"""The GTMG trace transfers' C ABI: a small C program compiled against include/fdb200.h prints
FDB_FORM_TRACE_PROLONG / _RESTRICT, which must equal _lib's constants; the header, the engine's form table and
op2.Kernel document them; and op2.Kernel gives the transfers their access descriptors.  The creation refusals run on
the device (tests/test_gtmg_gpu.py::test_creation_and_call_refusals)."""
import os
import shutil
import subprocess

import pytest

from firedrake_b200 import _lib, op2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROGRAM = r"""
#include <stdio.h>
#include "fdb200.h"
int main(void)
{
    printf("%d %d\n", (int)FDB_FORM_TRACE_PROLONG, (int)FDB_FORM_TRACE_RESTRICT);
    return 0;
}
"""


def test_trace_transfer_enums_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "tt.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "tt"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [_lib.FORM_TRACE_PROLONG, _lib.FORM_TRACE_RESTRICT] == [28, 29]


def test_forms_are_documented_and_described():
    with open(os.path.join(ROOT, "include", "fdb200.h")) as f:
        header = f.read()
    with open(os.path.join(ROOT, "firedrake_b200", "csrc", "global_kernel.cu")) as f:
        table = f.read()
    for name in ("TRACE_PROLONG", "TRACE_RESTRICT"):
        assert f"FDB_FORM_{name}" in header and f"FDB_FORM_{name}" in table
    assert "[lambda WRITE, c]" in header and "[c INC, lambda, w]" in header
    p = op2.Kernel("trace_prolong", degree=1, coarse_degree=1)
    r = op2.Kernel("trace_restrict", degree=2, coarse_degree=1)
    assert p.accesses == (op2.WRITE, op2.READ) and r.accesses == (op2.INC, op2.READ, op2.READ)
    assert "trace_prolong" in op2.Kernel.__doc__
    t = op2.trace_transfer_table(3)
    assert t.shape == (3, 2) and abs(t.sum(axis=1) - 1.0).max() < 1e-15
