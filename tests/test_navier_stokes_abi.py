"""The Navier-Stokes forms' C ABI: a small C program compiled against include/fdb200.h prints
FDB_FORM_NAVIER_STOKES[_JACOBIAN] and the descriptor layouts, which must equal _lib's constants and ctypes
mirrors (fdb_kernel_desc and fdb_space2_desc keep their layouts), and the header and the engine document the
Jacobian's argument order, the second space's arguments before the trailing u."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from firedrake_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROGRAM = r"""
#include <stddef.h>
#include <stdio.h>
#include "fdb200.h"
int main(void)
{
    printf("%d %d %d %zu %zu %zu %zu %zu %zu\n", (int)FDB_FORM_STOKES, (int)FDB_FORM_NAVIER_STOKES,
           (int)FDB_FORM_NAVIER_STOKES_JACOBIAN, sizeof(fdb_kernel_desc), offsetof(fdb_kernel_desc, lmbda),
           sizeof(fdb_space2_desc), offsetof(fdb_space2_desc, degree), offsetof(fdb_space2_desc, B),
           offsetof(fdb_space2_desc, offset));
    return 0;
}
"""


def test_navier_stokes_enums_and_descriptors_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "ns.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "ns"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    stokes, ns, nsj, size, off_lmbda, size2, off_deg, off_b, off_off = out
    assert (_lib.FORM_STOKES, _lib.FORM_NAVIER_STOKES, _lib.FORM_NAVIER_STOKES_JACOBIAN) == (stokes, ns, nsj) == \
        (10, 11, 12)
    K, S = _lib.KernelDesc, _lib.Space2Desc
    assert C.sizeof(K) == size and K._fields_[-1][0] == "lmbda" and size == off_lmbda + C.sizeof(C.c_double)
    assert C.sizeof(S) == size2
    assert (S.degree.offset, S.B.offset, S.offset.offset) == (off_deg, off_b, off_off)


def test_argument_order_is_documented():
    """The header gives the Jacobian's action arguments with u last, after the pressure pair, and the engine's
    comment at its argument check states the same order for a form with a second space and a coefficient."""
    with open(os.path.join(ROOT, "include", "fdb200.h")) as f:
        header = f.read()
    assert re.search(r"FDB_FORM_NAVIER_STOKES_JACOBIAN = 12.*?action\s+\[y_u INC, coords, w, y_p INC, r, u\]", header,
                     re.S)
    assert re.search(r"FDB_FORM_NAVIER_STOKES = 11.*?action\s+\[y_u INC, coords, u, y_p INC, p\]", header, re.S)
    with open(os.path.join(ROOT, "firedrake_b200", "csrc", "global_kernel.cu")) as f:
        engine = f.read()
    assert "[y, coords, x, y2, x2, coef]" in engine
    from firedrake_b200 import op2
    assert "(velocity output, coordinates, w, pressure output, r, u)" in " ".join(op2.Kernel.__doc__.split())
