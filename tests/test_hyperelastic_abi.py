"""The hyperelastic forms in the C ABI: a small C program compiled against include/fdb200.h prints
FDB_FORM_HYPERELASTICITY[_JACOBIAN] and the layout of fdb_kernel_desc, which the forms leave unchanged
(mu in alpha, lmbda and beta in their existing fields); _lib's values and ctypes mirror must match."""
import ctypes as C
import os
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
    printf("%zu %zu %zu %zu %zu %d %d\n", sizeof(fdb_kernel_desc), offsetof(fdb_kernel_desc, alpha),
           offsetof(fdb_kernel_desc, beta), offsetof(fdb_kernel_desc, dcoef), offsetof(fdb_kernel_desc, lmbda),
           (int)FDB_FORM_HYPERELASTICITY, (int)FDB_FORM_HYPERELASTICITY_JACOBIAN);
    return 0;
}
"""


def test_hyperelastic_forms_and_unchanged_desc_layout_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    size, o_alpha, o_beta, o_dcoef, o_lmbda, f7, f8 = (int(v) for v in subprocess.run(
        [str(exe)], capture_output=True, text=True, check=True).stdout.split())
    K = _lib.KernelDesc
    assert C.sizeof(K) == size
    assert (K.alpha.offset, K.beta.offset, K.dcoef.offset, K.lmbda.offset) == (o_alpha, o_beta, o_dcoef, o_lmbda)
    # lmbda is still the last field: the hyperelastic forms added none
    assert K._fields_[-1][0] == "lmbda" and size == o_lmbda + C.sizeof(C.c_double)
    assert _lib.FORM_HYPERELASTICITY == f7 == 7
    assert _lib.FORM_HYPERELASTICITY_JACOBIAN == f8 == 8
