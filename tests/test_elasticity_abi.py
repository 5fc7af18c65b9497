"""The ctypes mirror of fdb_kernel_desc against the C header after the elasticity form: a small C program
compiled against include/fdb200.h prints sizeof, the offsets of the trailing fields (lmbda appended after
dcoef) and FDB_FORM_ELASTICITY, which must equal _lib's."""
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
    printf("%zu %zu %zu %zu %zu %zu %d\n", sizeof(fdb_kernel_desc), offsetof(fdb_kernel_desc, alpha),
           offsetof(fdb_kernel_desc, beta), offsetof(fdb_kernel_desc, affine_cells),
           offsetof(fdb_kernel_desc, dcoef), offsetof(fdb_kernel_desc, lmbda), (int)FDB_FORM_ELASTICITY);
    return 0;
}
"""


def test_kernel_desc_layout_with_lmbda_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    size, o_alpha, o_beta, o_aff, o_dcoef, o_lmbda, f6 = (int(v) for v in subprocess.run(
        [str(exe)], capture_output=True, text=True, check=True).stdout.split())
    K = _lib.KernelDesc
    assert C.sizeof(K) == size
    assert (K.alpha.offset, K.beta.offset, K.affine_cells.offset, K.dcoef.offset, K.lmbda.offset) == \
        (o_alpha, o_beta, o_aff, o_dcoef, o_lmbda)
    assert K.lmbda.offset == K.dcoef.offset + 3 * C.sizeof(C.c_double)
    assert K.lmbda.size == C.sizeof(C.c_double)
    assert _lib.FORM_ELASTICITY == f6 == 6
