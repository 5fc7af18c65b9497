"""The ctypes mirror of fdb_kernel_desc against the C header: a small C program compiled against
include/fdb200.h prints sizeof and the offsets of the fields around the nonlinear diffusion
coefficients (dcoef, appended after affine_cells), which must equal _lib.KernelDesc's."""
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
    printf("%zu %zu %zu %zu %d %d\n", sizeof(fdb_kernel_desc), offsetof(fdb_kernel_desc, diagonal),
           offsetof(fdb_kernel_desc, affine_cells), offsetof(fdb_kernel_desc, dcoef),
           (int)FDB_FORM_NONLINEAR_DIFFUSION, (int)FDB_FORM_NONLINEAR_DIFFUSION_JACOBIAN);
    return 0;
}
"""


def test_kernel_desc_layout_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    size, off_diag, off_aff, off_dcoef, f4, f5 = (int(v) for v in subprocess.run(
        [str(exe)], capture_output=True, text=True, check=True).stdout.split())
    K = _lib.KernelDesc
    assert C.sizeof(K) == size
    assert (K.diagonal.offset, K.affine_cells.offset, K.dcoef.offset) == (off_diag, off_aff, off_dcoef)
    assert K.dcoef.size == 3 * C.sizeof(C.c_double)
    assert (_lib.FORM_NONLINEAR_DIFFUSION, _lib.FORM_NONLINEAR_DIFFUSION_JACOBIAN) == (f4, f5) == (4, 5)
