"""The advection-diffusion form's enum value against the C header: a small C program compiled against
include/fdb200.h prints FDB_FORM_ADVECTION_DIFFUSION, sizeof(fdb_kernel_desc) and the offset of its last
field, which must equal _lib's constant and _lib.KernelDesc's layout (the form adds no field)."""
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
    printf("%d %zu %zu\n", (int)FDB_FORM_ADVECTION_DIFFUSION, sizeof(fdb_kernel_desc),
           offsetof(fdb_kernel_desc, lmbda));
    return 0;
}
"""


def test_advection_diffusion_enum_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "enum.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "enum"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    form, size, off_lmbda = (int(v) for v in subprocess.run(
        [str(exe)], capture_output=True, text=True, check=True).stdout.split())
    assert _lib.FORM_ADVECTION_DIFFUSION == form == 9
    assert C.sizeof(_lib.KernelDesc) == size
    assert _lib.KernelDesc.lmbda.offset == off_lmbda
