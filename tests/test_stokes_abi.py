"""The Stokes form's C ABI: a small C program compiled against include/fdb200.h fills an fdb_space2_desc (the
pressure space passed to fdb_kernel_create_mixed) and prints FDB_FORM_STOKES, the descriptor sizes and the
second-space descriptor's field offsets, which must equal _lib's constant and ctypes mirrors.
fdb_kernel_desc keeps its layout: lmbda is still its last field."""
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
#include <string.h>
#include "fdb200.h"
int main(void)
{
    static const fdb_int off2[8] = {1, 1, 1, 1, 1, 1, 1, 1};
    fdb_space2_desc s;
    memset(&s, 0, sizeof(s));
    s.degree = 1;
    for (int q = 0; q < 3; q++)
        for (int a = 0; a < 2; a++) s.B[q * 2 + a] = q + 0.5 * a;
    s.offset = off2;
    printf("%d %zu %zu %zu %zu %zu %zu %g %d\n", (int)FDB_FORM_STOKES, sizeof(fdb_kernel_desc),
           offsetof(fdb_kernel_desc, lmbda), sizeof(fdb_space2_desc), offsetof(fdb_space2_desc, degree),
           offsetof(fdb_space2_desc, B), offsetof(fdb_space2_desc, offset), s.B[5], s.offset[7]);
    return 0;
}
"""

# compiled only (not linked): the entry point's prototype
PROTOTYPE = r"""
#include "fdb200.h"
int (*create)(const fdb_kernel_desc *, const fdb_space2_desc *, fdb_kernel_t *) = fdb_kernel_create_mixed;
"""


def test_stokes_descriptors_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "stokes.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "stokes"
    proto = tmp_path / "proto.c"
    proto.write_text(PROTOTYPE)
    subprocess.run([cc, "-std=c99", "-c", "-I", os.path.join(ROOT, "include"), str(proto), "-o",
                    str(tmp_path / "proto.o")], check=True)
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    form, size, off_lmbda, size2, off_deg, off_b, off_off = (int(v) for v in out[:7])
    assert float(out[7]) == 2.5 and int(out[8]) == 1
    assert _lib.FORM_STOKES == form == 10
    K, S = _lib.KernelDesc, _lib.Space2Desc
    assert C.sizeof(K) == size and K._fields_[-1][0] == "lmbda" and size == off_lmbda + C.sizeof(C.c_double)
    assert C.sizeof(S) == size2
    assert (S.degree.offset, S.B.offset, S.offset.offset) == (off_deg, off_b, off_off)
