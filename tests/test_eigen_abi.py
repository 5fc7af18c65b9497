"""The C ABI of the block-vector kernels: the prototypes of fdb_bv_dot and fdb_bv_mult compile against
include/fdb200.h with the argument types _lib declares, FDB_BV_MAX_COLUMNS equals _lib's constant, and the library
exports both symbols."""
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
/* the prototypes, checked by assignment to pointers of the exact types */
static int (*const dot)(size_t, int, const double *const *, int, const double *const *, double *) = fdb_bv_dot;
static int (*const mult)(size_t, int, double *const *, double, double, int, const double *const *, const double *) =
    fdb_bv_mult;
int main(void)
{
    printf("%d\n", (int)FDB_BV_MAX_COLUMNS);
    return dot == NULL || mult == NULL;
}
"""


def test_prototypes_and_max_columns_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "bv.c"
    src.write_text(PROGRAM)
    # compile only: the symbols live in libfdb200.so, which this check does not need
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                    str(tmp_path / "bv.o")], check=True)
    with open(os.path.join(ROOT, "include", "fdb200.h")) as f:
        assert "#define FDB_BV_MAX_COLUMNS 64" in f.read()
    assert _lib.BV_MAX_COLUMNS == 64


def test_signatures():
    S = _lib.SIGNATURES
    P, D = C.POINTER(C.c_void_p), C.POINTER(C.c_double)
    assert S["fdb_bv_dot"] == (C.c_int, [C.c_size_t, C.c_int, P, C.c_int, P, D])
    assert S["fdb_bv_mult"] == (C.c_int, [C.c_size_t, C.c_int, P, C.c_double, C.c_double, C.c_int, P, D])


def test_library_exports():
    lib = _lib.load()
    assert lib.fdb_bv_dot.argtypes == _lib.SIGNATURES["fdb_bv_dot"][1]
    assert lib.fdb_bv_mult.argtypes == _lib.SIGNATURES["fdb_bv_mult"][1]


def test_largest_block_fits_the_kernels():
    from firedrake_b200.eigensolver import MAX_BLOCKSIZE
    assert MAX_BLOCKSIZE == 21 and 3 * MAX_BLOCKSIZE <= _lib.BV_MAX_COLUMNS
