"""The C ABI of the vertex-star relaxation: the prototypes of fdb_fdm_star_* compile against include/fdb200.h with
the argument types _lib declares, and the library exports them."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from firedrake_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROGRAM = r"""
#include <stddef.h>
#include "fdb200.h"
static int (*const create)(int, int, int, const fdb_int *, const fdb_int *, fdb_int, int, const fdb_int *, int,
                           const fdb_int *, const fdb_int *, const fdb_int *, const long long *, int, const double *,
                           fdb_fdm_star_t *) = fdb_fdm_star_create;
static int (*const update)(fdb_fdm_star_t, double, double, const double *) = fdb_fdm_star_update;
static int (*const apply)(fdb_fdm_star_t, const double *, double *) = fdb_fdm_star_apply;
static int (*const destroy)(fdb_fdm_star_t) = fdb_fdm_star_destroy;
int main(void) { return create == NULL || update == NULL || apply == NULL || destroy == NULL; }
"""

NAMES = ("fdb_fdm_star_create", "fdb_fdm_star_update", "fdb_fdm_star_apply", "fdb_fdm_star_destroy")


def test_prototypes_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "fdm.c"
    src.write_text(PROGRAM)
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                    str(tmp_path / "fdm.o")], check=True)


def test_signatures():
    S, V, I = _lib.SIGNATURES, C.c_void_p, C.c_int
    assert S["fdb_fdm_star_create"] == (I, [I, I, I, V, V, C.c_int32, I, V, I, V, V, V, V, I, V, C.POINTER(V)])
    assert S["fdb_fdm_star_update"] == (I, [V, C.c_double, C.c_double, V])
    assert S["fdb_fdm_star_apply"] == (I, [V, V, V])
    assert S["fdb_fdm_star_destroy"] == (I, [V])


def test_library_exports():
    lib = _lib.load()
    for n in NAMES:
        assert getattr(lib, n).argtypes == _lib.SIGNATURES[n][1]
