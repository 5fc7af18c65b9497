"""The C ABI of the spectral-element wave equation: the enum values of FDB_FORM_SPECTRAL_HELMHOLTZ[_COEF] from
include/fdb200.h equal _lib's constants, the prototypes of fdb_vec_leapfrog, fdb_point_eval and fdb_point_load
compile against the header with the argument types _lib declares, op2.Kernel gives the documented accesses and the
GLL tables, and the engine's form table has the rows."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from firedrake_b200 import _lib, op2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROGRAM = r"""
#include <stddef.h>
#include <stdio.h>
#include "fdb200.h"
/* the prototypes, checked by assignment to pointers of the exact types */
static int (*const leapfrog)(size_t, double, const double *, const double *, const double *, double *) =
    fdb_vec_leapfrog;
static int (*const eval)(fdb_int, int, const fdb_int *, const double *, const double *, double *) = fdb_point_eval;
static int (*const load)(fdb_int, int, const fdb_int *, const double *, const double *, double, double *) =
    fdb_point_load;
int main(void)
{
    printf("%d %d %d\n", (int)FDB_FORM_SPECTRAL_HELMHOLTZ, (int)FDB_FORM_SPECTRAL_HELMHOLTZ_COEF,
           (int)FDB_FORM_P_INJECT);
    return leapfrog == NULL || eval == NULL || load == NULL;
}
"""


def _read(*path):
    with open(os.path.join(ROOT, *path)) as f:
        return f.read()


def test_enum_and_prototypes_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "sem.c"
    src.write_text(PROGRAM)
    obj = tmp_path / "sem.o"
    # compile only: the symbols live in libfdb200.so, which this check does not need
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                    str(obj)], check=True)
    assert _lib.FORM_SPECTRAL_HELMHOLTZ == 20 and _lib.FORM_SPECTRAL_HELMHOLTZ_COEF == 21
    header = _read("include", "fdb200.h")
    assert "FDB_FORM_SPECTRAL_HELMHOLTZ = 20," in header and "FDB_FORM_SPECTRAL_HELMHOLTZ_COEF = 21" in header


def test_signatures():
    S = _lib.SIGNATURES
    assert S["fdb_vec_leapfrog"] == (C.c_int, [C.c_size_t, C.c_double] + [C.c_void_p] * 4)
    assert S["fdb_point_eval"] == (C.c_int, [C.c_int32, C.c_int] + [C.c_void_p] * 4)
    assert S["fdb_point_load"] == (C.c_int, [C.c_int32, C.c_int] + [C.c_void_p] * 3 + [C.c_double, C.c_void_p])


def test_kernel_accesses_and_tables():
    INC, READ = op2.INC, op2.READ
    assert op2.Kernel("spectral_helmholtz", degree=3).accesses == (INC, READ, READ)
    assert op2.Kernel("spectral_helmholtz", degree=3, diagonal=True).accesses == (INC, READ)
    assert op2.Kernel("spectral_helmholtz_coef", degree=3).accesses == (INC, READ, READ, READ)
    assert op2.Kernel("spectral_helmholtz_coef", degree=3, diagonal=True).accesses == (INC, READ, READ)
    assert op2._FORMS["spectral_helmholtz"].enum == 20 and op2._FORMS["spectral_helmholtz_coef"].coefficient
    src = _read("firedrake_b200", "csrc", "global_kernel.cu")
    for name in ("spectral_helmholtz", "spectral_helmholtz_coef"):
        assert f'"{name}"' in src
    assert "no assembled SEM matrix" in src


def test_descriptor_gets_gll_tables():
    """GlobalKernel.compile fills the GLL rule in dof order for the spectral forms by default (B = I, xq = nodes)."""
    import numpy as np
    from firedrake_b200.fiat_lite import interval_element
    seen = {}

    class Fake:
        def fdb_kernel_create(self, d, h):
            seen["d"] = _lib.KernelDesc.from_buffer_copy(d._obj)        # byref(desc): copy it while it lives
            return 0

    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    saved = _lib.lib
    _lib.lib = lambda: Fake()
    try:
        mesh = ExtrudedHexMesh(2, 2, 2)
        W = mesh.function_space(4)
        m0 = op2.Map(op2.ExtrudedSet(op2.Set(4), 3), op2.Set(W.node_count), W.arity, W.cell_node_map,
                     offset=W.offset)
        m1 = op2.Map(op2.ExtrudedSet(op2.Set(4), 3), op2.Set(mesh.coord_space.node_count), 8, mesh.coord_map,
                     offset=mesh.coord_offset)
        op2.GlobalKernel(op2.Kernel("spectral_helmholtz", degree=4), [m0, m1], extruded=True).compile()
    finally:
        _lib.lib = saved
    d, el = seen["d"], interval_element(4, quadrature="gll")
    assert d.form == 20 and d.nq == 5
    assert np.array_equal(np.array(d.B[:25]).reshape(5, 5), np.eye(5))
    assert np.array_equal(np.array(d.xq[:5]), el.xq) and np.array_equal(np.array(d.wq[:5]), el.wq)
