"""The boundary mass form's C ABI: a small C program compiled against include/fdb200.h prints
FDB_FORM_BOUNDARY_MASS and the descriptor layouts, which must equal _lib's constants and ctypes mirrors
(fdb_kernel_desc, fdb_space2_desc and fdb_call_args keep their layouts); the header documents the argument
order with the facet numbers last, and the engine's form table gives the form its exterior-facet row and a
refusal naming it for each case it does not cover."""
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
    printf("%d %d %zu %zu %zu %zu %zu\n", (int)FDB_FORM_BOUNDARY_MASS, (int)FDB_INTEGRAL_EXTERIOR_FACET,
           sizeof(fdb_kernel_desc), offsetof(fdb_kernel_desc, lmbda), sizeof(fdb_space2_desc),
           sizeof(fdb_call_args), offsetof(fdb_call_args, layers_version));
    return 0;
}
"""


def test_boundary_mass_enum_and_descriptors_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "bm.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "bm"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    form, integral, size, off_lmbda, size2, size_call, off_lv = (
        int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    assert form == _lib.FORM_BOUNDARY_MASS == 13
    assert integral == _lib.INTEGRAL_EXTERIOR_FACET == 1
    assert C.sizeof(_lib.KernelDesc) == size and size == off_lmbda + C.sizeof(C.c_double)
    assert C.sizeof(_lib.Space2Desc) == size2
    assert C.sizeof(_lib.CallArgs) == size_call and _lib.CallArgs.layers_version.offset == off_lv


def test_argument_order_is_documented():
    with open(os.path.join(ROOT, "include", "fdb200.h")) as f:
        header = f.read()
    m = re.search(r"FDB_FORM_BOUNDARY_MASS = 13(.*?)\*/", header, re.S)
    assert m
    doc = " ".join(m.group(1).split())
    for args in ("action [y INC, coords, u, facet]", "diagonal [d INC, coords, facet]", "rank 2 [Mat, coords, facet]"):
        assert args in doc
    from firedrake_b200 import op2
    k = op2.Kernel("boundary_mass", degree=2, integral="exterior_facet")
    assert k.accesses == (op2.INC, op2.READ, op2.READ, op2.READ) and k.name == "form0_exterior_facet_integral"
    k2 = op2.Kernel("boundary_mass", degree=2, rank=2, cdim=3, integral="exterior_facet")
    assert k2.accesses == (op2.INC, op2.READ, op2.READ) and k2.name == "form00_exterior_facet_integral"
    assert op2.Kernel("boundary_mass", degree=2, diagonal=True, integral="exterior_facet").accesses == \
        (op2.INC, op2.READ, op2.READ)


def test_engine_refusals_name_the_form():
    """Every refusal of the form is in the engine with the form's name; the existing rows keep their cell-only
    message."""
    with open(os.path.join(ROOT, "firedrake_b200", "csrc", "global_kernel.cu")) as f:
        engine = f.read()
    assert re.search(r'\{FDB_FORM_BOUNDARY_MASS, "boundary_mass", -1, .*?\{5, 4, 5\}, 1, nullptr,\s*'
                     r'FDB_INTEGRAL_EXTERIOR_FACET\}', engine, re.S)
    assert engine.count("FDB_INTEGRAL_CELL},") == 11
    for msg in ("%s has cell integrals only", "%s has exterior-facet integrals only",
                "interior facets are not supported", "takes a scalar space or a vector space of value size 3",
                "%s on extruded cells needs the layer offsets", "%s takes device-resident Dats only"):
        assert msg in engine, msg
