"""The C ABI of FDB_FORM_DG_TRANSPORT: the enum value from include/fdb200.h equals _lib's constant and the descriptor
keeps its layout; the header documents the argument orders and the coefficient slots, op2.Kernel gives the
documented accesses, names and descriptor fields, and the engine's form table has the row and a refusal naming the
form for each case it does not cover."""
import os
import re
import shutil
import subprocess

import pytest

from firedrake_b200 import _lib, op2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROGRAM = r"""
#include <stddef.h>
#include <stdio.h>
#include "fdb200.h"
int main(void)
{
    printf("%d %zu %zu %zu\n", (int)FDB_FORM_DG_TRANSPORT, offsetof(fdb_kernel_desc, dcoef),
           offsetof(fdb_kernel_desc, lmbda), sizeof(fdb_kernel_desc));
    return 0;
}
"""


def _read(*path):
    with open(os.path.join(ROOT, *path)) as f:
        return f.read()


def test_enum_and_layout_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "tr.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "tr"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    form, off_dcoef, off_lmbda, size = (int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True,
                                                                       check=True).stdout.split())
    assert form == _lib.FORM_DG_TRANSPORT == 16
    assert _lib.KernelDesc.dcoef.offset == off_dcoef
    assert _lib.KernelDesc.lmbda.offset == off_lmbda
    import ctypes
    assert ctypes.sizeof(_lib.KernelDesc) == size


def test_argument_orders_are_documented():
    m = re.search(r"FDB_FORM_DG_TRANSPORT = 16(.*?)\*/", _read("include", "fdb200.h"), re.S)
    doc = " ".join(m.group(1).split())
    for s in ("cell action [y INC, coords, u, b]", "diagonal [d INC, coords, b]",
              "facets action [y INC, coords, u, b, facets]", "diagonal [d INC, coords, b, facets]",
              "c_out = dcoef[0], c_in = dcoef[1]", "read through maps[1]", "B must be the identity",
              "there is no assembled DG matrix", "Device mode only"):
        assert s in doc, s
    assert "FDB_FORM_DG_TRANSPORT (exterior facets): c_out = dcoef[0], c_in = dcoef[1]" in _read("include", "fdb200.h")


def test_kernel_accesses_names_and_descriptor():
    from firedrake_b200.fiat_lite import interval_element
    el = interval_element(2, variant="gl")
    R, I = op2.READ, op2.INC
    cases = {("cell", False): (I, R, R, R), ("cell", True): (I, R, R),
             ("interior_facet", False): (I, R, R, R, R), ("interior_facet", True): (I, R, R, R),
             ("exterior_facet", False): (I, R, R, R, R), ("exterior_facet", True): (I, R, R, R)}
    for (integral, diag), acc in cases.items():
        k = op2.Kernel("dg_transport", degree=2, integral=integral, diagonal=diag, element=el)
        assert k.accesses == acc and k.name == f"form0_{integral}_integral"
    assert op2._FORMS["dg_transport"].enum == _lib.FORM_DG_TRANSPORT
    assert op2._FORMS["dg_transport"].facet and op2._FORMS["dg_transport"].velocity
    k = op2.Kernel("dg_transport", degree=2, integral="exterior_facet", element=el, c_out=0.0, c_in=-1.0)
    assert (k.c_out, k.c_in) == (0.0, -1.0)
    assert (op2.Kernel("dg_transport", degree=1).c_out, op2.Kernel("dg_transport", degree=1).c_in) == (1.0, 0.0)


def test_form_table_row_and_refusals():
    engine = _read("firedrake_b200", "csrc", "global_kernel.cu")
    assert re.search(r'\{FDB_FORM_DG_TRANSPORT, "dg_transport", 1, false, "b", 3, false, LAUNCH_DG_TRANSPORT, '
                     r'\{4, 0, 4\}, 1, nullptr, -1\}', engine)
    kernels = engine + _read("firedrake_b200", "csrc", "dg_transport_hex.cu") + \
        _read("firedrake_b200", "csrc", "dg_facet_hex.cu")
    for msg in ("%s has no rank-2 form: there is no assembled DG matrix",      # rank 2
                "degree %d outside %d..%d",                                      # degree
                "%s %s takes %s (cdim %d)",                                      # cdim (scalar spaces only)
                "%s needs nq == degree+1 Gauss points per axis",                 # nq
                "%s needs the collocated Gauss-Legendre element (B must be the ",
                "%s takes device-resident Dats only",                            # host location
                "%s takes a cell, exterior-facet or interior-facet integral",
                "dg transport cell kernel: degree %d not instantiated (1..4)",
                "dg upwind kernel: degree %d not instantiated (1..4)"):
        assert msg in kernels, msg
    # the rank-2 refusal applies to the transport launcher and comes before the degree check
    assert "f->launcher == LAUNCH_DG_TRANSPORT) && mode == MODE_MATRIX" in engine
    assert engine.index("no assembled DG matrix") < engine.index("degree %d outside %d..%d")
