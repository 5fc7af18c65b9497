"""The C ABI of the p-multigrid transfers and the fused Chebyshev step: the enum values from include/fdb200.h equal
_lib's constants, the descriptor layouts are unchanged, the header documents the tables, argument and map orders,
op2.Kernel gives the documented accesses, and the engine's form table has the rows, the per-row second-space degree
rule and a refusal naming the form for each case it does not cover."""
import ctypes
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
    printf("%d %d %d %zu %zu %zu %zu %zu\n", (int)FDB_FORM_P_PROLONG, (int)FDB_FORM_P_RESTRICT, (int)FDB_FORM_P_INJECT,
           sizeof(fdb_kernel_desc), offsetof(fdb_kernel_desc, lmbda), sizeof(fdb_space2_desc),
           offsetof(fdb_space2_desc, B), offsetof(fdb_space2_desc, offset));
    (void)sizeof(fdb_vec_chebyshev((size_t)0, 0.0, 0.0, (const double *)0, (const double *)0, (const double *)0,
                                   (double *)0, (double *)0));   /* the prototype, unevaluated */
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
    src = tmp_path / "pmg.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "pmg"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out[:3] == [_lib.FORM_P_PROLONG, _lib.FORM_P_RESTRICT, _lib.FORM_P_INJECT] == [17, 18, 19]
    assert out[3:] == [ctypes.sizeof(_lib.KernelDesc), _lib.KernelDesc.lmbda.offset, ctypes.sizeof(_lib.Space2Desc),
                       _lib.Space2Desc.B.offset, _lib.Space2Desc.offset.offset]
    assert "fdb_vec_chebyshev" in _lib.SIGNATURES


def test_argument_orders_are_documented():
    header = _read("include", "fdb200.h")
    m = re.search(r"FDB_FORM_P_PROLONG = 17,(.*?)\*/", header, re.S)
    doc = " ".join(m.group(1).split())
    for s in ("P (p+1, q+1), the coarse basis at the fine nodes: fdb_space2_desc.B",
              "R (q+1, p+1), the fine basis at the coarse nodes: fdb_kernel_desc.B, with nq = q+1",
              "P_PROLONG [fine WRITE, coarse] maps [fine map, coarse map]",
              "P_RESTRICT [coarse INC, fine, w] maps [coarse map, fine map]",
              "P_INJECT [coarse WRITE, fine] maps [coarse map, fine map]",
              "{(2, 1), (3, 1), (3, 2)}", "exact unit vectors", "Device mode only", "bit-reproducible"):
        assert s in doc, s
    assert re.search(r"fdb_vec_chebyshev\(size_t n, double c_d, double c_z, const double \*b, const double \*ax,\s+"
                     r"const double \*dinv,\s+double \*d, double \*x\)", header)


def test_kernel_accesses_and_names():
    R, I, W = op2.READ, op2.INC, op2.WRITE
    for form, acc in (("p_prolong", (W, R)), ("p_restrict", (I, R, R)), ("p_inject", (W, R))):
        k = op2.Kernel(form, degree=3, coarse_degree=1, cdim=3)
        assert k.accesses == acc and k.name == form and k.coarse_degree == 1
        assert op2._FORMS[form].transfer and op2._FORMS[form].enum == getattr(_lib, "FORM_" + form.upper())


def test_form_table_rows_and_refusals():
    engine = _read("firedrake_b200", "csrc", "global_kernel.cu")
    for form, name, extra in (("PROLONG", "p_prolong", "coarse"), ("RESTRICT", "p_restrict", "fine, w"),
                              ("INJECT", "p_inject", "fine")):
        assert re.search(r'\{FDB_FORM_P_%s, "%s", -1, false, nullptr, 0, false, LAUNCH_P_TRANSFER, \{3, 0, 0\}, 2, '
                         r'"%s",\s+FDB_INTEGRAL_CELL, SPACE2_COARSER\}' % (form, name, extra), engine)
    # the Stokes-specific degree check is now a property of the rows
    assert "enum { SPACE2_PRESSURE = 0, SPACE2_COARSER };" in engine
    assert "f->space2 && f->space2_degree == SPACE2_PRESSURE && s2->degree != d->degree - 1" in engine
    kernels = engine + _read("firedrake_b200", "csrc", "p_transfer_hex.cu")
    for msg in ("%s: degree pair (fine %d, coarse %d) not instantiated: (2, 1), ",      # other pairs
                "%s needs GLL elements: row %d of P (space2.B) must be the ",           # GL (DQ) element
                "%s needs GLL elements: row %d of R (desc.B) must be the ",
                "%s expects %d device args (%s, %s) and 2 maps (%s), got %d/%d",         # counts, host mode
                "%s needs hex cells (extruded or native), got cell %d",                  # triangles, quads
                "%s is a mixed form, a rank-1 action only",                              # rank 2, diagonal
                "p transfer: degree pair (%d, %d) not instantiated"):
        assert msg in kernels, msg
