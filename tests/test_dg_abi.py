"""The C ABI of the DG facet forms: a small C program compiled against include/fdb200.h prints
FDB_FORM_INTERIOR_PENALTY and FDB_FORM_DG_BOUNDARY, which must equal _lib's constants (the descriptor keeps its
layout); the header documents the argument orders and the coefficient slots, op2.Kernel gives the documented
accesses and names, and the engine's form table has the two rows and a refusal naming the form for each case it
does not cover."""
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
    printf("%d %d %d %zu\n", (int)FDB_FORM_INTERIOR_PENALTY, (int)FDB_FORM_DG_BOUNDARY,
           (int)FDB_INTEGRAL_INTERIOR_FACET, offsetof(fdb_kernel_desc, lmbda));
    return 0;
}
"""


def test_enums_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "dg.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "dg"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    ip, db, integral, off_lmbda = (int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True,
                                                                  check=True).stdout.split())
    assert ip == _lib.FORM_INTERIOR_PENALTY == 14
    assert db == _lib.FORM_DG_BOUNDARY == 15
    assert integral == _lib.INTEGRAL_INTERIOR_FACET == 2
    assert _lib.KernelDesc.lmbda.offset == off_lmbda


def _doc(header, form):
    m = re.search(form + r" = \d+,?(.*?)\*/", header, re.S)
    assert m, form
    return " ".join(m.group(1).split())


def test_argument_orders_are_documented():
    with open(os.path.join(ROOT, "include", "fdb200.h")) as f:
        header = f.read()
    ip = _doc(header, "FDB_FORM_INTERIOR_PENALTY")
    for s in ("action [y INC, coords, u, facets]", "diagonal [d INC, coords, facets]", "alpha = alpha, eta = beta",
              "arity 2*(degree+1)^3", "no assembled DG matrix"):
        assert s in ip, s
    db = _doc(header, "FDB_FORM_DG_BOUNDARY")
    for s in ("action [y INC, coords, u, facet]", "diagonal [d INC, coords, facet]",
              "c_f = alpha, c_p = beta, c_m = dcoef[0], c_s = dcoef[1]", "(0, alpha*eta, alpha, alpha)",
              "(0, alpha*eta, alpha, 0)", "(1, 0, 0, 0)"):
        assert s in db, s


def test_kernel_accesses_and_names():
    k = op2.Kernel("interior_penalty", degree=2, beta=27.0, integral="interior_facet")
    assert k.accesses == (op2.INC, op2.READ, op2.READ, op2.READ) and k.name == "form0_interior_facet_integral"
    kd = op2.Kernel("interior_penalty", degree=2, diagonal=True, integral="interior_facet")
    assert kd.accesses == (op2.INC, op2.READ, op2.READ)
    kb = op2.Kernel("dg_boundary", degree=3, c_m=1.0, integral="exterior_facet")
    assert kb.accesses == (op2.INC, op2.READ, op2.READ, op2.READ) and kb.name == "form0_exterior_facet_integral"
    # the element does not take part in equality: a CG and a DQ kernel of one degree compare equal, so nothing may
    # be keyed on a Kernel alone
    from firedrake_b200.fiat_lite import interval_element
    assert op2.Kernel("helmholtz", degree=2, element=interval_element(2, variant="gl")) == \
        op2.Kernel("helmholtz", degree=2)


def test_form_table_rows_and_refusals():
    with open(os.path.join(ROOT, "firedrake_b200", "csrc", "global_kernel.cu")) as f:
        engine = f.read()
    assert re.search(r'\{FDB_FORM_INTERIOR_PENALTY, "interior_penalty", 1, false, "facets", 1, false, '
                     r'LAUNCH_DG_FACET, \{4, 0, 4\}, 1,\s*nullptr, FDB_INTEGRAL_INTERIOR_FACET\}', engine)
    assert re.search(r'\{FDB_FORM_DG_BOUNDARY, "dg_boundary", 1, false, "facet", 1, false, LAUNCH_DG_FACET, '
                     r'\{4, 0, 4\}, 1, nullptr,\s*FDB_INTEGRAL_EXTERIOR_FACET\}', engine)
    for msg in ("%s has no rank-2 form: there is no assembled DG matrix", "%s has interior-facet integrals only",
                "%s has exterior-facet integrals only", "interior facets are not supported",
                "%s on extruded cells needs the layer offsets", "%s takes device-resident Dats only",
                "dg facet kernel: degree %d not instantiated (1..4)"):
        assert msg in engine or msg in open(os.path.join(ROOT, "firedrake_b200", "csrc", "dg_facet_hex.cu")).read(), \
            msg
    # the rank-2 refusal comes before the degree check, whose range would read 1..0
    assert engine.index("no assembled DG matrix") < engine.index("degree %d outside %d..%d")
