"""The Boussinesq forms' C ABI: a small C program compiled against include/fdb200.h prints
FDB_FORM_BOUSSINESQ[_JACOBIAN] and the descriptor layouts, which must equal _lib's constants and ctypes mirrors
(fdb_kernel_desc and fdb_space2_desc keep their layouts); the header, the engine's form table and op2.Kernel
document the argument lists; and the engine's existing argument-count message is unchanged for the forms without
a third field."""
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
    printf("%d %d %d %zu %zu %zu %zu %zu\n", (int)FDB_FORM_MIXED_POISSON_SCHUR, (int)FDB_FORM_BOUSSINESQ,
           (int)FDB_FORM_BOUSSINESQ_JACOBIAN, sizeof(fdb_kernel_desc), offsetof(fdb_kernel_desc, dcoef),
           offsetof(fdb_kernel_desc, lmbda), sizeof(fdb_space2_desc), offsetof(fdb_space2_desc, offset));
    return 0;
}
"""


def test_boussinesq_enums_and_descriptors_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "rb.c"
    src.write_text(PROGRAM)
    exe = tmp_path / "rb"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    schur, rb, rbj, size, off_dcoef, off_lmbda, size2, off_off = out
    assert (_lib.FORM_MIXED_POISSON_SCHUR, _lib.FORM_BOUSSINESQ, _lib.FORM_BOUSSINESQ_JACOBIAN) == (schur, rb, rbj) \
        == (23, 24, 25)
    K, S = _lib.KernelDesc, _lib.Space2Desc
    assert C.sizeof(K) == size and K.dcoef.offset == off_dcoef and K.lmbda.offset == off_lmbda
    assert K._fields_[-1][0] == "lmbda" and size == off_lmbda + C.sizeof(C.c_double)
    assert C.sizeof(S) == size2 and S.offset.offset == off_off


def test_argument_lists_are_documented():
    with open(os.path.join(ROOT, "include", "fdb200.h")) as f:
        header = f.read()
    assert re.search(r"FDB_FORM_BOUSSINESQ = 24.*?action\s+\[y_u INC, coords, u, y_p INC, p, y_T INC, T\]\s+"
                     r"maps \[V map, coord map, Q map\]", header, re.S)
    assert re.search(r"FDB_FORM_BOUSSINESQ_JACOBIAN = 25.*?action\s+\[y_u INC, coords, w, y_p INC, r, y_T INC, s, "
                     r"u0, T0\]\s+maps \[V map, coord map, Q map\]", header, re.S)
    assert re.search(r"FDB_FORM_BOUSSINESQ\[_JACOBIAN\]: the buoyancy vector \(Ra/Pr\) g = dcoef\[0\.\.2\]", header)
    assert re.search(r"FDB_FORM_BOUSSINESQ\[_JACOBIAN\]: the temperature diffusivity 1/Pr", header)
    with open(os.path.join(ROOT, "firedrake_b200", "csrc", "global_kernel.cu")) as f:
        engine = f.read()
    assert '"boussinesq", 3, false, nullptr, 0, true, LAUNCH_STOKES' in engine
    assert '"boussinesq_jacobian", 3, false, "u0, T0", 3, false, LAUNCH_STOKES' in engine
    # the argument-count message prints the third field between the second space's arguments and the coefficients;
    # both are empty strings for every form without them
    assert ('"fdb_kernel_call: %s %s expects %d %sargs (%s%s%s%s%s%s%s) and %d maps, got %d/%d"' in
            " ".join(engine.split()))
    from firedrake_b200 import op2
    doc = " ".join(op2.Kernel.__doc__.split())
    assert "(velocity output, coordinates, w, pressure output, r, temperature output, s, u0, T0)" in doc
    k = op2.Kernel("boussinesq_jacobian", degree=2, bg=(0, 0, -3), kt=0.5)
    assert k.accesses == (op2.INC, op2.READ, op2.READ, op2.INC, op2.READ, op2.INC, op2.READ, op2.READ, op2.READ)
    assert op2.Kernel("boussinesq", degree=3).accesses == (op2.INC, op2.READ, op2.READ, op2.INC, op2.READ, op2.INC,
                                                          op2.READ)
    with pytest.raises(ValueError, match="three values"):
        op2.Kernel("boussinesq", degree=2, bg=(0, 1))
