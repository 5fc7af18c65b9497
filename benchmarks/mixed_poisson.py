#!/usr/bin/env python
"""Speed of mixed Poisson on NCF_k x DQ_{k-1} hexahedra on one GPU, on a warped extruded mesh with device-resident
vectors:

* ``action``   -- the fused hand-written action (FDB_FORM_MIXED_POISSON, csrc/hdiv_hex.cu);
* ``generic``  -- ``mixed_poisson_kernel`` through the generic wrapper builder with MixedDat arguments;
* ``schur``    -- the selfp Schur complement S_p = B W B^T (FDB_FORM_MIXED_POISSON_SCHUR): its action (two passes
                  and the zeroing of the NCF scratch) and its diagonal.

One JSON line per (degree, n): ms per call (CUDA events over ``--steps`` calls after ``--warmup``), DoF/s of the
action counting flux plus DQ dofs, and the max-norm difference between the hand-written and generic actions
relative to max|y|.  Then one line per mesh size of the unit-cube solve (u = sin sin sin, natural u = 0, k = 2,
GMRES with the "full" selfp fieldsplit and inner Jacobi-CG, rtol 1e-8) with iterations and seconds.  FGMRES(30)
keeps about 61 MixedDats, which bounds the solve sizes.  Every line carries the card's name and power limit,
read in the same run.

    python benchmarks/mixed_poisson.py                        # the cases of DESIGN.md section 4.21
    python benchmarks/mixed_poisson.py --cases 2:16 --steps 3 --solve 8
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from firedrake_b200 import _lib                                                     # noqa: E402
from firedrake_b200.assemble import (FunctionSpace, MixedPoisson, MixedPoissonMatrixContext,  # noqa: E402
                                     MixedPoissonSchur, StokesAssembler, assemble, mass, solve)
from firedrake_b200.utility_meshes import ExtrudedHexMesh                           # noqa: E402

from coefficient_action import card, timed                                        # noqa: E402

SOLVER = {"ksp_type": "gmres", "ksp_rtol": 1e-8, "pc_type": "fieldsplit", "pc_fieldsplit_type": "schur",
          "pc_fieldsplit_schur_fact_type": "full", "pc_fieldsplit_schur_precondition": "selfp",
          "fieldsplit_0_ksp_type": "preonly", "fieldsplit_0_pc_type": "jacobi", "fieldsplit_1_ksp_type": "cg",
          "fieldsplit_1_pc_type": "jacobi", "fieldsplit_1_ksp_rtol": 1e-5}


def case(L, k, n, a, info):
    from firedrake_b200.assemble import assemble_mixed_poisson_generic
    mesh = ExtrudedHexMesh(n, n, n, warp=0.05)
    S, Q = FunctionSpace(mesh, k, family="NCF"), FunctionSpace(mesh, k - 1, family="DQ")
    F = MixedPoisson(S, Q, 1.0)
    rng = np.random.default_rng(0)
    up = F.dat(rng.standard_normal(S.node_count), rng.standard_normal(Q.node_count))
    y1, y2 = F.dat(), F.dat()
    asm = StokesAssembler(F, up)
    asm.assemble(y1)
    loop = asm._loop
    ms_action = timed(L, loop, a.warmup, a.steps)
    asm.assemble(y1)
    t0 = time.perf_counter()
    assemble_mixed_poisson_generic(F, up, y2)
    _lib.check(L.fdb_synchronize())
    ms_generic = None
    if not a.no_generic:
        ms_generic = timed(L, lambda: assemble_mixed_poisson_generic(F, up, y2), 1, max(1, a.steps // 5))
    diff = max(np.abs(p.data_ro - q.data_ro).max() for p, q in zip(y1, y2)) / max(np.abs(p.data_ro).max()
                                                                               for p in y1)
    Sp = MixedPoissonSchur(F, MixedPoissonMatrixContext(F).getDiagonal())
    x, z = Q.dat(rng.standard_normal(Q.node_count)), Q.dat()
    ms_sp = timed(L, lambda: Sp.mult(x, z), a.warmup, a.steps)
    ms_spd = timed(L, lambda: Sp.getDiagonal(z), a.warmup, a.steps)
    ndof = S.node_count + Q.node_count
    print(json.dumps({"k": k, "n": n, "flux_dofs": S.node_count, "dq_dofs": Q.node_count,
                      "action_ms": ms_action, "action_dofs_per_s": ndof / (ms_action * 1e-3),
                      "generic_ms": ms_generic, "generic_first_call_s": time.perf_counter() - t0,
                      "max_rel_diff": diff, "schur_action_ms": ms_sp, "schur_diagonal_ms": ms_spd, **info}),
          flush=True)


def solve_case(L, n, info):
    mesh = ExtrudedHexMesh(n, n, n)
    S, Q = FunctionSpace(mesh, 2, family="NCF"), FunctionSpace(mesh, 1, family="DQ")
    F = MixedPoisson(S, Q)
    X = Q.V.dof_coordinates()
    f = Q.dat(3 * np.pi ** 2 * np.sin(np.pi * X[:, 0]) * np.sin(np.pi * X[:, 1]) * np.sin(np.pi * X[:, 2]))
    b = F.dat()
    b.zero()
    b[1].axpy(-1.0, assemble(mass(Q), u=f))
    out = {}
    # one Jacobi application of S_p needs O(1/h^2) outer iterations: recorded on the smaller meshes only
    for inner in ("cg", "preonly") if n <= 32 else ("cg",):
        up = F.dat()
        _lib.check(L.fdb_synchronize())
        t0 = time.perf_counter()
        its, hist = solve(F, b, up, (), {**SOLVER, "fieldsplit_1_ksp_type": inner, "ksp_max_it": 20000})
        _lib.check(L.fdb_synchronize())
        out[inner] = {"its": its, "s": time.perf_counter() - t0, "rel_res": hist[-1] / hist[0]}
    print(json.dumps({"solve_n": n, "k": 2, **out, **info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="2:128,3:128,4:96")
    ap.add_argument("--solve", default="16,32,64")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-generic", action="store_true")
    a = ap.parse_args()
    L = _lib.init()
    info = card()
    for c in a.cases.split(","):
        if c:
            k, n = (int(v) for v in c.split(":"))
            case(L, k, n, a, info)
    for n in a.solve.split(","):
        if n:
            solve_case(L, int(n), info)


if __name__ == "__main__":
    main()
