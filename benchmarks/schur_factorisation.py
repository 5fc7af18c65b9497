#!/usr/bin/env python
"""Newton on the lid-driven cavity with the diagonal, lower and upper Schur factorisations of the Taylor-Hood
fieldsplit, on one GPU.

The 3-D lid-driven cavity (Q2-Q1, lid (1, 0, 0), nu = 1/Re, from rest) with the velocity V-cycle, the inverse
diagonal of (1/nu) M_p on the pressure, the constant-pressure nullspace, snes_rtol 1e-8 and GMRES(30) with
ksp_rtol 1e-6 and at most 3000 iterations per step; one JSON line per (Re, n, pc_fieldsplit_schur_fact_type)
with the Newton steps, the GMRES iterations per step, whether it converged and the synchronised wall time
(including the preconditioner set-up).  Every line carries the card's name and power limit, read in the same run.

    python benchmarks/schur_factorisation.py                 # the table of DESIGN.md section 4.13
    python benchmarks/schur_factorisation.py --solve-n 8 --re 10 --fact diag,lower
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
from firedrake_b200.assemble import (ConvergenceError, DirichletBC, FunctionSpace, NavierStokes,  # noqa: E402
                                     solve_nonlinear)
from firedrake_b200.utility_meshes import ExtrudedHexMesh                           # noqa: E402

from coefficient_action import card                                                # noqa: E402


def cavity(L, re, n, fact, info):
    from firedrake_b200.mg import MeshHierarchy
    mesh = ExtrudedHexMesh(n, n, n)
    V, Q = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1)
    F = NavierStokes(V, Q, 1.0 / re)
    lid = np.zeros((V.node_count, 3))
    lid[:, 0] = 1.0
    bcs = [DirichletBC(V, 0.0, (1, 2, 3, 4, "bottom")), DirichletBC(V, V.dat(lid), "top")]
    levels = int(np.log2(n // 2))
    sp = {"snes_rtol": 1e-8, "snes_max_it": 25, "ksp_rtol": 1e-6, "ksp_max_it": 3000, "pc_type": "fieldsplit",
          "pc_fieldsplit_type": "schur", "pc_fieldsplit_schur_fact_type": fact, "fieldsplit_0_pc_type": "mg",
          "fieldsplit_1_pc_type": "jacobi"}
    up = F.dat()
    _lib.check(L.fdb_synchronize())
    t0 = time.perf_counter()
    reason = None
    try:
        hist, kits = solve_nonlinear(F, F.dat(), up, bcs, sp, hierarchy=MeshHierarchy(2, 2, 2, levels),
                                     nullspace="constant")
    except ConvergenceError as e:
        hist, kits, reason = [float("nan")], [], e.reason
    _lib.check(L.fdb_synchronize())
    dt = time.perf_counter() - t0
    converged = reason is None and hist[-1] <= 1e-8 * hist[0]
    return {"workload": f"lid-driven cavity, Navier-Stokes Re = {re:g}, Q2-Q1 on {n}^3, Newton from rest, "
                        f"fieldsplit schur {fact}, velocity V-cycle ({levels + 1} levels from 2^3)",
            "re": re, "n": n, "dofs": 3 * V.node_count + Q.node_count, "pc_fieldsplit_schur_fact_type": fact,
            "snes_rtol": 1e-8, "ksp_rtol": 1e-6, "converged": converged, "reason": reason,
            "newton_steps": len(kits), "gmres_iterations_per_step": kits, "residual_norms": hist,
            "seconds": dt, "gpu": info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solve-n", default="16,32", help="cavity sizes, comma separated")
    ap.add_argument("--re", default="1,10,100", help="Reynolds numbers of the cavity, comma separated")
    ap.add_argument("--fact", default="diag,lower,upper", help="pc_fieldsplit_schur_fact_type values")
    a = ap.parse_args()
    L = _lib.lib()
    info = card()
    for re in (float(v) for v in a.re.split(",") if v):
        for n in (int(v) for v in a.solve_n.split(",") if v):
            for fact in (v for v in a.fact.split(",") if v):
                print(json.dumps(cavity(L, re, n, fact, info)), flush=True)


if __name__ == "__main__":
    main()
