#!/usr/bin/env python
"""Speed of the Boussinesq (Rayleigh-Benard) residual and Jacobian action on Taylor-Hood hexahedra with the
temperature on the pressure numbering, on one GPU, and Newton with the demo's fieldsplit on the heated cavity.

Actions, on the same warped extruded mesh and device-resident vectors:

* ``residual``          -- the hand-written residual (FDB_FORM_BOUSSINESQ, EL_RB_RESIDUAL);
* ``jacobian``          -- the hand-written Jacobian action at (u, T) (FDB_FORM_BOUSSINESQ_JACOBIAN, EL_RB_JACOBIAN);
* ``ns_residual``, ``ns_jacobian`` -- the Navier-Stokes kernels on the same velocity and pressure spaces;
* ``generic_residual``, ``generic_jacobian`` -- ``boussinesq_kernel`` through the generic wrapper builder.

One JSON line per (degree, n): ms per action (CUDA events over ``--steps`` launches after ``--warmup``, outputs
accumulated; the generic path over ``--generic-steps`` after one), the ratios to the Navier-Stokes kernels and of
the generic path to the hand-written one, and the max-norm difference to the generic path relative to max|y| over the
three blocks.

Newton: the differentially heated cube (no slip on every wall, T = 1 on x = 0, T = 0 on x = 1, adiabatic elsewhere,
g = (0, 0, -1), Q2-Q1-Q1, from rest) with the demo's options -- outer fgmres, multiplicative fieldsplit, fieldsplit_0
gmres (rtol 1e-2) with the lower Schur factorisation, fieldsplit_1 gmres (rtol 1e-4) -- with the velocity and
temperature preconditioned by Jacobi or V-cycles, snes_rtol 1e-8, ksp_rtol 1e-6 and the constant-pressure
nullspace.  One line per (Ra, n, pc) with the Newton steps, the outer iterations per step, the inner iterations per
step and the synchronised wall time.  Every line carries the card's name and power limit, read in the same run.

    python benchmarks/boussinesq.py                     # the cases of DESIGN.md section 4.22
    python benchmarks/boussinesq.py --cases 2:32 --steps 3 --solve-n 8 --ra 1000
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

from firedrake_b200 import _lib, op2                                                # noqa: E402
from firedrake_b200.assemble import (Boussinesq, ConvergenceError, DirichletBC, FunctionSpace,  # noqa: E402
                                     NavierStokes, StokesAssembler, boussinesq_kernel, solve_nonlinear)
from firedrake_b200.utility_meshes import ExtrudedHexMesh                           # noqa: E402

from coefficient_action import card, timed                                        # noqa: E402

RA, PR = 1.0e3, 6.8


def _diff(a, b):
    d = max(float(np.abs(x.data_ro - y.data_ro).max()) for x, y in zip(a, b))
    return d / max(float(np.abs(x.data_ro).max()) for x in a)


def case(L, p, n, a, info):
    mesh = ExtrudedHexMesh(n, n, n, warp=0.05)
    V, Q, W = FunctionSpace(mesh, p, 3), FunctionSpace(mesh, p - 1), FunctionSpace(mesh, p - 1)
    F = Boussinesq(V, Q, W, RA, PR)
    N = NavierStokes(V, Q, 1.0)
    rng = np.random.default_rng(0)
    upT = F.dat(rng.standard_normal((V.node_count, 3)), rng.standard_normal(Q.node_count),
                rng.standard_normal(W.node_count))
    wrs = F.dat(rng.standard_normal((V.node_count, 3)), rng.standard_normal(Q.node_count),
                rng.standard_normal(W.node_count))
    up, wr = op2.MixedDat([upT[0], upT[1]]), op2.MixedDat([wrs[0], wrs[1]])
    y1, y2, yn = F.dat(), F.dat(), N.dat()
    for y in (y1, y2, yn):
        y.zero()
        for d in y:
            d.device_ptr
    loops = {}
    for key, form, x, y in (("residual", F, upT, y1), ("jacobian", F.jacobian(upT), wrs, y1),
                            ("ns_residual", N, up, yn), ("ns_jacobian", N.jacobian(up), wr, yn)):
        asm = StokesAssembler(form, x)
        asm.assemble(y)
        loops[key] = asm._loop
    mm = op2.MixedMap(F.block_maps)
    kr, kj = boussinesq_kernel(p, RA, PR), boussinesq_kernel(p, RA, PR, jacobian=True)
    X = V.coordinates(op2.READ, V.coord_map)

    def gen_res():
        op2.par_loop(kr, V.cell_set, y2(op2.INC, mm), X, upT(op2.READ, mm))

    def gen_jac():
        op2.par_loop(kj, V.cell_set, y2(op2.INC, mm), X, wrs(op2.READ, mm), upT[0](op2.READ, V.cell_node_map),
                     upT[2](op2.READ, F.temperature_map))

    ms = {k: timed(L, lp, a.warmup, a.steps) for k, lp in loops.items()}
    ms["generic_residual"] = timed(L, gen_res, 1, a.generic_steps)
    ms["generic_jacobian"] = timed(L, gen_jac, 1, a.generic_steps)
    diffs = {}
    for key, gen in (("residual", gen_res), ("jacobian", gen_jac)):
        y1.zero()
        loops[key]()
        y2.zero()
        gen()
        diffs[key] = _diff(y1, y2)
    dofs = 3 * V.node_count + Q.node_count + W.node_count
    return {"workload": f"Boussinesq residual and Jacobian action, Q{p}-Q{p - 1}-Q{p - 1} on {n}^3 warped extruded "
                        f"hexes",
            "degree": p, "n": n, "dofs": dofs, "ms": ms, "dofs_per_s": {k: dofs / (t * 1e-3) for k, t in ms.items()},
            "residual_over_ns": ms["residual"] / ms["ns_residual"],
            "jacobian_over_ns": ms["jacobian"] / ms["ns_jacobian"],
            "generic_over_handwritten": {"residual": ms["generic_residual"] / ms["residual"],
                                         "jacobian": ms["generic_jacobian"] / ms["jacobian"]},
            "rel_diff_vs_generic": diffs, "steps": {"handwritten": a.steps, "generic": a.generic_steps},
            "warmup": a.warmup, "gpu": info}


def cavity(L, ra, n, pc, info):
    from firedrake_b200.mg import MeshHierarchy
    mesh = ExtrudedHexMesh(n, n, n)
    V, Q, W = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1), FunctionSpace(mesh, 1)
    F = Boussinesq(V, Q, W, ra, PR)
    bcs = [DirichletBC(V, 0.0, (1, 2, 3, 4, "bottom", "top")), DirichletBC(W, 1.0, 1), DirichletBC(W, 0.0, 2)]
    levels = int(np.log2(n // 2))
    hier = MeshHierarchy(2, 2, 2, levels) if pc == "mg" else None
    sp = {"snes_rtol": 1e-8, "snes_max_it": 25, "ksp_type": "fgmres", "ksp_rtol": 1e-6, "ksp_max_it": 1000,
          "pc_type": "fieldsplit", "pc_fieldsplit_type": "multiplicative",
          "pc_fieldsplit_0_fields": "0,1", "pc_fieldsplit_1_fields": "2",
          "fieldsplit_0": {"ksp_type": "gmres", "ksp_rtol": 1e-2, "pc_type": "fieldsplit",
                           "pc_fieldsplit_type": "schur", "pc_fieldsplit_schur_fact_type": "lower",
                           "fieldsplit_0": {"ksp_type": "preonly", "pc_type": pc},
                           "fieldsplit_1": {"ksp_type": "preonly", "pc_type": "jacobi"}},
          "fieldsplit_1": {"ksp_type": "gmres", "ksp_rtol": 1e-4, "pc_type": pc}}
    upT = F.dat()
    _lib.check(L.fdb_synchronize())
    t0 = time.perf_counter()
    reason = None
    try:
        hist, kits, inner = solve_nonlinear(F, F.dat(), upT, bcs, sp, hierarchy=hier, nullspace="constant")
    except ConvergenceError as e:
        hist, kits, inner, reason = [float("nan")], [], [], e.reason
    _lib.check(L.fdb_synchronize())
    dt = time.perf_counter() - t0
    converged = reason is None and hist[-1] <= 1e-8 * hist[0]
    return {"workload": f"heated cavity, Boussinesq Ra = {ra:g}, Pr = {PR:g}, Q2-Q1-Q1 on {n}^3, Newton from rest, "
                        f"multiplicative fieldsplit, velocity and temperature pc {pc}"
                        + (f" ({levels + 1} levels from 2^3)" if pc == "mg" else ""),
            "ra": ra, "pr": PR, "n": n, "dofs": 3 * V.node_count + 2 * Q.node_count, "pc": pc,
            "snes_rtol": 1e-8, "ksp_rtol": 1e-6, "converged": converged, "reason": reason,
            "newton_steps": len(kits), "outer_iterations_per_step": kits,
            "inner_iterations_per_step": [list(c) for c in inner], "residual_norms": hist,
            "seconds": dt, "gpu": info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="2:128,3:128,4:64", help="degree:n,...")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--generic-steps", type=int, default=2)
    ap.add_argument("--solve-n", default="16,32", help="cavity sizes, comma separated; empty: no solves")
    ap.add_argument("--ra", default="1000,10000", help="Rayleigh numbers of the cavity, comma separated")
    ap.add_argument("--pc", default="mg,jacobi", help="velocity and temperature pc types, comma separated")
    a = ap.parse_args()
    L = _lib.lib()
    info = card()
    for c in a.cases.split(","):
        if c:
            p, n = (int(v) for v in c.split(":"))
            print(json.dumps(case(L, p, n, a, info)), flush=True)
    for ra in (float(v) for v in a.ra.split(",") if v):
        for n in (int(v) for v in a.solve_n.split(",") if v):
            for pc in (v for v in a.pc.split(",") if v):
                print(json.dumps(cavity(L, ra, n, pc, info)), flush=True)


if __name__ == "__main__":
    main()
