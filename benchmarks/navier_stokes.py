#!/usr/bin/env python
"""Speed of the steady Navier-Stokes residual and Jacobian action on Taylor-Hood hexahedra on one GPU, and Newton
on the lid-driven cavity.

Actions, on the same warped extruded mesh and device-resident vectors:

* ``residual``          -- the hand-written residual (FDB_FORM_NAVIER_STOKES, EL_NS_RESIDUAL);
* ``jacobian``          -- the hand-written Jacobian action at u (FDB_FORM_NAVIER_STOKES_JACOBIAN, EL_NS_JACOBIAN);
* ``stokes``            -- the Stokes action on the same spaces (FDB_FORM_STOKES, EL_STOKES);
* ``generic_residual``, ``generic_jacobian`` -- ``navier_stokes_kernel`` through the generic wrapper builder.

One JSON line per (degree, n): ms per action (CUDA events over ``--steps`` launches after ``--warmup``, outputs
accumulated, no zeroing inside the window; the generic path over ``--generic-steps`` after one), the ratios to
the Stokes action, the max-norm differences to the generic path relative to max|y| over both blocks, and the
Taylor figure max|J w - (R(u + h w) - R(u - h w)) / 2h| / max|J w| at h = 1e-3.

Newton: the 3-D lid-driven cavity (Q2-Q1, lid (1, 0, 0), nu = 1/Re, from rest) with the diagonal Schur
fieldsplit (velocity Jacobi or V-cycle), the constant-pressure nullspace, snes_rtol 1e-8 and ksp_rtol 1e-6;
one line per (Re, n, fieldsplit_0_pc_type) with the Newton steps, the GMRES iterations per step, whether it
converged and the synchronised wall time.  Every line carries the card's name and power limit, read in the same
run.

    python benchmarks/navier_stokes.py                       # the cases of DESIGN.md section 4.12
    python benchmarks/navier_stokes.py --cases 2:32 --steps 3 --solve-n 8 --re 10
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
from firedrake_b200.assemble import (ConvergenceError, DirichletBC, FunctionSpace, NavierStokes,  # noqa: E402
                                     Stokes, StokesAssembler, navier_stokes_kernel, solve_nonlinear)
from firedrake_b200.utility_meshes import ExtrudedHexMesh                           # noqa: E402

from coefficient_action import card, timed                                        # noqa: E402

NU, BETA = 0.1, 0.0


def _diff(a, b):
    d = max(float(np.abs(x.data_ro - y.data_ro).max()) for x, y in zip(a, b))
    return d / max(float(np.abs(x.data_ro).max()) for x in a)


def case(L, p, n, a, info):
    mesh = ExtrudedHexMesh(n, n, n, warp=0.05)
    V, Q = FunctionSpace(mesh, p, 3), FunctionSpace(mesh, p - 1)
    F = NavierStokes(V, Q, NU, BETA)
    rng = np.random.default_rng(0)
    up = F.dat(rng.standard_normal((V.node_count, 3)), rng.standard_normal(Q.node_count))
    wr = F.dat(rng.standard_normal((V.node_count, 3)), rng.standard_normal(Q.node_count))
    y1, y2 = F.dat(), F.dat()
    for y in (y1, y2):
        y.zero()
        for d in y:
            d.device_ptr
    loops = {}
    for key, form, x in (("residual", F, up), ("jacobian", F.jacobian(up), wr), ("stokes", Stokes(V, Q, NU, BETA), up)):
        asm = StokesAssembler(form, x)
        asm.assemble(y1)
        loops[key] = asm._loop
    mm = op2.MixedMap([V.cell_node_map, F.pressure_map])
    kr, kj = navier_stokes_kernel(p, NU, BETA), navier_stokes_kernel(p, NU, BETA, jacobian=True)
    X = V.coordinates(op2.READ, V.coord_map)

    def gen_res():
        op2.par_loop(kr, V.cell_set, y2(op2.INC, mm), X, up(op2.READ, mm))

    def gen_jac():
        op2.par_loop(kj, V.cell_set, y2(op2.INC, mm), X, wr(op2.READ, mm), up[0](op2.READ, V.cell_node_map))

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
    # Taylor figure of the device kernels: R is quadratic in u, so the central difference is exact up to rounding
    h = 1e-3
    jw = [d.data_ro.copy() for d in StokesAssembler(F.jacobian(up), wr).assemble()]
    rs = []
    for s in (h, -h):
        us = F.dat(up[0].data_ro + s * wr[0].data_ro, up[1].data_ro + s * wr[1].data_ro)
        rs.append([d.data_ro.copy() for d in StokesAssembler(F, us).assemble()])
    taylor = max(float(np.abs(j - (r1 - r2) / (2 * h)).max()) for j, r1, r2 in zip(jw, *rs)) / \
        max(float(np.abs(j).max()) for j in jw)
    vd, pd = 3 * V.node_count, Q.node_count
    return {"workload": f"Navier-Stokes residual and Jacobian action, Q{p}-Q{p - 1} on {n}^3 warped extruded hexes",
            "degree": p, "n": n, "velocity_dofs": vd, "pressure_dofs": pd, "ms": ms,
            "dofs_per_s": {k: (vd + pd) / (t * 1e-3) for k, t in ms.items()},
            "residual_over_stokes": ms["residual"] / ms["stokes"], "jacobian_over_stokes": ms["jacobian"] / ms["stokes"],
            "generic_over_handwritten": {"residual": ms["generic_residual"] / ms["residual"],
                                         "jacobian": ms["generic_jacobian"] / ms["jacobian"]},
            "rel_diff_vs_generic": diffs, "taylor_central_difference": taylor,
            "steps": {"handwritten": a.steps, "generic": a.generic_steps}, "warmup": a.warmup, "gpu": info}


def cavity(L, re, n, pc0, info):
    from firedrake_b200.mg import MeshHierarchy
    mesh = ExtrudedHexMesh(n, n, n)
    V, Q = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1)
    F = NavierStokes(V, Q, 1.0 / re)
    lid = np.zeros((V.node_count, 3))
    lid[:, 0] = 1.0
    bcs = [DirichletBC(V, 0.0, (1, 2, 3, 4, "bottom")), DirichletBC(V, V.dat(lid), "top")]
    levels = int(np.log2(n // 2))
    hier = MeshHierarchy(2, 2, 2, levels) if pc0 == "mg" else None
    sp = {"snes_rtol": 1e-8, "snes_max_it": 25, "ksp_rtol": 1e-6, "ksp_max_it": 3000, "pc_type": "fieldsplit",
          "pc_fieldsplit_type": "schur", "pc_fieldsplit_schur_fact_type": "diag", "fieldsplit_0_pc_type": pc0,
          "fieldsplit_1_pc_type": "jacobi"}
    up = F.dat()
    _lib.check(L.fdb_synchronize())
    t0 = time.perf_counter()
    reason = None
    try:
        hist, kits = solve_nonlinear(F, F.dat(), up, bcs, sp, hierarchy=hier, nullspace="constant")
    except ConvergenceError as e:
        hist, kits, reason = [float("nan")], [], e.reason
    _lib.check(L.fdb_synchronize())
    dt = time.perf_counter() - t0
    converged = reason is None and hist[-1] <= 1e-8 * hist[0]
    return {"workload": f"lid-driven cavity, Navier-Stokes Re = {re:g}, Q2-Q1 on {n}^3, Newton from rest, "
                        f"fieldsplit schur diag, fieldsplit_0_pc_type {pc0}"
                        + (f" ({levels + 1} levels from 2^3)" if pc0 == "mg" else ""),
            "re": re, "n": n, "dofs": 3 * V.node_count + Q.node_count, "fieldsplit_0_pc_type": pc0,
            "snes_rtol": 1e-8, "ksp_rtol": 1e-6, "converged": converged, "reason": reason,
            "newton_steps": len(kits), "gmres_iterations_per_step": kits, "residual_norms": hist,
            "seconds": dt, "gpu": info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="2:128,2:256,3:128,4:64,4:128", help="degree:n,...")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--generic-steps", type=int, default=2)
    ap.add_argument("--solve-n", default="16,32", help="cavity sizes, comma separated; empty: no solves")
    ap.add_argument("--re", default="1,10,100", help="Reynolds numbers of the cavity, comma separated")
    ap.add_argument("--pc", default="mg,jacobi", help="fieldsplit_0_pc_type values, comma separated")
    a = ap.parse_args()
    L = _lib.lib()
    info = card()
    for c in a.cases.split(","):
        if c:
            p, n = (int(v) for v in c.split(":"))
            print(json.dumps(case(L, p, n, a, info)), flush=True)
    for re in (float(v) for v in a.re.split(",") if v):
        for n in (int(v) for v in a.solve_n.split(",") if v):
            for pc0 in (v for v in a.pc.split(",") if v):
                print(json.dumps(cavity(L, re, n, pc0, info)), flush=True)


if __name__ == "__main__":
    main()
