#!/usr/bin/env python
"""Speed of the Stokes saddle-point action on Taylor-Hood hexahedra on one GPU, four ways on the same warped
extruded mesh and the same device-resident vectors:

* ``stokes``     -- the fused hand-written action (FDB_FORM_STOKES, the EL_STOKES mode of
                    csrc/elasticity_hex.cu): velocity CG_p and pressure CG_(p-1) in and out;
* ``elasticity`` -- the linear elasticity action on the velocity space (the same kernel family);
* ``vector``     -- the cdim = 3 vector Poisson action on the velocity space (FDB_FORM_HELMHOLTZ);
* ``generic``    -- ``stokes_kernel`` through the generic wrapper builder with MixedDat arguments.

One JSON line per (degree, n): ms per action (CUDA events over ``--steps`` launches after ``--warmup``,
outputs accumulated, no zeroing inside the window), DoF/s counting velocity plus pressure DoFs for stokes
and generic (velocity DoFs for the other two), and the max-norm difference between the fused and generic
results relative to max|y| over both blocks.  Then one line per velocity preconditioner for the lid-driven
cavity (Q2-Q1, GMRES with the diagonal Schur fieldsplit, constant-pressure nullspace, rtol 1e-8) with its
iterations and seconds.  Every line carries the card's name and power limit, read in the same run.

    python benchmarks/stokes.py                          # the cases of DESIGN.md section 4.11
    python benchmarks/stokes.py --cases 2:32 --steps 3 --solve-n 8
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
from firedrake_b200.assemble import (DirichletBC, FunctionSpace, Stokes, StokesAssembler, solve,  # noqa: E402
                                     stokes_kernel)
from firedrake_b200.utility_meshes import ExtrudedHexMesh                           # noqa: E402

from coefficient_action import card, timed                                        # noqa: E402

MU, BETA = 1.0, 0.0


def case(L, p, n, a, info):
    mesh = ExtrudedHexMesh(n, n, n, warp=0.05)
    V, Q = FunctionSpace(mesh, p, 3), FunctionSpace(mesh, p - 1)
    F = Stokes(V, Q, MU, BETA)
    rng = np.random.default_rng(0)
    up = F.dat(rng.standard_normal((V.node_count, 3)), rng.standard_normal(Q.node_count))
    y1, y2 = F.dat(), F.dat()
    for y in (y1, y2):
        y.zero()
        for d in y:
            d.device_ptr
    u = up[0]
    asm = StokesAssembler(F, up)
    asm.assemble(y1)
    stokes = asm._loop
    base = [V.coordinates(op2.READ, V.coord_map), u(op2.READ, V.cell_node_map)]
    gk = lambda k: op2.GlobalKernel(k, [V.cell_node_map, V.coord_map], extruded=True)
    elas = op2.Parloop(gk(op2.Kernel("elasticity", degree=p, mu=MU, lmbda=0.0, beta=BETA, cdim=3)),
                       V.cell_set, [y1[0](op2.INC, V.cell_node_map)] + base)
    vec = op2.Parloop(gk(op2.Kernel("helmholtz", degree=p, alpha=1.0, beta=0.0, cdim=3)), V.cell_set,
                      [y1[0](op2.INC, V.cell_node_map)] + base)
    sk = stokes_kernel(p, MU, BETA)
    mm = op2.MixedMap([V.cell_node_map, F.pressure_map])

    def generic():
        op2.par_loop(sk, V.cell_set, y2(op2.INC, mm), V.coordinates(op2.READ, V.coord_map), up(op2.READ, mm))

    t_st = timed(L, stokes, a.warmup, a.steps)
    t_el = timed(L, elas, a.warmup, a.steps)
    t_vec = timed(L, vec, a.warmup, a.steps)
    t_gen = timed(L, generic, 1, a.generic_steps)
    asm.assemble(y1)
    y2.zero()
    generic()
    diff, scale = 0.0, 0.0
    for b1, b2 in zip(y1, y2):
        h1, h2 = b1.data_ro, b2.data_ro
        scale = max(scale, float(np.abs(h1).max()))
        diff = max(diff, float(np.abs(h1 - h2).max()))
    vd, pd = 3 * V.node_count, Q.node_count
    return {"workload": f"Stokes action, Q{p}-Q{p - 1} on {n}^3 warped extruded hexes",
            "degree": p, "n": n, "velocity_dofs": vd, "pressure_dofs": pd,
            "ms": {"stokes": t_st, "elasticity": t_el, "vector": t_vec, "generic": t_gen},
            "dofs_per_s": {"stokes": (vd + pd) / (t_st * 1e-3), "elasticity": vd / (t_el * 1e-3),
                           "vector": vd / (t_vec * 1e-3), "generic": (vd + pd) / (t_gen * 1e-3)},
            "stokes_over_elasticity": t_st / t_el, "generic_over_stokes": t_gen / t_st,
            "rel_diff_stokes_vs_generic": diff / scale,
            "steps": {"stokes": a.steps, "elasticity": a.steps, "vector": a.steps, "generic": a.generic_steps},
            "warmup": a.warmup, "gpu": info}


def cavity(L, n, pc0, info):
    from firedrake_b200.mg import MeshHierarchy
    mesh = ExtrudedHexMesh(n, n, n)
    V, Q = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1)
    F = Stokes(V, Q, 1.0)
    lid = np.zeros((V.node_count, 3))
    lid[:, 0] = 1.0
    bcs = [DirichletBC(V, 0.0, (1, 2, 3, 4, "bottom")), DirichletBC(V, V.dat(lid), "top")]
    levels = int(np.log2(n // 2))
    hier = MeshHierarchy(2, 2, 2, levels) if pc0 == "mg" else None
    sp = {"ksp_type": "gmres", "ksp_rtol": 1e-8, "ksp_max_it": 5000, "pc_type": "fieldsplit",
          "pc_fieldsplit_type": "schur", "pc_fieldsplit_schur_fact_type": "diag", "fieldsplit_0_pc_type": pc0,
          "fieldsplit_1_pc_type": "jacobi"}
    up = F.dat()
    _lib.check(L.fdb_synchronize())
    t0 = time.perf_counter()
    its, _ = solve(F, F.dat(), up, bcs, sp, hierarchy=hier, nullspace="constant")
    _lib.check(L.fdb_synchronize())
    dt = time.perf_counter() - t0
    return {"workload": f"lid-driven cavity, Q2-Q1 on {n}^3, fieldsplit schur diag, fieldsplit_0_pc_type {pc0}"
                        + (f" ({levels + 1} levels from 2^3)" if pc0 == "mg" else ""),
            "n": n, "dofs": 3 * V.node_count + Q.node_count, "fieldsplit_0_pc_type": pc0, "ksp_rtol": 1e-8,
            "iterations": its, "seconds": dt, "gpu": info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="2:128,2:256,3:128,4:64,4:128", help="degree:n,...")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--generic-steps", type=int, default=2)
    ap.add_argument("--solve-n", default="16,32", help="cavity sizes, comma separated; empty: no solves")
    a = ap.parse_args()
    L = _lib.lib()
    info = card()
    for c in a.cases.split(","):
        if c:
            p, n = (int(v) for v in c.split(":"))
            print(json.dumps(case(L, p, n, a, info)), flush=True)
    for n in (int(v) for v in a.solve_n.split(",") if v):
        for pc0 in ("mg", "jacobi"):
            print(json.dumps(cavity(L, n, pc0, info)), flush=True)


if __name__ == "__main__":
    main()
