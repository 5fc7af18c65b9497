#!/usr/bin/env python
"""Speed of the linear elasticity action  inner(sigma(u), grad v)*dx + beta*inner(u, v)*dx  on one GPU,
three ways on the same warped extruded mesh and the same device-resident vector u (3 components):

* ``elasticity`` -- the hand-written kernel (FDB_FORM_ELASTICITY, csrc/elasticity_hex.cu);
* ``vector``     -- the cdim = 3 vector Helmholtz action (FDB_FORM_HELMHOLTZ, alpha = 1, beta = 1): the
                    same sum-factorised contractions on three uncoupled components;
* ``generic``    -- ``elasticity_kernel`` through the generic wrapper builder (one thread per cell, NVRTC).

One JSON line per (degree, n): ms per action (CUDA events over ``--steps`` launches after ``--warmup``,
output accumulated, no zeroing inside the window), DoF/s counting 3 DoFs per node, the elasticity /
vector and generic / elasticity time ratios, the max-norm difference between the elasticity and generic
results relative to max|y| (one fresh action each).  Then one line per preconditioner for a solve of the
manufactured problem of tests/test_elasticity_gpu.py (CG1, clamped, nu = 0.3) with its iterations and
seconds.  Every line carries the card's name, power limit and maximum SM clock, read in the same run.

    python benchmarks/elasticity.py                         # the cases of DESIGN.md section 4.8
    python benchmarks/elasticity.py --cases 3:64 --steps 5 --solve-n 16
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from firedrake_b200 import _lib, op2                                              # noqa: E402
from firedrake_b200.assemble import FunctionSpace, elasticity_kernel, interpolate  # noqa: E402
from firedrake_b200.utility_meshes import ExtrudedHexMesh                         # noqa: E402

from coefficient_action import card, timed                                      # noqa: E402

MU, LMBDA, BETA = 1.0, 1.5, 0.0
U = ["sin(2.0 * x[0]) * cos(x[1]) + x[2] * x[2]", "x[0] * x[1] - cos(x[2])", "sin(x[0] + 2.0 * x[2])"]


def case(L, p, n, a, info):
    V = FunctionSpace(ExtrudedHexMesh(n, n, n, warp=0.05), p, 3)
    u = interpolate(V, U)
    y1, y2 = V.dat(), V.dat()
    for y in (y1, y2):
        y.zero()
        y.device_ptr
    base = [V.coordinates(op2.READ, V.coord_map), u(op2.READ, V.cell_node_map)]
    gk = lambda k: op2.GlobalKernel(k, [V.cell_node_map, V.coord_map], extruded=True)
    elas = op2.Parloop(gk(op2.Kernel("elasticity", degree=p, mu=MU, lmbda=LMBDA, beta=BETA, cdim=3)),
                       V.cell_set, [y1(op2.INC, V.cell_node_map)] + base)
    vec = op2.Parloop(gk(op2.Kernel("helmholtz", degree=p, alpha=1.0, beta=1.0, cdim=3)), V.cell_set,
                      [y1(op2.INC, V.cell_node_map)] + base)
    ek = elasticity_kernel(p, MU, LMBDA, BETA)

    def generic():
        op2.par_loop(ek, V.cell_set, y2(op2.INC, V.cell_node_map), *base)

    t_el = timed(L, elas, a.warmup, a.steps)
    t_vec = timed(L, vec, a.warmup, a.steps)
    t_gen = timed(L, generic, 1, a.generic_steps)
    for y in (y1, y2):
        y.zero()
        y.device_ptr
    elas()
    generic()
    h = np.empty(y1._data.size)
    _lib.check(L.fdb_memcpy_d2h(h.ctypes.data, y1.device_ptr, h.nbytes))
    scale = float(np.abs(h).max())
    _lib.check(L.fdb_vec_axpy(h.size, -1.0, y1.device_ptr, y2.device_ptr))             # y2 = generic - elas
    _lib.check(L.fdb_memcpy_d2h(h.ctypes.data, y2.device_ptr, h.nbytes))
    dofs = 3 * V.node_count
    return {"workload": f"linear elasticity action, vector CG{p} on {n}^3 warped extruded hexes",
            "degree": p, "n": n, "dofs": dofs,
            "ms": {"elasticity": t_el, "vector": t_vec, "generic": t_gen},
            "dofs_per_s": {"elasticity": dofs / (t_el * 1e-3), "vector": dofs / (t_vec * 1e-3),
                           "generic": dofs / (t_gen * 1e-3)},
            "elasticity_over_vector": t_el / t_vec, "generic_over_elasticity": t_gen / t_el,
            "rel_diff_elasticity_vs_generic": float(np.abs(h).max()) / scale,
            "steps": {"elasticity": a.steps, "vector": a.steps, "generic": a.generic_steps}, "warmup": a.warmup,
            "gpu": info}


def solve_case(L, n, pc, info):
    import test_elasticity_gpu as tg
    from firedrake_b200.assemble import solve
    refinements = int(np.log2(n // 2))
    V, h, F, rhs, bcs, ui = tg.manufactured(n, 1, refinements if pc == "mg" else 0)
    u = V.dat()
    _lib.check(L.fdb_synchronize())
    t0 = time.perf_counter()
    its, hist = solve(F, rhs, u, bcs=bcs, hierarchy=h,
                      solver_parameters={"pc_type": pc, "ksp_rtol": 1e-8, "ksp_max_it": 5000})
    _lib.check(L.fdb_synchronize())
    dt = time.perf_counter() - t0
    return {"workload": f"elasticity solve, CG1 on {n}^3 unit cube, clamped, nu = 0.3, pc_type {pc}"
                        + (f" ({refinements + 1} levels from 2^3)" if pc == "mg" else ""),
            "n": n, "dofs": 3 * V.node_count, "pc_type": pc, "ksp_rtol": 1e-8, "iterations": its,
            "seconds": dt, "l2_error": tg.l2_error(V, u, ui), "gpu": info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="1:256,2:128,2:256,3:128,4:64,4:128", help="degree:n,...")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--generic-steps", type=int, default=2)
    ap.add_argument("--solve-n", type=int, default=32, help="0: no solves")
    a = ap.parse_args()
    L = _lib.lib()
    info = card()
    for c in a.cases.split(","):
        p, n = (int(v) for v in c.split(":"))
        print(json.dumps(case(L, p, n, a, info)), flush=True)
    if a.solve_n:
        for pc in ("mg", "jacobi"):
            print(json.dumps(solve_case(L, a.solve_n, pc, info)), flush=True)


if __name__ == "__main__":
    main()
