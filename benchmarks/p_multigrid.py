#!/usr/bin/env python
"""p-multigrid against geometric multigrid and Jacobi on one GPU: Poisson with Dirichlet conditions on the bottom
and top, on warped extruded meshes, CG_p on n^3 cells.  For each case and preconditioner (one JSON line each):

* ``jacobi``   -- Jacobi-CG;
* ``gmg``      -- ``pc_type mg`` on a MeshHierarchy (coarsest mesh 4 cells per axis);
* ``p1pc_cg``  -- ``firedrake.P1PC``, Chebyshev-Jacobi levels, coarse CG1 solved by Jacobi-CG to rtol 1e-3;
* ``p1pc_mg``  -- ``firedrake.P1PC`` with a ``preonly`` + ``mg`` coarse solve on the same hierarchy.

``its`` / ``seconds``: outer iterations and time to rtol 1e-8, set-up included, from a host clock ending in
fdb_synchronize (after one untimed solve of the same case, which warms every kernel and the NVRTC cache).  Then, per
case, one line with the prolong and restrict kernel times (CUDA events over ``--steps`` calls after ``--warmup``)
and their GB/s from the algorithmic bytes (below), and the fused Chebyshev step against the unfused fdb_vec_*
sequence it replaces (aypx, pointwise_mult, aypx-style update of d, axpy).  The card's name and power limit are read
in the same run.

Algorithmic bytes per call: prolong reads the coarse values once per cell ((q+1)^3 doubles and ints) and writes
every fine node once per cell ((p+1)^3 doubles and ints); restrict reads (p+1)^3 fine values, weights and ints per
cell and adds (q+1)^3 coarse values (read + write) with their ints.

    python benchmarks/p_multigrid.py
    python benchmarks/p_multigrid.py --cases 3:64 --solvers gmg,p1pc_mg
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from firedrake_b200 import _lib, mg                                               # noqa: E402
from firedrake_b200.assemble import DirichletBC, Form, FunctionSpace, assemble, mass, solve  # noqa: E402

HBM_TBPS = 3.35
SOLVERS = {
    "jacobi": {"pc_type": "jacobi"},
    "gmg": {"pc_type": "mg"},
    "p1pc_cg": {"pc_type": "python", "pc_python_type": "firedrake.P1PC"},
    "p1pc_mg": {"pc_type": "python", "pc_python_type": "firedrake.P1PC",
                "pmg_mg_coarse": {"ksp_type": "preonly", "pc_type": "mg"}},
}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (f.strip() for f in r.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power}


def timed(L, fn, warmup, steps):
    for _ in range(warmup):
        fn()
    t = C.c_void_p()
    _lib.check(L.fdb_timer_create(C.byref(t)))
    ms = C.c_float()
    _lib.check(L.fdb_synchronize())
    _lib.check(L.fdb_timer_start(t))
    for _ in range(steps):
        fn()
    _lib.check(L.fdb_timer_stop(t, C.byref(ms)))
    _lib.check(L.fdb_timer_destroy(t))
    return ms.value / steps


def run_solve(V, h, sp):
    bcs = [DirichletBC(V, 0.0, s) for s in ("bottom", "top")]
    X = V.V.dof_coordinates() if V.node_count < 2_000_000 else None
    f = V.dat(np.sin(3 * X[:, 0]) * np.cos(2 * X[:, 1]) if X is not None else np.ones(V.node_count))
    L = assemble(mass(V), u=f)
    u = V.dat()
    t0 = time.perf_counter()
    its, _ = solve(Form(V), L, u, bcs=bcs, hierarchy=h, solver_parameters=dict(sp, ksp_rtol=1e-8, ksp_max_it=20000))
    _lib.check(_lib.lib().fdb_synchronize())
    return its, time.perf_counter() - t0


def kernels(L, V, warmup, steps):
    p = V.degree
    Vc = FunctionSpace(V.mesh, 1)
    T = mg.PTransfer(Vc, V)
    xc, xf, yc, yf = Vc.dat(np.ones(Vc.node_count)), V.dat(np.ones(V.node_count)), Vc.dat(), V.dat()
    T.weight
    cells = V.mesh.num_cells
    nf, nc = (p + 1) ** 3, 8
    t_p = timed(L, lambda: T.prolong(xc, yf), warmup, steps)
    t_r = timed(L, lambda: T._loop("p_restrict", yc(mg.op2.INC, T.cmap), xf(mg.op2.READ, V.cell_node_map),
                                   T.weight(mg.op2.READ, V.cell_node_map)), warmup, steps)
    b_p = cells * (nc * 12 + nf * 12)
    b_r = cells * (nf * 20 + nc * 20)
    n = V.node_count
    v = [V.dat(np.ones(n)) for _ in range(5)]
    b, ax, dinv, d, x = (w.device_ptr for w in v)
    scratch = V.dat()
    t = scratch.device_ptr
    t_f = timed(L, lambda: _lib.check(L.fdb_vec_chebyshev(n, 0.5, 1.1, b, ax, dinv, d, x)), warmup, steps)

    def unfused():
        _lib.check(L.fdb_memcpy_d2d(t, ax, 8 * n))
        _lib.check(L.fdb_vec_aypx(n, -1.0, b, t))                  # t = b - ax
        _lib.check(L.fdb_vec_pointwise_mult(n, t, dinv, t))        # t = dinv t
        _lib.check(L.fdb_vec_aypx(n, 0.5 / 1.1, t, d))             # d = t + c d
        _lib.check(L.fdb_vec_scale(n, 1.1, d))
        _lib.check(L.fdb_vec_axpy(n, 1.0, d, x))
    t_u = timed(L, unfused, warmup, steps)
    return {"prolong_ms": round(t_p, 4), "prolong_GBps": round(b_p / t_p / 1e6, 1),
            "restrict_ms": round(t_r, 4), "restrict_GBps": round(b_r / t_r / 1e6, 1),
            "chebyshev_fused_ms": round(t_f, 4), "chebyshev_unfused_ms": round(t_u, 4), "hbm_TBps": HBM_TBPS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="3:64,3:128,2:128", help="p:n pairs")
    ap.add_argument("--solvers", default=",".join(SOLVERS))
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    L = _lib.init()
    info = card()
    for case in a.cases.split(","):
        p, n = (int(v) for v in case.split(":"))
        levels = int(np.log2(n // 4))
        h = mg.MeshHierarchy(4, 4, 4, levels, warp=0.05)
        V = FunctionSpace(h[levels], p)
        for name in a.solvers.split(","):
            run_solve(V, h, SOLVERS[name])                         # warm-up: modules, NVRTC, colour plans
            its, sec = run_solve(V, h, SOLVERS[name])
            print(json.dumps({"case": f"CG{p} {n}^3", "dofs": V.node_count, "solver": name, "its": its,
                              "seconds": round(sec, 3), **info}), flush=True)
        print(json.dumps({"case": f"CG{p} {n}^3", "kernels": kernels(L, V, a.warmup, a.steps), **info}), flush=True)


if __name__ == "__main__":
    main()
