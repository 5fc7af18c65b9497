#!/usr/bin/env python
"""The fast-diagonalisation vertex-star relaxation (FDMPC + ASMExtrudedStarPC, csrc/fdm_star_hex.cu) on one GPU.
One JSON line per measurement; the card's name and power limit are read in the same run.

* ``kernel``: the star apply (patch.FDMStar.apply: one memset and 8 colour launches) for CG1..CG5, CUDA events over
  ``--steps`` calls after ``--warmup``, beside the matrix-free action of the same Form (OneFormAssembler) at the
  same size.  FLOP/s from 12 m^4 flops per star (m = 2p - 1: six 1-D contractions of m^3 points by m), GB/s from the
  algorithmic bytes per star: m^3 values of r read, m^3 values of z read and written and m^3 map entries (28 m^3
  bytes), plus the memset of z.  ``chebyshev_unit_dinv_ms``: the fdb_vec_chebyshev call of one star-preconditioned
  Chebyshev step (unit dinv, zero ax), and its share of the step (action, residual, star apply, that call), the
  most a fused variant could save.  ``setup_s``: FDMStar construction (host tables, upload), ``table_MB`` its device
  memory.  Warped meshes at 64^3; at 128^3 unwarped meshes, whose table pool is a handful of entries (the warped
  pools at 128^3 hold 3 (n+1)^3 entries).
* ``solve``: Poisson with Dirichlet bottom and top on warped meshes to rtol 1e-8, CG_p on n^3 cells: Jacobi-CG (CG
  without a preconditioner at CG4 and CG5, which have no diagonal kernel),
  GMG (pc_type mg, coarsest mesh 4^3), P1PC with Chebyshev-Jacobi levels and FDMPC + P1PC with the star smoother,
  and FDMPC with the one-level star relaxation.  ``seconds`` includes the set-up; ``star_setup_s`` is the FDMStar
  construction on the fine level alone, timed separately.

    python benchmarks/fdm_star.py
    python benchmarks/fdm_star.py --kernels 3:64 --solves 3:64 --solvers jacobi,p1pc_star
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

from firedrake_b200 import _lib, mg                                                          # noqa: E402
from firedrake_b200.assemble import (DirichletBC, Form, FunctionSpace, OneFormAssembler, assemble,  # noqa: E402
                                     mass, solve)
from firedrake_b200.patch import FDMStar                                                     # noqa: E402
from firedrake_b200.utility_meshes import ExtrudedHexMesh                                    # noqa: E402

HBM_TBPS = 3.35
STAR_LEVELS = {"ksp_type": "chebyshev", "ksp_max_it": 2, "pc_type": "python",
               "pc_python_type": "firedrake.ASMExtrudedStarPC", "pc_star_sub_sub_pc_type": "lu"}
SOLVERS = {
    "none": {"pc_type": "none"},
    "jacobi": {"pc_type": "jacobi"},
    "gmg": {"pc_type": "mg"},
    "p1pc_jacobi": {"pc_type": "python", "pc_python_type": "firedrake.P1PC"},
    "p1pc_star": {"pc_type": "python", "pc_python_type": "firedrake.FDMPC",
                  "fdm": {"pc_type": "python", "pc_python_type": "firedrake.P1PC", "pmg_mg_levels": STAR_LEVELS}},
    "star": {"pc_type": "python", "pc_python_type": "firedrake.FDMPC",
             "fdm": {"pc_type": "python", "pc_python_type": "firedrake.ASMExtrudedStarPC",
                     "pc_star_sub_sub_pc_type": "lu"}},
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


def kernel(L, p, n, warmup, steps):
    warp = 0.05 if n <= 64 else 0.0
    V = FunctionSpace(ExtrudedHexMesh(n, n, n, warp=warp), p)
    form = Form(V)
    t0 = time.perf_counter()
    star = FDMStar(form, [DirichletBC(V, 0.0, s) for s in ("bottom", "top")])
    _lib.check(L.fdb_synchronize())
    setup = time.perf_counter() - t0
    r, z = V.dat(np.ones(V.node_count)), V.dat()
    t_s = timed(L, lambda: star.apply(r, z), warmup, steps)
    asm = OneFormAssembler(form, r)
    y = V.dat()
    t_a = timed(L, lambda: asm.assemble(tensor=y), warmup, steps)
    # the vector work of one star-preconditioned Chebyshev step of mg.PMG: the residual (aypx) and
    # fdb_vec_chebyshev with a unit dinv and a zero ax, which a fused variant could at most remove
    nn = V.node_count
    b, ax, s, d, x, zero, one = (V.dat(np.full(nn, v)) for v in (1.0, 0.5, 0.25, 0.0, 0.0, 0.0, 1.0))
    t_y = timed(L, lambda: _lib.check(L.fdb_vec_aypx(nn, -1.0, b.device_ptr, ax.device_ptr)), warmup, steps)
    t_c = timed(L, lambda: _lib.check(L.fdb_vec_chebyshev(nn, 0.5, 1.1, s.device_ptr, zero.device_ptr, one.device_ptr,
                                                          d.device_ptr, x.device_ptr)), warmup, steps)
    m = 2 * p - 1
    nstar = len(star.tables.star_vert)
    flops = 12 * m ** 4 * nstar
    byts = 28 * m ** 3 * nstar + 8 * V.node_count
    return {"case": f"CG{p} {n}^3", "warp": warp, "dofs": V.node_count, "stars": nstar, "star_ms": round(t_s, 4),
            "star_GFLOPs": round(flops / t_s / 1e6, 1), "star_GBps": round(byts / t_s / 1e6, 1),
            "action_ms": round(t_a, 4), "residual_aypx_ms": round(t_y, 4), "chebyshev_unit_dinv_ms": round(t_c, 4),
            "chebyshev_share_of_step": round(t_c / (t_a + t_y + t_s + t_c), 4), "setup_s": round(setup, 2),
            "pool_entries": len(star.tables.pool),
            "table_MB": round(star.tables.nbytes / 1e6, 1), "hbm_TBps": HBM_TBPS}


def run_solve(V, h, sp):
    bcs = [DirichletBC(V, 0.0, s) for s in ("bottom", "top")]
    L = assemble(mass(V), u=V.dat(np.sin(np.arange(V.node_count) * 0.37)))
    u = V.dat()
    t0 = time.perf_counter()
    its, _ = solve(Form(V), L, u, bcs=bcs, hierarchy=h, solver_parameters=dict(sp, ksp_rtol=1e-8, ksp_max_it=20000))
    _lib.check(_lib.lib().fdb_synchronize())
    return its, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernels", default="1:64,2:64,3:64,4:64,5:64,1:128,2:128,3:128,4:128,5:128", help="p:n pairs")
    ap.add_argument("--solves", default="2:64,3:64,2:128,3:128", help="p:n pairs")
    ap.add_argument("--solvers", default="jacobi,gmg,p1pc_jacobi,p1pc_star,star")
    ap.add_argument("--one-level", default="2:64,3:64,4:64,5:64", help="p:n pairs for star against jacobi")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    L = _lib.init()
    info = card()
    pairs = lambda s: [tuple(int(v) for v in c.split(":")) for c in s.split(",") if c]
    for p, n in pairs(a.kernels):
        print(json.dumps({"kernel": kernel(L, p, n, a.warmup, a.steps), **info}), flush=True)
    runs = [(p, n, a.solvers.split(",")) for p, n in pairs(a.solves)]
    # at CG4 and CG5 there is no diagonal kernel: the one-level star against unpreconditioned CG
    runs += [(p, n, ["jacobi" if p <= 3 else "none", "star"]) for p, n in pairs(a.one_level)
             if (p, n) not in pairs(a.solves)]
    for p, n, names in runs:
        levels = int(np.log2(n // 4))
        h = mg.MeshHierarchy(4, 4, 4, levels, warp=0.05)
        V = FunctionSpace(h[levels], p)
        t0 = time.perf_counter()
        FDMStar(Form(V), [DirichletBC(V, 0.0, s) for s in ("bottom", "top")])
        _lib.check(L.fdb_synchronize())
        setup = time.perf_counter() - t0
        h0 = mg.MeshHierarchy(4, 4, 4, 1, warp=0.05)
        for name in names:
            if name in ("gmg", "p1pc_jacobi", "p1pc_star") and p > 3:
                continue
            run_solve(FunctionSpace(h0[1], p), h0, SOLVERS[name])           # warm-up: modules, NVRTC
            its, sec = run_solve(V, h, SOLVERS[name])
            print(json.dumps({"solve": f"CG{p} {n}^3", "dofs": V.node_count, "solver": name, "its": its,
                              "seconds": round(sec, 3), "star_setup_s": round(setup, 2), **info}), flush=True)


if __name__ == "__main__":
    main()
