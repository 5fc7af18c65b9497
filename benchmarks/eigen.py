#!/usr/bin/env python
"""The eigensolver on one GPU (one JSON line each):

* ``bv``     -- fdb_bv_dot and fdb_bv_mult alone at n = --bv-n (57,066,625 = the CG3 dofs of 128^3) with m = k in
                --bv-cols: ms per call, GB/s of algorithmic traffic (every x and y column read once; fdb_bv_mult with
                beta = 0 reads x and writes y) against the HBM peak (MEASURED_PEAKS.json, else the data sheet's
                3.35 TB/s), fp64 TFLOP/s (2 m k n) against 33.5, and the time of the m k fdb_vec_dot and m k
                fdb_vec_axpy calls they replace.
* ``lobpcg`` -- the Dirichlet Laplacian at CG3 on warped n^3 meshes, n_evals = 8, eps_tol 1e-8, st_pc_type jacobi, mg
                and P1PC: iterations and wall time (set-up included), then a second, instrumented run whose per-iteration
                split into A actions, M actions, preconditioner, fdb_bv_dot, fdb_bv_mult and the host Rayleigh-Ritz
                synchronises the device around every part.

CUDA events time the kernels after --warmup calls.  The card's name, power limit and SM clock are read in the same
run.

    python benchmarks/eigen.py
    python benchmarks/eigen.py --only lobpcg --n 64 --pcs mg
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

from firedrake_b200 import _lib, mg                                                      # noqa: E402
from firedrake_b200.assemble import DirichletBC, Form, FunctionSpace, mass               # noqa: E402
from firedrake_b200.eigensolver import LinearEigenproblem, LinearEigensolver             # noqa: E402
from firedrake_b200.utility_meshes import ExtrudedHexMesh                                # noqa: E402

WALLS = [1, 2, 3, 4, "bottom", "top"]
FP64_TFLOPS = 33.5          # H100 SXM data sheet, non-tensor fp64


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    name, power, sm, smax = (f.strip() for f in r.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "clocks_sm": sm, "clocks_max_sm": smax}


def peak_gbs():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"], "MEASURED_PEAKS.json"
    except Exception:
        return 3350.0, "H100 SXM data sheet"


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


def bench_bv(L, n, cols, warmup, steps):
    peak, src = peak_gbs()
    for m in cols:
        k = m
        bufs = [L.fdb_malloc(n * 8) for _ in range(m + k)]
        if not all(bufs):
            raise MemoryError(f"fdb_malloc of {m + k} columns of {n} doubles")
        for i, b in enumerate(bufs):
            _lib.check(L.fdb_vec_fill(n, 1.0 + 1e-3 * i, b))
        xs = (C.c_void_p * m)(*bufs[:m])
        ys = (C.c_void_p * k)(*bufs[m:])
        g = np.empty(m * k)
        gp = g.ctypes.data_as(C.POINTER(C.c_double))
        Q = np.random.default_rng(0).standard_normal(m * k)
        qp = Q.ctypes.data_as(C.POINTER(C.c_double))
        out = C.c_double()
        t_dot = timed(L, lambda: _lib.check(L.fdb_bv_dot(n, m, xs, k, ys, gp)), warmup, steps)
        t_mult = timed(L, lambda: _lib.check(L.fdb_bv_mult(n, k, ys, 0.0, 1.0, m, xs, qp)), warmup, steps)

        def dots():
            for i in range(m):
                for j in range(k):
                    _lib.check(L.fdb_vec_dot(n, bufs[i], bufs[m + j], C.byref(out)))

        def axpys():
            for j in range(k):
                for i in range(m):
                    _lib.check(L.fdb_vec_axpy(n, 1e-3, bufs[i], bufs[m + j]))

        t_dots = timed(L, dots, 1, 1)
        t_axpys = timed(L, axpys, 1, 1)
        nbytes = 8.0 * n * (m + k)
        flops = 2.0 * m * k * n
        for name, ms, ref in (("fdb_bv_dot", t_dot, t_dots), ("fdb_bv_mult", t_mult, t_axpys)):
            gbs = nbytes / (ms * 1e-3) / 1e9
            tf = flops / (ms * 1e-3) / 1e12
            print(json.dumps({"bench": "bv", "kernel": name, "n": n, "m": m, "k": k, "ms": round(ms, 3),
                              "GB/s": round(gbs, 1), "hbm_fraction": round(gbs / peak, 3), "peak_source": src,
                              "fp64_TFLOP/s": round(tf, 2), "fp64_fraction": round(tf / FP64_TFLOPS, 3),
                              "replaced_calls": m * k,
                              "replaced_ms": round(ref, 1), "speedup": round(ref / ms, 1), "card": CARD}),
                  flush=True)
        for b in bufs:
            L.fdb_free(b)


class Split:
    """Synchronised wall time of each part of an iteration, accumulated by wrapping the solver's methods."""

    def __init__(self, L, es):
        self.L, self.t = L, {}
        orig_setup = es._setup

        def setup():
            orig_setup()
            self.wrap(es, "_precondition", "preconditioner")
            self.wrap(es._bv, "dot", "fdb_bv_dot")
            self.wrap(es._bv, "mult", "fdb_bv_mult")
            self.wrap(es, "_ritz", "rayleigh_ritz")
            self.wrap(es, "_normaliser", "rayleigh_ritz")
            apply = es._apply

            def timed_apply(op, x, out):
                return self.run(f"{op}_action", apply, op, x, out)
            es._apply = timed_apply
        es._setup = setup

    def run(self, key, fn, *a, **kw):
        _lib.check(self.L.fdb_synchronize())
        t0 = time.perf_counter()
        r = fn(*a, **kw)
        _lib.check(self.L.fdb_synchronize())
        self.t[key] = self.t.get(key, 0.0) + time.perf_counter() - t0
        return r

    def wrap(self, obj, name, key):
        fn = getattr(obj, name)
        setattr(obj, name, lambda *a, **kw: self.run(key, fn, *a, **kw))


def bench_lobpcg(L, sizes, pcs, max_it):
    for n in sizes:
        for pc in pcs:
            h = None
            if pc == "mg":
                lev = int(np.log2(n // 4))
                h = mg.MeshHierarchy(4, 4, 4, lev, warp=0.05)
                mesh = h[len(h) - 1]
            else:
                mesh = ExtrudedHexMesh(n, n, n, warp=0.05)
            V = FunctionSpace(mesh, 3)
            bc = DirichletBC(V, 0.0, WALLS)
            sp = {"eps_tol": 1e-8, "eps_max_it": max_it}
            if pc == "P1PC":
                sp.update({"st_pc_type": "python", "st_pc_python_type": "firedrake.P1PC"})
            else:
                sp["st_pc_type"] = pc
            prob = LinearEigenproblem(Form(V, 1.0, 0.0), mass(V), bcs=[bc])
            res = {"bench": "lobpcg", "n": n, "degree": 3, "dofs": V.node_count, "st_pc_type": pc, "n_evals": 8}
            try:
                es = LinearEigensolver(prob, 8, solver_parameters=sp, hierarchy=h)
                _lib.check(L.fdb_synchronize())
                t0 = time.perf_counter()
                es.solve()
                _lib.check(L.fdb_synchronize())
                res.update(iterations=es.iterations, wall_s=round(time.perf_counter() - t0, 2),
                           eigenvalues_over_pi2=[round(es.eigenvalue(i) / np.pi ** 2, 6) for i in range(8)])
                del es
                es = LinearEigensolver(prob, 8, solver_parameters=sp, hierarchy=h)
                split = Split(L, es)
                es.solve()
                its = max(es.iterations, 1)
                res["split_ms_per_iteration"] = {k: round(1e3 * v / its, 2) for k, v in split.t.items()}
                del es
            except Exception as e:                   # a configuration that does not fit or converge is reported
                res["error"] = f"{type(e).__name__}: {e}"
            res["card"] = CARD
            print(json.dumps(res), flush=True)


def main():
    global CARD
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["bv", "lobpcg"])
    ap.add_argument("--bv-n", type=int, default=385 ** 3)
    ap.add_argument("--bv-cols", type=int, nargs="+", default=[24, 48, 63])
    ap.add_argument("--n", type=int, nargs="+", default=[64, 128])
    ap.add_argument("--pcs", nargs="+", default=["jacobi", "mg", "P1PC"])
    ap.add_argument("--max-it", type=int, default=3000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    L = _lib.init()
    CARD = card()
    if args.only in (None, "bv"):
        bench_bv(L, args.bv_n, args.bv_cols, args.warmup, args.steps)
    if args.only in (None, "lobpcg"):
        bench_lobpcg(L, args.n, args.pcs, args.max_it)


CARD = None

if __name__ == "__main__":
    main()
