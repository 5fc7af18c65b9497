#!/usr/bin/env python
"""The spectral-element wave equation on one GPU, on warped extruded meshes of n^3 cells (one JSON line each):

* ``action``   -- for CG_p: the collocated SEM action (FDB_FORM_SPECTRAL_HELMHOLTZ_COEF), helmholtz_coef given the
                  GLL tables through ``op2.Kernel(element=...)`` (the same discrete operator) and the Gauss
                  helmholtz_coef action, atomic scatter, with kappa; ms per action and DoF/s;
* ``step``     -- one leapfrog step of CG_p split into the SEM action (coloured scatter, as ``leapfrog`` runs it),
                  the point load of one source, the fused step fdb_vec_leapfrog and the evaluation at 64 receivers,
                  then the fused step's GB/s (5 doubles per entry: minv, r, u, uprev read, uprev written) against the
                  unfused fdb_vec_* sequence that computes the same update.

Kernel times are CUDA events over ``--steps`` calls after ``--warmup``.  The card's name and power limit are read in
the same run.

    python benchmarks/wave.py
    python benchmarks/wave.py --degrees 3 --n 64
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from firedrake_b200 import _lib, op2                                                    # noqa: E402
from firedrake_b200.assemble import (FunctionSpace, OneFormAssembler, PointEvaluator, SpectralForm,  # noqa: E402
                                     lumped_mass)
from firedrake_b200.fiat_lite import interval_element                                     # noqa: E402
from firedrake_b200.utility_meshes import ExtrudedHexMesh                                 # noqa: E402


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


def actions(L, V, kap, x, warmup, steps):
    p = V.degree
    sem = OneFormAssembler(SpectralForm(V, 1.0, 0.0, kap), x)
    out = {"sem": sem.assemble}
    for name, el in (("coef_gll", interval_element(p, quadrature="gll")), ("coef_gauss", None)):
        y = V.dat()
        k = op2.Kernel("helmholtz_coef", degree=p, alpha=1.0, beta=0.0, element=el)
        loop = op2.Parloop(op2.GlobalKernel(k, [V.cell_node_map, V.coord_map], extruded=True), V.cell_set,
                           [y(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                            x(op2.READ, V.cell_node_map), kap(op2.READ, V.cell_node_map)], location="device")

        def run(y=y, loop=loop):
            y.zero()
            loop()
        out[name] = run
    y = V.dat()
    res = {}
    for name, fn in out.items():
        ms = timed(L, (lambda fn=fn: fn(y)) if name == "sem" else fn, warmup, steps)
        res[f"{name}_ms"] = round(ms, 3)
        res[f"{name}_dofs_per_s"] = float(f"{V.node_count / ms * 1e3:.3g}")
    return res


def step(L, V, kap, x, warmup, steps):
    n = V.node_count
    F = SpectralForm(V, 1.0, 0.0, kap)
    m = lumped_mass(V)
    X = V.mesh.coordinates
    lo, hi = X.min(axis=0), X.max(axis=0)
    rng = np.random.default_rng(0)
    src = PointEvaluator(V, [0.5 * (lo + hi)])
    rec = PointEvaluator(V, lo + (hi - lo) * rng.uniform(0.1, 0.9, (64, 3)))
    amp = op2.DeviceArray.from_host(np.ones(1))
    tr = op2.DeviceArray(8 * 64)
    r, up = V.dat(), V.dat(np.zeros(n))
    asm = OneFormAssembler(F, x, scatter="coloured")
    minv = V.dat(1.0 / m.data_ro)
    res = {"action_ms": timed(L, lambda: asm.assemble(tensor=r), warmup, steps),
           "load_ms": timed(L, lambda: src._load_into(amp.ptr, -1.0, r), warmup, steps),
           "eval_ms": timed(L, lambda: rec._eval_into(x, tr.ptr), warmup, steps)}
    rp, xp, upp, mp = r.device_ptr, x.device_ptr, up.device_ptr, minv.device_ptr
    res["leapfrog_ms"] = timed(L, lambda: _lib.check(L.fdb_vec_leapfrog(n, 1e-6, mp, rp, xp, upp)), warmup, steps)
    t = V.dat(np.zeros(n))
    tp = t.device_ptr

    def unfused():
        _lib.check(L.fdb_vec_pointwise_mult(n, rp, mp, tp))          # t = minv r
        _lib.check(L.fdb_vec_aypx(n, -1.0, xp, upp))                 # uprev = u - uprev
        _lib.check(L.fdb_vec_axpy(n, 1.0, xp, upp))                  # uprev += u
        _lib.check(L.fdb_vec_axpy(n, -1e-6, tp, upp))                # uprev -= dt2 t
    res["unfused_ms"] = timed(L, unfused, warmup, steps)
    res["leapfrog_GBps"] = 5 * 8 * n / res["leapfrog_ms"] / 1e6
    res["step_ms"] = res["action_ms"] + res["load_ms"] + res["leapfrog_ms"] + res["eval_ms"]
    return {k: round(v, 4) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--degrees", default="2,3,4,5")
    ap.add_argument("--n", type=int, default=128)
    ap.add_argument("--step-degree", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    L = _lib.init()
    info = card()
    mesh = ExtrudedHexMesh(a.n, a.n, a.n, warp=0.05)
    for p in (int(v) for v in a.degrees.split(",")):
        V = FunctionSpace(mesh, p)
        rng = np.random.default_rng(p)
        kap = V.dat(rng.uniform(1.0, 2.0, V.node_count))
        x = V.dat(rng.standard_normal(V.node_count))
        print(json.dumps({"case": f"CG{p} {a.n}^3", "dofs": V.node_count,
                          "action": actions(L, V, kap, x, a.warmup, a.steps), **info}), flush=True)
        if p == a.step_degree:
            print(json.dumps({"case": f"CG{p} {a.n}^3", "dofs": V.node_count,
                              "step": step(L, V, kap, x, a.warmup, a.steps), **info}), flush=True)
        del V, kap, x


if __name__ == "__main__":
    main()
