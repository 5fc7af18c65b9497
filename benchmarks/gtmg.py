#!/usr/bin/env python
"""GTMG (mg.GTMG, csrc/trace_transfer_hex.cu) against Jacobi-CG for the hybridised mixed Poisson trace system on one
GPU, on an unwarped unit cube with natural conditions and a seeded random load (which excites every mode of H).

* Trace CG to ``--rtol`` from lambda = 0: iterations and seconds (host clock around work ending in a device
  synchronise) for Jacobi-CG, GTMG with the (cg, jacobi) coarse solve to 1e-3, and GTMG with one CG1 V-cycle
  (preonly, mg) on a hierarchy down to 4^3.  Chebyshev-Jacobi with ``--nu`` iterations on the trace level.
* The split of one GTMG application (coarse cg): trace SpMVs (2 nu + 1 per cycle), fused Chebyshev vector passes
  (2 nu), the two transfers and the coarse solve, each timed on its own with CUDA events.
* The transfer kernels: time per call (CUDA events over ``--steps`` calls after ``--warmup``) and bytes/s, bytes
  counted from the shapes as the per-cell traffic through the maps (prolong: 6k^2 trace writes and map entries, 8
  vertex reads and map entries; restrict: 6k^2 reads of lambda, w and the map, 8 vertex read-modify-writes and map
  entries), hand-written against the generic wrapper path.

Every line carries the card's name and power limit, read in the same run.  A case that is not run is reported as
"not measured".

    python benchmarks/gtmg.py                          # k = 2 on 16^3, 32^3, 64^3 and k = 3 on 16^3, 32^3
    python benchmarks/gtmg.py --cases 2:16 --steps 5
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

from firedrake_b200 import _lib, mg                                         # noqa: E402
from firedrake_b200.assemble import FunctionSpace, HybridizationPC, MixedPoisson  # noqa: E402
from firedrake_b200.utility_meshes import ExtrudedHexMesh                   # noqa: E402

from coefficient_action import card, timed                                # noqa: E402

DEFAULT = "2:16,2:32,2:64,3:16,3:32"


def transfer_bytes(k, ncells):
    nt = 6 * k * k
    return ncells * (nt * (8 + 4) + 8 * (8 + 4)), ncells * (nt * (8 + 8 + 4) + 8 * (8 + 8 + 4))


def wall(L, fn):
    _lib.check(L.fdb_synchronize())
    t0 = time.perf_counter()
    out = fn()
    _lib.check(L.fdb_synchronize())
    return time.perf_counter() - t0, out


def case(L, k, n, a, info):
    levels = max(int(np.log2(n // 4)), 1)
    hier = mg.MeshHierarchy(n >> levels, n >> levels, n >> levels, levels)
    mesh = hier[len(hier) - 1]
    S, Q = FunctionSpace(mesh, k, family="NCF"), FunctionSpace(mesh, k - 1, family="DQ")
    F = MixedPoisson(S, Q, 1.0)
    pc = HybridizationPC(F)
    T = pc.trace
    rng = np.random.default_rng(0)
    Ld = F.dat(np.zeros(S.node_count), rng.standard_normal(Q.node_count))
    r = pc.forward(Ld)
    lam = T.dat()
    out = dict(info, k=k, n=n, trace_dofs=T.node_count, nnz=int(pc.mat.csr()[2].size))
    # trace solves
    routes = {"jacobi": None,
              "gtmg_cg": lambda: mg.GTMG(pc, nu=a.nu),
              "gtmg_mg": lambda: mg.GTMG(pc, nu=a.nu, coarse_ksp="preonly", coarse_pc="mg", hierarchy=hier)}
    cycles = {}
    for name, make in routes.items():
        setup, cyc = wall(L, make) if make else (0.0, None)
        cycles[name] = cyc
        pc.trace_solve(r, lam, a.rtol, 20000, "jacobi", cycle=cyc)           # warm-up
        sec, (its, hist) = wall(L, lambda: pc.trace_solve(r, lam, a.rtol, 20000, "jacobi", cycle=cyc))
        out[name] = dict(iterations=its, seconds=sec, setup_seconds=setup, reached=hist[-1] / hist[0])
    # the split of one GTMG application (coarse cg)
    g = cycles["gtmg_cg"]
    w1, w0 = g._work[1], g._work[0]
    tt = g.transfers[0]
    z = T.dat()
    tt.restrict(r, w0["b"])
    split = {
        "cycle": timed(L, lambda: g(r, z), a.warmup, a.steps),
        "trace_spmv": timed(L, lambda: pc.mat.mult(r, w1["t"]), a.warmup, a.steps) * (2 * a.nu + 1),
        "chebyshev_pass": timed(L, lambda: L.fdb_vec_chebyshev(T.node_count, 0.5, 0.5, r.device_ptr,
                                                                  w1["t"].device_ptr, g.invdiag[1].device_ptr,
                                                                  w1["d"].device_ptr, w1["x"].device_ptr),
                                a.warmup, a.steps) * 2 * a.nu,
        "prolong": timed(L, lambda: tt.prolong(w0["x"], w1["e"]), a.warmup, a.steps),
        "restrict": timed(L, lambda: tt.restrict(r, w0["b"]), a.warmup, a.steps),
        "coarse_solve": timed(L, lambda: g._coarse_solve(w0["b"], w0["x"]), a.warmup, a.steps),
    }
    out["split_ms"] = split
    # transfer kernels, hand-written against generic
    ncells = mesh.num_cells
    bp, br = transfer_bytes(k, ncells)
    c = tt.Vc.dat(rng.standard_normal(tt.Vc.node_count))
    lt, ct = T.dat(), tt.Vc.dat()
    tr = {}
    for tag, pro, res in (("hand", tt.prolong, tt.restrict), ("generic", tt.prolong_generic, tt.restrict_generic)):
        mp = timed(L, lambda: pro(c, lt), a.warmup, a.steps)
        mr = timed(L, lambda: res(r, ct), a.warmup, a.steps)
        tr[tag] = dict(prolong_ms=mp, restrict_ms=mr, prolong_GBs=bp / mp / 1e6, restrict_GBs=br / mr / 1e6)
    tr["speedup_prolong"] = tr["generic"]["prolong_ms"] / tr["hand"]["prolong_ms"]
    tr["speedup_restrict"] = tr["generic"]["restrict_ms"] / tr["hand"]["restrict_ms"]
    out["transfers"] = tr
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=DEFAULT)
    ap.add_argument("--skip", default="", help="cases to report as not measured")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--nu", type=int, default=3)
    ap.add_argument("--rtol", type=float, default=1e-8)
    a = ap.parse_args()
    _lib.init()
    L = _lib.lib()
    info = {"card": card()}
    skip = set(a.skip.split(",")) - {""}
    for spec in a.cases.split(","):
        k, n = (int(v) for v in spec.split(":"))
        if spec in skip:
            print(json.dumps(dict(info, k=k, n=n, result="not measured")), flush=True)
            continue
        print(json.dumps(case(L, k, n, a, info)), flush=True)


if __name__ == "__main__":
    main()
