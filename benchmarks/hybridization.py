#!/usr/bin/env python
"""Speed of the hybridised mixed Poisson solver (HybridizationPC, csrc/hybrid_hex.cu) on one GPU, on a warped extruded
mesh with device-resident vectors.

* Kernel times (CUDA events over ``--steps`` calls after ``--warmup``): HY_CONDENSE (the trace matrix, into a zeroed
  CSR without lgmaps), HY_ELIMINATE and HY_RECONSTRUCT, with FLOP/s from the local algebra counted from the shapes:
  the flux mass matrix entry by entry (2 flops per point per lower-triangle entry) and the symmetric elimination (2
  flops per updated entry of the packed triangle, dense: the kernel skips rows whose multiplier is exactly zero, so
  the rates slightly overstate the work done); the CSR's nnz and bytes.  At k = 2 also the generic-wrapper-path
  condensation (``assemble_hybrid_trace_generic``, one thread per cell) and its difference from the hand-written H.
* Solves: the unit-cube problem of DESIGN.md section 4.21 (u = sin sin sin, natural u = 0), hybridised ("preonly",
  Jacobi-CG on the trace system, ``--trace-rtol``) and the existing "full" selfp fieldsplit with inner Jacobi-CG
  (GMRES rtol 1e-8), each with its iterations, seconds and the relative residual of the mixed system it reached.
  ``load`` "sin" is that smooth load, "random" a seeded random u-load (and zero flux load), which excites every mode
  of the trace system.

Every line carries the card's name and power limit, read in the same run.

    python benchmarks/hybridization.py                       # the cases of DESIGN.md section 4.23
    python benchmarks/hybridization.py --cases 2:16 --solve 2:8 --steps 3
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
from firedrake_b200.assemble import (FunctionSpace, HybridizationPC, MixedPoisson,  # noqa: E402
                                     MixedPoissonMatrixContext, assemble, assemble_hybrid_trace_generic, mass,
                                     solve)
from firedrake_b200.utility_meshes import ExtrudedHexMesh                           # noqa: E402

from coefficient_action import card, timed                                        # noqa: E402

SCHUR = {"ksp_type": "gmres", "ksp_rtol": 1e-8, "pc_type": "fieldsplit", "pc_fieldsplit_type": "schur",
         "pc_fieldsplit_schur_fact_type": "full", "pc_fieldsplit_schur_precondition": "selfp",
         "fieldsplit_0_ksp_type": "preonly", "fieldsplit_0_pc_type": "jacobi", "fieldsplit_1_ksp_type": "cg",
         "fieldsplit_1_pc_type": "jacobi", "fieldsplit_1_ksp_rtol": 1e-5, "ksp_max_it": 20000}


def local_flops(k):
    """Counted flops per cell of (condense, eliminate, reconstruct): the mass matrix and the elimination."""
    ns, nu, nf, npts = 3 * k * k * (k + 1), k ** 3, 6 * k * k, (k + 1) ** 3
    nl = ns + nu
    mass_flops = ns * (ns + 1) // 2 * npts * 2

    def elim(n):
        return sum(2 * (n - j - 1) * (n - j) // 2 for j in range(nl))
    back = nl * (nl - 1)                           # the back substitution
    return mass_flops + elim(nl + nf), mass_flops + elim(nl + 1) + back, mass_flops + elim(nl + 1) + back


def kernels(L, k, n, a, info):
    mesh = ExtrudedHexMesh(n, n, n, warp=0.05)
    S, Q = FunctionSpace(mesh, k, family="NCF"), FunctionSpace(mesh, k - 1, family="DQ")
    F = MixedPoisson(S, Q, 1.0)
    t0 = time.perf_counter()
    pc = HybridizationPC(F)
    _lib.check(L.fdb_synchronize())
    setup_s = time.perf_counter() - t0
    rng = np.random.default_rng(0)
    Ld = F.dat(rng.standard_normal(S.node_count), rng.standard_normal(Q.node_count))
    lam, r, up = pc.trace.dat(rng.standard_normal(pc.trace.node_count)), pc.trace.dat(), F.dat()
    cond = op2.Parloop(pc._gk[2], S.cell_set, [pc.mat(op2.INC, (pc.trace_map, pc.trace_map)),
                                               S.coordinates(op2.READ, S.coord_map)])
    elim = op2.Parloop(pc._gk[1], S.cell_set, [r(op2.INC, pc.trace_map), S.coordinates(op2.READ, S.coord_map),
                                               Ld[0](op2.READ, S.cell_node_map), pc.w(op2.READ, S.cell_node_map),
                                               Ld[1](op2.READ, F.pressure_map)])
    rec = op2.Parloop(pc._gkr, S.cell_set, [up[0](op2.INC, S.cell_node_map), S.coordinates(op2.READ, S.coord_map),
                                            lam(op2.READ, pc.trace_map), Ld[0](op2.READ, S.cell_node_map),
                                            pc.w(op2.READ, S.cell_node_map), up[1](op2.INC, F.pressure_map),
                                            Ld[1](op2.READ, F.pressure_map)])
    for d in (r, up[0], up[1]):
        d.zero()
        d.device_ptr
    ms = {name: timed(L, fn, a.warmup, a.steps) for name, fn in (("condense", cond), ("eliminate", elim),
                                                                   ("reconstruct", rec))}
    gen = {}
    if k == 2:
        pc.assemble()                            # the timed condensations above added into pc.mat
        Hg = assemble_hybrid_trace_generic(pc)
        a_, b_ = pc.mat.csr()[2], Hg.csr()[2]
        gen = {"generic_condense_ms": timed(L, lambda: assemble_hybrid_trace_generic(pc, Hg), 1, max(1, a.steps // 2)),
               "generic_max_rel_diff": float(np.abs(a_ - b_).max() / np.abs(a_).max())}
        del Hg
    ncell = mesh.num_cells
    fl = dict(zip(("condense", "eliminate", "reconstruct"), local_flops(k)))
    print(json.dumps({"k": k, "n": n, "cells": ncell, "trace_dofs": pc.trace.node_count, "csr_nnz": pc.mat.nnz,
                      "csr_bytes": pc.mat.nnz * 12 + (pc.mat.nrows + 1) * 8, "setup_s": setup_s,
                      **{f"{m}_ms": ms[m] for m in ms},
                      **{f"{m}_gflops": fl[m] * ncell / (ms[m] * 1e-3) / 1e9 for m in ms},
                      **{f"{m}_flops_per_cell": fl[m] for m in ms}, **gen, **info}), flush=True)


def mixed_residual(F, b, up):
    A = MixedPoissonMatrixContext(F)
    y = F.dat()
    A.mult(up, y)
    y.axpy(-1.0, b)
    return float(np.sqrt(sum(d.inner(d) for d in y)) / np.sqrt(sum(d.inner(d) for d in b)))


def solve_case(L, k, n, load, a, info):
    mesh = ExtrudedHexMesh(n, n, n)
    S, Q = FunctionSpace(mesh, k, family="NCF"), FunctionSpace(mesh, k - 1, family="DQ")
    F = MixedPoisson(S, Q)
    X = Q.V.dof_coordinates()
    f = Q.dat(3 * np.pi ** 2 * np.sin(np.pi * X[:, 0]) * np.sin(np.pi * X[:, 1]) * np.sin(np.pi * X[:, 2]))
    b = F.dat()
    b.zero()
    if load == "sin":
        b[1].axpy(-1.0, assemble(mass(Q), u=f))
    else:
        b[1].axpy(1.0, Q.dat(np.random.default_rng(7).standard_normal(Q.node_count)))
    hyb = {"mat_type": "matfree", "ksp_type": "preonly", "pc_type": "python",
           "pc_python_type": "firedrake.HybridizationPC",
           "hybridization": {"ksp_type": "cg", "pc_type": "jacobi", "ksp_rtol": a.trace_rtol, "ksp_max_it": 100000}}
    out = {}
    for name, sp in (("hybrid", hyb), ("schur_full", SCHUR)):
        up = F.dat()
        solve(F, b, up, (), sp)                  # warm-up: module loads, sparsity build, first launches
        up = F.dat()
        _lib.check(L.fdb_synchronize())
        t0 = time.perf_counter()
        its, hist = solve(F, b, up, (), sp)
        _lib.check(L.fdb_synchronize())
        out[name] = {"its": its, "s": time.perf_counter() - t0, "mixed_rel_res": mixed_residual(F, b, up)}
    print(json.dumps({"solve_n": n, "k": k, "load": load, **out, **info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="2:128,3:64")
    ap.add_argument("--solve", default="2:16,2:32,2:64,3:16,3:32")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--trace-rtol", type=float, default=1e-8)
    ap.add_argument("--loads", default="sin,random")
    a = ap.parse_args()
    L = _lib.init()
    info = card()
    for c in a.cases.split(","):
        if c:
            kernels(L, *(int(v) for v in c.split(":")), a, info)
    for c in a.solve.split(","):
        if c:
            for load in a.loads.split(","):
                solve_case(L, *(int(v) for v in c.split(":")), load, a, info)


if __name__ == "__main__":
    main()
