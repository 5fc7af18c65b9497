#!/usr/bin/env python
"""Speed of the boundary mass term gamma*inner(u, v)*ds on one GPU, on warped extruded meshes with device-resident
u:

* ``facet``    -- the hand-written exterior-facet kernel (FDB_FORM_BOUNDARY_MASS) over ds("on_boundary"): every
                  vertical facet x every layer, plus the bottom and top faces (two launches);
* ``cell``     -- the cell action of the volume form on the same space: the Poisson action (FDB_FORM_HELMHOLTZ)
                  on a scalar space, the elasticity action (FDB_FORM_ELASTICITY) on a vector space;
* ``generic``  -- ``boundary_mass_kernel`` through the generic wrapper builder over the same facet sets.

One JSON line per case: ms per call (CUDA events over ``--steps`` calls after ``--warmup``, output accumulated, no
zeroing inside the window), the facet-to-cell and generic-to-facet time ratios, the max-norm difference of the
hand-written and generic results relative to max|y|, and the card's name, power limit and maximum SM clock read in
the same run.  Then, unless ``--no-solve``, one JSON line of a Robin-Helmholtz solve with the V-cycle.

    python benchmarks/boundary_terms.py
    python benchmarks/boundary_terms.py --cases s3:64 --steps 5 --no-solve
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

from firedrake_b200 import _lib, mg, op2                                          # noqa: E402
from firedrake_b200.assemble import (BoundaryMass, DirichletBC, Elasticity, Form, FunctionSpace,  # noqa: E402
                                     OneFormAssembler, _boundary_groups, assemble, boundary_mass_kernel, mass,
                                     solve)
from firedrake_b200.utility_meshes import ExtrudedHexMesh                         # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (f.strip() for f in r.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


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


def case(L, kind, p, n, a, info):
    cdim = 3 if kind == "v" else 1
    V = FunctionSpace(ExtrudedHexMesh(n, n, n, warp=0.05), p, cdim)
    u = V.dat(np.random.default_rng(p).standard_normal(V.node_count * cdim).reshape(V.node_count, cdim)
              if cdim == 3 else np.random.default_rng(p).standard_normal(V.node_count))
    y1, y2 = V.dat(), V.dat()
    for y in (y1, y2):
        y.zero()
        y.device_ptr
    groups = _boundary_groups(V, "on_boundary")
    facet_loops = []
    for fset, fmap, cmap, facet in groups:
        gk = op2.GlobalKernel(op2.Kernel("boundary_mass", degree=p, alpha=1.0, cdim=cdim, integral="exterior_facet"),
                              [fmap, cmap], extruded=True)
        facet_loops.append(op2.Parloop(gk, fset, [y1(op2.INC, fmap), V.coordinates(op2.READ, cmap), u(op2.READ, fmap),
                                                  facet(op2.READ)]))
    k = op2.Kernel("elasticity", degree=p, mu=1.0, lmbda=1.0, cdim=3) if cdim == 3 else \
        op2.Kernel("helmholtz", degree=p, alpha=1.0, beta=0.0)
    cell = op2.Parloop(op2.GlobalKernel(k, [V.cell_node_map, V.coord_map], extruded=True), V.cell_set,
                       [y1(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                        u(op2.READ, V.cell_node_map)])

    def facets():
        for loop in facet_loops:
            loop()

    gk = boundary_mass_kernel(p, 1.0, cdim)

    def generic():
        for fset, fmap, cmap, facet in groups:
            op2.par_loop(gk, fset, y2(op2.INC, fmap), V.coordinates(op2.READ, cmap), u(op2.READ, fmap),
                         facet(op2.READ))

    t_facet = timed(L, facets, a.warmup, a.steps)
    t_cell = timed(L, cell, a.warmup, a.steps)
    t_gen = timed(L, generic, 1, a.generic_steps)
    for y in (y1, y2):
        y.zero()
        y.device_ptr
    facets()
    generic()
    h = np.empty(y1._data.size)
    _lib.check(L.fdb_memcpy_d2h(h.ctypes.data, y1.device_ptr, h.nbytes))
    scale = float(np.abs(h).max())
    _lib.check(L.fdb_vec_axpy(h.size, -1.0, y1.device_ptr, y2.device_ptr))          # y2 = generic - facet
    _lib.check(L.fdb_memcpy_d2h(h.ctypes.data, y2.device_ptr, h.nbytes))
    nfacets = sum(fset.total_size * (fset.layers - 1) for fset, _, _, _ in groups)
    return {"workload": f"gamma*inner(u, v)*ds('on_boundary') action vs the {'elasticity' if cdim == 3 else 'Poisson'}"
                        f" cell action, {'vector ' if cdim == 3 else ''}CG{p} on {n}^3 warped extruded hexes",
            "degree": p, "cdim": cdim, "n": n, "dofs": V.node_count * cdim, "facets": nfacets,
            "cells": V.mesh.num_cells,
            "ms": {"facet": t_facet, "cell": t_cell, "generic": t_gen},
            "facet_over_cell": t_facet / t_cell, "generic_over_facet": t_gen / t_facet,
            "rel_diff_facet_vs_generic": float(np.abs(h).max()) / scale,
            "steps": {"facet": a.steps, "cell": a.steps, "generic": a.generic_steps}, "warmup": a.warmup,
            "gpu": info}


def robin_solve(L, levels, info):
    """-div grad u + u/2 = 1, u = 0 on "bottom", Robin h = 2, u_inf = 0.3 on the four sides and "top": CG2 with
    the V-cycle on the finest level of a hierarchy over a 2^3 mesh."""
    h = mg.MeshHierarchy(2, 2, 2, levels)
    V = FunctionSpace(h[levels], 2)
    sides = (1, 2, 3, 4, "top")
    rhs = assemble(mass(V), u=V.dat(np.ones(V.node_count)))
    rhs.axpy(1.0, OneFormAssembler(BoundaryMass(V, 2.0, sides), V.dat(np.full(V.node_count, 0.3))).assemble())
    u = V.dat()
    _lib.check(L.fdb_synchronize())
    t0 = time.perf_counter()
    its, hist = solve(Form(V, 1.0, 0.5, ds=((2.0, sides),)), rhs, u, bcs=[DirichletBC(V, 0.0, "bottom")],
                      hierarchy=h, solver_parameters={"pc_type": "mg", "ksp_rtol": 1e-8})
    _lib.check(L.fdb_synchronize())
    n = 2 * 2 ** levels
    print(json.dumps({"workload": f"Robin-Helmholtz solve, CG2 on {n}^3, CG + V-cycle", "n": n,
                      "dofs": V.node_count, "iterations": its, "wall_s": time.perf_counter() - t0,
                      "rel_residual": hist[-1] / hist[0], "gpu": info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="s3:128,s3:256,v2:128,v3:128", help="s|v degree:n,...")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--generic-steps", type=int, default=3)
    ap.add_argument("--solve-levels", type=int, default=5)
    ap.add_argument("--no-solve", action="store_true")
    a = ap.parse_args()
    L = _lib.lib()
    info = card()
    for c in a.cases.split(","):
        kind_p, n = c.split(":")
        print(json.dumps(case(L, kind_p[0], int(kind_p[1:]), int(n), a, info)), flush=True)
    if not a.no_solve:
        robin_solve(L, a.solve_levels, info)


if __name__ == "__main__":
    main()
