#!/usr/bin/env python
"""Speed of the advection-diffusion action  inner(grad u, grad v)*dx + inner(dot(b, grad u), v)*dx  on one GPU,
four ways on the same warped extruded mesh and the same device-resident u (and b, kappa):

* ``adv``      -- the hand-written slab-thread kernel in its advection mode (FDB_FORM_ADVECTION_DIFFUSION);
* ``coef``     -- the coefficient form's action (FDB_FORM_HELMHOLTZ_COEF), the kernel whose layout it extends
                  (one coefficient buffer instead of three);
* ``const``    -- the constant-coefficient Poisson action (FDB_FORM_HELMHOLTZ);
* ``generic``  -- ``advection_diffusion_kernel`` through the generic wrapper builder (one thread per cell,
                  NVRTC), the path the form had before; degrees 1..3 (``null`` at degree 4).

One JSON line per (degree, n): ms per action (CUDA events over ``--steps`` launches after ``--warmup``,
output accumulated, no zeroing inside the window), DoF/s, the time ratios, the max-norm difference between
the adv and generic results relative to max|y| (one fresh action each), and the card's name, power limit
and maximum SM clock read in the same run.  Then, unless ``--no-solve``, one JSON line per
(mesh, pc_type) of the manufactured CG1 problem solved with GMRES: iterations and wall time.

    python benchmarks/advection_diffusion.py                    # CG1..CG4 at 128^3, CG1..CG3 at 256^3
    python benchmarks/advection_diffusion.py --cases 3:128 --steps 5 --no-solve
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
from firedrake_b200.assemble import (AdvectionDiffusion, DirichletBC, FunctionSpace, OneFormAssembler,  # noqa: E402
                                     advection_diffusion_kernel, interpolate, mass, solve)
from firedrake_b200.utility_meshes import ExtrudedHexMesh                         # noqa: E402

KAPPA = "2.0 + sin(3.0 * x[0]) * x[1]"
U = "sin(2.0 * x[0]) * cos(x[1]) + x[2] * x[2]"


def velocity(X):
    return np.stack([1.0 + 0.5 * X[:, 1], 0.5 - 0.25 * X[:, 0], np.full(len(X), 0.25)], axis=1)


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


def case(L, p, n, a, info):
    V = FunctionSpace(ExtrudedHexMesh(n, n, n, warp=0.05), p)
    u, kap = interpolate(V, U), interpolate(V, KAPPA)
    b = op2.Dat(V.vector_dset(3), velocity(V.V.dof_coordinates()))
    y1, y2 = V.dat(), V.dat()
    for y in (y1, y2):
        y.zero()
        y.device_ptr
    base = [V.coordinates(op2.READ, V.coord_map), u(op2.READ, V.cell_node_map)]
    gk = lambda k: op2.GlobalKernel(k, [V.cell_node_map, V.coord_map], extruded=True)
    out = [y1(op2.INC, V.cell_node_map)]
    adv = op2.Parloop(gk(op2.Kernel("advection_diffusion", degree=p)), V.cell_set,
                      out + base + [b(op2.READ, V.cell_node_map)])
    coef = op2.Parloop(gk(op2.Kernel("helmholtz_coef", degree=p)), V.cell_set,
                       out + base + [kap(op2.READ, V.cell_node_map)])
    const = op2.Parloop(gk(op2.Kernel("helmholtz", degree=p)), V.cell_set, out + base)
    t_adv = timed(L, adv, a.warmup, a.steps)
    t_coef = timed(L, coef, a.warmup, a.steps)
    t_const = timed(L, const, a.warmup, a.steps)
    t_gen = diff = None
    if p <= 3:                       # the generic statement takes degrees 1..3 (assemble.advection_diffusion_kernel)
        ak = advection_diffusion_kernel(p)

        def generic():
            op2.par_loop(ak, V.cell_set, y2(op2.INC, V.cell_node_map), *base, b(op2.READ, V.cell_node_map))

        t_gen = timed(L, generic, 1, a.generic_steps)
        for y in (y1, y2):
            y.zero()
            y.device_ptr
        adv()
        generic()
        h = np.empty(y1._data.size)
        _lib.check(L.fdb_memcpy_d2h(h.ctypes.data, y1.device_ptr, h.nbytes))
        scale = float(np.abs(h).max())
        _lib.check(L.fdb_vec_axpy(h.size, -1.0, y1.device_ptr, y2.device_ptr))         # y2 = generic - adv
        _lib.check(L.fdb_memcpy_d2h(h.ctypes.data, y2.device_ptr, h.nbytes))
        diff = float(np.abs(h).max()) / scale
    dofs = V.node_count
    times = (("adv", t_adv), ("coef", t_coef), ("const", t_const), ("generic", t_gen))
    return {"workload": f"inner(grad u, grad v)*dx + inner(dot(b, grad u), v)*dx action, CG{p} on {n}^3 "
                        f"warped extruded hexes",
            "degree": p, "n": n, "dofs": dofs,
            "ms": dict(times),
            "dofs_per_s": {k: dofs / (t * 1e-3) for k, t in times if t is not None},
            "adv_over_coef": t_adv / t_coef, "adv_over_const": t_adv / t_const,
            "generic_over_adv": t_gen / t_adv if t_gen else None, "rel_diff_adv_vs_generic": diff,
            "steps": {"adv": a.steps, "coef": a.steps, "const": a.steps, "generic": a.generic_steps},
            "warmup": a.warmup, "gpu": info}


def solves(L, levels, info):
    """-div grad u + b.grad u + u/2 = f, u = sin(pi x) sin(pi y) sin(pi z) + x + y z, Dirichlet values on
    every side, CG1 on the finest level of a hierarchy over a 2^3 mesh."""
    h = mg.MeshHierarchy(2, 2, 2, levels)
    V = FunctionSpace(h[levels], 1)
    X = V.V.dof_coordinates()
    x, y, z = X[:, 0], X[:, 1], X[:, 2]
    s, c, pi = np.sin, np.cos, np.pi
    S = s(pi * x) * s(pi * y) * s(pi * z)
    ue = S + x + y * z
    grad = np.stack([pi * c(pi * x) * s(pi * y) * s(pi * z) + 1.0, pi * s(pi * x) * c(pi * y) * s(pi * z) + z,
                     pi * s(pi * x) * s(pi * y) * c(pi * z) + y], axis=1)
    bn = velocity(X)
    f = 3.0 * pi ** 2 * S + (bn * grad).sum(axis=1) + 0.5 * ue
    F = AdvectionDiffusion(V, op2.Dat(V.vector_dset(3), bn), 1.0, 0.5)
    rhs = OneFormAssembler(mass(V), V.dat(f)).assemble()
    bcs = [DirichletBC(V, V.dat(ue), [1, 2, 3, 4, "bottom", "top"])]
    n = 2 * 2 ** levels
    for pc in ("none", "jacobi", "mg"):
        u = V.dat()
        _lib.check(L.fdb_synchronize())
        t0 = time.perf_counter()
        its, hist = solve(F, rhs, u, bcs=bcs, hierarchy=h,
                          solver_parameters={"pc_type": pc, "ksp_rtol": 1e-8, "ksp_max_it": 5000})
        _lib.check(L.fdb_synchronize())
        wall = time.perf_counter() - t0
        print(json.dumps({"workload": f"advection-diffusion solve, CG1 on {n}^3, GMRES(30)", "n": n,
                          "pc_type": pc, "iterations": its, "wall_s": wall,
                          "err_max": float(np.abs(u.data_ro - ue).max()), "gpu": info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="1:128,2:128,3:128,4:128,1:256,2:256,3:256", help="degree:n,...")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--generic-steps", type=int, default=2)
    ap.add_argument("--solve-levels", default="3,4", help="hierarchy levels of the solves (2^3 base)")
    ap.add_argument("--no-solve", action="store_true")
    a = ap.parse_args()
    L = _lib.lib()
    info = card()
    for c in a.cases.split(","):
        p, n = (int(v) for v in c.split(":"))
        print(json.dumps(case(L, p, n, a, info)), flush=True)
    if not a.no_solve:
        for lv in a.solve_levels.split(","):
            solves(L, int(lv), info)


if __name__ == "__main__":
    main()
