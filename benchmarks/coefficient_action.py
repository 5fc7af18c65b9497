#!/usr/bin/env python
"""Speed of the variable-coefficient action  inner(kappa*grad u, grad v)*dx  on one GPU, three ways on the
same warped extruded mesh and the same device-resident u and kappa:

* ``coef``     -- the hand-written slab-thread kernel in its coefficient mode (FDB_FORM_HELMHOLTZ_COEF);
* ``const``    -- the constant-coefficient Poisson action (FDB_FORM_HELMHOLTZ), the kernel it extends;
* ``generic``  -- ``variable_coefficient_kernel`` through the generic wrapper builder (one thread per
                  cell, NVRTC), the path the form took before.

One JSON line per (degree, n): ms per action (CUDA events over ``--steps`` launches after ``--warmup``,
output accumulated, no zeroing inside the window), DoF/s, the coef / const time ratio, the max-norm
difference between the coef and generic results relative to max|y| (one fresh action each), and the
card's name, power limit and maximum SM clock read in the same run.

    python benchmarks/coefficient_action.py                         # p = 2, 3 at 128^3 and 256^3, p = 4 at 128^3
    python benchmarks/coefficient_action.py --cases 3:128 --steps 5
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

from firedrake_b200 import _lib, op2                                              # noqa: E402
from firedrake_b200.assemble import FunctionSpace, interpolate, variable_coefficient_kernel  # noqa: E402
from firedrake_b200.utility_meshes import ExtrudedHexMesh                         # noqa: E402

KAPPA = "2.0 + sin(3.0 * x[0]) * x[1]"
U = "sin(2.0 * x[0]) * cos(x[1]) + x[2] * x[2]"


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
    y1, y2 = V.dat(), V.dat()
    for y in (y1, y2):
        y.zero()
        y.device_ptr
    base = [V.coordinates(op2.READ, V.coord_map), u(op2.READ, V.cell_node_map)]
    gk = lambda k: op2.GlobalKernel(k, [V.cell_node_map, V.coord_map], extruded=True)
    coef = op2.Parloop(gk(op2.Kernel("helmholtz_coef", degree=p)), V.cell_set,
                       [y1(op2.INC, V.cell_node_map)] + base + [kap(op2.READ, V.cell_node_map)])
    const = op2.Parloop(gk(op2.Kernel("helmholtz", degree=p)), V.cell_set, [y1(op2.INC, V.cell_node_map)] + base)
    vk = variable_coefficient_kernel(p)

    def generic():
        op2.par_loop(vk, V.cell_set, y2(op2.INC, V.cell_node_map), *base, kap(op2.READ, V.cell_node_map))

    t_coef = timed(L, coef, a.warmup, a.steps)
    t_const = timed(L, const, a.warmup, a.steps)
    t_gen = timed(L, generic, 1, a.generic_steps)
    # one fresh action each on the timed inputs
    for y in (y1, y2):
        y.zero()
        y.device_ptr
    coef()
    generic()
    h = np.empty(y1._data.size)
    _lib.check(L.fdb_memcpy_d2h(h.ctypes.data, y1.device_ptr, h.nbytes))
    scale = float(np.abs(h).max())
    _lib.check(L.fdb_vec_axpy(h.size, -1.0, y1.device_ptr, y2.device_ptr))             # y2 = generic - coef
    _lib.check(L.fdb_memcpy_d2h(h.ctypes.data, y2.device_ptr, h.nbytes))
    dofs = V.node_count
    return {"workload": f"inner(kappa*grad u, grad v)*dx action, CG{p} on {n}^3 warped extruded hexes",
            "degree": p, "n": n, "dofs": dofs,
            "ms": {"coef": t_coef, "const": t_const, "generic": t_gen},
            "dofs_per_s": {"coef": dofs / (t_coef * 1e-3), "const": dofs / (t_const * 1e-3),
                           "generic": dofs / (t_gen * 1e-3)},
            "coef_over_const": t_coef / t_const, "generic_over_coef": t_gen / t_coef,
            "rel_diff_coef_vs_generic": float(np.abs(h).max()) / scale,
            "steps": {"coef": a.steps, "const": a.steps, "generic": a.generic_steps}, "warmup": a.warmup,
            "gpu": info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="2:128,2:256,3:128,3:256,4:128", help="degree:n,...")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--generic-steps", type=int, default=3)
    a = ap.parse_args()
    L = _lib.lib()
    info = card()
    for c in a.cases.split(","):
        p, n = (int(v) for v in c.split(":"))
        print(json.dumps(case(L, p, n, a, info)), flush=True)


if __name__ == "__main__":
    main()
