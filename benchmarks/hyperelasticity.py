#!/usr/bin/env python
"""Speed of the Neo-Hookean hyperelasticity residual and Jacobian action on one GPU, on the same warped
extruded mesh and the same device-resident vectors (3 components):

* ``residual``  -- R(u), the hand-written kernel (FDB_FORM_HYPERELASTICITY, csrc/elasticity_hex.cu);
* ``jacobian``  -- J(u) w, the hand-written kernel (FDB_FORM_HYPERELASTICITY_JACOBIAN);
* ``linear``    -- the linear elasticity action (FDB_FORM_ELASTICITY), the same kernel's linear mode;
* ``generic_residual``, ``generic_jacobian`` -- ``hyperelasticity_kernel`` through the generic wrapper
  builder (one thread per cell, NVRTC).

One JSON line per (degree, n): ms per call (CUDA events over ``--steps`` launches after ``--warmup``,
output accumulated, no zeroing inside the window), DoF/s counting 3 DoFs per node, the ratios to the
linear action and generic / hand-written, and the max-norm differences between the hand-written and
generic results relative to max|y| (one fresh call each).  Then one line per preconditioner for the
twisted-cube Newton solve of tests/test_hyperelastic_gpu.py (CG1, clamped bottom, 30 degree twist and 10 %
compression of the top in ``--increments`` load increments): Newton steps and GMRES iterations per step for
every increment and seconds, or the error that ended the solve.  Every line carries the card's name, power limit and maximum SM clock, read in
the same run.

    python benchmarks/hyperelasticity.py                    # the cases of DESIGN.md section 4.9
    python benchmarks/hyperelasticity.py --cases 3:64 --steps 5 --solve-n 16
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from firedrake_b200 import _lib, op2                                                   # noqa: E402
from firedrake_b200.assemble import FunctionSpace, hyperelasticity_kernel, interpolate  # noqa: E402
from firedrake_b200.utility_meshes import ExtrudedHexMesh                              # noqa: E402

from coefficient_action import card, timed                                           # noqa: E402

MU, LMBDA, BETA = 1.0, 1.5, 0.0
# a smooth displacement with det F > 0 on the unit cube, and a direction
U = ["0.1 * sin(2.0 * x[0]) * cos(x[1]) + 0.05 * x[2] * x[2]", "0.1 * x[0] * x[1] - 0.05 * cos(x[2])",
     "0.1 * sin(x[0] + 2.0 * x[2])"]
W = ["sin(2.0 * x[0]) * cos(x[1]) + x[2] * x[2]", "x[0] * x[1] - cos(x[2])", "sin(x[0] + 2.0 * x[2])"]


def _diff(L, a, b):
    """max|b - a| / max|a| of two device vectors (b is overwritten)."""
    h = np.empty(a._data.size)
    _lib.check(L.fdb_memcpy_d2h(h.ctypes.data, a.device_ptr, h.nbytes))
    scale = float(np.abs(h).max())
    _lib.check(L.fdb_vec_axpy(h.size, -1.0, a.device_ptr, b.device_ptr))
    _lib.check(L.fdb_memcpy_d2h(h.ctypes.data, b.device_ptr, h.nbytes))
    return float(np.abs(h).max()) / scale


def case(L, p, n, a, info):
    V = FunctionSpace(ExtrudedHexMesh(n, n, n, warp=0.05), p, 3)
    u, w = interpolate(V, U), interpolate(V, W)
    y1, y2 = V.dat(), V.dat()
    for y in (y1, y2):
        y.zero()
        y.device_ptr
    X = V.coordinates(op2.READ, V.coord_map)
    rd = lambda d: d(op2.READ, V.cell_node_map)
    gk = lambda name: op2.GlobalKernel(op2.Kernel(name, degree=p, mu=MU, lmbda=LMBDA, beta=BETA, cdim=3),
                                       [V.cell_node_map, V.coord_map], extruded=True)
    res = op2.Parloop(gk("hyperelasticity"), V.cell_set, [y1(op2.INC, V.cell_node_map), X, rd(u)])
    jac = op2.Parloop(gk("hyperelasticity_jacobian"), V.cell_set, [y1(op2.INC, V.cell_node_map), X, rd(w), rd(u)])
    lin = op2.Parloop(gk("elasticity"), V.cell_set, [y1(op2.INC, V.cell_node_map), X, rd(w)])
    kr, kj = hyperelasticity_kernel(p, MU, LMBDA, BETA), hyperelasticity_kernel(p, MU, LMBDA, BETA, jacobian=True)
    gres = lambda: op2.par_loop(kr, V.cell_set, y2(op2.INC, V.cell_node_map), X, rd(u))
    gjac = lambda: op2.par_loop(kj, V.cell_set, y2(op2.INC, V.cell_node_map), X, rd(w), rd(u))
    t = {"residual": timed(L, res, a.warmup, a.steps), "jacobian": timed(L, jac, a.warmup, a.steps),
         "linear": timed(L, lin, a.warmup, a.steps),
         "generic_residual": timed(L, gres, 1, a.generic_steps),
         "generic_jacobian": timed(L, gjac, 1, a.generic_steps)}
    diff = {}
    for name, mine, gen in (("residual", res, gres), ("jacobian", jac, gjac)):
        for y in (y1, y2):
            y.zero()
            y.device_ptr
        mine()
        gen()
        diff[name] = _diff(L, y1, y2)
    dofs = 3 * V.node_count
    return {"workload": f"hyperelasticity residual and Jacobian action, vector CG{p} on {n}^3 warped extruded hexes",
            "degree": p, "n": n, "dofs": dofs, "ms": t,
            "dofs_per_s": {k: dofs / (v * 1e-3) for k, v in t.items()},
            "residual_over_linear": t["residual"] / t["linear"], "jacobian_over_linear": t["jacobian"] / t["linear"],
            "generic_over_residual": t["generic_residual"] / t["residual"],
            "generic_over_jacobian": t["generic_jacobian"] / t["jacobian"],
            "rel_diff_vs_generic": diff,
            "steps": {"hand-written": a.steps, "generic": a.generic_steps}, "warmup": a.warmup, "gpu": info}


def solve_case(L, n, pc, increments, info):
    import test_hyperelastic_gpu as tg
    from firedrake_b200 import mg
    from firedrake_b200.assemble import ConvergenceError
    refinements = int(np.log2(n // 2))
    h = mg.MeshHierarchy(2, 2, 2, refinements) if pc == "mg" else None
    out = {"workload": f"hyperelasticity Newton solve, twisted cube, CG1 on {n}^3, {increments} load increments, "
                       f"pc_type {pc}" + (f" ({refinements + 1} levels from 2^3)" if pc == "mg" else ""),
           "n": n, "pc_type": pc, "ksp_rtol": 1e-6, "snes_rtol": 1e-11, "gpu": info}
    _lib.check(L.fdb_synchronize())
    t0 = time.perf_counter()
    try:
        V, u, hists, kits = tg.twisted_cube(n, 1, pc, h, ksp_rtol=1e-6, steps=increments)
    except ConvergenceError as e:
        out.update(diverged=str(e), seconds=time.perf_counter() - t0)
        return out
    _lib.check(L.fdb_synchronize())
    out.update(dofs=3 * V.node_count, newton_steps=[len(k) for k in kits], gmres_iterations=kits,
               final_residual_ratio=[hh[-1] / hh[0] for hh in hists], seconds=time.perf_counter() - t0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="1:256,2:128,2:256,3:128,4:64,4:128", help="degree:n,...")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--generic-steps", type=int, default=2)
    ap.add_argument("--solve-n", type=int, default=32, help="0: no solves")
    # full-step Newton needs the top's jump per increment below the layer height (4 increments suffice on 4^3
    # and invert elements on 32^3)
    ap.add_argument("--increments", type=int, default=16)
    a = ap.parse_args()
    L = _lib.lib()
    info = card()
    for c in a.cases.split(","):
        p, n = (int(v) for v in c.split(":"))
        print(json.dumps(case(L, p, n, a, info)), flush=True)
    if a.solve_n:
        for pc in ("mg", "jacobi", "none"):
            print(json.dumps(solve_case(L, a.solve_n, pc, a.increments, info)), flush=True)


if __name__ == "__main__":
    main()
