#!/usr/bin/env python
"""Speed of nonlinear diffusion on one GPU: the residual and the Jacobian action of
alpha*inner(D(u)*grad u, grad v)*dx (D(s) = 1 + 0.1 s^2), against the coefficient action (kappa a field)
and the constant-coefficient action, on the same warped extruded mesh and device-resident vectors;
then one Newton solve of a manufactured problem.

Per (degree, n) one JSON line: ms per action (CUDA events over ``--steps`` launches after
``--warmup``, output accumulated, no zeroing inside the window), the ratios to the coefficient action,
and the Taylor figure max|J w - (R(u + h w) - R(u - h w)) / 2h| / max|J w| (h = 1e-4).  The solve line:
u* = cos(2 pi x) cos(2 pi y) cos(2 pi z) on the unit cube with natural conditions, CG3 on
``--solve-n``^3, Newton from u = 0 to snes_rtol 1e-8 with GMRES (ksp_rtol 1e-6) and pc_type jacobi
and mg; Newton and Krylov iterations and synchronised wall time per Newton step.  Every line carries
the card's name, power limit and maximum SM clock read in the same run.

    python benchmarks/nonlinear_diffusion.py                      # the cases of DESIGN.md section 4.6
    python benchmarks/nonlinear_diffusion.py --cases 3:128 --solve-n 0
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from coefficient_action import card, timed                                       # noqa: E402
from firedrake_b200 import _lib, op2                                              # noqa: E402
from firedrake_b200.assemble import FunctionSpace, interpolate                    # noqa: E402
from firedrake_b200.utility_meshes import ExtrudedHexMesh                         # noqa: E402

D = (1.0, 0.0, 0.1)
U = "sin(2.0 * x[0]) * cos(x[1]) + x[2] * x[2]"
W = "cos(3.0 * x[0]) + x[1] * x[2]"


def case(L, p, n, a, info):
    V = FunctionSpace(ExtrudedHexMesh(n, n, n, warp=0.05), p)
    u, w = interpolate(V, U), interpolate(V, W)
    kap = V.dat()
    op2.par_loop(op2.Kernel("static void dk(double *k, const double *u) { *k = 1.0 + 0.1 * u[0] * u[0]; }", "dk"),
                 V.node_set, kap(op2.WRITE), u(op2.READ))
    y = V.dat()
    y.zero()
    y.device_ptr
    X = V.coordinates(op2.READ, V.coord_map)
    m = V.cell_node_map
    gk = lambda k: op2.GlobalKernel(k, [V.cell_node_map, V.coord_map], extruded=True)
    loops = {
        "residual": op2.Parloop(gk(op2.Kernel("nonlinear_diffusion", degree=p, d=D)), V.cell_set,
                                [y(op2.INC, m), X, u(op2.READ, m)]),
        "jacobian": op2.Parloop(gk(op2.Kernel("nonlinear_diffusion_jacobian", degree=p, d=D)), V.cell_set,
                                [y(op2.INC, m), X, w(op2.READ, m), u(op2.READ, m)]),
        "coef": op2.Parloop(gk(op2.Kernel("helmholtz_coef", degree=p)), V.cell_set,
                            [y(op2.INC, m), X, u(op2.READ, m), kap(op2.READ, m)]),
        "const": op2.Parloop(gk(op2.Kernel("helmholtz", degree=p)), V.cell_set, [y(op2.INC, m), X, u(op2.READ, m)]),
    }
    ms = {k: timed(L, f, a.warmup, a.steps) for k, f in loops.items()}
    # the Taylor figure: fresh residuals at u +- h w and one Jacobian action
    from firedrake_b200.assemble import NonlinearDiffusion, assemble
    F = NonlinearDiffusion(V, 1.0, 0.0, D)
    h = 1e-4
    up, um = V.dat(), V.dat()
    u.copy(up)
    up.axpy(h, w)
    u.copy(um)
    um.axpy(-h, w)
    rp, rm, jw = assemble(F, u=up), assemble(F, u=um), assemble(F.jacobian(u), u=w)
    nn = rp._data.size
    _lib.check(L.fdb_vec_axpy(nn, -1.0, rm.device_ptr, rp.device_ptr))
    _lib.check(L.fdb_vec_scale(nn, 1.0 / (2 * h), rp.device_ptr))
    _lib.check(L.fdb_vec_axpy(nn, -1.0, jw.device_ptr, rp.device_ptr))            # rp = fd - J w
    buf = np.empty(nn)

    def absmax(d):
        _lib.check(L.fdb_memcpy_d2h(buf.ctypes.data, d.device_ptr, buf.nbytes))
        return float(np.abs(buf).max())
    taylor = absmax(rp) / absmax(jw)
    dofs = V.node_count
    return {"workload": f"nonlinear diffusion, D(u) = 1 + 0.1 u^2, CG{p} on {n}^3 warped extruded hexes",
            "degree": p, "n": n, "dofs": dofs, "ms": ms,
            "dofs_per_s": {k: dofs / (t * 1e-3) for k, t in ms.items()},
            "residual_over_coef": ms["residual"] / ms["coef"], "jacobian_over_coef": ms["jacobian"] / ms["coef"],
            "taylor_rel": taylor, "steps": a.steps, "warmup": a.warmup, "gpu": info}


def solve_case(L, n, pc, info):
    from firedrake_b200 import mg
    from firedrake_b200.assemble import NonlinearDiffusion, assemble, mass, solve_nonlinear
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_nonlinear_gpu import FSRC, USTAR
    p = 3
    h = mg.MeshHierarchy(n // 4, n // 4, n // 4, 2) if pc == "mg" else None
    V = FunctionSpace(h[2] if h is not None else ExtrudedHexMesh(n, n, n), p)
    F = NonlinearDiffusion(V, 1.0, 1.0, D)
    Lf = assemble(mass(V), u=interpolate(V, FSRC))
    ui = interpolate(V, USTAR)
    u = V.dat()
    u.zero()
    u.device_ptr
    _lib.check(L.fdb_synchronize())
    t0 = time.perf_counter()
    hist, kits = solve_nonlinear(F, Lf, u, hierarchy=h,
                                 solver_parameters={"pc_type": pc, "snes_rtol": 1e-8, "ksp_rtol": 1e-6})
    _lib.check(L.fdb_synchronize())
    t = time.perf_counter() - t0
    err = float(np.abs(u.data_ro - ui.data_ro).max())
    return {"workload": f"Newton solve of the manufactured problem, CG3 on {n}^3 unit cube", "pc_type": pc,
            "dofs": V.node_count, "newton_its": len(kits), "krylov_its": kits,
            "residual_history": hist, "s_per_newton_step": t / max(1, len(kits)), "s_total": t,
            "max_err_vs_interpolant": err, "gpu": info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="2:128,2:256,3:128,3:256,4:128", help="degree:n,...")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--solve-n", type=int, default=64, help="mesh of the Newton solve (0: skip)")
    a = ap.parse_args()
    L = _lib.lib()
    info = card()
    for c in filter(None, a.cases.split(",")):
        p, n = (int(v) for v in c.split(":"))
        print(json.dumps(case(L, p, n, a, info)), flush=True)
    if a.solve_n:
        for pc in ("jacobi", "mg"):
            print(json.dumps(solve_case(L, a.solve_n, pc, info)), flush=True)


if __name__ == "__main__":
    main()
