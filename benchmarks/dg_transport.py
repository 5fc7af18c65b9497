#!/usr/bin/env python
"""Speed of upwind DG transport (DGTransport, FDB_FORM_DG_TRANSPORT) on DQ_p on one GPU, on warped extruded meshes
with device-resident u and a random vertex velocity b:

* ``cell``    -- the transport cell term -u*dot(b, grad v)*dx (csrc/dg_transport_hex.cu);
* ``dS_v``    -- the upwind flux over the vertical interior facets x all layers;
* ``dS_h``    -- the same over the horizontal interior facets;
* ``ds``      -- the outflow term over the exterior facets (vertical, bottom, top);
* ``action``  -- assemble(F, u=x) end to end (zeroing included), also as DoF/s;
* ``ssprk3``  -- one SSPRK3 step (three actions and the vector updates);
* ``generic`` -- the same transport terms through the generic wrapper builder (dg_transport_kernels), at
                 --generic-max cells per axis and below, with the same warm-up and step count; larger sizes print
                 "not measured".

Times are ms per call from CUDA events over ``--steps`` calls after ``--warmup`` (output accumulated, no zeroing
inside the window, except ``action``, ``ssprk3`` and ``generic``).  ``facet_GBps`` is the upwind facet kernels'
algorithmic bytes (values of both cells read once, the result added once, the '+' cell's vertices and b, maps and
facet numbers) over their time, beside the H100's 3.35 TB/s.  The card's name and power limit are read in the same
run.  One JSON line per case.

    python benchmarks/dg_transport.py
    python benchmarks/dg_transport.py --cases 1:64,2:64 --steps 20
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
from firedrake_b200.assemble import (DGTransport, FunctionSpace, OneFormAssembler, _boundary_groups,  # noqa: E402
                                     assemble_dg_transport_generic, ssprk3)
from firedrake_b200.utility_meshes import ExtrudedHexMesh                         # noqa: E402

HBM_TBPS = 3.35


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


def facet_bytes(groups, nd, sides, nlay_of):
    """Algorithmic bytes of one pass over facet groups: per facet, sides * (nd values read + nd results added) doubles,
    sides * 8 vertices (3 doubles), the map rows and the facet numbers once per column."""
    b = 0
    for fset, fmap, cmap, facet in groups:
        nf = fset.total_size * nlay_of(fset)
        b += nf * sides * (2 * nd * 8 + 8 * 3 * 8)
        b += fset.total_size * (sides * (nd + 8) * 4 + sides * 4)
    return b


def facet_bytes(groups, nd, sides, nlay_of):
    """Algorithmic bytes of one upwind pass over facet groups: per facet, sides * (nd values read + nd results
    added) doubles and the '+' cell's 8 vertices and b (6 doubles each); the map rows and facet numbers once per
    column."""
    b = 0
    for fset, fmap, cmap, facet in groups:
        nf = fset.total_size * nlay_of(fset)
        b += nf * (sides * 2 * nd * 8 + 8 * 6 * 8)
        b += fset.total_size * (sides * (nd + 8) * 4 + sides * 4)
    return b


def case(L, p, n, args, info):
    mesh = ExtrudedHexMesh(n, n, n, warp=0.05)
    V = FunctionSpace(mesh, p, family="DQ")
    nd = (p + 1) ** 3
    rng = np.random.default_rng(p)
    x = V.dat(rng.standard_normal(V.node_count))
    b = op2.Dat(op2.DataSet(V.vertex_set, 3), rng.standard_normal((mesh.coord_space.node_count, 3)))
    y = V.dat()
    y.zero()
    y.device_ptr
    F = DGTransport(V, b)
    terms = F.facet_terms()
    loops = terms.action_loops(y, x)
    nint = len(terms.interior)
    vert = [lp for lp, g in zip(loops[:nint], terms.interior) if g[0].layers == mesh.layers]
    horiz = [lp for lp, g in zip(loops[:nint], terms.interior) if g[0].layers != mesh.layers]
    ext = loops[nint:]
    cell = op2.Parloop(op2.GlobalKernel(F.kernel(1), [V.cell_node_map, V.coord_map], extruded=True),
                       V.cell_set, [y(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                                    x(op2.READ, V.cell_node_map)] + F.coefficient_args())
    run = lambda ls: (lambda: [lp() for lp in ls])
    rec = dict(info, p=p, n=n, dofs=V.node_count, cells=mesh.num_cells)
    rec["cell_ms"] = timed(L, cell, args.warmup, args.steps)
    rec["dS_v_ms"] = timed(L, run(vert), args.warmup, args.steps)
    rec["dS_h_ms"] = timed(L, run(horiz), args.warmup, args.steps)
    rec["ds_ms"] = timed(L, run(ext), args.warmup, args.steps)
    asm = OneFormAssembler(F, x)
    out = V.dat()
    rec["action_ms"] = timed(L, lambda: asm.assemble(out), args.warmup, args.steps)
    rec["action_dofs_per_s"] = V.node_count / (rec["action_ms"] * 1e-3)
    q = V.dat(np.ones(V.node_count))
    ssprk3(F, q, 1e-6, 1)
    # --steps steps in one call: the one-off set-up (M^-1, the operator) is amortised over them
    rec["ssprk3_step_ms"] = timed(L, lambda: ssprk3(F, q, 1e-6, args.steps), 0, 1) / args.steps
    nl = lambda fs: fs.layers - 1
    fb = facet_bytes(terms.interior, nd, 2, nl) + facet_bytes(_boundary_groups(V, "on_boundary"), nd, 1, nl)
    fms = rec["dS_v_ms"] + rec["dS_h_ms"] + rec["ds_ms"]
    rec["facet_GBps"] = fb / (fms * 1e-3) / 1e9
    rec["facet_fraction_of_hbm"] = rec["facet_GBps"] / (HBM_TBPS * 1e3)
    if n <= args.generic_max:
        gout = V.dat()
        rec["generic_ms"] = timed(L, lambda: assemble_dg_transport_generic(F, x, gout), args.warmup, args.steps)
        rec["generic_over_handwritten"] = rec["generic_ms"] / (rec["cell_ms"] + fms)
        yh = asm.assemble(V.dat()).data_ro
        yg = assemble_dg_transport_generic(F, x).data_ro
        rec["generic_max_rel_diff"] = float(np.abs(yh - yg).max() / np.abs(yg).max())
    else:
        rec["generic_ms"] = "not measured"
    print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="1:64,2:64,3:64,4:64,1:128,2:128,3:128,4:128")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--generic-max", type=int, default=64)
    args = ap.parse_args()
    L = _lib.init(0)
    info = card()
    for c in args.cases.split(","):
        p, n = (int(v) for v in c.split(":"))
        case(L, p, n, args, info)


if __name__ == "__main__":
    main()
