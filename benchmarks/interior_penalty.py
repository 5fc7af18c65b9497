#!/usr/bin/env python
"""Speed of the symmetric interior penalty (SIPG) operator on DQ_p on one GPU, on warped extruded meshes with
device-resident u, eta = 3 (p+1)^2 and Nitsche conditions on the whole boundary:

* ``cell``   -- the cell term alpha*inner(grad u, grad v)*dx + beta*u*v*dx (FDB_FORM_HELMHOLTZ, GL tables);
* ``dS_v``   -- FDB_FORM_INTERIOR_PENALTY over the vertical interior facets x all layers;
* ``dS_h``   -- the same over the horizontal interior facets;
* ``ds``     -- FDB_FORM_DG_BOUNDARY (Nitsche) over the exterior facets (vertical, bottom, top);
* ``action`` -- assemble(F, u=x) end to end (zeroing included), also as DoF/s;
* ``generic``-- the facet terms through the generic wrapper builder (interior_penalty_kernels), at --generic-max
                cells per axis and below, with the same warm-up and step count; larger sizes print "not measured".

Times are ms per call from CUDA events over ``--steps`` calls after ``--warmup`` (output accumulated, no zeroing
inside the window, except ``action``).  ``facet_GBps`` is the facet kernels' algorithmic bytes (values of both cells
read once, the result added once, coordinates, maps and facet numbers) over their time, beside the H100's 3.35 TB/s.
The card's name and power limit are read in the same run.  One JSON line per case.

    python benchmarks/interior_penalty.py
    python benchmarks/interior_penalty.py --cases 1:64,2:64 --steps 20
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
from firedrake_b200.assemble import (Form, FunctionSpace, InteriorPenalty, OneFormAssembler,  # noqa: E402
                                     _boundary_groups, _dg_interior_groups, assemble_interior_penalty_generic)
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


def case(L, p, n, args, info):
    mesh = ExtrudedHexMesh(n, n, n, warp=0.05)
    V = FunctionSpace(mesh, p, family="DQ")
    nd = (p + 1) ** 3
    x = V.dat(np.random.default_rng(p).standard_normal(V.node_count))
    y = V.dat()
    y.zero()
    y.device_ptr
    F = InteriorPenalty(V, 1.0, 0.0, 3.0 * (p + 1) ** 2)
    terms = F.facet_terms()
    loops = terms.action_loops(y, x)
    nint = len(terms.interior)
    vert = [lp for lp, g in zip(loops[:nint], terms.interior) if g[0].layers == mesh.layers]
    horiz = [lp for lp, g in zip(loops[:nint], terms.interior) if g[0].layers != mesh.layers]
    ext = loops[nint:]
    cell = op2.Parloop(op2.GlobalKernel(Form(V, 1.0, 0.0).kernel(1), [V.cell_node_map, V.coord_map], extruded=True),
                       V.cell_set, [y(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                                    x(op2.READ, V.cell_node_map)])
    run = lambda ls: (lambda: [lp() for lp in ls])
    rec = dict(info, p=p, n=n, dofs=V.node_count, cells=mesh.num_cells, eta=F.eta)
    rec["cell_ms"] = timed(L, cell, args.warmup, args.steps)
    rec["dS_v_ms"] = timed(L, run(vert), args.warmup, args.steps)
    rec["dS_h_ms"] = timed(L, run(horiz), args.warmup, args.steps)
    rec["ds_ms"] = timed(L, run(ext), args.warmup, args.steps)
    asm = OneFormAssembler(F, x)
    out = V.dat()
    rec["action_ms"] = timed(L, lambda: asm.assemble(out), args.warmup, args.steps)
    rec["action_dofs_per_s"] = V.node_count / (rec["action_ms"] * 1e-3)
    nl = lambda fs: fs.layers - 1
    fb = facet_bytes(terms.interior, nd, 2, nl) + facet_bytes(_boundary_groups(V, "on_boundary"), nd, 1, nl)
    fms = rec["dS_v_ms"] + rec["dS_h_ms"] + rec["ds_ms"]
    rec["facet_GBps"] = fb / (fms * 1e-3) / 1e9
    rec["facet_fraction_of_hbm"] = rec["facet_GBps"] / (HBM_TBPS * 1e3)
    if n <= args.generic_max:
        gout = V.dat()
        rec["generic_facets_ms"] = timed(L, lambda: assemble_interior_penalty_generic(F, x, gout), args.warmup,
                                         args.steps)
        rec["generic_over_handwritten"] = rec["generic_facets_ms"] / fms
        yh = asm.assemble(V.dat()).data_ro - OneFormAssembler(Form(V, 1.0, 0.0), x).assemble().data_ro
        yg = assemble_interior_penalty_generic(F, x).data_ro
        rec["generic_max_rel_diff"] = float(np.abs(yh - yg).max() / np.abs(yg).max())
    else:
        rec["generic_facets_ms"] = "not measured"
    print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="1:64,2:64,3:64,4:64,1:128,2:128,3:128")
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
