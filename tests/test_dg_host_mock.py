"""Host logic of the DG forms on the CPU, against a recording stand-in for the engine (tests/_mock_engine.py with
fdb_kernel_create / fdb_kernel_call replaced by recorders): every descriptor and every call the Python layer hands
to the engine.  The CG paths that the DG change touches (Form.kernel, the Helmholtz diagonal kernel of getDiagonal,
the facet hooks of OneFormAssembler and getDiagonal) must make exactly the calls they made before DQ spaces existed,
pinned in CG_CALLS; InteriorPenalty must issue its cell loop, its interior-facet loops (dS_v, dS_h) and its
DG_BOUNDARY loops, with the documented coefficients, for the action, the diagonal and the loads."""
import numpy as np
import pytest

import _mock_engine as me
from firedrake_b200 import _lib
from firedrake_b200.utility_meshes import ExtrudedHexMesh


class RecordingEngine(me.MockEngine):
    """Records (descriptor fields) per fdb_kernel_create and (kernel index, argument and map counts, range, location,
    layers, map sizes in ints) per fdb_kernel_call; computes nothing."""

    def __init__(self):
        super().__init__(None)
        self.creates, self.calls, self._index = [], [], {}

    def fdb_kernel_create(self, desc, out):
        d = me._obj(desc)
        self.creates.append((int(d.form), int(d.rank), int(d.cell), int(d.integral), int(d.degree), int(d.nq),
                             int(d.cdim), int(d.scatter), round(float(d.alpha), 12), round(float(d.beta), 12),
                             int(d.diagonal), int(d.affine_cells), round(float(d.dcoef[0]), 12),
                             round(float(d.dcoef[1]), 12), round(float(d.B[0]), 9)))
        self._next += 1
        self._index[self._next] = len(self.creates) - 1
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        a = me._obj(ca)
        layers = (int(a.layers[0]), int(a.layers[1])) if me._addr(a.layers) else None
        sizes = tuple(len(self.bufs[a.maps[i]]) // 4 if a.maps[i] in self.bufs else None for i in range(a.nmaps))
        self.calls.append((self._index[me._addr(h)], int(a.nargs), int(a.nmaps), int(a.start), int(a.end),
                           int(a.location), layers, sizes))
        return 0


class recording(me.install):
    def __init__(self):
        self.engine = RecordingEngine()


def cg_engine_calls():
    """The engine calls of the CG paths the DG change touches, as (creates, calls)."""
    from firedrake_b200.assemble import (BoundaryMass, Form, FunctionSpace, ImplicitMatrixContext, OneFormAssembler,
                                         assemble, mass, poisson)
    out = []
    with recording() as eng:
        mesh = ExtrudedHexMesh(3, 2, 2, warp=0.05)
        V = FunctionSpace(mesh, 2)
        x = V.dat(np.ones(V.node_count))
        assemble(Form(V, 1.3, 0.7), u=x)
        assemble(mass(V), u=x)
        assemble(poisson(V), u=x)
        ImplicitMatrixContext(Form(V, 1.3, 0.7)).getDiagonal(V.dat())
        OneFormAssembler(Form(V, 1.0, 0.0, ds=((2.0, "on_boundary"),)), x, scatter="coloured").assemble()
        ImplicitMatrixContext(Form(V, 1.0, 0.0, ds=((2.0, "top"),))).getDiagonal(V.dat())
        assemble(BoundaryMass(V, 1.5, (1, "bottom")), u=x)
        ImplicitMatrixContext(BoundaryMass(V, 1.5, 3)).getDiagonal(V.dat())
        box = ExtrudedHexMesh(2, 2, 2)                     # parallelepipeds: the affine variant
        for p in (1, 3):
            W = FunctionSpace(box, p)
            assemble(poisson(W), u=W.dat(np.ones(W.node_count)))
            ImplicitMatrixContext(mass(W)).getDiagonal(W.dat())
        Vv = FunctionSpace(mesh, 2, 3)
        assemble(Form(Vv, 1.0, 1.0), u=Vv.dat(np.ones((Vv.node_count, 3))))
        import gc
        gc.collect()
        out = (list(eng.creates), list(eng.calls))
    return out


# cg_engine_calls() run on the parent commit, the last one before DQ spaces: (creates, calls)
CG_CALLS = \
    ([(1, 1, 1, 0, 2, 3, 1, 0, 1.3, 0.7, 0, 0, 1.0, 0.0, 0.687298335),
      (1, 1, 1, 0, 2, 3, 1, 0, 0.0, 1.0, 0, 0, 1.0, 0.0, 0.687298335),
      (1, 1, 1, 0, 2, 3, 1, 0, 1.0, 0.0, 0, 0, 1.0, 0.0, 0.687298335),
      (1, 1, 1, 0, 2, 3, 1, 0, 1.3, 0.7, 1, 0, 1.0, 0.0, 0.687298335),
      (1, 1, 1, 0, 2, 3, 1, 1, 1.0, 0.0, 0, 0, 1.0, 0.0, 0.687298335),
      (13, 1, 1, 1, 2, 3, 1, 1, 2.0, 0.0, 0, 0, 1.0, 0.0, 0.687298335),
      (13, 1, 1, 1, 2, 3, 1, 1, 2.0, 0.0, 0, 0, 1.0, 0.0, 0.687298335),
      (1, 1, 1, 0, 2, 3, 1, 0, 1.0, 0.0, 1, 0, 1.0, 0.0, 0.687298335),
      (13, 1, 1, 1, 2, 3, 1, 0, 2.0, 0.0, 1, 0, 1.0, 0.0, 0.687298335),
      (13, 1, 1, 1, 2, 3, 1, 0, 1.5, 0.0, 0, 0, 1.0, 0.0, 0.687298335),
      (13, 1, 1, 1, 2, 3, 1, 0, 1.5, 0.0, 0, 0, 1.0, 0.0, 0.687298335),
      (13, 1, 1, 1, 2, 3, 1, 0, 1.5, 0.0, 1, 0, 1.0, 0.0, 0.687298335),
      (1, 1, 1, 0, 1, 2, 1, 0, 1.0, 0.0, 0, 1, 1.0, 0.0, 0.788675135),
      (1, 1, 1, 0, 1, 2, 1, 0, 0.0, 1.0, 1, 0, 1.0, 0.0, 0.788675135),
      (1, 1, 1, 0, 3, 4, 1, 0, 1.0, 0.0, 0, 1, 1.0, 0.0, 0.629943166),
      (1, 1, 1, 0, 3, 4, 1, 0, 0.0, 1.0, 1, 0, 1.0, 0.0, 0.629943166),
      (1, 1, 1, 0, 2, 3, 3, 0, 1.0, 1.0, 0, 0, 1.0, 0.0, 0.687298335)],
     [(0, 3, 2, 0, 6, 1, (0, 3), (162, 48)), (1, 3, 2, 0, 6, 1, (0, 3), (162, 48)),
      (2, 3, 2, 0, 6, 1, (0, 3), (162, 48)), (3, 2, 2, 0, 6, 1, (0, 3), (162, 48)),
      (4, 3, 2, 0, 6, 1, (0, 3), (162, 48)), (5, 4, 2, 0, 10, 1, (0, 3), (270, 80)),
      (6, 4, 2, 0, 12, 1, (0, 2), (324, 96)), (7, 2, 2, 0, 6, 1, (0, 3), (162, 48)),
      (8, 3, 2, 0, 6, 1, (0, 2), (162, 48)), (9, 4, 2, 0, 2, 1, (0, 3), (54, 16)),
      (10, 4, 2, 0, 6, 1, (0, 2), (162, 48)), (11, 3, 2, 0, 3, 1, (0, 3), (81, 24)),
      (12, 3, 2, 0, 4, 1, (0, 3), (32, 32)), (13, 2, 2, 0, 4, 1, (0, 3), (32, 32)),
      (14, 3, 2, 0, 4, 1, (0, 3), (256, 32)), (15, 2, 2, 0, 4, 1, (0, 3), (256, 32)),
      (16, 3, 2, 0, 6, 1, (0, 3), (162, 48))])


def test_cg_forms_make_the_same_engine_calls():
    creates, calls = cg_engine_calls()
    assert creates == CG_CALLS[0]
    assert calls == CG_CALLS[1]


def _dg_space(p=2):
    from firedrake_b200.assemble import FunctionSpace
    mesh = ExtrudedHexMesh(3, 2, 3, warp=0.05)
    return mesh, FunctionSpace(mesh, p, family="DQ")


def _facet_counts(mesh):
    nx, ny, nz = mesh.nx, mesh.ny, mesh.nz
    nv = (nx - 1) * ny + nx * (ny - 1)
    ext = 2 * ny + 2 * nx
    return nv, nx * ny, ext


@pytest.mark.parametrize("weak", ["on_boundary", ()])
def test_interior_penalty_action_loops(weak):
    """assemble(F, u=x): the cell loop (Helmholtz with the GL tables), then dS_v (all layers) and dS_h (nz - 1 facet
    layers) with (alpha, eta), then the Nitsche loops (0, alpha eta, alpha, alpha) on the vertical and the bottom/top
    facets of weak_bcs."""
    from firedrake_b200.assemble import InteriorPenalty, assemble
    mesh, V = _dg_space()
    nd = 27
    nv, nh, ne = _facet_counts(mesh)
    with recording() as eng:
        assemble(InteriorPenalty(V, 1.3, 0.2, 27.0, weak_bcs=weak), u=V.dat(np.ones(V.node_count)))
        creates, calls = list(eng.creates), list(eng.calls)
    kinds = [(creates[c[0]][0], creates[c[0]][3]) for c in calls]
    want = [(_lib.FORM_HELMHOLTZ, _lib.INTEGRAL_CELL), (_lib.FORM_INTERIOR_PENALTY, _lib.INTEGRAL_INTERIOR_FACET),
            (_lib.FORM_INTERIOR_PENALTY, _lib.INTEGRAL_INTERIOR_FACET)]
    if weak:
        want += [(_lib.FORM_DG_BOUNDARY, _lib.INTEGRAL_EXTERIOR_FACET)] * 2
    assert kinds == want
    cell, dsv, dsh = calls[:3]
    assert creates[cell[0]][8:11] == (1.3, 0.2, 0) and abs(creates[cell[0]][14] - 1.0) < 1e-12   # GL: B = I
    assert cell[1:3] == (3, 2) and cell[6] == (0, mesh.layers)
    for c, n, lay in ((dsv, nv, mesh.layers), (dsh, nh, mesh.nz)):
        cr = creates[c[0]]
        assert cr[8:11] == (1.3, 27.0, 0) and cr[5] == 3 and cr[6] == 1
        assert c[1:5] == (4, 2, 0, n) and c[6] == (0, lay)
        assert c[7] == (n * 2 * nd, n * 16)                     # '+' row then '-' row; 8 + 8 vertices
    if weak:
        vert, horiz = calls[3:]
        for c, n, lay in ((vert, ne, mesh.layers), (horiz, 2 * nh, 2)):
            cr = creates[c[0]]
            assert cr[8:10] == (1.3, round(1.3 * 27.0, 12)) and cr[12:14] == (0.0, 1.3) and cr[10] == 0
            assert c[1:5] == (4, 2, 0, n) and c[6] == (0, lay) and c[7] == (n * nd, n * 8)


def test_interior_penalty_diagonal_and_loads():
    """getDiagonal: the Helmholtz diagonal, then the diagonal kernels of every facet group; nitsche_load and
    dg_flux_load: one DG_BOUNDARY action loop per facet group of their sub-domains, with (0, alpha eta, alpha, 0)
    and (1, 0, 0, 0)."""
    from firedrake_b200.assemble import ImplicitMatrixContext, InteriorPenalty, dg_flux_load, nitsche_load
    mesh, V = _dg_space()
    F = InteriorPenalty(V, 0.5, 0.0, 27.0, weak_bcs=(2, "top"))
    with recording() as eng:
        ImplicitMatrixContext(F).getDiagonal(V.dat())
        n_diag = len(eng.calls)
        g = V.dat(np.ones(V.node_count))
        nitsche_load(F, g)
        n_nitsche = len(eng.calls)
        dg_flux_load(V, g, "bottom")
        creates, calls = list(eng.creates), list(eng.calls)
    diag = [creates[c[0]] for c in calls[:n_diag]]
    assert [(d[0], d[10], d[1]) for d in diag] == [(_lib.FORM_HELMHOLTZ, 1, 1)] + \
        [(_lib.FORM_INTERIOR_PENALTY, 1, 1)] * 2 + [(_lib.FORM_DG_BOUNDARY, 1, 1)] * 2
    assert [c[1] for c in calls[:n_diag]] == [2, 3, 3, 3, 3]     # [d, coords] / [d, coords, facets]
    nit = [creates[c[0]] for c in calls[n_diag:n_nitsche]]
    assert len(nit) == 2 and all(d[0] == _lib.FORM_DG_BOUNDARY and d[10] == 0 for d in nit)
    assert all((d[8], d[9], d[12], d[13]) == (0.0, 13.5, 0.0, 0.5) for d in nit)
    flux = [creates[c[0]] for c in calls[n_nitsche:]]
    assert len(flux) == 1 and (flux[0][8], flux[0][9], flux[0][12], flux[0][13]) == (0.0, 0.0, 1.0, 0.0)
    assert calls[-1][6] == (0, 2)                            # "bottom": one cell layer


def test_refusals_before_the_engine():
    """DQ4's cell diagonal, multigrid and a V-cycle on a DQ form refuse before any kernel is created."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import ImplicitMatrixContext, InteriorPenalty, solve
    mesh, V = _dg_space(4)
    F = InteriorPenalty(V, 1.0, 0.0, 75.0)
    with recording() as eng:
        with pytest.raises(NotImplementedError, match="diagonal of the DQ4 cell term"):
            ImplicitMatrixContext(F).getDiagonal(V.dat())
        with pytest.raises(NotImplementedError, match="use pc_type 'none' on DQ4"):
            solve(F, V.dat(), V.dat(), solver_parameters={"pc_type": "jacobi"})
        h = mg.MeshHierarchy(2, 2, 2, 1)
        _, W = _dg_space(1)
        with pytest.raises(NotImplementedError, match="VCycle does not take DQ spaces"):
            mg.VCycle(h, 1, lambda V_: InteriorPenalty(W, 1.0, 0.0, 12.0))
        assert not [c for c in eng.creates if c[0] != _lib.FORM_HELMHOLTZ or c[10] == 1]
