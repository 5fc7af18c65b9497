"""Host logic of DGTransport on the CPU, against the recording stand-in for the engine of tests/test_dg_host_mock.py:
the loops, descriptors, argument and map counts and layer ranges of the action, the diagonal, inflow_load and
ssprk3, with and without the Helmholtz and interior penalty parts."""
import numpy as np
import pytest

import _mock_engine as me
from firedrake_b200 import _lib, op2
from test_dg_host_mock import RecordingEngine, _dg_space, _facet_counts

F_TR, F_H, F_IP, F_DB = _lib.FORM_DG_TRANSPORT, _lib.FORM_HELMHOLTZ, _lib.FORM_INTERIOR_PENALTY, _lib.FORM_DG_BOUNDARY
CELL, EXT, INT = _lib.INTEGRAL_CELL, _lib.INTEGRAL_EXTERIOR_FACET, _lib.INTEGRAL_INTERIOR_FACET


class _Recorder(RecordingEngine):
    """Also records the generated-wrapper calls (ssprk3's reciprocal) as ('jit',)."""

    def fdb_wrapper_create(self, desc, out):
        self._next += 1
        self._index[self._next] = "jit"
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        if self._index.get(me._addr(h)) == "jit":
            self.calls.append(("jit",))
            return 0
        return super().fdb_kernel_call(h, ca)


class recording(me.install):
    def __init__(self):
        self.engine = _Recorder()


def _velocity(V, mesh):
    return op2.Dat(op2.DataSet(V.vertex_set, 3), np.ones((mesh.coord_space.node_count, 3)))


def _kinds(creates, calls):
    return [(creates[c[0]][0], creates[c[0]][3]) for c in calls if c[0] != "jit"]


@pytest.mark.parametrize("parts", ["transport", "reaction", "diffusion"])
def test_action_loops(parts):
    """The transport cell loop [y, coords, u, b], the Helmholtz cell loop (alpha or beta nonzero), InteriorPenalty's
    dS_v, dS_h and Nitsche loops (alpha > 0), the upwind dS_v and dS_h loops [y, coords, u, b, facets] and the outflow
    loops (c_out, c_in) = (1, 0) on the vertical and bottom/top boundary facets."""
    from firedrake_b200.assemble import DGTransport, assemble
    mesh, V = _dg_space()
    nd = 27
    nv, nh, ne = _facet_counts(mesh)
    kw = {"transport": {}, "reaction": dict(beta=0.5), "diffusion": dict(beta=0.5, alpha=1.3, eta=27.0,
                                                                          weak_bcs="on_boundary")}[parts]
    with recording() as eng:
        F = DGTransport(V, _velocity(V, mesh), **kw)
        assemble(F, u=V.dat(np.ones(V.node_count)))
        creates, calls = list(eng.creates), list(eng.calls)
    want = [(F_TR, CELL)]
    if parts != "transport":
        want += [(F_H, CELL)]
    if parts == "diffusion":
        want += [(F_IP, INT)] * 2 + [(F_DB, EXT)] * 2
    want += [(F_TR, INT)] * 2 + [(F_TR, EXT)] * 2
    assert _kinds(creates, calls) == want
    cell = calls[0]
    assert creates[cell[0]][1:3] == (1, _lib.CELL_HEX_EXTRUDED) and creates[cell[0]][10] == 0
    assert abs(creates[cell[0]][14] - 1.0) < 1e-12                   # GL: B = I
    assert cell[1:3] == (4, 2) and cell[6] == (0, mesh.layers) and cell[7] == (V.cell_set.size * nd, V.cell_set.size * 8)
    if parts != "transport":
        h = creates[calls[1][0]]
        assert h[8:10] == (kw.get("alpha", 0.0), 0.5) and calls[1][1:3] == (3, 2)
    dsv, dsh, vert, horiz = calls[-4:]
    for c, n, lay in ((dsv, nv, mesh.layers), (dsh, nh, mesh.nz)):
        assert c[1:5] == (5, 2, 0, n) and c[6] == (0, lay) and c[7] == (n * 2 * nd, n * 16)
    for c, n, lay in ((vert, ne, mesh.layers), (horiz, 2 * nh, 2)):
        cr = creates[c[0]]
        assert cr[12:14] == (1.0, 0.0) and cr[10] == 0
        assert c[1:5] == (5, 2, 0, n) and c[6] == (0, lay) and c[7] == (n * nd, n * 8)


def test_diagonal_and_inflow_load():
    """getDiagonal: the transport cell diagonal [d, coords, b], the Helmholtz diagonal (beta), then the upwind and
    outflow diagonals [d, coords, b, facets]; inflow_load: the exterior action with (c_out, c_in) = (0, -1)."""
    from firedrake_b200.assemble import DGTransport, ImplicitMatrixContext, inflow_load
    mesh, V = _dg_space()
    with recording() as eng:
        F = DGTransport(V, _velocity(V, mesh), beta=0.5)
        ImplicitMatrixContext(F).getDiagonal(V.dat())
        n_diag = len(eng.calls)
        inflow_load(F, V.dat(np.ones(V.node_count)))
        creates, calls = list(eng.creates), list(eng.calls)
    diag = calls[:n_diag]
    assert _kinds(creates, diag) == [(F_TR, CELL), (F_H, CELL), (F_TR, INT), (F_TR, INT), (F_TR, EXT), (F_TR, EXT)]
    assert all(creates[c[0]][10] == 1 for c in diag)
    assert diag[0][1:3] == (3, 2) and diag[1][1:3] == (2, 2) and all(c[1:3] == (4, 2) for c in diag[2:])
    load = calls[n_diag:]
    assert _kinds(creates, load) == [(F_TR, EXT)] * 2
    assert all(creates[c[0]][12:14] == (0.0, -1.0) and creates[c[0]][10] == 0 and c[1] == 5 for c in load)


def test_dq4_jacobi_only_with_the_helmholtz_part():
    """Pure transport takes Jacobi at DQ4 (its diagonal covers p = 1..4); with beta the Helmholtz diagonal stops at
    DQ3 and solve refuses before anything is assembled."""
    from firedrake_b200.assemble import DGTransport, ImplicitMatrixContext, solve
    mesh, V = _dg_space(4)
    with recording() as eng:
        b = _velocity(V, mesh)
        ImplicitMatrixContext(DGTransport(V, b)).getDiagonal(V.dat())
        n = len(eng.calls)
        with pytest.raises(NotImplementedError, match="degrees 1..3"):
            solve(DGTransport(V, b, beta=1.0), V.dat(), V.dat(), solver_parameters={"pc_type": "jacobi"})
        assert len(eng.calls) == n
        with pytest.raises(ValueError, match="ksp_type cg needs a symmetric operator"):
            solve(DGTransport(V, b), V.dat(), V.dat(), solver_parameters={"ksp_type": "cg"})
        with pytest.raises(NotImplementedError, match="no DQ multigrid"):
            solve(DGTransport(V, b), V.dat(), V.dat(), solver_parameters={"pc_type": "mg"})
        with pytest.raises(NotImplementedError, match="DG transport"):
            ImplicitMatrixContext(DGTransport(V, b)).multTranspose(V.dat(), V.dat())


@pytest.mark.parametrize("steps", [1, 3])
def test_ssprk3_three_actions_per_step(steps):
    """ssprk3: the mass action on ones once (M^-1 by its reciprocal), then three transport actions per step."""
    from firedrake_b200.assemble import DGTransport, ssprk3
    mesh, V = _dg_space()
    with recording() as eng:
        F = DGTransport(V, _velocity(V, mesh))
        q = V.dat(np.ones(V.node_count))
        ssprk3(F, q, 1e-3, steps, load=V.dat())
        creates, calls = list(eng.creates), list(eng.calls)
    kinds = _kinds(creates, calls)
    assert kinds[0] == (F_H, CELL) and creates[calls[0][0]][8:10] == (0.0, 1.0)
    assert kinds.count((F_TR, CELL)) == 3 * steps
    assert kinds[1:] == [(F_TR, CELL), (F_TR, INT), (F_TR, INT), (F_TR, EXT), (F_TR, EXT)] * (3 * steps)
