"""Host logic of Stokes flow on the CPU: a mock engine that emulates FDB_FORM_STOKES through the NumPy oracle
(tests/_stokes_oracle.py) runs the Python layers -- the MixedDat assembler, the matrix-free operator with
velocity conditions, the lifting, the constant-pressure nullspace, GMRES over MixedDats with the diagonal
Schur fieldsplit -- against scipy, and every refusal of the Python layer.  The device code itself is what
`-m gpu` checks (tests/test_stokes_gpu.py)."""
import numpy as np
import pytest

import _mock_engine as me
import _stokes_oracle as so
import test_coefficient_host_mock as cm
import test_stokes_gpu as tg
from firedrake_b200 import _lib
from firedrake_b200.fiat_lite import interval_element


class StokesMockEngine(cm.CoefMockEngine):
    """CoefMockEngine plus the Stokes action, extruded and native hexes, device location."""

    def fdb_kernel_create_mixed(self, desc, space2, out):
        d, s2 = me._obj(desc), me._obj(space2)
        if d.form != _lib.FORM_STOKES:
            return self._fail("mock engine: only stokes is a form on two spaces")
        if d.cell not in (_lib.CELL_HEX_EXTRUDED, _lib.CELL_HEX) or d.cdim != 3 or d.rank != 1 or d.diagonal:
            return self._fail("mock engine: stokes is a rank-1 action on a 3-component hex space")
        p = d.degree
        ext = d.cell == _lib.CELL_HEX_EXTRUDED
        n, n2 = (p + 1) ** 3, p ** 3
        self._next += 1
        self.kernels[self._next] = dict(
            kind="stokes", degree=p, mu=d.alpha, beta=d.beta, extruded=ext,
            off0=np.array(d.offset0[:n] if ext else [0] * n, dtype=np.int32),
            off1=np.array(d.offset1[:8] if ext else [0] * 8, dtype=np.int32),
            off2=np.array(s2.offset[:n2] if ext else [0] * n2, dtype=np.int32))
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        k = self.kernels[me._addr(h)]
        if k["kind"] != "stokes":
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        self.launches += 1
        if a.nargs != 5 or a.nmaps != 3 or a.location != _lib.LOC_DEVICE:
            return self._fail("mock engine: stokes action expects 5 device args (y, coords, x, y_p, p) and 3 maps")
        p = k["degree"]
        nlay = a.layers[1] - 1 if k["extruded"] else 1
        ar0, ar2 = (p + 1) ** 3, p ** 3
        map0 = me._view(a.maps[0], a.end * ar0, np.int32).reshape(a.end, ar0)
        map1 = me._view(a.maps[1], a.end * 8, np.int32).reshape(a.end, 8)
        map2 = me._view(a.maps[2], a.end * ar2, np.int32).reshape(a.end, ar2)
        cols = np.arange(a.start, a.end)
        top = lambda m, o: int(m.max() + o.max() * (nlay - 1)) + 1
        nvert, nnode, nq = top(map1, k["off1"]), top(map0, k["off0"]), top(map2, k["off2"])
        coords = me._view(a.args[1], nvert * 3)
        geo = (map0[cols], k["off0"], map1[cols], k["off1"], nlay)
        yu, yp = so.action(interval_element(p), coords, me._view(a.args[2], 3 * nnode).copy(),
                           me._view(a.args[4], nq).copy(), geo, (map2[cols], k["off2"]), k["mu"], k["beta"])
        me._view(a.args[0], 3 * nnode)[:] += yu
        me._view(a.args[3], nq)[:] += yp
        return 0


class install(me.install):
    def __init__(self, oracle):
        self.engine = StokesMockEngine(oracle)


@pytest.fixture()
def mock(oracle):
    with install(oracle) as eng:
        yield eng


def test_matfree_mult_host_logic(mock):
    tg.test_matfree_mult_with_velocity_bcs_matches_oracle(mock)


def _reference(mesh, V, Q, bcs, g):
    """scipy's solution of the oracle's constrained system with one pressure pinned, mean removed."""
    import scipy.sparse as sps
    import scipy.sparse.linalg as spla
    geo = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    K = so.global_matrix(interval_element(V.degree), mesh.coordinates, geo, (Q.V.cell_node_map, Q.V.offset),
                         V.node_count, Q.node_count, 1.0)
    bd = so.velocity_dofs(np.unique(np.concatenate([bc.nodes for bc in bcs])))
    nv = 3 * V.node_count
    gfull = np.concatenate([g.ravel(), np.zeros(Q.node_count)])
    rhs = -(K @ gfull)
    rhs[bd] = 0.0
    rhs[nv] = 0.0
    x = spla.spsolve(sps.csc_matrix(so.constrained(K, np.concatenate([bd, [nv]]))), rhs) + gfull
    return K, x[:nv], x[nv:] - x[nv:].mean()


@pytest.mark.parametrize("pc0", ["jacobi", "mg"])
def test_fieldsplit_gmres_matches_scipy(mock, pc0):
    """The lid-driven cavity on 4^3 (Q2-Q1): GMRES with the diagonal Schur fieldsplit and the constant
    nullspace gives scipy's velocity and, modulo a constant, its pressure; the pressure comes back with
    zero mean."""
    from firedrake_b200.assemble import solve
    from firedrake_b200.mg import MeshHierarchy
    mesh, V, Q, F, bcs = tg._cavity(4)
    g = np.zeros((V.node_count, 3))
    g[bcs[1].nodes, 0] = 1.0
    up = F.dat()
    its, hist = solve(F, F.dat(), up, bcs, tg._fieldsplit(pc0),
                      hierarchy=MeshHierarchy(2, 2, 2, 1) if pc0 == "mg" else None, nullspace="constant")
    assert hist[-1] <= 1e-12 * hist[0]
    _, u_ref, p_ref = _reference(mesh, V, Q, bcs, g)
    assert np.abs(up[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    p = up[1].data_ro
    assert abs(p.mean()) < 1e-12 * np.abs(p_ref).max()
    assert np.abs(p - p_ref).max() < 1e-7 * np.abs(p_ref).max()


def test_lifting_fills_the_pressure_rows(mock):
    """The right-hand side of the lifted system is L - A (g, 0): its pressure rows are -q div g, nonzero for
    a lid velocity (x (1 - x), y (1 - y), 0) (tangential on the side walls, so the system stays consistent,
    but not divergence-free), and solve's solution is the one scipy gets from the same lifting."""
    from firedrake_b200.assemble import DirichletBC, assemble, solve
    mesh, V, Q, F, bcs = tg._cavity(3)
    X = V.V.dof_coordinates()
    lid = np.stack([X[:, 0] * (1 - X[:, 0]), X[:, 1] * (1 - X[:, 1]), np.zeros(V.node_count)], axis=1)
    bcs = [bcs[0], DirichletBC(V, V.dat(lid), "top")]
    g = F.dat()
    for bc in bcs:
        bc.apply(g[0])
    Kg = assemble(F, u=g)
    K, _, _ = _reference(mesh, V, Q, bcs, np.zeros((V.node_count, 3)))
    want = K @ np.concatenate([g[0].data_ro.ravel(), np.zeros(Q.node_count)])
    nv = 3 * V.node_count
    assert np.abs(want[nv:]).max() > 1e-3 * np.abs(want[:nv]).max()
    assert np.abs(Kg[1].data_ro - want[nv:]).max() < 1e-12 * np.abs(want[nv:]).max()
    up = F.dat()
    solve(F, F.dat(), up, bcs, {**tg._fieldsplit("jacobi")}, nullspace="constant")
    _, u_ref, p_ref = _reference(mesh, V, Q, bcs, g[0].data_ro.copy())
    assert np.abs(up[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    assert np.abs(up[1].data_ro - p_ref).max() < 1e-7 * np.abs(p_ref).max()


def test_without_nullspace_no_pc(mock):
    """pc_type none and no nullspace: GMRES still converges on the singular but consistent system (the
    right-hand side is orthogonal to the constant pressure), and the velocity is scipy's."""
    from firedrake_b200.assemble import solve
    mesh, V, Q, F, bcs = tg._cavity(3)
    g = np.zeros((V.node_count, 3))
    g[bcs[1].nodes, 0] = 1.0
    up = F.dat()
    solve(F, F.dat(), up, bcs, {"ksp_rtol": 1e-12, "ksp_max_it": 3000})
    _, u_ref, _ = _reference(mesh, V, Q, bcs, g)
    assert np.abs(up[0].data_ro.ravel() - u_ref).max() < 1e-7 * np.abs(u_ref).max()


def test_refusals_host_logic(mock):
    tg.test_solver_refusals(mock)


def test_partitioned_spaces_are_refused(mock):
    from firedrake_b200.assemble import FunctionSpace, Stokes
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    mesh = ExtrudedHexMesh(2, 2, 2)
    V, Q = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1)
    V.cell_set.owner_computes = True
    with pytest.raises(NotImplementedError, match="partitioned"):
        Stokes(V, Q)


def test_other_solver_options_are_refused(mock):
    from firedrake_b200.assemble import Form, solve
    _, V, Q, F, bcs = tg._cavity(2)
    up = F.dat()
    fs = {"pc_type": "fieldsplit", "pc_fieldsplit_type": "schur", "pc_fieldsplit_schur_fact_type": "diag"}
    for extra, msg in (({"ksp_type": "minres"}, "gmres"), ({"mat_type": "aij"}, "matfree"),
                       ({"pc_type": "jacobi"}, "'none' or 'fieldsplit'"),
                       ({**fs, "fieldsplit_0_pc_type": "ilu"}, "'jacobi' or 'mg'"),
                       ({**fs, "fieldsplit_1_pc_type": "mg"}, "fieldsplit_1_pc_type"),
                       ({**fs, "fieldsplit_0_ksp_type": "cg"}, "preonly")):
        with pytest.raises(NotImplementedError, match=msg):
            solve(F, F.dat(), up, bcs, extra)
    with pytest.raises(ValueError, match="hierarchy"):
        solve(F, F.dat(), up, bcs, {**fs, "fieldsplit_0_pc_type": "mg"})
    with pytest.raises(NotImplementedError, match="Stokes forms only"):
        solve(Form(Q), Q.dat(), Q.dat(), nullspace="constant")
