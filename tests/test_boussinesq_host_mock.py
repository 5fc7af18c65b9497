"""Host logic of the Boussinesq system on the CPU: a mock engine that emulates FDB_FORM_BOUSSINESQ[_JACOBIAN] through
the NumPy oracle (tests/_boussinesq_oracle.py) runs the Python layers -- the 3-block assemblers, the matrix-free
Jacobian with a condition on each block, the block Gauss-Seidel fieldsplit and Newton -- and the Stokes and
Navier-Stokes solves are checked to make the engine calls that the version before the third block made.  The
device code itself is what `-m gpu` checks (tests/test_boussinesq_gpu.py)."""
import json
import os

import numpy as np
import pytest

import _boussinesq_oracle as bo
import _mock_engine as me
import _stokes_recorder as sr
import test_boussinesq_gpu as tb
import test_navier_stokes_host_mock as nm
from firedrake_b200 import _lib
from firedrake_b200.fiat_lite import interval_element

_KINDS = {_lib.FORM_BOUSSINESQ: "boussinesq", _lib.FORM_BOUSSINESQ_JACOBIAN: "boussinesq_jacobian"}


class BoussinesqMockEngine(nm.NavierStokesMockEngine):
    """NavierStokesMockEngine plus the Boussinesq residual and Jacobian action, device location."""

    def fdb_kernel_create_mixed(self, desc, space2, out):
        d, s2 = me._obj(desc), me._obj(space2)
        kind = _KINDS.get(d.form)
        if kind is None:
            return super().fdb_kernel_create_mixed(desc, space2, out)
        if d.cell not in (_lib.CELL_HEX_EXTRUDED, _lib.CELL_HEX) or d.cdim != 3 or d.rank != 1 or d.diagonal:
            return self._fail(f"mock engine: {kind} is a rank-1 action on a 3-component hex space")
        p = d.degree
        ext = d.cell == _lib.CELL_HEX_EXTRUDED
        n, n2 = (p + 1) ** 3, p ** 3
        self._next += 1
        self.kernels[self._next] = dict(
            kind=kind, degree=p, bg=tuple(d.dcoef[:3]), kt=d.lmbda, extruded=ext,
            off0=np.array(d.offset0[:n] if ext else [0] * n, dtype=np.int32),
            off1=np.array(d.offset1[:8] if ext else [0] * 8, dtype=np.int32),
            off2=np.array(s2.offset[:n2] if ext else [0] * n2, dtype=np.int32))
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        k = self.kernels[me._addr(h)]
        if k["kind"] not in _KINDS.values():
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        self.launches += 1
        jac = k["kind"] == "boussinesq_jacobian"
        want = 9 if jac else 7
        if a.nargs != want or a.nmaps != 3 or a.location != _lib.LOC_DEVICE:
            return self._fail(f"mock engine: {k['kind']} action expects {want} device args and 3 maps")
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
        geo2 = (map2[cols], k["off2"])
        x, q, t = me._view(a.args[2], 3 * nnode).copy(), me._view(a.args[4], nq).copy(), me._view(a.args[6], nq).copy()
        el = interval_element(p)
        if jac:
            yu, yp, yt = bo.jacobian_action(el, coords, me._view(a.args[7], 3 * nnode).copy(),
                                            me._view(a.args[8], nq).copy(), x, q, t, geo, geo2, k["bg"], k["kt"])
        else:
            yu, yp, yt = bo.residual(el, coords, x, q, t, geo, geo2, k["bg"], k["kt"])
        me._view(a.args[0], 3 * nnode)[:] += yu
        me._view(a.args[3], nq)[:] += yp
        me._view(a.args[5], nq)[:] += yt
        return 0


class install(me.install):
    def __init__(self, oracle):
        self.engine = BoussinesqMockEngine(oracle)


@pytest.fixture()
def mock(oracle):
    with install(oracle) as eng:
        yield eng


def _geo(F):
    mesh, V, Q = F.V.mesh, F.V, F.Q
    return (mesh, (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz),
            (Q.V.cell_node_map, Q.V.offset))


def test_assemblers_follow_the_linearisation_point(mock):
    """assemble(F, u=upT) and assemble(F.jacobian(upT), u=wrs) hand the right Dats to the engine; the Jacobian reads
    upT[0] and upT[2] in place."""
    from firedrake_b200.assemble import assemble
    F = tb._form(2)
    upT, wrs = tb._random(F, 1), tb._random(F, 2)
    mesh, geo, geo2 = _geo(F)
    el = interval_element(2)
    fl = lambda d: d.data_ro.ravel().copy()
    want = np.concatenate(bo.residual(el, mesh.coordinates, fl(upT[0]), fl(upT[1]), fl(upT[2]), geo, geo2, F.bg,
                                      F.kt))
    assert tb.relerr(tb._flat(assemble(F, u=upT)), want) < 1e-13
    J = F.jacobian(upT)
    for _ in range(2):
        want = np.concatenate(bo.jacobian_action(el, mesh.coordinates, fl(upT[0]), fl(upT[2]), fl(wrs[0]),
                                                 fl(wrs[1]), fl(wrs[2]), geo, geo2, F.bg, F.kt))
        assert tb.relerr(tb._flat(assemble(J, u=wrs)), want) < 1e-13
        upT[0].data[:] *= 2.0
        upT[2].data[:] *= -1.5


def test_bcs_act_on_the_block_of_their_space(mock):
    """A condition on W constrains the temperature block only, one on V the velocity block only: the matrix-free
    Jacobian is the identity on those rows and leaves the other blocks' rows with the same node numbers alone."""
    from firedrake_b200.assemble import DirichletBC, assemble
    F = tb._form(2)
    upT, wrs = tb._random(F, 3), tb._random(F, 4)
    J = F.jacobian(upT)
    plain = [d.data_ro.copy() for d in assemble(J, u=wrs)]
    bcT = DirichletBC(F.W, 1.0, 1)
    bcV = DirichletBC(F.V, 0.0, "top")
    A = assemble(J, bcs=[bcT, bcV], mat_type="matfree")
    Y = F.dat()
    A.mult(wrs, Y)
    # rows: identity on the constrained nodes of each block
    assert np.array_equal(Y[2].data_ro[bcT.nodes], wrs[2].data_ro[bcT.nodes])
    assert np.array_equal(Y[0].data_ro[bcV.nodes], wrs[0].data_ro[bcV.nodes])
    # the pressure block has no condition: it differs from the plain action only through the zeroed columns
    x = F.dat(*[d.data_ro.copy() for d in wrs])
    x[2].data[bcT.nodes] = 0.0
    x[0].data[bcV.nodes] = 0.0
    want = [d.data_ro.copy() for d in assemble(J, u=x)]
    assert tb.relerr(Y[1].data_ro, want[1]) < 1e-13
    free = np.setdiff1d(np.arange(F.W.node_count), bcT.nodes)
    assert tb.relerr(Y[2].data_ro[free], want[2][free]) < 1e-13
    assert not np.allclose(want[1], plain[1])            # the zeroed columns do enter the pressure rows
    # the residual zeroes the temperature rows of bcT, and the velocity rows of the same node numbers are kept
    R = assemble(F, u=upT, bcs=[bcT])
    R0 = assemble(F, u=upT)
    assert np.all(R[2].data_ro[bcT.nodes] == 0.0)
    assert np.array_equal(R[0].data_ro, R0[0].data_ro) and np.array_equal(R[1].data_ro, R0[1].data_ro)


def _dense_jacobian(A, F):
    """The matrix of a matrix-free operator on 3-block vectors, column by column."""
    sizes = [3 * F.V.node_count, F.Q.node_count, F.W.node_count]
    n = sum(sizes)
    K = np.empty((n, n))
    for j in range(n):
        e = np.zeros(n)
        e[j] = 1.0
        x = F.dat(e[:sizes[0]].reshape(-1, 3), e[sizes[0]:sizes[0] + sizes[1]], e[sizes[0] + sizes[1]:])
        Y = F.dat()
        A.mult(x, Y)
        K[:, j] = tb._flat(Y)
    return K, sizes


@pytest.mark.parametrize("split", ["multiplicative", "additive"])
def test_block_gauss_seidel_with_exact_inverses(mock, split):
    """With the exact inverses of the diagonal blocks, multiplicative M is the inverse of A's block lower triangle L,
    so A M - I = (A - L) L^-1 has zero temperature rows (the (u, p) rows keep the buoyancy coupling, which block
    Gauss-Seidel does not remove).  Additive M leaves A_10 A_00^-1 in the temperature rows."""
    from firedrake_b200.assemble import DirichletBC, _block_gauss_seidel, assemble
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    F = tb._form(2, mesh=ExtrudedHexMesh(2, 1, 2, warp=0.05, permute_seed=3))
    upT = tb._random(F, 5, 0.3)
    # no slip on the bottom only: the (u, p) block is then invertible (no constant-pressure mode)
    A = assemble(F.jacobian(upT), bcs=[DirichletBC(F.V, 0.0, "bottom"), DirichletBC(F.W, 0.0, 1)],
                 mat_type="matfree")
    K, sizes = _dense_jacobian(A, F)
    n0 = sizes[0] + sizes[1]
    inv0, inv1 = np.linalg.inv(K[:n0, :n0]), np.linalg.inv(K[n0:, n0:])

    def S0(r, z):
        v = inv0 @ np.concatenate([r[0].data_ro.ravel(), r[1].data_ro])
        z[0].data[:] = v[:sizes[0]].reshape(-1, 3)
        z[1].data[:] = v[sizes[0]:]

    def S1(r, z):
        z.data[:] = inv1 @ r.data_ro

    M = _block_gauss_seidel(S0, S1, A, F.dat, split == "multiplicative")
    AM = np.empty_like(K)
    n = K.shape[0]
    for j in range(n):
        e = np.zeros(n)
        e[j] = 1.0
        r = F.dat(e[:sizes[0]].reshape(-1, 3), e[sizes[0]:n0], e[n0:])
        z = F.dat()
        M(r, z)
        Y = F.dat()
        A.mult(z, Y)
        AM[:, j] = tb._flat(Y)
    E = AM - np.eye(n)
    assert np.abs(E[n0:, n0:]).max() < 1e-9              # both: the temperature block is inverted exactly
    if split == "multiplicative":
        assert np.abs(E[n0:]).max() < 1e-9
    else:
        assert np.abs(E[n0:, :n0]).max() > 1e-3


def test_newton_on_the_heated_cavity_matches_scipy(mock):
    """3^3 at Ra = 1e3, Pr = 6.8, the demo's multiplicative fieldsplit and the constant nullspace."""
    F, bcs = tb._cavity(3, 1e3, 6.8)
    upT = F.dat()
    from firedrake_b200.assemble import solve_nonlinear
    hist, kits, inner = solve_nonlinear(F, F.dat(), upT, bcs, tb._demo_options(), nullspace="constant")
    assert hist[-1] <= 1e-10 * hist[0] and len(kits) < 10, (hist, kits)
    assert len(inner) == len(kits) and all(a > 0 and b > 0 for a, b in inner)
    mesh, geo, geo2 = _geo(F)
    nv, nq = F.V.node_count, F.Q.node_count
    walls = bcs[0].nodes
    fixed = np.concatenate([(3 * walls[:, None] + np.arange(3)).ravel(), [3 * nv], 3 * nv + nq + bcs[1].nodes,
                            3 * nv + nq + bcs[2].nodes])
    values = np.concatenate([np.zeros(3 * len(walls) + 1), np.ones(len(bcs[1].nodes)), np.zeros(len(bcs[2].nodes))])
    u_ref, p_ref, T_ref, _ = bo.newton(interval_element(2), mesh.coordinates, geo, geo2, nv, nq, F.bg, F.kt, fixed,
                                       values)
    assert np.abs(upT[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    assert np.abs(upT[2].data_ro - T_ref).max() < 1e-8 * np.abs(T_ref).max()
    p = upT[1].data_ro
    assert np.abs(p - p.mean() - p_ref).max() < 1e-7 * np.abs(p_ref).max()


def test_divergence_is_reported(mock):
    from firedrake_b200.assemble import ConvergenceError, solve_nonlinear
    F, bcs = tb._cavity(2, 1e3, 6.8)
    L = F.dat()
    L[2].data[:] = np.nan
    with pytest.raises(ConvergenceError) as e:
        solve_nonlinear(F, L, F.dat(), bcs)
    assert e.value.reason == "DIVERGED_FNORM_NAN"


def test_refusals_host_logic(mock):
    tb.test_solver_refusals(mock)


def test_partitioned_and_mismatched_spaces_are_refused(mock):
    from firedrake_b200.assemble import Boussinesq, FunctionSpace
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    mesh = ExtrudedHexMesh(2, 2, 2)
    V, Q, W = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1), FunctionSpace(mesh, 1)
    W.cell_set.owner_computes = True
    with pytest.raises(NotImplementedError, match="Boussinesq on a partitioned mesh"):
        Boussinesq(V, Q, W, 1e3, 6.8)


@pytest.mark.parametrize("case", sr.CASES)
def test_stokes_and_navier_stokes_engine_calls_are_unchanged(oracle, case):
    """The Stokes and Navier-Stokes solves make exactly the engine calls that the version before the 3-block
    assembler made (tests/golden/stokes_engine_calls.json, recorded with tests/_stokes_recorder.py)."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stokes_engine_calls.json")) as f:
        golden = json.load(f)
    assert sr.solve_calls(oracle, case) == golden[case]
