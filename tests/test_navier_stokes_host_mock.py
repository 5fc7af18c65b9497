"""Host logic of steady Navier-Stokes on the CPU: a mock engine that emulates FDB_FORM_NAVIER_STOKES[_JACOBIAN]
through the NumPy oracle (tests/_navier_stokes_oracle.py) runs the Python layers -- the residual and Jacobian
assemblers on MixedDats, the matrix-free Jacobian with velocity conditions, Newton with matrix-free GMRES and
both fieldsplit variants, the constant-pressure nullspace -- against scipy's Newton, and every refusal of the
Python layer.  The device code itself is what `-m gpu` checks (tests/test_navier_stokes_gpu.py)."""
import numpy as np
import pytest

import _mock_engine as me
import _navier_stokes_oracle as nso
import test_navier_stokes_gpu as tn
import test_stokes_host_mock as sm
from firedrake_b200 import _lib
from firedrake_b200.fiat_lite import interval_element

_KINDS = {_lib.FORM_NAVIER_STOKES: "navier_stokes", _lib.FORM_NAVIER_STOKES_JACOBIAN: "navier_stokes_jacobian"}


class NavierStokesMockEngine(sm.StokesMockEngine):
    """StokesMockEngine plus the Navier-Stokes residual and Jacobian action, extruded and native hexes, device
    location."""

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
            kind=kind, degree=p, mu=d.alpha, beta=d.beta, extruded=ext,
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
        jac = k["kind"] == "navier_stokes_jacobian"
        want = 6 if jac else 5
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
        x, q = me._view(a.args[2], 3 * nnode).copy(), me._view(a.args[4], nq).copy()
        el = interval_element(p)
        if jac:
            yu, yp = nso.jacobian_action(el, coords, me._view(a.args[5], 3 * nnode).copy(), x, q, geo, geo2,
                                         k["mu"], k["beta"])
        else:
            yu, yp = nso.residual(el, coords, x, q, geo, geo2, k["mu"], k["beta"])
        me._view(a.args[0], 3 * nnode)[:] += yu
        me._view(a.args[3], nq)[:] += yp
        return 0


class install(me.install):
    def __init__(self, oracle):
        self.engine = NavierStokesMockEngine(oracle)


@pytest.fixture()
def mock(oracle):
    with install(oracle) as eng:
        yield eng


def test_matfree_mult_host_logic(mock):
    tn.test_matfree_mult_with_velocity_bcs_matches_oracle(mock)


def test_residual_and_jacobian_assemblers_host_logic(mock):
    """assemble(F, u=up) and assemble(F.jacobian(up), u=wr) hand the right Dats to the engine: the Jacobian
    reads up[0] in place, so it follows an update of up without being rebuilt."""
    from firedrake_b200.assemble import assemble
    F = tn._form(2)
    up, wr = tn._random(F, 1), tn._random(F, 2)
    mesh, V, Q = F.V.mesh, F.V, F.Q
    geo = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    geo2 = (Q.V.cell_node_map, Q.V.offset)
    el = interval_element(2)
    want = np.concatenate(nso.residual(el, mesh.coordinates, up[0].data_ro.ravel().copy(), up[1].data_ro.copy(),
                                       geo, geo2, F.nu, F.beta))
    assert tn.relerr(tn._flat(assemble(F, u=up)), want) < 1e-13
    J = F.jacobian(up)
    for _ in range(2):
        want = np.concatenate(nso.jacobian_action(el, mesh.coordinates, up[0].data_ro.ravel().copy(),
                                                  wr[0].data_ro.ravel().copy(), wr[1].data_ro.copy(), geo, geo2,
                                                  F.nu, F.beta))
        assert tn.relerr(tn._flat(assemble(J, u=wr)), want) < 1e-13
        up[0].data[:] *= 2.0


@pytest.mark.parametrize("pc0", ["jacobi", "mg"])
def test_newton_fieldsplit_matches_scipy(mock, pc0):
    """The lid-driven cavity on 4^3 (Q2-Q1) at Re = 10: Newton with matrix-free GMRES, the diagonal Schur
    fieldsplit and the constant nullspace gives scipy's Newton velocity and, modulo a constant, its pressure;
    the pressure comes back with zero mean."""
    from firedrake_b200.assemble import solve_nonlinear
    from firedrake_b200.mg import MeshHierarchy
    mesh, V, Q, F, bcs = tn._cavity(4, 0.1)
    up = F.dat()
    hist, kits = solve_nonlinear(F, F.dat(), up, bcs, tn._fieldsplit(pc0, 1e-10),
                                 hierarchy=MeshHierarchy(2, 2, 2, 1) if pc0 == "mg" else None, nullspace="constant")
    assert hist[-1] <= 1e-10 * hist[0] and 2 <= len(kits) < 10, (hist, kits)
    u_ref, p_ref, ref_hist = tn._scipy_cavity(mesh, V, Q, F, bcs)
    assert len(ref_hist) >= 3
    assert np.abs(up[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    p = up[1].data_ro
    assert abs(p.mean()) < 1e-12 * np.abs(p_ref).max()
    assert np.abs(p - p_ref).max() < 1e-7 * np.abs(p_ref).max()


def test_newton_without_preconditioner(mock):
    """pc_type none with the nullspace, from rest: the same solution as scipy's Newton."""
    from firedrake_b200.assemble import solve_nonlinear
    mesh, V, Q, F, bcs = tn._cavity(3, 0.2)
    up = F.dat()
    hist, _ = solve_nonlinear(F, F.dat(), up, bcs, {"snes_rtol": 1e-10, "ksp_rtol": 1e-11, "ksp_max_it": 3000},
                              nullspace="constant")
    assert hist[-1] <= 1e-10 * hist[0]
    u_ref, p_ref, _ = tn._scipy_cavity(mesh, V, Q, F, bcs)
    assert np.abs(up[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    assert np.abs(up[1].data_ro - p_ref).max() < 1e-7 * np.abs(p_ref).max()


def test_divergence_is_reported(mock):
    """A non-finite residual ends Newton with DIVERGED_FNORM_NAN."""
    from firedrake_b200.assemble import ConvergenceError, solve_nonlinear
    _, V, Q, F, bcs = tn._cavity(2, 0.1)
    up = F.dat()
    L = F.dat()
    L[0].data[:] = np.inf
    with pytest.raises(ConvergenceError) as e:
        solve_nonlinear(F, L, up, bcs)
    assert e.value.reason == "DIVERGED_FNORM_NAN"


def test_refusals_host_logic(mock):
    tn.test_solver_refusals(mock)


def test_partitioned_spaces_are_refused(mock):
    from firedrake_b200.assemble import FunctionSpace, NavierStokes
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    mesh = ExtrudedHexMesh(2, 2, 2)
    V, Q = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1)
    V.cell_set.owner_computes = True
    with pytest.raises(NotImplementedError, match="Navier-Stokes on a partitioned mesh"):
        NavierStokes(V, Q)


def test_op2_kernel_accesses():
    from firedrake_b200 import op2
    INC, READ = op2.INC, op2.READ
    k = op2.Kernel("navier_stokes", degree=2)
    assert k.cdim == 3 and k.accesses == (INC, READ, READ, INC, READ)
    k = op2.Kernel("navier_stokes_jacobian", degree=3)
    assert k.cdim == 3 and k.accesses == (INC, READ, READ, INC, READ, READ)
