"""The CPU oracle of the Boussinesq system on Taylor-Hood hexahedra (tests/_boussinesq_oracle.py) against
independent statements: the Jacobian against central differences of the residual, the Navier-Stokes oracle and the
temperature's stiffness matrix at Ra = 0, the exact conduction profile of the differentially heated cube at Ra = 0,
and the L2 rates of a manufactured solution on Q2-Q1-Q1."""
import numpy as np
import pytest

import _boussinesq_oracle as bo
import _coef_oracle as co
import _navier_stokes_oracle as nso
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

BG = (0.3, -0.2, -1.7)
KT = 0.6


def _setup(p, n=(3, 2, 3), warp=0.08, seed=1):
    mesh = ExtrudedHexMesh(*n, warp=warp, permute_seed=seed)
    V, Q = mesh.function_space(p), mesh.function_space(p - 1)
    geo = (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    return mesh, V, Q, geo, (Q.cell_node_map, Q.offset)


def _fields(V, Q, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(3 * V.node_count), rng.standard_normal(Q.node_count), rng.standard_normal(Q.node_count)


@pytest.mark.parametrize("p", [2, 3, 4])
def test_jacobian_is_the_derivative_of_the_residual(p):
    mesh, V, Q, geo, geo2 = _setup(p)
    el = interval_element(p)
    u, pr, T = _fields(V, Q, 1)
    w, r, s = _fields(V, Q, 2)
    R = lambda a, b, c: np.concatenate(bo.residual(el, mesh.coordinates, a, b, c, geo, geo2, BG, KT))
    Jw = np.concatenate(bo.jacobian_action(el, mesh.coordinates, u, T, w, r, s, geo, geo2, BG, KT))
    h = 1e-3
    fd = (R(u + h * w, pr + h * r, T + h * s) - R(u - h * w, pr - h * r, T - h * s)) / (2 * h)
    assert np.abs(fd - Jw).max() < 1e-9 * np.abs(Jw).max()


@pytest.mark.parametrize("p", [2, 3])
def test_jacobian_matrix_matches_its_action(p):
    mesh, V, Q, geo, geo2 = _setup(p)
    el = interval_element(p)
    u, _, T = _fields(V, Q, 3)
    w, r, s = _fields(V, Q, 4)
    K = bo.jacobian_matrix(el, mesh.coordinates, u, T, geo, geo2, V.node_count, Q.node_count, BG, KT)
    want = np.concatenate(bo.jacobian_action(el, mesh.coordinates, u, T, w, r, s, geo, geo2, BG, KT))
    assert np.abs(K @ np.concatenate([w, r, s]) - want).max() < 1e-12 * np.abs(want).max()


def _stiffness(el_q, mesh, Q, geo2, kt):
    """kt K_W as scipy CSR from the scalar coefficient oracle on the CG_(p-1) element at the velocity's rule."""
    import scipy.sparse as sps
    i2 = co._cells(Q.cell_node_map, Q.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    i0, i1 = i2
    Xc = mesh.coordinates.reshape(-1, 3)[i1]
    Ke = co.cell_matrices(el_q, Xc, np.ones(i0.shape), kt, 0.0)
    nd = i0.shape[1]
    return sps.csr_matrix((Ke.ravel(), (np.repeat(i0, nd, axis=1).ravel(), np.tile(i0, (1, nd)).ravel())),
                          shape=(Q.node_count, Q.node_count))


@pytest.mark.parametrize("p", [2, 3, 4])
def test_ra_zero_is_navier_stokes_and_conduction(p):
    """With Ra = 0 and zero velocity the (u, p) rows are the Navier-Stokes oracle's and the T rows are kt K_W T."""
    mesh, V, Q, geo, geo2 = _setup(p)
    el = interval_element(p)
    _, pr, T = _fields(V, Q, 5)
    z = np.zeros(3 * V.node_count)
    yu, yp, yT = bo.residual(el, mesh.coordinates, z, pr, T, geo, geo2, (0.0, 0.0, 0.0), KT)
    wu, wp = nso.residual(el, mesh.coordinates, z, pr, geo, geo2, 1.0)
    assert np.abs(yu - wu).max() <= 1e-13 * np.abs(wu).max()
    assert np.abs(yp - wp).max() <= 1e-13 * np.abs(wp).max()
    elq = interval_element(p - 1, p + 1)
    want = _stiffness(elq, mesh, Q, geo2, KT) @ T
    assert np.abs(yT - want).max() < 1e-12 * np.abs(want).max()
    # and with a velocity, the (u, p) rows still are Navier-Stokes at Ra = 0
    u, _, _ = _fields(V, Q, 6)
    yu, yp, _ = bo.residual(el, mesh.coordinates, u, pr, T, geo, geo2, (0.0, 0.0, 0.0), KT)
    wu, wp = nso.residual(el, mesh.coordinates, u, pr, geo, geo2, 1.0)
    assert np.abs(yu - wu).max() < 1e-13 * np.abs(wu).max()
    assert np.abs(yp - wp).max() < 1e-13 * np.abs(wp).max()


def cavity(n, p=2, warp=0.0):
    """The differentially heated cube: u = 0 on every wall, T = 1 on face 1 (x = 0), T = 0 on face 2 (x = 1),
    adiabatic elsewhere.  Returns the mesh, spaces, geometry, the fixed global dofs (with the first pressure dof
    pinned) and their values."""
    mesh, V, Q, geo, geo2 = _setup(p, (n, n, n), warp=warp, seed=0)
    nv, nq = V.node_count, Q.node_count
    walls = np.unique(np.concatenate([V.boundary_nodes(s) for s in (1, 2, 3, 4, "bottom", "top")]))
    hot, cold = Q.boundary_nodes(1), Q.boundary_nodes(2)
    fixed = np.concatenate([(3 * walls[:, None] + np.arange(3)).ravel(), [3 * nv], 3 * nv + nq + hot,
                            3 * nv + nq + cold])
    values = np.concatenate([np.zeros(3 * len(walls)), [0.0], np.ones(len(hot)), np.zeros(len(cold))])
    return mesh, V, Q, geo, geo2, fixed, values


def test_conduction_profile_at_ra_zero():
    """At Ra = 0 scipy's Newton on the heated cavity gives u = 0 and T = 1 - x exactly (T is in the space)."""
    mesh, V, Q, geo, geo2, fixed, values = cavity(3, warp=0.0)
    el = interval_element(2)
    u, p, T, hist = bo.newton(el, mesh.coordinates, geo, geo2, V.node_count, Q.node_count, (0.0, 0.0, 0.0),
                              1 / 6.8, fixed, values)
    x = _q1_x(mesh, Q)
    assert np.abs(u).max() < 1e-12
    assert np.abs(T - (1.0 - x)).max() < 1e-12
    assert np.abs(p).max() < 1e-12


def _q1_x(mesh, Q):
    """x of every CG1 node: CG1 nodes are the mesh vertices, so the coordinates through the two maps."""
    i2 = co._cells(Q.cell_node_map, Q.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    x = np.empty(Q.node_count)
    x[i2[0].ravel()] = mesh.coordinates.reshape(-1, 3)[i2[1]].reshape(-1, 3)[:, 0]
    return x


@pytest.mark.parametrize("p", [2, 3])
def test_generic_path_host_build_matches_the_oracle(oracle, p):
    import _mock_engine as me
    from firedrake_b200.assemble import Boussinesq, FunctionSpace, assemble_boussinesq_generic
    mesh, V0, Q0, geo, geo2 = _setup(p, seed=2)
    el = interval_element(p)
    u0, p0, T0 = _fields(V0, Q0, 8)
    w0, r0, s0 = _fields(V0, Q0, 9)
    Ra, Pr, g = 900.0, 2.5, (0.2, -0.1, -1.0)
    bg, kt = tuple(Ra / Pr * c for c in g), 1.0 / Pr
    want_r = bo.residual(el, mesh.coordinates, u0, p0, T0, geo, geo2, bg, kt)
    want_j = bo.jacobian_action(el, mesh.coordinates, u0, T0, w0, r0, s0, geo, geo2, bg, kt)
    with me.install(oracle):
        F = Boussinesq(FunctionSpace(mesh, p, 3), FunctionSpace(mesh, p - 1), FunctionSpace(mesh, p - 1), Ra, Pr, g)
        upT = F.dat(u0.reshape(-1, 3).copy(), p0.copy(), T0.copy())
        yr = [d.data_ro.copy() for d in assemble_boussinesq_generic(F, upT)]
        wrs = F.dat(w0.reshape(-1, 3).copy(), r0.copy(), s0.copy())
        yj = [d.data_ro.copy() for d in assemble_boussinesq_generic(F, upT, wrs)]
    for y, want in ((yr, want_r), (yj, want_j)):
        for b in range(3):
            assert np.abs(y[b].ravel() - want[b]).max() < 1e-12 * np.abs(want[b]).max()


def test_boussinesq_form_refusals():
    from firedrake_b200.assemble import Boussinesq, FunctionSpace, boussinesq_kernel
    mesh = ExtrudedHexMesh(2, 2, 2)
    V, Q, W = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1), FunctionSpace(mesh, 1)
    with pytest.raises(ValueError, match="FunctionSpace object of its own"):
        Boussinesq(V, Q, Q, 1e3, 6.8)
    with pytest.raises(ValueError, match="scalar CG_\\(p-1\\) on the pressure space's mesh"):
        Boussinesq(V, Q, FunctionSpace(mesh, 2), 1e3, 6.8)
    with pytest.raises(ValueError, match="scalar CG_\\(p-1\\) on the pressure space's mesh"):
        Boussinesq(V, Q, FunctionSpace(ExtrudedHexMesh(2, 2, 2), 1), 1e3, 6.8)
    with pytest.raises(ValueError, match="Boussinesq velocity space is a vector space"):
        Boussinesq(FunctionSpace(mesh, 2), Q, W, 1e3, 6.8)
    with pytest.raises(ValueError, match="Pr must be nonzero"):
        Boussinesq(V, Q, W, 1e3, 0.0)
    with pytest.raises(ValueError, match="3-vector"):
        Boussinesq(V, Q, W, 1e3, 6.8, g=(0.0, -1.0))
    F = Boussinesq(V, Q, W, 1e3, 6.8)
    assert F.bg == pytest.approx((0.0, 0.0, -1e3 / 6.8)) and F.kt == pytest.approx(1 / 6.8)
    with pytest.raises(ValueError, match="1-form"):
        F.kernel(2)
    for jac in (False, True):
        with pytest.raises(NotImplementedError, match="degrees 2..4"):
            boussinesq_kernel(5, 1e3, 6.8, jacobian=jac)



def _manufactured(Ra, Pr, g):
    """u = curl psi (divergence free, zero on the boundary of the unit cube), p and T, and the sources f_u, f_T of
    R = L."""
    import sympy as sp
    x, y, z = X3 = sp.symbols("x y z")
    psi = (sp.sin(sp.pi * x) * sp.sin(sp.pi * y) * sp.sin(sp.pi * z)) ** 2
    A = sp.Matrix([0, psi, psi * sp.cos(x)])
    ue = sp.Matrix([sp.diff(A[2], y) - sp.diff(A[1], z), sp.diff(A[0], z) - sp.diff(A[2], x),
                    sp.diff(A[1], x) - sp.diff(A[0], y)])
    pe = sp.cos(sp.pi * x) * sp.cos(sp.pi * y) * sp.cos(sp.pi * z)
    Te = 1 - x + sp.sin(sp.pi * x) * sp.sin(sp.pi * y) * sp.cos(sp.pi * z) / 4
    fu = [-sum(sp.diff(ue[i], v, 2) for v in X3) + sum(ue[k] * sp.diff(ue[i], X3[k]) for k in range(3))
          + sp.diff(pe, X3[i]) - Ra / Pr * g[i] * Te for i in range(3)]
    fT = sum(ue[k] * sp.diff(Te, X3[k]) for k in range(3)) - sum(sp.diff(Te, v, 2) for v in X3) / Pr
    lam = lambda e: sp.lambdify(X3, e, "numpy")
    return [lam(e) for e in ue], lam(pe), lam(Te), [lam(e) for e in fu], lam(fT)


def _trilinear(t, X):
    """The trilinear map of the cells X (nc, 8, 3) at the tensor points of the 1-D coordinates t: (nc, len(t)^3, 3)."""
    t = np.asarray(t)
    CB = np.stack([1.0 - t, t], axis=1)
    return np.einsum("qv,cvd->cqd", np.kron(np.kron(CB, CB), CB), X)


def _node_coordinates(mesh, S, el):
    """Physical coordinates of every node of the CG space S, whose 1-D element ``el`` lists its nodes in dof order."""
    i0, i1 = co._cells(S.cell_node_map, S.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    out = np.empty((S.node_count, 3))
    out[i0.ravel()] = _trilinear(el.nodes, mesh.coordinates.reshape(-1, 3)[i1]).reshape(-1, 3)
    return out


def test_manufactured_solution_rates():
    """Q2-Q1-Q1 on the unit cube, u, p and T manufactured, their sources assembled on the same rule, u and T
    prescribed on the whole boundary: L2 rates (on the Gauss rule) from 4^3 to 8^3 of at least 2.8 for u, 1.8 for
    p modulo a constant and 1.8 for T."""
    Ra, Pr, g = 200.0, 0.9, (0.0, 0.0, -1.0)
    bg, kt = tuple(Ra / Pr * c for c in g), 1.0 / Pr
    uex, pex, Tex, fu, fT = _manufactured(Ra, Pr, g)
    el = interval_element(2)
    errs = []
    for n in (4, 8):
        mesh, V, Q, geo, geo2 = _setup(2, (n, n, n), warp=0.0, seed=0)
        nv, nq = V.node_count, Q.node_count
        i0, i2, Xc = bo._gather(el, mesh.coordinates, geo, geo2)
        PV, PT, _ = bo._bases(el)
        _, detw = bo._metric(el, Xc)
        xq = _trilinear(el.xq, Xc)
        at = lambda f: np.broadcast_to(f(xq[..., 0], xq[..., 1], xq[..., 2]), xq.shape[:2])
        Lu, LT = np.zeros((nv, 3)), np.zeros(nq)
        for d in range(3):
            np.add.at(Lu[:, d], i0, np.einsum("cq,qa->ca", detw * at(fu[d]), PV))
        np.add.at(LT, i2, np.einsum("cq,qi->ci", detw * at(fT), PT))
        walls = np.unique(np.concatenate([V.boundary_nodes(s) for s in WALLS]))
        tnodes = np.unique(np.concatenate([Q.boundary_nodes(s) for s in WALLS]))
        xv, xt = _node_coordinates(mesh, V, el)[walls], _node_coordinates(mesh, Q, interval_element(1))[tnodes]
        ub = np.stack([np.broadcast_to(f(*xv.T), len(walls)) for f in uex], axis=1)
        fixed = np.concatenate([(3 * walls[:, None] + np.arange(3)).ravel(), [3 * nv], 3 * nv + nq + tnodes])
        values = np.concatenate([ub.ravel(), [0.0], Tex(*xt.T)])
        u, p, T, hist = bo.newton(el, mesh.coordinates, geo, geo2, nv, nq, bg, kt, fixed, values,
                                  L=np.concatenate([Lu.ravel(), np.zeros(nq), LT]))
        assert hist[-1] <= 1e-10 * hist[0], hist
        uq = np.einsum("qa,cad->cqd", PV, u.reshape(-1, 3)[i0])
        dp = p[i2] @ PT.T - at(pex)
        dp = dp - np.sum(detw * dp) / np.sum(detw)
        eu = np.sqrt(np.sum(detw * sum((uq[..., d] - at(uex[d])) ** 2 for d in range(3))))
        eT = np.sqrt(np.sum(detw * (T[i2] @ PT.T - at(Tex)) ** 2))
        errs.append((eu, np.sqrt(np.sum(detw * dp ** 2)), eT))
    rates = np.log2(np.array(errs[0]) / np.array(errs[1]))
    assert rates[0] >= 2.8 and rates[1] >= 1.8 and rates[2] >= 1.8, (errs, rates)


WALLS = (1, 2, 3, 4, "bottom", "top")
