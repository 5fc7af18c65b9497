"""CPU checks of the pressure convection-diffusion oracle (tests/_pcd_oracle.py) and of the premise of a PCD
Schur approximation on this engine's lid-driven cavity.

The oracle: F_p at u = 0 is nu K + beta M from the scalar Helmholtz oracle on Q with the same rule; F_p is
linear in u and r; the convective part of a linear pressure at a constant velocity is exact; a point-by-point
restatement of one warped cell agrees.  The premise: with exact inner solves, the "lower" factorisation with the
exact Schur complement converges in two iterations (the sign check), and exact PCD with natural pressure
conditions takes more iterations than the exact (1/nu) M_p approximation (the measurement DESIGN.md section 4.13
records, and the reason the engine has no F_p kernel)."""
import numpy as np
import pytest

import _navier_stokes_oracle as nso
import _pcd_oracle as po
import _stokes_oracle as so
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh


def _spaces(p, n=(3, 2, 2), warp=0.05):
    mesh = ExtrudedHexMesh(*n, warp=warp, permute_seed=2)
    V, Q = mesh.function_space(p), mesh.function_space(p - 1)
    geo = (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    return mesh, V, Q, geo, (Q.cell_node_map, Q.offset)


@pytest.mark.parametrize("p", [2, 3, 4])
def test_zero_velocity_is_helmholtz(p):
    mesh, V, Q, geo, geo2 = _spaces(p)
    el = interval_element(p)
    Fp = po.matrix(el, mesh.coordinates, np.zeros(3 * V.node_count), geo, geo2, Q.node_count, 0.7, 0.3)
    K = po.helmholtz_matrix(el, mesh.coordinates, geo, geo2, Q.node_count, 1.0, 0.0)
    M = po.helmholtz_matrix(el, mesh.coordinates, geo, geo2, Q.node_count, 0.0, 1.0)
    want = (0.7 * K + 0.3 * M).toarray()
    assert np.abs(Fp.toarray() - want).max() < 1e-13 * np.abs(want).max()


@pytest.mark.parametrize("p", [2, 3])
def test_linear_in_u_and_r(p):
    mesh, V, Q, geo, geo2 = _spaces(p)
    el = interval_element(p)
    rng = np.random.default_rng(p)
    u1, u2 = rng.standard_normal((2, 3 * V.node_count))
    r1, r2 = rng.standard_normal((2, Q.node_count))
    F = lambda r, u: po.action(el, mesh.coordinates, r, u, geo, geo2, 0.0, 0.0)
    ref = np.abs(F(r1, u1)).max()
    assert np.abs(F(r1, 2 * u1 - 3 * u2) - 2 * F(r1, u1) + 3 * F(r1, u2)).max() < 1e-13 * ref
    assert np.abs(F(2 * r1 - 3 * r2, u1) - 2 * F(r1, u1) + 3 * F(r2, u1)).max() < 1e-13 * ref
    # nu and beta enter linearly beside the convective part
    full = po.action(el, mesh.coordinates, r1, u1, geo, geo2, 0.7, 0.3)
    assert np.abs(full - F(r1, u1) - po.action(el, mesh.coordinates, r1, 0 * u1, geo, geo2, 0.7, 0.3)).max() \
        < 1e-13 * np.abs(full).max()


@pytest.mark.parametrize("p", [2, 3, 4])
def test_constant_velocity_on_a_linear_pressure(p):
    """u = c and r = a . x (in Q on the trilinear cells): inner(u, grad r) q = (c . a) q, so F_p r = (c . a) M 1
    at nu = beta = 0."""
    mesh, V, Q, geo, geo2 = _spaces(p)
    el = interval_element(p)
    c, a = np.array([0.3, -0.7, 1.1]), np.array([1.0, 2.0, -3.0])
    y = po.action(el, mesh.coordinates, Q.dof_coordinates() @ a, np.tile(c, V.node_count), geo, geo2, 0.0, 0.0)
    M = po.helmholtz_matrix(el, mesh.coordinates, geo, geo2, Q.node_count, 0.0, 1.0)
    want = (c @ a) * (M @ np.ones(Q.node_count))
    assert np.abs(y - want).max() < 1e-13 * np.abs(want).max()


@pytest.mark.parametrize("p", [2, 3])
def test_pointwise_restatement_of_one_cell(p):
    """One warped cell, element matrix summed point by point: nu gq . gr + beta q r + (u . gr) q times |det J| w."""
    mesh, V, Q, geo, geo2 = _spaces(p, (1, 1, 1), warp=0.15)
    el = interval_element(p)
    pe = po.pressure_element(el)
    X = mesh.coordinates.reshape(-1, 3)[mesh.coord_map[0]].reshape(1, 8, 3)
    rng = np.random.default_rng(5)
    u = rng.standard_normal((1, (p + 1) ** 3, 3))
    nu, beta = 0.4, 0.9
    got = np.swapaxes(po.cell_actions(el, X, np.eye(p ** 3)[None], u, nu, beta)[0], 0, 1)
    xq, wq = el.xq, el.wq
    Bv, Bq, Dq = np.asarray(el.B), np.asarray(pe.B), np.asarray(pe.D)
    Xv = X[0].reshape(2, 2, 2, 3)
    want = np.zeros((p ** 3, p ** 3))
    for i, j, k in np.ndindex(len(xq), len(xq), len(xq)):
        s = xq[[i, j, k]]
        lin = np.stack([1 - s, s], axis=1)
        dl = np.array([-1.0, 1.0])
        J = np.stack([np.einsum("a,b,c,abcd->d", dl, lin[1], lin[2], Xv),
                      np.einsum("a,b,c,abcd->d", lin[0], dl, lin[2], Xv),
                      np.einsum("a,b,c,abcd->d", lin[0], lin[1], dl, Xv)], axis=1)
        w = wq[i] * wq[j] * wq[k] * abs(np.linalg.det(J))
        phi = np.einsum("a,b,c->abc", Bq[i], Bq[j], Bq[k]).ravel()
        gref = np.stack([np.einsum("a,b,c->abc", Dq[i], Bq[j], Bq[k]).ravel(),
                         np.einsum("a,b,c->abc", Bq[i], Dq[j], Bq[k]).ravel(),
                         np.einsum("a,b,c->abc", Bq[i], Bq[j], Dq[k]).ravel()], axis=1)
        g = gref @ np.linalg.inv(J)                       # physical gradients, one row per basis function
        uq = np.einsum("a,b,c,abcd->d", Bv[i], Bv[j], Bv[k], u[0].reshape(p + 1, p + 1, p + 1, 3))
        want += w * (nu * g @ g.T + beta * np.outer(phi, phi) + np.outer(phi, g @ uq))
    assert np.abs(got - want).max() < 1e-13 * np.abs(want).max()


def _cavity_system(n, nu):
    mesh = ExtrudedHexMesh(n, n, n)
    V, Q = mesh.function_space(2), mesh.function_space(1)
    geo = (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    geo2 = (Q.cell_node_map, Q.offset)
    X = V.dof_coordinates()
    bd = so.velocity_dofs(np.where(np.any((X < 1e-12) | (X > 1 - 1e-12), axis=1))[0])
    g = np.zeros((V.node_count, 3))
    g[X[:, 2] > 1 - 1e-12, 0] = 1.0
    el = interval_element(2)
    nv, nq = V.node_count, Q.node_count
    u, _, _ = nso.newton(el, mesh.coordinates, geo, geo2, nv, nq, nu, bd, g.ravel(), rtol=1e-6)
    J = so.constrained(nso.jacobian_matrix(el, mesh.coordinates, u, geo, geo2, nv, nq, nu), bd)
    Fp = po.matrix(el, mesh.coordinates, u, geo, geo2, nq, nu)
    Kp = po.helmholtz_matrix(el, mesh.coordinates, geo, geo2, nq, 1.0, po.KP_MASS)
    Mp = po.helmholtz_matrix(el, mesh.coordinates, geo, geo2, nq, 0.0, 1.0)
    return J, bd, 3 * nv, Fp, Kp, Mp


def test_pcd_premise_on_the_cavity():
    """Q2-Q1 cavity on 4^3 at Re = 100, the Jacobian at the Newton solution, exact velocity solves (sparse LU):
    flexible GMRES to 1e-8 with the "lower" factorisation takes 2 iterations with the exact Schur complement and
    more with the opposite sign; with (1/nu) M_p it beats "diag" with (1/nu) M_p; and exact PCD, K_p^-1 F_p
    M_p^-1, takes more iterations than (1/nu) M_p in both factorisations."""
    import scipy.sparse.linalg as spla
    nu = 0.01
    J, bd, n, Fp, Kp, Mp = _cavity_system(4, nu)
    A, Bt, B, _ = so.blocks(J, n // 3)
    Flu, Klu, Mlu = spla.splu(A.tocsc()), spla.splu(Kp.tocsc()), spla.splu(Mp.tocsc())
    Sinv = np.linalg.pinv(B @ Flu.solve(Bt.toarray()))           # (B F^-1 B^T)^-1
    P1 = {"exact": lambda r: Sinv @ r, "wrong_sign": lambda r: -(Sinv @ r), "mass": lambda r: nu * Mlu.solve(r),
          "pcd": lambda r: Klu.solve(Fp @ Mlu.solve(r))}
    b = np.random.default_rng(0).standard_normal(J.shape[0])
    b[bd] = 0.0
    b[n:] -= b[n:].mean()

    def project(z):
        z = z.copy()
        z[n:] -= z[n:].mean()
        return z

    def pc(fact, s1):
        def prec(r):
            if fact == "upper":
                zp = -P1[s1](r[n:])
                return np.concatenate([Flu.solve(r[:n] - Bt @ zp), zp])
            zu = Flu.solve(r[:n])
            zp = P1[s1](r[n:]) if fact == "diag" else -P1[s1](r[n:] - B @ zu)
            return np.concatenate([zu, zp])
        return prec

    def its(fact, s1):
        _, k, ok = po.fgmres(lambda v: J @ v, b, pc(fact, s1), rtol=1e-8, maxit=400, project=project)
        assert ok
        return k

    # with the exact Schur complement J P - I is nilpotent, (J P - I)^2 = 0, for the triangular factorisations;
    # with the opposite sign J P has the eigenvalues 1 and -1 instead (GMRES also takes 2 iterations then)
    T = lambda prec, v: J @ project(prec(v)) - v
    for fact in ("lower", "upper"):
        assert its(fact, "exact") <= 2
        assert np.abs(T(pc(fact, "exact"), T(pc(fact, "exact"), b))).max() < 1e-8 * np.abs(b).max()
        assert np.abs(T(pc(fact, "wrong_sign"), T(pc(fact, "wrong_sign"), b))).max() > 0.1 * np.abs(b).max()
    assert its("diag", "exact") <= 3
    lower_mass, diag_mass = its("lower", "mass"), its("diag", "mass")
    assert lower_mass < diag_mass
    assert its("lower", "pcd") > lower_mass
    assert its("diag", "pcd") > diag_mass
