"""CPU checks of the spectral-element (collocated GLL) tables and oracle (tests/_sem_oracle.py), and of the host-side
point location of assemble.PointEvaluator: the GLL rule's exactness, B = I, the lumped (diagonal) mass, symmetry and
the constant null vector of the stiffness, the Rayleigh quotient's convergence to 3 pi^2, the leapfrog energy and
point location against brute force."""
import numpy as np
import pytest

import _boundary_oracle as bo
import _sem_oracle as so
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh


class _Space:
    """The host-side attributes of assemble.FunctionSpace that point location reads (no engine needed)."""

    def __init__(self, mesh, p):
        self.mesh, self.degree, self.cdim, self.family = mesh, p, 1, "CG"
        self.V = mesh.function_space(p)


def warped(n=3, seed=1):
    return bo.perturb(ExtrudedHexMesh(n, n - 1, n, Lx=1.2, Ly=0.9, Lz=1.1, warp=0.05, permute_seed=seed), 0.08, seed)


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
def test_gll_rule(p):
    """The p+1 GLL weights integrate x^k exactly for k <= 2p-1 (and not 2p); B is exactly I in dof order, D the
    derivative of the Lagrange basis at the nodes, and the default Gauss tables are unchanged."""
    el = interval_element(p, quadrature="gll")
    for k in range(2 * p):
        assert abs(el.wq @ el.xq ** k - 1.0 / (k + 1)) < 1e-14, k
    assert abs(el.wq @ el.xq ** (2 * p) - 1.0 / (2 * p + 1)) > 1e-6
    assert np.array_equal(el.B, np.eye(p + 1))
    assert el.xq[0] == 0.0 and el.xq[1] == 1.0 and np.array_equal(el.xq, el.nodes)
    _, D = el.tabulate(el.xq)
    assert np.allclose(el.D, D, atol=1e-13, rtol=0)
    g = interval_element(p)
    assert g.quadrature == "gauss" and np.allclose(g.xq, np.polynomial.legendre.leggauss(p + 1)[0] * 0.5 + 0.5)
    with pytest.raises(ValueError, match="collocated"):
        interval_element(p, nq=p + 2, quadrature="gll")


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
def test_lumped_mass_is_diagonal_and_equals_gauss_load(p):
    """On an affine mesh the GLL mass matrix is diagonal and its diagonal is the Gauss load of 1 (Firedrake's
    test_spectral_mass_lumping); on a warped mesh it stays diagonal."""
    mesh = ExtrudedHexMesh(2, 3, 2, Lx=1.3, Ly=0.7, Lz=0.9)
    W = mesh.function_space(p)
    M = so.operator(mesh, W, p, 0.0, 1.0).toarray()
    assert np.abs(M - np.diag(np.diag(M))).max() < 1e-15 * np.abs(M).max()
    assert np.abs(np.diag(M) - so.gauss_load_of_one(mesh, W, p)).max() < 1e-13 * np.diag(M).max()
    mw = warped(2, p)
    Mw = so.operator(mw, mw.function_space(p), p, 0.0, 1.0).toarray()
    assert np.abs(Mw - np.diag(np.diag(Mw))).max() < 1e-15 * np.abs(Mw).max()


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
def test_stiffness_symmetric_null_and_diagonal(p):
    mesh = warped(2, 10 + p)
    W = mesh.function_space(p)
    kappa = 1.0 + np.random.default_rng(p).uniform(0, 1, W.node_count)
    K = so.operator(mesh, W, p, 1.0, 0.0, kappa).toarray()
    assert np.abs(K - K.T).max() < 1e-13 * np.abs(K).max()
    assert np.abs(K @ np.ones(W.node_count)).max() < 1e-12 * np.abs(K).max()
    A = so.operator(mesh, W, p, 0.7, 0.3, kappa)
    assert np.all(np.linalg.eigvalsh(A.toarray()) > 0)


def test_rayleigh_quotient_rate():
    """The Rayleigh quotient u^T K u / u^T M u of the interpolated mode cos(pi x) cos(pi y) cos(pi z) on the unit cube
    (lumped M) tends to 3 pi^2 at an observed rate of at least p + 1 between 3^3 and 6^3 cells: 1.96, 3.97 and 5.98
    for p = 1, 2, 3 (2p, DESIGN.md section 4.18).  At p = 1, where p + 1 = 2p, the rate approaches 2 from below."""
    rates = {}
    for p in (1, 2, 3):
        errs = []
        for n in (3, 6):
            mesh = ExtrudedHexMesh(n, n, n)
            W = mesh.function_space(p)
            X = W.dof_coordinates()
            u = np.cos(np.pi * X[:, 0]) * np.cos(np.pi * X[:, 1]) * np.cos(np.pi * X[:, 2])
            K = so.operator(mesh, W, p, 1.0, 0.0)
            m = so.operator(mesh, W, p, 0.0, 1.0).diagonal()
            errs.append(abs(u @ (K @ u) / (u @ (m * u)) - 3 * np.pi ** 2))
        rates[p] = np.log2(errs[0] / errs[1])
        assert rates[p] >= (p + 1 if p > 1 else 1.9), (p, errs, rates)


def test_leapfrog_energy():
    """500 oracle leapfrog steps at 0.9 of the stability bound conserve the discrete energy to 1e-11 relative."""
    p = 2
    mesh = warped(3, 4)
    W = mesh.function_space(p)
    kappa = np.where(W.dof_coordinates()[:, 2] > 0.5, 2.0, 1.0)
    K = so.operator(mesh, W, p, 1.0, 0.0, kappa)
    m = so.operator(mesh, W, p, 0.0, 1.0).diagonal()
    lmax = np.linalg.eigvalsh((K.toarray() / np.sqrt(m)[:, None]) / np.sqrt(m)[None, :]).max()
    dt = 0.9 * 2.0 / np.sqrt(lmax)
    u0 = np.random.default_rng(0).standard_normal(W.node_count)
    u1, u0_ = so.leapfrog(K, m, u0, u0, dt, 1)[:2]
    E0 = so.energy(K, m, u1, u0_, dt)
    u, up, _ = so.leapfrog(K, m, u1, u0_, dt, 500)
    assert abs(so.energy(K, m, u, up, dt) - E0) < 1e-11 * abs(E0)


@pytest.mark.parametrize("p", [1, 3])
def test_point_location_matches_brute_force(p):
    from firedrake_b200.assemble import locate_points, point_weights
    mesh = warped(3, 20 + p)
    V = _Space(mesh, p)
    X = mesh.coordinates
    rng = np.random.default_rng(p)
    pts = rng.uniform(X.min(axis=0), X.max(axis=0), (60, 3))
    cells, xi = locate_points(V, pts, 1e-8)
    bc, bxi = so.locate_brute_force(mesh, V.V, pts)
    assert np.array_equal(cells, bc)
    ok = cells >= 0
    assert ok.sum() > 30 and (~ok).any()          # the warped box leaves some of its bounding box outside
    assert np.abs(xi[ok] - bxi[ok]).max() < 1e-10
    idx, w = point_weights(V, cells, xi)
    # the weights reproduce the coordinates (Q1 geometry is in Q_p) and sum to one
    Xd = V.V.dof_coordinates()
    assert np.abs(np.einsum("kj,kji->ki", w[ok], Xd[idx[ok]]) - pts[ok]).max() < 1e-10
    assert np.abs(w[ok].sum(axis=1) - 1.0).max() < 1e-13
    assert (idx[~ok] == -1).all() and (w[~ok] == 0).all()


def test_point_location_shared_entities_and_missing():
    """Points on shared faces, edges and vertices go to the lowest cell number; a point outside is -1, and
    PointEvaluator's "error" names its index."""
    from firedrake_b200.assemble import PointEvaluator, locate_points
    mesh = ExtrudedHexMesh(3, 3, 3, permute_seed=2)
    V = _Space(mesh, 2)
    pts = np.array([[1 / 3, 0.5, 0.5], [1 / 3, 2 / 3, 0.5], [1 / 3, 2 / 3, 1 / 3], [2.0, 0.5, 0.5],
                    [0.0, 0.0, 0.0], [1.0, 1.0, 1.0]])
    cells, _ = locate_points(V, pts, 1e-8)
    bc, _ = so.locate_brute_force(mesh, V.V, pts)
    assert np.array_equal(cells, bc) and cells[3] == -1 and (cells[[0, 1, 2, 4, 5]] >= 0).all()
    # every point on a shared entity lies in several cells; the lowest of them is taken, the same every time
    assert np.array_equal(locate_points(V, pts[::-1], 1e-8)[0][::-1], cells)
    with pytest.raises(ValueError, match="point 3 "):
        PointEvaluator(V, pts)
    with pytest.raises(ValueError, match="missing_points_behaviour"):
        PointEvaluator(V, pts, missing_points_behaviour="warn")


def test_point_adjoint():
    """<E u, a> = <u, E^T a> with the located weights, points sharing cells and nodes included."""
    from firedrake_b200.assemble import locate_points, point_weights
    mesh = warped(3, 7)
    V = _Space(mesh, 3)
    X = V.V.dof_coordinates()
    rng = np.random.default_rng(7)
    pts = np.concatenate([X[rng.choice(len(X), 5)], X[rng.choice(len(X), 5)] * 0.98 + 0.01])
    pw = point_weights(V, *locate_points(V, pts, 1e-8))
    u, a = rng.standard_normal(len(X)), rng.standard_normal(len(pts))
    lhs = so.evaluate(pw, u) @ a
    assert abs(lhs - u @ so.adjoint(pw, a, len(X))) < 1e-12 * np.abs(u).sum()
