"""CPU checks of the p-multigrid reference (tests/_pmg_oracle.py) and of the host-side pieces the kernels and the
smoother rely on: exact endpoint rows, inject o prolong = id, polynomial exactness, the weighted restriction = P^T,
and the Chebyshev coefficients against the recurrence written out on a scipy matrix."""
import numpy as np
import pytest
import scipy.sparse as sp

import _pmg_oracle as po
from firedrake_b200 import mg, op2
from firedrake_b200.utility_meshes import ExtrudedHexMesh

PAIRS = [(2, 1), (3, 1), (3, 2)]


@pytest.mark.parametrize("p,q", PAIRS)
def test_endpoint_rows_exact(p, q):
    """The tables the engine receives: endpoint rows exact unit vectors, the rest equal to the oracle's."""
    P, R = op2.p_transfer_tables(p, q)
    Po, Ro = po.tables(p, q)
    for T, To in ((P, Po), (R, Ro)):
        assert np.array_equal(T[0], np.eye(T.shape[1])[0]) and np.array_equal(T[1], np.eye(T.shape[1])[1])
        np.testing.assert_allclose(T, To, rtol=0, atol=1e-14)
    # P's columns sum to one (partition of unity), and R P = I (the coarse nodes are nested in the fine space)
    np.testing.assert_allclose(P.sum(axis=1), 1.0, atol=1e-14)
    np.testing.assert_allclose(R @ P, np.eye(q + 1), atol=1e-14)


@pytest.mark.parametrize("p,q", PAIRS)
def test_inject_prolong_identity(p, q):
    mesh = ExtrudedHexMesh(3, 2, 2, warp=0.05, permute_seed=3)
    Vf, Vc = mesh.function_space(p), mesh.function_space(q)
    G = po.global_injection(Vf, Vc) @ po.global_prolongation(Vf, Vc)
    np.testing.assert_allclose(G, np.eye(Vc.node_count), atol=1e-13)


@pytest.mark.parametrize("p,q", PAIRS)
def test_polynomial_prolonged_exactly(p, q):
    """On an affine mesh a degree-q polynomial in CG_q is the same polynomial in CG_p."""
    mesh = ExtrudedHexMesh(3, 2, 4, Lx=1.5, Ly=0.7, Lz=1.1, permute_seed=1)
    Vf, Vc = mesh.function_space(p), mesh.function_space(q)

    def f(X):
        x, y, z = X.T
        return (1 + x - 2 * y + 0.5 * z) ** q + x ** q * y * z ** min(q, 1)
    cf = po.prolong(Vf, Vc, f(Vc.dof_coordinates()))
    np.testing.assert_allclose(cf, f(Vf.dof_coordinates()), rtol=0, atol=1e-12)


@pytest.mark.parametrize("p,q", PAIRS)
@pytest.mark.parametrize("cdim", [1, 3])
def test_weighted_restrict_is_transpose(p, q, cdim):
    """coarse += P^T (w o fine) cell by cell, w = 1 / multiplicity, is exactly the transpose of the global
    prolongation: dense check with a permuted numbering."""
    mesh = ExtrudedHexMesh(3, 3, 2, warp=0.05, permute_seed=7)
    Vf, Vc = mesh.function_space(p), mesh.function_space(q)
    fine = np.random.default_rng(0).standard_normal((Vf.node_count, cdim)).squeeze()
    want = np.einsum("ji,j...->i...", po.global_prolongation(Vf, Vc), fine)
    np.testing.assert_allclose(po.restrict_cellwise(Vf, Vc, fine), want, rtol=1e-13, atol=1e-13)


def test_level_degrees():
    assert mg.pmg_degrees(3) == [1, 3] and mg.pmg_degrees(2) == [1, 2]
    assert mg.pmg_degrees(3, 2) == [2, 3] and mg.pmg_degrees(3, 1, halve=False) == [1, 3]
    assert mg.pmg_degrees(5) == [1, 2, 5] and mg.pmg_degrees(5, halve=False) == [1, 5]


@pytest.mark.parametrize("k", [1, 2, 4])
def test_chebyshev_recurrence(k):
    """The fused steps with mg.chebyshev_coefficients reproduce the recurrence written out, and the error after k
    steps is T_k((theta - D^-1 A) / delta) / T_k(theta / delta) applied to the initial error."""
    n = 40
    A = sp.diags([-1.0, 2.5, -1.0], [-1, 0, 1], shape=(n, n)).tocsr() + sp.diags(np.linspace(0, 1, n))
    rng = np.random.default_rng(2)
    b, x0 = rng.standard_normal(n), rng.standard_normal(n)
    dinv = 1.0 / A.diagonal()
    lam = np.linalg.eigvals(np.diag(dinv) @ A.toarray()).real
    emin, emax = 0.1 * lam.max(), 1.1 * lam.max()
    x, d = x0.copy(), np.zeros(n)
    for cd, cz in mg.chebyshev_coefficients(emin, emax, k):
        po.chebyshev_step(cd, cz, b, A @ x, dinv, d, x)
    np.testing.assert_allclose(x, po.chebyshev(A, b, x0, dinv, emin, emax, k), rtol=1e-13, atol=1e-13)
    # the error polynomial
    xs = np.linalg.solve(A.toarray(), b)
    S = np.diag(np.sqrt(dinv))                              # D^-1 A = S M S^-1, M = D^-1/2 A D^-1/2
    M = np.diag(np.sqrt(dinv)) @ A.toarray() @ np.diag(np.sqrt(dinv))
    ev, Q = np.linalg.eigh(M)
    theta, delta = 0.5 * (emax + emin), 0.5 * (emax - emin)
    T = np.polynomial.chebyshev.Chebyshev.basis(k)
    g = T((theta - ev) / delta) / T(theta / delta)
    e = S @ Q @ np.diag(g) @ Q.T @ np.linalg.inv(S) @ (x0 - xs)
    np.testing.assert_allclose(x - xs, e, atol=1e-11)


def _stiffness(V, h):
    """The assembled Poisson operator of CG_p on a mesh of cubes of side h, from the Kronecker cell matrix
    h (K (x) M (x) M + M (x) K (x) M + M (x) M (x) K) of the 1-D GLL tables (Gauss rule of p+1 points)."""
    from firedrake_b200.fiat_lite import interval_element
    el = interval_element(V.degree)
    W = np.diag(el.wq)
    M1, K1 = el.B.T @ W @ el.B, el.D.T @ W @ el.D
    Ke = h * (np.kron(np.kron(K1, M1), M1) + np.kron(np.kron(M1, K1), M1) + np.kron(np.kron(M1, M1), K1))
    cells = V.full_cell_node_list().astype(np.int64)
    n = Ke.shape[0]
    rows, cols = np.repeat(cells, n, axis=1).ravel(), np.tile(cells, (1, n)).ravel()
    return sp.csr_matrix((np.tile(Ke.ravel(), len(cells)), (rows, cols)), shape=(V.node_count,) * 2)


def two_level_radius(p, n, nu=2):
    """The spectral radius of the error propagation E = S (I - P Ac^-1 P^T A) S of two-level PMG (CG_p over a
    rediscretised CG1, Dirichlet bottom and top) on n^3 unit cubes, S = nu Chebyshev-Jacobi iterations with the
    coefficients of mg.chebyshev_coefficients and PETSc's bounds (0.1, 1.1) x lmax(D^-1 A)."""
    import scipy.sparse.linalg as sla
    mesh = ExtrudedHexMesh(n, n, n)
    Vf, Vc = mesh.function_space(p), mesh.function_space(1)

    def free(V):
        bc = np.union1d(V.boundary_nodes("bottom"), V.boundary_nodes("top"))
        return np.setdiff1d(np.arange(V.node_count), bc)
    ff, fc = free(Vf), free(Vc)
    A = _stiffness(Vf, 1.0 / n)[ff][:, ff].tocsc()
    Ac = sla.splu(_stiffness(Vc, 1.0 / n)[fc][:, fc].tocsc())
    P = sp.csr_matrix(po.global_prolongation(Vf, Vc)[np.ix_(ff, fc)])
    dinv = 1.0 / A.diagonal()
    Dh = sp.diags(np.sqrt(dinv))
    lmax = sla.eigsh(Dh @ A @ Dh, k=1, which="LA", return_eigenvectors=False)[0]
    coef = mg.chebyshev_coefficients(0.1 * lmax, 1.1 * lmax, nu)

    def smooth(e):
        d = np.zeros_like(e)
        for cd, cz in coef:
            po.chebyshev_step(cd, cz, np.zeros_like(e), A @ e, dinv, d, e)
        return e

    def E(e):
        e = smooth(np.array(e, dtype=float).ravel())
        e = e - P @ Ac.solve(P.T @ (A @ e))
        return smooth(e)
    op = sla.LinearOperator((len(ff),) * 2, matvec=E, dtype=float)
    return float(np.abs(sla.eigs(op, k=1, which="LM", return_eigenvectors=False, tol=1e-6)[0]))


@pytest.mark.parametrize("p", [2, 3])
def test_two_level_spectral_radius(p):
    """Two-level PMG contracts and does not degrade from 4^3 to 8^3 (0.282 and 0.283 at CG2, 0.324 and 0.326 at
    CG3)."""
    r4, r8 = two_level_radius(p, 4), two_level_radius(p, 8)
    print(f"CG{p}: rho(4^3) = {r4:.3f}, rho(8^3) = {r8:.3f}")
    assert r4 < 0.5 and r8 < 0.5
    assert r8 <= r4 + 0.05
