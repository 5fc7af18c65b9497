"""CPU checks of the GTMG oracle (tests/_gtmg_oracle.py): P reproduces constants and affine functions at the trace
points, the energy identity (P p)^T H (P p) = p^T A p / alpha for affine p that makes Form(P1, 1/alpha, 0) the right
coarse operator, and a SciPy two-level cycle whose trace-CG iteration count stays bounded under refinement while
Jacobi-CG grows -- with natural data, flux conditions, and flux conditions everywhere with the constant nullspace."""
import numpy as np
import pytest
import scipy.sparse as sp

import _gtmg_oracle as go
import _hybrid_oracle as ho
from firedrake_b200.fiat_lite import gauss_legendre
from firedrake_b200.utility_meshes import ExtrudedHexMesh


def _spaces(n, k, warp=0.0, permute_seed=None):
    mesh = ExtrudedHexMesh(*n, warp=warp, permute_seed=permute_seed)
    return mesh, mesh.hdiv_function_space(k), mesh.dg_function_space(k - 1), mesh.trace_function_space(k - 1), \
        mesh.function_space(1)


@pytest.mark.parametrize("k", [2, 3])
def test_prolongation_reproduces_constants_and_affine_functions(k):
    """P 1 = 1, and P applied to the vertex values of an affine function gives its values at the trace points,
    which on a warped mesh are the trilinear images of the reference points (so the coordinates themselves)."""
    mesh, S, Q, T, V1 = _spaces((3, 2, 2), k, warp=0.05, permute_seed=3)
    P = go.prolongation(T, V1)
    assert np.abs(P @ np.ones(V1.node_count) - 1.0).max() < 1e-14
    X = mesh.coordinates                      # CG1 and the coordinates share one numbering
    assert X.shape[0] == V1.node_count
    ft, fc = T.full_cell_node_list(), mesh.coord_space.full_cell_node_list()
    Pl = go.trilinear(go.reference_points(k))
    ref = np.zeros((T.node_count, 3))
    for c in range(ft.shape[0]):
        ref[ft[c]] = Pl @ X[fc[c]]
    a, b = np.array([0.3, -1.2, 0.7]), 0.4
    assert np.abs(P @ (X @ a + b) - (ref @ a + b)).max() < 1e-13
    # on an unwarped mesh the points are the GL points of every face
    mesh, S, Q, T, V1 = _spaces((2, 2, 2), k)
    P = go.prolongation(T, V1)
    x, _ = gauss_legendre(k)
    Y = P @ mesh.coordinates
    ft = T.full_cell_node_list()
    pts = go.reference_points(k)
    for c in (0, ft.shape[0] - 1):
        lo = mesh.coordinates[mesh.coord_space.full_cell_node_list()[c][0]]
        assert np.abs(Y[ft[c]] - (lo + pts * 0.5)).max() < 1e-14
    assert set(np.round(pts[pts[:, 0] == 0.0][:, 1], 14)) == set(np.round(x, 14))


@pytest.mark.parametrize("k", [2, 3])
def test_energy_identity_for_affine_functions(k):
    """(P p)^T H (P p) = p^T A p / alpha to 1e-12 for affine p, alpha != 1, no masked faces."""
    alpha = 0.6
    mesh, S, Q, T, V1 = _spaces((2, 3, 2), k)
    H = go.trace_matrix(mesh, S, Q, T, alpha)
    A = go.stiffness(mesh, V1)
    P = go.prolongation(T, V1)
    X = mesh.coordinates
    for a, b in [((1.0, 0.0, 0.0), 0.0), ((0.2, -0.7, 1.3), 2.0)]:
        p = X @ np.array(a) + b
        lhs = (P @ p) @ (H @ (P @ p))
        rhs = p @ (A @ p) / alpha
        assert abs(lhs - rhs) < 1e-12 * abs(rhs), (lhs, rhs)


def _iterations(n, k, flux_subs, nullspace, coarse_rtol=None, warp=0.0, alpha=1.0):
    mesh, S, Q, T, V1 = _spaces(n, k, warp=warp)
    nat_subs = [s for s in ho.SUBS if s not in flux_subs]
    nat_t = ho.natural_nodes(T, flux_subs)
    nat_c = go.cg1_boundary_nodes(V1, nat_subs)
    H = go.masked(go.trace_matrix(mesh, S, Q, T, alpha), nat_t)
    A = go.masked(go.stiffness(mesh, V1, 1.0 / alpha), nat_c)
    P = go.prolongation(T, V1)
    r = np.random.default_rng(7).standard_normal(T.node_count)
    r[nat_t] = 0.0
    dinv = 1.0 / H.diagonal()
    _, it_j = go.pcg(H, r, lambda v: dinv * v, nullspace=nullspace)
    M = go.TwoLevel(H, A, P, nat_t, nat_c, nu=3, coarse_rtol=coarse_rtol, nullspace=nullspace)
    x, it_g = go.pcg(H, r, M, nullspace=nullspace)
    rr = r - r.mean() if nullspace else r
    assert np.linalg.norm(rr - H @ x) <= 1e-7 * np.linalg.norm(rr)
    return it_j, it_g


@pytest.mark.parametrize("case", ["natural", "flux", "all_flux"])
def test_two_level_cycle_keeps_iterations_bounded(case):
    """k = 2 at 4^3 and 8^3: GTMG-CG needs at most 10 iterations at both sizes, while Jacobi-CG grows."""
    flux = {"natural": (), "flux": (1, "top"), "all_flux": ho.SUBS}[case]
    ns = case == "all_flux"
    j4, g4 = _iterations((4, 4, 4), 2, flux, ns)
    j8, g8 = _iterations((8, 8, 8), 2, flux, ns)
    assert g4 <= 10 and g8 <= 10, (g4, g8)
    assert j8 > j4 * 1.5, (j4, j8)
    assert g8 < j8 / 3


def test_inexact_coarse_solve_and_k3():
    """A Jacobi-CG coarse solve to 1e-3 on a warped mesh, and k = 3, stay bounded as well."""
    _, g = _iterations((6, 6, 6), 2, (), False, coarse_rtol=1e-3, warp=0.06)
    assert g <= 10, g
    j, g = _iterations((4, 4, 4), 3, (2,), False, alpha=0.5, warp=0.06)
    assert g <= 10 and g < j, (j, g)


def test_restriction_is_the_weighted_transpose():
    """sum over cells of P_K^T (w o lambda_K) = P^T lambda: the weights make the cell-wise restriction exact."""
    mesh, S, Q, T, V1 = _spaces((2, 2, 3), 2, warp=0.04)
    P = go.prolongation(T, V1)
    lam = np.random.default_rng(1).standard_normal(T.node_count)
    w = go.trace_weights(T)
    Pl = go.trilinear(go.reference_points(2))
    ft, fv = T.full_cell_node_list(), V1.full_cell_node_list()
    c = np.zeros(V1.node_count)
    for i in range(ft.shape[0]):
        np.add.at(c, fv[i], Pl.T @ (w[ft[i]] * lam[ft[i]]))
    assert np.abs(c - P.T @ lam).max() < 1e-13 * np.abs(c).max()
    assert isinstance(P, sp.csr_matrix)
