"""The eigenvalue oracle on the CPU: the Dirichlet Laplacian of the unit cube, assembled from the element-matrix
oracles, converges to pi^2 (l^2 + m^2 + n^2) at the expected rate 2p, and the symmetry of an unwarped cube shows as
degenerate triples."""
import numpy as np
import pytest

import _eigen_oracle as eo


@pytest.mark.parametrize("p", [1, 2])
def test_unit_cube_rates(p):
    """Observed rates between 4^3 and 8^3 in [2p - 0.3, 2p + 0.5] for the first 7 eigenvalues."""
    l4, exact = eo.unit_cube_dirichlet(4, p, 7)
    l8, _ = eo.unit_cube_dirichlet(8, p, 7)
    assert np.all(l4 >= exact) and np.all(l8 >= exact)          # conforming: the discrete values lie above
    rates = np.log2((l4 - exact) / (l8 - exact))
    assert np.all(rates >= 2 * p - 0.3) and np.all(rates <= 2 * p + 0.5), rates


@pytest.mark.parametrize("p", [1, 2])
def test_unwarped_cube_triples(p):
    """On an unwarped cube 6 pi^2 and 9 pi^2 are triple: the three computed values of each agree to 1e-10."""
    lam, _ = eo.unit_cube_dirichlet(4, p, 7)
    for tri in (lam[1:4], lam[4:7]):
        assert (tri.max() - tri.min()) <= 1e-10 * tri.max(), tri


def test_restricted_eigh_vectors():
    """The reference pairs are M-orthonormal, zero on the constrained rows and solve K x = lambda M x."""
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    mesh = ExtrudedHexMesh(3, 3, 2, warp=0.05, permute_seed=2)
    W = mesh.function_space(2)
    K, M = eo.helmholtz(mesh, W, 2), eo.helmholtz(mesh, W, 2, 0.0, 1.0)
    bd = eo.boundary(W)
    lam, X = eo.restricted_eigh(K, M, bd, 5)
    assert np.abs(X.T @ (M @ X) - np.eye(5)).max() < 1e-12
    assert np.abs(X[bd]).max() == 0.0
    free = np.setdiff1d(np.arange(W.node_count), bd)
    R = (K @ X - (M @ X) * lam)[free]
    assert np.abs(R).max() < 1e-10 * lam.max()
