"""TEST INFRASTRUCTURE: global stiffness and mass matrices (scipy.sparse) of the forms the eigensolver takes, built from
the NumPy element-matrix oracles (tests/_coef_oracle.py, _elasticity_oracle.py, _sem_oracle.py, _dg_oracle.py), and the
reference eigenpairs of the restricted problems from scipy.linalg.eigh on dense matrices (small sizes only)."""
import numpy as np
import scipy.linalg as sl
import scipy.sparse as sps

import _coef_oracle as co
import _dg_oracle as do
import _elasticity_oracle as eo
import _sem_oracle as so
from firedrake_b200.fiat_lite import interval_element


def _geo(mesh, W):
    return (W.cell_node_map, W.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)


def _scatter(i0, A, n):
    nd = i0.shape[1]
    r = np.repeat(i0, nd, axis=1).ravel()
    c = np.tile(i0, (1, nd)).ravel()
    return sps.csr_matrix((A.ravel(), (r, c)), shape=(n, n))


def helmholtz(mesh, W, p, alpha=1.0, beta=0.0, kappa=None):
    """Form(V, alpha, beta, kappa) on the scalar CG_p space W = mesh.function_space(p)."""
    k = np.ones(W.node_count) if kappa is None else np.asarray(kappa)
    i0, A = co.element_matrices(interval_element(p), mesh.coordinates, k, *_geo(mesh, W), alpha=alpha, beta=beta)
    return _scatter(i0, A, W.node_count)


def elasticity(mesh, W, p, mu, lmbda, beta=0.0):
    """Elasticity(V, mu, lmbda, beta) on the vector CG_p space (3 dofs per node, AoS)."""
    return eo.global_matrix(interval_element(p), mesh.coordinates, _geo(mesh, W), W.node_count, mu, lmbda,
                            beta).tocsr()


def vector_mass(mesh, W, p):
    """mass(V) on the vector space: the scalar mass on each component (AoS)."""
    return sps.kron(helmholtz(mesh, W, p, 0.0, 1.0), sps.eye(3)).tocsr()


def spectral(mesh, W, p, alpha=1.0, beta=0.0, kappa=None):
    """SpectralForm(V, alpha, beta, kappa): the GLL-collocated operator; (0, 1) is the lumped (diagonal) mass."""
    return so.operator(mesh, W, p, alpha, beta, kappa)


def interior_penalty(mesh, W, p, alpha, beta, eta, weak_bcs="on_boundary"):
    """InteriorPenalty(V, alpha, beta, eta, weak_bcs) on DQ_p (W = mesh.dg_function_space(p))."""
    return do.operator(mesh, W, do.element(p), alpha, beta, eta, weak_bcs).tocsr()


def dg_mass(mesh, W, p):
    return do.cell_matrix(mesh, W, do.element(p), 0.0, 1.0).tocsr()


WALLS = (1, 2, 3, 4, "bottom", "top")


def boundary(W, sub_domains=WALLS):
    """The nodes of W on the given sub-domains (all six walls by default)."""
    return np.unique(np.concatenate([W.boundary_nodes(s) for s in sub_domains]))


def restricted_eigh(K, M, constrained=(), n=None):
    """The eigenpairs of K x = lambda M x on the rows and columns not in ``constrained`` (dense eigh), ascending; the
    eigenvectors are M-orthonormal and zero on the constrained rows."""
    N = K.shape[0]
    free = np.setdiff1d(np.arange(N), np.asarray(constrained, dtype=np.int64))
    Kf, Mf = K[free][:, free], M[free][:, free]
    if n is not None and len(free) > 1500:
        # the smallest n by shift-and-invert about 0 (a sparse LU of Kf), converged to machine precision
        import scipy.sparse.linalg as spla
        lam, U = spla.eigsh(Kf.tocsc(), k=n, M=Mf.tocsc(), sigma=0.0, which="LM", tol=0.0)
        o = np.argsort(lam)
        lam, U = lam[o], U[:, o]
        U = U / np.sqrt(np.einsum("ij,ij->j", U, Mf @ U))
    else:
        Kf, Mf = Kf.toarray(), Mf.toarray()
        sub = None if n is None else (0, min(n, len(free)) - 1)
        lam, U = sl.eigh((Kf + Kf.T) / 2, (Mf + Mf.T) / 2, subset_by_index=sub)
    X = np.zeros((N, U.shape[1]))
    X[free] = U
    return lam, X


def unit_cube_dirichlet(n, p, count=10):
    """The smallest ``count`` Dirichlet-Laplacian eigenvalues on the unit cube, CG_p on an n^3 unwarped mesh, and the
    exact ones pi^2 (l^2 + m^2 + n^2)."""
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    mesh = ExtrudedHexMesh(n, n, n)
    W = mesh.function_space(p)
    K = helmholtz(mesh, W, p, 1.0, 0.0)
    M = helmholtz(mesh, W, p, 0.0, 1.0)
    lam, _ = restricted_eigh(K, M, boundary(W), count)
    return lam, exact_cube(count)


def exact_cube(count):
    v = sorted(l * l + m * m + k * k for l in range(1, 8) for m in range(1, 8) for k in range(1, 8))
    return np.pi ** 2 * np.array(v[:count], dtype=float)
