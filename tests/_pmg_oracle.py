"""NumPy reference for the p-multigrid transfers and the Chebyshev smoother: 1-D tables from Lagrange interpolation
on GLL nodes, dense global transfer matrices assembled cell by cell, and the Chebyshev iteration on a dense or
scipy matrix.  Test infrastructure only."""
import numpy as np

from firedrake_b200.fiat_lite import gll_points


def dof_nodes(p):
    """GLL nodes of CG_p in 1-D dof numbering: the two ends first, then the interior."""
    x = gll_points(p)
    return x[np.array([0, p] + list(range(1, p)))]


def lagrange(nodes, pts):
    """(len(pts), len(nodes)): the Lagrange basis through ``nodes`` at ``pts``."""
    out = np.ones((len(pts), len(nodes)))
    for a, xa in enumerate(nodes):
        for b, xb in enumerate(nodes):
            if a != b:
                out[:, a] *= (pts - xb) / (xa - xb)
    return out


def tables(p, q):
    """P (p+1, q+1): the coarse basis at the fine nodes; R (q+1, p+1): the fine basis at the coarse nodes."""
    return lagrange(dof_nodes(q), dof_nodes(p)), lagrange(dof_nodes(p), dof_nodes(q))


def _kron3(T):
    return np.kron(np.kron(T, T), T)


def global_prolongation(Vf, Vc):
    """Dense (fine nodes, coarse nodes) matrix of the prolongation, cell by cell: a node shared by several cells
    gets the same row from each."""
    P, _ = tables(Vf.degree, Vc.degree)
    loc = _kron3(P)
    ff, cf = Vf.full_cell_node_list(), Vc.full_cell_node_list()
    G = np.zeros((Vf.node_count, Vc.node_count))
    for rf, rc in zip(ff, cf):
        G[np.ix_(rf, rc)] = loc
    return G


def global_injection(Vf, Vc):
    """Dense (coarse nodes, fine nodes) matrix of the injection."""
    _, R = tables(Vf.degree, Vc.degree)
    loc = _kron3(R)
    ff, cf = Vf.full_cell_node_list(), Vc.full_cell_node_list()
    G = np.zeros((Vc.node_count, Vf.node_count))
    for rf, rc in zip(ff, cf):
        G[np.ix_(rc, rf)] = loc
    return G


def weights(Vf):
    """1 / (number of cells containing each fine node)."""
    return 1.0 / np.bincount(Vf.full_cell_node_list().ravel(), minlength=Vf.node_count)


def restrict_cellwise(Vf, Vc, fine):
    """The kernel's algorithm on the host: coarse += P^T (w o fine) cell by cell.  ``fine``: (nodes,) or (nodes,
    cdim)."""
    P, _ = tables(Vf.degree, Vc.degree)
    loc = _kron3(P)
    w = weights(Vf)
    wf = fine * (w if fine.ndim == 1 else w[:, None])
    out = np.zeros((Vc.node_count,) + fine.shape[1:])
    for rf, rc in zip(Vf.full_cell_node_list(), Vc.full_cell_node_list()):
        np.add.at(out, rc, loc.T @ wf[rf])
    return out


def prolong(Vf, Vc, coarse):
    return np.einsum("ij,j...->i...", global_prolongation(Vf, Vc), coarse)


def inject(Vf, Vc, fine):
    return np.einsum("ij,j...->i...", global_injection(Vf, Vc), fine)


def chebyshev_step(cd, cz, b, ax, dinv, d, x):
    """The fused step of fdb_vec_chebyshev: d = cd d + cz dinv (b - ax); x += d (in place)."""
    z = cz * (dinv * (b - ax))
    d[:] = z if cd == 0.0 else cd * d + z
    x += d


def chebyshev(A, b, x, dinv, emin, emax, k):
    """k Chebyshev-Jacobi iterations on A x = b from x (Saad, Algorithm 12.1), written out directly."""
    theta, delta = 0.5 * (emax + emin), 0.5 * (emax - emin)
    sigma = theta / delta
    rho = 1.0 / sigma
    x = x.copy()
    d = dinv * (b - A @ x) / theta
    x += d
    for _ in range(k - 1):
        rho_new = 1.0 / (2.0 * sigma - rho)
        d = rho_new * rho * d + 2.0 * rho_new / delta * (dinv * (b - A @ x))
        x += d
        rho = rho_new
    return x
