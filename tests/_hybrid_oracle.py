"""Dense NumPy oracle of the hybridised mixed Poisson problem (FDB_FORM_MIXED_POISSON_HYBRID, _RECONSTRUCT): the cell
blocks A_K = alpha M_K and B_K of tests/_mixed_poisson_oracle.py, the trace coupling C_K, and every local solve as a
dense ``numpy.linalg.solve`` of the cell's saddle-point matrix -- no elimination order, no packed storage.

    K_K = [[A_K, B_K^T], [B_K, 0]],  C^_K = [C_K 0],  H = sum_K C^_K K_K^-1 C^_K^T,  r = sum_K C^_K K_K^-1 f_K
    (sigma_K, u_K) = K_K^-1 (f_K - C^_K^T lambda),  sigma = sum_K w o sigma_K

C_K[t, sigma-dof(t)] = o_t w_t0 w_t1 for trace dof t (face 2d + s, GL indices t0, t1): o = -1 on side 0, +1 on side 1,
w the k-point Gauss-Legendre weights on [0, 1]."""
import numpy as np

import _mixed_poisson_oracle as mo
from firedrake_b200.fiat_lite import gauss_legendre

SUBS = (1, 2, 3, 4, "bottom", "top")


def face_dof(k, t):
    """(local flux dof, d, s, t0, t1) of trace dof t."""
    f, r = divmod(t, k * k)
    d, s = divmod(f, 2)
    t0, t1 = divmod(r, k)
    idx = [0, 0, 0]
    idx[d] = s
    others = [e for e in range(3) if e != d]
    idx[others[0]], idx[others[1]] = t0, t1
    dims = [k + 1 if e == d else k for e in range(3)]
    return d * k * k * (k + 1) + (idx[0] * dims[1] + idx[1]) * dims[2] + idx[2], d, s, t0, t1


def trace_coupling(k):
    """C_K (6k^2 x 3k^2(k+1)), metric-free."""
    _, w = gauss_legendre(k)
    ns = 3 * k * k * (k + 1)
    C = np.zeros((6 * k * k, ns))
    for t in range(6 * k * k):
        i, d, s, t0, t1 = face_dof(k, t)
        C[t, i] = (1.0 if s else -1.0) * w[t0] * w[t1]
    return C


def cell_data(mesh, S, Q, T):
    """(flux rows, DQ rows, trace rows, vertex coordinates) of every cell."""
    fs, fq, ft = S.full_cell_node_list(), Q.full_cell_node_list(), T.full_cell_node_list()
    fc = mesh.coord_space.full_cell_node_list()
    return [(fs[c], fq[c], ft[c], mesh.coordinates[fc[c]]) for c in range(fs.shape[0])]


def weights(S):
    counts = np.bincount(S.full_cell_node_list().ravel(), minlength=S.node_count)
    return 1.0 / counts


def local_saddle(k, Xv, alpha):
    M, B = mo.element_matrices(k, Xv, alpha)
    nu = B.shape[0]
    return np.block([[M, B.T], [B, np.zeros((nu, nu))]])


def trace_matrix(mesh, S, Q, T, alpha):
    """Dense H (no boundary rows modified)."""
    k = S.degree
    C = trace_coupling(k)
    nu = k ** 3
    Ch = np.hstack([C, np.zeros((C.shape[0], nu))])
    H = np.zeros((T.node_count, T.node_count))
    for rs, rq, rt, Xv in cell_data(mesh, S, Q, T):
        Kk = local_saddle(k, Xv, alpha)
        H[np.ix_(rt, rt)] += Ch @ np.linalg.solve(Kk, Ch.T)
    return H


def eliminate(mesh, S, Q, T, alpha, L0, L1, w=None):
    """r = sum_K C^ K_K^-1 (w o L0, L1)."""
    k = S.degree
    w = weights(S) if w is None else w
    C = trace_coupling(k)
    r = np.zeros(T.node_count)
    for rs, rq, rt, Xv in cell_data(mesh, S, Q, T):
        x = np.linalg.solve(local_saddle(k, Xv, alpha), np.concatenate([w[rs] * L0[rs], L1[rq]]))
        r[rt] += C @ x[:len(rs)]
    return r


def reconstruct(mesh, S, Q, T, alpha, lam, L0, L1, w=None, per_cell=False):
    """(sigma, u) = sum_K (w o sigma_K, u_K); with ``per_cell`` also the list of (flux rows, sigma_K)."""
    k = S.degree
    w = weights(S) if w is None else w
    C = trace_coupling(k)
    sigma, u, cells = np.zeros(S.node_count), np.zeros(Q.node_count), []
    for rs, rq, rt, Xv in cell_data(mesh, S, Q, T):
        g = np.concatenate([w[rs] * L0[rs], L1[rq]])
        g[:len(rs)] -= C.T @ lam[rt]
        x = np.linalg.solve(local_saddle(k, Xv, alpha), g)
        sigma[rs] += w[rs] * x[:len(rs)]
        u[rq] = x[len(rs):]
        cells.append((rs, x[:len(rs)]))
    return (sigma, u, cells) if per_cell else (sigma, u)


def natural_nodes(T, flux_subs):
    subs = [s for s in SUBS if s not in flux_subs]
    return np.unique(np.concatenate([T.boundary_nodes(s) for s in subs])) if subs else np.zeros(0, dtype=int)


def hybrid_solve(mesh, S, Q, T, alpha, L0, L1, flux_subs=(), nullspace=False):
    """The hybridised (sigma, u, lambda): L0 zeroed on the flux-condition rows, lambda = 0 on the natural faces,
    the plain means of L1 and u removed with ``nullspace``."""
    L0, L1 = L0.copy(), L1.copy()
    for s in flux_subs:
        L0[S.boundary_nodes(s)] = 0.0
    if nullspace:
        L1 -= L1.mean()
    H = trace_matrix(mesh, S, Q, T, alpha)
    r = eliminate(mesh, S, Q, T, alpha, L0, L1)
    nat = natural_nodes(T, flux_subs)
    H[nat, :] = 0.0
    H[:, nat] = 0.0
    H[nat, nat] = 1.0
    r[nat] = 0.0
    lam = np.linalg.lstsq(H, r, rcond=None)[0] if nullspace else np.linalg.solve(H, r)
    sigma, u = reconstruct(mesh, S, Q, T, alpha, lam, L0, L1)
    if nullspace:
        u -= u.mean()
    return sigma, u, lam
