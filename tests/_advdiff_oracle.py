"""TEST INFRASTRUCTURE: NumPy oracle of advection-diffusion (FDB_FORM_ADVECTION_DIFFUSION)

    alpha*inner(grad(u), grad(v))*dx + inner(dot(b, grad(u)), v)*dx + beta*inner(u, v)*dx

on Q_p (x) P_p hexahedra with a trilinear (Q1) coordinate field and the velocity b given by 3 values per
node of the scalar space (AoS).  Built on tests/_coef_oracle.py: its tables, geometry, cell lists and CSR
insertion, with the diffusion and mass terms taken from its coefficient form at kappa = 1.  The
convective term is the physical gradient J^{-T} ghat dotted with b at every Gauss point, weighted by
|det J| w_q and tested against the basis functions' values."""
import numpy as np
import scipy.sparse as sps
import scipy.sparse.linalg as spla

import _coef_oracle as co


def convective_actions(el, X, u, b):
    """The convective part C(b)[i] = inner(dot(b, grad(u)), phi_i)*dx for a batch of cells: X (nc, 8, 3),
    u (nc, ND) or (nc, m, ND), b (nc, ND, 3) -> the shape of u."""
    B, D, _, _ = co._tables(el)
    n = B.shape[1]
    Kinv, detw = co.geometry(el, X)
    uu = u.reshape(u.shape[:-1] + (n, n, n))
    extra = uu.ndim - 4
    ex = lambda a: a.reshape(a.shape[:1] + (1,) * extra + a.shape[1:])
    bq = np.stack([co._t3(B, B, B, b[..., c].reshape(-1, n, n, n)) for c in range(3)], axis=-1)
    g = np.stack([co._t3(D, B, B, uu), co._t3(B, D, B, uu), co._t3(B, B, D, uu)], axis=-1)
    grad = np.einsum("...ijkrd,...ijkr->...ijkd", ex(Kinv), g)          # grad_d = sum_r dxi_r/dx_d ghat_r
    conv = ex(detw) * np.einsum("...ijkd,...ijkd->...ijk", ex(bq), grad)
    return co._t3(B.T, B.T, B.T, conv).reshape(u.shape)


def cell_actions(el, X, u, b, alpha=1.0, beta=0.0):
    """Element actions A(b)[i] = a(u, phi_i): the coefficient form at kappa = 1 plus the convective part."""
    nd = el.ndof ** 3
    return co.cell_actions(el, X, u, np.ones((X.shape[0], nd)), alpha, beta) + convective_actions(el, X, u, b)


def cell_matrices(el, X, b, alpha=1.0, beta=0.0, convective_only=False):
    """Element matrices A[i, j] = a(phi_j, phi_i) (row = test, column = trial): (nc, ND, ND)."""
    nd = el.ndof ** 3
    step = max(1, 2048 // nd)
    out = np.empty((X.shape[0], nd, nd))
    for c in range(0, X.shape[0], step):
        e = min(c + step, X.shape[0])
        E = np.broadcast_to(np.eye(nd), (e - c, nd, nd))
        A = convective_actions(el, X[c:e], E, b[c:e]) if convective_only else \
            cell_actions(el, X[c:e], E, b[c:e], alpha, beta)
        out[c:e] = np.swapaxes(A, 1, 2)
    return out


def _b_cells(b, i0):
    return np.asarray(b).reshape(-1, 3)[i0]


def action(el, coords, u, b, map0, off0, map1, off1, nlay, alpha=1.0, beta=0.0, out=None):
    """assemble(action(a(b), u)) over every column and layer (native hexes: nlay = 1, zero offsets)."""
    i0, i1 = co._cells(map0, off0, map1, off1, nlay)
    y = np.zeros(len(u)) if out is None else out
    np.add.at(y, i0, cell_actions(el, coords.reshape(-1, 3)[i1], u[i0], _b_cells(b, i0), alpha, beta))
    return y


def element_matrices(el, coords, b, map0, off0, map1, off1, nlay, alpha=1.0, beta=0.0, convective_only=False):
    """(dof indices (ncells, ND), element matrices (ncells, ND, ND))."""
    i0, i1 = co._cells(map0, off0, map1, off1, nlay)
    return i0, cell_matrices(el, coords.reshape(-1, 3)[i1], _b_cells(b, i0), alpha, beta, convective_only)


def diagonal(el, coords, b, map0, off0, map1, off1, nlay, alpha=1.0, beta=0.0, out=None, nnodes=None):
    i0, A = element_matrices(el, coords, b, map0, off0, map1, off1, nlay, alpha, beta)
    d = np.zeros(nnodes if nnodes is not None else len(b) // 3) if out is None else out
    np.add.at(d, i0, np.diagonal(A, axis1=1, axis2=2))
    return d


def csr(el, coords, b, map0, off0, map1, off1, nlay, alpha=1.0, beta=0.0, nnodes=None, convective_only=False):
    """The global matrix (row = test dof, column = trial dof) as a scipy CSR matrix."""
    i0, A = element_matrices(el, coords, b, map0, off0, map1, off1, nlay, alpha, beta, convective_only)
    n = nnodes if nnodes is not None else len(b) // 3
    nd = i0.shape[1]
    rows = np.repeat(i0, nd, axis=1).ravel()
    cols = np.tile(i0, (1, nd)).ravel()
    return sps.csr_matrix((A.reshape(-1), (rows, cols)), shape=(n, n))


def solve(A, rhs, bc_nodes, bc_values):
    """A u = rhs with u = bc_values on bc_nodes (rows replaced by the identity, values lifted), by
    scipy's sparse LU."""
    A = sps.csr_matrix(A, copy=True)
    n = A.shape[0]
    g = np.zeros(n)
    g[bc_nodes] = np.asarray(bc_values)[bc_nodes] if np.ndim(bc_values) else bc_values
    r = rhs - A @ g
    free = np.ones(n, dtype=bool)
    free[bc_nodes] = False
    u = g.copy()
    u[free] = spla.spsolve(A[free][:, free].tocsc(), r[free])
    return u
