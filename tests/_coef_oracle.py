"""TEST INFRASTRUCTURE: NumPy oracle of the coefficient form (FDB_FORM_HELMHOLTZ_COEF)

    alpha*inner(kappa*grad(u), grad(v))*dx + beta*inner(u, v)*dx

on Q_p (x) P_p hexahedra with a trilinear (Q1) coordinate field, kappa in the argument space.  A
restatement written for the tests, in the conventions of oracle/hex_kernels.inc: dof (ax*N + ay)*N + az,
vertex (bx*2 + by)*2 + bz, tables B[q][a] / D[q][a] on [0, 1].  Element kernels are batched over cells
and sum-factorised with einsum; the geometry (J, det J, J^{-1}) is taken at every quadrature point.
The wrappers gather / scatter through an extruded map (column map + layer offset) or a native hex map
(offsets zero, one layer)."""
import numpy as np


def _tables(el):
    return np.asarray(el.B), np.asarray(el.D), np.asarray(el.wq), np.asarray(el.xq)


def _t3(A0, A1, A2, x):
    """out[..., i, j, k] = sum_abc A0[i, a] A1[j, b] A2[k, c] x[..., a, b, c]"""
    return np.einsum("ia,jb,kc,...abc->...ijk", A0, A1, A2, x, optimize=True)


def geometry(el, X):
    """X (nc, 8, 3) vertex coordinates -> Kinv (nc, Q, Q, Q, 3, 3) = J^{-1} [reference, physical] and
    detw (nc, Q, Q, Q) = |det J| w_q."""
    _, _, wq, xq = _tables(el)
    CB = np.stack([1.0 - xq, xq], axis=1)                   # (Q, 2) P1 basis at the points
    CD = np.tile([-1.0, 1.0], (len(xq), 1))                 # (Q, 2) its derivative
    Xv = X.reshape(-1, 2, 2, 2, 3)
    J = np.stack([np.einsum("ia,jb,kc,nabcd->nijkd", CD, CB, CB, Xv),
                  np.einsum("ia,jb,kc,nabcd->nijkd", CB, CD, CB, Xv),
                  np.einsum("ia,jb,kc,nabcd->nijkd", CB, CB, CD, Xv)], axis=-1)   # J[..., d, r] = dx_d/dxi_r
    det = np.linalg.det(J)
    w3 = wq[:, None, None] * wq[None, :, None] * wq[None, None, :]
    return np.linalg.inv(J), np.abs(det) * w3


def cell_actions(el, X, u, kappa, alpha=1.0, beta=0.0):
    """Element actions A(kappa)[i] = a(u, phi_i) for a batch of cells: X (nc, 8, 3), u and kappa
    (nc, ND) -> (nc, ND).  ``u`` may carry extra leading batch axes after the cell axis:
    (nc, m, ND) -> (nc, m, ND)."""
    B, D, _, _ = _tables(el)
    n = B.shape[1]
    Kinv, detw = geometry(el, X)
    uu = u.reshape(u.shape[:-1] + (n, n, n))
    extra = uu.ndim - 4                                     # batch axes between cell and dofs
    kq = _t3(B, B, B, kappa.reshape(-1, n, n, n))
    g = np.stack([_t3(D, B, B, uu), _t3(B, D, B, uu), _t3(B, B, D, uu)], axis=-1)      # reference gradient
    ex = lambda a: a.reshape(a.shape[:1] + (1,) * extra + a.shape[1:])
    # flux in reference coordinates: fhat = alpha kappa |det| w  J^{-1} J^{-T} ghat
    M = np.einsum("nijkrd,nijksd->nijkrs", Kinv, Kinv)
    s = alpha * kq * detw
    f = np.einsum("...ijkrs,...ijks->...ijkr", ex(M), g) * ex(s)[..., None]
    m = beta * ex(detw) * _t3(B, B, B, uu)
    out = (_t3(D.T, B.T, B.T, f[..., 0]) + _t3(B.T, D.T, B.T, f[..., 1]) + _t3(B.T, B.T, D.T, f[..., 2])
           + _t3(B.T, B.T, B.T, m))
    return out.reshape(u.shape)


def cell_matrices(el, X, kappa, alpha=1.0, beta=0.0):
    """Element matrices A[i, j] = a(phi_j, phi_i) (row = test, column = trial): (nc, ND, ND)."""
    nd = el.ndof ** 3
    step = max(1, 2048 // nd)                               # cells per batch (memory)
    out = np.empty((X.shape[0], nd, nd))
    for c in range(0, X.shape[0], step):
        e = min(c + step, X.shape[0])
        E = np.broadcast_to(np.eye(nd), (e - c, nd, nd))
        out[c:e] = np.swapaxes(cell_actions(el, X[c:e], E, kappa[c:e], alpha, beta), 1, 2)
    return out


def _cells(map0, off0, map1, off1, nlay):
    """Per (column, layer) cell: dof indices (ncells, ND) and vertex indices (ncells, 8)."""
    lay = np.arange(nlay)
    i0 = (map0[:, None, :] + np.asarray(off0)[None, None, :] * lay[None, :, None]).reshape(-1, map0.shape[1])
    i1 = (map1[:, None, :] + np.asarray(off1)[None, None, :] * lay[None, :, None]).reshape(-1, 8)
    return i0, i1


def action(el, coords, u, kappa, map0, off0, map1, off1, nlay, alpha=1.0, beta=0.0, out=None):
    """assemble(action(a(kappa), u)) over every column and layer (native hexes: nlay = 1 and zero
    offsets)."""
    i0, i1 = _cells(map0, off0, map1, off1, nlay)
    y = np.zeros(len(u)) if out is None else out
    A = cell_actions(el, coords.reshape(-1, 3)[i1], u[i0], kappa[i0], alpha, beta)
    np.add.at(y, i0, A)
    return y


def element_matrices(el, coords, kappa, map0, off0, map1, off1, nlay, alpha=1.0, beta=0.0):
    """(dof indices (ncells, ND), element matrices (ncells, ND, ND))."""
    i0, i1 = _cells(map0, off0, map1, off1, nlay)
    return i0, cell_matrices(el, coords.reshape(-1, 3)[i1], kappa[i0], alpha, beta)


def diagonal(el, coords, kappa, map0, off0, map1, off1, nlay, alpha=1.0, beta=0.0, out=None, nnodes=None):
    i0, A = element_matrices(el, coords, kappa, map0, off0, map1, off1, nlay, alpha, beta)
    d = np.zeros(nnodes if nnodes is not None else len(kappa)) if out is None else out
    np.add.at(d, i0, np.diagonal(A, axis1=1, axis2=2))
    return d


def add_to_csr(rowptr, colidx, vals, i0, A, row_lg=None, col_lg=None):
    """MatSetValuesLocal(ADD_VALUES) of every element matrix into a CSR pattern whose column indices
    are sorted within each row; rows / columns mapped to a negative index by the lgmaps are dropped."""
    nd = i0.shape[1]
    r = np.repeat(i0, nd, axis=1).ravel()
    c = np.tile(i0, (1, nd)).ravel()
    v = A.reshape(-1)
    if row_lg is not None:
        r = np.asarray(row_lg)[r]
    if col_lg is not None:
        c = np.asarray(col_lg)[c]
    keep = (r >= 0) & (c >= 0)
    r, c, v = r[keep].astype(np.int64), c[keep].astype(np.int64), v[keep]
    n = len(rowptr) - 1
    prow = np.repeat(np.arange(n, dtype=np.int64), np.diff(rowptr))
    key = prow * (n + 1) + np.asarray(colidx, dtype=np.int64)
    pos = np.searchsorted(key, r * (n + 1) + c)
    assert np.array_equal(key[pos], r * (n + 1) + c), "entry outside the sparsity pattern"
    np.add.at(vals, pos, v)
    return vals
