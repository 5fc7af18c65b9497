"""TEST INFRASTRUCTURE: NumPy oracle of linear elasticity (FDB_FORM_ELASTICITY)

    a(u, v) = inner(sigma(u), grad(v))*dx + beta*inner(u, v)*dx,
    sigma(u) = mu (grad u + grad u^T) + lmbda tr(grad u) I

on vector (3 components, AoS) Q_p (x) P_p hexahedra with a trilinear coordinate field.  Built on the
coefficient oracle's geometry, tensor contraction, cell gather and CSR insertion (tests/_coef_oracle.py):
dof (ax*N + ay)*N + az, vertex (bx*2 + by)*2 + bz, component fastest (dof index 3*node + component)."""
import numpy as np

from _coef_oracle import _cells, _t3, add_to_csr, geometry


def cell_actions(el, X, u, mu, lmbda, beta=0.0):
    """Element actions for a batch of cells: X (nc, 8, 3), u (nc, [m,] ND, 3) -> same shape as u."""
    B, D = np.asarray(el.B), np.asarray(el.D)
    n = B.shape[1]
    Kinv, detw = geometry(el, X)                            # Kinv[..., m, k] = dxi_m / dx_k
    uu = np.moveaxis(u, -1, -2).reshape(u.shape[:-2] + (3, n, n, n))     # (..., d, a, b, c)
    extra = uu.ndim - 5
    ex = lambda a: a.reshape(a.shape[:1] + (1,) * extra + a.shape[1:])
    gh = np.stack([_t3(D, B, B, uu), _t3(B, D, B, uu), _t3(B, B, D, uu)], axis=-1)   # (..., d, Q, Q, Q, m)
    G = np.einsum("...dijkm,...ijkme->...ijkde", gh, ex(Kinv))                        # (..., Q, Q, Q, d, e)
    tr = np.trace(G, axis1=-2, axis2=-1)
    S = mu * (G + np.swapaxes(G, -1, -2)) + lmbda * tr[..., None, None] * np.eye(3)
    f = np.einsum("...ijkme,...ijkde->...dijkm", ex(Kinv), S) * ex(detw)[..., None, :, :, :, None]
    m = beta * ex(detw)[..., None, :, :, :] * _t3(B, B, B, uu)
    out = (_t3(D.T, B.T, B.T, f[..., 0]) + _t3(B.T, D.T, B.T, f[..., 1]) + _t3(B.T, B.T, D.T, f[..., 2])
           + _t3(B.T, B.T, B.T, m))
    return np.moveaxis(out.reshape(u.shape[:-2] + (3, n ** 3)), -2, -1)


def cell_matrices(el, X, mu, lmbda, beta=0.0):
    """Element matrices A[3i + a, 3j + b] = a(phi_j e_b, phi_i e_a): (nc, 3 ND, 3 ND)."""
    nd = el.ndof ** 3
    step = max(1, 1024 // nd)
    out = np.empty((X.shape[0], 3 * nd, 3 * nd))
    E = np.eye(3 * nd).reshape(3 * nd, nd, 3)
    for c in range(0, X.shape[0], step):
        e = min(c + step, X.shape[0])
        Y = cell_actions(el, X[c:e], np.broadcast_to(E, (e - c,) + E.shape), mu, lmbda, beta)   # (nc, col, ND, 3)
        out[c:e] = np.swapaxes(Y.reshape(e - c, 3 * nd, 3 * nd), 1, 2)
    return out


def dofs(i0):
    """Dof indices (ncells, 3 ND) of node indices (ncells, ND)."""
    return (3 * i0[:, :, None] + np.arange(3)).reshape(i0.shape[0], -1)


def action(el, coords, u, map0, off0, map1, off1, nlay, mu, lmbda, beta=0.0, out=None):
    """assemble(action(a, u)) over every column and layer; u and the result are flat AoS (3 per node)."""
    i0, i1 = _cells(map0, off0, map1, off1, nlay)
    y = np.zeros(len(u)) if out is None else out
    uv = np.asarray(u).reshape(-1, 3)
    A = cell_actions(el, coords.reshape(-1, 3)[i1], uv[i0], mu, lmbda, beta)
    np.add.at(y.reshape(-1, 3), i0, A)
    return y


def element_matrices(el, coords, map0, off0, map1, off1, nlay, mu, lmbda, beta=0.0):
    """(dof indices (ncells, 3 ND), element matrices (ncells, 3 ND, 3 ND))."""
    i0, i1 = _cells(map0, off0, map1, off1, nlay)
    return dofs(i0), cell_matrices(el, coords.reshape(-1, 3)[i1], mu, lmbda, beta)


def diagonal(el, coords, map0, off0, map1, off1, nlay, mu, lmbda, beta=0.0, nnodes=None, out=None):
    di, A = element_matrices(el, coords, map0, off0, map1, off1, nlay, mu, lmbda, beta)
    d = np.zeros(3 * (nnodes if nnodes is not None else int(di.max()) // 3 + 1)) if out is None else out
    np.add.at(d, di, np.diagonal(A, axis1=1, axis2=2))
    return d


def add_to_bcsr(rowptr, colidx, vals, di, A, row_lg=None, col_lg=None, bs=3):
    """MatSetValuesLocal(ADD_VALUES) into a blocked CSR (node pattern, bs x bs row-major blocks) with
    dof-level lgmaps: the node pattern is expanded to the equivalent dof-level CSR, the entries are added
    there by ``add_to_csr`` and moved back into the block layout."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    colidx = np.asarray(colidx, dtype=np.int64)
    n = len(rowptr) - 1
    cnt = np.diff(rowptr)
    # dof row r*bs + a holds, for every stored block k of node row r, the columns colidx[k]*bs + b
    drow = np.repeat(np.arange(n * bs), np.repeat(cnt, bs) * bs)
    blk = np.concatenate([np.tile(np.arange(rowptr[r], rowptr[r + 1]), bs) for r in range(n)]) if n else \
        np.zeros(0, dtype=np.int64)
    k = np.repeat(blk, bs)
    b = np.tile(np.arange(bs), len(blk))
    a = (drow % bs)
    perm = (k * bs + a) * bs + b                            # block-layout position of each dof-CSR entry
    dcol = colidx[k] * bs + b
    drowptr = np.concatenate([[0], np.cumsum(np.repeat(cnt, bs) * bs)])
    tmp = np.zeros(len(dcol))
    add_to_csr(drowptr, dcol, tmp, di, A, row_lg, col_lg)
    vals[perm] += tmp
    return vals


def to_dense(rowptr, colidx, vals, bs=3):
    n = len(rowptr) - 1
    A = np.zeros((n * bs, n * bs))
    blocks = np.asarray(vals).reshape(-1, bs, bs)
    for r in range(n):
        for k in range(rowptr[r], rowptr[r + 1]):
            c = colidx[k]
            A[r * bs:(r + 1) * bs, c * bs:(c + 1) * bs] = blocks[k]
    return A


def global_matrix(el, coords, geo, nnodes, mu, lmbda, beta=0.0):
    """The assembled operator as a scipy CSR matrix (3 nnodes square)."""
    import scipy.sparse as sps
    di, A = element_matrices(el, coords, *geo, mu, lmbda, beta)
    nd = di.shape[1]
    r = np.repeat(di, nd, axis=1).ravel()
    c = np.tile(di, (1, nd)).ravel()
    return sps.csr_matrix((A.ravel(), (r, c)), shape=(3 * nnodes, 3 * nnodes))


def rigid_body_modes(Xn):
    """The 6 rigid-body modes at node positions Xn (nnodes, 3): 3 translations and 3 infinitesimal
    rotations omega x x, flat AoS (6, 3 nnodes)."""
    out = []
    for a in range(3):
        t = np.zeros_like(Xn)
        t[:, a] = 1.0
        out.append(t.ravel())
    for a in range(3):
        w = np.zeros(3)
        w[a] = 1.0
        out.append(np.cross(w, Xn).ravel())
    return np.array(out)
