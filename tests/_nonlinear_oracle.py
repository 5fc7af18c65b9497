"""TEST INFRASTRUCTURE: NumPy oracle of nonlinear diffusion (FDB_FORM_NONLINEAR_DIFFUSION[_JACOBIAN])

    F(u; v)    = alpha*inner(D(u) grad u, grad v)*dx + beta*inner(u, v)*dx,   D(s) = d0 + d1 s + d2 s^2
    J(u)[w; v] = alpha*inner(D(u) grad w + D'(u) w grad u, grad v)*dx + beta*inner(w, v)*dx

on Q_p (x) P_p hexahedra with a trilinear coordinate field, built on tests/_coef_oracle.py (same dof /
vertex conventions, same p+1 Gauss points per axis).  D(u) is evaluated at each quadrature point from
the interpolated u, so J is the exact derivative of the discrete F.  ``newton`` solves F(u) = L with
scipy's sparse direct solver at every step: the reference solution of the GPU solves."""
import numpy as np
import scipy.sparse as sps
import scipy.sparse.linalg as spla

import _coef_oracle as co


def _D(d, s):
    return d[0] + s * (d[1] + d[2] * s)


def _dD(d, s):
    return d[1] + 2.0 * d[2] * s


def _quad(el, X, u):
    """geometry, u at the points and u's reference gradient: (M = J^-1 J^-T, detw, uq, gu)."""
    B, D, _, _ = co._tables(el)
    n = B.shape[1]
    Kinv, detw = co.geometry(el, X)
    uu = u.reshape(-1, n, n, n)
    uq = co._t3(B, B, B, uu)
    gu = np.stack([co._t3(D, B, B, uu), co._t3(B, D, B, uu), co._t3(B, B, D, uu)], axis=-1)
    M = np.einsum("nijkrd,nijksd->nijkrs", Kinv, Kinv)
    return M, detw, uq, gu


def _test(el, f, m):
    """sum_q (grad phi_i . f + phi_i m): f (..., Q, Q, Q, 3) reference flux, m (..., Q, Q, Q)."""
    B, D, _, _ = co._tables(el)
    return (co._t3(D.T, B.T, B.T, f[..., 0]) + co._t3(B.T, D.T, B.T, f[..., 1]) + co._t3(B.T, B.T, D.T, f[..., 2])
            + co._t3(B.T, B.T, B.T, m))


def cell_residuals(el, X, u, d, alpha=1.0, beta=0.0):
    """Element residuals F(u; phi_i): X (nc, 8, 3), u (nc, ND) -> (nc, ND)."""
    M, detw, uq, gu = _quad(el, X, u)
    f = np.einsum("nijkrs,nijks->nijkr", M, gu) * (alpha * _D(d, uq) * detw)[..., None]
    return _test(el, f, beta * detw * uq).reshape(u.shape)


def cell_jacobian_actions(el, X, u, w, d, alpha=1.0, beta=0.0):
    """Element actions J(u)[w; phi_i]: u (nc, ND), w (nc, ND) or (nc, m, ND) -> w's shape."""
    B, D, _, _ = co._tables(el)
    n = B.shape[1]
    M, detw, uq, gu = _quad(el, X, u)
    ww = w.reshape(w.shape[:-1] + (n, n, n))
    extra = ww.ndim - 4
    ex = lambda a: a.reshape(a.shape[:1] + (1,) * extra + a.shape[1:])
    wq = co._t3(B, B, B, ww)
    gw = np.stack([co._t3(D, B, B, ww), co._t3(B, D, B, ww), co._t3(B, B, D, ww)], axis=-1)
    g = ex(_D(d, uq))[..., None] * gw + (ex(_dD(d, uq)) * wq)[..., None] * ex(gu)
    f = np.einsum("...ijkrs,...ijks->...ijkr", ex(M), g) * ex(alpha * detw)[..., None]
    return _test(el, f, beta * ex(detw) * wq).reshape(w.shape)


def cell_jacobian_matrices(el, X, u, d, alpha=1.0, beta=0.0):
    """A[i, j] = J(u)[phi_j; phi_i] (row = test, column = trial): (nc, ND, ND)."""
    nd = el.ndof ** 3
    step = max(1, 2048 // nd)
    out = np.empty((X.shape[0], nd, nd))
    for c in range(0, X.shape[0], step):
        e = min(c + step, X.shape[0])
        E = np.broadcast_to(np.eye(nd), (e - c, nd, nd))
        out[c:e] = np.swapaxes(cell_jacobian_actions(el, X[c:e], u[c:e], E, d, alpha, beta), 1, 2)
    return out


def residual(el, coords, u, map0, off0, map1, off1, nlay, d, alpha=1.0, beta=0.0):
    i0, i1 = co._cells(map0, off0, map1, off1, nlay)
    y = np.zeros(len(u))
    np.add.at(y, i0, cell_residuals(el, coords.reshape(-1, 3)[i1], u[i0], d, alpha, beta))
    return y


def jacobian_action(el, coords, u, w, map0, off0, map1, off1, nlay, d, alpha=1.0, beta=0.0):
    i0, i1 = co._cells(map0, off0, map1, off1, nlay)
    y = np.zeros(len(u))
    np.add.at(y, i0, cell_jacobian_actions(el, coords.reshape(-1, 3)[i1], u[i0], w[i0], d, alpha, beta))
    return y


def jacobian_matrices(el, coords, u, map0, off0, map1, off1, nlay, d, alpha=1.0, beta=0.0):
    """(dof indices (ncells, ND), element matrices (ncells, ND, ND))."""
    i0, i1 = co._cells(map0, off0, map1, off1, nlay)
    return i0, cell_jacobian_matrices(el, coords.reshape(-1, 3)[i1], u[i0], d, alpha, beta)


def jacobian_diagonal(el, coords, u, map0, off0, map1, off1, nlay, d, alpha=1.0, beta=0.0):
    i0, A = jacobian_matrices(el, coords, u, map0, off0, map1, off1, nlay, d, alpha, beta)
    out = np.zeros(len(u))
    np.add.at(out, i0, np.diagonal(A, axis1=1, axis2=2))
    return out


def jacobian_csr(el, coords, u, geo, d, alpha=1.0, beta=0.0, bc_nodes=()):
    """The global Jacobian as a scipy CSR matrix; rows and columns of ``bc_nodes`` replaced by the
    identity (what assemble(J, bcs) gives)."""
    i0, A = jacobian_matrices(el, coords, u, *geo, d, alpha, beta)
    nd = i0.shape[1]
    r = np.repeat(i0, nd, axis=1).ravel()
    c = np.tile(i0, (1, nd)).ravel()
    v = A.reshape(-1)
    bc = np.zeros(len(u), dtype=bool)
    bc[np.asarray(bc_nodes, dtype=np.int64)] = True
    keep = ~(bc[r] | bc[c])
    K = sps.coo_matrix((v[keep], (r[keep], c[keep])), shape=(len(u), len(u))).tocsr()
    bn = np.flatnonzero(bc)
    K = K + sps.coo_matrix((np.ones(len(bn)), (bn, bn)), shape=K.shape).tocsr()
    return K


def newton(el, coords, geo, L, d, alpha=1.0, beta=0.0, u0=None, bc_nodes=(), bc_values=None, rtol=1e-10,
           maxit=50):
    """Newton with the full step and exact linear solves: returns (u, residual norms).  ``bc_values``
    (full-length array) supplies the Dirichlet values on ``bc_nodes``."""
    u = np.zeros(len(L)) if u0 is None else np.array(u0, dtype=float)
    bn = np.asarray(bc_nodes, dtype=np.int64)
    if len(bn):
        u[bn] = np.asarray(bc_values)[bn]

    def R(u):
        r = residual(el, coords, u, *geo, d, alpha, beta) - L
        r[bn] = 0.0
        return r

    r = R(u)
    hist = [np.linalg.norm(r)]
    while hist[-1] > rtol * hist[0] and len(hist) <= maxit:
        du = spla.spsolve(jacobian_csr(el, coords, u, geo, d, alpha, beta, bn), r)
        du[bn] = 0.0
        u -= du
        r = R(u)
        hist.append(np.linalg.norm(r))
    return u, hist
