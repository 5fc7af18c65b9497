"""TEST INFRASTRUCTURE: NumPy oracle of steady incompressible Navier-Stokes on Taylor-Hood hexahedra
(FDB_FORM_NAVIER_STOKES[_JACOBIAN])

    R((u, p); (v, q))    = nu*inner(grad u, grad v)*dx + beta*inner(u, v)*dx + inner(dot(grad u, u), v)*dx
                           - p*div(v)*dx - q*div(u)*dx
    J(u)[(w, r); (v, q)] = Stokes((w, r); (v, q)) + inner(dot(grad w, u), v)*dx + inner(dot(grad u, w), v)*dx

with dot(grad a, b)_d = sum_k da_d/dx_k b_k.  The Stokes part is the Stokes oracle (tests/_stokes_oracle.py)
with mu = nu; the convective term is added here on the same (p+1)-point Gauss rule, geometry and tensor
contractions (tests/_coef_oracle.py).  Global numbering as in the Stokes oracle: velocity dof 3*node +
component, then the pressures.  ``newton`` is scipy's Newton on the oracle system, the reference of the
lid-driven cavity."""
import numpy as np

import _stokes_oracle as so
from _coef_oracle import _cells, _t3, geometry


def _grad(el, X, a):
    """Physical gradient G[..., i, j, k, d, e] = d a_d / d x_e at the points: a (nc, [m,] ND, 3)."""
    B, D = np.asarray(el.B), np.asarray(el.D)
    n = B.shape[1]
    Kinv, _ = geometry(el, X)
    aa = np.moveaxis(a, -1, -2).reshape(a.shape[:-2] + (3, n, n, n))
    extra = aa.ndim - 5
    ex = lambda t: t.reshape(t.shape[:1] + (1,) * extra + t.shape[1:])
    gh = np.stack([_t3(D, B, B, aa), _t3(B, D, B, aa), _t3(B, B, D, aa)], axis=-1)
    return np.einsum("...dijkm,...ijkme->...ijkde", gh, ex(Kinv))


def _values(el, a):
    B = np.asarray(el.B)
    n = B.shape[1]
    aa = np.moveaxis(a, -1, -2).reshape(a.shape[:-2] + (3, n, n, n))
    return np.moveaxis(_t3(B, B, B, aa), -4, -1)                  # (..., i, j, k, 3)


def convective(el, X, a, b):
    """Element vectors of inner(dot(grad a, b), v)*dx: a, b (nc, [m,] ND, 3) -> (nc, [m,] ND, 3)."""
    B = np.asarray(el.B)
    n = B.shape[1]
    _, detw = geometry(el, X)
    extra = a.ndim - 3
    ex = lambda t: t.reshape(t.shape[:1] + (1,) * extra + t.shape[1:])
    c = np.einsum("...ijkde,...ijke->...dijk", _grad(el, X, a), _values(el, b)) * ex(detw)[..., None, :, :, :]
    y = _t3(B.T, B.T, B.T, c)
    return np.moveaxis(y.reshape(a.shape[:-2] + (3, n ** 3)), -2, -1)


def cell_residual(el, X, u, p, nu, beta=0.0):
    yu, yp = so.cell_actions(el, X, u, p, nu, beta)
    return yu + convective(el, X, u, u), yp


def cell_jacobian(el, X, u, w, r, nu, beta=0.0):
    """J(u) applied to (w, r); w and r may carry a batch axis after the cell axis, u does not."""
    yu, yp = so.cell_actions(el, X, w, r, nu, beta)
    ub = np.broadcast_to(u.reshape(u.shape[:1] + (1,) * (w.ndim - 3) + u.shape[1:]), w.shape)
    return yu + convective(el, X, w, ub) + convective(el, X, ub, w), yp


def _gather(el, coords, u, geo, geo2):
    i0, i1 = _cells(*geo)
    i2 = so._pressure_cells(*geo2, geo[4])
    return i0, i1, i2, coords.reshape(-1, 3)[i1], np.asarray(u).reshape(-1, 3)[i0]


def residual(el, coords, u, p, geo, geo2, nu, beta=0.0):
    """R(u, p): u flat AoS (3 per node), p one per pressure node -> (y_u, y_p).  geo = (map0, off0, map1, off1,
    nlay), geo2 = (map2, off2)."""
    i0, _, i2, Xc, uc = _gather(el, coords, u, geo, geo2)
    yu, yp = np.zeros(len(u)), np.zeros(len(p))
    au, ap = cell_residual(el, Xc, uc, np.asarray(p)[i2], nu, beta)
    np.add.at(yu.reshape(-1, 3), i0, au)
    np.add.at(yp, i2, ap)
    return yu, yp


def jacobian_action(el, coords, u, w, r, geo, geo2, nu, beta=0.0):
    """J(u) (w, r) -> (y_u, y_p), all flat as in :func:`residual`."""
    i0, _, i2, Xc, uc = _gather(el, coords, u, geo, geo2)
    yu, yp = np.zeros(len(w)), np.zeros(len(r))
    au, ap = cell_jacobian(el, Xc, uc, np.asarray(w).reshape(-1, 3)[i0], np.asarray(r)[i2], nu, beta)
    np.add.at(yu.reshape(-1, 3), i0, au)
    np.add.at(yp, i2, ap)
    return yu, yp


def jacobian_matrix(el, coords, u, geo, geo2, nv, nq, nu, beta=0.0):
    """J(u) as scipy CSR over (3 nv velocity dofs, nq pressures), row = test, column = trial."""
    import scipy.sparse as sps
    i0, _, i2, Xc, uc = _gather(el, coords, u, geo, geo2)
    nd, npd = el.ndof ** 3, (el.ndof - 1) ** 3
    nt = 3 * nd + npd
    E = np.eye(nt)
    Eu, Ep = E[:, :3 * nd].reshape(nt, nd, 3), E[:, 3 * nd:]
    K = np.empty((len(Xc), nt, nt))
    step = max(1, 512 // nd)
    for c in range(0, len(Xc), step):
        e = min(c + step, len(Xc))
        bu = np.broadcast_to(Eu, (e - c,) + Eu.shape)
        bp = np.broadcast_to(Ep, (e - c,) + Ep.shape)
        yu, yp = cell_jacobian(el, Xc[c:e], uc[c:e], bu, bp, nu, beta)
        K[c:e] = np.swapaxes(np.concatenate([yu.reshape(e - c, nt, 3 * nd), yp], axis=2), 1, 2)
    di = np.concatenate([(3 * i0[:, :, None] + np.arange(3)).reshape(i0.shape[0], -1), 3 * nv + i2], axis=1)
    rr = np.repeat(di, nt, axis=1).ravel()
    cc = np.tile(di, (1, nt)).ravel()
    return sps.csr_matrix((K.ravel(), (rr, cc)), shape=(3 * nv + nq, 3 * nv + nq))


def newton(el, coords, geo, geo2, nv, nq, nu, bdofs, g, beta=0.0, rtol=1e-12, maxit=30):
    """scipy's Newton for R(u, p) = 0 with the velocity dofs ``bdofs`` fixed to ``g`` (flat, 3 nv) and the
    pressure fixed by pinning its first dof, then its mean removed.  Returns (u, p, residual norms)."""
    import scipy.sparse as sps
    import scipy.sparse.linalg as spla
    x = np.zeros(3 * nv + nq)
    x[bdofs] = g[bdofs]
    fixed = np.concatenate([bdofs, [3 * nv]])

    def res(x):
        yu, yp = residual(el, coords, x[:3 * nv], x[3 * nv:], geo, geo2, nu, beta)
        R = np.concatenate([yu, yp])
        R[fixed] = 0.0
        return R

    R = res(x)
    hist = [np.linalg.norm(R)]
    while hist[-1] > rtol * hist[0] and len(hist) <= maxit:
        K = jacobian_matrix(el, coords, x[:3 * nv], geo, geo2, nv, nq, nu, beta)
        x -= spla.spsolve(sps.csc_matrix(so.constrained(K, fixed)), R)
        R = res(x)
        hist.append(np.linalg.norm(R))
    return x[:3 * nv], x[3 * nv:] - x[3 * nv:].mean(), hist
