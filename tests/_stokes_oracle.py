"""TEST INFRASTRUCTURE: NumPy oracle of Stokes flow on Taylor-Hood hexahedra (FDB_FORM_STOKES)

    a((u, p), (v, q)) = mu*inner(grad u, grad v)*dx + beta*inner(u, v)*dx - p*div(v)*dx - q*div(u)*dx

with u in vector (3 components, AoS) Q_p and p in scalar Q_(p-1) on the same hexahedra, a trilinear
coordinate field and the (p+1)-point Gauss rule per axis.  Built on the coefficient oracle's geometry,
tensor contraction and cell gather (tests/_coef_oracle.py): velocity dof 3*node + component, pressure dofs
after the velocity's in the global saddle-point numbering."""
import numpy as np

from _coef_oracle import _cells, _t3, geometry
from firedrake_b200.fiat_lite import interval_element


def pressure_element(el):
    """The CG_(p-1) element tabulated at the velocity element's Gauss points."""
    return interval_element(el.ndof - 2, el.nq)


def cell_actions(el, X, u, p, mu, beta=0.0):
    """Element actions for a batch of cells: X (nc, 8, 3), u (nc, [m,] ND, 3), p (nc, [m,] NP) ->
    (y_u like u, y_p like p)."""
    B, D = np.asarray(el.B), np.asarray(el.D)
    Bq = np.asarray(pressure_element(el).B)
    n, nqp = B.shape[1], Bq.shape[1]
    Kinv, detw = geometry(el, X)
    uu = np.moveaxis(u, -1, -2).reshape(u.shape[:-2] + (3, n, n, n))
    pp = p.reshape(p.shape[:-1] + (nqp, nqp, nqp))
    extra = uu.ndim - 5
    ex = lambda a: a.reshape(a.shape[:1] + (1,) * extra + a.shape[1:])
    gh = np.stack([_t3(D, B, B, uu), _t3(B, D, B, uu), _t3(B, B, D, uu)], axis=-1)
    G = np.einsum("...dijkm,...ijkme->...ijkde", gh, ex(Kinv))
    pq = _t3(Bq, Bq, Bq, pp)
    S = mu * G - pq[..., None, None] * np.eye(3)
    f = np.einsum("...ijkme,...ijkde->...dijkm", ex(Kinv), S) * ex(detw)[..., None, :, :, :, None]
    m = beta * ex(detw)[..., None, :, :, :] * _t3(B, B, B, uu)
    yu = (_t3(D.T, B.T, B.T, f[..., 0]) + _t3(B.T, D.T, B.T, f[..., 1]) + _t3(B.T, B.T, D.T, f[..., 2])
          + _t3(B.T, B.T, B.T, m))
    t = -ex(detw) * np.trace(G, axis1=-2, axis2=-1)
    yp = _t3(Bq.T, Bq.T, Bq.T, t)
    return np.moveaxis(yu.reshape(u.shape[:-2] + (3, n ** 3)), -2, -1), yp.reshape(p.shape)


def cell_matrices(el, X, mu, beta=0.0):
    """Element saddle-point matrices over (3 ND velocity dofs, NP pressure dofs), row = test, column = trial."""
    nd, npd = el.ndof ** 3, (el.ndof - 1) ** 3
    nt = 3 * nd + npd
    out = np.empty((X.shape[0], nt, nt))
    E = np.eye(nt)
    Eu, Ep = E[:, :3 * nd].reshape(nt, nd, 3), E[:, 3 * nd:]
    step = max(1, 512 // nd)
    for c in range(0, X.shape[0], step):
        e = min(c + step, X.shape[0])
        bu = np.broadcast_to(Eu, (e - c,) + Eu.shape)
        bp = np.broadcast_to(Ep, (e - c,) + Ep.shape)
        yu, yp = cell_actions(el, X[c:e], bu, bp, mu, beta)        # (nc, col, ND, 3), (nc, col, NP)
        Y = np.concatenate([yu.reshape(e - c, nt, 3 * nd), yp], axis=2)
        out[c:e] = np.swapaxes(Y, 1, 2)
    return out


def _pressure_cells(map2, off2, nlay):
    lay = np.arange(nlay)
    return (map2[:, None, :] + np.asarray(off2)[None, None, :] * lay[None, :, None]).reshape(-1, map2.shape[1])


def action(el, coords, u, p, geo, geo2, mu, beta=0.0):
    """assemble(action(a, (u, p))): u flat AoS (3 per node), p one per pressure node -> (y_u, y_p).
    geo = (map0, off0, map1, off1, nlay), geo2 = (map2, off2)."""
    i0, i1 = _cells(*geo)
    i2 = _pressure_cells(*geo2, geo[4])
    yu, yp = np.zeros(len(u)), np.zeros(len(p))
    au, ap = cell_actions(el, coords.reshape(-1, 3)[i1], np.asarray(u).reshape(-1, 3)[i0], np.asarray(p)[i2],
                          mu, beta)
    np.add.at(yu.reshape(-1, 3), i0, au)
    np.add.at(yp, i2, ap)
    return yu, yp


def global_matrix(el, coords, geo, geo2, nv, nq, mu, beta=0.0):
    """The saddle-point matrix [[A, B^T], [B, 0]] as scipy CSR over (3 nv velocity dofs, nq pressures)."""
    import scipy.sparse as sps
    i0, i1 = _cells(*geo)
    i2 = _pressure_cells(*geo2, geo[4])
    di = np.concatenate([(3 * i0[:, :, None] + np.arange(3)).reshape(i0.shape[0], -1), 3 * nv + i2], axis=1)
    K = cell_matrices(el, coords.reshape(-1, 3)[i1], mu, beta)
    nt = di.shape[1]
    r = np.repeat(di, nt, axis=1).ravel()
    c = np.tile(di, (1, nt)).ravel()
    return sps.csr_matrix((K.ravel(), (r, c)), shape=(3 * nv + nq, 3 * nv + nq))


def blocks(K, nv):
    """(A, B^T, B, C) of the saddle-point matrix."""
    K = K.tocsr()
    n = 3 * nv
    return K[:n, :n], K[:n, n:], K[n:, :n], K[n:, n:]


def constrained(K, bdofs):
    """The matrix-free operator's matrix: constrained velocity rows and columns replaced by the identity."""
    import scipy.sparse as sps
    n = K.shape[0]
    keep = np.ones(n)
    keep[bdofs] = 0.0
    Dk = sps.diags(keep)
    return (Dk @ K @ Dk + sps.diags(1.0 - keep)).tocsr()


def velocity_dofs(nodes):
    return (3 * np.asarray(nodes)[:, None] + np.arange(3)).ravel()
