"""TEST INFRASTRUCTURE: NumPy oracle of compressible Neo-Hookean hyperelasticity
(FDB_FORM_HYPERELASTICITY[_JACOBIAN])

    F = I + grad u,  J = det F,  psi = mu/2 (tr(F^T F) - 3) - mu ln J + lmbda/2 (ln J)^2
    P(F) = mu (F - F^{-T}) + lmbda ln(J) F^{-T}
    R(u; v)    = inner(P(F(u)), grad v)*dx + beta*inner(u, v)*dx
    J(u)[w; v] = inner(dP[grad w], grad v)*dx + beta*inner(w, v)*dx
    dP[H] = mu H + (mu - lmbda ln J) F^{-T} H^T F^{-T} + lmbda tr(F^{-1} H) F^{-T}

on vector (3 components, AoS) Q_p (x) P_p hexahedra, with the layout, geometry and CSR helpers of the
linear elasticity oracle (tests/_elasticity_oracle.py).  Also the discrete energy
E(u) = int psi(F(u)) + beta/2 |u|^2 dx, whose gradient is R, and a scipy Newton solve."""
import numpy as np

from _coef_oracle import _cells, _t3, geometry
from _elasticity_oracle import dofs


def _extra(u):
    """Broadcasts cell arrays over the optional extra axis of u (nc, [m,] ND, 3)."""
    extra = u.ndim - 3
    return lambda a: a.reshape(a.shape[:1] + (1,) * extra + a.shape[1:])


def _at_points(el, X, u):
    """Values (..., d, Q, Q, Q), physical gradients (..., Q, Q, Q, d, e) of u (nc, [m,] ND, 3), and the
    geometry (Kinv, w |det|)."""
    B, D = np.asarray(el.B), np.asarray(el.D)
    n = B.shape[1]
    Kinv, detw = geometry(el, X)
    ex = _extra(u)
    uu = np.moveaxis(u, -1, -2).reshape(u.shape[:-2] + (3, n, n, n))
    gh = np.stack([_t3(D, B, B, uu), _t3(B, D, B, uu), _t3(B, B, D, uu)], axis=-1)
    G = np.einsum("...dijkm,...ijkme->...ijkde", gh, ex(Kinv))
    return _t3(B, B, B, uu), G, Kinv, detw


def _integrate(el, Kinv, detw, S, vals, beta, ex, shape):
    """sum_q w |det J| (S : grad v + beta vals . v) for every basis function v: the shape of u."""
    B, D = np.asarray(el.B), np.asarray(el.D)
    n = B.shape[1]
    f = np.einsum("...ijkme,...ijkde->...dijkm", ex(Kinv), S) * ex(detw)[..., None, :, :, :, None]
    m = beta * ex(detw)[..., None, :, :, :] * vals
    out = (_t3(D.T, B.T, B.T, f[..., 0]) + _t3(B.T, D.T, B.T, f[..., 1]) + _t3(B.T, B.T, D.T, f[..., 2])
           + _t3(B.T, B.T, B.T, m))
    return np.moveaxis(out.reshape(shape[:-2] + (3, n ** 3)), -2, -1)


def piola(F, mu, lmbda):
    Fit = np.swapaxes(np.linalg.inv(F), -1, -2)
    return mu * (F - Fit) + lmbda * np.log(np.linalg.det(F))[..., None, None] * Fit


def dpiola(F, H, mu, lmbda):
    Fi = np.linalg.inv(F)
    Fit = np.swapaxes(Fi, -1, -2)
    lnJ = np.log(np.linalg.det(F))[..., None, None]
    trA = np.trace(Fi @ H, axis1=-2, axis2=-1)[..., None, None]
    return mu * H + (mu - lmbda * lnJ) * (Fit @ np.swapaxes(H, -1, -2) @ Fit) + lmbda * trA * Fit


def energy_density(F, mu, lmbda):
    lnJ = np.log(np.linalg.det(F))
    return mu / 2 * ((F * F).sum(axis=(-2, -1)) - 3) - mu * lnJ + lmbda / 2 * lnJ ** 2


def cell_residuals(el, X, u, mu, lmbda, beta=0.0):
    """X (nc, 8, 3), u (nc, ND, 3) -> (nc, ND, 3)."""
    vals, G, Kinv, detw = _at_points(el, X, u)
    return _integrate(el, Kinv, detw, piola(np.eye(3) + G, mu, lmbda), vals, beta, _extra(u), u.shape)


def cell_jacobian_actions(el, X, u, w, mu, lmbda, beta=0.0):
    """J(u) w per cell: u (nc, ND, 3), w (nc, [m,] ND, 3) -> the shape of w."""
    _, Gu, _, _ = _at_points(el, X, u)
    vals, H, Kinv, detw = _at_points(el, X, w)
    ex = _extra(w)
    return _integrate(el, Kinv, detw, dpiola(ex(np.eye(3) + Gu), H, mu, lmbda), vals, beta, ex, w.shape)


def cell_jacobians(el, X, u, mu, lmbda, beta=0.0):
    """Element Jacobians A[3i + a, 3j + b] = J(u)[phi_j e_b; phi_i e_a]: (nc, 3 ND, 3 ND)."""
    nd = el.ndof ** 3
    step = max(1, 1024 // nd)
    out = np.empty((X.shape[0], 3 * nd, 3 * nd))
    E = np.eye(3 * nd).reshape(3 * nd, nd, 3)
    for c in range(0, X.shape[0], step):
        e = min(c + step, X.shape[0])
        Y = cell_jacobian_actions(el, X[c:e], u[c:e], np.broadcast_to(E, (e - c,) + E.shape), mu, lmbda, beta)
        out[c:e] = np.swapaxes(Y.reshape(e - c, 3 * nd, 3 * nd), 1, 2)
    return out


def cell_energies(el, X, u, mu, lmbda, beta=0.0):
    vals, G, _, detw = _at_points(el, X, u)
    psi = energy_density(np.eye(3) + G, mu, lmbda) + beta / 2 * (vals ** 2).sum(axis=-4)
    return (psi * detw).sum(axis=(-3, -2, -1))


def _gather(coords, u, geo):
    i0, i1 = _cells(*geo)
    return i0, coords.reshape(-1, 3)[i1], np.asarray(u).reshape(-1, 3)[i0]


def residual(el, coords, u, map0, off0, map1, off1, nlay, mu, lmbda, beta=0.0, out=None):
    """assemble(R(u)) over every column and layer; u and the result are flat AoS (3 per node)."""
    i0, X, uc = _gather(coords, u, (map0, off0, map1, off1, nlay))
    y = np.zeros(len(u)) if out is None else out
    np.add.at(y.reshape(-1, 3), i0, cell_residuals(el, X, uc, mu, lmbda, beta))
    return y


def jacobian_action(el, coords, u, w, map0, off0, map1, off1, nlay, mu, lmbda, beta=0.0, out=None):
    i0, X, uc = _gather(coords, u, (map0, off0, map1, off1, nlay))
    y = np.zeros(len(w)) if out is None else out
    wc = np.asarray(w).reshape(-1, 3)[i0]
    np.add.at(y.reshape(-1, 3), i0, cell_jacobian_actions(el, X, uc, wc, mu, lmbda, beta))
    return y


def element_matrices(el, coords, u, map0, off0, map1, off1, nlay, mu, lmbda, beta=0.0):
    """(dof indices (ncells, 3 ND), element Jacobians (ncells, 3 ND, 3 ND))."""
    i0, X, uc = _gather(coords, u, (map0, off0, map1, off1, nlay))
    return dofs(i0), cell_jacobians(el, X, uc, mu, lmbda, beta)


def diagonal(el, coords, u, map0, off0, map1, off1, nlay, mu, lmbda, beta=0.0, out=None):
    di, A = element_matrices(el, coords, u, map0, off0, map1, off1, nlay, mu, lmbda, beta)
    d = np.zeros(len(u)) if out is None else out
    np.add.at(d, di, np.diagonal(A, axis1=1, axis2=2))
    return d


def energy(el, coords, u, geo, mu, lmbda, beta=0.0):
    _, X, uc = _gather(coords, u, geo)
    return float(cell_energies(el, X, uc, mu, lmbda, beta).sum())


def global_jacobian(el, coords, u, geo, mu, lmbda, beta=0.0):
    import scipy.sparse as sps
    di, A = element_matrices(el, coords, u, *geo, mu, lmbda, beta)
    nd = di.shape[1]
    n = len(u)
    return sps.csr_matrix((A.ravel(), (np.repeat(di, nd, axis=1).ravel(), np.tile(di, (1, nd)).ravel())),
                          shape=(n, n))


def newton(el, coords, geo, mu, lmbda, beta, L, u, bc_dofs, rtol=1e-12, maxit=30):
    """Newton with the full step on R(u) - L with u fixed on ``bc_dofs`` (u carries their values);
    scipy's sparse direct solve for every step.  Returns (u, residual norms)."""
    import scipy.sparse.linalg as spla
    u = np.array(u, dtype=float)
    free = np.setdiff1d(np.arange(len(u)), bc_dofs)
    hist = []
    for _ in range(maxit):
        r = residual(el, coords, u, *geo, mu, lmbda, beta) - L
        hist.append(float(np.linalg.norm(r[free])))
        if hist[-1] <= rtol * hist[0] or hist[-1] == 0.0:
            break
        K = global_jacobian(el, coords, u, geo, mu, lmbda, beta).tocsr()
        u[free] -= spla.spsolve(K[free][:, free].tocsc(), r[free])
    return u, hist


# a homogeneous deformation u* = (A - I) X with det A > 0, small enough that Newton from zero interior
# values does not invert the elements next to the boundary on a 3^3 CG2 mesh
HOMOGENEOUS_A = np.array([[1.08, 0.04, -0.02], [0.02, 0.96, 0.04], [0.0, -0.04, 1.04]])


def converges_quadratically(hist):
    """Some Newton step from a relative residual r in (1e-11, 1e-2) reaches r**1.8 or less (rounding
    ends the sequence before the rate can show on the last steps)."""
    r = np.asarray(hist) / hist[0]
    return any(1e-11 < r[k] < 1e-2 and r[k + 1] <= r[k] ** 1.8 for k in range(len(r) - 1))


def rotation(axis, angle):
    """The rotation matrix about ``axis`` by ``angle`` (Rodrigues)."""
    k = np.asarray(axis, dtype=float) / np.linalg.norm(axis)
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(angle) * Kx + (1 - np.cos(angle)) * Kx @ Kx


def rotated_rigid_modes(Xn, Q):
    """The 6 null vectors of J at u = (Q - I) X (beta = 0): the translations and S Q X for skew S,
    flat AoS (6, 3 nnodes)."""
    out = []
    for a in range(3):
        t = np.zeros_like(Xn)
        t[:, a] = 1.0
        out.append(t.ravel())
    QX = Xn @ Q.T
    for a in range(3):
        w = np.zeros(3)
        w[a] = 1.0
        out.append(np.cross(w, QX).ravel())
    return np.array(out)
