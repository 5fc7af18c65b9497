"""TEST INFRASTRUCTURE: NumPy oracle of the Boussinesq (Rayleigh-Benard) system on Taylor-Hood hexahedra with the
temperature in CG_(p-1) on the pressure numbering (FDB_FORM_BOUSSINESQ[_JACOBIAN])

    R((u, p, T); (v, q, S)) = NavierStokes(nu = 1)((u, p); (v, q)) - T inner(bg, v)*dx
                              + dot(grad T, u) S*dx + kt inner(grad T, grad S)*dx
    J(u0, T0)[(w, r, s)]    = NavierStokesJacobian(u0)[(w, r)] - s inner(bg, v)*dx
                              + (dot(grad s, u0) + dot(grad T0, w)) S*dx + kt inner(grad s, grad S)*dx

bg = (Ra/Pr) g, kt = 1/Pr.  The (u, p) part is the Navier-Stokes oracle (tests/_navier_stokes_oracle.py); the
buoyancy and temperature terms are added here with the full 3-D bases (Kronecker products of the 1-D tables,
not sum-factorised) on the same (p+1)-point Gauss rule and geometry.  Global numbering: velocity dof 3*node +
component, then the pressures, then the temperatures.  ``newton`` is scipy's Newton on the oracle system."""
import numpy as np

import _navier_stokes_oracle as nso
import _stokes_oracle as so
from _coef_oracle import _cells, geometry


def _bases(el):
    """Velocity basis PV (Q, ND), scalar CG_(p-1) basis PT (Q, NP) and its reference gradients DT (Q, NP, 3) at the
    Q = nq^3 points, in the local dof orders of the kernels."""
    B, D = np.asarray(el.B), np.asarray(el.D)
    elq = so.pressure_element(el)
    Bq, Dq = np.asarray(elq.B), np.asarray(elq.D)
    k3 = lambda a, b, c: np.kron(np.kron(a, b), c)
    PV = k3(B, B, B)
    PT = k3(Bq, Bq, Bq)
    DT = np.stack([k3(Dq, Bq, Bq), k3(Bq, Dq, Bq), k3(Bq, Bq, Dq)], axis=-1)
    return PV, PT, DT


def _metric(el, X):
    Kinv, detw = geometry(el, X)
    nc = X.shape[0]
    return Kinv.reshape(nc, -1, 3, 3), detw.reshape(nc, -1)


def _temperature_terms(el, X, a, b, c, gc, bg, kt):
    """Velocity rows -c inner(bg, v) and temperature rows (dot(grad c, a) + dot(grad gc, b)) S + kt inner(grad c,
    grad S): a, b (nc, ND, 3) velocities, c, gc (nc, NP) temperatures (b or gc None: that term is absent)."""
    PV, PT, DT = _bases(el)
    Kinv, detw = _metric(el, X)
    grad = lambda f: np.einsum("qir,ci,cqre->cqe", DT, f, Kinv)          # physical gradient at the points
    gS = np.einsum("qir,cqre->cqie", DT, Kinv)                           # test-function gradients
    cq = c @ PT.T
    gcq = grad(c)
    aq = np.einsum("qa,cad->cqd", PV, a)
    val = np.einsum("cqe,cqe->cq", gcq, aq)
    if b is not None:
        val = val + np.einsum("cqe,cqe->cq", grad(gc), np.einsum("qa,cad->cqd", PV, b))
    yT = np.einsum("cq,qi->ci", detw * val, PT) + kt * np.einsum("cq,cqe,cqie->ci", detw, gcq, gS)
    yu = -np.einsum("cq,qa,d->cad", detw * cq, PV, np.asarray(bg, dtype=float))
    return yu, yT


def cell_residual(el, X, u, p, T, bg, kt):
    yu, yp = nso.cell_residual(el, X, u, p, 1.0)
    bu, yT = _temperature_terms(el, X, u, None, T, None, bg, kt)
    return yu + bu, yp, yT


def cell_jacobian(el, X, u0, T0, w, r, s, bg, kt):
    yu, yp = nso.cell_jacobian(el, X, u0, w, r, 1.0)
    bu, yT = _temperature_terms(el, X, u0, w, s, T0, bg, kt)
    return yu + bu, yp, yT


def _gather(el, coords, geo, geo2):
    i0, i1 = _cells(*geo)
    i2 = so._pressure_cells(*geo2, geo[4])
    return i0, i2, coords.reshape(-1, 3)[i1]


def residual(el, coords, u, p, T, geo, geo2, bg, kt):
    """R(u, p, T): u flat AoS (3 per node), p and T one per pressure node -> (y_u, y_p, y_T).  geo = (map0, off0,
    map1, off1, nlay), geo2 = (map2, off2)."""
    i0, i2, Xc = _gather(el, coords, geo, geo2)
    u, p, T = np.asarray(u, dtype=float), np.asarray(p, dtype=float), np.asarray(T, dtype=float)
    au, ap, aT = cell_residual(el, Xc, u.reshape(-1, 3)[i0], p[i2], T[i2], bg, kt)
    yu, yp, yT = np.zeros(len(u)), np.zeros(len(p)), np.zeros(len(T))
    np.add.at(yu.reshape(-1, 3), i0, au)
    np.add.at(yp, i2, ap)
    np.add.at(yT, i2, aT)
    return yu, yp, yT


def jacobian_action(el, coords, u0, T0, w, r, s, geo, geo2, bg, kt):
    """J(u0, T0) (w, r, s) -> (y_u, y_p, y_T), all flat as in :func:`residual`."""
    i0, i2, Xc = _gather(el, coords, geo, geo2)
    u0, T0 = np.asarray(u0, dtype=float), np.asarray(T0, dtype=float)
    w, r, s = np.asarray(w, dtype=float), np.asarray(r, dtype=float), np.asarray(s, dtype=float)
    au, ap, aT = cell_jacobian(el, Xc, u0.reshape(-1, 3)[i0], T0[i2], w.reshape(-1, 3)[i0], r[i2], s[i2], bg, kt)
    yu, yp, yT = np.zeros(len(w)), np.zeros(len(r)), np.zeros(len(s))
    np.add.at(yu.reshape(-1, 3), i0, au)
    np.add.at(yp, i2, ap)
    np.add.at(yT, i2, aT)
    return yu, yp, yT


def jacobian_matrix(el, coords, u0, T0, geo, geo2, nv, nq, bg, kt):
    """J(u0, T0) as scipy CSR over (3 nv velocity dofs, nq pressures, nq temperatures), row = test, column = trial:
    the element matrices column by column from unit directions."""
    import scipy.sparse as sps
    i0, i2, Xc = _gather(el, coords, geo, geo2)
    nc = len(Xc)
    nd, npd = el.ndof ** 3, (el.ndof - 1) ** 3
    nt = 3 * nd + 2 * npd
    uc, Tc = np.asarray(u0, dtype=float).reshape(-1, 3)[i0], np.asarray(T0, dtype=float)[i2]
    K = np.empty((nc, nt, nt))
    for j in range(nt):
        e = np.zeros(nt)
        e[j] = 1.0
        w = np.broadcast_to(e[:3 * nd].reshape(nd, 3), (nc, nd, 3))
        r = np.broadcast_to(e[3 * nd:3 * nd + npd], (nc, npd))
        s = np.broadcast_to(e[3 * nd + npd:], (nc, npd))
        yu, yp, yT = cell_jacobian(el, Xc, uc, Tc, w, r, s, bg, kt)
        K[:, :, j] = np.concatenate([yu.reshape(nc, -1), yp, yT], axis=1)
    di = np.concatenate([(3 * i0[:, :, None] + np.arange(3)).reshape(nc, -1), 3 * nv + i2, 3 * nv + nq + i2], axis=1)
    rr = np.repeat(di, nt, axis=1).ravel()
    cc = np.tile(di, (1, nt)).ravel()
    n = 3 * nv + 2 * nq
    return sps.csr_matrix((K.ravel(), (rr, cc)), shape=(n, n))


def newton(el, coords, geo, geo2, nv, nq, bg, kt, fixed, values, rtol=1e-12, maxit=30, L=None):
    """scipy's Newton for R(u, p, T) = L (L None: 0; flat over the three blocks) with the global dofs ``fixed`` set to
    ``values`` (velocity and temperature conditions; pin one pressure dof here to fix the constant).  Returns (u, p
    with its mean removed, T, residual norms)."""
    import scipy.sparse.linalg as spla
    n = 3 * nv + 2 * nq
    x = np.zeros(n)
    x[fixed] = values

    def res(x):
        R = np.concatenate(residual(el, coords, x[:3 * nv], x[3 * nv:3 * nv + nq], x[3 * nv + nq:], geo, geo2, bg,
                                    kt))
        if L is not None:
            R -= L
        R[fixed] = 0.0
        return R

    R = res(x)
    hist = [np.linalg.norm(R)]
    while hist[-1] > rtol * max(hist[0], 1e-300) and len(hist) <= maxit:
        K = jacobian_matrix(el, coords, x[:3 * nv], x[3 * nv + nq:], geo, geo2, nv, nq, bg, kt)
        x -= spla.spsolve(so.constrained(K, fixed).tocsc(), R)
        R = res(x)
        hist.append(np.linalg.norm(R))
    p = x[3 * nv:3 * nv + nq]
    return x[:3 * nv], p - p.mean(), x[3 * nv + nq:], hist
