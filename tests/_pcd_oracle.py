"""TEST INFRASTRUCTURE: NumPy oracle of the pressure convection-diffusion operator of a PCD Schur approximation
(DESIGN.md section 4.13)

    F_p(u)[r; q] = nu*inner(grad r, grad q)*dx + beta*r*q*dx + inner(u, grad r)*q*dx

with r, q in scalar Q_(p-1) and u in vector (3 components, AoS) Q_p on the same hexahedra, the velocity's
(p+1)-point Gauss rule per axis and a trilinear coordinate field: the pressure space and rule of the
Taylor-Hood forms (tests/_stokes_oracle.py), the velocity values of the Navier-Stokes oracle
(tests/_navier_stokes_oracle.py).  Also the other two PCD operators as scipy CSR -- the pressure Laplacian
K_p (regularised with 1e-6 of the mass) and the pressure mass M_p, both from the scalar Helmholtz oracle
(tests/_coef_oracle.py) on Q with the same rule -- and a flexible GMRES for the preconditioner checks."""
import numpy as np

import _navier_stokes_oracle as nso
import _stokes_oracle as so
from _coef_oracle import _cells, _t3, geometry
from _coef_oracle import cell_matrices as _coef_cell_matrices
from firedrake_b200.fiat_lite import interval_element

KP_MASS = 1e-6


def pressure_element(el):
    return so.pressure_element(el)


def cell_actions(el, X, r, u, nu, beta=0.0):
    """Element actions of F_p(u) for a batch of cells: X (nc, 8, 3), r (nc, [m,] NP), u (nc, ND, 3) ->
    like r."""
    pe = pressure_element(el)
    Bq, Dq = np.asarray(pe.B), np.asarray(pe.D)
    nqp = Bq.shape[1]
    Kinv, detw = geometry(el, X)
    rr = r.reshape(r.shape[:-1] + (nqp, nqp, nqp))
    extra = rr.ndim - 4
    ex = lambda a: a.reshape(a.shape[:1] + (1,) * extra + a.shape[1:])
    gh = np.stack([_t3(Dq, Bq, Bq, rr), _t3(Bq, Dq, Bq, rr), _t3(Bq, Bq, Dq, rr)], axis=-1)
    g = np.einsum("...ijks,...ijkse->...ijke", gh, ex(Kinv))               # physical gradient of r
    f = nu * np.einsum("...ijkre,...ijke->...ijkr", ex(Kinv), g) * ex(detw)[..., None]
    uq = nso._values(el, u)                                                # (nc, i, j, k, 3)
    v = ex(detw) * (beta * _t3(Bq, Bq, Bq, rr) + np.einsum("...ijke,...ijke->...ijk", ex(uq), g))
    y = (_t3(Dq.T, Bq.T, Bq.T, f[..., 0]) + _t3(Bq.T, Dq.T, Bq.T, f[..., 1]) + _t3(Bq.T, Bq.T, Dq.T, f[..., 2])
         + _t3(Bq.T, Bq.T, Bq.T, v))
    return y.reshape(r.shape)


def _gather(el, coords, u, geo, geo2):
    i0, i1 = _cells(*geo)
    i2 = so._pressure_cells(*geo2, geo[4])
    return i0, i2, coords.reshape(-1, 3)[i1], np.asarray(u).reshape(-1, 3)[i0]


def action(el, coords, r, u, geo, geo2, nu, beta=0.0):
    """assemble(action(F_p(u), r)): r one per pressure node, u flat AoS (3 per velocity node).
    geo = (map0, off0, map1, off1, nlay), geo2 = (map2, off2)."""
    _, i2, Xc, uc = _gather(el, coords, u, geo, geo2)
    y = np.zeros(len(r))
    np.add.at(y, i2, cell_actions(el, Xc, np.asarray(r)[i2], uc, nu, beta))
    return y


def _csr(i2, K, nq):
    import scipy.sparse as sps
    nt = i2.shape[1]
    return sps.csr_matrix((K.ravel(), (np.repeat(i2, nt, axis=1).ravel(), np.tile(i2, (1, nt)).ravel())),
                          shape=(nq, nq))


def matrix(el, coords, u, geo, geo2, nq, nu, beta=0.0):
    """F_p(u) as scipy CSR over the pressure nodes, row = test, column = trial."""
    _, i2, Xc, uc = _gather(el, coords, u, geo, geo2)
    npd = i2.shape[1]
    K = np.empty((len(Xc), npd, npd))
    step = max(1, 4096 // npd)
    for c in range(0, len(Xc), step):
        e = min(c + step, len(Xc))
        E = np.broadcast_to(np.eye(npd), (e - c, npd, npd))
        K[c:e] = np.swapaxes(cell_actions(el, Xc[c:e], E, uc[c:e], nu, beta), 1, 2)
    return _csr(i2, K, nq)


def helmholtz_matrix(el, coords, geo, geo2, nq, alpha, beta):
    """alpha*inner(grad r, grad q)*dx + beta*r*q*dx on Q, from the scalar Helmholtz oracle with the velocity's
    rule: K_p = helmholtz_matrix(.., 1, KP_MASS), M_p = helmholtz_matrix(.., 0, 1)."""
    _, i1 = _cells(*geo)
    i2 = so._pressure_cells(*geo2, geo[4])
    pe = interval_element(el.ndof - 2, el.nq)
    K = _coef_cell_matrices(pe, coords.reshape(-1, 3)[i1], np.ones(i2.shape), alpha, beta)
    return _csr(i2, K, nq)


def fgmres(A, b, prec, rtol=1e-8, maxit=500, restart=None, project=None):
    """Right-preconditioned flexible GMRES from x = 0 (no restart unless ``restart``): A and prec are
    callables.  ``project`` is applied to every preconditioned vector.  Returns (x, iterations, converged)."""
    restart = restart or maxit
    x = np.zeros_like(b)
    nb = np.linalg.norm(b)
    its = 0
    while True:
        r = b - A(x)
        beta = np.linalg.norm(r)
        if beta <= rtol * nb:
            return x, its, True
        if its >= maxit:
            return x, its, False
        m = min(restart, maxit - its)
        V = np.zeros((m + 1, len(b)))
        Z = np.zeros((m, len(b)))
        H = np.zeros((m + 1, m))
        V[0] = r / beta
        k = 0
        for k in range(m):
            z = prec(V[k])
            Z[k] = project(z) if project else z
            w = A(Z[k])
            for i in range(k + 1):
                H[i, k] = w @ V[i]
                w = w - H[i, k] * V[i]
            H[k + 1, k] = np.linalg.norm(w)
            its += 1
            e1 = np.zeros(k + 2)
            e1[0] = beta
            y, *_ = np.linalg.lstsq(H[:k + 2, :k + 1], e1, rcond=None)
            res = np.linalg.norm(H[:k + 2, :k + 1] @ y - e1)
            if res <= rtol * nb or H[k + 1, k] == 0.0:
                break
            V[k + 1] = w / H[k + 1, k]
        x = x + Z[:k + 1].T @ y
        if res <= rtol * nb:
            return x, its, True
