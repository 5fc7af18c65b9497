"""TEST INFRASTRUCTURE: NumPy oracle of the spectral-element (collocated GLL) Helmholtz operator on scalar CG_p
hexahedra

    a(u, v) = alpha*inner(kappa*grad u, grad v)*dx(GLL) + beta*inner(u, v)*dx(GLL)

with a trilinear (Q1) coordinate field, the full 3-D basis tabulated at the (p+1)^3 GLL points (not assuming B = I)
and the full 3-D Jacobian at every point, assembled element by element into a scipy matrix; kappa is nodal,
interpolated to the points by the same basis.  Also: the Gauss-rule load of 1, the leapfrog recurrence with point
sources and receivers, its discrete energy, and point location by brute force.  Conventions as tests/_dg_oracle.py
(dof (ax*N + ay)*N + az in 1-D dof numbering, vertex (bx*2 + by)*2 + bz, cell rows c*nz + l)."""
import numpy as np

from firedrake_b200.fiat_lite import interval_element

import _dg_oracle as do


def element(p):
    return interval_element(p, quadrature="gll")


def points(el):
    return np.stack(np.meshgrid(el.xq, el.xq, el.xq, indexing="ij"), axis=-1).reshape(-1, 3)


def cell_matrices(el, Xc, alpha, beta, kc=None, chunk=256):
    """(nc, N^3, N^3): the element matrices, row = test; kc (nc, N^3) the cells' nodal kappa or None."""
    if len(Xc) > chunk:
        return np.concatenate([cell_matrices(el, Xc[i:i + chunk], alpha, beta, None if kc is None else kc[i:i + chunk])
                               for i in range(0, len(Xc), chunk)])
    q = points(el)
    w = np.einsum("a,b,c->abc", el.wq, el.wq, el.wq).ravel()
    val, grad = do.basis3(el, q)
    J = do.jacobians(Xc, q)
    G = np.einsum("cqdi,qjd->cqji", np.linalg.inv(J), grad)
    wd = np.abs(np.linalg.det(J)) * w[None, :]
    kq = np.ones_like(wd) if kc is None else np.einsum("qj,cj->cq", val, kc)
    K = alpha * np.einsum("cqji,cqki->cjk", (wd * kq)[..., None, None] * G, G, optimize=True)
    M = beta * np.einsum("cq,qj,qk->cjk", wd, val, val)
    return K + M


def operator(mesh, W, p, alpha=1.0, beta=0.0, kappa=None):
    """The global matrix (scipy CSR) of SpectralForm on W = mesh.function_space(p); kappa a nodal array or None."""
    rows, Xc = do.cells(mesh, W)
    rows = rows.astype(np.int64)
    kc = None if kappa is None else np.asarray(kappa)[rows]
    return do._scatter(rows, cell_matrices(element(p), Xc, alpha, beta, kc), W.node_count).tocsr()


def gauss_load_of_one(mesh, W, p):
    """The load int(phi_i) dx with the (p+1)-point Gauss rule (exact on affine cells)."""
    rows, Xc = do.cells(mesh, W)
    el = interval_element(p)
    q = np.stack(np.meshgrid(el.xq, el.xq, el.xq, indexing="ij"), axis=-1).reshape(-1, 3)
    w = np.einsum("a,b,c->abc", el.wq, el.wq, el.wq).ravel()
    val, _ = do.basis3(el, q)
    wd = np.abs(np.linalg.det(do.jacobians(Xc, q))) * w[None, :]
    out = np.zeros(W.node_count)
    np.add.at(out, rows.astype(np.int64), np.einsum("cq,qj->cj", wd, val))
    return out


def leapfrog(K, m, u, u_prev, dt, steps, src=None, amp=None, rec=None, fixed=()):
    """u^{n+1} = 2 u^n - u^{n-1} - dt^2 M^-1 (K u^n - f^n), M = diag(m); f^n = E_src^T amp[n]; rows in ``fixed``
    held at zero.  src / rec: (idx, w) pairs of point_weights.  Returns (u^steps, u^{steps-1}, traces (steps, nrec))."""
    minv = 1.0 / np.asarray(m, dtype=float)
    minv[list(fixed)] = 0.0
    u, up = np.array(u, dtype=float), np.array(u_prev, dtype=float)
    u[list(fixed)] = 0.0
    up[list(fixed)] = 0.0
    tr = []
    for s in range(steps):
        r = K @ u
        if src is not None:
            r -= adjoint(src, amp[s], len(u))
        u, up = 2.0 * u - up - dt * dt * minv * r, u
        if rec is not None:
            tr.append(evaluate(rec, u))
    return u, up, (np.array(tr) if rec is not None else None)


def energy(K, m, u_new, u_old, dt):
    """The conserved leapfrog energy 1/2 v^T M v + 1/2 u^{n+1 T} K u^n, v = (u^{n+1} - u^n) / dt."""
    v = (u_new - u_old) / dt
    return 0.5 * v @ (np.asarray(m) * v) + 0.5 * u_new @ (K @ u_old)


def evaluate(pw, u):
    idx, w = pw
    out = np.einsum("kj,kj->k", w, np.asarray(u)[np.maximum(idx, 0)])
    out[idx[:, 0] < 0] = np.nan
    return out


def adjoint(pw, a, n):
    idx, w = pw
    y = np.zeros(n)
    ok = idx[:, 0] >= 0
    np.add.at(y, idx[ok].ravel(), (np.asarray(a)[ok, None] * w[ok]).ravel())
    return y


def locate_brute_force(mesh, W, pts, tol=1e-8):
    """(cell, xi) by Newton on EVERY cell, the lowest cell number whose reference point is within [-tol, 1+tol]^3."""
    _, Xc = do.cells(mesh, W)
    cells, xis = np.full(len(pts), -1), np.zeros((len(pts), 3))
    b = np.array([[(v >> 2) & 1, (v >> 1) & 1, v & 1] for v in range(8)], dtype=float)
    for k, x in enumerate(pts):
        xi = np.full((len(Xc), 3), 0.5)
        for _ in range(40):
            f = np.where(b[None] > 0, xi[:, None, :], 1.0 - xi[:, None, :])
            X = np.einsum("cv,cvi->ci", f.prod(axis=2), Xc)
            dN = [np.where(b[None, :, d] > 0, 1.0, -1.0) * np.prod(np.delete(f, d, axis=2), axis=2) for d in range(3)]
            J = np.stack([np.einsum("cv,cvi->ci", g, Xc) for g in dN], axis=2)
            xi = np.clip(xi - np.linalg.solve(J, (X - x)[..., None])[..., 0], -1.0, 2.0)
        ok = np.flatnonzero(((xi >= -tol) & (xi <= 1 + tol)).all(axis=1))
        if len(ok):
            cells[k], xis[k] = ok[0], np.clip(xi[ok[0]], 0.0, 1.0)
    return cells, xis
