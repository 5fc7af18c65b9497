"""SciPy oracle of the GTMG trace preconditioner (FDB_FORM_TRACE_PROLONG / _RESTRICT and mg.GTMG): the CG1 -> trace
interpolation P as a sparse matrix built from the trace numbering and the cell vertices, the Q1 stiffness matrix, and a
two-level cycle (Chebyshev-Jacobi on H, exact or Jacobi-CG coarse solve) -- no engine code.

Trace dof t of a cell (face 2d + s, GL indices t0, t1 along the tangential axes e0 < e1) is the point xi with xi_d = s,
xi_e0 = x_t0, xi_e1 = x_t1 (x the k Gauss-Legendre points on [0, 1]); P[t, v] is the trilinear basis of local vertex
v = (a0 * 2 + a1) * 2 + a2 there."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from firedrake_b200.fiat_lite import gauss_legendre


def reference_points(k):
    """(6k^2, 3) reference coordinates of the trace dofs of a cell."""
    x, _ = gauss_legendre(k)
    pts = np.zeros((6 * k * k, 3))
    for t in range(6 * k * k):
        f, r = divmod(t, k * k)
        d, s = divmod(f, 2)
        t0, t1 = divmod(r, k)
        e0, e1 = [e for e in range(3) if e != d]
        pts[t, d], pts[t, e0], pts[t, e1] = s, x[t0], x[t1]
    return pts


def trilinear(pts):
    """(npts, 8): the Q1 basis of local vertex (a0 * 2 + a1) * 2 + a2 at reference points."""
    out = np.ones((len(pts), 8))
    for v in range(8):
        for e in range(3):
            a = (v >> (2 - e)) & 1
            out[:, v] *= pts[:, e] if a else 1.0 - pts[:, e]
    return out


def prolongation(T, V1):
    """P (trace nodes x CG1 nodes), CSR; a shared face's rows are set (both cells give the same row)."""
    k = T.k
    Pl = trilinear(reference_points(k))
    ft, fv = T.full_cell_node_list(), V1.full_cell_node_list()
    P = sp.lil_matrix((T.node_count, V1.node_count))
    for c in range(ft.shape[0]):
        for t in range(6 * k * k):
            for v in range(8):
                if Pl[t, v] != 0.0:
                    P[ft[c, t], fv[c, v]] = Pl[t, v]
    return P.tocsr()


def trace_weights(T):
    return 1.0 / np.bincount(T.full_cell_node_list().ravel(), minlength=T.node_count)


def stiffness(mesh, V1, kappa=1.0):
    """kappa * (grad u, grad v) on CG1 with 2^3 Gauss points per cell (exact on parallelepipeds)."""
    xq, wq = gauss_legendre(2)
    fv = V1.full_cell_node_list()
    fc = mesh.coord_space.full_cell_node_list()
    rows, cols, vals = [], [], []
    pts = np.array([[a, b, c] for a in xq for b in xq for c in xq])
    wts = np.array([a * b * c for a in wq for b in wq for c in wq])
    grads = []
    for p in pts:
        g = np.zeros((8, 3))
        for v in range(8):
            a = [(v >> (2 - e)) & 1 for e in range(3)]
            f = [p[e] if a[e] else 1.0 - p[e] for e in range(3)]
            df = [1.0 if a[e] else -1.0 for e in range(3)]
            g[v] = [df[0] * f[1] * f[2], f[0] * df[1] * f[2], f[0] * f[1] * df[2]]
        grads.append(g)
    for c in range(fv.shape[0]):
        X = mesh.coordinates[fc[c]]
        K = np.zeros((8, 8))
        for g, w in zip(grads, wts):
            J = X.T @ g                       # dx/dxi
            G = g @ np.linalg.inv(J)          # physical gradients
            K += w * abs(np.linalg.det(J)) * kappa * (G @ G.T)
        rows.append(np.repeat(fv[c], 8))
        cols.append(np.tile(fv[c], 8))
        vals.append(K.ravel())
    n = V1.node_count
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))


def masked(A, rows):
    """A with ``rows`` and their columns replaced by the identity (Dirichlet / natural-face rows)."""
    A = sp.lil_matrix(A)
    for r in rows:
        A.rows[r], A.data[r] = [], []
    A = A.tocsc()
    keep = np.ones(A.shape[0])
    keep[rows] = 0.0
    D = sp.diags(keep)
    return (D @ A @ D + sp.diags(1.0 - keep)).tocsr()


def lanczos_bounds(H, dinv, rhs, steps=10):
    """(lmin, lmax) of D^-1 H from ``steps`` Jacobi-CG steps (mg.jacobi_lanczos_bounds)."""
    r = rhs.copy()
    z = dinv * r
    p = z.copy()
    rz = r @ z
    al, be = [], []
    for _ in range(steps):
        Ap = H @ p
        a = rz / (p @ Ap)
        r = r - a * Ap
        z = dinv * r
        rzn = r @ z
        al.append(a)
        be.append(rzn / rz)
        p = z + rzn / rz * p
        rz = rzn
    m = len(al)
    Tm = np.zeros((m, m))
    for j in range(m):
        Tm[j, j] = 1.0 / al[j] + (be[j - 1] / al[j - 1] if j else 0.0)
        if j + 1 < m:
            Tm[j, j + 1] = Tm[j + 1, j] = np.sqrt(be[j]) / al[j]
    ev = np.linalg.eigvalsh(Tm)
    return ev[0], ev[-1]


def chebyshev(H, dinv, b, x, lo, hi, nu):
    theta, delta = 0.5 * (hi + lo), 0.5 * (hi - lo)
    sigma = theta / delta
    rho = 1.0 / sigma
    d = dinv * (b - H @ x) / theta
    x = x + d
    for _ in range(nu - 1):
        rn = 1.0 / (2.0 * sigma - rho)
        d = rn * rho * d + 2.0 * rn / delta * dinv * (b - H @ x)
        x = x + d
        rho = rn
    return x


class TwoLevel:
    """The GTMG cycle on the masked trace matrix H (natural rows identity) with the masked coarse A = stiffness / alpha
    (Dirichlet rows identity on the natural sub-domains' CG1 nodes): pre-smooth, restrict P^T, coarse solve (exact,
    or Jacobi-CG to ``coarse_rtol``), prolong, post-smooth."""

    def __init__(self, H, A, P, nat_t, nat_c, nu=3, coarse_rtol=None, nullspace=False, seed=0):
        self.H, self.A, self.P, self.nu = H, A, P, nu
        self.nat_t, self.nat_c, self.coarse_rtol, self.nullspace = nat_t, nat_c, coarse_rtol, nullspace
        self.dinv = 1.0 / H.diagonal()
        self.adinv = 1.0 / A.diagonal()
        rhs = np.random.default_rng(seed).standard_normal(H.shape[0])
        rhs[nat_t] = 0.0
        lo, hi = lanczos_bounds(H, self.dinv, rhs)
        self.lo, self.hi = 0.1 * hi, 1.1 * hi
        self.Ad = None if nullspace or coarse_rtol is not None else spla.factorized(A.tocsc())

    def coarse(self, b):
        if self.nullspace:
            b = b - b.mean()
        if self.Ad is not None:
            return self.Ad(b)
        if self.coarse_rtol is None:                      # singular, consistent: least squares
            return spla.lsqr(self.A, b, atol=1e-14, btol=1e-14, iter_lim=10000)[0]
        x, _ = spla.cg(self.A, b, rtol=self.coarse_rtol, maxiter=500, M=sp.diags(self.adinv))
        return x

    def __call__(self, r):
        x = chebyshev(self.H, self.dinv, r, np.zeros_like(r), self.lo, self.hi, self.nu)
        res = r - self.H @ x
        res[self.nat_t] = 0.0
        bc = self.P.T @ res
        bc[self.nat_c] = 0.0
        e = self.P @ self.coarse(bc)
        e[self.nat_t] = 0.0
        return chebyshev(self.H, self.dinv, r, x + e, self.lo, self.hi, self.nu)


def pcg(H, b, M, rtol=1e-8, maxit=2000, nullspace=False):
    """Preconditioned CG from 0; returns (x, iterations)."""
    def proj(v):
        return v - v.mean() if nullspace else v
    b = proj(b)
    x = np.zeros_like(b)
    r = b.copy()
    z = proj(M(r))
    p = z.copy()
    rz = r @ z
    r0 = np.linalg.norm(r)
    it = 0
    while np.linalg.norm(r) > rtol * r0 and it < maxit:
        Ap = H @ p
        a = rz / (p @ Ap)
        x += a * p
        r -= a * Ap
        z = proj(M(r))
        rzn = r @ z
        p = z + rzn / rz * p
        rz = rzn
        it += 1
    return x, it


def trace_matrix(mesh, S, Q, T, alpha):
    """H = sum_K C^ K_K^-1 C^^T (tests/_hybrid_oracle.py) assembled sparse, no boundary rows modified."""
    import _hybrid_oracle as ho
    k = S.degree
    C = ho.trace_coupling(k)
    Ch = np.hstack([C, np.zeros((C.shape[0], k ** 3))])
    rows, cols, vals = [], [], []
    for rs, rq, rt, Xv in ho.cell_data(mesh, S, Q, T):
        HK = Ch @ np.linalg.solve(ho.local_saddle(k, Xv, alpha), Ch.T)
        rows.append(np.repeat(rt, len(rt)))
        cols.append(np.tile(rt, len(rt)))
        vals.append(HK.ravel())
    n = T.node_count
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))


def cg1_boundary_nodes(V1, subs):
    return (np.unique(np.concatenate([V1.boundary_nodes(s) for s in subs])) if subs
            else np.zeros(0, dtype=np.int64))
