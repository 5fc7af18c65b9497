"""NumPy oracle of mixed Poisson on NCF_k x DQ_{k-1} hexahedra (FDB_FORM_MIXED_POISSON, _SCHUR): every 3-D basis
function is tabulated at every 3-D quadrature point as a dense array, the contravariant Piola map is applied with
the point's Jacobian, and the element matrices are dense sums over the points.  Nothing here is sum-factorised:
it states the form the way a textbook does, independently of the kernels' 1-D tables.

    a((sigma, u), (tau, v)) = alpha*dot(sigma, tau)*dx + div(tau)*u*dx + div(sigma)*v*dx

Reference flux basis: component d of the local dof in block d is phi_{i_d}(x_d) prod_{e != d} psi_{i_e}(x_e), CG_k
(GLL, FIAT entity order) along d, DG_{k-1} (Gauss-Legendre, ascending) along the others; block index (i0 * n1 +
i1) * n2 + i2.  Physical sigma = J sigma^ / det J, div sigma = div^ sigma^ / det J."""
import itertools

import numpy as np
import scipy.sparse as sps

from firedrake_b200.fiat_lite import gauss_legendre, interval_element


def _tables(k, x):
    """CG_k and DG_{k-1} values / derivatives at the 1-D points x."""
    Bc, Dc = interval_element(k).tabulate(x)
    Bg, Dg = interval_element(k - 1, variant="gl").tabulate(x)
    return Bc, Dc, Bg, Dg


def ncf_dofs(k):
    """(d, (i0, i1, i2)) of every local flux dof, in the local numbering."""
    out = []
    for d in range(3):
        dims = [k + 1 if e == d else k for e in range(3)]
        out += [(d, idx) for idx in itertools.product(*(range(n) for n in dims))]
    return out


def tabulate(k, pts):
    """Reference flux basis at 3-D points (n, 3): values (arity, n, 3) and divergences (arity, n); the DQ_{k-1}
    basis (k^3, n)."""
    T = [_tables(k, pts[:, e]) for e in range(3)]
    dofs = ncf_dofs(k)
    val = np.zeros((len(dofs), len(pts), 3))
    div = np.zeros((len(dofs), len(pts)))
    for j, (d, idx) in enumerate(dofs):
        f = np.ones(len(pts))
        df = np.ones(len(pts))
        for e in range(3):
            Bc, Dc, Bg, _ = T[e]
            if e == d:
                f = f * Bc[:, idx[e]]
                df = df * Dc[:, idx[e]]
            else:
                f = f * Bg[:, idx[e]]
                df = df * Bg[:, idx[e]]
        val[j, :, d] = f
        div[j] = df
    psi = np.array([T[0][2][:, a] * T[1][2][:, b] * T[2][2][:, c]
                    for a, b, c in itertools.product(range(k), repeat=3)])
    return val, div, psi


def points(n):
    x, w = gauss_legendre(n)
    P = np.array(list(itertools.product(x, x, x)))
    W = np.array([a * b * c for a, b, c in itertools.product(w, w, w)])
    return P, W


def jacobians(Xv, pts):
    """J (n, 3, 3) of the trilinear map of the 8 vertices Xv (vertex (b0*2 + b1)*2 + b2 at (b0, b1, b2))."""
    J = np.zeros((len(pts), 3, 3))
    for v in range(8):
        b = [(v >> 2) & 1, (v >> 1) & 1, v & 1]
        f = [pts[:, e] if b[e] else 1.0 - pts[:, e] for e in range(3)]
        for r in range(3):
            g = (1.0 if b[r] else -1.0) * np.prod([f[e] for e in range(3) if e != r], axis=0)
            J[:, :, r] += Xv[v][None, :] * g[:, None]
    return J


def trilinear(Xv, pts):
    out = np.zeros((len(pts), Xv.shape[1]))
    for v in range(8):
        b = [(v >> 2) & 1, (v >> 1) & 1, v & 1]
        out += np.prod([pts[:, e] if b[e] else 1.0 - pts[:, e] for e in range(3)], axis=0)[:, None] * Xv[v][None]
    return out


def element_matrices(k, Xv, alpha=1.0):
    """Dense alpha*M (arity x arity) and B (k^3 x arity) of one cell, by the (k+1)^3-point Gauss rule."""
    P, W = points(k + 1)
    val, div, psi = tabulate(k, P)
    J = jacobians(Xv, P)
    det = np.linalg.det(J)
    sig = np.einsum("qab,jqb->jqa", J, val) / det[None, :, None]          # physical basis
    M = alpha * np.einsum("q,iqa,jqa->ij", W * det, sig, sig)
    Bm = np.einsum("q,vq,jq->vj", W * det, psi, div / det[None, :])
    return M, Bm


def cells(mesh, S, Q):
    """(flux rows, DQ rows, vertex coordinates (8, 3)) of every cell."""
    fs, fq = S.full_cell_node_list(), Q.full_cell_node_list()
    fc = mesh.coord_space.full_cell_node_list()
    for c in range(fs.shape[0]):
        yield fs[c], fq[c], mesh.coordinates[fc[c]]


def global_matrices(mesh, S, Q, alpha=1.0):
    """Sparse alpha*M (nS x nS) and B (nQ x nS): the element matrices of :func:`element_matrices`, all cells at
    once."""
    Xv = mesh.coordinates[mesh.coord_space.full_cell_node_list()]               # (ncell, 8, 3)
    return matrices_from_rows(S.degree, Xv, S.full_cell_node_list(), Q.full_cell_node_list(), S.node_count,
                              Q.node_count, alpha)


def matrices_from_rows(k, Xv, fs, fq, nS, nQ, alpha=1.0):
    """The same from the cells' vertex coordinates (ncell, 8, 3), flux rows (ncell, 3k^2(k+1)) and DQ rows
    (ncell, k^3)."""
    P, W = points(k + 1)
    val, div, psi = tabulate(k, P)
    J = np.stack([jacobians(x, P) for x in Xv])                                  # (ncell, nq, 3, 3)
    det = np.linalg.det(J)
    G = np.einsum("cqka,cqkb->cqab", J, J) / det[:, :, None, None]
    Me = alpha * np.einsum("q,cqab,iqa,jqb->cij", W, G, val, val)
    Be = np.broadcast_to(np.einsum("q,vq,jq->vj", W, psi, div), (len(fs),) + (psi.shape[0], val.shape[0]))
    ar, aq = fs.shape[1], fq.shape[1]
    M = sps.csr_matrix((Me.ravel(), (np.repeat(fs, ar, axis=1).ravel(), np.tile(fs, (1, ar)).ravel())),
                       shape=(nS, nS))
    Bm = sps.csr_matrix((Be.ravel(), (np.repeat(fq, ar, axis=1).ravel(), np.tile(fs, (1, aq)).ravel())),
                        shape=(nQ, nS))
    return M, Bm


def saddle(M, Bm):
    return sps.bmat([[M, Bm.T], [Bm, None]], format="csr")


def constrained(K, rows):
    """K with the rows and columns of ``rows`` replaced by the identity."""
    K = sps.lil_matrix(K)
    K[rows, :] = 0.0
    K[:, rows] = 0.0
    K[rows, rows] = 1.0
    return K.tocsr()


def dq_mass(mesh, Q):
    """The DQ_{k-1} mass matrix (block diagonal), exact (the k-point rule)."""
    k = Q.degree + 1
    P, W = points(k + 1)
    _, _, psi = tabulate(k, P)
    rows, cols, vals = [], [], []
    fq, fc = Q.full_cell_node_list(), mesh.coord_space.full_cell_node_list()
    for c in range(fq.shape[0]):
        det = np.linalg.det(jacobians(mesh.coordinates[fc[c]], P))
        Me = np.einsum("q,vq,wq->vw", W * det, psi, psi)
        rows.append(np.repeat(fq[c], len(fq[c])))
        cols.append(np.tile(fq[c], len(fq[c])))
        vals.append(Me.ravel())
    n = Q.node_count
    return sps.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))


def dirichlet_load(mesh, S, g, sub_domain):
    """The natural condition u = g: the load int (tau.n) g ds over ``sub_domain`` (1..4, "bottom", "top"), g given
    at the vertices (trilinear).  tau.n ds = tau^.n^ ds^ under the contravariant Piola map."""
    k = S.degree
    side = {1: (0, 0), 2: (0, 1), 3: (1, 0), 4: (1, 1), "bottom": (2, 0), "top": (2, 1)}[sub_domain]
    d, s = side
    nx, ny, nz = mesh.nx, mesh.ny, mesh.nz
    x, w = gauss_legendre(k + 1)
    out = np.zeros(S.node_count)
    fs, fc = S.full_cell_node_list(), mesh.coord_space.full_cell_node_list()
    cix = np.repeat(mesh.cell_ix, nz)
    ciy = np.repeat(mesh.cell_iy, nz)
    ciz = np.tile(np.arange(nz), mesh.num_base_cells)
    pos = (cix, ciy, ciz)
    last = (nx - 1, ny - 1, nz - 1)
    fp = np.array(list(itertools.product(x, x)))
    fw = np.array([a * b for a, b in itertools.product(w, w)])
    pts = np.insert(fp, d, float(s), axis=1)
    val, _, _ = tabulate(k, pts)
    for c in np.nonzero(pos[d] == (last[d] if s else 0))[0]:
        gq = trilinear(g[fc[c]][:, None], pts)[:, 0]
        out[fs[c]] += (2 * s - 1) * np.einsum("q,jq->j", fw * gq, val[:, :, d])
    return out


def field_errors(mesh, S, Q, sigma, u, u_exact, grad_exact, nq=None):
    """L2 errors of the discrete (sigma, u) against u_exact(x) and its gradient, (n, 3) -> (n,) / (n, 3)."""
    k = S.degree
    P, W = points(nq or k + 3)
    val, _, psi = tabulate(k, P)
    eu = es = 0.0
    for rs, rq, Xv in cells(mesh, S, Q):
        J = jacobians(Xv, P)
        det = np.linalg.det(J)
        X = trilinear(Xv, P)
        sh = np.einsum("j,jqa->qa", sigma[rs], val)
        sp = np.einsum("qab,qb->qa", J, sh) / det[:, None]
        uh = psi.T @ u[rq]
        eu += np.sum(W * det * (uh - u_exact(X)) ** 2)
        es += np.sum(W * det * np.sum((sp - grad_exact(X)) ** 2, axis=1))
    return np.sqrt(eu), np.sqrt(es)
