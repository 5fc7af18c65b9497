"""TEST INFRASTRUCTURE: NumPy oracle of the symmetric interior penalty (SIPG) discretisation on scalar DQ_p hexahedra

    a(u, v) = alpha*inner(grad u, grad v)*dx + beta*u*v*dx
              + alpha*( -inner(avg(grad u), jump(v, n)) - inner(jump(u, n), avg(grad v))
                        + (eta/avg(h))*inner(jump(u, n), jump(v, n)) )*dS
              + ( c_m*u*v + (c_p/h)*u*v - c_s*u*dot(grad v, n) - c_f*dot(grad u, n)*v )*ds(D)

with a trilinear (Q1) coordinate field, assembled element by element with the full 3-D basis and the full 3-D
Jacobian at every quadrature point (no sum factorisation).  Conventions: dof (ax*N + ay)*N + az with the 1-D Gauss-
Legendre nodes ascending, vertex (bx*2 + by)*2 + bz, local facet f = 2*direction + side whose face is parametrised by
the other two reference axes (s, t) in increasing order.  h is the largest distance between two of a cell's 8
vertices; the unit normal is the normalised dX/ds x dX/dt of the '+' cell, turned to point away from that cell's
centroid.  The facet lists are built here from the mesh, independently of firedrake_b200.assemble."""
import numpy as np
import scipy.sparse as sp

from firedrake_b200.fiat_lite import interval_element

import _boundary_oracle as bo


def element(p):
    return interval_element(p, variant="gl")


def basis3(el, pts):
    """The tensor basis at reference points pts (m, 3): values (m, N^3) and reference gradients (m, N^3, 3)."""
    n = el.ndof
    tabs = [el.tabulate(pts[:, d]) for d in range(3)]            # (B, D) per axis, each (m, n)
    B = [t[0] for t in tabs]
    D = [t[1] for t in tabs]
    val = np.einsum("ma,mb,mc->mabc", B[0], B[1], B[2]).reshape(len(pts), n ** 3)
    g0 = np.einsum("ma,mb,mc->mabc", D[0], B[1], B[2]).reshape(len(pts), n ** 3)
    g1 = np.einsum("ma,mb,mc->mabc", B[0], D[1], B[2]).reshape(len(pts), n ** 3)
    g2 = np.einsum("ma,mb,mc->mabc", B[0], B[1], D[2]).reshape(len(pts), n ** 3)
    return val, np.stack([g0, g1, g2], axis=-1)


def jacobians(Xc, pts):
    """J[c, q, i, d] = dX_i/dxi_d of the trilinear maps of cells Xc (nc, 8, 3) at pts (m, 3)."""
    b = np.array([[(v >> 2) & 1, (v >> 1) & 1, v & 1] for v in range(8)], dtype=float)     # (8, 3)
    f = np.where(b[None, :, :] > 0, pts[:, None, :], 1.0 - pts[:, None, :])                # (m, 8, 3)
    s = np.where(b > 0, 1.0, -1.0)                                                          # (8, 3)
    dN = np.empty((len(pts), 8, 3))
    for d in range(3):
        o = [e for e in range(3) if e != d]
        dN[:, :, d] = s[None, :, d] * f[:, :, o[0]] * f[:, :, o[1]]
    return np.einsum("cvi,qvd->cqid", Xc, dN)


def diameters(Xc):
    d = Xc[:, :, None, :] - Xc[:, None, :, :]
    return np.sqrt((d ** 2).sum(-1)).reshape(len(Xc), -1).max(axis=1)


def face_points(el, f):
    """The reference points of facet f's Gauss points (N^2, 3), (a along s, b along t)."""
    d, side = int(f) // 2, int(f) % 2
    s_ax, t_ax = [e for e in range(3) if e != d]
    a, b = np.divmod(np.arange(el.nq ** 2), el.nq)
    pts = np.empty((el.nq ** 2, 3))
    pts[:, d] = side
    pts[:, s_ax] = el.xq[a]
    pts[:, t_ax] = el.xq[b]
    return pts


def face_weights(el):
    a, b = np.divmod(np.arange(el.nq ** 2), el.nq)
    return el.wq[a] * el.wq[b]


def cell_matrices(el, Xc, alpha, beta):
    """(nc, N^3, N^3): alpha*inner(grad u, grad v)*dx + beta*u*v*dx with N^3 Gauss points."""
    n = el.nq
    q = np.stack(np.meshgrid(el.xq, el.xq, el.xq, indexing="ij"), axis=-1).reshape(-1, 3)
    w = np.einsum("a,b,c->abc", el.wq, el.wq, el.wq).ravel()
    assert len(q) == n ** 3
    val, grad = basis3(el, q)
    J = jacobians(Xc, q)
    Ki = np.linalg.inv(J)                                            # (nc, m, d, i)
    det = np.abs(np.linalg.det(J))
    G = np.einsum("cqdi,qjd->cqji", Ki, grad)                        # physical gradients (nc, m, ND, 3)
    wd = det * w[None, :]
    return alpha * np.einsum("cq,cqji,cqki->cjk", wd, G, G) + beta * np.einsum("cq,qj,qk->cjk", wd, val, val)


def _side_data(el, Xc, f):
    """Values (m, ND), physical gradients (nf, m, ND, 3), J (nf, m, 3, 3) of cells Xc on their facets f (one facet
    number per entry, grouped here by value)."""
    nd = el.ndof ** 3
    m = el.nq ** 2
    val = np.empty((len(f), m, nd))
    grad = np.empty((len(f), m, nd, 3))
    J = np.empty((len(f), m, 3, 3))
    for fv in np.unique(f):
        sel = f == fv
        pts = face_points(el, fv)
        v, g = basis3(el, pts)
        Js = jacobians(Xc[sel], pts)
        val[sel] = v[None]
        J[sel] = Js
        grad[sel] = np.einsum("cqdi,qjd->cqji", np.linalg.inv(Js), g)
    return val, grad, J


def _normal_and_weight(el, Xc, f, J):
    """Unit normal outward from cells Xc on facets f and the surface weights w_s w_t |dX/ds x dX/dt|."""
    d = np.asarray(f) // 2
    s_ax = np.where(d == 0, 1, 0)
    t_ax = np.where(d == 2, 1, 2)
    idx = np.arange(len(f))
    Xs = J[idx, :, :, s_ax]                                          # (nf, m, 3)
    Xt = J[idx, :, :, t_ax]
    c = np.cross(Xs, Xt)
    area = np.linalg.norm(c, axis=-1)
    n = c / area[..., None]
    cen = Xc.mean(axis=1)
    fvs = np.stack([Xc[i, bo.face_vertices(fi)].mean(axis=0) for i, fi in enumerate(f)])
    sgn = np.sign(np.einsum("fi,fi->f", n.mean(axis=1), fvs - cen))
    return n * sgn[:, None, None], area * face_weights(el)[None, :]


def interior_matrices(el, Xp, Xm, fp, fm, alpha, eta):
    """(nf, 2 N^3, 2 N^3) element matrices of the dS terms, rows/columns '+' dofs then '-' dofs."""
    vp, gp, Jp = _side_data(el, Xp, fp)
    vm, gm, _ = _side_data(el, Xm, fm)
    n, W = _normal_and_weight(el, Xp, fp, Jp)
    sig = eta / (0.5 * (diameters(Xp) + diameters(Xm)))
    val = np.concatenate([np.broadcast_to(vp, gp.shape[:3]), -np.broadcast_to(vm, gm.shape[:3])], axis=2)   # s*phi
    dn = np.concatenate([np.einsum("fqji,fqi->fqj", gp, n), np.einsum("fqji,fqi->fqj", gm, n)], axis=2)
    # -avg(dn u) s_v v - s_u u avg(dn v) + sig s_u u s_v v
    A = -0.5 * np.einsum("fq,fqi,fqj->fij", W, val, dn) - 0.5 * np.einsum("fq,fqj,fqi->fij", W, val, dn) \
        + np.einsum("fq,f,fqi,fqj->fij", W, sig, val, val)
    return alpha * A


def exterior_matrices(el, Xc, f, c_m, c_p, c_s, c_f):
    """(nf, N^3, N^3) element matrices of (c_m u v + (c_p/h) u v - c_s u dn(v) - c_f dn(u) v) ds; row = test."""
    v, g, J = _side_data(el, Xc, f)
    n, W = _normal_and_weight(el, Xc, f, J)
    v = np.broadcast_to(v, g.shape[:3])
    dn = np.einsum("fqji,fqi->fqj", g, n)
    h = diameters(Xc)
    return (np.einsum("fq,fqi,fqj->fij", W * (c_m + c_p / h[:, None]), v, v)
            - c_s * np.einsum("fq,fqi,fqj->fij", W, dn, v) - c_f * np.einsum("fq,fqi,fqj->fij", W, v, dn))


# ------------------------------------------------------------------------------------------------- mesh level
def cells(mesh, W):
    """Every cell of an extruded mesh: dof rows (nc, N^3), vertex coordinates (nc, 8, 3), row c*nz + l."""
    return (W.full_cell_node_list().astype(np.int64),
            mesh.coordinates[mesh.coord_space.full_cell_node_list().astype(np.int64)])


def interior_facets(mesh):
    """(cell '+', cell '-', f '+', f '-') over all interior facets, cells as rows c*nz + l of :func:`cells`."""
    nz = mesh.nz
    cp, cm, local = mesh.interior_vertical_facets()
    lay = np.arange(nz)
    P = [(cp[:, None] * nz + lay).ravel()]
    M = [(cm[:, None] * nz + lay).ravel()]
    FP = [np.repeat(local[:, 0], nz)]
    FM = [np.repeat(local[:, 1], nz)]
    c = np.arange(mesh.num_base_cells)
    for l in range(nz - 1):
        P.append(c * nz + l)
        M.append(c * nz + l + 1)
        FP.append(np.full(len(c), 5))
        FM.append(np.full(len(c), 4))
    return tuple(np.concatenate(a).astype(np.int64) for a in (P, M, FP, FM))


def exterior_facets(mesh, sub_domain):
    """(cell, f) over the exterior facets of ``ds(sub_domain)``."""
    nz = mesh.nz
    cells_, local = mesh.exterior_vertical_facets()
    C, F = [], []
    for s in bo.subs_of(sub_domain):
        if s in ("bottom", "top"):
            c = np.arange(mesh.num_base_cells)
            C.append(c * nz + (0 if s == "bottom" else nz - 1))
            F.append(np.full(len(c), 4 if s == "bottom" else 5))
        else:
            c = cells_[local == s - 1].astype(np.int64)
            C.append((c[:, None] * nz + np.arange(nz)).ravel())
            F.append(np.full(len(c) * nz, s - 1))
    if not C:
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)
    return np.concatenate(C).astype(np.int64), np.concatenate(F).astype(np.int64)


def _scatter(rows, M, n):
    r = np.repeat(rows, rows.shape[1], axis=1).ravel()
    c = np.tile(rows, (1, rows.shape[1])).ravel()
    return sp.csr_matrix((M.ravel(), (r, c)), shape=(n, n))


def cell_matrix(mesh, W, el, alpha, beta):
    rows, Xc = cells(mesh, W)
    return _scatter(rows, cell_matrices(el, Xc, alpha, beta), W.node_count)


def interior_matrix(mesh, W, el, alpha, eta):
    rows, Xc = cells(mesh, W)
    P, M, FP, FM = interior_facets(mesh)
    A = interior_matrices(el, Xc[P], Xc[M], FP, FM, alpha, eta)
    return _scatter(np.concatenate([rows[P], rows[M]], axis=1), A, W.node_count)


def exterior_matrix(mesh, W, el, sub_domain, c_m, c_p, c_s, c_f):
    rows, Xc = cells(mesh, W)
    C, F = exterior_facets(mesh, sub_domain)
    if len(C) == 0:
        return sp.csr_matrix((W.node_count, W.node_count))
    return _scatter(rows[C], exterior_matrices(el, Xc[C], F, c_m, c_p, c_s, c_f), W.node_count)


def operator(mesh, W, el, alpha, beta, eta, weak_bcs="on_boundary"):
    """The global matrix of a (scipy CSR)."""
    A = cell_matrix(mesh, W, el, alpha, beta) + interior_matrix(mesh, W, el, alpha, eta)
    if weak_bcs:
        A = A + exterior_matrix(mesh, W, el, weak_bcs, 0.0, alpha * eta, alpha, alpha)
    return A.tocsr()


def nitsche_load(mesh, W, el, alpha, eta, weak_bcs, g):
    return exterior_matrix(mesh, W, el, weak_bcs, 0.0, alpha * eta, alpha, 0.0) @ g


def flux_load(mesh, W, el, sub_domain, g):
    return exterior_matrix(mesh, W, el, sub_domain, 1.0, 0.0, 0.0, 0.0) @ g
