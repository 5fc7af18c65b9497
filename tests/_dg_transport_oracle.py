"""TEST INFRASTRUCTURE: NumPy oracle of upwind DG transport on scalar DQ_p hexahedra

    a(u, v) = - u*dot(b, grad v)*dx + dot(b, n('+'))*u_up*(v('+') - v('-'))*dS
              + (c_out*max(dot(b, n), 0) + c_in*min(dot(b, n), 0))*u*v*ds

with b given at the mesh vertices and interpolated trilinearly, a trilinear coordinate field, the full 3-D basis and
the full 3-D Jacobian at every quadrature point (p+1 Gauss points per axis on cells and faces), assembled element by
element into a sparse matrix.  Conventions, facet lists, normals and face weights are those of tests/_dg_oracle.py,
whose helpers this reuses."""
import numpy as np

import _dg_oracle as do


def vertex_weights(pts):
    """(m, 8): the trilinear weight of vertex (bx*2 + by)*2 + bz at reference points pts (m, 3)."""
    b = np.array([[(v >> 2) & 1, (v >> 1) & 1, v & 1] for v in range(8)], dtype=float)
    return np.prod(np.where(b[None] > 0, pts[:, None, :], 1.0 - pts[:, None, :]), axis=-1)


def cell_matrices(el, Xc, Bc):
    """(nc, N^3, N^3): -u*dot(b, grad v)*dx, row = test; Bc (nc, 8, 3) the vertex values of b."""
    q = np.stack(np.meshgrid(el.xq, el.xq, el.xq, indexing="ij"), axis=-1).reshape(-1, 3)
    w = np.einsum("a,b,c->abc", el.wq, el.wq, el.wq).ravel()
    val, grad = do.basis3(el, q)
    J = do.jacobians(Xc, q)
    G = np.einsum("cqdi,qjd->cqji", np.linalg.inv(J), grad)
    wd = np.abs(np.linalg.det(J)) * w[None, :]
    bq = np.einsum("qv,cvi->cqi", vertex_weights(q), Bc)
    return -np.einsum("cq,cqi,cqji,qk->cjk", wd, bq, G, val)


def _bn(el, Xc, Bc, f):
    """b.n and the face weights on facets f of cells Xc (n outward from the cell), and the trace tables."""
    v, g, J = do._side_data(el, Xc, f)
    n, W = do._normal_and_weight(el, Xc, f, J)
    bq = np.empty(n.shape)
    for fv in np.unique(f):
        sel = f == fv
        bq[sel] = np.einsum("qv,cvi->cqi", vertex_weights(do.face_points(el, fv)), Bc[sel])
    return np.einsum("fqi,fqi->fq", bq, n), W, np.broadcast_to(v, g.shape[:3])


def interior_matrices(el, Xp, Xm, Bp, fp, fm):
    """(nf, 2 N^3, 2 N^3) upwind flux matrices, rows/columns '+' dofs then '-' dofs."""
    bn, W, vp = _bn(el, Xp, Bp, fp)
    vm = np.broadcast_to(do._side_data(el, Xm, fm)[0], vp.shape)
    up = (bn >= 0)[..., None]
    trial = np.concatenate([vp * up, vm * ~up], axis=2)
    test = np.concatenate([vp, -vm], axis=2)
    return np.einsum("fq,fqi,fqj->fij", W * bn, test, trial)


def exterior_matrices(el, Xc, Bc, f, c_out, c_in):
    bn, W, v = _bn(el, Xc, Bc, f)
    c = c_out * np.maximum(bn, 0.0) + c_in * np.minimum(bn, 0.0)
    return np.einsum("fq,fqi,fqj->fij", W * c, v, v)


# ------------------------------------------------------------------------------------------------- mesh level
def cell_velocities(mesh, bv):
    """(nc, 8, 3): b at every cell's vertices, row c*nz + l as in _dg_oracle.cells."""
    return np.asarray(bv)[mesh.coord_space.full_cell_node_list().astype(np.int64)]


def cell_matrix(mesh, W, el, bv):
    rows, Xc = do.cells(mesh, W)
    return do._scatter(rows, cell_matrices(el, Xc, cell_velocities(mesh, bv)), W.node_count)


def interior_matrix(mesh, W, el, bv):
    rows, Xc = do.cells(mesh, W)
    Bc = cell_velocities(mesh, bv)
    P, M, FP, FM = do.interior_facets(mesh)
    A = interior_matrices(el, Xc[P], Xc[M], Bc[P], FP, FM)
    return do._scatter(np.concatenate([rows[P], rows[M]], axis=1), A, W.node_count)


def exterior_matrix(mesh, W, el, bv, c_out, c_in):
    rows, Xc = do.cells(mesh, W)
    C, F = do.exterior_facets(mesh, "on_boundary")
    return do._scatter(rows[C], exterior_matrices(el, Xc[C], cell_velocities(mesh, bv)[C], F, c_out, c_in),
                       W.node_count)


def operator(mesh, W, el, bv, beta=0.0, alpha=0.0, eta=None, weak_bcs=()):
    """The global matrix of DGTransport(V, b, beta, alpha, eta, weak_bcs) (scipy CSR)."""
    A = cell_matrix(mesh, W, el, bv) + interior_matrix(mesh, W, el, bv) + exterior_matrix(mesh, W, el, bv, 1.0, 0.0)
    if alpha or beta:
        A = A + do.cell_matrix(mesh, W, el, alpha, beta)
    if alpha > 0:
        A = A + do.interior_matrix(mesh, W, el, alpha, eta)
        if weak_bcs:
            A = A + do.exterior_matrix(mesh, W, el, weak_bcs, 0.0, alpha * eta, alpha, alpha)
    return A.tocsr()


def inflow_load(mesh, W, el, bv, g):
    return exterior_matrix(mesh, W, el, bv, 0.0, -1.0) @ g


def outflow_integral(mesh, W, el, bv, q):
    """The outflow flux  sum over boundary faces of  max(b.n, 0)*q*ds, from the traces of q."""
    rows, Xc = do.cells(mesh, W)
    C, F = do.exterior_facets(mesh, "on_boundary")
    bn, Wt, v = _bn(el, Xc[C], cell_velocities(mesh, bv)[C], F)
    return float(np.einsum("fq,fqi,fi->", Wt * np.maximum(bn, 0.0), v, np.asarray(q)[rows[C]]))


def mass_diagonal(mesh, W, el):
    return do.cell_matrix(mesh, W, el, 0.0, 1.0).diagonal()


def ssprk3_step(A, m, q, dt, load=None):
    """One step of the three-stage SSP Runge-Kutta method for M dq/dt = load - A q, M = diag(m)."""
    f = (lambda x: (load - A @ x) / m) if load is not None else (lambda x: -(A @ x) / m)
    q1 = q + dt * f(q)
    q2 = 0.75 * q + 0.25 * (q1 + dt * f(q1))
    return q / 3.0 + 2.0 / 3.0 * (q2 + dt * f(q2))

