"""TEST INFRASTRUCTURE: NumPy oracle of the boundary mass term (FDB_FORM_BOUNDARY_MASS)

    gamma * inner(u, v) * ds(sub_domain)

on Q_p (x) P_p hexahedra with a trilinear (Q1) coordinate field.  A restatement written for the tests, in the
conventions of tests/_coef_oracle.py: dof (ax*N + ay)*N + az with 1-D dof index 0 / 1 at the 0 / 1 end of the
reference interval, vertex (bx*2 + by)*2 + bz, tables B[q][a] on [0, 1].  A facet is local facet f =
2*direction + side of a cell; its face is parametrised by the other two reference axes (s, t) in increasing
order, and the surface measure at a point is |dX/ds x dX/dt| of the cell's trilinear map restricted to the face.

The facet lists are built here from the mesh (the base mesh's exterior facets x all layers for sides 1..4,
layer 0 / nz - 1 of every column for "bottom" / "top"), independently of the facet sets of
firedrake_b200.assemble; the global matrices are scipy CSR, inserted with tests/_coef_oracle.py's CSR helper."""
import numpy as np
import scipy.sparse as sp

import _coef_oracle as co

ALL = (1, 2, 3, 4, "bottom", "top")


def subs_of(sub_domain):
    if isinstance(sub_domain, str) and sub_domain == "on_boundary":
        return ALL
    return tuple(sub_domain) if isinstance(sub_domain, (list, tuple)) else (sub_domain,)


def face_dofs(n, f):
    """The cell-local dofs of facet f's face nodes, (n*n,), in (a along s, b along t) order."""
    d, side = f // 2, f % 2
    a, b = np.divmod(np.arange(n * n), n)
    return {0: (side * n + a) * n + b, 1: (a * n + side) * n + b, 2: (a * n + b) * n + side}[d]


def face_vertices(f):
    """The cell-local vertices of facet f, (4,), in (sa*2 + sb) order."""
    d, side = f // 2, f % 2
    out = []
    for sa in (0, 1):
        for sb in (0, 1):
            bx, by, bz = {0: (side, sa, sb), 1: (sa, side, sb), 2: (sa, sb, side)}[d]
            out.append((bx * 2 + by) * 2 + bz)
    return np.array(out)


def surface_weights(el, Xf, gamma=1.0):
    """Xf (nf, 4, 3) face vertices -> W (nf, Q, Q) = gamma w_s w_t |dX/ds x dX/dt| at the Gauss points."""
    xq, wq = np.asarray(el.xq), np.asarray(el.wq)
    s, t = xq[:, None, None], xq[None, :, None]
    X00, X01, X10, X11 = (Xf[:, k][:, None, None, :] for k in range(4))
    xs = (1 - t) * (X10 - X00) + t * (X11 - X01)
    xt = (1 - s) * (X01 - X00) + s * (X11 - X10)
    return gamma * wq[:, None] * wq[None, :] * np.linalg.norm(np.cross(xs, xt), axis=-1)


def facet_matrices(el, Xf, gamma=1.0):
    """Face element matrices M[i, j] = gamma*inner(phi_j, phi_i)*ds over the face nodes: (nf, n^2, n^2)."""
    B = np.asarray(el.B)
    n = B.shape[1]
    W = surface_weights(el, Xf, gamma)
    M = np.einsum("qa,qc,rb,rd,nqr->nabcd", B, B, B, B, W, optimize=True)
    return M.reshape(-1, n * n, n * n)


def extruded_facets(mesh, V, sub_domain):
    """Facets of ``ds(sub_domain)`` on an extruded mesh: cell dof rows (nf, N^3), vertex rows (nf, 8), local
    facet numbers (nf,)."""
    nz = mesh.nz
    cmap, off = V.cell_node_map.astype(np.int64), np.asarray(V.offset, dtype=np.int64)
    xmap, xoff = mesh.coord_map.astype(np.int64), np.asarray(mesh.coord_offset, dtype=np.int64)
    cols, lays, fs = [], [], []
    cells, local = mesh.exterior_vertical_facets()
    for s in subs_of(sub_domain):
        if s in ("bottom", "top"):
            c = np.arange(mesh.num_base_cells)
            cols.append(c)
            lays.append(np.full(len(c), 0 if s == "bottom" else nz - 1))
            fs.append(np.full(len(c), 4 if s == "bottom" else 5))
        else:
            c = cells[local == s - 1].astype(np.int64)
            cols.append(np.repeat(c, nz))
            lays.append(np.tile(np.arange(nz), len(c)))
            fs.append(np.full(len(c) * nz, s - 1))
    col, lay, f = (np.concatenate(a) for a in (cols, lays, fs))
    return (cmap[col] + off[None, :] * lay[:, None], xmap[col] + xoff[None, :] * lay[:, None], f)


def element_data(el, coords, rows, vrows, facets, gamma=1.0):
    """(face dof indices (nf, n^2), face element matrices (nf, n^2, n^2))."""
    n = el.ndof
    X = coords.reshape(-1, 3)
    i0 = np.empty((len(facets), n * n), dtype=np.int64)
    Xf = np.empty((len(facets), 4, 3))
    for f in range(6):
        sel = facets == f
        i0[sel] = rows[sel][:, face_dofs(n, f)]
        Xf[sel] = X[vrows[sel][:, face_vertices(f)]]
    return i0, facet_matrices(el, Xf, gamma)


def action(el, coords, u, rows, vrows, facets, gamma=1.0, cdim=1):
    i0, M = element_data(el, coords, rows, vrows, facets, gamma)
    uu = u.reshape(-1, cdim)
    y = np.zeros_like(uu)
    np.add.at(y, i0, np.einsum("nij,njc->nic", M, uu[i0]))
    return y.reshape(u.shape)


def matrix(el, coords, nnodes, rows, vrows, facets, gamma=1.0, cdim=1):
    """The global matrix of a_G as scipy CSR over dofs node*cdim + c (components uncoupled)."""
    i0, M = element_data(el, coords, rows, vrows, facets, gamma)
    r = np.repeat(i0, i0.shape[1], axis=1).ravel()
    c = np.tile(i0, (1, i0.shape[1])).ravel()
    A = sp.csr_matrix((M.ravel(), (r, c)), shape=(nnodes, nnodes))
    return sp.kron(A, sp.identity(cdim), format="csr") if cdim > 1 else A


def add_to_csr(rowptr, colidx, vals, el, coords, rows, vrows, facets, gamma=1.0, row_lg=None, col_lg=None):
    """The face element matrices of a scalar space added into a CSR pattern (tests/_coef_oracle.py)."""
    i0, M = element_data(el, coords, rows, vrows, facets, gamma)
    return co.add_to_csr(rowptr, colidx, vals, i0, M, row_lg, col_lg)


def perturb(mesh, amplitude=0.08, seed=0):
    """Move every vertex of the coordinate field by up to ``amplitude`` times the smallest cell size in every
    direction (seeded): boundary faces become non-planar bilinear surfaces and their vertices move in plane
    too (the mesh's own warp vanishes on the box boundary)."""
    h = min(mesh.Lx / mesh.nx_global, mesh.Ly / mesh.ny, mesh.Lz / mesh.nz)
    rng = np.random.default_rng(seed)
    mesh.coordinates += amplitude * h * rng.uniform(-1.0, 1.0, mesh.coordinates.shape)
    return mesh
