"""Synthetic meshes that produce *Firedrake-shaped* arrays (host side, NumPy only).

Mesh generation itself is out of scope for the engine (SURVEY.md section 2.1
row 14): in a real deployment these arrays come from Firedrake's DMPlex layer
(``mesh.coordinates.dat``, ``V.cell_node_map().values_with_halo``,
``V.cell_node_map().offset``).  This module builds the same data layout for the
benchmark and test workloads of SURVEY.md section 8(d), so that the launcher is
exercised with exactly the shapes it would receive behind ``assemble()``:

* extruded meshes store the cell->node map for the BOTTOM cell of each column
  only, plus a per-dof layer ``offset`` (reference
  pyop2/codegen/builder.py:80-128, firedrake/extrusion_utils.py:342-366);
* dofs are numbered contiguously up each column, per base entity, interleaved
  per layer as [dofs on the level | dofs in the layer interior] (reference
  firedrake/extrusion_utils.py:236-252, firedrake/mesh.py:1932-1951);
* the local dof index of a tensor-product element is
  ``(ax * n + ay) * n + az`` with ax, ay, az the 1-D *entity ordered* dof numbers
  (0 = left vertex, 1 = right vertex, 2.. = interior);
* vector spaces are AoS (node major, component fastest).
"""
from __future__ import annotations

import numpy as np

from .fiat_lite import gauss_legendre, gll_points

IntType = np.int32
ScalarType = np.float64

__all__ = ["ExtrudedHexMesh", "ExtrudedFunctionSpace", "ExtrudedDGFunctionSpace", "UnitSquareTriMesh",
           "QuadMesh"]


def _first_touch_rank(keys_per_cell: np.ndarray, nent: int) -> np.ndarray:
    """Number entities in the order a cell-by-cell closure walk first meets
    them (the locality DMPlex reordering gives the reference's numbering)."""
    flat = keys_per_cell.ravel()
    uniq, first = np.unique(flat, return_index=True)
    assert len(uniq) == nent
    order = np.argsort(first, kind="stable")
    rank = np.empty(nent, dtype=np.int64)
    rank[uniq[order]] = np.arange(nent)
    return rank


class ExtrudedHexMesh:
    """nx x ny quadrilateral base mesh on [0,Lx]x[0,Ly] extruded into nz layers.

    Parameters
    ----------
    warp : amplitude of the smooth non-affine warp of SURVEY.md section 8(d):
        ``x += warp * sin(2 pi x) sin(2 pi y) sin(2 pi z)`` applied to every
        coordinate component, so the Jacobian varies inside each cell.
    permute_seed : if not None, base cells are visited in a seeded random order
        (the "unstructured element->dof map" stress case).
    """

    def __init__(self, nx, ny, nz, Lx=1.0, Ly=1.0, Lz=1.0, warp=0.0,
                 permute_seed=None, ix0=0, nx_global=None, ghost_left=False, halo_right=False):
        """``ix0``/``nx_global``/``ghost_left`` describe one slab of a larger
        mesh partitioned along x (firedrake_b200.partition): this mesh holds
        base cells ix0 .. ix0+nx-1 of an nx_global-wide mesh of x-extent Lx;
        with ``ghost_left`` the entities on the slab's left face belong to the
        neighbouring rank: their dof columns are numbered LAST (the ghost tail
        of pyop2/types/set.py:38-52) and the cells touching them come last in
        the cell order (owned-but-not-core cells, pyop2/types/set.py:119-125)."""
        self.nx, self.ny, self.nz = int(nx), int(ny), int(nz)
        self.Lx, self.Ly, self.Lz = float(Lx), float(Ly), float(Lz)
        self.warp = float(warp)
        self.ix0 = int(ix0)
        self.nx_global = int(nx_global) if nx_global is not None else self.nx
        self.ghost_left = bool(ghost_left)
        self.halo_right = bool(halo_right)
        nx, ny = self.nx, self.ny
        ncell = nx * ny
        ix, iy = np.divmod(np.arange(ncell, dtype=np.int64), ny)
        if permute_seed is not None:
            perm = np.random.default_rng(permute_seed).permutation(ncell)
            ix, iy = ix[perm], iy[perm]
        # cell classes: 0 core, 1 owned (touches the left ghost plane), 2 exec halo
        cls = np.zeros(ncell, dtype=np.int64)
        if self.ghost_left:
            cls[ix == 0] = 1
        if self.halo_right:
            cls[ix == nx - 1] = 2
        if self.ghost_left or self.halo_right:
            order = np.argsort(cls, kind="stable")
            ix, iy, cls = ix[order], iy[order], cls[order]
        self.num_core_cells = int((cls == 0).sum())
        self.num_owned_cells = int((cls <= 1).sum())
        self.cell_ix, self.cell_iy = ix, iy
        self.num_base_cells = ncell
        self.layers = self.nz + 1          # node layers, as in ExtrudedSet
        # structured base entity ids
        NV = (nx + 1) * (ny + 1)
        NEy = (nx + 1) * ny                # edges running along y (point x interval)
        NEx = nx * (ny + 1)                # edges running along x (interval x point)
        self._nent = (NV, NEy, NEx, ncell)
        self._ent_base = np.cumsum([0, NV, NEy, NEx])
        clo = np.empty((ncell, 9), dtype=np.int64)
        k = 0
        for ax in (0, 1):
            for ay in (0, 1):
                clo[:, k] = self._vertex(ix + ax, iy + ay); k += 1
        for ax in (0, 1):
            clo[:, k] = self._yedge(ix + ax, iy); k += 1
        for ay in (0, 1):
            clo[:, k] = self._xedge(ix, iy + ay); k += 1
        clo[:, k] = self._face(ix, iy)
        self.closure = clo
        self.num_entities = NV + NEy + NEx + ncell
        self._rank = _first_touch_rank(clo, self.num_entities)
        self.ghost_entities = np.zeros(0, dtype=np.int64)
        if self.ghost_left or self.halo_right:
            # canonical plane order: vertices iy = 0..ny, then y-edges iy = 0..ny-1; the right
            # halo region follows in the order of column_region_entities()
            parts = []
            if self.ghost_left:
                parts.append(self.plane_entities(0))
            if self.halo_right:
                parts.append(self.column_region_entities(nx - 1))
            ghosts = np.concatenate(parts)
            is_ghost = np.zeros(self.num_entities, dtype=bool)
            is_ghost[ghosts] = True
            owned = np.nonzero(~is_ghost)[0]
            owned = owned[np.argsort(self._rank[owned], kind="stable")]
            rank = np.empty(self.num_entities, dtype=np.int64)
            rank[owned] = np.arange(len(owned))
            rank[ghosts] = len(owned) + np.arange(len(ghosts))
            self._rank = rank
            self.ghost_entities = ghosts
        self._fs_cache = {}
        # coordinates: VectorFunctionSpace(Q1 x P1, dim=3)
        V1 = self.function_space(1)
        self.coord_space = V1
        self.coord_map = V1.cell_node_map
        self.coord_offset = V1.offset
        self.coordinates = self._vertex_coordinates(V1)

    # -- structured entity ids -------------------------------------------
    def _vertex(self, i, j):
        return i * (self.ny + 1) + j

    def _yedge(self, i, j):
        return self._ent_base[1] + i * self.ny + j

    def _xedge(self, i, j):
        return self._ent_base[2] + i * (self.ny + 1) + j

    def _face(self, i, j):
        return self._ent_base[3] + i * self.ny + j

    @property
    def num_cells(self):
        return self.num_base_cells * self.nz

    def plane_entities(self, i):
        """Base entities on the plane x-index ``i`` (local), canonical order."""
        return np.concatenate([self._vertex(i, np.arange(self.ny + 1)),
                               self._yedge(i, np.arange(self.ny))]).astype(np.int64)

    def column_region_entities(self, c):
        """Base entities of cell column ``c`` (local) that lie strictly to the right of the plane
        ``c``: x-edges, faces, then the plane ``c + 1`` -- canonical order shared by both sides of
        an exec-halo exchange."""
        return np.concatenate([self._xedge(c, np.arange(self.ny + 1)),
                               self._face(c, np.arange(self.ny)),
                               self.plane_entities(c + 1)]).astype(np.int64)

    def exterior_vertical_facets(self):
        """(base cells, local facet numbers) of the base mesh's exterior facets: local facet
        2*direction + side of the hex (0: x-, 1: x+, 2: y-, 3: y+; 4 / 5 are the bottom / top
        faces, reached through iteration regions).  In a slab of a partitioned mesh only
        facets on the GLOBAL boundary count (mesh.exterior_facets, firedrake/mesh.py:1211-1260)."""
        gx = self.cell_ix + self.ix0
        sel = [(gx == 0, 0), (gx == self.nx_global - 1, 1), (self.cell_iy == 0, 2),
               (self.cell_iy == self.ny - 1, 3)]
        cells = np.concatenate([np.nonzero(m)[0] for m, _ in sel]).astype(IntType)
        local = np.concatenate([np.full(int(m.sum()), k, dtype=np.uint32) for m, k in sel])
        return cells, local

    def interior_vertical_facets(self):
        """(cells '+', cells '-', local facet pairs (nfacets, 2)) of the base mesh's interior
        facets within this (unpartitioned) mesh: x-normal facets carry local facets (1, 0),
        y-normal ones (3, 2) (mesh.interior_facets, firedrake/mesh.py:1262-1300)."""
        col = np.full((self.nx, self.ny), -1, dtype=np.int64)
        col[self.cell_ix, self.cell_iy] = np.arange(self.num_base_cells)
        xp, xm = col[:-1, :].ravel(), col[1:, :].ravel()
        yp, ym = col[:, :-1].ravel(), col[:, 1:].ravel()
        local = np.concatenate([np.tile([1, 0], (len(xp), 1)), np.tile([3, 2], (len(yp), 1))]).astype(np.uint32)
        return (np.concatenate([xp, yp]).astype(IntType), np.concatenate([xm, ym]).astype(IntType), local)

    def function_space(self, degree: int) -> "ExtrudedFunctionSpace":
        if degree not in self._fs_cache:
            self._fs_cache[degree] = ExtrudedFunctionSpace(self, degree)
        return self._fs_cache[degree]

    def dg_function_space(self, degree: int) -> "ExtrudedDGFunctionSpace":
        """Scalar DQ_p (p = 1..4) with Firedrake's default "spectral" variant: Gauss-Legendre nodes."""
        cache = self.__dict__.setdefault("_dg_fs_cache", {})
        if degree not in cache:
            cache[degree] = ExtrudedDGFunctionSpace(self, degree)
        return cache[degree]

    def hdiv_function_space(self, degree: int) -> "ExtrudedHDivFunctionSpace":
        """NCF_k (k = 2..4), Firedrake's H(div) element on hexahedra in its default "spectral" variant."""
        cache = self.__dict__.setdefault("_hdiv_fs_cache", {})
        if degree not in cache:
            cache[degree] = ExtrudedHDivFunctionSpace(self, degree)
        return cache[degree]

    def trace_function_space(self, degree: int) -> "ExtrudedTraceFunctionSpace":
        """Firedrake's "HDiv Trace" space of degree ``degree`` = k - 1 (1..3): Q_{k-1} on every face, the Lagrange
        multiplier of the hybridised NCF_k x DQ_{k-1} mixed Poisson problem."""
        cache = self.__dict__.setdefault("_trace_fs_cache", {})
        if degree not in cache:
            cache[degree] = ExtrudedTraceFunctionSpace(self, degree)
        return cache[degree]

    def _apply_warp(self, X):
        if self.warp == 0.0:
            return X
        s = self.warp * (np.sin(2 * np.pi * X[:, 0] / self.Lx)
                         * np.sin(2 * np.pi * X[:, 1] / self.Ly)
                         * np.sin(2 * np.pi * X[:, 2] / self.Lz))
        return X + s[:, None]

    def _vertex_coordinates(self, V1):
        nx, ny, nz = self.nx, self.ny, self.nz
        NV = self._nent[0]
        vid = np.arange(NV, dtype=np.int64)
        vi, vj = np.divmod(vid, ny + 1)
        start = V1._ent_start[vid]                       # column starts, stride 1
        X = np.empty((V1.node_count, 3), dtype=ScalarType)
        lay = np.arange(nz + 1, dtype=np.int64)
        idx = (start[:, None] + lay[None, :]).ravel()
        X[idx, 0] = np.repeat((vi + self.ix0) * (self.Lx / self.nx_global), nz + 1)
        X[idx, 1] = np.repeat(vj * (self.Ly / ny), nz + 1)
        X[idx, 2] = np.tile(lay * (self.Lz / nz), NV)
        return self._apply_warp(X)


class ExtrudedFunctionSpace:
    """Scalar Q_p (x) P_p space on an :class:`ExtrudedHexMesh` (GLL nodes)."""

    def __init__(self, mesh: ExtrudedHexMesh, degree: int):
        self.mesh = mesh
        self.degree = p = int(degree)
        n = p + 1
        self.n = n
        self.arity = n ** 3
        nz = mesh.nz
        NV, NEy, NEx, NF = mesh._nent
        nb_kind = np.array([1, p - 1, p - 1, (p - 1) ** 2], dtype=np.int64)
        nb = np.repeat(nb_kind, [NV, NEy, NEx, NF])      # base dofs per entity
        colsize = nb * (p * nz + 1)
        # columns laid out in first-touch order
        order = np.argsort(mesh._rank, kind="stable")
        start_sorted = np.concatenate([[0], np.cumsum(colsize[order])[:-1]])
        ent_start = np.empty(mesh.num_entities, dtype=np.int64)
        ent_start[order] = start_sorted
        self._ent_start = ent_start
        self._ent_nb = nb
        self._ent_colsize = colsize
        self.node_count = int(colsize.sum())
        self.ghost_node_count = int(colsize[mesh.ghost_entities].sum())
        self.owned_node_count = self.node_count - self.ghost_node_count
        if self.node_count >= 2 ** 31:
            raise ValueError("node count exceeds int32 IntType")
        ix, iy = mesh.cell_ix, mesh.cell_iy
        cmap = np.empty((mesh.num_base_cells, self.arity), dtype=IntType)
        off = np.empty(self.arity, dtype=IntType)
        for ax in range(n):
            for ay in range(n):
                if ax < 2 and ay < 2:
                    ent = mesh._vertex(ix + ax, iy + ay); nbe = 1; eb = 0
                elif ax < 2:
                    ent = mesh._yedge(ix + ax, iy); nbe = p - 1; eb = ay - 2
                elif ay < 2:
                    ent = mesh._xedge(ix, iy + ay); nbe = p - 1; eb = ax - 2
                else:
                    ent = mesh._face(ix, iy); nbe = (p - 1) ** 2
                    eb = (ax - 2) * (p - 1) + (ay - 2)
                st = ent_start[ent]
                for v in range(n):
                    if v == 0:
                        pos = eb
                    elif v == 1:
                        pos = nbe * p + eb
                    else:
                        pos = nbe + eb * (p - 1) + (v - 2)
                    loc = (ax * n + ay) * n + v
                    cmap[:, loc] = st + pos
                    off[loc] = nbe * p
        self.cell_node_map = cmap
        self.offset = off

    # ------------------------------------------------------------------
    def full_cell_node_list(self):
        """(num_cells, arity) map with the layer loop expanded: row
        ``c*nz + l`` is column c, layer l (small meshes / tests)."""
        nz = self.mesh.nz
        lay = np.arange(nz, dtype=np.int64)
        full = (self.cell_node_map[:, None, :].astype(np.int64)
                + lay[None, :, None] * self.offset[None, None, :])
        return full.reshape(-1, self.arity).astype(IntType)

    def dof_coordinates(self):
        """Physical positions of all nodes, (node_count, 3).  The geometry is
        Q1: a node's position is the trilinear image of its reference position.
        Small meshes only (allocates arity x num_cells)."""
        mesh = self.mesh
        n = self.n
        ref1d = gll_points(self.degree)
        a2pos = np.array([0, n - 1] + list(range(1, n - 1)))
        xi = ref1d[a2pos]                                  # by dof number
        full = self.full_cell_node_list().astype(np.int64)
        cfull = mesh.coord_space.full_cell_node_list().astype(np.int64)
        XV = mesh.coordinates[cfull]                       # (ncell, 8, 3)
        out = np.empty((self.node_count, 3), dtype=ScalarType)
        for ax in range(n):
            for ay in range(n):
                for az in range(n):
                    pt = np.zeros((full.shape[0], 3))
                    for bx in (0, 1):
                        for by in (0, 1):
                            for bz in (0, 1):
                                wgt = ((xi[ax] if bx else 1 - xi[ax])
                                       * (xi[ay] if by else 1 - xi[ay])
                                       * (xi[az] if bz else 1 - xi[az]))
                                pt += wgt * XV[:, (bx * 2 + by) * 2 + bz, :]
                    out[full[:, (ax * n + ay) * n + az]] = pt
        return out

    def plane_nodes(self, i):
        """All nodes on the plane x-index ``i`` in canonical order (entity by
        entity, bottom to top): the send/recv lists of the slab halo."""
        ents = self.mesh.plane_entities(i)
        st, sz = self._ent_start[ents], self._ent_colsize[ents]
        return np.concatenate([np.arange(a, a + b) for a, b in zip(st, sz)]).astype(IntType)

    def column_region_nodes(self, c):
        """All nodes of the base entities ``mesh.column_region_entities(c)`` (entity by entity,
        bottom to top): send/recv list of the exec-halo region of cell column ``c``."""
        ents = self.mesh.column_region_entities(c)
        st, sz = self._ent_start[ents], self._ent_colsize[ents]
        return np.concatenate([np.arange(a, a + b) for a, b in zip(st, sz)]).astype(IntType)

    def dof_lattice(self):
        """Integer position of every node on the global p-refined lattice,
        (node_count, 3): identifies dofs across partitions (tests)."""
        mesh, n, p = self.mesh, self.n, self.degree
        a2pos = np.array([0, n - 1] + list(range(1, n - 1)))
        full = self.full_cell_node_list().astype(np.int64)
        nz = mesh.nz
        cix = np.repeat(mesh.cell_ix + mesh.ix0, nz)
        ciy = np.repeat(mesh.cell_iy, nz)
        ciz = np.tile(np.arange(nz), mesh.num_base_cells)
        out = np.empty((self.node_count, 3), dtype=np.int64)
        for ax in range(n):
            for ay in range(n):
                for az in range(n):
                    idx = full[:, (ax * n + ay) * n + az]
                    out[idx, 0] = cix * p + a2pos[ax]
                    out[idx, 1] = ciy * p + a2pos[ay]
                    out[idx, 2] = ciz * p + a2pos[az]
        return out

    def boundary_nodes(self, sub_domain):
        """Node indices of a Dirichlet boundary (reference
        firedrake/functionspacedata.py:272-300 for "bottom"/"top"; integer ids
        1..4 = x==0, x==Lx, y==0, y==Ly as in firedrake/utility_meshes.py)."""
        mesh = self.mesh
        p, nz = self.degree, mesh.nz
        st, nb = self._ent_start, self._ent_nb
        if sub_domain in ("bottom", "top"):
            base = st if sub_domain == "bottom" else st + nb * p * nz
            reps = np.repeat(base, nb)
            within = np.concatenate([np.arange(k) for k in nb]) if len(nb) else np.array([], dtype=np.int64)
            return np.sort(reps + within).astype(IntType)
        nx, ny = mesh.nx, mesh.ny
        if sub_domain == 1:
            ents = [mesh._vertex(0, np.arange(ny + 1)), mesh._yedge(0, np.arange(ny))]
        elif sub_domain == 2:
            ents = [mesh._vertex(nx, np.arange(ny + 1)), mesh._yedge(nx, np.arange(ny))]
        elif sub_domain == 3:
            ents = [mesh._vertex(np.arange(nx + 1), 0), mesh._xedge(np.arange(nx), 0)]
        elif sub_domain == 4:
            ents = [mesh._vertex(np.arange(nx + 1), ny), mesh._xedge(np.arange(nx), ny)]
        else:
            raise ValueError(f"unknown sub_domain {sub_domain!r}")
        ents = np.concatenate(ents)
        size = nb[ents] * (p * nz + 1)
        idx = np.concatenate([np.arange(s, s + k) for s, k in zip(st[ents], size)])
        return np.sort(idx).astype(IntType)


class ExtrudedDGFunctionSpace:
    """Scalar DQ_p = dQ_p (x) dP_p space on an :class:`ExtrudedHexMesh` with Gauss-Legendre nodes (the default
    "spectral" variant of a DG element, SURVEY.md section 7).  Every dof belongs to one cell: the numbering is
    cell-major, base column c (in the mesh's cell order) holds the ``nz * (p+1)^3`` dofs ``c * nz * (p+1)^3 ..``
    layer by layer, so the layer offset of every local dof is ``(p+1)^3``.  The local index is ``(ax*n + ay)*n +
    az`` with the 1-D indices in ascending node position."""

    def __init__(self, mesh: ExtrudedHexMesh, degree: int):
        p = int(degree)
        if not 1 <= p <= 4:
            raise ValueError(f"DQ degree {p} outside 1..4")
        self.mesh = mesh
        self.degree = p
        self.n = n = p + 1
        self.arity = n ** 3
        nz = mesh.nz
        self.node_count = mesh.num_base_cells * nz * self.arity
        self.owned_node_count = self.node_count
        self.ghost_node_count = 0
        if self.node_count >= 2 ** 31:
            raise ValueError("node count exceeds int32 IntType")
        self.cell_node_map = (np.arange(mesh.num_base_cells, dtype=np.int64)[:, None] * (nz * self.arity)
                              + np.arange(self.arity)[None, :]).astype(IntType)
        self.offset = np.full(self.arity, self.arity, dtype=IntType)

    def full_cell_node_list(self):
        """(num_cells, arity) map with the layer loop expanded: row ``c*nz + l`` is column c, layer l."""
        nz = self.mesh.nz
        lay = np.arange(nz, dtype=np.int64)
        full = (self.cell_node_map[:, None, :].astype(np.int64)
                + lay[None, :, None] * self.offset[None, None, :])
        return full.reshape(-1, self.arity).astype(IntType)

    def dof_coordinates(self):
        """Physical positions of all dofs, (node_count, 3): the trilinear image of the Gauss-Legendre points."""
        mesh, n = self.mesh, self.n
        xi, _ = gauss_legendre(n)
        full = self.full_cell_node_list().astype(np.int64)
        XV = mesh.coordinates[mesh.coord_space.full_cell_node_list().astype(np.int64)]     # (ncell, 8, 3)
        out = np.empty((self.node_count, 3), dtype=ScalarType)
        for ax in range(n):
            for ay in range(n):
                for az in range(n):
                    pt = np.zeros((full.shape[0], 3))
                    for v in range(8):
                        bx, by, bz = (v >> 2) & 1, (v >> 1) & 1, v & 1
                        pt += ((xi[ax] if bx else 1 - xi[ax]) * (xi[ay] if by else 1 - xi[ay])
                               * (xi[az] if bz else 1 - xi[az])) * XV[:, v, :]
                    out[full[:, (ax * n + ay) * n + az]] = pt
        return out

    def boundary_nodes(self, sub_domain):
        raise ValueError("a DQ space has no boundary nodes: every dof is interior to its cell.  Impose Dirichlet "
                         "conditions weakly (InteriorPenalty's weak_bcs and nitsche_load)")


class ExtrudedHDivFunctionSpace:
    """NCF_k (k = 2..4) on an :class:`ExtrudedHexMesh`: Firedrake's H(div) element on hexahedra in its default
    "spectral" variant.  Component d of the reference field (the contravariant Piola pull-back sigma^ = det J J^-1
    sigma) is CG_k on GLL nodes along axis d times DG_{k-1} on Gauss-Legendre nodes along the other two axes; a dof
    is the value of one component at its node.

    Local numbering is component-major: block d holds n0*n1*n2 dofs (n_d = k+1, the others k), index
    ``(i0*n1 + i1)*n2 + i2`` with the CG index in FIAT entity order (0 at 0, 1 at 1, then the interior nodes) and
    the GL indices in ascending position.  Arity 3 k^2 (k+1).

    Global numbering follows :class:`ExtrudedFunctionSpace`'s entity columns in first-touch order: an x-normal
    vertical face belongs to its base y-edge, a y-normal one to its base x-edge (``nz * k^2`` dofs per column), and a
    base face holds its horizontal faces and the cell interiors as ``[hface_0, interior_0, hface_1, ..., hface_nz]``
    (k^2 per face, 3 (k-1) k^2 per interior).  Every local dof has a constant layer offset.  All cells have the
    reference orientation of the structured mesh, so two cells sharing a face parametrise it alike and see the same
    sigma^.n^: no sign flips are needed."""

    def __init__(self, mesh: ExtrudedHexMesh, degree: int):
        k = int(degree)
        if not 2 <= k <= 4:
            raise ValueError(f"NCF degree {k} outside 2..4")
        self.mesh = mesh
        self.degree = k
        self.arity = 3 * k * k * (k + 1)
        nz = mesh.nz
        NV, NEy, NEx, NF = mesh._nent
        k2 = k * k
        self.layer_stride = (3 * k - 2) * k2                       # hface + interior per layer of a base face
        colsize = np.concatenate([np.zeros(NV, dtype=np.int64), np.full(NEy + NEx, nz * k2, dtype=np.int64),
                                  np.full(NF, nz * self.layer_stride + k2, dtype=np.int64)])
        order = np.argsort(mesh._rank, kind="stable")
        start_sorted = np.concatenate([[0], np.cumsum(colsize[order])[:-1]])
        ent_start = np.empty(mesh.num_entities, dtype=np.int64)
        ent_start[order] = start_sorted
        self._ent_start, self._ent_colsize = ent_start, colsize
        self.node_count = int(colsize.sum())
        self.owned_node_count, self.ghost_node_count = self.node_count, 0
        if self.node_count >= 2 ** 31:
            raise ValueError("node count exceeds int32 IntType")
        ix, iy = mesh.cell_ix, mesh.cell_iy
        cmap = np.empty((mesh.num_base_cells, self.arity), dtype=np.int64)
        off = np.empty(self.arity, dtype=IntType)
        face = ent_start[mesh._face(ix, iy)]
        loc = 0
        for d in range(3):
            dims = [k + 1 if e == d else k for e in range(3)]
            for i0 in range(dims[0]):
                for i1 in range(dims[1]):
                    for i2 in range(dims[2]):
                        idx = (i0, i1, i2)
                        a = idx[d]
                        t0, t1 = [idx[e] for e in range(3) if e != d]   # the two GL indices, axis order
                        within = t0 * k + t1
                        if a >= 2:
                            cmap[:, loc] = face + k2 + (d * (k - 1) + a - 2) * k2 + within
                            off[loc] = self.layer_stride
                        elif d == 2:
                            cmap[:, loc] = face + a * self.layer_stride + within
                            off[loc] = self.layer_stride
                        else:
                            ent = mesh._yedge(ix + a, iy) if d == 0 else mesh._xedge(ix, iy + a)
                            cmap[:, loc] = ent_start[ent] + within
                            off[loc] = k2
                        loc += 1
        self.cell_node_map = cmap.astype(IntType)
        self.offset = off

    def full_cell_node_list(self):
        """(num_cells, arity) map with the layer loop expanded: row ``c*nz + l`` is column c, layer l."""
        nz = self.mesh.nz
        lay = np.arange(nz, dtype=np.int64)
        full = (self.cell_node_map[:, None, :].astype(np.int64)
                + lay[None, :, None] * self.offset[None, None, :])
        return full.reshape(-1, self.arity).astype(IntType)

    def boundary_nodes(self, sub_domain):
        """The face dofs on a boundary: sub-domains 1..4 (x == 0, x == Lx, y == 0, y == Ly) and "bottom" / "top".
        A DirichletBC on them is the flux condition sigma.n = 0."""
        mesh, k2 = self.mesh, self.degree ** 2
        nx, ny = mesh.nx, mesh.ny
        if sub_domain in ("bottom", "top"):
            st = self._ent_start[mesh._face(mesh.cell_ix, mesh.cell_iy)]
            if sub_domain == "top":
                st = st + mesh.nz * self.layer_stride
            return np.sort((st[:, None] + np.arange(k2)[None, :]).ravel()).astype(IntType)
        ents = {1: lambda: mesh._yedge(0, np.arange(ny)), 2: lambda: mesh._yedge(nx, np.arange(ny)),
                3: lambda: mesh._xedge(np.arange(nx), 0), 4: lambda: mesh._xedge(np.arange(nx), ny)}
        if sub_domain not in ents:
            raise ValueError(f"unknown sub_domain {sub_domain!r}")
        e = np.atleast_1d(ents[sub_domain]())
        st, sz = self._ent_start[e], self._ent_colsize[e]
        return np.sort(np.concatenate([np.arange(a, a + b) for a, b in zip(st, sz)])).astype(IntType)


class ExtrudedTraceFunctionSpace:
    """Firedrake's "HDiv Trace" space of degree k - 1 (k = 2..4) on an :class:`ExtrudedHexMesh`: Q_{k-1} on every
    face of the mesh, its k^2 dofs the values at the k x k Gauss-Legendre points of the face -- the points of the NCF_k
    face dofs of that face.

    Local numbering (arity 6k^2): face ``2d + s`` (normal axis d, side s), then ``t0 * k + t1`` with the two GL
    indices in axis order: exactly the order of the NCF_k face dofs of component d at CG index s
    (:class:`ExtrudedHDivFunctionSpace`).  Global numbering: the NCF_k entity columns with the cell interiors removed,
    in the same first-touch order: a base edge holds its ``nz`` vertical faces (``nz * k^2`` dofs), a base face its
    ``nz + 1`` horizontal faces (``(nz + 1) * k^2``).  Every local dof has the layer offset k^2."""

    def __init__(self, mesh: ExtrudedHexMesh, degree: int):
        p = int(degree)
        if not 1 <= p <= 3:
            raise ValueError(f"HDiv Trace degree {p} outside 1..3")
        self.mesh = mesh
        self.degree = p
        self.k = k = p + 1
        k2 = k * k
        self.arity = 6 * k2
        nz = mesh.nz
        NV, NEy, NEx, NF = mesh._nent
        colsize = np.concatenate([np.zeros(NV, dtype=np.int64), np.full(NEy + NEx, nz * k2, dtype=np.int64),
                                  np.full(NF, (nz + 1) * k2, dtype=np.int64)])
        order = np.argsort(mesh._rank, kind="stable")
        start_sorted = np.concatenate([[0], np.cumsum(colsize[order])[:-1]])
        ent_start = np.empty(mesh.num_entities, dtype=np.int64)
        ent_start[order] = start_sorted
        self._ent_start, self._ent_colsize = ent_start, colsize
        self.node_count = int(colsize.sum())
        self.owned_node_count, self.ghost_node_count = self.node_count, 0
        if self.node_count >= 2 ** 31:
            raise ValueError("node count exceeds int32 IntType")
        ix, iy = mesh.cell_ix, mesh.cell_iy
        within = np.arange(k2, dtype=np.int64)
        starts = [ent_start[mesh._yedge(ix, iy)], ent_start[mesh._yedge(ix + 1, iy)],
                  ent_start[mesh._xedge(ix, iy)], ent_start[mesh._xedge(ix, iy + 1)],
                  ent_start[mesh._face(ix, iy)], ent_start[mesh._face(ix, iy)] + k2]
        self.cell_node_map = np.concatenate([st[:, None] + within[None, :] for st in starts],
                                            axis=1).astype(IntType)
        self.offset = np.full(self.arity, k2, dtype=IntType)

    def full_cell_node_list(self):
        """(num_cells, arity) map with the layer loop expanded: row ``c*nz + l`` is column c, layer l."""
        nz = self.mesh.nz
        lay = np.arange(nz, dtype=np.int64)
        full = (self.cell_node_map[:, None, :].astype(np.int64)
                + lay[None, :, None] * self.offset[None, None, :])
        return full.reshape(-1, self.arity).astype(IntType)

    def boundary_nodes(self, sub_domain):
        """The trace dofs on a boundary: sub-domains 1..4 (x == 0, x == Lx, y == 0, y == Ly) and "bottom" / "top",
        the names of the NCF space's."""
        mesh, k2 = self.mesh, self.k ** 2
        nx, ny = mesh.nx, mesh.ny
        if sub_domain in ("bottom", "top"):
            st = self._ent_start[mesh._face(mesh.cell_ix, mesh.cell_iy)]
            if sub_domain == "top":
                st = st + mesh.nz * k2
            return np.sort((st[:, None] + np.arange(k2)[None, :]).ravel()).astype(IntType)
        ents = {1: lambda: mesh._yedge(0, np.arange(ny)), 2: lambda: mesh._yedge(nx, np.arange(ny)),
                3: lambda: mesh._xedge(np.arange(nx), 0), 4: lambda: mesh._xedge(np.arange(nx), ny)}
        if sub_domain not in ents:
            raise ValueError(f"unknown sub_domain {sub_domain!r}")
        e = np.atleast_1d(ents[sub_domain]())
        st, sz = self._ent_start[e], self._ent_colsize[e]
        return np.sort(np.concatenate([np.arange(a, a + b) for a, b in zip(st, sz)])).astype(IntType)


class UnitSquareTriMesh:
    """``UnitSquareMesh(nx, ny)``: each cell of the nx x ny grid split with the
    "left" diagonal (reference firedrake/utility_meshes.py:599-600, 802-812).
    P1 only: the cell->node map is the vertex list, (ncell, 3)."""

    def __init__(self, nx, ny, L=1.0):
        self.nx, self.ny = nx, ny
        xs = np.linspace(0.0, L, nx + 1)
        ys = np.linspace(0.0, L, ny + 1)
        X, Y = np.meshgrid(xs, ys, indexing="ij")
        self.coordinates = np.stack([X.ravel(), Y.ravel()], axis=1).astype(ScalarType)
        i, j = np.meshgrid(np.arange(nx), np.arange(ny), indexing="ij")
        i, j = i.ravel(), j.ravel()
        v = lambda a, b: a * (ny + 1) + b
        v00, v10, v01, v11 = v(i, j), v(i + 1, j), v(i, j + 1), v(i + 1, j + 1)
        # "left" diagonal joins (i, j+1) and (i+1, j)
        t0 = np.stack([v00, v10, v01], axis=1)
        t1 = np.stack([v10, v11, v01], axis=1)
        self.cell_node_map = np.concatenate([t0, t1], axis=0).astype(IntType)
        self.num_cells = self.cell_node_map.shape[0]
        self.node_count = self.coordinates.shape[0]

    def boundary_nodes(self):
        X = self.coordinates
        on = (np.isclose(X[:, 0], 0) | np.isclose(X[:, 0], X[:, 0].max())
              | np.isclose(X[:, 1], 0) | np.isclose(X[:, 1], X[:, 1].max()))
        return np.nonzero(on)[0].astype(IntType)


class QuadMesh:
    """nx x ny quadrilateral mesh (non-extruded) with the facet data the DG
    advection demo needs (reference demos/DG_advection/DG_advection.py.rst):

    * ``coord_map`` (ncell, 4): Q1 vertices, local index ax*2+ay
    * DQ1 space: 4 dofs per cell, numbered cell*4 + (ax*2+ay)
    * interior facets: ``int_facet_cells`` (nf, 2) = [cell+, cell-],
      ``int_facet_local`` (nf, 2) local facet numbers; exterior likewise.
      Local facet numbering of the reference quad: 0: x==0, 1: x==1, 2: y==0,
      3: y==1 (edges of FInAT dimension (0,1) first; reference
      firedrake/cython/dmcommon.pyx:1496-1499).
    * ``nbr`` / ``nbr_facet`` (ncell, 4): neighbour cell across each local facet
      (-1 on the domain boundary) and the neighbour's local facet number -- the
      cell-centred view used by the fused owner-computes kernel.

    Slab of a larger mesh (``ix0``, ``nx_global``, ``ghost_left/right``): the
    local mesh holds the owned columns ix0 .. ix0+nx-1 plus one ghost column of
    cells on each interior side; owned cells are numbered first, ghost cells
    last (their DQ dofs form the ghost tail of the Dat).  Facet lists are only
    built for an unpartitioned mesh.
    """

    def __init__(self, nx, ny, Lx=1.0, Ly=1.0, ix0=0, nx_global=None, ghost_left=False,
                 ghost_right=False):
        self.nx, self.ny = nx, ny
        nxg = nx if nx_global is None else nx_global
        gl, gr = int(ghost_left), int(ghost_right)
        nxl = nx + gl + gr                                   # local columns incl. ghosts
        xs = (np.arange(nxl + 1) + ix0 - gl) * (Lx / nxg)
        ys = np.linspace(0.0, Ly, ny + 1)
        X, Y = np.meshgrid(xs, ys, indexing="ij")
        self.coordinates = np.stack([X.ravel(), Y.ravel()], axis=1).astype(ScalarType)
        # local cell ids: owned (columns gl .. gl+nx-1) first, then left ghost, right ghost
        col_order = list(range(gl, gl + nx)) + ([0] if gl else []) + ([nxl - 1] if gr else [])
        cid_of = -np.ones((nxl, ny), dtype=np.int64)
        k = 0
        for c in col_order:
            cid_of[c, :] = k + np.arange(ny)
            k += ny
        ncell = nxl * ny
        ii = np.empty(ncell, dtype=np.int64)
        jj = np.empty(ncell, dtype=np.int64)
        for c in range(nxl):
            ii[cid_of[c, :]] = c
            jj[cid_of[c, :]] = np.arange(ny)
        v = lambda a, b: a * (ny + 1) + b
        self.coord_map = np.stack([v(ii, jj), v(ii, jj + 1), v(ii + 1, jj), v(ii + 1, jj + 1)],
                                  axis=1).astype(IntType)
        self.num_cells = ncell
        self.num_owned_cells = nx * ny
        self.node_count = self.coordinates.shape[0]
        self.dg1_map = (np.arange(ncell, dtype=np.int64)[:, None] * 4
                        + np.arange(4)[None, :]).astype(IntType)
        # neighbour tables (global domain boundary: -1)
        nbr = -np.ones((ncell, 4), dtype=np.int64)
        gi = ii + ix0 - gl                                   # global column of each local cell
        for f, (di, dj) in enumerate([(-1, 0), (1, 0), (0, -1), (0, 1)]):
            ni, nj = ii + di, jj + dj
            ok = (ni >= 0) & (ni < nxl) & (nj >= 0) & (nj < ny)
            nbr[ok, f] = cid_of[ni[ok], nj[ok]]
        self.nbr = nbr.astype(IntType)
        self.nbr_facet = np.tile(np.array([1, 0, 3, 2], dtype=np.uint32), (ncell, 1))
        self.cell_global_column = gi
        self.ghost_cells_left = cid_of[0, :].copy() if gl else np.zeros(0, dtype=np.int64)
        self.ghost_cells_right = cid_of[nxl - 1, :].copy() if gr else np.zeros(0, dtype=np.int64)
        self.first_owned_column = cid_of[gl, :].copy()
        self.last_owned_column = cid_of[gl + nx - 1, :].copy()
        if gl or gr:
            return
        i, j = ii, jj
        cid = lambda a, b: a * ny + b
        # interior facets normal to x (between (i,j) and (i+1,j)): '+' local 1, '-' local 0
        a, b = np.meshgrid(np.arange(nx - 1), np.arange(ny), indexing="ij")
        fx_cells = np.stack([cid(a, b).ravel(), cid(a + 1, b).ravel()], axis=1)
        fx_loc = np.tile(np.array([1, 0]), (fx_cells.shape[0], 1))
        a, b = np.meshgrid(np.arange(nx), np.arange(ny - 1), indexing="ij")
        fy_cells = np.stack([cid(a, b).ravel(), cid(a, b + 1).ravel()], axis=1)
        fy_loc = np.tile(np.array([3, 2]), (fy_cells.shape[0], 1))
        self.int_facet_cells = np.concatenate([fx_cells, fy_cells]).astype(IntType)
        self.int_facet_local = np.concatenate([fx_loc, fy_loc]).astype(np.uint32)
        ext_cells, ext_loc = [], []
        b = np.arange(ny)
        ext_cells += [cid(0, b), cid(nx - 1, b)]
        ext_loc += [np.full(ny, 0), np.full(ny, 1)]
        a = np.arange(nx)
        ext_cells += [cid(a, 0), cid(a, ny - 1)]
        ext_loc += [np.full(nx, 2), np.full(nx, 3)]
        self.ext_facet_cells = np.concatenate(ext_cells).astype(IntType)
        self.ext_facet_local = np.concatenate(ext_loc).astype(np.uint32)
