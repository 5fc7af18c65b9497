"""Additive Schwarz patch smoother on the device (SURVEY.md section 8f row f4).

Mirrors the pieces of the reference a patch preconditioner is made of:

* ``vertex_star_patches`` -- the dof sets ``firedrake.ASMStarPC`` builds with
  ``construct_dim = 0`` (firedrake/preconditioners/asm.py:150-230): for every mesh vertex, the dofs
  of all entities in its OPEN star (the vertex, and every edge / face / cell that contains it);
* ``PatchASM`` -- TinyASM's ``BlockJacobi`` (tinyasm/tinyasm.cpp:27-120): ``update`` extracts the
  dense patch blocks of the assembled operator and inverts them, ``apply`` adds
  ``inv(A[d_p, d_p]) b[d_p]`` into ``x[d_p]`` for every patch.  Both run in ``csrc/patch_asm.cu``.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib, op2


def vertex_star_patches(V, exclude=()):
    """(patch_ptr, patch_dofs) of the vertex-star patches of the scalar space ``V.V`` (an
    ``ExtrudedFunctionSpace``): on the p-refined lattice a dof belongs to the open star of the
    vertex at lattice position ``p * (i, j, k)`` iff it is closer than ``p`` to it in every
    direction.  ``exclude``: node indices to leave out of every patch (Dirichlet rows).
    Small / medium meshes (uses ``dof_lattice``)."""
    fs = V.V
    p = fs.degree
    lat = fs.dof_lattice()
    lo, hi = lat.min(axis=0), lat.max(axis=0)
    skip = np.zeros(fs.node_count, dtype=bool)
    skip[np.asarray(exclude, dtype=np.int64)] = True
    ptr, dofs = [0], []
    for i in range(lo[0], hi[0] + 1, p):
        in_i = np.abs(lat[:, 0] - i) < p
        for j in range(lo[1], hi[1] + 1, p):
            in_ij = in_i & (np.abs(lat[:, 1] - j) < p)
            for k in range(lo[2], hi[2] + 1, p):
                sel = np.nonzero(in_ij & (np.abs(lat[:, 2] - k) < p) & ~skip)[0]
                if len(sel):
                    dofs.append(sel)
                    ptr.append(ptr[-1] + len(sel))
    return (np.asarray(ptr, dtype=np.int64),
            np.concatenate(dofs).astype(np.int32) if dofs else np.zeros(0, dtype=np.int32))


class PatchASM:
    """``PatchASM(mat, patch_ptr, patch_dofs)``: additive Schwarz over dof patches of the assembled
    matrix ``mat`` (an ``op2.Mat``).  ``update()`` after (re)assembly, ``apply(b, x)`` computes
    ``x = sum_p R_p^T inv(R_p A R_p^T) R_p b`` on device-resident Dats."""

    def __init__(self, mat: op2.Mat, patch_ptr, patch_dofs):
        self.mat = mat
        self.ptr = np.ascontiguousarray(patch_ptr, dtype=np.int64)
        self.dofs = np.ascontiguousarray(patch_dofs, dtype=np.int32)
        h = C.c_void_p()
        _lib.check(_lib.lib().fdb_asm_create(len(self.ptr) - 1, self.ptr.ctypes.data, self.dofs.ctypes.data,
                                             C.byref(h)), "fdb_asm_create")
        self._handle = h
        self.update()

    def update(self):
        ns = C.c_int()
        _lib.check(_lib.lib().fdb_asm_update(self._handle, self.mat.handle, C.byref(ns)), "fdb_asm_update")
        if ns.value:
            raise np.linalg.LinAlgError(f"{ns.value} singular patch block(s)")

    def apply(self, b: op2.Dat, x: op2.Dat):
        x.zero()
        _lib.check(_lib.lib().fdb_asm_apply(self._handle, b.device_ptr, x.device_ptr), "fdb_asm_apply")
        x._device_written()
        return x

    def inverse_blocks(self):
        """The inverted patch blocks, one (n_p, n_p) array per patch (tests)."""
        n = np.diff(self.ptr)
        out = np.empty(int((n * n).sum()))
        _lib.check(_lib.lib().fdb_asm_get_blocks(self._handle, out.ctypes.data), "fdb_asm_get_blocks")
        off = np.concatenate([[0], np.cumsum(n * n)])
        return [out[off[k]:off[k + 1]].reshape(n[k], n[k]) for k in range(len(n))]

    def __del__(self):
        try:
            if self._handle is not None and _lib._initialised is not None:
                _lib._lib.fdb_asm_destroy(self._handle)
        except Exception:
            pass


# ------------------------------------------------------------------ fast-diagonalisation vertex stars
# Dirichlet sub-domains at the low and high end of each reference direction
_FACES = ((1, 2), (3, 4), ("bottom", "top"))


def reference_matrices(p):
    """(K, M): the 1-D stiffness and mass of CG_p on [0, 1] with the GLL Lagrange basis and (p+1)-point Gauss
    quadrature (the action's tables), rows and columns in ascending node position."""
    from .fiat_lite import interval_element
    el = interval_element(p)
    pos = np.argsort(el.nodes)
    B, D, w = el.B[:, pos], el.D[:, pos], el.wq
    return D.T @ (w[:, None] * D), B.T @ (w[:, None] * B)


def star_matrices(p, flags, hl, hr):
    """The 1-D stiffness K and mass M of star directions on the star's m = 2p - 1 nodes, one per row of ``flags``
    (bit 0: a cell on the low side, bit 1: on the high side, bit 2: the centre node is removed by a Dirichlet
    condition) with the interval lengths ``hl``, ``hr`` on the two sides: (1/h) K_ref and h M_ref assembled over the
    one or two intervals, the nodes at offsets -p and p dropped.  Node i of the star is at offset i - (p - 1) from
    its vertex.  Returns (K, M, act, has), shapes (n, m, m) and (n, m): ``act`` marks the nodes in the patch, ``has``
    those some cell of the star holds."""
    Kh, Mh = reference_matrices(p)
    m = 2 * p - 1
    flags = np.asarray(flags, dtype=np.int64)
    hl, hr = np.asarray(hl, dtype=float), np.asarray(hr, dtype=float)
    o = np.arange(m) - (p - 1)
    f = flags[:, None]
    has = np.where(o < 0, (f & 1) != 0, np.where(o > 0, (f & 2) != 0, True))
    act = has & ~((o == 0)[None, :] & ((f & 4) != 0))
    lo, hi = (flags & 1) != 0, (flags & 2) != 0
    K2, M2 = np.zeros((len(flags), 2 * p + 1, 2 * p + 1)), np.zeros((len(flags), 2 * p + 1, 2 * p + 1))
    K2[lo, :p + 1, :p + 1] += Kh / hl[lo, None, None]
    M2[lo, :p + 1, :p + 1] += Mh * hl[lo, None, None]
    K2[hi, p:, p:] += Kh / hr[hi, None, None]
    M2[hi, p:, p:] += Mh * hr[hi, None, None]
    return K2[:, 1:-1, 1:-1], M2[:, 1:-1, 1:-1], act, has


def star_tables(p, flags, hl, hr):
    """The fast-diagonalisation tables of the star directions of :func:`star_matrices`: (S, lam, act, has) with
    K S = M S diag(lam) and S^T M S = I on the active nodes (Cholesky transform of M, then a batched eigh), zero
    rows and columns and lam = 1 elsewhere."""
    K, M, act, has = star_matrices(p, flags, hl, hr)
    n, m = K.shape[0], K.shape[1]
    S, lam = np.zeros((n, m, m)), np.ones((n, m))
    keys = act @ (1 << np.arange(m))
    for key in np.unique(keys):
        sel = np.nonzero(keys == key)[0]
        a = np.nonzero(act[sel[0]])[0]
        if not len(a):
            continue
        L = np.linalg.cholesky(M[sel][:, a][:, :, a])
        Lit = np.swapaxes(np.linalg.inv(L), 1, 2)
        lam_a, Q = np.linalg.eigh(np.swapaxes(Lit, 1, 2) @ K[sel][:, a][:, :, a] @ Lit)
        S[np.ix_(sel, a, np.arange(len(a)))] = Lit @ Q
        lam[sel, :len(a)] = lam_a
    return S, lam, act.astype(float), has.astype(float)


def _side_means(E, axis):
    """Per vertex-lattice point, the mean over the existing cells on its low and high side along ``axis`` of the
    cell quantity ``E`` (shape (nx, ny, nz)), and the number of those cells (0: no cell on that side)."""
    Ep = np.pad(E, 1)
    Cp = np.pad(np.ones_like(E), 1)
    others = [d for d in range(3) if d != axis]

    def window(A):
        # sum over the 2 x 2 cells around each lattice line in the other two directions
        for d in others:
            lo = [slice(None)] * 3
            hi = [slice(None)] * 3
            lo[d], hi[d] = slice(None, -1), slice(1, None)
            A = A[tuple(lo)] + A[tuple(hi)]
        return A
    W, N = window(Ep), window(Cp)
    lo = [slice(None)] * 3
    hi = [slice(None)] * 3
    lo[axis], hi[axis] = slice(None, -1), slice(1, None)
    out = []
    for s in (lo, hi):
        w, c = W[tuple(s)], N[tuple(s)]
        out.append((np.where(c > 0, w / np.maximum(c, 1), 0.0), c))
    return out


class StarTables:
    """The host side of :class:`FDMStar` on the scalar CG_p space ``V`` with Dirichlet conditions on the sub-domains
    ``domains``: the vertex -> base-column table ``vert_cols``, the stars sorted by colour (``star_vert``,
    ``star_layer``, ``colour_ptr``), and the deduplicated 1-D tables (``pool``; ``S``, ``lam``, ``act``, ``has`` as
    returned by :func:`star_tables`) with each star's entries per direction (``star_table``).  NumPy only.

    Per reference direction, h on each side of v is the mean over the star's cells on that side of the mean length
    of each cell's four edges along that direction."""

    def __init__(self, V, domains=()):
        mesh, p = V.mesh, V.degree
        nx, ny, nz = mesh.nx, mesh.ny, mesh.nz
        self.degree = p
        domains = set(domains)
        for s in domains:
            if not any(s in f for f in _FACES):
                raise ValueError(f"FDMStar: unknown Dirichlet sub_domain {s!r}")
        # vertex -> base columns, quadrant sx*2 + sy (sx = 0: the cell on the low-x side)
        col = np.full((nx + 2, ny + 2), -1, dtype=np.int64)
        col[mesh.cell_ix + 1, mesh.cell_iy + 1] = np.arange(mesh.num_base_cells)
        vcols = np.stack([col[sx:sx + nx + 1, sy:sy + ny + 1] for sx in (0, 1) for sy in (0, 1)], axis=-1)
        self.vert_cols = np.ascontiguousarray(vcols.reshape(-1, 4), dtype=np.int32)
        # per cell, the mean length of its four edges along each reference direction, on the (ix, iy, layer) grid
        X = mesh.coordinates
        cm, co = mesh.coord_map.astype(np.int64), np.asarray(mesh.coord_offset, dtype=np.int64)
        lay = np.arange(nz, dtype=np.int64)

        def vx(v):
            return X[cm[:, v, None] + lay[None, :] * co[v]]           # (ncols, nz, 3)
        E = np.zeros((3, nx, ny, nz))
        for d, bit in enumerate((4, 2, 1)):
            e = np.zeros((mesh.num_base_cells, nz))
            for v in range(8):
                if not v & bit:
                    e += np.linalg.norm(vx(v | bit) - vx(v), axis=-1)
            E[d][mesh.cell_ix, mesh.cell_iy] = e / 4.0
        # per star and direction: flags and side lengths
        shape = (nx + 1, ny + 1, nz + 1)
        I, J, K = np.meshgrid(*(np.arange(s) for s in shape), indexing="ij")
        idx = (I, J, K)
        keys = []
        for d in range(3):
            (hl, cl), (hr, cr) = _side_means(E[d], d)
            f = (cl > 0).astype(np.int64) + 2 * (cr > 0)
            lo_face, hi_face = _FACES[d]
            removed = np.zeros(shape, dtype=bool)
            if lo_face in domains:
                removed |= idx[d] == 0
            if hi_face in domains:
                removed |= idx[d] == shape[d] - 1
            f = f + 4 * removed
            keys.append((f.ravel(), np.where(f & 1, hl, 0.0).ravel(), np.where(f & 2, hr, 0.0).ravel()))
        # stars sorted by colour (parities of i, j, layer), then lexicographically
        colour = ((I % 2) * 4 + (J % 2) * 2 + K % 2).ravel()
        order = np.argsort(colour, kind="stable")
        self.colour_ptr = np.concatenate([[0], np.cumsum(np.bincount(colour, minlength=8))]).astype(np.int64)
        self.star_vert = np.ascontiguousarray((I * (ny + 1) + J).ravel()[order], dtype=np.int32)
        self.star_layer = np.ascontiguousarray(K.ravel()[order], dtype=np.int32)
        # deduplicated table pool over all directions; lengths equal to ~1e-12 share an entry
        flags = np.concatenate([k[0][order] for k in keys])
        hl = np.concatenate([k[1][order] for k in keys])
        hr = np.concatenate([k[2][order] for k in keys])
        q = np.stack([flags, hl.view(np.int64) >> 12, hr.view(np.int64) >> 12], axis=1)
        _, first, inv = np.unique(q, axis=0, return_index=True, return_inverse=True)
        nstar = len(order)
        self.star_table = np.ascontiguousarray(np.reshape(inv, (3, nstar)).T, dtype=np.int32)
        self.flags, self.hl, self.hr = flags[first], hl[first], hr[first]
        self.S, self.lam, self.act, self.has = star_tables(p, self.flags, self.hl, self.hr)
        m = 2 * p - 1
        self.pool = np.ascontiguousarray(np.concatenate(
            [self.S.reshape(-1, m * m), self.lam, self.act, self.has], axis=1))

    @property
    def nbytes(self):
        """Device memory of the tables and the per-star data."""
        return (self.pool.nbytes + self.star_table.nbytes + self.star_vert.nbytes + self.star_layer.nbytes
                + self.vert_cols.nbytes + 8 * len(self.star_vert))


class FDMStar:
    """``FDMStar(form, bcs)``: the fast-diagonalisation vertex-star relaxation of ``form`` (a :class:`assemble.Form`
    on a scalar CG_p space, p = 1..5, of an unpartitioned extruded hex mesh) with the Dirichlet conditions ``bcs``:
    ``apply(r, z)`` overwrites z with sum_v R_v^T A_v^-1 R_v r on device-resident Dats, A_v the separable patch
    operator of DESIGN.md section 4.20 (csrc/fdm_star_hex.cu).  ``update()`` after ``form.kappa`` changed.

    The patch of vertex v is its open star (:func:`vertex_star_patches`, without the Dirichlet nodes); the tables
    are :class:`StarTables`, built on the host."""

    def __init__(self, form, bcs=()):
        from .assemble import Form
        if type(form) is not Form or form.ds:
            raise NotImplementedError(f"FDMStar takes a Form without ds terms (its star operators are those of "
                                      f"alpha*kappa*grad.grad + beta*mass with the Gauss rule), not "
                                      f"{type(form).__name__}{' with ds terms' if type(form) is Form else ''}")
        V = form.V
        if getattr(V, "family", "CG") == "NCF":
            raise NotImplementedError("FDMStar does not take NCF (H(div)) spaces: the only form on NCF is "
                                      "MixedPoisson")
        if getattr(V, "family", "CG") != "CG" or V.cdim != 1:
            raise NotImplementedError("FDMStar: scalar CG spaces only")
        if V.dof_dset.halo is not None:
            raise NotImplementedError("FDMStar: partitioned spaces are not supported")
        if not 1 <= V.degree <= 5:
            raise NotImplementedError(f"FDMStar: degree {V.degree} outside 1..5")
        self.form, self.V = form, V
        self._handle = None
        t = self.tables = StarTables(V, {s for bc in bcs for s in bc.sub_domains})
        mesh, p = V.mesh, V.degree
        # the kernel reads the space's own device cell map; the handle keeps no copy, this object keeps V alive
        self._offset = op2.DeviceArray.from_host(np.ascontiguousarray(V.V.offset, dtype=np.int32))
        h = C.c_void_p()
        _lib.check(_lib.lib().fdb_fdm_star_create(
            p, mesh.nz, mesh.num_base_cells, V.cell_node_map.device_ptr, self._offset.ptr, V.node_count,
            len(t.vert_cols),
            t.vert_cols.ctypes.data, len(t.star_vert), t.star_vert.ctypes.data, t.star_layer.ctypes.data,
            t.star_table.ctypes.data, t.colour_ptr.ctypes.data, len(t.pool), t.pool.ctypes.data,
            C.byref(h)), "fdb_fdm_star_create")
        self._handle = h
        self.update()

    def update(self):
        """Recompute the per-star coefficient alpha * mean(kappa) after ``form.kappa`` changed (on the device)."""
        k = self.form.kappa
        _lib.check(_lib.lib().fdb_fdm_star_update(self._handle, float(self.form.alpha), float(self.form.beta),
                                                  None if k is None else k.device_ptr), "fdb_fdm_star_update")

    def apply(self, r: op2.Dat, z: op2.Dat):
        _lib.check(_lib.lib().fdb_fdm_star_apply(self._handle, r.device_ptr, z.device_ptr), "fdb_fdm_star_apply")
        z._device_written()
        return z

    def __del__(self):
        try:
            if self._handle is not None and _lib._initialised is not None:
                _lib._lib.fdb_fdm_star_destroy(self._handle)
        except Exception:
            pass
