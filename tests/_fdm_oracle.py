"""TEST INFRASTRUCTURE: a NumPy restatement of the fast-diagonalisation vertex-star relaxation (patch.FDMStar), star
by star on the dof lattice, and the separable star operators of DESIGN.md section 4.20 (small meshes only)."""
import numpy as np

from firedrake_b200.patch import star_matrices


def star_nodes(V, t):
    """(nstar, m, m, m): the node at every lattice point of every star of ``t`` (a patch.StarTables on the space
    ``V``), in the tables' star order, -1 outside the mesh; and the stars' vertex lattice indices (I, J, K)."""
    fs, mesh = V.V, V.mesh
    p = fs.degree
    m = 2 * p - 1
    lat = fs.dof_lattice()
    grid = np.full(tuple(lat.max(axis=0) + 1), -1, dtype=np.int64)
    grid[lat[:, 0], lat[:, 1], lat[:, 2]] = np.arange(fs.node_count)
    I, J = np.divmod(t.star_vert.astype(np.int64), mesh.ny + 1)
    K = t.star_layer.astype(np.int64)
    o = np.arange(m) - (p - 1)
    pos = [c[:, None] * p + o[None, :] for c in (I, J, K)]
    ok = [(x >= 0) & (x < n) for x, n in zip(pos, grid.shape)]
    P = [np.clip(x, 0, n - 1) for x, n in zip(pos, grid.shape)]
    nodes = grid[P[0][:, :, None, None], P[1][:, None, :, None], P[2][:, None, None, :]]
    inside = ok[0][:, :, None, None] & ok[1][:, None, :, None] & ok[2][:, None, None, :]
    return np.where(inside, nodes, -1), (I, J, K)


def _dirs(t, what):
    return [getattr(t, what)[t.star_table[:, d]] for d in range(3)]


def _outer(a, b, c):
    return a[:, :, None, None] * b[:, None, :, None] * c[:, None, None, :]


def star_coefficient(t, nodes, alpha, kappa=None):
    """alpha * the mean of kappa (None: 1) over every star's existing nodes."""
    has = _outer(*_dirs(t, "has")) != 0
    k = np.ones(nodes.max() + 1) if kappa is None else np.asarray(kappa)
    vals = np.where(has, k[np.where(has, nodes, 0)], 0.0)
    return alpha * vals.sum(axis=(1, 2, 3)) / has.sum(axis=(1, 2, 3))


def apply(t, nodes, r, alpha=1.0, beta=0.0, kappa=None):
    """z = sum_v R_v^T A_v^-1 R_v r."""
    Sx, Sy, Sz = _dirs(t, "S")
    act = _outer(*_dirs(t, "act")) != 0
    u = np.where(act, r[np.where(act, nodes, 0)], 0.0)
    uh = np.einsum("sia,sjb,skc,sijk->sabc", Sx, Sy, Sz, u, optimize=True)
    lx, ly, lz = _dirs(t, "lam")
    ak = star_coefficient(t, nodes, alpha, kappa)
    D = ak[:, None, None, None] * (lx[:, :, None, None] + ly[:, None, :, None] + lz[:, None, None, :]) + beta
    y = np.einsum("sia,sjb,skc,sabc->sijk", Sx, Sy, Sz, uh / D, optimize=True)
    z = np.zeros(len(r))
    np.add.at(z, nodes[act], y[act])
    return z


def separable_operator(t, s, alpha=1.0, beta=0.0, kbar=1.0):
    """The separable A_v of star s on its active nodes (lattice order), from its 1-D K and M rebuilt from the
    tables' flags and lengths."""
    K, M, act = [], [], []
    for d in range(3):
        e = t.star_table[s, d]
        k, mm, a, _ = star_matrices(t.degree, t.flags[e:e + 1], t.hl[e:e + 1], t.hr[e:e + 1])
        sel = np.nonzero(a[0])[0]
        K.append(k[0][np.ix_(sel, sel)])
        M.append(mm[0][np.ix_(sel, sel)])
    kron = lambda a, b, c: np.kron(np.kron(a, b), c)
    return (alpha * kbar * (kron(K[0], M[1], M[2]) + kron(M[0], K[1], M[2]) + kron(M[0], M[1], K[2]))
            + beta * kron(M[0], M[1], M[2]))


# ---------------------------------------------------------------------------------------------------------------
# The engine calls fdb_fdm_star_* in NumPy, from the arrays of the C ABI alone: a mock engine mixin for the host
# tests (tests/test_fdm_host_mock.py), whose gather restates the kernel's (csrc/fdm_star_hex.cu line_nodes).

def abi_star_nodes(p, nz, cmap, off, vcols, svert, slay):
    """(nstar, m, m, m) nodes of every star from the extruded cell-node map and the vertex -> column table."""
    m, n = 2 * p - 1, p + 1
    o = np.arange(m) - (p - 1)
    pos2dof = lambda a: np.where(a == 0, 0, np.where(a == p, 1, a + 1))
    vc = vcols[svert]                                               # (nstar, 4)
    rx = (vc[:, 2] >= 0) | (vc[:, 3] >= 0)
    ry = (vc[:, 1] >= 0) | (vc[:, 3] >= 0)
    rz = slay < nz

    def side(r):
        return np.where(o[None, :] < 0, 0, np.where(o[None, :] > 0, 1, r[:, None].astype(int)))
    sx, sy, sz = side(rx), side(ry), side(rz)
    dx, dy, dz = (pos2dof(np.where(s == 1, o[None, :], o[None, :] + p)) for s in (sx, sy, sz))
    S = np.arange(len(svert))[:, None, None, None]
    col = vc[S, sx[:, :, None, None] * 2 + sy[:, None, :, None]]
    layer = slay[:, None, None, None] - 1 + sz[:, None, None, :]
    loc = (dx[:, :, None, None] * n + dy[:, None, :, None]) * n + dz[:, None, None, :]
    ok = (col >= 0) & (layer >= 0) & (layer < nz)
    node = cmap[np.where(ok, col, 0), loc] + layer * off[loc]
    return np.where(ok, node, -1)


class FDMMixin:
    """fdb_fdm_star_create / update / apply / destroy on the host; ``trace`` records ("fdb_fdm_star_apply", n)."""

    def fdb_fdm_star_create(self, degree, nz, ncols, cmap, off, node_count, nvert, vcols, nstar, svert, slay, stab,
                            cptr, npool, pool, out):
        import types
        from _mock_engine import _obj, _view
        p, n3, m = degree, (degree + 1) ** 3, 2 * degree - 1
        iv = lambda a, c: _view(a, c, np.int32).astype(np.int64)
        E = m * m + 3 * m
        P = _view(pool, npool * E).reshape(npool, E).copy()
        t = types.SimpleNamespace(S=P[:, :m * m].reshape(-1, m, m), lam=P[:, m * m:m * m + m],
                                  act=P[:, m * m + m:m * m + 2 * m], has=P[:, m * m + 2 * m:],
                                  star_table=iv(stab, 3 * nstar).reshape(nstar, 3))
        nodes = abi_star_nodes(p, nz, iv(cmap, ncols * n3).reshape(ncols, n3), iv(off, n3),
                               iv(vcols, 4 * nvert).reshape(nvert, 4), iv(svert, nstar), iv(slay, nstar))
        self._next += 1
        self.stars = getattr(self, "stars", {})
        self.stars[self._next] = dict(t=t, nodes=nodes, n=node_count, alpha=1.0, beta=0.0, kappa=None)
        _obj(out).value = self._next
        return 0

    def fdb_fdm_star_update(self, h, alpha, beta, kappa):
        from _mock_engine import _addr, _view
        st = self.stars[_addr(h)]
        st.update(alpha=alpha, beta=beta, kappa=None if not kappa else _view(kappa, st["n"]).copy())
        return 0

    def fdb_fdm_star_apply(self, h, r, z):
        from _mock_engine import _addr, _view
        st = self.stars[_addr(h)]
        self.trace.append(("fdb_fdm_star_apply", st["n"]))
        if getattr(self, "compute", True):
            _view(z, st["n"])[:] = apply(st["t"], st["nodes"], _view(r, st["n"]), st["alpha"], st["beta"],
                                         st["kappa"])
        return 0

    def fdb_fdm_star_destroy(self, h):
        return 0
