"""Host logic of mixed Poisson on the CPU: a mock engine that emulates FDB_FORM_MIXED_POISSON and _SCHUR from the ABI
arrays alone, with the dense NumPy oracle (tests/_mixed_poisson_oracle.py), runs the Python layers -- the MixedDat
assembler, the matrix-free operator with flux conditions, the Schur fieldsplit in every factorisation and
fieldsplit_1 variant, the constant nullspace -- against scipy, and every refusal of the solver options.  The
generic-path statements (the action and the natural-condition load) run through the host build of their generated
wrappers and are checked against the oracle.  The device code itself is what `-m gpu` checks
(tests/test_mixed_poisson_gpu.py)."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import _mixed_poisson_oracle as mo
import _mock_engine as me
from firedrake_b200 import _lib, op2
from firedrake_b200.utility_meshes import ExtrudedHexMesh

SUBS = (1, 2, 3, 4, "bottom", "top")


class MixedPoissonMockEngine(me.MockEngine):
    """MockEngine plus the two mixed Poisson forms on extruded hexes, device location.  The operators are the oracle's
    sparse alpha*M and B, assembled from the maps, offsets and coordinates of the call."""

    def fdb_kernel_create_mixed(self, desc, space2, out):
        d, s2 = me._obj(desc), me._obj(space2)
        if d.form not in (_lib.FORM_MIXED_POISSON, _lib.FORM_MIXED_POISSON_SCHUR):
            return self._fail("mock engine: only the mixed Poisson forms are forms on two spaces here")
        if d.cell != _lib.CELL_HEX_EXTRUDED or d.rank != 1 or s2.degree != d.degree - 1:
            return self._fail("mock engine: mixed Poisson is rank 1 on extruded hexes, DQ_(k-1) second space")
        k = d.degree
        schur = d.form == _lib.FORM_MIXED_POISSON_SCHUR
        self._next += 1
        self.kernels[self._next] = dict(
            kind="mixed_poisson", k=k, schur=schur, alpha=d.alpha, diagonal=bool(d.diagonal),
            off_s=np.array(d.offset0[:3 * k * k * (k + 1)], dtype=np.int64),
            off_c=None if schur else np.array(d.offset1[:8], dtype=np.int64),
            off_u=np.array(s2.offset[:k ** 3], dtype=np.int64), cache={})
        me._obj(out).value = self._next
        return 0

    def _matrices(self, kk, a, map_s, map_u, map_c):
        """alpha*M and B over the call's cells (built once per set of maps)."""
        key = (me._addr(a.maps[0]), me._addr(a.maps[1]), a.end, a.layers[1])
        if key in kk["cache"]:
            return kk["cache"][key]
        k, nlay = kk["k"], a.layers[1] - 1
        lay = np.arange(nlay)
        rows = lambda m, o: (m[:, None, :] + lay[None, :, None] * o[None, None, :]).reshape(-1, m.shape[1])
        fs = rows(map_s, kk["off_s"])
        # (the diagonal of alpha*M is called without the DQ map: any distinct rows serve)
        fq = rows(map_u, kk["off_u"]) if map_u is not None else np.arange(len(fs) * k ** 3).reshape(len(fs), -1)
        nS, nQ = int(fs.max()) + 1, int(fq.max()) + 1
        if map_c is not None:
            fc = rows(map_c, kk["off_c"])
            Xv = me._view(a.args[1], (int(fc.max()) + 1) * 3).reshape(-1, 3)[fc]
        else:
            # B is metric-free: any cell gives it; the unit cube stands in
            Xv = np.broadcast_to(np.array([[(v >> 2) & 1, (v >> 1) & 1, v & 1] for v in range(8)], dtype=float),
                                 (len(fs), 8, 3))
        kk["cache"][key] = mo.matrices_from_rows(k, Xv, fs, fq, nS, nQ, kk["alpha"])
        return kk["cache"][key]

    def fdb_kernel_call(self, h, ca):
        kk = self.kernels[me._addr(h)]
        if kk["kind"] != "mixed_poisson":
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        self.launches += 1
        k = kk["k"]
        want = (2 if kk["diagonal"] else 4) if kk["schur"] else (2 if kk["diagonal"] else 5)
        want_maps = 3 if not kk["schur"] and not kk["diagonal"] else 2
        if a.location != _lib.LOC_DEVICE or a.nargs != want or a.nmaps != want_maps:
            return self._fail(f"mock engine: mixed Poisson expects {want} device args and {want_maps} maps")
        ns, nu = 3 * k * k * (k + 1), k ** 3
        if kk["schur"]:
            map_u = me._view(a.maps[0], a.end * nu, np.int32).reshape(a.end, nu).astype(np.int64)
            map_s = me._view(a.maps[1], a.end * ns, np.int32).reshape(a.end, ns).astype(np.int64)
            _, B = self._matrices(kk, a, map_s, map_u, None)
            nQ, nS = B.shape
            y = me._view(a.args[0], nQ)
            if kk["diagonal"]:
                y += B.multiply(B) @ me._view(a.args[1], nS)
            else:
                t = me._view(a.args[3], nS)
                t += B.T @ me._view(a.args[1], nQ)
                y += B @ (me._view(a.args[2], nS) * t)
            return 0
        map_s = me._view(a.maps[0], a.end * ns, np.int32).reshape(a.end, ns).astype(np.int64)
        map_c = me._view(a.maps[1], a.end * 8, np.int32).reshape(a.end, 8).astype(np.int64)
        if kk["diagonal"]:
            M, _ = self._matrices(kk, a, map_s, None, map_c)
            me._view(a.args[0], M.shape[0])[:] += M.diagonal()
            return 0
        map_u = me._view(a.maps[2], a.end * nu, np.int32).reshape(a.end, nu).astype(np.int64)
        M, B = self._matrices(kk, a, map_s, map_u, map_c)
        nQ, nS = B.shape
        s, u = me._view(a.args[2], nS).copy(), me._view(a.args[4], nQ).copy()
        me._view(a.args[0], nS)[:] += M @ s + B.T @ u
        me._view(a.args[3], nQ)[:] += B @ s
        return 0


@pytest.fixture()
def mock(oracle):
    inst = me.install(oracle)
    inst.engine = MixedPoissonMockEngine(oracle)
    with inst as eng:
        yield eng


def _spaces(k=2, n=(3, 3, 3), warp=0.05, permute_seed=1, alpha=1.3):
    from firedrake_b200.assemble import FunctionSpace, MixedPoisson
    mesh = ExtrudedHexMesh(*n, warp=warp, permute_seed=permute_seed)
    S, Q = FunctionSpace(mesh, k, family="NCF"), FunctionSpace(mesh, k - 1, family="DQ")
    return mesh, S, Q, MixedPoisson(S, Q, alpha)


@pytest.mark.parametrize("k", [2, 3])
def test_generic_path_host_build_matches_the_oracle(oracle, k):
    """``mixed_poisson_kernel`` through the host build of its generated wrapper gives the oracle's action."""
    from firedrake_b200.assemble import assemble_mixed_poisson_generic
    with me.install(oracle):
        mesh, S, Q, F = _spaces(k, n=(2, 3, 2))
        M, B = mo.global_matrices(mesh, S.V, Q.V, F.alpha)
        rng = np.random.default_rng(k)
        s, u = rng.standard_normal(S.node_count), rng.standard_normal(Q.node_count)
        y = [d.data_ro.copy() for d in assemble_mixed_poisson_generic(F, F.dat(s.copy(), u.copy()))]
    assert np.abs(y[0] - (M @ s + B.T @ u)).max() < 1e-12 * np.abs(M @ s + B.T @ u).max()
    assert np.abs(y[1] - B @ s).max() < 1e-12 * np.abs(B @ s).max()


@pytest.mark.parametrize("k", [2, 3])
def test_natural_condition_load_matches_the_oracle(oracle, k):
    """``mixed_dirichlet_load`` on every sub-domain, and on all of them at once, equals the oracle's int (tau.n) g ds
    on a warped, permuted mesh, with g a nonconstant trilinear field."""
    from firedrake_b200.assemble import mixed_dirichlet_load
    with me.install(oracle):
        mesh, S, Q, F = _spaces(k, n=(2, 3, 2))
        X = mesh.coordinates
        gv = 1.0 + X[:, 0] - 2.0 * X[:, 1] * X[:, 2] + 0.5 * X[:, 2]
        g = op2.Dat(op2.DataSet(S.vertex_set, 1), gv.copy())
        for sub in SUBS:
            want = mo.dirichlet_load(mesh, S.V, gv, sub)
            got = mixed_dirichlet_load(F, g, sub).data_ro
            assert np.abs(got - want).max() < 1e-13 * np.abs(want).max(), sub
            assert np.abs(want).max() > 0
        want = sum(mo.dirichlet_load(mesh, S.V, gv, s) for s in SUBS)
        got = mixed_dirichlet_load(F, g).data_ro
        assert np.abs(got - want).max() < 1e-13 * np.abs(want).max()


def test_matfree_mult_and_diagonal_with_flux_conditions(mock):
    """The operator is the oracle's saddle matrix with identity rows and columns on the flux conditions; the
    diagonal is diag(alpha M) with 1 there."""
    from firedrake_b200.assemble import DirichletBC, assemble
    mesh, S, Q, F = _spaces()
    bcs = [DirichletBC(S, 0.0, s) for s in (1, "top")]
    M, B = mo.global_matrices(mesh, S.V, Q.V, F.alpha)
    rows = np.unique(np.concatenate([bc.nodes for bc in bcs]))
    K = mo.constrained(mo.saddle(M, B), rows)
    x = np.random.default_rng(0).standard_normal(S.node_count + Q.node_count)
    A = assemble(F, bcs=bcs, mat_type="matfree")
    Y = F.dat()
    A.mult(F.dat(x[:S.node_count].copy(), x[S.node_count:].copy()), Y)
    y = np.concatenate([Y[0].data_ro, Y[1].data_ro])
    assert np.abs(y - K @ x).max() < 1e-12 * np.abs(K @ x).max()
    d = A.getDiagonal().data_ro
    assert np.abs(d - K.diagonal()[:S.node_count]).max() < 1e-12 * np.abs(d).max()


SOLVER = {"ksp_type": "gmres", "ksp_rtol": 1e-11, "pc_type": "fieldsplit", "pc_fieldsplit_type": "schur",
          "pc_fieldsplit_schur_fact_type": "full", "pc_fieldsplit_schur_precondition": "selfp",
          "fieldsplit_0_ksp_type": "preonly", "fieldsplit_0_pc_type": "jacobi", "fieldsplit_1_ksp_type": "cg",
          "fieldsplit_1_pc_type": "jacobi", "fieldsplit_1_ksp_rtol": 1e-5}


def _load(mesh, S, Q, F, flux_bcs):
    """(sigma load, u load) with a source, and natural data g on the sides without flux conditions."""
    from firedrake_b200.assemble import mixed_dirichlet_load
    X = Q.V.dof_coordinates()
    f = np.sin(np.pi * X[:, 0]) * np.cos(np.pi * X[:, 1]) + X[:, 2]
    L = F.dat(np.zeros(S.node_count), -(mo.dq_mass(mesh, Q.V) @ f))
    if not flux_bcs:
        gv = mesh.coordinates[:, 0] * mesh.coordinates[:, 1]
        mixed_dirichlet_load(F, op2.Dat(op2.DataSet(S.vertex_set, 1), gv.copy()), (2, 4), tensor=L[0])
    return L


def _scipy(mesh, S, Q, F, L, bcs, nullspace):
    M, B = mo.global_matrices(mesh, S.V, Q.V, F.alpha)
    rows = np.unique(np.concatenate([bc.nodes for bc in bcs])) if bcs else np.zeros(0, dtype=np.int64)
    rhs = np.concatenate([L[0].data_ro, L[1].data_ro])
    rhs[rows] = 0.0
    pin = []
    if nullspace:
        rhs[S.node_count:] -= rhs[S.node_count:].mean()
        pin = [S.node_count]
        rhs[pin] = 0.0
    x = spla.spsolve(mo.constrained(mo.saddle(M, B), np.concatenate([rows, pin]).astype(np.int64)).tocsc(), rhs)
    if nullspace:
        x[S.node_count:] -= x[S.node_count:].mean()
    return x[:S.node_count], x[S.node_count:]


@pytest.mark.parametrize("fact", ["full", "diag", "lower", "upper"])
@pytest.mark.parametrize("inner", ["cg", "preonly"])
def test_fieldsplit_gmres_matches_scipy(mock, fact, inner):
    """Natural conditions (g on two sides) and a source: every factorisation and fieldsplit_1 variant converges to
    scipy's solution."""
    from firedrake_b200.assemble import solve
    mesh, S, Q, F = _spaces()
    L = _load(mesh, S, Q, F, False)
    up = F.dat()
    its, hist = solve(F, L, up, (), {**SOLVER, "pc_fieldsplit_schur_fact_type": fact,
                                     "fieldsplit_1_ksp_type": inner, "ksp_max_it": 2000})
    assert hist[-1] <= 1e-11 * hist[0]
    s_ref, u_ref = _scipy(mesh, S, Q, F, L, (), False)
    assert np.abs(up[0].data_ro - s_ref).max() < 1e-8 * np.abs(s_ref).max()
    assert np.abs(up[1].data_ro - u_ref).max() < 1e-8 * np.abs(u_ref).max()


@pytest.mark.parametrize("fact", ["full", "lower"])
@pytest.mark.parametrize("inner", ["cg", "preonly"])
def test_flux_conditions_with_constant_nullspace(mock, fact, inner):
    """Flux conditions on the whole boundary: the constant nullspace, also inside the inner CG; u comes back with
    zero mean, and sigma.n = 0 on the boundary."""
    from firedrake_b200.assemble import DirichletBC, solve
    mesh, S, Q, F = _spaces()
    bcs = [DirichletBC(S, 0.0, s) for s in SUBS]
    L = _load(mesh, S, Q, F, True)
    up = F.dat()
    solve(F, L, up, bcs, {**SOLVER, "pc_fieldsplit_schur_fact_type": fact, "fieldsplit_1_ksp_type": inner,
                          "ksp_max_it": 2000}, nullspace="constant")
    s_ref, u_ref = _scipy(mesh, S, Q, F, L, bcs, True)
    assert np.abs(up[0].data_ro - s_ref).max() < 1e-8 * np.abs(s_ref).max()
    assert np.abs(up[1].data_ro - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    assert abs(up[1].data_ro.mean()) < 1e-12 * np.abs(u_ref).max()
    assert np.all(up[0].data_ro[np.concatenate([bc.nodes for bc in bcs])] == 0.0)


def test_unpreconditioned_gmres_matches_scipy(mock):
    from firedrake_b200.assemble import solve
    mesh, S, Q, F = _spaces(n=(2, 2, 2))
    L = _load(mesh, S, Q, F, False)
    up = F.dat()
    solve(F, L, up, (), {"ksp_rtol": 1e-12, "ksp_max_it": 5000, "ksp_gmres_restart": 200})
    s_ref, u_ref = _scipy(mesh, S, Q, F, L, (), False)
    assert np.abs(up[0].data_ro - s_ref).max() < 1e-8 * np.abs(s_ref).max()
    assert np.abs(up[1].data_ro - u_ref).max() < 1e-8 * np.abs(u_ref).max()


@pytest.mark.parametrize("opts, exc, msg", [
    ({"ksp_type": "cg"}, ValueError, "indefinite"),
    ({"ksp_type": "minres"}, NotImplementedError, "ksp_type 'minres'"),
    ({"mat_type": "aij"}, NotImplementedError, "mat_type 'aij'"),
    ({"pc_type": "jacobi"}, NotImplementedError, "pc_type 'jacobi'"),
    ({"pc_type": "fieldsplit", "pc_fieldsplit_type": "additive"}, NotImplementedError, "pc_fieldsplit_type"),
    ({"pc_type": "fieldsplit", "pc_fieldsplit_schur_fact_type": "lu"}, NotImplementedError,
     "pc_fieldsplit_schur_fact_type"),
    ({"pc_type": "fieldsplit", "pc_fieldsplit_schur_precondition": "a11"}, NotImplementedError,
     "pc_fieldsplit_schur_precondition"),
    ({"pc_type": "fieldsplit", "fieldsplit_0_ksp_type": "cg"}, NotImplementedError, "fieldsplit_0_ksp_type"),
    ({"pc_type": "fieldsplit", "fieldsplit_0_pc_type": "mg"}, NotImplementedError, "fieldsplit_0_pc_type"),
    ({"pc_type": "fieldsplit", "fieldsplit_1_ksp_type": "gmres"}, NotImplementedError, "fieldsplit_1_ksp_type"),
    ({"pc_type": "fieldsplit", "fieldsplit_1_pc_type": "hypre"}, NotImplementedError, "fieldsplit_1_pc_type"),
    ({"ksp_monitor": None}, NotImplementedError, "ksp_monitor"),
    ({"fieldsplit_1_pc_hypre_type": "boomeramg"}, NotImplementedError, "fieldsplit_1_pc_hypre_type"),
])
def test_solver_option_refusals(mock, opts, exc, msg):
    from firedrake_b200.assemble import solve
    _, S, Q, F = _spaces(n=(1, 1, 1))
    with pytest.raises(exc, match=msg):
        solve(F, F.dat(), F.dat(), (), opts)


def test_other_solver_refusals(mock):
    from firedrake_b200.assemble import DirichletBC, FunctionSpace, MixedPoisson, assemble, solve
    mesh, S, Q, F = _spaces(n=(1, 1, 1))
    with pytest.raises(NotImplementedError, match="nullspace 'pressure'"):
        solve(F, F.dat(), F.dat(), (), {}, nullspace="pressure")
    other = FunctionSpace(mesh, 2, family="NCF")
    with pytest.raises(ValueError, match="flux conditions on its NCF space"):
        solve(F, F.dat(), F.dat(), [DirichletBC(other, 0.0, 1)], {})
    with pytest.raises(NotImplementedError, match="nonzero flux value"):
        DirichletBC(S, 1.0, 1)
    with pytest.raises(NotImplementedError, match="mat_type 'aij'"):
        assemble(F)
    with pytest.raises(NotImplementedError, match="no assembled matrix"):
        F.kernel(2)
    with pytest.raises(ValueError, match="NCF_k"):
        MixedPoisson(Q, Q)
    with pytest.raises(ValueError, match="same mesh"):
        MixedPoisson(S, FunctionSpace(ExtrudedHexMesh(1, 1, 1), 1, family="DQ"))
    with pytest.raises(ValueError, match="vertex"):
        from firedrake_b200.assemble import mixed_dirichlet_load
        mixed_dirichlet_load(F, Q.dat(), 1)
