"""Mixed Poisson on NCF_k x DQ_{k-1} on the H100: the hand-written kernels (FDB_FORM_MIXED_POISSON, _SCHUR) against
the dense NumPy oracle (tests/_mixed_poisson_oracle.py) and the generic wrapper path, and the Schur fieldsplit solve
against scipy."""
import numpy as np
import pytest

import _mixed_poisson_oracle as mo
from firedrake_b200 import _lib, op2
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu


def _spaces(k, n=3, warp=0.05, permute_seed=0, alpha=1.7):
    from firedrake_b200.assemble import FunctionSpace, MixedPoisson
    mesh = ExtrudedHexMesh(n, n + 1, n, warp=warp, permute_seed=permute_seed)
    S = FunctionSpace(mesh, k, family="NCF")
    Q = FunctionSpace(mesh, k - 1, family="DQ")
    return mesh, S, Q, MixedPoisson(S, Q, alpha)


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _native(S, Q, mesh, kernel, scatter, args_of):
    """Run ``kernel`` on native hexes: one map row per cell (the extruded maps with the layer loop expanded)."""
    cells = op2.Set(mesh.num_cells)
    ms = op2.Map(cells, S.node_set, S.V.arity, S.V.full_cell_node_list())
    mc = op2.Map(cells, S.vertex_set, 8, mesh.coord_space.full_cell_node_list())
    mq = op2.Map(cells, Q.node_set, Q.V.arity, Q.V.full_cell_node_list())
    maps = [ms, mc, mq] if kernel.form == "mixed_poisson" else [mq, ms]
    gk = op2.GlobalKernel(kernel, maps, extruded=False, scatter=scatter)
    op2.Parloop(gk, cells, args_of(ms, mc, mq), location="device")()


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("extruded", [True, False])
@pytest.mark.parametrize("scatter", ["atomic", "coloured"])
def test_action_and_diagonal_match_oracle(k, extruded, scatter):
    """y = (alpha M s + B^T u, B s) and diag(alpha M) on a warped, permuted mesh, to 1e-12 relative."""
    from firedrake_b200.assemble import StokesAssembler
    mesh, S, Q, F = _spaces(k)
    M, B = mo.global_matrices(mesh, S.V, Q.V, F.alpha)
    rng = np.random.default_rng(k)
    s, u = rng.standard_normal(S.node_count), rng.standard_normal(Q.node_count)
    up = F.dat(s, u)
    y = F.dat()
    d = S.dat()
    if extruded:
        StokesAssembler(F, up, scatter=scatter).assemble(y)
        from firedrake_b200.assemble import MixedPoissonMatrixContext
        MixedPoissonMatrixContext(F).getDiagonal(d, scatter=scatter)
    else:
        y.zero()
        for t in y:
            t.device_ptr
        _native(S, Q, mesh, F.kernel(1), scatter, lambda ms, mc, mq: [
            y[0](op2.INC, ms), S.coordinates(op2.READ, mc), up[0](op2.READ, ms), y[1](op2.INC, mq),
            up[1](op2.READ, mq)])
        d.zero()
        _native(S, Q, mesh, F.kernel(1, diagonal=True), scatter, lambda ms, mc, mq: [
            d(op2.INC, ms), S.coordinates(op2.READ, mc)])
    assert _rel(y[0].data_ro, M @ s + B.T @ u) < 1e-12
    assert _rel(y[1].data_ro, B @ s) < 1e-12
    assert _rel(d.data_ro, M.diagonal()) < 1e-12


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("extruded", [True, False])
@pytest.mark.parametrize("scatter", ["atomic", "coloured"])
def test_schur_action_and_diagonal_match_dense(k, extruded, scatter):
    """S_p u and diag(S_p) against the dense B W B^T, W positive with zeros on some flux rows."""
    from firedrake_b200.assemble import MixedPoissonSchur
    mesh, S, Q, F = _spaces(k)
    _, B = mo.global_matrices(mesh, S.V, Q.V, F.alpha)
    rng = np.random.default_rng(10 + k)
    wv = rng.uniform(0.5, 2.0, S.node_count)
    wv[S.boundary_nodes(1)] = 0.0
    u = rng.standard_normal(Q.node_count)
    Sp = (B @ np.diag(wv) @ B.T.toarray())
    w, x, y, d = S.dat(wv), Q.dat(u), Q.dat(), Q.dat()
    if extruded:
        op = MixedPoissonSchur(F, w, scatter=scatter)
        op.mult(x, y)
        op.getDiagonal(d)
    else:
        t = S.dat()
        t.zero()
        y.zero()
        d.zero()
        for v in (t, y, d):
            v.device_ptr
        _native(S, Q, mesh, op2.Kernel("mixed_poisson_schur", degree=k), scatter, lambda ms, mc, mq: [
            y(op2.INC, mq), x(op2.READ, mq), w(op2.READ, ms), t(op2.INC, ms)])
        _native(S, Q, mesh, op2.Kernel("mixed_poisson_schur", degree=k, diagonal=True), scatter,
                lambda ms, mc, mq: [d(op2.INC, mq), w(op2.READ, ms)])
    assert _rel(y.data_ro, Sp @ u) < 1e-12
    assert _rel(d.data_ro, np.diag(Sp)) < 1e-12


@pytest.mark.parametrize("k", [2, 3, 4])
def test_action_matches_generic_path(k):
    from firedrake_b200.assemble import assemble, assemble_mixed_poisson_generic
    mesh, S, Q, F = _spaces(k, permute_seed=3)
    rng = np.random.default_rng(20 + k)
    up = F.dat(rng.standard_normal(S.node_count), rng.standard_normal(Q.node_count))
    y = assemble(F, u=up)
    yg = assemble_mixed_poisson_generic(F, up)
    for a, b in zip(y, yg):
        assert _rel(a.data_ro, b.data_ro) < 1e-12


def _reference_solve(mesh, S, Q, F, bcs, L, nullspace):
    import scipy.sparse.linalg as spla
    M, B = mo.global_matrices(mesh, S.V, Q.V, F.alpha)
    K = mo.saddle(M, B)
    rows = np.unique(np.concatenate([bc.nodes for bc in bcs])) if bcs else np.zeros(0, dtype=int)
    rhs = np.concatenate([L[0].data_ro, L[1].data_ro])
    rhs[rows] = 0.0
    pin = [S.node_count] if nullspace else []
    if nullspace:
        rhs[S.node_count:] -= rhs[S.node_count:].mean()
        rhs[pin] = 0.0                       # u_0 = 0, then the mean is removed
    x = spla.spsolve(mo.constrained(K, np.concatenate([rows, pin]).astype(int)).tocsc(), rhs)
    if nullspace:
        x[S.node_count:] -= x[S.node_count:].mean()
    return x[:S.node_count], x[S.node_count:], M, B


SOLVER = {"ksp_type": "gmres", "ksp_rtol": 1e-10, "pc_type": "fieldsplit", "pc_fieldsplit_type": "schur",
          "pc_fieldsplit_schur_fact_type": "full", "pc_fieldsplit_schur_precondition": "selfp",
          "fieldsplit_0_ksp_type": "preonly", "fieldsplit_0_pc_type": "jacobi", "fieldsplit_1_ksp_type": "cg",
          "fieldsplit_1_pc_type": "jacobi", "fieldsplit_1_ksp_rtol": 1e-5}


def _problem(n, k=2, warp=0.0, flux_bcs=False):
    from firedrake_b200.assemble import DirichletBC, assemble, mass, mixed_dirichlet_load
    mesh, S, Q, F = _spaces(k, n=n, warp=warp, permute_seed=None, alpha=1.0)
    X = Q.V.dof_coordinates()
    f = Q.dat(3 * np.pi ** 2 * np.sin(np.pi * X[:, 0]) * np.sin(np.pi * X[:, 1]) * np.sin(np.pi * X[:, 2])
              + (np.cos(2 * np.pi * X[:, 0]) if flux_bcs else 0.0))
    L = F.dat()
    L.zero()
    Mf = assemble(mass(Q), u=f)
    L[1].axpy(-1.0, Mf)
    bcs = [DirichletBC(S, 0.0, s) for s in (1, 2, 3, 4, "bottom", "top")] if flux_bcs else []
    if not flux_bcs:
        g = op2.Dat(op2.DataSet(S.vertex_set, 1), mesh.coordinates[:, 0].copy())
        mixed_dirichlet_load(F, g, 2, tensor=L[0])
    return mesh, S, Q, F, L, bcs


@pytest.mark.parametrize("fact", ["full", "diag", "lower", "upper"])
@pytest.mark.parametrize("inner", ["cg", "preonly"])
def test_solve_matches_scipy(fact, inner):
    """8^3, k = 2, natural conditions (u = x on x == 1, u = 0 elsewhere) and a source: GMRES with every Schur
    factorisation matches scipy to 1e-8; div sigma_h = -Pi f cellwise (the u-block residual is at the tolerance)."""
    from firedrake_b200.assemble import solve
    mesh, S, Q, F, L, bcs = _problem(8)
    up = F.dat()
    its, hist = solve(F, L, up, bcs, {**SOLVER, "pc_fieldsplit_schur_fact_type": fact,
                                      "fieldsplit_1_ksp_type": inner, "ksp_max_it": 3000})
    s_ref, u_ref, M, B = _reference_solve(mesh, S, Q, F, bcs, L, False)
    assert _rel(up[0].data_ro, s_ref) < 1e-8
    assert _rel(up[1].data_ro, u_ref) < 1e-8
    r = B @ up[0].data_ro - L[1].data_ro
    assert np.abs(r).max() < 1e-8 * np.abs(L[1].data_ro).max()


def test_solve_with_flux_conditions_and_constant_nullspace():
    from firedrake_b200.assemble import solve
    mesh, S, Q, F, L, bcs = _problem(6, warp=0.03, flux_bcs=True)
    up = F.dat()
    solve(F, L, up, bcs, SOLVER, nullspace="constant")
    s_ref, u_ref, _, _ = _reference_solve(mesh, S, Q, F, bcs, L, True)
    assert _rel(up[0].data_ro, s_ref) < 1e-8
    assert _rel(up[1].data_ro, u_ref) < 1e-8
    assert abs(up[1].data_ro.mean()) < 1e-12 * np.abs(u_ref).max()


def test_iterations_grow_slowly_with_full_and_inner_cg():
    """Outer GMRES iterations with "full" and inner CG at 16^3 are at most those at 8^3 plus 2; the preonly-Jacobi
    counts are printed."""
    from firedrake_b200.assemble import solve
    counts = {}
    for n in (8, 16):
        for inner in ("cg", "preonly"):
            _, S, Q, F, L, bcs = _problem(n)
            up = F.dat()
            its, _ = solve(F, L, up, bcs, {**SOLVER, "ksp_rtol": 1e-8, "fieldsplit_1_ksp_type": inner,
                                           "ksp_max_it": 5000})
            counts[(n, inner)] = its
    print("outer GMRES iterations", counts)
    assert counts[(16, "cg")] <= counts[(8, "cg")] + 2


def test_create_call_and_solver_refusals():
    from firedrake_b200.assemble import solve
    mesh, S, Q, F = _spaces(2)
    lib = _lib.lib()
    import ctypes as C
    base = op2.GlobalKernel(F.kernel(1), [S.cell_node_map, S.coord_map, F.pressure_map], extruded=True)
    base.compile()

    def create(**kw):
        d = _lib.KernelDesc()
        from firedrake_b200.fiat_lite import interval_element
        el = interval_element(kw.get("degree", 2))
        d.form, d.rank, d.cell, d.integral = _lib.FORM_MIXED_POISSON, kw.get("rank", 1), _lib.CELL_HEX, 0
        d.degree, d.nq, d.cdim = kw.get("degree", 2), kw.get("nq", el.nq), 1
        d.affine_cells = kw.get("affine", 0)
        n = d.degree + 1
        for q in range(el.nq):
            d.wq[q], d.xq[q] = el.wq[q], el.xq[q]
            for a in range(n):
                d.B[q * n + a], d.D[q * n + a] = el.B[q, a], el.D[q, a]
        s2 = _lib.Space2Desc()
        s2.degree = kw.get("degree2", d.degree - 1)
        h = C.c_void_p()
        rc = lib.fdb_kernel_create_mixed(C.byref(d), C.byref(s2), C.byref(h))
        return rc, lib.fdb_last_error().decode()

    assert create()[0] == 0
    for kw, msg in [({"degree": 5}, "degree 5 outside 2..4"), ({"degree": 1, "degree2": 0}, "outside 2..4"),
                    ({"degree2": 2}, "second space of degree 1"), ({"rank": 2}, "no rank-2"),
                    ({"affine": 1}, "affine"), ({"nq": 4}, "nq == degree+1")]:
        rc, err = create(**kw)
        assert rc != 0 and msg in err, (kw, err)
    with pytest.raises(_lib.EngineError, match="expects 5 device args"):
        base(0, 1, np.array([0, mesh.layers], dtype=np.int32), None, [S.coordinates.device_ptr] * 3, None, None,
             [S.cell_node_map.device_ptr] * 3, None, _lib.LOC_DEVICE, False, False)
    with pytest.raises(_lib.EngineError, match="host-pointer"):
        base(0, 1, np.array([0, mesh.layers], dtype=np.int32), None, [S.coordinates.device_ptr] * 5, [8] * 5,
             [0] * 5, [S.cell_node_map.device_ptr] * 3, [8] * 3, _lib.LOC_HOST, False, False)
    with pytest.raises(ValueError, match="indefinite"):
        solve(F, F.dat(), F.dat(), (), {"ksp_type": "cg"})
    with pytest.raises(NotImplementedError, match="ksp_monitor"):
        solve(F, F.dat(), F.dat(), (), {"ksp_monitor": None})
