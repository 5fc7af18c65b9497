"""Hybridised mixed Poisson on the H100: the condensation, elimination and reconstruction kernels
(FDB_FORM_MIXED_POISSON_HYBRID / _RECONSTRUCT) against the dense oracle (tests/_hybrid_oracle.py), their
bit-reproducibility, and the HybridizationPC solves against scipy and the Schur fieldsplit solve."""
import numpy as np
import pytest

import _hybrid_oracle as ho
import _mixed_poisson_oracle as mo
from firedrake_b200 import _lib, op2
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

HYBRID = {"mat_type": "matfree", "ksp_type": "preonly", "pc_type": "python",
          "pc_python_type": "firedrake.HybridizationPC",
          "hybridization": {"ksp_type": "cg", "pc_type": "jacobi", "ksp_rtol": 1e-12, "ksp_max_it": 20000}}


def _spaces(k, n=3, warp=0.05, permute_seed=1, alpha=1.4):
    from firedrake_b200.assemble import FunctionSpace, MixedPoisson
    mesh = ExtrudedHexMesh(n, n + 1, n, warp=warp, permute_seed=permute_seed)
    S, Q = FunctionSpace(mesh, k, family="NCF"), FunctionSpace(mesh, k - 1, family="DQ")
    return mesh, S, Q, MixedPoisson(S, Q, alpha)


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _masked(H, nat):
    H = H.copy()
    H[nat, :] = 0.0
    H[:, nat] = 0.0
    H[nat, nat] = 1.0
    return H


def _native_run(pc, S, Q, mesh, flux_subs, L0, L1, lam):
    """The three kernels on native hexes: one map row per cell (the extruded maps with the layer loop expanded)."""
    F, T = pc.form, pc.trace
    cells = op2.Set(mesh.num_cells)
    mt = op2.Map(cells, T.node_set, T.V.arity, T.V.full_cell_node_list())
    mc = op2.Map(cells, S.vertex_set, 8, mesh.coord_space.full_cell_node_list())
    ms = op2.Map(cells, S.node_set, S.V.arity, S.V.full_cell_node_list())
    mq = op2.Map(cells, Q.node_set, Q.V.arity, Q.V.full_cell_node_list())
    maps = [mt, mc, ms, mq]
    k = S.degree
    gk = {r: op2.GlobalKernel(op2.Kernel("mixed_poisson_hybrid", degree=k, alpha=F.alpha, rank=r), maps)
          for r in (1, 2)}
    gkr = op2.GlobalKernel(op2.Kernel("mixed_poisson_reconstruct", degree=k, alpha=F.alpha), maps)
    mat = op2.Mat(op2.Sparsity((T.node_set, T.node_set), [(mt, mt, None)]))
    mat.zero()
    lg = np.arange(T.node_count, dtype=np.int32)
    lg[pc.natural_nodes] = -1
    op2.Parloop(gk[2], cells, [mat(op2.INC, (mt, mt), lgmaps=(lg, lg)), S.coordinates(op2.READ, mc)])()
    mat.set_local_diagonal_entries(pc.natural_nodes, 1.0)
    f0, f1 = S.dat(L0.copy()), Q.dat(L1.copy())
    r = T.dat()
    r.zero()
    r.device_ptr
    op2.Parloop(gk[1], cells, [r(op2.INC, mt), S.coordinates(op2.READ, mc), f0(op2.READ, ms),
                               pc.w(op2.READ, ms), f1(op2.READ, mq)])()
    ys, yu = S.dat(), Q.dat()
    for d in (ys, yu):
        d.zero()
        d.device_ptr
    op2.Parloop(gkr, cells, [ys(op2.INC, ms), S.coordinates(op2.READ, mc), T.dat(lam.copy())(op2.READ, mt),
                             f0(op2.READ, ms), pc.w(op2.READ, ms), yu(op2.INC, mq), f1(op2.READ, mq)])()
    return mat.values, r.data_ro.copy(), ys.data_ro.copy(), yu.data_ro.copy()


@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("extruded", [True, False])
def test_kernels_match_oracle(k, extruded):
    """H's CSR values (natural faces masked, unit diagonal), r and the reconstructed (sigma, u) against the dense
    oracle to 1e-12 relative on a warped, permuted mesh with flux conditions on two sides."""
    from firedrake_b200.assemble import DirichletBC, HybridizationPC
    mesh, S, Q, F = _spaces(k)
    flux = (1, "top")
    pc = HybridizationPC(F, [DirichletBC(S, 0.0, s) for s in flux])
    T = pc.trace
    rng = np.random.default_rng(k)
    L0, L1 = rng.standard_normal(S.node_count), rng.standard_normal(Q.node_count)
    lam = rng.standard_normal(T.node_count)
    nat = ho.natural_nodes(T.V, flux)
    H_ref = _masked(ho.trace_matrix(mesh, S.V, Q.V, T.V, F.alpha), nat)
    r_ref = ho.eliminate(mesh, S.V, Q.V, T.V, F.alpha, L0, L1)
    r_ref[nat] = 0.0
    s_ref, u_ref = ho.reconstruct(mesh, S.V, Q.V, T.V, F.alpha, lam, L0, L1)
    if extruded:
        H = pc.mat.values
        r = pc.forward(F.dat(L0.copy(), L1.copy())).data_ro.copy()
        up = pc.backward(T.dat(lam.copy()), F.dat(L0.copy(), L1.copy()), F.dat())
        ys, yu = up[0].data_ro.copy(), up[1].data_ro.copy()
    else:
        H, r, ys, yu = _native_run(pc, S, Q, mesh, flux, L0, L1, lam)
        r[nat] = 0.0
    assert _rel(H, H_ref) < 1e-12
    assert _rel(r, r_ref) < 1e-12
    assert _rel(ys, s_ref) < 1e-12
    assert _rel(yu, u_ref) < 1e-12


def test_two_condensations_are_bitwise_identical():
    from firedrake_b200.assemble import HybridizationPC
    mesh, S, Q, F = _spaces(3, n=4)
    pc = HybridizationPC(F)
    v1 = pc.mat.csr()[2].copy()
    pc.assemble()
    v2 = pc.mat.csr()[2].copy()
    assert v1.tobytes() == v2.tobytes()
    rng = np.random.default_rng(3)
    L = F.dat(rng.standard_normal(S.node_count), rng.standard_normal(Q.node_count))
    r1 = pc.forward(L).data_ro.copy()
    r2 = pc.forward(L).data_ro.copy()
    assert r1.tobytes() == r2.tobytes()
    lam = pc.trace.dat(rng.standard_normal(pc.trace.node_count))
    a = [d.data_ro.copy() for d in pc.backward(lam, L, F.dat())]
    b = [d.data_ro.copy() for d in pc.backward(lam, L, F.dat())]
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _problem(n, k=2, warp=0.0, flux_bcs=False):
    from firedrake_b200.assemble import DirichletBC, assemble, mass, mixed_dirichlet_load
    mesh, S, Q, F = _spaces(k, n=n, warp=warp, permute_seed=None, alpha=1.0)
    X = Q.V.dof_coordinates()
    f = Q.dat(3 * np.pi ** 2 * np.sin(np.pi * X[:, 0]) * np.sin(np.pi * X[:, 1]) * np.sin(np.pi * X[:, 2])
              + (np.cos(2 * np.pi * X[:, 0]) if flux_bcs else 0.0))
    L = F.dat()
    L.zero()
    L[1].axpy(-1.0, assemble(mass(Q), u=f))
    bcs = [DirichletBC(S, 0.0, s) for s in (1, 2, 3, 4, "bottom", "top")] if flux_bcs else []
    if not flux_bcs:
        g = op2.Dat(op2.DataSet(S.vertex_set, 1), mesh.coordinates[:, 0].copy())
        mixed_dirichlet_load(F, g, 2, tensor=L[0])
    return mesh, S, Q, F, L, bcs


def _scipy(mesh, S, Q, F, L, bcs, nullspace):
    import scipy.sparse.linalg as spla
    M, B = mo.global_matrices(mesh, S.V, Q.V, F.alpha)
    rows = np.unique(np.concatenate([bc.nodes for bc in bcs])) if bcs else np.zeros(0, dtype=int)
    rhs = np.concatenate([L[0].data_ro, L[1].data_ro])
    rhs[rows] = 0.0
    pin = [S.node_count] if nullspace else []
    if nullspace:
        rhs[S.node_count:] -= rhs[S.node_count:].mean()
        rhs[pin] = 0.0
    x = spla.spsolve(mo.constrained(mo.saddle(M, B), np.concatenate([rows, pin]).astype(int)).tocsc(), rhs)
    if nullspace:
        x[S.node_count:] -= x[S.node_count:].mean()
    return x[:S.node_count], x[S.node_count:]


SCHUR = {"ksp_type": "gmres", "ksp_rtol": 1e-10, "pc_type": "fieldsplit", "pc_fieldsplit_type": "schur",
         "pc_fieldsplit_schur_fact_type": "full", "pc_fieldsplit_schur_precondition": "selfp",
         "fieldsplit_0_ksp_type": "preonly", "fieldsplit_0_pc_type": "jacobi", "fieldsplit_1_ksp_type": "cg",
         "fieldsplit_1_pc_type": "jacobi", "fieldsplit_1_ksp_rtol": 1e-5, "ksp_max_it": 3000}


@pytest.mark.parametrize("flux_bcs", [False, True])
def test_solve_matches_scipy_and_the_schur_solve(flux_bcs):
    """8^3, k = 2: the hybridised solve ("preonly") matches scipy and the "full" Schur fieldsplit solve to 1e-8;
    with flux conditions on the whole boundary and the constant nullspace as well."""
    from firedrake_b200.assemble import solve
    mesh, S, Q, F, L, bcs = _problem(8, warp=0.03 if flux_bcs else 0.0, flux_bcs=flux_bcs)
    ns = "constant" if flux_bcs else None
    up = F.dat()
    rtol = 1e-10 if flux_bcs else 1e-12
    its, hist = solve(F, L, up, bcs, {**HYBRID, "hybridization": {**HYBRID["hybridization"], "ksp_rtol": rtol}},
                      nullspace=ns)
    assert hist[-1] <= rtol * hist[0]
    s_ref, u_ref = _scipy(mesh, S, Q, F, L, bcs, flux_bcs)
    assert _rel(up[0].data_ro, s_ref) < 1e-8
    assert _rel(up[1].data_ro, u_ref) < 1e-8
    us = F.dat()
    solve(F, L, us, bcs, SCHUR, nullspace=ns)
    assert _rel(up[0].data_ro, us[0].data_ro) < 1e-8
    assert _rel(up[1].data_ro, us[1].data_ro) < 1e-8
    if flux_bcs:
        assert abs(up[1].data_ro.mean()) < 1e-12 * np.abs(u_ref).max()
        assert np.all(up[0].data_ro[np.concatenate([bc.nodes for bc in bcs])] == 0.0)


@pytest.mark.parametrize("k", [2, 3])
def test_gmres_with_hybridization_pc_converges_at_once(k):
    """Outer GMRES right-preconditioned by HybridizationPC with a 1e-12 trace solve: at most 2 iterations."""
    from firedrake_b200.assemble import solve
    mesh, S, Q, F, L, bcs = _problem(6, k=k)
    up = F.dat()
    its, hist = solve(F, L, up, bcs, {**HYBRID, "ksp_type": "gmres", "ksp_rtol": 1e-9})
    assert its <= 2, hist
    s_ref, u_ref = _scipy(mesh, S, Q, F, L, bcs, False)
    assert _rel(up[0].data_ro, s_ref) < 1e-8
    assert _rel(up[1].data_ro, u_ref) < 1e-8


def test_flat_options_and_pc_none():
    from firedrake_b200.assemble import solve
    mesh, S, Q, F, L, bcs = _problem(4)
    up = F.dat()
    flat = {"mat_type": "matfree", "ksp_type": "preonly", "pc_type": "python",
            "pc_python_type": "firedrake.HybridizationPC", "hybridization_ksp_type": "cg",
            "hybridization_pc_type": "none", "hybridization_ksp_rtol": 1e-12, "hybridization_mat_type": "aij"}
    solve(F, L, up, bcs, flat)
    s_ref, u_ref = _scipy(mesh, S, Q, F, L, bcs, False)
    assert _rel(up[0].data_ro, s_ref) < 1e-8
    assert _rel(up[1].data_ro, u_ref) < 1e-8


def _create(form, rank=1, degree=2, scatter=0):
    import ctypes as C
    from firedrake_b200.fiat_lite import interval_element
    lib = _lib.lib()
    d = _lib.KernelDesc()
    el = interval_element(degree)
    d.form, d.rank, d.cell, d.integral = form, rank, _lib.CELL_HEX, 0
    d.degree, d.nq, d.cdim, d.scatter = degree, el.nq, 1, scatter
    n = degree + 1
    for q in range(el.nq):
        d.wq[q], d.xq[q] = el.wq[q], el.xq[q]
        for a in range(n):
            d.B[q * n + a], d.D[q * n + a] = el.B[q, a], el.D[q, a]
    s2 = _lib.Space2Desc()
    s2.degree = degree - 1
    h = C.c_void_p()
    rc = lib.fdb_kernel_create_mixed(C.byref(d), C.byref(s2), C.byref(h))
    if rc == 0:
        lib.fdb_kernel_destroy(h)
    return rc, lib.fdb_last_error().decode()


def test_creation_call_and_solver_refusals():
    from firedrake_b200.assemble import FunctionSpace, HybridizationPC, MixedPoisson, assemble, solve
    H, R = _lib.FORM_MIXED_POISSON_HYBRID, _lib.FORM_MIXED_POISSON_RECONSTRUCT
    assert _create(H)[0] == 0 and _create(H, rank=2, degree=3)[0] == 0 and _create(R, degree=3)[0] == 0
    for args, msg in [((H, 1, 4), "shared memory"), ((H, 2, 4), "shared memory"), ((R, 2, 2), "no rank-2"),
                      ((H, 1, 2, 1), "atomic scatter only"), ((H, 1, 5), "outside 2..3")]:
        rc, err = _create(*args)
        assert rc != 0 and msg in err, (args, err)
    rc, err = _create(_lib.FORM_MIXED_POISSON, rank=2)
    assert rc != 0 and "no rank-2" in err
    mesh, S, Q, F = _spaces(2)
    pc = HybridizationPC(F)
    with pytest.raises(_lib.EngineError, match="expects 5 device args"):
        pc._gk[1](0, 1, np.array([0, mesh.layers], dtype=np.int32), None, [S.coordinates.device_ptr] * 3, None,
                  None, [S.cell_node_map.device_ptr] * 4, None, _lib.LOC_DEVICE, False, False)
    with pytest.raises(_lib.EngineError, match="host-pointer"):
        pc._gkr(0, 1, np.array([0, mesh.layers], dtype=np.int32), None, [S.coordinates.device_ptr] * 7, [8] * 7,
                [0] * 7, [S.cell_node_map.device_ptr] * 4, [8] * 4, _lib.LOC_HOST, False, False)
    with pytest.raises(NotImplementedError, match="no assembled matrix"):
        F.kernel(2)
    with pytest.raises(NotImplementedError, match="mat_type 'aij'"):
        assemble(F)
    m4 = ExtrudedHexMesh(1, 1, 1)
    F4 = MixedPoisson(FunctionSpace(m4, 4, family="NCF"), FunctionSpace(m4, 3, family="DQ"))
    with pytest.raises(NotImplementedError, match="shared memory"):
        HybridizationPC(F4)
    FunctionSpace(m4, 3, family="HDiv Trace")
    for opts, exc, msg in [
            ({"hybridization": {"pc_type": "lu"}}, NotImplementedError, "hybridization_pc_type 'lu'"),
            ({"hybridization": {"pc_type": "gamg"}}, NotImplementedError, "hybridization_pc_type 'gamg'"),
            ({"hybridization": {"ksp_type": "preonly"}}, NotImplementedError, "direct solver"),
            ({"hybridization": {"mat_type": "matfree"}}, NotImplementedError, "hybridization_mat_type 'matfree'"),
            ({"hybridization": {"localsolve": {"ksp_type": "preonly"}}}, NotImplementedError, "localsolve"),
            ({"pc_python_type": "firedrake.GTMGPC"}, NotImplementedError, "pc_python_type"),
            ({"ksp_type": "cg"}, ValueError, "indefinite"),
            ({"ksp_type": "minres"}, NotImplementedError, "ksp_type 'minres'")]:
        with pytest.raises(exc, match=msg):
            solve(F, F.dat(), F.dat(), (), {**HYBRID, **opts})
    with pytest.raises(NotImplementedError, match="ksp_type 'preonly'"):
        solve(F, F.dat(), F.dat(), (), {"ksp_type": "preonly"})


def test_generic_path_matches_the_hand_written_trace_matrix():
    """k = 2: the generic wrapper path (hybridization_kernel, one thread per cell, dense Cholesky) gives the
    hand-written H to 1e-12, natural faces masked, on a warped, permuted mesh with flux conditions."""
    from firedrake_b200.assemble import DirichletBC, HybridizationPC, assemble_hybrid_trace_generic
    mesh, S, Q, F = _spaces(2, n=4, permute_seed=3)
    pc = HybridizationPC(F, [DirichletBC(S, 0.0, s) for s in (3, "bottom")])
    Hg = assemble_hybrid_trace_generic(pc)
    a, b = pc.mat.csr()[2], Hg.csr()[2]
    assert _rel(b, a) < 1e-12
