"""GTMG for the hybridised trace system on the H100: the CG1 <-> trace transfer kernels (FDB_FORM_TRACE_PROLONG /
_RESTRICT) against the oracle's P (tests/_gtmg_oracle.py), on extruded and native hexes, their adjointness and
bit-reproducibility, the generic-path statement, and GTMG-preconditioned hybrid solves against the Jacobi-CG ones."""
import ctypes as C

import numpy as np
import pytest

import _gtmg_oracle as go
import _hybrid_oracle as ho
from firedrake_b200 import _lib, op2
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu


def _spaces(k, n=(4, 3, 5), warp=0.05, permute_seed=2, alpha=1.3):
    from firedrake_b200.assemble import FunctionSpace, MixedPoisson
    mesh = ExtrudedHexMesh(*n, warp=warp, permute_seed=permute_seed)
    S, Q = FunctionSpace(mesh, k, family="NCF"), FunctionSpace(mesh, k - 1, family="DQ")
    return mesh, S, Q, MixedPoisson(S, Q, alpha)


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _native(tt, c, lam, scatter="atomic"):
    """prolong and restrict on native hexes: one map row per cell (the extruded maps with the layer loop expanded)."""
    mesh, T, V1 = tt.Vc.mesh, tt.Vf, tt.Vc
    cells = op2.Set(mesh.num_cells)
    mt = op2.Map(cells, T.node_set, T.V.arity, T.V.full_cell_node_list())
    mv = op2.Map(cells, V1.node_set, 8, V1.V.full_cell_node_list())
    kw = dict(degree=tt.k - 1, coarse_degree=1)
    gp = op2.GlobalKernel(op2.Kernel("trace_prolong", **kw), [mt, mv])
    gr = op2.GlobalKernel(op2.Kernel("trace_restrict", **kw), [mv, mt], scatter=scatter)
    out_t = T.dat()
    op2.Parloop(gp, cells, [out_t(op2.WRITE, mt), V1.dat(c.copy())(op2.READ, mv)])()
    out_c = V1.dat()
    out_c.zero()
    out_c.device_ptr
    op2.Parloop(gr, cells, [out_c(op2.INC, mv), T.dat(lam.copy())(op2.READ, mt), tt.weight(op2.READ, mt)])()
    return out_t.data_ro.copy(), out_c.data_ro.copy()


@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("extruded", [True, False])
def test_transfers_match_the_oracle(k, extruded):
    """P c and P^T lambda against the oracle to 1e-14 on a warped, permuted mesh, atomic and coloured; the adjoint
    identity <P c, f> = <c, P^T f> to 1e-13; the hand-written kernels against the generic path."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import HybridizationPC
    mesh, S, Q, F = _spaces(k)
    pc = HybridizationPC(F)
    rng = np.random.default_rng(10 + k)
    for scatter in ("atomic", "coloured"):
        tt = mg.TraceTransfer(pc, scatter=scatter)
        T, V1 = pc.trace, tt.Vc
        P = go.prolongation(T.V, V1.V)
        c, lam = rng.standard_normal(V1.node_count), rng.standard_normal(T.node_count)
        if extruded:
            pt = tt.prolong(V1.dat(c.copy()), T.dat()).data_ro.copy()
            rc = tt.restrict(T.dat(lam.copy()), V1.dat()).data_ro.copy()
        else:
            pt, rc = _native(tt, c, lam, scatter)
        assert _rel(pt, P @ c) < 1e-14
        assert _rel(rc, P.T @ lam) < 1e-14
        assert abs(pt @ lam - c @ rc) < 1e-13 * np.abs(pt).sum() * np.abs(lam).max()
    gp = tt.prolong_generic(V1.dat(c.copy()), T.dat()).data_ro
    gr = tt.restrict_generic(T.dat(lam.copy()), V1.dat()).data_ro
    assert _rel(pt, gp) < 1e-14
    assert _rel(rc, gr) < 1e-14


def test_repeats_are_bitwise_identical():
    """The prolongation (both writers of a shared face store the same bits) and the coloured restriction give
    bitwise the same result on every repeat."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import HybridizationPC
    mesh, S, Q, F = _spaces(3, n=(6, 5, 6))
    pc = HybridizationPC(F)
    tt = mg.TraceTransfer(pc, scatter="coloured")
    rng = np.random.default_rng(4)
    c = tt.Vc.dat(rng.standard_normal(tt.Vc.node_count))
    lam = pc.trace.dat(rng.standard_normal(pc.trace.node_count))
    a = [tt.prolong(c, pc.trace.dat()).data_ro.copy() for _ in range(3)]
    b = [tt.restrict(lam, tt.Vc.dat()).data_ro.copy() for _ in range(3)]
    assert all(x.tobytes() == a[0].tobytes() for x in a)
    assert all(x.tobytes() == b[0].tobytes() for x in b)


def _problem(mesh, k=2, flux=(), seed=0):
    from firedrake_b200.assemble import DirichletBC, FunctionSpace, MixedPoisson
    S, Q = FunctionSpace(mesh, k, family="NCF"), FunctionSpace(mesh, k - 1, family="DQ")
    F = MixedPoisson(S, Q, 1.0)
    rng = np.random.default_rng(seed)
    L = F.dat(rng.standard_normal(S.node_count), rng.standard_normal(Q.node_count))
    return S, Q, F, L, [DirichletBC(S, 0.0, s) for s in flux]


def _opts(coarse, ksp="preonly", rtol=1e-10):
    gt = {"mg_levels": {"ksp_type": "chebyshev", "pc_type": "jacobi", "ksp_max_it": 3},
          "mg_coarse": {"ksp_type": "cg", "pc_type": "jacobi", "ksp_rtol": 1e-3} if coarse == "cg"
          else {"ksp_type": "preonly", "pc_type": "mg"}}
    return {"mat_type": "matfree", "ksp_type": ksp, "ksp_rtol": 1e-9, "pc_type": "python",
            "pc_python_type": "firedrake.HybridizationPC",
            "hybridization": {"ksp_type": "cg", "ksp_rtol": rtol, "pc_type": "python",
                              "pc_python_type": "firedrake.GTMGPC", "gt": gt}}


JACOBI = {"mat_type": "matfree", "ksp_type": "preonly", "pc_type": "python",
          "pc_python_type": "firedrake.HybridizationPC",
          "hybridization": {"ksp_type": "cg", "pc_type": "jacobi", "ksp_rtol": 1e-10, "ksp_max_it": 20000}}


def _solve(n, k, coarse, flux=(), ns=None, ksp="preonly"):
    from firedrake_b200 import mg
    from firedrake_b200.assemble import solve
    hier = mg.MeshHierarchy(n // 4, n // 4, n // 4, 2) if coarse == "mg" else None
    mesh = hier[len(hier) - 1] if hier is not None else ExtrudedHexMesh(n, n, n)
    S, Q, F, L, bcs = _problem(mesh, k, flux)
    up, uj = F.dat(), F.dat()
    its, hist = solve(F, L, up, bcs, _opts(coarse, ksp), hierarchy=hier, nullspace=ns)
    itj, _ = solve(F, L, uj, bcs, JACOBI, nullspace=ns)
    assert _rel(up[0].data_ro, uj[0].data_ro) < 1e-8
    assert _rel(up[1].data_ro, uj[1].data_ro) < 1e-8
    return its, itj


@pytest.mark.parametrize("coarse", ["cg", "mg"])
def test_gtmg_solves_match_jacobi_cg_and_iterations_stay_bounded(coarse):
    """k = 2 at 8^3 and 16^3: the GTMG solve equals the Jacobi-CG hybrid solve to 1e-8; its trace-CG iterations at
    16^3 are at most those at 8^3 + 2, and below the Jacobi-CG count at 16^3."""
    g8, j8 = _solve(8, 2, coarse)
    g16, j16 = _solve(16, 2, coarse)
    assert g16 <= g8 + 2, (g8, g16)
    assert g16 < j16, (g16, j16)


def test_gtmg_k3_and_flux_conditions():
    g, j = _solve(8, 3, "cg", flux=(1, "top"))
    assert g < j, (g, j)


def test_all_flux_with_the_nullspace_and_outer_gmres():
    _solve(8, 2, "cg", flux=ho.SUBS, ns="constant")
    its, _ = _solve(8, 2, "cg", ksp="gmres")
    assert its <= 2


def _create(form, degree=1, s2degree=1, rank=1, cdim=1):
    lib = _lib.lib()
    d = _lib.KernelDesc()
    d.form, d.rank, d.cell, d.integral = form, rank, _lib.CELL_HEX, 0
    d.degree, d.nq, d.cdim, d.scatter = degree, degree + 1, cdim, 0
    s2 = _lib.Space2Desc()
    s2.degree = s2degree
    h = C.c_void_p()
    rc = lib.fdb_kernel_create_mixed(C.byref(d), C.byref(s2), C.byref(h))
    if rc == 0:
        lib.fdb_kernel_destroy(h)
    return rc, lib.fdb_last_error().decode()


def test_creation_and_call_refusals():
    from firedrake_b200 import mg
    from firedrake_b200.assemble import HybridizationPC
    TP, TR = _lib.FORM_TRACE_PROLONG, _lib.FORM_TRACE_RESTRICT
    assert _create(TP)[0] == 0 and _create(TR, degree=2)[0] == 0
    for args, msg in [((TP, 3), "trace degree 3 not instantiated"), ((TR, 0), "trace degree 0"),
                      ((TP, 1, 2), "must be CG1"), ((TR, 1, 1, 2), "no rank-2"), ((TP, 1, 1, 1, 3), "scalar")]:
        rc, err = _create(*args)
        assert rc != 0 and msg in err, (args, err)
    lib = _lib.lib()
    d = _lib.KernelDesc()
    d.form, d.rank, d.cell, d.degree, d.nq, d.cdim = TP, 1, _lib.CELL_HEX, 1, 2, 1
    h = C.c_void_p()
    assert lib.fdb_kernel_create(C.byref(d), C.byref(h)) != 0
    assert "fdb_kernel_create_mixed" in lib.fdb_last_error().decode()
    mesh, S, Q, F = _spaces(2, n=(2, 2, 2))
    pc = HybridizationPC(F)
    tt = mg.TraceTransfer(pc)
    with pytest.raises(_lib.EngineError, match="host-pointer"):
        op2.Parloop(tt._gk["trace_prolong"], tt.cell_set, [pc.trace.dat()(op2.WRITE, tt.tmap),
                                                           tt.Vc.dat()(op2.READ, tt.cmap)], location="host")()
