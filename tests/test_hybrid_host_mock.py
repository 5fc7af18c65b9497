"""Host logic of the hybridised mixed Poisson solver on the CPU: a mock engine that emulates
FDB_FORM_MIXED_POISSON_HYBRID and _RECONSTRUCT from the ABI arrays alone, with the dense oracle
(tests/_hybrid_oracle.py), runs HybridizationPC (forward, trace_solve, backward) and ``solve`` with "preonly" and
"gmres" against scipy, and every refusal of the options.  The generic-path statement of the condensation runs through
the host build of its generated wrapper and is checked against the oracle.  The device code itself is what `-m gpu`
checks (tests/test_hybrid_gpu.py)."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import _hybrid_oracle as ho
import _mixed_poisson_oracle as mo
import _mock_engine as me
from firedrake_b200 import _lib
from firedrake_b200.utility_meshes import ExtrudedHexMesh
from test_mixed_poisson_host_mock import MixedPoissonMockEngine

HYBRID = {"mat_type": "matfree", "ksp_type": "preonly", "pc_type": "python",
          "pc_python_type": "firedrake.HybridizationPC",
          "hybridization": {"ksp_type": "cg", "pc_type": "jacobi", "ksp_rtol": 1e-13, "ksp_max_it": 5000}}


class HybridMockEngine(MixedPoissonMockEngine):
    """The mixed Poisson mock plus the two hybrid forms on extruded hexes, device location, and
    fdb_mat_get_diagonal.  Each cell's saddle system is solved densely with the oracle's element matrices."""

    def fdb_kernel_create_mixed(self, desc, space2, out):
        d, s2 = me._obj(desc), me._obj(space2)
        if d.form not in (_lib.FORM_MIXED_POISSON_HYBRID, _lib.FORM_MIXED_POISSON_RECONSTRUCT):
            return super().fdb_kernel_create_mixed(desc, space2, out)
        k = d.degree
        if d.cell != _lib.CELL_HEX_EXTRUDED or k not in (2, 3) or s2.degree != k - 1:
            return self._fail("mock engine: the hybrid forms are k = 2..3 on extruded hexes")
        nf, ns = 6 * k * k, 3 * k * k * (k + 1)
        off0 = np.array(d.offset0[:nf + ns], dtype=np.int64)
        self._next += 1
        self.kernels[self._next] = dict(
            kind="hybrid", k=k, rank=d.rank, reconstruct=d.form == _lib.FORM_MIXED_POISSON_RECONSTRUCT,
            alpha=d.alpha, off_t=off0[:nf], off_s=off0[nf:], off_c=np.array(d.offset1[:8], dtype=np.int64),
            off_u=np.array(s2.offset[:k ** 3], dtype=np.int64))
        me._obj(out).value = self._next
        return 0

    def fdb_mat_get_diagonal(self, h, d):
        m = self.mats[me._addr(h)]
        out = me._view(d, m.nrows)
        for r in range(m.nrows):
            cols = m.colidx[m.rowptr[r]:m.rowptr[r + 1]]
            j = np.searchsorted(cols, r)
            out[r] = m.vals[m.rowptr[r] + j] if j < len(cols) and cols[j] == r else 0.0
        return 0

    def fdb_kernel_call(self, h, ca):
        kk = self.kernels[me._addr(h)]
        if kk["kind"] != "hybrid":
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        self.launches += 1
        k, nlay = kk["k"], a.layers[1] - 1
        want = 2 if kk["rank"] == 2 else (7 if kk["reconstruct"] else 5)
        want_maps = 2 if kk["rank"] == 2 else 4
        if a.location != _lib.LOC_DEVICE or a.nargs != want or a.nmaps != want_maps:
            return self._fail(f"mock engine: the hybrid form expects {want} device args and {want_maps} maps")
        nf, ns, nu = 6 * k * k, 3 * k * k * (k + 1), k ** 3
        lay = np.arange(nlay)

        def rows(slot, arity, off):
            m = me._view(a.maps[slot], a.end * arity, np.int32).reshape(a.end, arity).astype(np.int64)
            return (m[:, None, :] + lay[None, :, None] * off[None, None, :]).reshape(-1, arity)

        ft = rows(0 if not kk["reconstruct"] else 2, nf, kk["off_t"])
        fc = rows(1, 8, kk["off_c"])
        X = me._view(a.args[1], (int(fc.max()) + 1) * 3).reshape(-1, 3)
        C = ho.trace_coupling(k)
        if kk["rank"] == 2:
            m = self.mats[a.args[0]]
            Ch = np.hstack([C, np.zeros((nf, nu))])
            for c in range(len(ft)):
                HK = Ch @ np.linalg.solve(ho.local_saddle(k, X[fc[c]], kk["alpha"]), Ch.T)
                for i, gi in enumerate(ft[c]):
                    r = m.row_lg[gi] if m.row_lg is not None else gi
                    if r < 0:
                        continue
                    cols = m.colidx[m.rowptr[r]:m.rowptr[r + 1]]
                    for j, gj in enumerate(ft[c]):
                        cc = m.col_lg[gj] if m.col_lg is not None else gj
                        if cc >= 0:
                            m.vals[m.rowptr[r] + np.searchsorted(cols, cc)] += HK[i, j]
            return 0
        fs = rows(2 if not kk["reconstruct"] else 0, ns, kk["off_s"])
        fq = rows(3, nu, kk["off_u"])
        nT, nS, nQ = int(ft.max()) + 1, int(fs.max()) + 1, int(fq.max()) + 1
        if kk["reconstruct"]:
            ys, lam, f0, w, yu, f1 = (me._view(a.args[i], n) for i, n in
                                      ((0, nS), (2, nT), (3, nS), (4, nS), (5, nQ), (6, nQ)))
        else:
            r, f0, w, f1 = (me._view(a.args[i], n) for i, n in ((0, nT), (2, nS), (3, nS), (4, nQ)))
        for c in range(len(ft)):
            g = np.concatenate([w[fs[c]] * f0[fs[c]], f1[fq[c]]])
            if kk["reconstruct"]:
                g[:ns] -= C.T @ lam[ft[c]]
            x = np.linalg.solve(ho.local_saddle(k, X[fc[c]], kk["alpha"]), g)
            if kk["reconstruct"]:
                ys[fs[c]] += w[fs[c]] * x[:ns]
                yu[fq[c]] += x[ns:]
            else:
                r[ft[c]] += C @ x[:ns]
        return 0


@pytest.fixture()
def mock(oracle):
    inst = me.install(oracle)
    inst.engine = HybridMockEngine(oracle)
    with inst as eng:
        yield eng


def _spaces(k=2, n=(3, 2, 3), warp=0.05, permute_seed=1, alpha=1.3):
    from firedrake_b200.assemble import FunctionSpace, MixedPoisson
    mesh = ExtrudedHexMesh(*n, warp=warp, permute_seed=permute_seed)
    S, Q = FunctionSpace(mesh, k, family="NCF"), FunctionSpace(mesh, k - 1, family="DQ")
    return mesh, S, Q, MixedPoisson(S, Q, alpha)


def _load(S, Q, F, seed=0):
    rng = np.random.default_rng(seed)
    return F.dat(rng.standard_normal(S.node_count), rng.standard_normal(Q.node_count))


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


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def test_generic_path_host_build_matches_the_oracle(mock):
    """``hybridization_kernel(2)`` through the host build of its generated wrapper gives the oracle's H, with the
    natural faces masked and a unit diagonal; k = 3 is refused by name."""
    from firedrake_b200.assemble import (DirichletBC, HybridizationPC, assemble_hybrid_trace_generic,
                                         hybridization_kernel)
    mesh, S, Q, F = _spaces(2)
    flux = (2, "bottom")
    pc = HybridizationPC(F, [DirichletBC(S, 0.0, s) for s in flux])
    T = pc.trace
    H_ref = ho.trace_matrix(mesh, S.V, Q.V, T.V, F.alpha)
    nat = ho.natural_nodes(T.V, flux)
    H_ref[nat, :] = 0.0
    H_ref[:, nat] = 0.0
    H_ref[nat, nat] = 1.0
    assert _rel(assemble_hybrid_trace_generic(pc).values, H_ref) < 1e-12
    assert _rel(pc.mat.values, H_ref) < 1e-12
    with pytest.raises(NotImplementedError, match="stack"):
        hybridization_kernel(3)


@pytest.mark.parametrize("k", [2, 3])
def test_forward_trace_solve_backward_match_the_oracle(mock, k):
    from firedrake_b200.assemble import DirichletBC, HybridizationPC
    mesh, S, Q, F = _spaces(k, n=(2, 2, 2))
    flux = (1, "top")
    bcs = [DirichletBC(S, 0.0, s) for s in flux]
    pc = HybridizationPC(F, bcs)
    L = _load(S, Q, F, k)
    for bc in bcs:
        bc.zero(L[0])
    L0, L1 = L[0].data_ro.copy(), L[1].data_ro.copy()
    r = pc.forward(L)
    r_ref = ho.eliminate(mesh, S.V, Q.V, pc.trace.V, F.alpha, L0, L1)
    r_ref[ho.natural_nodes(pc.trace.V, flux)] = 0.0
    assert _rel(r.data_ro, r_ref) < 1e-12
    lam = pc.trace.dat()
    its, hist = pc.trace_solve(r, lam, rtol=1e-13)
    assert hist[-1] <= 1e-13 * hist[0]
    s_ref, u_ref, lam_ref = ho.hybrid_solve(mesh, S.V, Q.V, pc.trace.V, F.alpha, L0, L1, flux)
    assert _rel(lam.data_ro, lam_ref) < 1e-10
    up = pc.backward(lam, L, F.dat())
    assert _rel(up[0].data_ro, s_ref) < 1e-10
    assert _rel(up[1].data_ro, u_ref) < 1e-10


@pytest.mark.parametrize("ksp", ["preonly", "gmres"])
def test_solve_with_natural_data_matches_scipy(mock, ksp):
    from firedrake_b200.assemble import solve
    mesh, S, Q, F = _spaces()
    L = _load(S, Q, F, 1)
    up = F.dat()
    its, hist = solve(F, L, up, (), {**HYBRID, "ksp_type": ksp, "ksp_rtol": 1e-11})
    if ksp == "gmres":
        assert its <= 2
    s_ref, u_ref = _scipy(mesh, S, Q, F, L, (), False)
    assert _rel(up[0].data_ro, s_ref) < 1e-8
    assert _rel(up[1].data_ro, u_ref) < 1e-8


@pytest.mark.parametrize("ksp", ["preonly", "gmres"])
def test_solve_with_flux_conditions_and_constant_nullspace(mock, ksp):
    from firedrake_b200.assemble import DirichletBC, solve
    mesh, S, Q, F = _spaces()
    bcs = [DirichletBC(S, 0.0, s) for s in ho.SUBS]
    L = _load(S, Q, F, 2)
    up = F.dat()
    flat = {"mat_type": "matfree", "ksp_type": ksp, "ksp_rtol": 1e-10, "pc_type": "python",
            "pc_python_type": "firedrake.HybridizationPC", "hybridization_ksp_type": "cg",
            "hybridization_pc_type": "jacobi", "hybridization_ksp_rtol": 1e-12}
    solve(F, L, up, bcs, flat, nullspace="constant")
    s_ref, u_ref = _scipy(mesh, S, Q, F, L, bcs, True)
    assert _rel(up[0].data_ro, s_ref) < 1e-8
    assert _rel(up[1].data_ro, u_ref) < 1e-8
    assert abs(up[1].data_ro.mean()) < 1e-12 * np.abs(u_ref).max()
    assert np.all(up[0].data_ro[np.concatenate([bc.nodes for bc in bcs])] == 0.0)


@pytest.mark.parametrize("opts, exc, msg", [
    ({"hybridization": {"pc_type": "lu"}}, NotImplementedError, "hybridization_pc_type 'lu'"),
    ({"hybridization": {"pc_type": "gamg"}}, NotImplementedError, "hybridization_pc_type 'gamg'"),
    ({"hybridization": {"pc_type": "hypre"}}, NotImplementedError, "hybridization_pc_type 'hypre'"),
    ({"hybridization": {"pc_type": "mg"}}, NotImplementedError, "hybridization_pc_type 'mg'"),
    ({"hybridization": {"pc_type": "python"}}, NotImplementedError, "hybridization_pc_type 'python'"),
    ({"hybridization": {"ksp_type": "preonly"}}, NotImplementedError, "direct solver"),
    ({"hybridization": {"ksp_type": "gmres"}}, NotImplementedError, "hybridization_ksp_type 'gmres'"),
    ({"hybridization": {"mat_type": "matfree"}}, NotImplementedError, "hybridization_mat_type 'matfree'"),
    ({"hybridization": {"localsolve": {"ksp_type": "preonly"}}}, NotImplementedError, "localsolve"),
    ({"pc_python_type": "firedrake.GTMGPC"}, NotImplementedError, "pc_python_type 'firedrake.GTMGPC'"),
    ({"pc_python_type": "drop"}, NotImplementedError, "needs pc_python_type"),
    ({"pc_type": "fieldsplit"}, NotImplementedError, "pc_type 'fieldsplit'"),
    ({"mat_type": "aij"}, NotImplementedError, "mat_type 'aij'"),
    ({"ksp_type": "cg"}, ValueError, "indefinite"),
    ({"ksp_type": "minres"}, NotImplementedError, "ksp_type 'minres'"),
    ({"ksp_monitor": None}, NotImplementedError, "ksp_monitor"),
])
def test_solver_option_refusals(mock, opts, exc, msg):
    from firedrake_b200.assemble import solve
    _, S, Q, F = _spaces(n=(1, 1, 1))
    sp = {**HYBRID, **opts}
    sp = {k: v for k, v in sp.items() if v != "drop"}
    with pytest.raises(exc, match=msg):
        solve(F, F.dat(), F.dat(), (), sp)


def test_other_refusals(mock):
    from firedrake_b200.assemble import DirichletBC, Form, FunctionSpace, HybridizationPC, MixedPoisson, solve
    mesh, S, Q, F = _spaces(n=(1, 1, 1))
    with pytest.raises(NotImplementedError, match="pc_type 'python' needs pc_python_type"):
        solve(F, F.dat(), F.dat(), (), {"pc_type": "python"})
    with pytest.raises(NotImplementedError, match="hybridization options need pc_type 'python'"):
        solve(F, F.dat(), F.dat(), (), {"hybridization_ksp_type": "cg"})
    with pytest.raises(NotImplementedError, match="nullspace 'pressure'"):
        solve(F, F.dat(), F.dat(), (), HYBRID, nullspace="pressure")
    with pytest.raises(NotImplementedError, match="ksp_type 'preonly'"):
        solve(F, F.dat(), F.dat(), (), {"ksp_type": "preonly"})
    m4 = ExtrudedHexMesh(1, 1, 1)
    with pytest.raises(NotImplementedError, match="shared memory"):
        HybridizationPC(MixedPoisson(FunctionSpace(m4, 4, family="NCF"), FunctionSpace(m4, 3, family="DQ")))
    T = FunctionSpace(mesh, 1, family="HDiv Trace")
    with pytest.raises(NotImplementedError, match="does not take HDiv Trace spaces"):
        Form(T, 1.0, 0.0)
    with pytest.raises(NotImplementedError, match="does not take HDiv Trace spaces"):
        DirichletBC(T, 0.0, 1)
    with pytest.raises(ValueError, match="NCF_k"):
        MixedPoisson(T, Q)
    with pytest.raises(ValueError, match="HDiv Trace degree 4"):
        FunctionSpace(mesh, 4, family="HDiv Trace")
    with pytest.raises(ValueError, match="family 'RT'"):
        FunctionSpace(mesh, 1, family="RT")
    with pytest.raises(NotImplementedError, match="partitioned HDiv Trace"):
        FunctionSpace(mesh, 1, family="HDiv Trace", partition=object())
