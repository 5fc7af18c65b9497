"""Host logic of the GTMG trace preconditioner on the CPU: a mock engine that emulates FDB_FORM_TRACE_PROLONG and
_RESTRICT from the ABI arrays alone with the oracle's P (tests/_gtmg_oracle.py), on top of the hybridisation mock.
It runs mg.TraceTransfer, the generic-path statement of the transfers through the host build of its generated
wrapper, and ``solve`` with the GTMGPC options on both outer routes against scipy, and checks every refusal of the
options.  The device code itself is what `-m gpu` checks (tests/test_gtmg_gpu.py)."""
import numpy as np
import pytest

import _gtmg_oracle as go
import _hybrid_oracle as ho
import _mock_engine as me
from firedrake_b200 import _lib
from firedrake_b200.fiat_lite import gauss_legendre
from test_hybrid_host_mock import HybridMockEngine, _load, _rel, _scipy, _spaces

GTMG = {"mat_type": "matfree", "ksp_type": "preonly", "pc_type": "python",
        "pc_python_type": "firedrake.HybridizationPC",
        "hybridization": {"ksp_type": "cg", "ksp_rtol": 1e-12, "pc_type": "python",
                          "pc_python_type": "firedrake.GTMGPC",
                          "gt": {"mg_levels": {"ksp_type": "chebyshev", "pc_type": "jacobi", "ksp_max_it": 3},
                                 "mg_coarse": {"ksp_type": "cg", "pc_type": "jacobi", "ksp_rtol": 1e-3}}}}


class GTMGMockEngine(HybridMockEngine):
    """The hybridisation mock plus the two trace transfers on extruded hexes, device location."""

    def fdb_kernel_create_mixed(self, desc, space2, out):
        d, s2 = me._obj(desc), me._obj(space2)
        if d.form not in (_lib.FORM_TRACE_PROLONG, _lib.FORM_TRACE_RESTRICT):
            return super().fdb_kernel_create_mixed(desc, space2, out)
        k = d.degree + 1
        if d.cell != _lib.CELL_HEX_EXTRUDED or k not in (2, 3) or s2.degree != 1:
            return self._fail("mock engine: the trace transfers are k = 2..3 on extruded hexes, with CG1")
        table = np.array(s2.B[:2 * k]).reshape(k, 2)
        x, _ = gauss_legendre(k)
        if np.abs(table - np.stack([1.0 - x, x], axis=1)).max() > 1e-15:
            return self._fail("mock engine: space2.B must be the CG1 basis at the Gauss-Legendre points")
        self._next += 1
        self.kernels[self._next] = dict(kind="trace", k=k, prolong=d.form == _lib.FORM_TRACE_PROLONG,
                                        off_t=np.array(d.offset0[:6 * k * k], dtype=np.int64),
                                        off_v=np.array(s2.offset[:8], dtype=np.int64))
        me._obj(out).value = self._next
        return 0

    def fdb_vec_chebyshev(self, n, cd, cz, b, ax, dinv, d, x):
        """d = c_d d + c_z dinv o (b - ax); x += d."""
        dv, xv = me._view(d, n), me._view(x, n)
        dv[:] = cd * dv + cz * me._view(dinv, n) * (me._view(b, n) - me._view(ax, n))
        xv += dv
        return 0

    def fdb_kernel_call(self, h, ca):
        kk = self.kernels[me._addr(h)]
        if kk["kind"] != "trace":
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        self.launches += 1
        k, nlay, nt = kk["k"], a.layers[1] - 1, 6 * kk["k"] ** 2
        want = 2 if kk["prolong"] else 3
        if a.location != _lib.LOC_DEVICE or a.nargs != want or a.nmaps != 2:
            return self._fail(f"mock engine: the trace transfer expects {want} device args and 2 maps")
        lay = np.arange(nlay)

        def rows(slot, arity, off):
            m = me._view(a.maps[slot], a.end * arity, np.int32).reshape(a.end, arity).astype(np.int64)
            return (m[:, None, :] + lay[None, :, None] * off[None, None, :]).reshape(-1, arity)

        ft = rows(0 if kk["prolong"] else 1, nt, kk["off_t"])
        fv = rows(1 if kk["prolong"] else 0, 8, kk["off_v"])
        Pl = go.trilinear(go.reference_points(k))
        nT, nV = int(ft.max()) + 1, int(fv.max()) + 1
        if kk["prolong"]:
            lam, c = me._view(a.args[0], nT), me._view(a.args[1], nV)
            for i in range(len(ft)):
                lam[ft[i]] = Pl @ c[fv[i]]
        else:
            c, lam, w = me._view(a.args[0], nV), me._view(a.args[1], nT), me._view(a.args[2], nT)
            for i in range(len(ft)):
                np.add.at(c, fv[i], Pl.T @ (w[ft[i]] * lam[ft[i]]))
        return 0


@pytest.fixture()
def mock(oracle):
    inst = me.install(oracle)
    inst.engine = GTMGMockEngine(oracle)
    with inst as eng:
        yield eng


@pytest.mark.parametrize("k", [2, 3])
def test_transfers_and_generic_path_match_the_oracle(mock, k):
    """TraceTransfer on the emulated forms and on the host build of the generic-path kernels both give P c and
    P^T lambda of the oracle."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import HybridizationPC
    mesh, S, Q, F = _spaces(k, n=(2, 3, 2))
    pc = HybridizationPC(F)
    tt = mg.TraceTransfer(pc)
    T, V1 = pc.trace, tt.Vc
    P = go.prolongation(T.V, V1.V)
    rng = np.random.default_rng(k)
    c, lam = rng.standard_normal(V1.node_count), rng.standard_normal(T.node_count)
    for pro, res in ((tt.prolong, tt.restrict), (tt.prolong_generic, tt.restrict_generic)):
        out = pro(V1.dat(c.copy()), T.dat())
        assert _rel(out.data_ro, P @ c) < 1e-14
        out = res(T.dat(lam.copy()), V1.dat())
        assert _rel(out.data_ro, P.T @ lam) < 1e-14


@pytest.mark.parametrize("ksp", ["preonly", "gmres"])
@pytest.mark.parametrize("flux", [(), (1, "top")])
def test_solve_with_gtmg_matches_scipy(mock, ksp, flux):
    from firedrake_b200.assemble import DirichletBC, solve
    mesh, S, Q, F = _spaces(n=(3, 3, 3))
    bcs = [DirichletBC(S, 0.0, s) for s in flux]
    L = _load(S, Q, F, 4)
    up = F.dat()
    its, hist = solve(F, L, up, bcs, {**GTMG, "ksp_type": ksp, "ksp_rtol": 1e-11})
    if ksp == "preonly":
        assert hist[-1] <= 1e-12 * hist[0] and its <= 15, (its, hist)
    s_ref, u_ref = _scipy(mesh, S, Q, F, L, bcs, False)
    assert _rel(up[0].data_ro, s_ref) < 1e-8
    assert _rel(up[1].data_ro, u_ref) < 1e-8


def test_all_flux_with_the_nullspace_and_flat_options(mock):
    from firedrake_b200.assemble import DirichletBC, solve
    mesh, S, Q, F = _spaces(n=(3, 2, 3))
    bcs = [DirichletBC(S, 0.0, s) for s in ho.SUBS]
    L = _load(S, Q, F, 5)
    up = F.dat()
    flat = {"mat_type": "matfree", "ksp_type": "preonly", "pc_type": "python",
            "pc_python_type": "firedrake.HybridizationPC", "hybridization_ksp_type": "cg",
            "hybridization_ksp_rtol": 1e-12, "hybridization_pc_type": "python",
            "hybridization_pc_python_type": "firedrake.GTMGPC", "hybridization_gt_mg_levels_ksp_max_it": 3,
            "hybridization_gt_mg_coarse_pc_type": "none", "hybridization_gt_pc_mg_type": "multiplicative"}
    solve(F, L, up, bcs, flat, nullspace="constant")
    s_ref, u_ref = _scipy(mesh, S, Q, F, L, bcs, True)
    assert _rel(up[0].data_ro, s_ref) < 1e-8
    assert _rel(up[1].data_ro, u_ref) < 1e-8
    assert abs(up[1].data_ro.mean()) < 1e-12 * np.abs(u_ref).max()


def _gt(**gt):
    return {**GTMG, "hybridization": {**GTMG["hybridization"], "gt": gt}}


@pytest.mark.parametrize("opts, exc, msg", [
    (_gt(pc_mg_galerkin=True), NotImplementedError, "hybridization_gt_pc_mg_galerkin"),
    (_gt(pc_mg_type="full"), NotImplementedError, "hybridization_gt_pc_mg_type 'full'"),
    (_gt(mg_coarse={"pc_mg_type": "full"}), NotImplementedError, "hybridization_gt_mg_coarse_pc_mg_type"),
    (_gt(mg_coarse={"ksp_type": "preonly", "pc_type": "mg", "mg_levels": {"ksp_type": "chebyshev"}}),
     NotImplementedError, "hybridization_gt_mg_coarse_mg_levels_ksp_type"),
    (_gt(mg_coarse={"ksp_type": "preonly", "pc_type": "lu"}), NotImplementedError, "direct coarse solvers"),
    (_gt(mg_coarse={"ksp_type": "preonly", "pc_type": "mg"}), ValueError, "hierarchy"),
    (_gt(mg_coarse={"ksp_type": "gmres", "pc_type": "jacobi"}), NotImplementedError, "cg with jacobi or none"),
    (_gt(mg_levels={"pc_type": "sor"}), NotImplementedError, "hybridization_gt_mg_levels_pc_type 'sor'"),
    (_gt(mg_levels={"ksp_type": "gmres"}), NotImplementedError, "hybridization_gt_mg_levels_ksp_type 'gmres'"),
    (_gt(mg_coarse_degree=2), NotImplementedError, "unknown GTMG option hybridization_gt_mg_coarse_degree"),
    (_gt(appctx=1), NotImplementedError, "unknown GTMG option hybridization_gt_appctx"),
    ({**GTMG, "hybridization": {**GTMG["hybridization"], "pc_python_type": "firedrake.PMGPC"}},
     NotImplementedError, "hybridization_pc_python_type 'firedrake.PMGPC'"),
    ({**GTMG, "hybridization": {**GTMG["hybridization"], "pc_type": "jacobi"}},
     NotImplementedError, "hybridization_pc_python_type needs hybridization_pc_type 'python'"),
    ({**GTMG, "hybridization": {**GTMG["hybridization"], "mat_type": "matfree"}},
     NotImplementedError, "hybridization_mat_type 'matfree'"),
    # the refusals of the hybridisation options stand as they were
    ({"hybridization": {"pc_type": "python"}}, NotImplementedError, "hybridization_pc_type 'python'"),
    ({"hybridization": {"pc_type": "mg"}}, NotImplementedError, "hybridization_pc_type 'mg'"),
    ({"hybridization": {"pc_type": "gamg"}}, NotImplementedError, "hybridization_pc_type 'gamg'"),
    ({"hybridization": {"pc_type": "hypre"}}, NotImplementedError, "hybridization_pc_type 'hypre'"),
    ({"hybridization": {"pc_type": "lu"}}, NotImplementedError, "hybridization_pc_type 'lu'"),
    ({"pc_python_type": "firedrake.GTMGPC"}, NotImplementedError, "pc_python_type 'firedrake.GTMGPC'"),
    ({"hybridization": {"mat_type": "matfree"}}, NotImplementedError, "hybridization_mat_type 'matfree'"),
])
def test_option_refusals(mock, opts, exc, msg):
    from firedrake_b200.assemble import solve
    from test_hybrid_host_mock import HYBRID
    _, S, Q, F = _spaces(n=(1, 1, 1))
    sp = opts if "hybridization" in opts and opts.get("pc_python_type") else {**HYBRID, **opts}
    with pytest.raises(exc, match=msg):
        solve(F, F.dat(), F.dat(), (), sp)


def test_trace_transfer_refuses_other_spaces(mock):
    from firedrake_b200 import mg
    from firedrake_b200.assemble import FunctionSpace, HybridizationPC
    mesh, S, Q, F = _spaces(n=(1, 1, 1))
    pc = HybridizationPC(F)
    with pytest.raises(ValueError, match="scalar CG1"):
        mg.TraceTransfer(pc, FunctionSpace(mesh, 2))
    with pytest.raises(NotImplementedError, match="k = 4"):
        mg.trace_transfer_kernels(4)
    with pytest.raises(NotImplementedError, match="coarse solve"):
        mg.GTMG(pc, coarse_ksp="preonly", coarse_pc="lu")
