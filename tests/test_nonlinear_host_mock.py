"""Host logic of nonlinear diffusion on the CPU: a mock engine that emulates the residual and Jacobian
forms through the NumPy oracle (tests/_nonlinear_oracle.py) runs the tests of
tests/test_nonlinear_gpu.py -- argument lists, NonlinearDiffusion / assemble / ImplicitMatrixContext
plumbing, GMRES and the Newton solver -- plus GMRES against scipy on a nonsymmetric operator and a
gloo world-2 run on a slab partition, whose owned rows must equal the serial result (the
linearisation point's ghost rows are refreshed by Parloop like any other READ argument).  The device
code itself is what `-m gpu` checks."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sps
import scipy.sparse.linalg as spla
import torch.multiprocessing as mp

import _mock_engine as me
import _nonlinear_oracle as no
import test_coefficient_host_mock as cm
import test_nonlinear_gpu as tg
from firedrake_b200 import _lib
from firedrake_b200.fiat_lite import interval_element
from test_partition_gloo import ROOT, _free_port

NL_FORMS = (_lib.FORM_NONLINEAR_DIFFUSION, _lib.FORM_NONLINEAR_DIFFUSION_JACOBIAN)


class NonlinearMockEngine(cm.CoefMockEngine):
    """CoefMockEngine plus the nonlinear diffusion forms, extruded and native hexes, device or host
    location."""

    def fdb_kernel_create(self, desc, out):
        d = me._obj(desc)
        if d.form not in NL_FORMS:
            return super().fdb_kernel_create(desc, out)
        if d.cell not in (_lib.CELL_HEX_EXTRUDED, _lib.CELL_HEX) or d.cdim != 1 or d.affine_cells:
            return self._fail("mock engine: nonlinear diffusion takes scalar hex spaces, no affine variant")
        if d.form == _lib.FORM_NONLINEAR_DIFFUSION and (d.rank != 1 or d.diagonal):
            return self._fail("mock engine: nonlinear_diffusion is a 1-form action only")
        n = (d.degree + 1) ** 3
        ext = d.cell == _lib.CELL_HEX_EXTRUDED
        k = dict(kind="nl", jac=d.form == _lib.FORM_NONLINEAR_DIFFUSION_JACOBIAN, degree=d.degree, rank=d.rank,
                 alpha=d.alpha, beta=d.beta, diagonal=d.diagonal, dc=tuple(d.dcoef), extruded=ext,
                 off0=np.array(d.offset0[:n] if ext else [0] * n, dtype=np.int32),
                 off1=np.array(d.offset1[:8] if ext else [0] * 8, dtype=np.int32))
        self._next += 1
        self.kernels[self._next] = k
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        k = self.kernels[me._addr(h)]
        if k["kind"] != "nl":
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        self.launches += 1
        want = 4 if (k["jac"] and k["rank"] == 1 and not k["diagonal"]) else 3
        if a.nargs != want or a.nmaps != 2:
            return self._fail(f"mock engine: nonlinear diffusion expects {want} args and 2 maps")
        el = interval_element(k["degree"])
        nlay = a.layers[1] - 1 if k["extruded"] else 1
        arity = (k["degree"] + 1) ** 3
        map0 = me._view(a.maps[0], a.end * arity, np.int32).reshape(a.end, arity)
        map1 = me._view(a.maps[1], a.end * 8, np.int32).reshape(a.end, 8)
        cols = me._view(a.subset, a.end, np.int32)[a.start:a.end] if me._addr(a.subset) else \
            np.arange(a.start, a.end)
        nvert = int(map1.max() + k["off1"].max() * (nlay - 1)) + 1
        nnode = int(map0.max() + k["off0"].max() * (nlay - 1)) + 1
        coords = me._view(a.args[1], nvert * 3)
        u = me._view(a.args[a.nargs - 1], nnode).copy()
        geo = (map0[cols], k["off0"], map1[cols], k["off1"], nlay)
        ab = dict(alpha=k["alpha"], beta=k["beta"])
        if k["rank"] == 2:
            m = self.mats[a.args[0]]
            i0, A = no.jacobian_matrices(el, coords, u, *geo, k["dc"], **ab)
            cm.co.add_to_csr(m.rowptr, m.colidx, m.vals, i0, A, m.row_lg, m.col_lg)
            return 0
        y = me._view(a.args[0], nnode)
        if k["diagonal"]:
            y += no.jacobian_diagonal(el, coords, u, *geo, k["dc"], **ab)
            return 0
        if a.location == _lib.LOC_HOST and a.output_is_zero:
            y[:] = 0.0
        if k["jac"]:
            w = me._view(a.args[2], nnode).copy()
            y += no.jacobian_action(el, coords, u, w, *geo, k["dc"], **ab)
        else:
            y += no.residual(el, coords, u, *geo, k["dc"], **ab)
        return 0


class install(me.install):
    def __init__(self, oracle):
        self.engine = NonlinearMockEngine(oracle)


@pytest.fixture()
def mock(oracle):
    with install(oracle) as eng:
        yield eng


@pytest.mark.parametrize("p", [1, 3])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
def test_action_host_logic(mock, p, native):
    tg.test_nl_residual_and_jacobian_action_match_oracle(mock, p, native, 0.6)


@pytest.mark.parametrize("p", [1, 2])
def test_merged_kernels_host_logic(mock, p):
    tg.test_nl_forms_against_the_merged_kernels(mock, p)


def test_taylor_host_logic(mock):
    tg.test_nl_taylor_ratio(mock, 2)


@pytest.mark.parametrize("p", [1, 2])
def test_matrix_and_matfree_host_logic(mock, p):
    tg.test_nl_matrix_matches_oracle(mock, p)
    tg.test_nl_diagonal_equals_assembled_diagonal(mock, p)


def test_host_pointer_mode_host_logic(mock):
    tg.test_nl_host_pointer_mode_equals_device_mode(mock)


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
def test_newton_host_logic(mock, pc):
    tg.test_nl_newton_solve_manufactured(mock, pc)


def test_dirichlet_newton_host_logic(mock):
    """BC rows, the zero update on constrained nodes and the Newton step count against the oracle."""
    tg.test_nl_dirichlet_matches_oracle_newton(mock)


def test_cg1_rates_host_logic(mock):
    """The L2 rate check on the coarser half of its meshes (the finest one is for the GPU)."""
    from firedrake_b200.assemble import solve_nonlinear
    errs = []
    for n in (4, 8, 16):
        V, _, F, L, ui = tg.manufactured(n, 1)
        u = V.dat()
        solve_nonlinear(F, L, u, solver_parameters=dict(tg.NEWTON_PARAMS, pc_type="jacobi"))
        errs.append(tg.l2_error(V, u, ui))
    rates = np.log2(np.array(errs[:-1]) / np.array(errs[1:]))
    assert rates[-1] > 1.8, (errs, rates)


class _Dense:
    """A nonsymmetric operator on a plain device Dat (mult through the mock engine's memory)."""

    def __init__(self, K):
        self.K = K

    def mult(self, X, Y):
        Y.data[:] = self.K @ X.data_ro
        return Y


def _operator(n=120, seed=0):
    rng = np.random.default_rng(seed)
    K = sps.random(n, n, density=0.05, random_state=seed) + sps.diags(4.0 + rng.random(n))
    K = (K + 0.5 * sps.diags(np.ones(n - 1), 1) - 0.3 * sps.diags(np.ones(n - 1), -1)).tocsr()
    return K, rng.standard_normal(n)


@pytest.mark.parametrize("restart", [5, 30])
def test_gmres_matches_spsolve(mock, restart):
    from firedrake_b200 import op2
    from firedrake_b200.assemble import gmres
    K, b = _operator()
    assert abs(K - K.T).max() > 0.1
    S = op2.Set(len(b))
    x, bd = op2.Dat(S), op2.Dat(S, b.copy())
    x.device_ptr
    its, hist = gmres(_Dense(K), bd, x, rtol=1e-12, restart=restart)
    ref = spla.spsolve(K.tocsc(), b)
    assert np.abs(x.data_ro - ref).max() < 1e-9 * np.abs(ref).max(), (its, hist[-1])
    assert hist[-1] <= 1e-12 * hist[0] * 1.0001


def test_gmres_with_a_variable_preconditioner(mock):
    """The preconditioner changes at every application (a few inexact Jacobi sweeps whose count cycles):
    flexible GMRES still converges to the exact solution."""
    from firedrake_b200 import op2
    from firedrake_b200.assemble import gmres
    K, b = _operator(seed=1)
    dinv = 1.0 / K.diagonal()
    calls = []

    def M(r, z):
        rv = r.data_ro.copy()
        zv = dinv * rv
        for _ in range(len(calls) % 3):
            zv = zv + dinv * (rv - K @ zv)
        calls.append(1)
        z.data[:] = zv

    S = op2.Set(len(b))
    x, bd = op2.Dat(S), op2.Dat(S, b.copy())
    x.device_ptr
    its, hist = gmres(_Dense(K), bd, x, M=M, rtol=1e-12, restart=10)
    ref = spla.spsolve(K.tocsc(), b)
    assert np.abs(x.data_ro - ref).max() < 1e-9 * np.abs(ref).max(), (its, hist[-1])
    its0, _ = gmres(_Dense(K), bd, op2.Dat(S), rtol=1e-12, restart=10)
    assert its < its0, (its, its0)


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import test_nonlinear_host_mock as tm
    from firedrake_b200.assemble import FunctionSpace, NonlinearDiffusion, assemble, interpolate
    from firedrake_b200.partition import SlabPartition
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    from oracle import oracle
    key = lambda L: (L[:, 0] * 1000 + L[:, 1]) * 1000 + L[:, 2]
    out = {}
    d = (1.0, 0.3, 0.2)
    with tm.install(oracle) as eng:
        nx, ny, nz, p = 5, 3, 4, 2
        ue, we = "sin(2.0 * x[0]) + x[1] * x[2]", "x[0] - 2.0 * x[1] * x[2]"
        eng.dist = None
        G = FunctionSpace(ExtrudedHexMesh(nx, ny, nz, warp=0.05), p)
        FG = NonlinearDiffusion(G, 1.0, 0.4, d)
        gu = interpolate(G, ue)
        gy = assemble(FG.jacobian(gu), u=interpolate(G, we))
        gd = assemble(FG.jacobian(gu), mat_type="matfree").getDiagonal(G.dat())
        look_y = dict(zip(key(G.V.dof_lattice()).tolist(), gy.data_ro.tolist()))
        look_d = dict(zip(key(G.V.dof_lattice()).tolist(), gd.data_ro.tolist()))
        # this rank's slab; u's ghost rows are made stale on purpose before every parloop
        eng.dist = dist
        part = SlabPartition(nx, ny, nz, p, rank, world, warp=0.05)
        V = FunctionSpace(part.mesh, p, partition=part)
        F = NonlinearDiffusion(V, 1.0, 0.4, d)
        u = interpolate(V, ue)
        no_ = V.V.owned_node_count
        u.data[no_:] = -1.0e3
        u.halo_valid = False
        y = assemble(F.jacobian(u), u=interpolate(V, we))
        lat = V.V.dof_lattice()[:no_]
        out["action"] = float(np.abs(y.data_ro[:no_] - np.array([look_y[k] for k in key(lat).tolist()])).max())
        u.data[no_:] = -1.0e3
        u.halo_valid = False
        dd = assemble(F.jacobian(u), mat_type="matfree").getDiagonal(V.dat())
        out["diag"] = float(np.abs(dd.data_ro[:no_] - np.array([look_d[k] for k in key(lat).tolist()])).max())
        out["scale"] = float(np.abs(gy.data_ro).max())
        out["dscale"] = float(np.abs(gd.data_ro).max())
    q.put((rank, out))
    dist.destroy_process_group()


def test_partitioned_world2_owned_rows_equal_serial():
    from oracle import oracle
    oracle.build()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for pr in procs:
        pr.start()
    res = [q.get(timeout=300) for _ in range(2)]
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    for rank, out in res:
        assert out["action"] < 1e-12 * out["scale"], (rank, out)
        assert out["diag"] < 1e-12 * out["dscale"], (rank, out)
