"""Host logic of the coefficient form (FDB_FORM_HELMHOLTZ_COEF) on the CPU: a mock engine that
emulates the form through the NumPy oracle (tests/_coef_oracle.py) runs the tests of
tests/test_coefficient_gpu.py -- argument lists, Form / assemble / ImplicitMatrixContext / solve
plumbing, the coarsened coefficient of the V-cycle -- and a gloo world-2 run on a slab partition,
whose owned rows must equal the serial result (kappa's ghost rows are refreshed by Parloop like any
other READ argument).  The device code itself is what `-m gpu` checks."""
import os
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

import _coef_oracle as co
import _mock_engine as me
import test_coefficient_gpu as tg
from firedrake_b200 import _lib
from firedrake_b200.fiat_lite import interval_element
from test_partition_gloo import ROOT, _free_port


class CoefMockEngine(me.MockEngine):
    """MockEngine plus the coefficient form, extruded and native hexes, device or host location (the
    "mirrors" of host buffers are the buffers themselves)."""

    def fdb_kernel_create(self, desc, out):
        d = me._obj(desc)
        if d.form != _lib.FORM_HELMHOLTZ_COEF:
            return super().fdb_kernel_create(desc, out)
        if d.cell not in (_lib.CELL_HEX_EXTRUDED, _lib.CELL_HEX) or d.cdim != 1 or d.affine_cells:
            return self._fail("mock engine: helmholtz_coef takes scalar hex spaces, no affine variant")
        n = (d.degree + 1) ** 3
        ext = d.cell == _lib.CELL_HEX_EXTRUDED
        k = dict(kind="coef", degree=d.degree, rank=d.rank, alpha=d.alpha, beta=d.beta, diagonal=d.diagonal,
                 extruded=ext, off0=np.array(d.offset0[:n] if ext else [0] * n, dtype=np.int32),
                 off1=np.array(d.offset1[:8] if ext else [0] * 8, dtype=np.int32))
        self._next += 1
        self.kernels[self._next] = k
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        k = self.kernels[me._addr(h)]
        if k["kind"] != "coef":
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        self.launches += 1
        want = 3 if (k["rank"] == 2 or k["diagonal"]) else 4
        if a.nargs != want or a.nmaps != 2:
            return self._fail(f"mock engine: helmholtz_coef expects {want} args and 2 maps")
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
        kappa = me._view(a.args[a.nargs - 1], nnode)
        geo = (map0[cols], k["off0"], map1[cols], k["off1"], nlay)
        ab = dict(alpha=k["alpha"], beta=k["beta"])
        if k["rank"] == 2:
            m = self.mats[a.args[0]]
            i0, A = co.element_matrices(el, coords, kappa, *geo, **ab)
            co.add_to_csr(m.rowptr, m.colidx, m.vals, i0, A, m.row_lg, m.col_lg)
        elif k["diagonal"]:
            co.diagonal(el, coords, kappa, *geo, **ab, out=me._view(a.args[0], nnode))
        else:
            y = me._view(a.args[0], nnode)
            if a.location == _lib.LOC_HOST and a.output_is_zero:
                y[:] = 0.0                      # the engine zeroes the output's mirror
            co.action(el, coords, me._view(a.args[2], nnode).copy(), kappa, *geo, **ab, out=y)
        return 0


class install(me.install):
    def __init__(self, oracle):
        self.engine = CoefMockEngine(oracle)


@pytest.fixture()
def mock(oracle):
    with install(oracle) as eng:
        yield eng


@pytest.mark.parametrize("p", [1, 3])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
def test_action_host_logic(mock, p, native):
    tg.test_coef_action_matches_oracle(mock, p, native, 0.6)


@pytest.mark.parametrize("p", [1, 2])
def test_generic_path_and_constant_form_host_logic(mock, p):
    tg.test_coef_action_matches_generic_path_and_constant_form(mock, p)


@pytest.mark.parametrize("p", [1, 2])
def test_matrix_and_matfree_host_logic(mock, p):
    tg.test_coef_matrix_matches_oracle(mock, p)
    tg.test_coef_diagonal_equals_assembled_diagonal(mock, p)


def test_host_pointer_mode_host_logic(mock):
    tg.test_coef_host_pointer_mode_equals_device_mode(mock)


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
def test_solve_host_logic(mock, pc):
    tg.test_coef_solve(mock, pc)


def test_vcycle_coarsens_kappa_by_injection(mock):
    """Each coarser level's kappa is the injection of the next finer one; a kappa that is a
    polynomial of the space's degree on every level is reproduced exactly."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import Form, FunctionSpace, interpolate
    h = mg.MeshHierarchy(2, 2, 2, 2)
    V = FunctionSpace(h[2], 2)
    expr = "1.0 + x[0] * x[1] + x[2] * x[2]"
    kap = interpolate(V, expr)
    vc = mg.VCycle(h, 2, lambda W, k=None: Form(W, 1.0, 0.0, k), kappa=kap)
    assert vc.kappas[2] is not kap and np.array_equal(vc.kappas[2].data_ro, kap.data_ro)
    for l in (0, 1):
        want = interpolate(vc.spaces[l], expr)
        assert np.abs(vc.kappas[l].data_ro - want.data_ro).max() < 1e-13
        assert vc.ops[l].form.kappa is vc.kappas[l]


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import test_coefficient_host_mock as tm
    from firedrake_b200.assemble import Form, FunctionSpace, OneFormAssembler, assemble, interpolate
    from firedrake_b200.partition import SlabPartition
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    from oracle import oracle
    key = lambda L: (L[:, 0] * 1000 + L[:, 1]) * 1000 + L[:, 2]
    out = {}
    with tm.install(oracle) as eng:
        nx, ny, nz, p = 5, 3, 4, 2
        ue, ke = "sin(2.0 * x[0]) + x[1] * x[2]", "2.0 + sin(3.0 * x[0]) * x[1]"
        # serial reference on the whole mesh (no communication)
        eng.dist = None
        G = FunctionSpace(ExtrudedHexMesh(nx, ny, nz, warp=0.05), p)
        gk = interpolate(G, ke)
        gy = OneFormAssembler(Form(G, 1.0, 0.4, gk), interpolate(G, ue)).assemble()
        gd = assemble(Form(G, 1.0, 0.4, gk), mat_type="matfree").getDiagonal(G.dat())
        look_y = dict(zip(key(G.V.dof_lattice()).tolist(), gy.data_ro.tolist()))
        look_d = dict(zip(key(G.V.dof_lattice()).tolist(), gd.data_ro.tolist()))
        # this rank's slab; kappa's ghost rows are made stale on purpose before every parloop
        eng.dist = dist
        part = SlabPartition(nx, ny, nz, p, rank, world, warp=0.05)
        V = FunctionSpace(part.mesh, p, partition=part)
        kap = interpolate(V, ke)
        no = V.V.owned_node_count
        kap.data[no:] = -1.0e3
        kap.halo_valid = False
        y = OneFormAssembler(Form(V, 1.0, 0.4, kap), interpolate(V, ue)).assemble()
        lat = V.V.dof_lattice()[:no]
        out["action"] = float(np.abs(y.data_ro[:no] - np.array([look_y[k] for k in key(lat).tolist()])).max())
        kap.data[no:] = -1.0e3
        kap.halo_valid = False
        d = assemble(Form(V, 1.0, 0.4, kap), mat_type="matfree").getDiagonal(V.dat())
        out["diag"] = float(np.abs(d.data_ro[:no] - np.array([look_d[k] for k in key(lat).tolist()])).max())
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
