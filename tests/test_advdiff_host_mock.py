"""Host logic of advection-diffusion (FDB_FORM_ADVECTION_DIFFUSION) on the CPU: a mock engine that emulates
the form through the NumPy oracle (tests/_advdiff_oracle.py) runs the tests of tests/test_advdiff_gpu.py --
argument lists, AdvectionDiffusion / assemble / ImplicitMatrixContext plumbing, GMRES with each
preconditioner against scipy -- and a gloo world-2 run on a slab partition, whose owned rows must equal the
serial result (b's ghost rows are refreshed by Parloop like any other READ argument).  The device code
itself is what `-m gpu` checks."""
import os
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

import _advdiff_oracle as ao
import _mock_engine as me
import test_advdiff_gpu as tg
from firedrake_b200 import _lib
from firedrake_b200.fiat_lite import interval_element
from test_coefficient_host_mock import CoefMockEngine
from test_partition_gloo import ROOT, _free_port


class AdvMockEngine(CoefMockEngine):
    """The coefficient mock engine plus advection-diffusion, extruded and native hexes, device or host
    location (the "mirrors" of host buffers are the buffers themselves)."""

    def fdb_kernel_create(self, desc, out):
        d = me._obj(desc)
        if d.form != _lib.FORM_ADVECTION_DIFFUSION:
            return super().fdb_kernel_create(desc, out)
        if d.cell not in (_lib.CELL_HEX_EXTRUDED, _lib.CELL_HEX) or d.cdim != 1 or d.affine_cells:
            return self._fail("mock engine: advection_diffusion takes scalar hex spaces, no affine variant")
        n = (d.degree + 1) ** 3
        ext = d.cell == _lib.CELL_HEX_EXTRUDED
        k = dict(kind="adv", degree=d.degree, rank=d.rank, alpha=d.alpha, beta=d.beta, diagonal=d.diagonal,
                 extruded=ext, off0=np.array(d.offset0[:n] if ext else [0] * n, dtype=np.int32),
                 off1=np.array(d.offset1[:8] if ext else [0] * 8, dtype=np.int32))
        self._next += 1
        self.kernels[self._next] = k
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        k = self.kernels[me._addr(h)]
        if k["kind"] != "adv":
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        self.launches += 1
        want = 3 if (k["rank"] == 2 or k["diagonal"]) else 4
        if a.nargs != want or a.nmaps != 2:
            return self._fail(f"mock engine: advection_diffusion expects {want} args and 2 maps")
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
        b = me._view(a.args[a.nargs - 1], 3 * nnode)
        geo = (map0[cols], k["off0"], map1[cols], k["off1"], nlay)
        ab = dict(alpha=k["alpha"], beta=k["beta"])
        if k["rank"] == 2:
            m = self.mats[a.args[0]]
            i0, A = ao.element_matrices(el, coords, b, *geo, **ab)
            ao.co.add_to_csr(m.rowptr, m.colidx, m.vals, i0, A, m.row_lg, m.col_lg)
        elif k["diagonal"]:
            ao.diagonal(el, coords, b, *geo, **ab, out=me._view(a.args[0], nnode))
        else:
            y = me._view(a.args[0], nnode)
            if a.location == _lib.LOC_HOST and a.output_is_zero:
                y[:] = 0.0
            ao.action(el, coords, me._view(a.args[2], nnode).copy(), b, *geo, **ab, out=y)
        return 0


class install(me.install):
    def __init__(self, oracle):
        self.engine = AdvMockEngine(oracle)


@pytest.fixture()
def mock(oracle):
    with install(oracle) as eng:
        yield eng


@pytest.mark.parametrize("p", [1, 3])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
def test_action_host_logic(mock, p, native):
    tg.test_advdiff_action_matches_oracle(mock, p, native, 0.6)


@pytest.mark.parametrize("p", [1, 2])
def test_generic_path_and_constant_form_host_logic(mock, p):
    tg.test_advdiff_action_matches_generic_path_and_helmholtz(mock, p)


@pytest.mark.parametrize("p", [1, 2])
def test_matrix_and_matfree_host_logic(mock, p):
    tg.test_advdiff_matrix_matches_oracle(mock, p)
    tg.test_advdiff_diagonal_equals_assembled_diagonal(mock, p)


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
def test_gmres_solve_host_logic(mock, pc):
    """GMRES with each preconditioner against scipy's LU of the oracle's matrix."""
    tg.test_advdiff_solve_matches_scipy(mock, pc)


def test_solver_options_host_logic(mock):
    tg.test_advdiff_cg_refuses_and_gmres_is_the_default(mock)
    from firedrake_b200 import op2
    from firedrake_b200.assemble import AdvectionDiffusion, FunctionSpace, assemble
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    W = FunctionSpace(ExtrudedHexMesh(2, 2, 2), 1)
    F = AdvectionDiffusion(W, op2.Dat(W.vector_dset(3)))
    assert F.symmetric is False
    assert len(F.coefficient_args()) == 1 and F.coefficient_args()[0].data is F.b
    with pytest.raises(NotImplementedError, match="advection-diffusion"):
        assemble(F, mat_type="matfree").multTranspose(W.dat(), W.dat())


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import test_advdiff_host_mock as tm
    from firedrake_b200 import op2
    from firedrake_b200.assemble import AdvectionDiffusion, FunctionSpace, OneFormAssembler, assemble, interpolate
    from firedrake_b200.partition import SlabPartition
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    from oracle import oracle
    key = lambda L: (L[:, 0] * 1000 + L[:, 1]) * 1000 + L[:, 2]
    vel = lambda X: np.stack([1.0 + X[:, 1], 0.5 - X[:, 0] * X[:, 2], np.cos(X[:, 0])], axis=1)
    out = {}
    with tm.install(oracle) as eng:
        nx, ny, nz, p = 5, 3, 4, 2
        ue = "sin(2.0 * x[0]) + x[1] * x[2]"
        # serial reference on the whole mesh (no communication)
        eng.dist = None
        G = FunctionSpace(ExtrudedHexMesh(nx, ny, nz, warp=0.05), p)
        gb = op2.Dat(G.vector_dset(3), vel(G.V.dof_coordinates()))
        gy = OneFormAssembler(AdvectionDiffusion(G, gb, 1.0, 0.4), interpolate(G, ue)).assemble()
        gd = assemble(AdvectionDiffusion(G, gb, 1.0, 0.4), mat_type="matfree").getDiagonal(G.dat())
        look_y = dict(zip(key(G.V.dof_lattice()).tolist(), gy.data_ro.tolist()))
        look_d = dict(zip(key(G.V.dof_lattice()).tolist(), gd.data_ro.tolist()))
        # this rank's slab; b's ghost rows are made stale on purpose before every parloop
        eng.dist = dist
        part = SlabPartition(nx, ny, nz, p, rank, world, warp=0.05)
        V = FunctionSpace(part.mesh, p, partition=part)
        b = op2.Dat(V.vector_dset(3), vel(V.V.dof_coordinates()))
        no = V.V.owned_node_count
        out["has_halo"] = V.vector_dset(3).halo is not None
        b.data[no:] = -1.0e3
        b.halo_valid = False
        y = OneFormAssembler(AdvectionDiffusion(V, b, 1.0, 0.4), interpolate(V, ue)).assemble()
        lat = V.V.dof_lattice()[:no]
        out["action"] = float(np.abs(y.data_ro[:no] - np.array([look_y[k] for k in key(lat).tolist()])).max())
        b.data[no:] = -1.0e3
        b.halo_valid = False
        d = assemble(AdvectionDiffusion(V, b, 1.0, 0.4), mat_type="matfree").getDiagonal(V.dat())
        out["diag"] = float(np.abs(d.data_ro[:no] - np.array([look_d[k] for k in key(lat).tolist()])).max())
        out["scale"] = float(np.abs(gy.data_ro).max())
        out["dscale"] = float(np.abs(gd.data_ro).max())
    q.put((rank, out))
    dist.destroy_process_group()


def test_partitioned_world2_refreshes_the_velocity_ghost_rows():
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
        assert out["has_halo"], (rank, out)
        assert out["action"] < 1e-12 * out["scale"], (rank, out)
        assert out["diag"] < 1e-12 * out["dscale"], (rank, out)
