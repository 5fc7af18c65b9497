"""Host logic of hyperelasticity on the CPU: a mock engine that emulates FDB_FORM_HYPERELASTICITY[_JACOBIAN]
through the NumPy oracle (tests/_hyperelastic_oracle.py) runs the tests of tests/test_hyperelastic_gpu.py
-- argument lists, the blocked aij Jacobian with dof-level Dirichlet lgmaps, the matrix-free operator and
its diagonal, Newton with pc_type none / jacobi / mg and its NaN guard -- checks GMRES and Newton against
scipy, and runs a gloo world-2 slab partition in which u's ghost rows must be refreshed before the
Jacobian reads them.  The device code itself is what `-m gpu` checks."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse.linalg as spla
import torch.multiprocessing as mp

import _elasticity_oracle as eo
import _hyperelastic_oracle as ho
import _mock_engine as me
import test_elasticity_host_mock as em
import test_hyperelastic_gpu as tg
from firedrake_b200 import _lib
from firedrake_b200.fiat_lite import interval_element
from test_partition_gloo import ROOT, _free_port

_HYPER = (_lib.FORM_HYPERELASTICITY, _lib.FORM_HYPERELASTICITY_JACOBIAN)


class HyperElasticityMockEngine(em.ElasticityMockEngine):
    """ElasticityMockEngine plus the hyperelastic residual and Jacobian."""

    def fdb_kernel_create(self, desc, out):
        d = me._obj(desc)
        if d.form not in _HYPER:
            return super().fdb_kernel_create(desc, out)
        if d.cell not in (_lib.CELL_HEX_EXTRUDED, _lib.CELL_HEX) or d.cdim != 3 or d.affine_cells:
            return self._fail("mock engine: hyperelasticity takes 3-component hex spaces, no affine variant")
        if d.form == _lib.FORM_HYPERELASTICITY and (d.rank != 1 or d.diagonal):
            return self._fail("mock engine: hyperelasticity is the residual, a 1-form action only")
        n = (d.degree + 1) ** 3
        ext = d.cell == _lib.CELL_HEX_EXTRUDED
        k = dict(kind="hyperelasticity", jacobian=d.form == _lib.FORM_HYPERELASTICITY_JACOBIAN, degree=d.degree,
                 rank=d.rank, mu=d.alpha, lmbda=d.lmbda, beta=d.beta, diagonal=d.diagonal, extruded=ext,
                 off0=np.array(d.offset0[:n] if ext else [0] * n, dtype=np.int32),
                 off1=np.array(d.offset1[:8] if ext else [0] * 8, dtype=np.int32))
        self._next += 1
        self.kernels[self._next] = k
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        k = self.kernels[me._addr(h)]
        if k["kind"] != "hyperelasticity":
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        self.launches += 1
        want = 3 if (k["rank"] == 2 or k["diagonal"] or not k["jacobian"]) else 4
        if a.nargs != want or a.nmaps != 2:
            return self._fail(f"mock engine: hyperelasticity expects {want} args and 2 maps")
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
        geo = (map0[cols], k["off0"], map1[cols], k["off1"], nlay)
        lam = dict(mu=k["mu"], lmbda=k["lmbda"], beta=k["beta"])
        u = me._view(a.args[a.nargs - 1], 3 * nnode).copy()
        if k["rank"] == 2:
            m = self.mats[a.args[0]]
            if m.bs != 3:
                return self._fail(f"mock engine: Mat block size {m.bs} != value size 3 of the argument space")
            di, A = ho.element_matrices(el, coords, u, *geo, **lam)
            eo.add_to_bcsr(m.rowptr, m.colidx, m.vals, di, A, m.row_lg, m.col_lg)
            return 0
        y = me._view(a.args[0], 3 * nnode)
        if k["diagonal"]:
            ho.diagonal(el, coords, u, *geo, **lam, out=y)
            return 0
        if a.location == _lib.LOC_HOST and a.output_is_zero:
            y[:] = 0.0
        if k["jacobian"]:
            ho.jacobian_action(el, coords, u, me._view(a.args[2], 3 * nnode).copy(), *geo, **lam, out=y)
        else:
            with np.errstate(invalid="ignore"):
                ho.residual(el, coords, u, *geo, **lam, out=y)
        return 0


class install(me.install):
    def __init__(self, oracle):
        self.engine = HyperElasticityMockEngine(oracle)


@pytest.fixture()
def mock(oracle):
    with install(oracle) as eng:
        yield eng


@pytest.mark.parametrize("p", [1, 3])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
def test_residual_and_jacobian_action_host_logic(mock, p, native):
    tg.test_residual_matches_oracle(mock, p, native)
    tg.test_jacobian_action_matches_oracle(mock, p, native)


@pytest.mark.parametrize("p", [1, 2])
def test_generic_path_host_logic(mock, p):
    tg.test_matches_generic_path(mock, p)


def test_host_pointer_mode_host_logic(mock):
    tg.test_host_pointer_mode_equals_device_mode(mock)


@pytest.mark.parametrize("p", [1, 2])
def test_matrix_and_matfree_host_logic(mock, p):
    tg.test_jacobian_blocked_matrix_matches_oracle(mock, p)
    tg.test_mat_mult_equals_matfree(mock, p, True)
    tg.test_mat_mult_equals_matfree(mock, p, False)
    tg.test_diagonal_equals_assembled_diagonal(mock, p)
    tg.test_jacobian_at_zero_equals_elasticity(mock, p)


def test_invariants_host_logic(mock):
    tg.test_rigid_rotation_has_zero_residual(mock, 2)
    tg.test_taylor_ratio_is_four(mock, 1)


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
def test_patch_test_host_logic(mock, pc):
    tg.test_homogeneous_deformation_patch_test(mock, pc, 1)


def test_twisted_cube_host_logic(mock):
    tg.test_twisted_cube_matches_scipy_newton(mock, 1)


def test_nan_guard_host_logic(mock):
    tg.test_inverted_element_ends_the_solve(mock)


def test_gmres_step_matches_scipy(mock):
    """One Newton step's linear solve: GMRES with the Jacobi preconditioner on the assembled Jacobian with
    clamped rows equals scipy's direct solve of the oracle's Jacobian."""
    from firedrake_b200 import mg, op2
    from firedrake_b200.assemble import DirichletBC, FunctionSpace, HyperElasticity, assemble, gmres
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    V = FunctionSpace(ExtrudedHexMesh(3, 3, 3, warp=0.05), 1, 3)
    u = tg._u(V, 0.2)
    bcs = [DirichletBC(V, 0.0, "bottom")]
    J = HyperElasticity(V, tg.MU, tg.LMBDA).jacobian(u)
    A = assemble(J, bcs=bcs, mat_type="matfree")
    b = V.dat(tg.vec_values(V.node_count, 1))
    for bc in bcs:
        bc.zero(b)
    d = A.getDiagonal(V.dat())
    op2.par_loop(mg.reciprocal_kernel(3), V.node_set, d(op2.RW))
    x = V.dat()

    def M(r, z):
        _lib.check(_lib.lib().fdb_vec_pointwise_mult(3 * V.node_count, r.device_ptr, d.device_ptr, z.device_ptr))
        z._device_written()

    gmres(A, b, x, M, rtol=1e-12, restart=40, maxit=2000)
    mesh = V.mesh
    K = ho.global_jacobian(interval_element(1), mesh.coordinates, u.data_ro.ravel().copy(),
                           (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz),
                           tg.MU, tg.LMBDA).tocsr()
    bd = (3 * bcs[0].nodes[:, None] + np.arange(3)).ravel()
    free = np.setdiff1d(np.arange(3 * V.node_count), bd)
    ref = np.zeros(3 * V.node_count)
    ref[free] = spla.spsolve(K[free][:, free].tocsc(), b.data_ro.ravel()[free])
    assert np.abs(x.data_ro.ravel() - ref).max() < 1e-9 * np.abs(ref).max()


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import test_hyperelastic_host_mock as tm
    from firedrake_b200.assemble import FunctionSpace, HyperElasticity, assemble, interpolate
    from firedrake_b200.partition import SlabPartition
    from firedrake_b200.utility_meshes import ExtrudedHexMesh
    from oracle import oracle
    key = lambda L: (L[:, 0] * 1000 + L[:, 1]) * 1000 + L[:, 2]
    out = {}
    ue = ["0.1 * sin(2.0 * x[0]) + 0.05 * x[1] * x[2]", "0.1 * x[0] - 0.05 * x[1] * x[2]", "0.08 * cos(x[1]) * x[0]"]
    we = ["sin(2.0 * x[0]) + x[1] * x[2]", "x[0] - 2.0 * x[1] * x[2]", "cos(x[1]) * x[0]"]
    with tm.install(oracle) as eng:
        nx, ny, nz, p = 5, 3, 4, 2
        eng.dist = None
        G = FunctionSpace(ExtrudedHexMesh(nx, ny, nz, warp=0.05), p, 3)
        J = HyperElasticity(G, 1.0, 1.5, 0.4).jacobian(interpolate(G, ue))
        gy = assemble(J, u=interpolate(G, we))
        gd = assemble(J, mat_type="matfree").getDiagonal(G.dat())
        look_y = dict(zip(key(G.V.dof_lattice()).tolist(), gy.data_ro.tolist()))
        look_d = dict(zip(key(G.V.dof_lattice()).tolist(), gd.data_ro.tolist()))
        eng.dist = dist
        part = SlabPartition(nx, ny, nz, p, rank, world, warp=0.05)
        V = FunctionSpace(part.mesh, p, 3, partition=part)
        u = interpolate(V, ue)
        no_ = V.V.owned_node_count
        u.data[no_:] = -1.0e3                      # stale ghost rows of u: Parloop must refresh them
        u.halo_valid = False
        Jp = HyperElasticity(V, 1.0, 1.5, 0.4).jacobian(u)
        y = assemble(Jp, u=interpolate(V, we))
        lat = V.V.dof_lattice()[:no_]
        out["action"] = float(np.abs(y.data_ro[:no_] - np.array([look_y[k] for k in key(lat).tolist()])).max())
        u.data[no_:] = -1.0e3
        u.halo_valid = False
        dd = assemble(Jp, mat_type="matfree").getDiagonal(V.dat())
        out["diag"] = float(np.abs(dd.data_ro[:no_] - np.array([look_d[k] for k in key(lat).tolist()])).max())
        out["scale"] = float(np.abs(gy.data_ro).max())
        out["dscale"] = float(np.abs(gd.data_ro).max())
    q.put((rank, out))
    dist.destroy_process_group()


def test_partitioned_world2_jacobian_reads_refreshed_ghosts():
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
