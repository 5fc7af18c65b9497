"""p-multigrid on the H100: the transfer kernels against the NumPy oracle (every degree pair and value size, atomic
and coloured restriction), their determinism and adjointness, the fused Chebyshev step, and P1PC / PMGPC solves
against Jacobi-CG's solution on meshes no hierarchy produces, with the forms the solvers take."""

import numpy as np
import pytest

import _pmg_oracle as po
from firedrake_b200 import _lib, mg, op2
from firedrake_b200.assemble import (AdvectionDiffusion, DirichletBC, Elasticity, Form, FunctionSpace,
                                     HyperElasticity, NonlinearDiffusion, assemble, mass, solve, solve_nonlinear)
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

PAIRS = [(2, 1), (3, 1), (3, 2)]


def _spaces(p, q, cdim, nx=3, ny=3, nz=2):
    mesh = ExtrudedHexMesh(nx, ny, nz, warp=0.05, permute_seed=5)
    return FunctionSpace(mesh, q, cdim), FunctionSpace(mesh, p, cdim)


def _rand(W, seed):
    shape = (W.node_count, W.cdim) if W.cdim > 1 else (W.node_count,)
    return np.random.default_rng(seed).standard_normal(shape)


def _rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


@pytest.mark.parametrize("p,q", PAIRS)
@pytest.mark.parametrize("cdim", [1, 3])
@pytest.mark.parametrize("scatter", ["atomic", "coloured"])
def test_transfers_match_oracle(engine, p, q, cdim, scatter):
    Vc, Vf = _spaces(p, q, cdim)
    T = mg.PTransfer(Vc, Vf, scatter=scatter)
    xc, xf = _rand(Vc, 1), _rand(Vf, 2)
    fine = T.prolong(Vc.dat(xc), Vf.dat())
    assert _rel(fine.data_ro, po.prolong(Vf.V, Vc.V, xc)) < 1e-14
    coarse = T.restrict(Vf.dat(xf), Vc.dat())
    assert _rel(coarse.data_ro, po.restrict_cellwise(Vf.V, Vc.V, xf)) < 1e-14
    inj = T.inject(Vf.dat(xf), Vc.dat())
    assert _rel(inj.data_ro, po.inject(Vf.V, Vc.V, xf)) < 1e-14
    # <P x, y> = <x, P^T y>
    assert abs(np.vdot(fine.data_ro, xf) - np.vdot(xc, coarse.data_ro)) < 1e-12 * abs(np.vdot(xc, coarse.data_ro))


@pytest.mark.parametrize("p,q", PAIRS)
def test_transfers_deterministic(engine, p, q):
    """Two coloured restrictions and two prolongations are bitwise equal: the prolongation is WRITE from every
    cell sharing a node, which stores the same bits from each (exact endpoint rows, one contraction order)."""
    Vc, Vf = _spaces(p, q, 1, 10, 9, 8)
    T = mg.PTransfer(Vc, Vf, scatter="coloured")
    xc, xf = Vc.dat(_rand(Vc, 3)), Vf.dat(_rand(Vf, 4))
    a, b = T.restrict(xf, Vc.dat()).data_ro.copy(), T.restrict(xf, Vc.dat()).data_ro.copy()
    assert np.array_equal(a, b)
    f1, f2 = T.prolong(xc, Vf.dat()).data_ro.copy(), T.prolong(xc, Vf.dat()).data_ro.copy()
    assert np.array_equal(f1, f2)
    # and each shared fine node holds what every one of its cells computes: the same as the oracle's rows
    assert _rel(f1, po.prolong(Vf.V, Vc.V, xc.data_ro)) < 1e-14


@pytest.mark.parametrize("p,q", PAIRS)
def test_prolong_writers_agree(engine, p, q):
    """Every cell that shares a fine node stores the same bits there: the columns split in two halves (a permuted
    numbering, so most faces are shared between them), prolonged half after half in both orders.  The last writer
    of every node on the interface changes with the order, and the results are bitwise equal."""
    Vc, Vf = _spaces(p, q, 3, 10, 9, 8)
    T = mg.PTransfer(Vc, Vf)
    xc = Vc.dat(_rand(Vc, 6))
    cols = np.arange(Vf.cell_set.size)
    halves = op2.Subset(Vf.cell_set, cols[::2]), op2.Subset(Vf.cell_set, cols[1::2])
    gk = op2.GlobalKernel(T._k["p_prolong"], [Vf.cell_node_map, T.cmap], extruded=True, subset=True)

    def run(order):
        f = Vf.dat()
        for S in order:
            op2.Parloop(gk, S, [f(op2.WRITE, Vf.cell_node_map), xc(op2.READ, T.cmap)])()
        return f.data_ro.copy()
    a, b = run(halves), run(halves[::-1])
    assert np.array_equal(a, b)
    assert np.array_equal(a, T.prolong(xc, Vf.dat()).data_ro)


def test_gl_element_refused_by_the_engine(engine):
    """A Gauss-Legendre (DQ) fine element has no nodes at the ends: P and R have no unit endpoint rows, and
    fdb_kernel_create_mixed refuses them."""
    from firedrake_b200.fiat_lite import interval_element
    Vc, Vf = _spaces(2, 1, 1)
    T = mg.PTransfer(Vc, Vf)
    k = op2.Kernel("p_prolong", degree=2, coarse_degree=1, element=interval_element(2, variant="gl"))
    gk = op2.GlobalKernel(k, [Vf.cell_node_map, T.cmap], extruded=True)
    with pytest.raises(_lib.EngineError, match="p_prolong needs GLL elements: row 0 of P"):
        gk.compile()


def test_transfer_refusals(engine):
    mesh = ExtrudedHexMesh(2, 2, 2)
    Vc, Vf = FunctionSpace(mesh, 1), FunctionSpace(mesh, 4)
    with pytest.raises(_lib.EngineError, match="p_prolong action: degree 4 outside 2..3"):
        mg.PTransfer(Vc, Vf).prolong(Vc.dat(), Vf.dat())
    with pytest.raises(NotImplementedError, match="DQ"):
        mg.PTransfer(FunctionSpace(mesh, 1, family="DQ"), FunctionSpace(mesh, 2))


def test_chebyshev_kernel(engine):
    n = 100003
    rng = np.random.default_rng(7)
    b, ax, dinv, d, x = (rng.standard_normal(n) for _ in range(5))
    L = _lib.lib()
    bufs = [L.fdb_malloc(8 * n) for _ in range(5)]
    try:
        for buf, v in zip(bufs, (b, ax, dinv, d, x)):
            _lib.check(L.fdb_memcpy_h2d(buf, v.ctypes.data, 8 * n))
        for cd, cz in ((0.0, 0.7), (0.3, 1.9)):
            _lib.check(L.fdb_vec_chebyshev(n, cd, cz, *bufs))
            po.chebyshev_step(cd, cz, b, ax, dinv, d, x)
        out = np.empty(n), np.empty(n)
        _lib.check(L.fdb_memcpy_d2h(out[0].ctypes.data, bufs[3], 8 * n))
        _lib.check(L.fdb_memcpy_d2h(out[1].ctypes.data, bufs[4], 8 * n))
    finally:
        for buf in bufs:
            L.fdb_free(buf)
    assert _rel(out[0], d) < 1e-15 and _rel(out[1], x) < 1e-15


PMG = {"pc_type": "python", "pc_python_type": "firedrake.PMGPC"}
P1 = {"pc_type": "python", "pc_python_type": "firedrake.P1PC"}


def _poisson(V, sp, bcs_domains=("bottom", "top"), form=None):
    bcs = [DirichletBC(V, 0.0, s) for s in bcs_domains]
    f = V.dat(np.sin(np.arange(V.node_count * V.cdim) * 0.37).reshape((V.node_count, V.cdim)).squeeze())
    L = assemble(mass(V), u=f)
    u = V.dat()
    its, hist = solve(form or Form(V, 1.0, 0.0), L, u, bcs=bcs, solver_parameters=dict(sp, ksp_rtol=1e-11))
    return u.data_ro.copy(), its


def _close(u, v, tol=1e-8):
    assert _rel(u, v) < tol, _rel(u, v)


@pytest.mark.parametrize("p", [2, 3])
@pytest.mark.parametrize("sp", [PMG, P1], ids=["pmgpc", "p1pc"])
def test_poisson_unstructured_size(engine, p, sp):
    """A warped, permuted 6 x 5 x 7 mesh: no hierarchy can produce it."""
    V = FunctionSpace(ExtrudedHexMesh(6, 5, 7, warp=0.05, permute_seed=0), p)
    uj, _ = _poisson(V, {"pc_type": "jacobi"})
    u, its = _poisson(V, sp)
    _close(u, uj)


# P1PC's outer iterations on the mock engine (tests/test_pmg_host_mock.py::test_iterations_on_mock, which checks
# there that they grow by at most 2 from 8^3 to 16^3 and are at least 3x fewer than Jacobi-CG's 215 and 395 at 16^3)
MOCK_ITS = {2: {8: 11, 16: 11}, 3: {8: 12, 16: 14}}


@pytest.mark.parametrize("p", [2, 3])
def test_poisson_iterations(engine, p):
    """P1PC's outer iterations at 8^3 and 16^3 are the mock engine's plus at most 1 (the atomic scatters round
    differently from run to run), and at least 3x fewer than Jacobi-CG's at 16^3."""
    its = {}
    for n in (8, 16):
        V = FunctionSpace(ExtrudedHexMesh(n, n, n, warp=0.05), p)
        uj, its_j = _poisson(V, {"pc_type": "jacobi"})
        u, its[n] = _poisson(V, P1)
        _close(u, uj)
    print(f"CG{p}: P1PC {its}, Jacobi-CG at 16^3 {its_j}")
    assert all(its[n] <= MOCK_ITS[p][n] + 1 for n in its), its
    assert 3 * its[16] <= its_j


def test_p1pc_coarse_mg_reaches_gmg(engine):
    h = mg.MeshHierarchy(4, 4, 4, 1, warp=0.05)
    V = FunctionSpace(h[1], 3)
    bcs = [DirichletBC(V, 0.0, s) for s in ("bottom", "top")]
    L = assemble(mass(V), u=V.dat(np.cos(np.arange(V.node_count) * 0.11)))
    ug, ui = V.dat(), V.dat()
    solve(Form(V), L, ug, bcs=bcs, hierarchy=h, solver_parameters={"pc_type": "mg", "ksp_rtol": 1e-11})
    its, _ = solve(Form(V), L, ui, bcs=bcs, hierarchy=h,
                   solver_parameters=dict(P1, ksp_rtol=1e-11, pmg_mg_coarse={"ksp_type": "preonly", "pc_type": "mg"}))
    _close(ui.data_ro, ug.data_ro)


@pytest.mark.parametrize("case", ["kappa", "robin", "elasticity", "advection_diffusion"])
def test_forms(engine, case):
    """A kappa field of contrast 100, a Robin ds term, vector Elasticity CG2 and AdvectionDiffusion under GMRES: PMG reaches the
    Jacobi solution."""
    mesh = ExtrudedHexMesh(6, 5, 7, warp=0.05, permute_seed=0)
    V = FunctionSpace(mesh, 3)
    sp, tol = dict(PMG), 1e-8
    if case == "kappa":
        # a contrast of 100 across the mesh.  A nodal step would not do: its CG3 interpolant overshoots below zero
        # next to the jump, and the operator is then indefinite (its diagonal has negative entries)
        X = V.V.dof_coordinates()
        form = Form(V, 1.0, 0.0, V.dat(10.0 ** (2.0 * X[:, 0])))
    elif case == "robin":
        form = Form(V, 1.0, 0.0, ds=((2.0, 1),))
    elif case == "elasticity":
        V = FunctionSpace(mesh, 2, 3)
        form = Elasticity(V, 1.0, 2.0)
    else:
        bvel = op2.Dat(V.vector_dset(3), np.tile([0.5, -0.2, 0.1], (V.node_count, 1)))
        form, sp, tol = AdvectionDiffusion(V, bvel, 1.0, 0.0), dict(PMG, ksp_type="gmres"), 1e-7
    uj = _poisson(V, dict(sp, pc_type="jacobi"), form=form)[0]
    _close(_poisson(V, sp, form=form)[0], uj, tol)


def test_newton(engine):
    mesh = ExtrudedHexMesh(5, 4, 6, warp=0.05, permute_seed=1)
    V = FunctionSpace(mesh, 2)
    bcs = [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, 1.0, "top")]
    L = assemble(mass(V), u=V.dat(np.ones(V.node_count)))
    out = []
    for sp in ({"pc_type": "jacobi"}, PMG):
        u = V.dat()
        hist, _ = solve_nonlinear(NonlinearDiffusion(V, 1.0, 0.0, (1.0, 0.5, 0.2)), L, u, bcs=bcs,
                                  solver_parameters=dict(sp, snes_rtol=1e-10, ksp_rtol=1e-8))
        out.append(u.data_ro.copy())
    _close(out[1], out[0], 1e-7)
    W = FunctionSpace(mesh, 2, 3)
    bcs = [DirichletBC(W, 0.0, "bottom"), DirichletBC(W, 0.05, "top")]
    out = []
    for sp in ({"pc_type": "jacobi"}, PMG):
        u = W.dat()
        solve_nonlinear(HyperElasticity(W, 1.0, 2.0), W.dat(), u, bcs=bcs,
                        solver_parameters=dict(sp, snes_rtol=1e-10, ksp_rtol=1e-8))
        out.append(u.data_ro.copy())
    _close(out[1], out[0], 1e-7)
