"""GPU checks of the spectral-element wave equation: FDB_FORM_SPECTRAL_HELMHOLTZ[_COEF] (csrc/sem_hex.cu) against the
NumPy oracle (tests/_sem_oracle.py), helmholtz_coef on the GLL tables and the generic-path statement; the lumped
mass, solves, the engine's refusals, point sources and receivers (csrc/point_hex.cu), and the leapfrog stepper
(fdb_vec_leapfrog) against the oracle's recurrence, its energy and its second order in time."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import _boundary_oracle as bo
import _sem_oracle as so
from firedrake_b200 import _lib, op2
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

TOL = 1e-12


def relerr(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(b).max()


def warped(nx=3, ny=2, nz=3, seed=1):
    """Vertices moved in and out of plane (the mesh's warp and a seeded random perturbation)."""
    return bo.perturb(ExtrudedHexMesh(nx, ny, nz, Lx=1.2, Ly=0.9, Lz=1.1, warp=0.05, permute_seed=seed), 0.08, seed)


def space(mesh, p):
    from firedrake_b200.assemble import FunctionSpace
    return FunctionSpace(mesh, p)


def values(n, seed, lo=None):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(n) if lo is None else rng.uniform(lo, lo + 1.0, n)


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
def test_action_and_diagonal_match_oracle(engine, p):
    """Extruded warped mesh: action and diagonal, with and without kappa, atomic and coloured (coloured twice:
    bitwise the same)."""
    from firedrake_b200.assemble import ImplicitMatrixContext, OneFormAssembler, SpectralForm
    mesh = warped(seed=p)
    V = space(mesh, p)
    x = V.dat(values(V.node_count, p))
    kap = values(V.node_count, 50 + p, lo=0.5)
    for kappa in (None, kap):
        F = SpectralForm(V, 0.7, 0.4, None if kappa is None else V.dat(kappa))
        A = so.operator(mesh, V.V, p, 0.7, 0.4, kappa)
        want = A @ x.data_ro
        outs = []
        for scatter in ("atomic", "coloured", "coloured"):
            y = OneFormAssembler(F, x, scatter=scatter).assemble()
            assert relerr(y.data_ro, want) < TOL, (scatter, kappa is None)
            outs.append(y.data_ro.copy())
        assert np.array_equal(outs[1], outs[2])
        d = ImplicitMatrixContext(F).getDiagonal(V.dat())
        assert relerr(d.data_ro, A.diagonal()) < TOL
        dk = F.kernel(1, diagonal=True)
        dc = [V.dat(), V.dat()]
        for t in dc:
            op2.par_loop(dk, V.cell_set, t(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                         *F.coefficient_args(), scatter="coloured")
        assert relerr(dc[0].data_ro, A.diagonal()) < TOL and np.array_equal(dc[0].data_ro, dc[1].data_ro)


@pytest.mark.parametrize("p", [1, 3, 5])
def test_native_hexes(engine, p):
    """The op2 level on native hexes (permuted full rows): action and diagonal with kappa, atomic and coloured."""
    mesh = warped(3, 2, 3, seed=40 + p)
    W = mesh.function_space(p)
    perm = np.random.default_rng(p).permutation(mesh.num_cells)
    full, cfull = W.full_cell_node_list()[perm], mesh.coord_space.full_cell_node_list()[perm]
    nodes, vnodes = op2.Set(W.node_count), op2.Set(mesh.coord_space.node_count)
    X = op2.Dat(op2.DataSet(vnodes, 3), mesh.coordinates)
    kap = values(W.node_count, 9, lo=0.5)
    K = op2.Dat(nodes, kap)
    u = op2.Dat(nodes, values(W.node_count, 3))
    cset = op2.Set(mesh.num_cells)
    m0 = op2.Map(cset, nodes, W.arity, np.ascontiguousarray(full))
    m1 = op2.Map(cset, vnodes, 8, np.ascontiguousarray(cfull))
    A = so.operator(mesh, W, p, 1.3, 0.2, kap)
    k = op2.Kernel("spectral_helmholtz_coef", degree=p, alpha=1.3, beta=0.2)
    kd = op2.Kernel("spectral_helmholtz_coef", degree=p, alpha=1.3, beta=0.2, diagonal=True)
    outs = []
    for scatter in ("atomic", "coloured", "coloured"):
        y = op2.Dat(nodes)
        op2.par_loop(k, cset, y(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), K(op2.READ, m0), scatter=scatter)
        assert relerr(y.data_ro, A @ u.data_ro) < TOL, scatter
        outs.append(y.data_ro.copy())
        d = op2.Dat(nodes)
        op2.par_loop(kd, cset, d(op2.INC, m0), X(op2.READ, m1), K(op2.READ, m0), scatter=scatter)
        assert relerr(d.data_ro, A.diagonal()) < TOL, scatter
    assert np.array_equal(outs[1], outs[2])
    A0 = so.operator(mesh, W, p, 1.0, 0.0)
    y = op2.Dat(nodes)
    op2.par_loop(op2.Kernel("spectral_helmholtz", degree=p), cset, y(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0))
    assert relerr(y.data_ro, A0 @ u.data_ro) < TOL


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
def test_equals_helmholtz_coef_on_gll_tables(engine, p):
    """The same discrete operator as helmholtz_coef given the GLL tables, and (p <= 3) the generic-path statement."""
    from firedrake_b200 import codegen
    from firedrake_b200.assemble import OneFormAssembler, SpectralForm, spectral_helmholtz_kernel
    from firedrake_b200.fiat_lite import interval_element
    mesh = warped(seed=60 + p)
    V = space(mesh, p)
    x = V.dat(values(V.node_count, p))
    kap = V.dat(values(V.node_count, 70 + p, lo=0.5))
    y = OneFormAssembler(SpectralForm(V, 1.1, 0.3, kap), x).assemble()
    z = V.dat()
    k = op2.Kernel("helmholtz_coef", degree=p, alpha=1.1, beta=0.3, element=interval_element(p, quadrature="gll"))
    op2.par_loop(k, V.cell_set, z(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                 x(op2.READ, V.cell_node_map), kap(op2.READ, V.cell_node_map))
    assert relerr(y.data_ro, z.data_ro) < TOL
    if p <= 3:
        g = V.dat()
        codegen.par_loop(spectral_helmholtz_kernel(p, 1.1, 0.3, coef=True), V.cell_set, g(op2.INC, V.cell_node_map),
                         V.coordinates(op2.READ, V.coord_map), x(op2.READ, V.cell_node_map),
                         kap(op2.READ, V.cell_node_map))
        assert relerr(y.data_ro, g.data_ro) < TOL


@pytest.mark.parametrize("p", [2, 5])
def test_mass_action_is_lumped_mass(engine, p):
    from firedrake_b200.assemble import SpectralForm, assemble, lumped_mass
    mesh = warped(seed=80 + p)
    V = space(mesh, p)
    x = V.dat(values(V.node_count, p))
    rho = values(V.node_count, 3, lo=1.0)
    y = assemble(SpectralForm(V, 0.0, 1.0), u=x)
    m = lumped_mass(V)
    assert relerr(y.data_ro, m.data_ro * x.data_ro) < 1e-14
    assert relerr(lumped_mass(V, V.dat(rho)).data_ro, m.data_ro * rho) < 1e-15
    assert relerr(m.data_ro, so.operator(mesh, V.V, p, 0.0, 1.0).diagonal()) < TOL


def _desc(p, **kw):
    from firedrake_b200.fiat_lite import interval_element
    el = interval_element(p, quadrature="gll") if 1 <= p <= 7 else interval_element(1, quadrature="gll")
    d = _lib.KernelDesc()
    d.form, d.rank, d.cell, d.integral = _lib.FORM_SPECTRAL_HELMHOLTZ, 1, _lib.CELL_HEX, _lib.INTEGRAL_CELL
    d.degree, d.nq, d.cdim, d.alpha = p, el.nq, 1, 1.0
    n = el.nq
    for q in range(n):
        d.wq[q], d.xq[q] = el.wq[q], el.xq[q]
        for a in range(n):
            d.B[q * n + a], d.D[q * n + a] = el.B[q, a], el.D[q, a]
    for key, v in kw.items():
        if key == "B01":
            d.B[1] = v
        elif key == "xq0":
            d.xq[0] = v
        else:
            setattr(d, key, v)
    return d


@pytest.mark.parametrize("case, match", [
    (dict(B01=1e-17), "B must be exactly the identity"),
    (dict(nq=4), "nq == degree\\+1"),
    (dict(xq0=1e-300), "xq\\[0\\] == 0 and xq\\[1\\] == 1"),
    (dict(rank=2), "no assembled SEM matrix"),
    (dict(cdim=3), "scalar spaces only"),
    (dict(affine_cells=1), "no affine-cell variant"),
    (dict(degree=6, nq=7), "degree 6 outside 1..5"),
])
def test_create_refusals(engine, case, match):
    import ctypes as C
    d = _desc(2 if "degree" not in case else case["degree"], **{k: v for k, v in case.items() if k != "degree"})
    h = C.c_void_p()
    assert engine.fdb_kernel_create(C.byref(d), C.byref(h)) != 0
    msg = engine.fdb_last_error().decode()
    assert "spectral_helmholtz" in msg
    import re
    assert re.search(match, msg), msg


def test_host_pointer_mode_refused(engine):
    from firedrake_b200.assemble import SpectralForm
    V = space(ExtrudedHexMesh(2, 2, 2), 2)
    F = SpectralForm(V)
    x, y = V.dat(np.ones(V.node_count)), V.dat()
    with pytest.raises(_lib.EngineError, match="device-resident Dats only"):
        op2.par_loop(F.kernel(1), V.cell_set, y(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                     x(op2.READ, V.cell_node_map), location="host")


@pytest.mark.parametrize("p", [4, 5])
def test_solve_cg_and_jacobi(engine, p):
    from firedrake_b200.assemble import DirichletBC, SpectralForm, assemble, solve
    mesh = warped(3, 2, 2, seed=90 + p)
    V = space(mesh, p)
    kap = values(V.node_count, 5, lo=0.5)
    F = SpectralForm(V, 1.0, 0.5, V.dat(kap))
    f = V.dat(values(V.node_count, 6))
    L = assemble(SpectralForm(V, 0.0, 1.0), u=f)
    A = so.operator(mesh, V.V, p, 1.0, 0.5, kap).tocsc()
    bc = DirichletBC(V, 0.0, "bottom")
    fixed = np.asarray(bc.nodes)
    free = np.setdiff1d(np.arange(V.node_count), fixed)
    want = np.zeros(V.node_count)
    want[free] = spla.spsolve(A[free][:, free], L.data_ro[free])
    its = {}
    for pc in ("none", "jacobi"):
        u = V.dat()
        its[pc], _ = solve(F, L, u, bcs=[bc], solver_parameters={"pc_type": pc, "ksp_rtol": 1e-12,
                                                                  "ksp_max_it": 3000})
        assert relerr(u.data_ro, want) < 1e-9, pc
    assert its["jacobi"] < its["none"]


def _ricker_setup(p=3, n=16):
    from firedrake_b200.assemble import PointEvaluator, SpectralForm, lumped_mass, wave_dt_bound
    mesh = bo.perturb(ExtrudedHexMesh(n, n, n, warp=0.05, permute_seed=1), 0.05, 1)
    V = space(mesh, p)
    z = V.V.dof_coordinates()[:, 2]
    kap = np.where(z > 0.5, 2.25, 1.0)                         # two layers: c = 1 and 1.5
    F = SpectralForm(V, 1.0, 0.0, V.dat(kap))
    m = lumped_mass(V)
    src = PointEvaluator(V, [[0.5, 0.5, 0.3]])
    rec = PointEvaluator(V, [[0.2, 0.5, 0.6], [0.35, 0.5, 0.7], [0.5, 0.5, 0.8], [0.65, 0.45, 0.7],
                             [0.8, 0.55, 0.6]])
    return mesh, V, kap, F, m, src, rec, wave_dt_bound(F, m)


def test_ricker_traces_match_oracle(engine):
    """A Ricker source, five receivers, 200 steps on a warped 16^3 CG3 mesh with a two-layer kappa: the traces agree
    with the oracle's leapfrog to 1e-10 relative and are bitwise repeatable."""
    from firedrake_b200.assemble import leapfrog, ricker
    mesh, V, kap, F, m, src, rec, dtb = _ricker_setup()
    steps, dt = 200, 0.8 * dtb
    amp = ricker(np.arange(steps) * dt, 6.0, 0.2)[:, None] * 1e3
    traces = []
    for _ in range(2):
        u, up = V.dat(), V.dat()
        traces.append(leapfrog(F, u, up, dt, steps, m, sources=(src, amp), receivers=rec))
    assert np.array_equal(traces[0], traces[1])
    K = so.operator(mesh, V.V, 3, 1.0, 0.0, kap)
    uo, upo, tro = so.leapfrog(K, m.data_ro, np.zeros(V.node_count), np.zeros(V.node_count), dt, steps,
                               src=(src.idx, src.w), amp=amp, rec=(rec.idx, rec.w))
    assert np.abs(tro).max() > 0
    assert relerr(traces[0], tro) < 1e-10
    assert relerr(u.data_ro, uo) < 1e-10 and relerr(up.data_ro, upo) < 1e-10


def test_point_eval_and_load(engine):
    """evaluate and adjoint against the oracle's E and E^T; shared nodes and missing points; bitwise repeatable."""
    from firedrake_b200.assemble import PointEvaluator
    mesh = warped(3, 3, 3, seed=4)
    V = space(mesh, 3)
    Xd = V.V.dof_coordinates()
    pts = np.concatenate([Xd[[5, 5, 17]], Xd[[40, 41]] * 0.99 + 0.003, [[5.0, 5.0, 5.0]]])
    pe = PointEvaluator(V, pts, missing_points_behaviour="ignore")
    u = V.dat(values(V.node_count, 1))
    out = pe.evaluate(u)
    want = so.evaluate((pe.idx, pe.w), u.data_ro)
    assert np.isnan(out[-1]) and np.array_equal(np.isnan(out), np.isnan(want))
    assert relerr(out[:-1], want[:-1]) < 1e-14
    a = values(len(pts), 2)
    ys = [pe.adjoint(a).data_ro.copy() for _ in range(2)]
    assert np.array_equal(ys[0], ys[1])
    assert relerr(ys[0], so.adjoint((pe.idx, pe.w), a, V.node_count)) < 1e-14


def test_energy_drift(engine):
    """Without a source, 2000 steps at 0.9 wave_dt_bound keep the discrete energy to 1e-10 relative."""
    from firedrake_b200.assemble import SpectralForm, assemble, leapfrog, lumped_mass, wave_dt_bound
    mesh = warped(5, 4, 4, seed=11)
    V = space(mesh, 2)
    kap = np.where(V.V.dof_coordinates()[:, 2] > 0.5, 2.0, 1.0)
    F = SpectralForm(V, 1.0, 0.0, V.dat(kap))
    m = lumped_mass(V)
    dt = 0.9 * wave_dt_bound(F, m)
    mv = m.data_ro.copy()
    u0 = values(V.node_count, 3)

    def energy(un, uo):
        Ku = assemble(F, u=V.dat(uo)).data_ro
        v = (un - uo) / dt
        return 0.5 * v @ (mv * v) + 0.5 * un @ Ku

    u, up = V.dat(u0.copy()), V.dat(u0.copy())      # (a Dat wraps its array)
    leapfrog(F, u, up, dt, 1, m)
    E0 = energy(u.data_ro.copy(), up.data_ro.copy())
    leapfrog(F, u, up, dt, 2000, m)
    E1 = energy(u.data_ro.copy(), up.data_ro.copy())
    assert abs(E1 - E0) < 1e-10 * abs(E0), (E0, E1)


def test_second_order_in_time(engine):
    """The standing wave cos(pi x) cos(pi y) cos(pi z) cos(sqrt(3) pi t) on the unit cube (natural boundary) at CG5 on
    4^3 cells, where the time error dominates: halving dt divides the error at t = T by 3.5..4.5."""
    from firedrake_b200.assemble import SpectralForm, leapfrog, lumped_mass, wave_dt_bound
    mesh = ExtrudedHexMesh(4, 4, 4)
    V = space(mesh, 5)
    X = V.V.dof_coordinates()
    mode = np.cos(np.pi * X[:, 0]) * np.cos(np.pi * X[:, 1]) * np.cos(np.pi * X[:, 2])
    w = np.sqrt(3.0) * np.pi
    F = SpectralForm(V)
    m = lumped_mass(V)
    T = 0.6
    n0 = int(np.ceil(T / (0.9 * wave_dt_bound(F, m))))
    errs = []
    for steps in (n0, 2 * n0):
        dt = T / steps
        u, up = V.dat(mode.copy()), V.dat(mode * np.cos(-w * dt))
        leapfrog(F, u, up, dt, steps, m)
        errs.append(np.abs(u.data_ro - mode * np.cos(w * T)).max())
    assert 3.5 <= errs[0] / errs[1] <= 4.5, errs


def test_form_refusals(engine):
    from firedrake_b200.assemble import FunctionSpace, SpectralForm, assemble, solve
    mesh = ExtrudedHexMesh(2, 2, 2)
    V = space(mesh, 2)
    F = SpectralForm(V)
    with pytest.raises(NotImplementedError, match="no assembled SEM matrix"):
        assemble(F)
    L = V.dat(np.ones(V.node_count))
    for sp, match in ((dict(mat_type="aij"), "no assembled SEM matrix"), (dict(pc_type="mg"), "geometric multigrid"),
                      (dict(pc_type="python", pc_python_type="firedrake.PMGPC"), "p-multigrid")):
        with pytest.raises(NotImplementedError, match=match):
            solve(F, L, V.dat(), solver_parameters=sp)
    with pytest.raises(NotImplementedError, match="DQ"):
        SpectralForm(FunctionSpace(mesh, 2, family="DQ"))
    with pytest.raises(NotImplementedError, match="scalar"):
        SpectralForm(FunctionSpace(mesh, 2, cdim=3))
    with pytest.raises(NotImplementedError, match="ds terms"):
        SpectralForm(V, ds=((1.0, "bottom"),))
