"""GPU tests of Neo-Hookean hyperelasticity (FDB_FORM_HYPERELASTICITY[_JACOBIAN], csrc/elasticity_hex.cu):
the residual and the Jacobian action, blocked matrix and diagonal against the NumPy oracle
(tests/_hyperelastic_oracle.py) and the generic wrapper path; the Jacobian at u = 0 against linear
elasticity; frame indifference and the Taylor test; the refusals of fdb_kernel_create and
fdb_kernel_call; Newton solves (a homogeneous-deformation patch test with every preconditioner, a
twisted and compressed cube against scipy's Newton, the L2 rates of a manufactured solution, multigrid
iteration counts) and the solver's error on an inverted element.  Tolerance 1e-12 relative in the max
norm.

Every test takes the engine as its first argument, so tests/test_hyperelastic_host_mock.py runs the same
host logic on the CPU against a mock engine."""
import functools

import numpy as np
import pytest

import _hyperelastic_oracle as ho
from firedrake_b200 import op2
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh
from test_coefficient_gpu import relerr, setup
from test_hyperelastic_oracle import _smooth

pytestmark = pytest.mark.gpu

TOL = 1e-12
MU, LMBDA = 1.3, 2.1
ALL_FACES = (1, 2, 3, 4, "bottom", "top")


def vec_values(n, seed=0):
    return np.random.default_rng(seed).standard_normal((n, 3))


def _parity(engine, p, native, jacobian, beta):
    mesh, V, cells, nodes, m0, m1, X, omaps = setup(p, native)
    vset = op2.DataSet(nodes, 3)
    u = op2.Dat(vset, _smooth(V.dof_coordinates()).reshape(-1, 3))
    w = op2.Dat(vset, vec_values(V.node_count, p))
    el = interval_element(p)
    if jacobian:
        want = ho.jacobian_action(el, mesh.coordinates, u.data_ro.ravel().copy(), w.data_ro.ravel().copy(), *omaps,
                                  MU, LMBDA, beta)
        k = op2.Kernel("hyperelasticity_jacobian", degree=p, mu=MU, lmbda=LMBDA, beta=beta, cdim=3)
        ins = [w(op2.READ, m0), u(op2.READ, m0)]
    else:
        want = ho.residual(el, mesh.coordinates, u.data_ro.ravel().copy(), *omaps, MU, LMBDA, beta)
        k = op2.Kernel("hyperelasticity", degree=p, mu=MU, lmbda=LMBDA, beta=beta, cdim=3)
        ins = [u(op2.READ, m0)]
    y = op2.Dat(vset)
    op2.par_loop(k, cells, y(op2.INC, m0), X(op2.READ, m1), *ins)
    assert relerr(y.data_ro.ravel(), want) < TOL
    outs = []
    for _ in range(2):
        y.zero()
        op2.par_loop(k, cells, y(op2.INC, m0), X(op2.READ, m1), *ins, scatter="coloured")
        outs.append(y.data_ro.copy())
    assert np.array_equal(outs[0], outs[1])
    assert relerr(outs[0].ravel(), want) < TOL


@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
def test_residual_matches_oracle(engine, p, native):
    """Atomic and coloured scatter; coloured is bit-identical across calls."""
    _parity(engine, p, native, False, 0.6)


@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
def test_jacobian_action_matches_oracle(engine, p, native):
    _parity(engine, p, native, True, 0.6)


def _space(p, mesh=None):
    from firedrake_b200.assemble import FunctionSpace
    return FunctionSpace(mesh or ExtrudedHexMesh(4, 3, 5, warp=0.05, permute_seed=2), p, 3)


def _u(V, amp=0.1):
    return V.dat(_smooth(V.V.dof_coordinates(), amp).reshape(-1, 3))


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_matches_generic_path(engine, p):
    from firedrake_b200.assemble import HyperElasticity, assemble, assemble_hyperelasticity_generic
    V = _space(p)
    u, w = _u(V), V.dat(vec_values(V.node_count, 3))
    F = HyperElasticity(V, MU, LMBDA, 0.4)
    r = assemble(F, u=u).data_ro.copy()
    assert relerr(r, assemble_hyperelasticity_generic(V, u, MU, LMBDA, 0.4).data_ro) < TOL
    jw = assemble(F.jacobian(u), u=w).data_ro.copy()
    assert relerr(jw, assemble_hyperelasticity_generic(V, u, MU, LMBDA, 0.4, w=w).data_ro) < TOL


def test_host_pointer_mode_equals_device_mode(engine):
    """Host-resident Dats through the mirror cache (the monolithic path), residual and Jacobian action; a
    host write to u is picked up."""
    p = 3
    mesh, V, cells, nodes, m0, m1, X, _ = setup(p, False, ExtrudedHexMesh(4, 4, 6, warp=0.05))
    vset = op2.DataSet(nodes, 3)
    u = op2.Dat(vset, _smooth(V.dof_coordinates()).reshape(-1, 3))
    w = op2.Dat(vset, vec_values(V.node_count, 9))
    for name, ins in (("hyperelasticity", [u]), ("hyperelasticity_jacobian", [w, u])):
        k = op2.Kernel(name, degree=p, mu=MU, lmbda=LMBDA, beta=0.2, cdim=3)
        yd, yh = op2.Dat(vset), op2.Dat(vset)
        dev = lambda: op2.par_loop(k, cells, yd(op2.INC, m0), X(op2.READ, m1), *[a(op2.READ, m0) for a in ins])
        dev()
        gk = op2.GlobalKernel(k, [m0, m1], extruded=True)
        loop = op2.Parloop(gk, cells, [yh(op2.INC, m0), X(op2.READ, m1)] + [a(op2.READ, m0) for a in ins],
                           location="host")
        loop()
        assert relerr(yh.data_ro, yd.data_ro) < TOL
        u.data[:] *= 0.5
        yh.zero()
        loop()
        yd.zero()
        dev()
        assert relerr(yh.data_ro, yd.data_ro) < TOL


def _bcs(V):
    from firedrake_b200.assemble import DirichletBC
    return [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, 0.0, 2)]


def _block_diagonal(ro, ci, vals, n):
    blocks = vals.reshape(-1, 3, 3)
    return np.array([np.diagonal(blocks[ro[r] + np.searchsorted(ci[ro[r]:ro[r + 1]], r)]) for r in range(n)])


@pytest.mark.parametrize("p", [1, 2, 3])
def test_jacobian_blocked_matrix_matches_oracle(engine, p):
    """Entrywise against the oracle's element Jacobians added through the dof-level BC-masked lgmaps, unit
    diagonal on the constrained rows; symmetric."""
    import _elasticity_oracle as eo
    from firedrake_b200.assemble import HyperElasticity, assemble
    mesh = ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=2)
    V = _space(p, mesh)
    bcs = _bcs(V)
    u = _u(V, 0.2)
    A = assemble(HyperElasticity(V, MU, LMBDA, 0.7).jacobian(u), bcs=bcs)
    ro, ci, vals = A.csr()
    bn = np.unique(np.concatenate([bc.nodes for bc in bcs]))
    lg = np.arange(3 * V.node_count, dtype=np.int32).reshape(-1, 3)
    lg[bn] = -1
    lg = lg.ravel()
    di, Ae = ho.element_matrices(interval_element(p), mesh.coordinates, u.data_ro.ravel().copy(), V.V.cell_node_map,
                                 V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz, MU, LMBDA, 0.7)
    vo = eo.add_to_bcsr(ro, ci, np.zeros(len(vals)), di, Ae, lg, lg)
    blocks = vo.reshape(-1, 3, 3)
    for r in bn:
        k = ro[r] + np.searchsorted(ci[ro[r]:ro[r + 1]], r)
        blocks[k][np.diag_indices(3)] = 1.0
    scale = np.abs(vo).max()
    assert np.abs(vals - vo).max() < TOL * scale
    K = eo.to_dense(ro, ci, vals)
    assert np.abs(K - K.T).max() < TOL * scale


@pytest.mark.parametrize("p", [1, 2, 3])
@pytest.mark.parametrize("with_bcs", [False, True], ids=["nobc", "bc"])
def test_mat_mult_equals_matfree(engine, p, with_bcs):
    from firedrake_b200.assemble import HyperElasticity, assemble
    V = _space(p, ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=3))
    bcs = _bcs(V) if with_bcs else ()
    J = HyperElasticity(V, MU, LMBDA, 0.3).jacobian(_u(V))
    x = V.dat(vec_values(V.node_count, 6))
    y, ymf, yt = V.dat(), V.dat(), V.dat()
    assemble(J, bcs=bcs).mult(x, y)
    mf = assemble(J, bcs=bcs, mat_type="matfree")
    mf.mult(x, ymf)
    assert relerr(y.data_ro, ymf.data_ro) < TOL
    mf.multTranspose(x, yt)                      # symmetric: the same operator
    assert relerr(yt.data_ro, ymf.data_ro) < TOL


@pytest.mark.parametrize("p", [1, 2, 3])
def test_diagonal_equals_assembled_diagonal(engine, p):
    from firedrake_b200.assemble import HyperElasticity, assemble
    V = _space(p, ExtrudedHexMesh(3, 2, 4, warp=0.05, permute_seed=3))
    J = HyperElasticity(V, MU, LMBDA, 0.3).jacobian(_u(V))
    bcs = _bcs(V)
    d = assemble(J, bcs=bcs, mat_type="matfree").getDiagonal(V.dat()).data_ro.copy()
    ro, ci, vals = assemble(J, bcs=bcs).csr()
    assert relerr(d, _block_diagonal(ro, ci, vals, V.node_count)) < TOL


@pytest.mark.parametrize("p", [1, 2, 3])
def test_jacobian_at_zero_equals_elasticity(engine, p):
    """J(0) is Elasticity(V, mu, lmbda, beta): action, blocked matrix and diagonal."""
    from firedrake_b200.assemble import Elasticity, HyperElasticity, assemble
    V = _space(p, ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=1))
    J = HyperElasticity(V, MU, LMBDA, 0.5).jacobian(V.dat())
    E = Elasticity(V, MU, LMBDA, 0.5)
    w = V.dat(vec_values(V.node_count, 2))
    assert relerr(assemble(J, u=w).data_ro, assemble(E, u=w).data_ro) < TOL
    bcs = _bcs(V)
    _, _, vj = assemble(J, bcs=bcs).csr()
    _, _, ve = assemble(E, bcs=bcs).csr()
    assert relerr(vj, ve) < TOL
    dj = assemble(J, bcs=bcs, mat_type="matfree").getDiagonal(V.dat()).data_ro
    de = assemble(E, bcs=bcs, mat_type="matfree").getDiagonal(V.dat()).data_ro
    assert relerr(dj, de) < TOL


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_rigid_rotation_has_zero_residual(engine, p):
    """u = (Q - I) X for a 60 degree rotation, beta = 0: P(Q) = 0, so the residual vanishes to rounding."""
    from firedrake_b200.assemble import HyperElasticity, assemble
    V = _space(p, ExtrudedHexMesh(3, 3, 4, warp=0.06, permute_seed=1))
    Xn = V.V.dof_coordinates()
    Q = ho.rotation((1.0, 0.5, -0.3), np.pi / 3)
    F = HyperElasticity(V, MU, LMBDA)
    scale = np.abs(assemble(F, u=_u(V)).data_ro).max() / 0.1
    r = assemble(F, u=V.dat(Xn @ Q.T - Xn)).data_ro
    assert np.abs(r).max() < 1e-12 * scale


@pytest.mark.parametrize("p", [1, 2, 3])
def test_taylor_ratio_is_four(engine, p):
    """|R(u + h w) - R(u) - h J(u) w| falls by 4 when h halves."""
    from firedrake_b200.assemble import HyperElasticity, assemble
    V = _space(p)
    F = HyperElasticity(V, MU, LMBDA, 0.2)
    u = _u(V)
    w = V.dat(0.1 * vec_values(V.node_count, 4))
    r0 = assemble(F, u=u).data_ro.copy()
    jw = assemble(F.jacobian(u), u=w).data_ro.copy()
    e = []
    for h in (2e-3, 1e-3, 5e-4):
        r = assemble(F, u=V.dat(u.data_ro + h * w.data_ro)).data_ro
        e.append(np.abs(r - r0 - h * jw).max())
    ratios = np.array(e[:-1]) / np.array(e[1:])
    assert np.all(np.abs(ratios - 4.0) < 0.3), (e, ratios)


def test_refuses_what_it_does_not_cover(engine):
    """fdb_kernel_create: scalar or 2-component spaces, non-hex cells, the affine variant, another
    quadrature, the residual as a matrix or diagonal, degrees outside 1..4 (action) and 1..3 (matrix,
    diagonal).  fdb_kernel_call: a Mat whose block size is not 3, and wrong argument counts."""
    from firedrake_b200 import _lib
    mesh, V, cells, nodes, m0, m1, X, _ = setup(2, False, ExtrudedHexMesh(2, 2, 2))
    E = dict(mu=MU, lmbda=LMBDA)
    for form in ("hyperelasticity", "hyperelasticity_jacobian"):
        cases = [(dict(degree=2, cdim=1), "value size 3"), (dict(degree=2, cdim=2), "value size 3"),
                 (dict(degree=1, cdim=3, cell="triangle"), "hex cells"),
                 (dict(degree=2, cdim=3, affine=True), "affine"),
                 (dict(degree=2, cdim=3, element=interval_element(2, 4)), "nq == degree"),
                 (dict(degree=5, cdim=3), "degree 5 outside 1..4")]
        if form == "hyperelasticity":
            cases += [(dict(degree=2, cdim=3, rank=2), "1-form action only"),
                      (dict(degree=2, cdim=3, diagonal=True), "1-form action only")]
        else:
            cases += [(dict(degree=4, cdim=3, rank=2), "degree 4 outside 1..3"),
                      (dict(degree=4, cdim=3, diagonal=True), "degree 4 outside 1..3")]
        for kw, msg in cases:
            gk = op2.GlobalKernel(op2.Kernel(form, **E, **kw), [m0, m1], extruded=True)
            with pytest.raises(_lib.EngineError, match=msg):
                gk.compile()
    vset = op2.DataSet(nodes, 3)
    u, y = op2.Dat(vset), op2.Dat(vset)
    mat = op2.Mat(op2.Sparsity((nodes, nodes), [(m0, m0, None)]))
    with pytest.raises(_lib.EngineError, match="block size 1"):
        op2.par_loop(op2.Kernel("hyperelasticity_jacobian", degree=2, rank=2, cdim=3, **E), cells,
                     mat(op2.INC, (m0, m0)), X(op2.READ, m1), u(op2.READ, m0))
    # wrong argument counts straight through the C ABI (op2.Parloop checks them against the kernel first)
    layers = np.array([0, mesh.layers], dtype=np.int32)
    maps = [m0.device_ptr, m1.device_ptr]
    for kw, args, msg in ((dict(), [y, X, u], "expects 4 args"), (dict(diagonal=True), [y, X], "expects 3 device args"),
                          (dict(rank=2), [mat, X], "expects 3 args")):
        gk = op2.GlobalKernel(op2.Kernel("hyperelasticity_jacobian", degree=2, cdim=3, **E, **kw), [m0, m1],
                              extruded=True)
        ptrs = [a.handle.value if isinstance(a, op2.Mat) else a.device_ptr for a in args]
        with pytest.raises(_lib.EngineError, match=msg):
            gk(0, mesh.num_base_cells, layers, None, ptrs, None, None, maps, None, _lib.LOC_DEVICE, False, False)


# ------------------------------------------------------------------------------------------------ solves
def _newton_params(pc, **kw):
    sp = {"pc_type": pc, "snes_rtol": 1e-13, "snes_max_it": 12, "ksp_rtol": 1e-10, "ksp_max_it": 3000}
    sp.update(kw)
    return sp


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
@pytest.mark.parametrize("p", [1, 2])
def test_homogeneous_deformation_patch_test(engine, pc, p):
    """u* = (A - I) X with det A > 0 on all six faces, zero load, beta = 0: Newton recovers u* at every
    node of a warped mesh, and its last steps converge quadratically."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import DirichletBC, FunctionSpace, HyperElasticity, interpolate, solve_nonlinear
    h = mg.MeshHierarchy(2, 2, 2, 1, warp=0.05) if pc == "mg" else None
    V = FunctionSpace(h[1] if h is not None else ExtrudedHexMesh(4, 4, 4, warp=0.05, permute_seed=1), p, 3)
    A = ho.HOMOGENEOUS_A
    g = interpolate(V, [" + ".join([f"{float(A[a][k] - (a == k))!r} * x[{k}]" for k in range(3)]) for a in range(3)])
    u = V.dat()
    hist, kits = solve_nonlinear(HyperElasticity(V, MU, LMBDA), V.dat(), u, bcs=[DirichletBC(V, g, ALL_FACES)],
                                 hierarchy=h, solver_parameters=_newton_params(pc))
    assert np.abs(u.data_ro - g.data_ro).max() < 1e-9, (pc, hist, kits)
    assert ho.converges_quadratically(hist), hist


# twisted cube: clamped bottom; the top turned by TWIST about the vertical axis through its centre and
# moved down by SQUEEZE, in STEPS load increments
TWIST, SQUEEZE, STEPS, NEWTON_BUDGET = np.pi / 6, 0.1, 4, 8


def _top_expressions(s):
    t, d = TWIST * s, SQUEEZE * s
    c, sn = repr(float(np.cos(t))), repr(float(np.sin(t)))
    return [f"{c} * (x[0] - 0.5) - {sn} * (x[1] - 0.5) + 0.5 - x[0]",
            f"{sn} * (x[0] - 0.5) + {c} * (x[1] - 0.5) + 0.5 - x[1]", repr(-d)]


def twisted_cube(n, p, pc="none", hierarchy=None, beta=0.0, ksp_rtol=1e-8, steps=STEPS):
    """Solves the twisted cube on the n^3 unit cube (the finest mesh of ``hierarchy`` if given); returns
    (V, u, Newton histories, Krylov counts), one entry per load increment."""
    from firedrake_b200.assemble import DirichletBC, FunctionSpace, HyperElasticity, interpolate, solve_nonlinear
    mesh = hierarchy[len(hierarchy) - 1] if hierarchy is not None else ExtrudedHexMesh(n, n, n)
    V = FunctionSpace(mesh, p, 3)
    u = V.dat()
    F = HyperElasticity(V, MU, LMBDA, beta)
    hists, kits = [], []
    for step in range(1, steps + 1):
        bcs = [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, interpolate(V, _top_expressions(step / steps)), "top")]
        hist, its = solve_nonlinear(F, V.dat(), u, bcs=bcs, hierarchy=hierarchy,
                                    solver_parameters=_newton_params(pc, snes_rtol=1e-11, ksp_rtol=ksp_rtol,
                                                                     snes_max_it=NEWTON_BUDGET))
        hists.append(hist)
        kits.append(its)
    return V, u, hists, kits


def oracle_twisted_cube(V):
    """The same load increments through the oracle's scipy Newton."""
    mesh = V.mesh
    el = interval_element(V.degree)
    geo = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    Xn = V.V.dof_coordinates()
    bot, top = V.V.boundary_nodes("bottom"), V.V.boundary_nodes("top")
    bd = (3 * np.concatenate([bot, top])[:, None] + np.arange(3)).ravel()
    u = np.zeros(3 * V.node_count)
    for step in range(1, STEPS + 1):
        t, d = TWIST * step / STEPS, SQUEEZE * step / STEPS
        c = Xn[top] - [0.5, 0.5, 0.0]
        ut = np.stack([np.cos(t) * c[:, 0] - np.sin(t) * c[:, 1] - c[:, 0],
                       np.sin(t) * c[:, 0] + np.cos(t) * c[:, 1] - c[:, 1], np.full(len(top), -d)], axis=1)
        uv = u.reshape(-1, 3)
        uv[bot] = 0.0
        uv[top] = ut
        u, _ = ho.newton(el, mesh.coordinates, geo, MU, LMBDA, 0.0, np.zeros_like(u), u, bd, rtol=1e-13)
    return u


@pytest.mark.parametrize("p", [1, 2])
def test_twisted_cube_matches_scipy_newton(engine, p):
    """A 30 degree twist with 10 % axial compression in 4 increments on the 4^3 cube: every increment
    converges within the Newton budget, and the final field equals the oracle's at 1e-8."""
    V, u, hists, kits = twisted_cube(4, p)
    for hist in hists:
        assert hist[-1] <= 1e-11 * hist[0] and len(hist) <= NEWTON_BUDGET + 1, hists
    ref = oracle_twisted_cube(V)
    assert np.abs(u.data_ro.ravel() - ref).max() < 1e-8 * np.abs(ref).max(), hists


# manufactured solution, clamped on every face, beta = 0: u* = AMP (sin pi x sin pi y sin pi z) (1, 2, -1)
# with coupled x-dependence, f = -div P(I + grad u*)
MS_AMP = 0.05


@functools.lru_cache(maxsize=None)
def _manufactured_functions():
    """NumPy functions of the node positions (n, 3) -> (n, 3): u* and f, derived with sympy."""
    import sympy as sp
    x = sp.symbols("x0 x1 x2")
    s = sp.sin(sp.pi * x[0]) * sp.sin(sp.pi * x[1]) * sp.sin(sp.pi * x[2])
    us = [MS_AMP * s, 2 * MS_AMP * s * sp.cos(sp.pi * x[0] / 2), -MS_AMP * s * (1 + x[1])]
    F = sp.eye(3) + sp.Matrix(3, 3, lambda i, j: sp.diff(us[i], x[j]))
    J = F.det()
    Fit = F.adjugate().T / J
    P = MU * (F - Fit) + LMBDA * sp.log(J) * Fit
    f = [-sum(sp.diff(P[i, j], x[j]) for j in range(3)) for i in range(3)]
    lam = lambda e: sp.lambdify(x, e, "numpy", cse=True)
    fu, ff = lam(us), lam(f)
    field = lambda fn: lambda X: np.stack([np.broadcast_to(c, X.shape[:1]) for c in fn(*X.T)], axis=1)
    return field(fu), field(ff)


def manufactured_solve(n, p, pc="none", refinements=0):
    """Newton on the n^3 unit cube; returns (V, u, u* at the nodes, Newton history, Krylov counts)."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import DirichletBC, FunctionSpace, HyperElasticity, assemble, mass, solve_nonlinear
    ustar, fstar = _manufactured_functions()
    c = n >> refinements
    h = mg.MeshHierarchy(c, c, c, refinements) if refinements else None
    V = FunctionSpace(h[refinements] if h is not None else ExtrudedHexMesh(n, n, n), p, 3)
    Xn = V.V.dof_coordinates()
    L = assemble(mass(V), u=V.dat(fstar(Xn)))
    u = V.dat()
    hist, kits = solve_nonlinear(HyperElasticity(V, MU, LMBDA), L, u, bcs=[DirichletBC(V, 0.0, ALL_FACES)],
                                 hierarchy=h, solver_parameters=_newton_params(pc, snes_rtol=1e-10, ksp_rtol=1e-8))
    return V, u, V.dat(ustar(Xn)), hist, kits


def l2_error(V, u, ui):
    from firedrake_b200.assemble import assemble, mass
    e = V.dat(u.data_ro - ui.data_ro)
    return float(np.sqrt(np.dot(e.data_ro.ravel(), assemble(mass(V), u=e).data_ro.ravel())))


def rates(p, ns):
    errs = []
    for n in ns:
        V, u, ui, _, _ = manufactured_solve(n, p, "jacobi")
        errs.append(l2_error(V, u, ui))
    return errs, np.log2(np.array(errs[:-1]) / np.array(errs[1:]))


@pytest.mark.parametrize("p,ns,want", [(1, (8, 16), 1.8), (2, (4, 8), 2.8)])
def test_l2_convergence_rates(engine, p, ns, want):
    errs, r = rates(p, ns)
    assert np.all(r >= want), (errs, r)


def mg_iterations(n, refinements):
    """GMRES iterations per Newton step of the manufactured problem, CG1, V-cycle of J(0)."""
    _, _, _, hist, kits = manufactured_solve(n, 1, "mg", refinements)
    return kits


def test_mg_iterations(engine):
    """CG1, 8^3 and 16^3 from a 2^3 coarse mesh: the V-cycle of J(0) keeps the GMRES count per Newton step
    nearly flat under refinement."""
    k8, k16 = mg_iterations(8, 2), mg_iterations(16, 3)
    print(f"mg GMRES iterations per Newton step: 8^3 {k8}, 16^3 {k16}")
    assert max(k16) <= 1.5 * max(k8) + 2, (k8, k16)


def test_inverted_element_ends_the_solve(engine):
    """Top face pushed below the bottom: det F < 0 next to it, the first residual is NaN, and the solve
    stops there with DIVERGED_FNORM_NAN instead of running GMRES on NaNs."""
    from firedrake_b200.assemble import (ConvergenceError, DirichletBC, FunctionSpace, HyperElasticity,
                                         solve_nonlinear)
    V = FunctionSpace(ExtrudedHexMesh(3, 3, 3), 1, 3)
    bcs = [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, V.dat(np.tile([0.0, 0.0, -1.5], (V.node_count, 1))), "top")]
    with pytest.raises(ConvergenceError, match="DIVERGED_FNORM_NAN") as e:
        solve_nonlinear(HyperElasticity(V, MU, LMBDA), V.dat(), V.dat(), bcs=bcs,
                        solver_parameters=_newton_params("jacobi"))
    assert e.value.reason == "DIVERGED_FNORM_NAN" and "after 0 Newton steps" in str(e.value)
