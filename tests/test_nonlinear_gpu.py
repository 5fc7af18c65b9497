"""GPU parity of nonlinear diffusion (FDB_FORM_NONLINEAR_DIFFUSION[_JACOBIAN], the slab-thread kernel's
NL modes): residual, Jacobian action, element matrix and diagonal against the NumPy oracle
(tests/_nonlinear_oracle.py) and the merged coefficient and constant-coefficient kernels; Newton
solves of a manufactured problem (the 3-D analogue of Firedrake's
test_helmholtz_nonlinear_diffusion.py) with their L2 convergence rates; the refusals of
fdb_kernel_create.  Tolerance 1e-12 relative in the max norm.

Every test takes the engine as its first argument, so tests/test_nonlinear_host_mock.py runs the
same host logic on the CPU against a mock engine."""
import numpy as np
import pytest

import _coef_oracle as co
import _nonlinear_oracle as no
from firedrake_b200 import op2
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh
from test_coefficient_gpu import relerr, setup

pytestmark = pytest.mark.gpu

TOL = 1e-12
D = (1.0, 0.3, 0.2)

# the manufactured problem: u* = cos(2 pi x) cos(2 pi y) cos(2 pi z), D(u) = 1 + 0.1 u^2, beta = 1,
# zero normal derivative on every face of the unit cube, f = -D(u*) lap u* - D'(u*) |grad u*|^2 + u*
DM = (1.0, 0.0, 0.1)
_C = "cos(6.283185307179586 * x[{0}])"
_S = "sin(6.283185307179586 * x[{0}])"
USTAR = "{} * {} * {}".format(*(_C.format(i) for i in range(3)))
GRAD2 = " + ".join("pow({} * {} * {}, 2)".format(_S.format(i), _C.format((i + 1) % 3), _C.format((i + 2) % 3))
                   for i in range(3))
FSRC = (f"(1.0 + 0.1 * pow({USTAR}, 2)) * 118.43525281307230 * ({USTAR})"      # 12 pi^2
        f" - 0.2 * ({USTAR}) * 39.47841760435743 * ({GRAD2}) + ({USTAR})")      # 4 pi^2


def u_values(V, seed=0):
    X = V.dof_coordinates()
    return np.sin(2.0 * X[:, 0]) * X[:, 1] + X[:, 2] + 0.3 * np.random.default_rng(seed).standard_normal(len(X))


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
@pytest.mark.parametrize("beta", [0.0, 0.6])
def test_nl_residual_and_jacobian_action_match_oracle(engine, p, native, beta):
    """Atomic and coloured scatter (coloured bit-identical across calls); degree 5 on 6 layers takes
    the slim staging with atomics and the full one with colours."""
    mesh, V, cells, nodes, m0, m1, X, omaps = setup(p, native)
    u = op2.Dat(nodes, u_values(V, p))
    w = op2.Dat(nodes, np.random.default_rng(10 + p).standard_normal(V.node_count))
    alpha = 1.3
    el = interval_element(p)
    ro = no.residual(el, mesh.coordinates, u.data_ro.copy(), *omaps, D, alpha=alpha, beta=beta)
    jo = no.jacobian_action(el, mesh.coordinates, u.data_ro.copy(), w.data_ro.copy(), *omaps, D, alpha=alpha,
                            beta=beta)
    kr = op2.Kernel("nonlinear_diffusion", degree=p, alpha=alpha, beta=beta, d=D)
    kj = op2.Kernel("nonlinear_diffusion_jacobian", degree=p, alpha=alpha, beta=beta, d=D)
    for k, args, want in ((kr, (X(op2.READ, m1), u(op2.READ, m0)), ro),
                          (kj, (X(op2.READ, m1), w(op2.READ, m0), u(op2.READ, m0)), jo)):
        y = op2.Dat(nodes)
        op2.par_loop(k, cells, y(op2.INC, m0), *args)
        assert relerr(y.data_ro, want) < TOL, k.form
        outs = []
        for _ in range(2):
            y.zero()
            op2.par_loop(k, cells, y(op2.INC, m0), *args, scatter="coloured")
            outs.append(y.data_ro.copy())
        assert np.array_equal(outs[0], outs[1])
        assert relerr(outs[0], want) < TOL, k.form


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
def test_nl_forms_against_the_merged_kernels(engine, p):
    """d2 = 0: the residual is the coefficient form with kappa = d0 + d1 u.  d = (d0, 0, 0): the residual
    and the Jacobian are the constant-coefficient form with alpha*d0."""
    from firedrake_b200.assemble import Form, FunctionSpace, NonlinearDiffusion, OneFormAssembler, assemble
    mesh = ExtrudedHexMesh(4, 3, 5, warp=0.05, permute_seed=2)
    V = FunctionSpace(mesh, p)
    u = V.dat(u_values(V.V, 1))
    w = V.dat(np.random.default_rng(2).standard_normal(V.node_count))
    F = NonlinearDiffusion(V, 1.2, 0.5, (1.5, 0.7, 0.0))
    kap = V.dat(1.5 + 0.7 * u.data_ro)
    r = assemble(F, u=u)
    rc = OneFormAssembler(Form(V, 1.2, 0.5, kap), u).assemble()
    assert relerr(r.data_ro, rc.data_ro) < TOL
    F0 = NonlinearDiffusion(V, 1.2, 0.5, (1.5, 0.0, 0.0))
    r0 = assemble(F0, u=u).data_ro.copy()
    assert relerr(r0, assemble(Form(V, 1.2 * 1.5, 0.5), u=u).data_ro) < TOL
    j0 = assemble(F0.jacobian(u), u=w).data_ro.copy()
    assert relerr(j0, assemble(Form(V, 1.2 * 1.5, 0.5), u=w).data_ro) < TOL


@pytest.mark.parametrize("p", [2, 3])
def test_nl_taylor_ratio(engine, p):
    """(R(u + h w) - R(u - h w)) / 2h - J(u) w falls by 4 when h halves: J is the derivative of the
    discrete residual the kernels compute."""
    from firedrake_b200.assemble import FunctionSpace, NonlinearDiffusion, assemble
    V = FunctionSpace(ExtrudedHexMesh(3, 3, 4, warp=0.05), p)
    u0, w0 = u_values(V.V, 3), np.random.default_rng(4).standard_normal(V.node_count)
    F = NonlinearDiffusion(V, 1.0, 0.4, D)
    R = lambda x: assemble(F, u=V.dat(x)).data_ro.copy()
    Jw = assemble(F.jacobian(V.dat(u0)), u=V.dat(w0)).data_ro.copy()
    e = np.array([np.abs((R(u0 + h * w0) - R(u0 - h * w0)) / (2 * h) - Jw).max() for h in (0.04, 0.02, 0.01)])
    ratios = e[:-1] / e[1:]
    assert np.all((ratios > 3.6) & (ratios < 4.4)), (e, ratios)


def _bcs(V):
    from firedrake_b200.assemble import DirichletBC
    return [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, 0.0, "top")]


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_nl_matrix_matches_oracle(engine, p):
    """Entrywise against the oracle's element matrices added through the BC-masked lgmaps, unit diagonal
    on the constrained rows; measurably nonsymmetric; Mat.mult equals the matrix-free mult."""
    from firedrake_b200.assemble import FunctionSpace, NonlinearDiffusion, assemble
    mesh = ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=2) if p < 4 else \
        ExtrudedHexMesh(2, 2, 3, warp=0.05, permute_seed=2)
    V = FunctionSpace(mesh, p)
    u = V.dat(u_values(V.V, 5))
    bcs = _bcs(V)
    J = NonlinearDiffusion(V, 1.1, 0.7, D).jacobian(u)
    A = assemble(J, bcs=bcs)
    ro, ci, vals = A.csr()
    lg = np.arange(V.node_count, dtype=np.int32)
    bn = np.unique(np.concatenate([bc.nodes for bc in bcs]))
    lg[bn] = -1
    i0, Ae = no.jacobian_matrices(interval_element(p), mesh.coordinates, u.data_ro.copy(), V.V.cell_node_map,
                                  V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz, D, alpha=1.1, beta=0.7)
    vo = co.add_to_csr(ro, ci, np.zeros(len(ci)), i0, Ae, lg, lg)
    diag = ro[bn] + np.array([np.searchsorted(ci[ro[r]:ro[r + 1]], r) for r in bn], dtype=np.int64)
    vo[diag] = 1.0
    scale = np.abs(vo).max()
    assert np.abs(vals - vo).max() < TOL * scale
    import scipy.sparse as sps
    K = sps.csr_matrix((vals, ci, ro), shape=(V.node_count, V.node_count))
    assert abs(K - K.T).max() > 1e-3 * scale
    x = V.dat(np.random.default_rng(6).standard_normal(V.node_count))
    y, ymf = V.dat(), V.dat()
    A.mult(x, y)
    mf = assemble(J, bcs=bcs, mat_type="matfree")
    mf.mult(x, ymf)
    assert relerr(y.data_ro, ymf.data_ro) < TOL
    with pytest.raises(NotImplementedError):
        mf.multTranspose(x, ymf)


@pytest.mark.parametrize("p", [1, 2, 3])
def test_nl_diagonal_equals_assembled_diagonal(engine, p):
    from firedrake_b200.assemble import FunctionSpace, NonlinearDiffusion, assemble
    V = FunctionSpace(ExtrudedHexMesh(3, 2, 4, warp=0.05, permute_seed=3), p)
    u = V.dat(u_values(V.V, 7))
    J = NonlinearDiffusion(V, 1.0, 0.3, D).jacobian(u)
    bcs = _bcs(V)
    d = assemble(J, bcs=bcs, mat_type="matfree").getDiagonal(V.dat()).data_ro.copy()
    ro, ci, vals = assemble(J, bcs=bcs).csr()
    dA = np.array([vals[ro[r] + np.searchsorted(ci[ro[r]:ro[r + 1]], r)] for r in range(V.node_count)])
    assert relerr(d, dA) < TOL


def test_nl_host_pointer_mode_equals_device_mode(engine):
    """Host-resident Dats through the mirror cache (monolithic path); a host write to u is picked up."""
    p = 3
    mesh, V, cells, nodes, m0, m1, X, _ = setup(p, False, ExtrudedHexMesh(4, 4, 6, warp=0.05))
    u = op2.Dat(nodes, u_values(V, 9))
    w = op2.Dat(nodes, np.random.default_rng(9).standard_normal(V.node_count))
    for form, args in (("nonlinear_diffusion", [u]), ("nonlinear_diffusion_jacobian", [w, u])):
        k = op2.Kernel(form, degree=p, alpha=1.0, beta=0.2, d=D)
        yd = op2.Dat(nodes)
        op2.par_loop(k, cells, yd(op2.INC, m0), X(op2.READ, m1), *(a(op2.READ, m0) for a in args))
        ref = yd.data_ro.copy()
        yh = op2.Dat(nodes)
        gk = op2.GlobalKernel(k, [m0, m1], extruded=True)
        loop = op2.Parloop(gk, cells, [yh(op2.INC, m0), X(op2.READ, m1)] + [a(op2.READ, m0) for a in args],
                           location="host")
        loop()
        assert relerr(yh.data_ro, ref) < TOL, form
    u.data[:] *= 0.5
    yh.zero()
    loop()
    yd.zero()
    op2.par_loop(k, cells, yd(op2.INC, m0), X(op2.READ, m1), w(op2.READ, m0), u(op2.READ, m0))
    assert relerr(yh.data_ro, yd.data_ro) < TOL


def manufactured(n, p, refinements=0):
    """(V, hierarchy or None, F, L, interpolant of u*) on the n^3 unit cube, the finest level of a
    hierarchy with ``refinements`` coarser levels if that is nonzero."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import FunctionSpace, NonlinearDiffusion, assemble, interpolate, mass
    c = n >> refinements
    h = mg.MeshHierarchy(c, c, c, refinements) if refinements else None
    V = FunctionSpace(h[refinements] if h is not None else ExtrudedHexMesh(n, n, n), p)
    f = interpolate(V, FSRC)
    return V, h, NonlinearDiffusion(V, 1.0, 1.0, DM), assemble(mass(V), u=f), interpolate(V, USTAR)


NEWTON_PARAMS = {"snes_rtol": 1e-10, "ksp_rtol": 1e-12, "ksp_max_it": 5000}


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
def test_nl_newton_solve_manufactured(engine, pc):
    """CG2 on 8^3 from u = 0, exact Newton steps (ksp_rtol 1e-12): at most 6 steps for every
    preconditioner."""
    from firedrake_b200.assemble import solve_nonlinear
    V, h, F, L, ui = manufactured(8, 2, refinements=2 if pc == "mg" else 0)
    u = V.dat()
    hist, kits = solve_nonlinear(F, L, u, solver_parameters=dict(NEWTON_PARAMS, pc_type=pc), hierarchy=h)
    assert hist[-1] <= 1e-10 * hist[0] and len(kits) <= 6, (pc, hist, kits)
    assert np.abs(u.data_ro - ui.data_ro).max() < 0.1, pc       # the discretisation error at n = 8


def l2_error(V, u, ui):
    from firedrake_b200.assemble import assemble, mass
    e = V.dat(u.data_ro - ui.data_ro)
    return float(np.sqrt(np.dot(e.data_ro, assemble(mass(V), u=e).data_ro)))


@pytest.mark.parametrize("p,ns,rate", [(1, (8, 16, 32), 1.8), (2, (4, 8, 16), 2.8)])
def test_nl_l2_convergence_rates(engine, p, ns, rate):
    """The reference's thresholds: 1.8 for CG1 (test_helmholtz_nonlinear_diffusion.py), 2.8 for CG2
    (test_nonlinear_helmholtz.py); errors against the interpolant of u*."""
    from firedrake_b200.assemble import solve_nonlinear
    errs = []
    for n in ns:
        V, _, F, L, ui = manufactured(n, p)
        u = V.dat()
        solve_nonlinear(F, L, u, solver_parameters=dict(NEWTON_PARAMS, pc_type="jacobi", ksp_rtol=1e-11))
        errs.append(l2_error(V, u, ui))
    rates = np.log2(np.array(errs[:-1]) / np.array(errs[1:]))
    assert np.all(rates > rate), (errs, rates)


def test_nl_dirichlet_matches_oracle_newton(engine):
    """Nonzero Dirichlet values at the bottom (0.5) and the top (2.0), the source f = 1 + x y z."""
    from firedrake_b200.assemble import (DirichletBC, FunctionSpace, NonlinearDiffusion, assemble, interpolate,
                                         mass, solve_nonlinear)
    p = 2
    mesh = ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=1)
    V = FunctionSpace(mesh, p)
    f = interpolate(V, "1.0 + x[0] * x[1] * x[2]")
    L = assemble(mass(V), u=f)
    F = NonlinearDiffusion(V, 1.0, 0.3, (1.0, 0.5, 0.5))
    bcs = [DirichletBC(V, 0.5, "bottom"), DirichletBC(V, 2.0, "top")]
    u = V.dat()
    hist, kits = solve_nonlinear(F, L, u, bcs=bcs, solver_parameters=dict(NEWTON_PARAMS, pc_type="jacobi"))
    geo = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    g = np.zeros(V.node_count)
    g[bcs[0].nodes], g[bcs[1].nodes] = 0.5, 2.0
    uo, ho = no.newton(interval_element(p), mesh.coordinates, geo, L.data_ro.copy(), F.d, 1.0, 0.3,
                       bc_nodes=np.concatenate([bcs[0].nodes, bcs[1].nodes]), bc_values=g)
    assert np.abs(u.data_ro - uo).max() < 1e-9, (hist, ho)
    assert len(kits) == len(ho) - 1, (hist, ho)


def test_nl_kernel_refuses_what_it_does_not_cover(engine):
    """Vector spaces, the affine variant, another quadrature, non-hex cells, the residual as a matrix or
    diagonal, degrees outside the instantiated ranges: a clear error from fdb_kernel_create."""
    from firedrake_b200 import _lib
    mesh, V, cells, nodes, m0, m1, X, _ = setup(2, False, ExtrudedHexMesh(2, 2, 2))
    R, J = "nonlinear_diffusion", "nonlinear_diffusion_jacobian"
    cases = ((R, dict(degree=2, cdim=3), "scalar"), (J, dict(degree=2, cdim=3), "scalar"),
             (R, dict(degree=2, affine=True), "affine"), (J, dict(degree=2, affine=True), "affine"),
             (R, dict(degree=2, element=interval_element(2, 4)), "nq == degree"),
             (J, dict(degree=2, element=interval_element(2, 4)), "nq == degree"),
             (R, dict(degree=1, cell="triangle"), "hex cells"), (J, dict(degree=1, cell="triangle"), "hex cells"),
             (R, dict(degree=2, rank=2), "1-form action only"), (R, dict(degree=2, diagonal=True), "1-form action only"),
             (R, dict(degree=6), "degree 6"), (J, dict(degree=5, rank=2), "degree 5"),
             (J, dict(degree=4, diagonal=True), "degree 4"))
    for form, kw, msg in cases:
        gk = op2.GlobalKernel(op2.Kernel(form, d=D, **kw), [m0, m1], extruded=True)
        with pytest.raises(_lib.EngineError, match=msg):
            gk.compile()
