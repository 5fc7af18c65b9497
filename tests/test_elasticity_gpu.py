"""GPU parity of linear elasticity (FDB_FORM_ELASTICITY, csrc/elasticity_hex.cu): action, blocked element
matrix and diagonal against the NumPy oracle (tests/_elasticity_oracle.py) and the generic wrapper path;
the rigid-body modes; the assembled against the matrix-free operator; solves (the patch test with every
preconditioner, the L2 rates of a manufactured solution with coupled components, multigrid iteration
counts); the refusals of fdb_kernel_create and fdb_kernel_call.  Tolerance 1e-12 relative in the max norm.

Every test takes the engine as its first argument, so tests/test_elasticity_host_mock.py runs the same
host logic on the CPU against a mock engine."""
import numpy as np
import pytest

import _elasticity_oracle as eo
from firedrake_b200 import op2
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh
from test_coefficient_gpu import relerr, setup

pytestmark = pytest.mark.gpu

TOL = 1e-12
MU, LMBDA = 1.3, 2.1
ALL_FACES = (1, 2, 3, 4, "bottom", "top")


def vec_values(n, seed=0):
    return np.random.default_rng(seed).standard_normal((n, 3))


@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
@pytest.mark.parametrize("beta", [0.0, 0.6])
def test_elasticity_action_matches_oracle(engine, p, native, beta):
    """Atomic and coloured scatter; coloured is bit-identical across calls."""
    mesh, V, cells, nodes, m0, m1, X, omaps = setup(p, native)
    vset = op2.DataSet(nodes, 3)
    u = op2.Dat(vset, vec_values(V.node_count, p))
    want = eo.action(interval_element(p), mesh.coordinates, u.data_ro.ravel().copy(), *omaps, MU, LMBDA, beta)
    k = op2.Kernel("elasticity", degree=p, mu=MU, lmbda=LMBDA, beta=beta, cdim=3)
    y = op2.Dat(vset)
    op2.par_loop(k, cells, y(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0))
    assert relerr(y.data_ro.ravel(), want) < TOL
    outs = []
    for _ in range(2):
        y.zero()
        op2.par_loop(k, cells, y(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), scatter="coloured")
        outs.append(y.data_ro.copy())
    assert np.array_equal(outs[0], outs[1])
    assert relerr(outs[0].ravel(), want) < TOL


def _space(p, mesh=None):
    from firedrake_b200.assemble import FunctionSpace
    return FunctionSpace(mesh or ExtrudedHexMesh(4, 3, 5, warp=0.05, permute_seed=2), p, 3)


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_elasticity_action_matches_generic_path(engine, p):
    from firedrake_b200.assemble import Elasticity, assemble, assemble_elasticity_generic
    V = _space(p)
    w = V.dat(vec_values(V.node_count, 3))
    y = assemble(Elasticity(V, MU, LMBDA, 0.4), u=w).data_ro.copy()
    yg = assemble_elasticity_generic(V, w, MU, LMBDA, 0.4).data_ro.copy()
    assert relerr(y, yg) < TOL


def test_elasticity_host_pointer_mode_equals_device_mode(engine):
    """Host-resident Dats through the mirror cache (the monolithic path); a host write to u is picked up."""
    p = 3
    mesh, V, cells, nodes, m0, m1, X, _ = setup(p, False, ExtrudedHexMesh(4, 4, 6, warp=0.05))
    vset = op2.DataSet(nodes, 3)
    u = op2.Dat(vset, vec_values(V.node_count, 9))
    k = op2.Kernel("elasticity", degree=p, mu=MU, lmbda=LMBDA, beta=0.2, cdim=3)
    yd = op2.Dat(vset)
    op2.par_loop(k, cells, yd(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0))
    yh = op2.Dat(vset)
    gk = op2.GlobalKernel(k, [m0, m1], extruded=True)
    loop = op2.Parloop(gk, cells, [yh(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0)], location="host")
    loop()
    assert relerr(yh.data_ro, yd.data_ro) < TOL
    u.data[:] *= 0.5
    yh.zero()
    loop()
    yd.zero()
    op2.par_loop(k, cells, yd(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0))
    assert relerr(yh.data_ro, yd.data_ro) < TOL


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_rigid_body_modes_are_in_the_kernel(engine, p):
    """beta = 0, no boundary conditions: the 3 translations and 3 infinitesimal rotations, interpolated at
    the nodes of a warped mesh, are mapped to zero."""
    from firedrake_b200.assemble import Elasticity, assemble
    V = _space(p, ExtrudedHexMesh(3, 3, 4, warp=0.06, permute_seed=1))
    F = Elasticity(V, MU, LMBDA)
    ref = np.abs(assemble(F, u=V.dat(vec_values(V.node_count, 5))).data_ro).max()
    for r in eo.rigid_body_modes(V.V.dof_coordinates()):
        y = assemble(F, u=V.dat(r.reshape(-1, 3))).data_ro
        assert np.abs(y).max() <= 1e-11 * ref


def _bcs(V):
    from firedrake_b200.assemble import DirichletBC
    return [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, 0.0, 2)]


@pytest.mark.parametrize("p", [1, 2, 3])
def test_elasticity_blocked_matrix_matches_oracle(engine, p):
    """Entrywise against the oracle's element matrices added through the dof-level BC-masked lgmaps, unit
    diagonal on the constrained rows; symmetric, with nonzero off-diagonal component blocks."""
    from firedrake_b200.assemble import Elasticity, assemble
    mesh = ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=2)
    V = _space(p, mesh)
    bcs = _bcs(V)
    A = assemble(Elasticity(V, MU, LMBDA, 0.7), bcs=bcs)
    ro, ci, vals = A.csr()
    bn = np.unique(np.concatenate([bc.nodes for bc in bcs]))
    lg = np.arange(3 * V.node_count, dtype=np.int32).reshape(-1, 3)
    lg[bn] = -1
    lg = lg.ravel()
    di, Ae = eo.element_matrices(interval_element(p), mesh.coordinates, V.V.cell_node_map, V.V.offset,
                                 mesh.coord_map, mesh.coord_offset, mesh.nz, MU, LMBDA, 0.7)
    vo = eo.add_to_bcsr(ro, ci, np.zeros(len(vals)), di, Ae, lg, lg)
    blocks = vo.reshape(-1, 3, 3)
    for r in bn:
        k = ro[r] + np.searchsorted(ci[ro[r]:ro[r + 1]], r)
        blocks[k][np.diag_indices(3)] = 1.0
    scale = np.abs(vo).max()
    assert np.abs(vals - vo).max() < TOL * scale
    K = eo.to_dense(ro, ci, vals)
    assert np.abs(K - K.T).max() < TOL * scale
    off = vals.reshape(-1, 3, 3).copy()
    off[:, np.arange(3), np.arange(3)] = 0.0
    assert np.abs(off).max() > 1e-2 * scale


@pytest.mark.parametrize("p", [1, 2, 3])
@pytest.mark.parametrize("with_bcs", [False, True], ids=["nobc", "bc"])
def test_elasticity_mat_mult_equals_matfree(engine, p, with_bcs):
    from firedrake_b200.assemble import Elasticity, assemble
    V = _space(p, ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=3))
    bcs = _bcs(V) if with_bcs else ()
    F = Elasticity(V, MU, LMBDA, 0.3)
    x = V.dat(vec_values(V.node_count, 6))
    y, ymf, yt = V.dat(), V.dat(), V.dat()
    assemble(F, bcs=bcs).mult(x, y)
    mf = assemble(F, bcs=bcs, mat_type="matfree")
    mf.mult(x, ymf)
    assert relerr(y.data_ro, ymf.data_ro) < TOL
    mf.multTranspose(x, yt)                      # symmetric: the same operator
    assert relerr(yt.data_ro, ymf.data_ro) < TOL


@pytest.mark.parametrize("p", [1, 2, 3])
def test_elasticity_diagonal_equals_assembled_diagonal(engine, p):
    from firedrake_b200.assemble import Elasticity, assemble
    V = _space(p, ExtrudedHexMesh(3, 2, 4, warp=0.05, permute_seed=3))
    F = Elasticity(V, MU, LMBDA, 0.3)
    bcs = _bcs(V)
    d = assemble(F, bcs=bcs, mat_type="matfree").getDiagonal(V.dat()).data_ro.copy()
    ro, ci, vals = assemble(F, bcs=bcs).csr()
    blocks = vals.reshape(-1, 3, 3)
    dA = np.array([np.diagonal(blocks[ro[r] + np.searchsorted(ci[ro[r]:ro[r + 1]], r)])
                   for r in range(V.node_count)])
    assert relerr(d, dA) < TOL
    assert np.ptp(d[~np.isin(np.arange(V.node_count), np.concatenate([bc.nodes for bc in bcs]))], axis=1).max() > 0


def test_elasticity_refuses_what_it_does_not_cover(engine):
    """Scalar or 2-component spaces, non-hex cells, the affine variant, another quadrature, degrees outside
    1..4 (action) and 1..3 (matrix, diagonal): fdb_kernel_create; a Mat whose block size is not 3:
    fdb_kernel_call."""
    from firedrake_b200 import _lib
    mesh, V, cells, nodes, m0, m1, X, _ = setup(2, False, ExtrudedHexMesh(2, 2, 2))
    E = dict(mu=MU, lmbda=LMBDA)
    cases = ((dict(degree=2, cdim=1), "value size 3"), (dict(degree=2, cdim=2), "value size 3"),
             (dict(degree=1, cdim=3, cell="triangle"), "hex cells"),
             (dict(degree=2, cdim=3, affine=True), "affine"),
             (dict(degree=2, cdim=3, element=interval_element(2, 4)), "nq == degree"),
             (dict(degree=5, cdim=3), "degree 5 outside 1..4"),
             (dict(degree=4, cdim=3, rank=2), "degree 4 outside 1..3"),
             (dict(degree=4, cdim=3, diagonal=True), "degree 4 outside 1..3"))
    for kw, msg in cases:
        gk = op2.GlobalKernel(op2.Kernel("elasticity", **E, **kw), [m0, m1], extruded=True)
        with pytest.raises(_lib.EngineError, match=msg):
            gk.compile()
    mat = op2.Mat(op2.Sparsity((nodes, nodes), [(m0, m0, None)]))
    with pytest.raises(_lib.EngineError, match="block size 1"):
        op2.par_loop(op2.Kernel("elasticity", degree=2, rank=2, cdim=3, **E), cells,
                     mat(op2.INC, (m0, m0)), X(op2.READ, m1))


# ------------------------------------------------------------------------------------------------ solves
PATCH_M = ((0.3, -0.2, 0.5), (0.1, 0.4, -0.3), (-0.6, 0.2, 0.1))      # not symmetric
PATCH_C = (0.1, -0.2, 0.3)
PATCH = [" + ".join([f"{PATCH_M[a][k]!r} * x[{k}]" for k in range(3)] + [repr(PATCH_C[a])]) for a in range(3)]


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
@pytest.mark.parametrize("p", [1, 2])
def test_elasticity_patch_test(engine, pc, p):
    """Dirichlet data u = M x + c on all six faces of a warped mesh, zero load, beta = 0: every node
    of the solution carries the linear field."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import DirichletBC, Elasticity, FunctionSpace, interpolate, solve
    h = mg.MeshHierarchy(2, 2, 2, 1, warp=0.05) if pc == "mg" else None
    V = FunctionSpace(h[1] if h is not None else ExtrudedHexMesh(4, 4, 4, warp=0.05, permute_seed=1), p, 3)
    g = interpolate(V, PATCH)
    bcs = [DirichletBC(V, g, ALL_FACES)]
    u = V.dat()
    its, hist = solve(Elasticity(V, MU, LMBDA), V.dat(), u, bcs=bcs, hierarchy=h,
                      solver_parameters={"pc_type": pc, "ksp_rtol": 1e-13, "ksp_max_it": 5000})
    assert np.abs(u.data_ro - g.data_ro).max() < 1e-9, (pc, its, hist[-1])


# manufactured solution with coupled components, clamped on every face, nu = 0.3 (lmbda = 1.5 mu),
# f = -div sigma(u*) (beta = 0)
MS_MU, MS_LMBDA = 1.0, 1.5
_PI = "3.141592653589793"
USTAR = [e.replace("PI", _PI) for e in (
    "sin(PI*x[0])*sin(PI*x[1])*sin(PI*x[2])",
    "sin(2*PI*x[0])*sin(PI*x[1])*sin(PI*x[2])",
    "sin(PI*x[0])*sin(PI*x[1])*sin(2*PI*x[2])")]
FSTAR = [e.replace("PI", _PI) for e in (
    "(11.0/2.0)*pow(PI, 2)*sin(PI*x[0])*sin(PI*x[1])*sin(PI*x[2]) - 5*pow(PI, 2)*sin(PI*x[1])*cos(PI*x[0])"
    "*cos(2*PI*x[2]) - 5*pow(PI, 2)*sin(PI*x[2])*cos(2*PI*x[0])*cos(PI*x[1])",
    "-5*pow(PI, 2)*sin(PI*x[0])*cos(PI*x[1])*cos(2*PI*x[2]) + (17.0/2.0)*pow(PI, 2)*sin(2*PI*x[0])"
    "*sin(PI*x[1])*sin(PI*x[2]) - 5.0/2.0*pow(PI, 2)*sin(PI*x[2])*cos(PI*x[0])*cos(PI*x[1])",
    "32*pow(PI, 2)*sin(PI*x[0])*sin(PI*x[1])*sin(PI*x[2])*cos(PI*x[2]) - 5*pow(PI, 2)*sin(PI*x[0])"
    "*cos(PI*x[0])*cos(PI*x[1])*cos(PI*x[2]) - 5.0/2.0*pow(PI, 2)*sin(PI*x[1])*cos(PI*x[0])*cos(PI*x[2])")]


def manufactured(n, p, refinements=0):
    """(V, hierarchy or None, F, L, bcs, interpolant of u*) on the n^3 unit cube."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import DirichletBC, Elasticity, FunctionSpace, assemble, interpolate, mass
    c = n >> refinements
    h = mg.MeshHierarchy(c, c, c, refinements) if refinements else None
    V = FunctionSpace(h[refinements] if h is not None else ExtrudedHexMesh(n, n, n), p, 3)
    L = assemble(mass(V), u=interpolate(V, FSTAR))
    return V, h, Elasticity(V, MS_MU, MS_LMBDA), L, [DirichletBC(V, 0.0, ALL_FACES)], interpolate(V, USTAR)


def l2_error(V, u, ui):
    from firedrake_b200.assemble import assemble, mass
    e = V.dat(u.data_ro - ui.data_ro)
    return float(np.sqrt(np.dot(e.data_ro.ravel(), assemble(mass(V), u=e).data_ro.ravel())))


def rates(p, ns):
    from firedrake_b200.assemble import solve
    errs = []
    for n in ns:
        V, _, F, L, bcs, ui = manufactured(n, p)
        u = V.dat()
        solve(F, L, u, bcs=bcs, solver_parameters={"pc_type": "jacobi", "ksp_rtol": 1e-11, "ksp_max_it": 5000})
        errs.append(l2_error(V, u, ui))
    return errs, np.log2(np.array(errs[:-1]) / np.array(errs[1:]))


@pytest.mark.parametrize("p,ns", [(1, (8, 16)), (2, (4, 8))])
def test_elasticity_l2_convergence_rates(engine, p, ns):
    errs, r = rates(p, ns)
    assert np.all(r >= p + 0.8), (errs, r)


def iterations(n, refinements, pc):
    from firedrake_b200.assemble import solve
    V, h, F, L, bcs, _ = manufactured(n, 1, refinements if pc == "mg" else 0)
    its, _ = solve(F, L, V.dat(), bcs=bcs, hierarchy=h,
                   solver_parameters={"pc_type": pc, "ksp_rtol": 1e-8, "ksp_max_it": 5000})
    return its


def test_elasticity_mg_iterations(engine):
    """CG1, 8^3 and 16^3 from a 2^3 coarse mesh: the V-cycle's count grows by at most 25 % and stays
    below Jacobi's at both sizes."""
    mg8, mg16 = iterations(8, 2, "mg"), iterations(16, 3, "mg")
    j8, j16 = iterations(8, 2, "jacobi"), iterations(16, 3, "jacobi")
    assert mg16 <= 1.25 * mg8 and mg8 < j8 and mg16 < j16, (mg8, mg16, j8, j16)
