"""GPU parity of advection-diffusion alpha*inner(grad u, grad v)*dx + inner(dot(b, grad u), v)*dx +
beta*inner(u, v)*dx (FDB_FORM_ADVECTION_DIFFUSION, the slab-thread kernel's ADV mode): action, element
matrix, diagonal, host-pointer mode, refusals and GMRES solves, against the NumPy oracle
(tests/_advdiff_oracle.py), the generic wrapper path and the constant-coefficient kernels.  Tolerance 1e-12
relative in the max norm.

Every test takes the engine as its first argument, so tests/test_advdiff_host_mock.py runs the same host
logic on the CPU against a mock engine."""
import numpy as np
import pytest

import _advdiff_oracle as ao
import _coef_oracle as co
from firedrake_b200 import _lib, op2
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh
from test_coefficient_gpu import relerr, setup
from test_form_dispatch_gpu import _host_call

pytestmark = pytest.mark.gpu

TOL = 1e-12
SIDES = (1, 2, 3, 4, "bottom", "top")


def velocity(X, seed=0):
    """A varying velocity with per-node noise, (nnodes, 3)."""
    b = np.stack([1.0 + np.sin(2.0 * X[:, 1]), X[:, 0] * X[:, 2] - 0.5, 0.7 * np.cos(X[:, 0])], axis=1)
    return b + 0.1 * np.random.default_rng(seed).standard_normal(b.shape)


@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
@pytest.mark.parametrize("beta", [0.0, 0.6])
def test_advdiff_action_matches_oracle(engine, p, native, beta):
    """Atomic and coloured scatter; coloured is bit-identical across calls."""
    mesh, V, cells, nodes, m0, m1, X, omaps = setup(p, native)
    u = op2.Dat(nodes, np.random.default_rng(p).standard_normal(V.node_count))
    b = op2.Dat(op2.DataSet(nodes, 3), velocity(V.dof_coordinates(), p))
    alpha = 1.3
    yo = ao.action(interval_element(p), mesh.coordinates, u.data_ro.copy(), b.data_ro.ravel().copy(), *omaps,
                   alpha=alpha, beta=beta)
    k = op2.Kernel("advection_diffusion", degree=p, alpha=alpha, beta=beta)
    y = op2.Dat(nodes)
    op2.par_loop(k, cells, y(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), b(op2.READ, m0))
    assert relerr(y.data_ro, yo) < TOL
    outs = []
    for _ in range(2):
        y.zero()
        op2.par_loop(k, cells, y(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), b(op2.READ, m0),
                     scatter="coloured")
        outs.append(y.data_ro.copy())
    assert np.array_equal(outs[0], outs[1])
    assert relerr(outs[0], yo) < TOL


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_advdiff_action_matches_generic_path_and_helmholtz(engine, p):
    """The hand-written kernel against ``assemble_advection_diffusion_generic`` (the generic wrapper path,
    degrees 1..3; it refuses degree 4, DESIGN.md section 4.10), and b = 0 against the constant-coefficient
    ``Form`` (the helmholtz kernel) at every degree."""
    from firedrake_b200.assemble import (AdvectionDiffusion, Form, FunctionSpace, OneFormAssembler,
                                         assemble_advection_diffusion_generic)
    mesh = ExtrudedHexMesh(4, 3, 5, warp=0.05, permute_seed=2)
    V = FunctionSpace(mesh, p)
    u = V.dat(np.random.default_rng(1).standard_normal(V.node_count))
    b = op2.Dat(V.vector_dset(3), velocity(V.V.dof_coordinates(), 2))
    if p == 4:
        with pytest.raises(NotImplementedError, match="outside 1..3"):
            assemble_advection_diffusion_generic(V, u, b, alpha=0.9, beta=0.5)
    else:
        yg = assemble_advection_diffusion_generic(V, u, b, alpha=0.9, beta=0.5)
        ya = OneFormAssembler(AdvectionDiffusion(V, b, 0.9, 0.5), u).assemble()
        assert relerr(ya.data_ro, yg.data_ro) < TOL
    zero = op2.Dat(V.vector_dset(3))
    y0 = OneFormAssembler(AdvectionDiffusion(V, zero, 0.8, 0.5), u).assemble()
    yf = OneFormAssembler(Form(V, 0.8, 0.5), u).assemble()
    assert relerr(y0.data_ro, yf.data_ro) < TOL


def _bcs(V):
    from firedrake_b200.assemble import DirichletBC
    return [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, 0.0, "top")]


@pytest.mark.parametrize("p", [1, 2, 3])
def test_advdiff_matrix_matches_oracle(engine, p):
    """Entrywise against the oracle's element matrices (row = test, column = trial) added through the
    BC-masked lgmaps, unit diagonal on the constrained rows; Mat.mult equals the matrix-free operator's
    mult; the matrix is not symmetric."""
    from firedrake_b200.assemble import AdvectionDiffusion, FunctionSpace, assemble
    mesh = ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=2)
    V = FunctionSpace(mesh, p)
    b = op2.Dat(V.vector_dset(3), velocity(V.V.dof_coordinates(), 3))
    bcs = _bcs(V)
    form = AdvectionDiffusion(V, b, 1.1, 0.7)
    A = assemble(form, bcs=bcs)
    ro, ci, vals = A.csr()
    lg = np.arange(V.node_count, dtype=np.int32)
    bn = np.unique(np.concatenate([bc.nodes for bc in bcs]))
    lg[bn] = -1
    i0, Ae = ao.element_matrices(interval_element(p), mesh.coordinates, b.data_ro.ravel().copy(),
                                 V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz,
                                 alpha=1.1, beta=0.7)
    vo = co.add_to_csr(ro, ci, np.zeros(len(ci)), i0, Ae, lg, lg)
    diag = ro[bn] + np.array([np.searchsorted(ci[ro[r]:ro[r + 1]], r) for r in bn], dtype=np.int64)
    vo[diag] = 1.0
    assert np.abs(vals - vo).max() < TOL * np.abs(vo).max()
    import scipy.sparse as sps
    M = sps.csr_matrix((vals, ci, ro), shape=(V.node_count,) * 2)
    assert abs(M - M.T).max() > 1e-3 * np.abs(vals).max()
    x = V.dat(np.random.default_rng(4).standard_normal(V.node_count))
    y, ymf = V.dat(), V.dat()
    A.mult(x, y)
    assemble(form, bcs=bcs, mat_type="matfree").mult(x, ymf)
    assert relerr(y.data_ro, ymf.data_ro) < TOL


@pytest.mark.parametrize("p", [1, 2, 3])
def test_advdiff_diagonal_equals_assembled_diagonal(engine, p):
    from firedrake_b200.assemble import AdvectionDiffusion, FunctionSpace, ImplicitMatrixContext, assemble
    mesh = ExtrudedHexMesh(3, 2, 4, warp=0.05, permute_seed=3)
    V = FunctionSpace(mesh, p)
    b = op2.Dat(V.vector_dset(3), velocity(V.V.dof_coordinates(), 5))
    form = AdvectionDiffusion(V, b, 1.0, 0.3)
    bcs = _bcs(V)
    d = ImplicitMatrixContext(form, bcs).getDiagonal(V.dat()).data_ro.copy()
    ro, ci, vals = assemble(form, bcs=bcs).csr()
    dA = np.array([vals[ro[r] + np.searchsorted(ci[ro[r]:ro[r + 1]], r)] for r in range(V.node_count)])
    assert relerr(d, dA) < TOL
    do = ao.diagonal(interval_element(p), mesh.coordinates, b.data_ro.ravel().copy(), V.V.cell_node_map,
                     V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz, alpha=1.0, beta=0.3)
    do[np.unique(np.concatenate([bc.nodes for bc in bcs]))] = 1.0
    assert relerr(d, do) < TOL


def test_advdiff_host_pointer_modes_equal_device_mode(engine):
    """The action from host pointers (monolithic path, b mirrored by its byte size; a host write to b is
    picked up by the next call) and the matrix from host pointers equal the device-mode results."""
    p = 2
    mesh, V, cells, nodes, m0, m1, X, _ = setup(p, False, ExtrudedHexMesh(4, 4, 6, warp=0.05))
    u = op2.Dat(nodes, np.random.default_rng(9).standard_normal(V.node_count))
    b = op2.Dat(op2.DataSet(nodes, 3), velocity(V.dof_coordinates(), 9))
    k = op2.Kernel("advection_diffusion", degree=p, alpha=0.0, beta=0.0)      # the convective term alone
    yd = op2.Dat(nodes)
    op2.par_loop(k, cells, yd(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), b(op2.READ, m0))
    ref = yd.data_ro.copy()
    assert np.abs(ref).max() > 0
    yh = op2.Dat(nodes)
    gk = op2.GlobalKernel(k, [m0, m1], extruded=True)
    loop = op2.Parloop(gk, cells, [yh(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), b(op2.READ, m0)],
                       location="host")
    loop()
    assert relerr(yh.data_ro, ref) < TOL
    b.data[:] *= 2.0
    yh.zero()
    loop()
    assert relerr(yh.data_ro, 2.0 * ref) < TOL
    km = op2.Kernel("advection_diffusion", degree=p, alpha=1.0, beta=0.5, rank=2)
    sparsity = op2.Sparsity((op2.DataSet(nodes, 1),) * 2, [(m0, m0, None)])
    md = op2.Mat(sparsity)
    op2.par_loop(km, cells, md(op2.INC, (m0, m0)), X(op2.READ, m1), b(op2.READ, m0))
    mh = op2.Mat(sparsity)
    _host_call(op2.GlobalKernel(km, [m0, m1], extruded=True), mesh, m0, m1, mh, [X, b])
    assert np.abs(md.values).max() > 0
    assert relerr(mh.values, md.values) < TOL
    # a host-mode b with one value per node is too short for the kernel's 3 (action and matrix alike)
    short = op2.Dat(nodes, np.ones(V.node_count))
    with pytest.raises(_lib.EngineError, match="too few"):
        _host_call(op2.GlobalKernel(km, [m0, m1], extruded=True), mesh, m0, m1, op2.Mat(sparsity), [X, short])


def test_advdiff_generic_statement_every_column_at_degree_3(engine):
    """The generic statement's device build column by column on one cell at its highest degree: every unit
    vector, including the cell's first node (the node whose b the degree-4 build reads as u)."""
    from firedrake_b200.assemble import FunctionSpace, assemble_advection_diffusion_generic
    mesh = ExtrudedHexMesh(1, 1, 1, warp=0.05)
    V = FunctionSpace(mesh, 3)
    n = V.node_count
    bn = velocity(V.V.dof_coordinates(), 1)
    b = op2.Dat(V.vector_dset(3), bn)
    for j in range(n):
        e = np.zeros(n)
        e[j] = 1.0
        y = assemble_advection_diffusion_generic(V, V.dat(e), b, alpha=0.7, beta=0.4).data_ro
        yo = ao.action(interval_element(3), mesh.coordinates, e, bn.ravel(), V.V.cell_node_map, V.V.offset,
                       mesh.coord_map, mesh.coord_offset, mesh.nz, alpha=0.7, beta=0.4)
        assert relerr(y, yo) < TOL, j


def test_advdiff_kernel_refuses_what_it_does_not_cover(engine):
    """Vector spaces, the affine variant, a non-Gauss rule, degrees outside the instantiated ranges, non-hex
    cells and periodic sets: a clear error, never a silent fall-back; multTranspose raises."""
    from firedrake_b200 import _lib
    from firedrake_b200.assemble import AdvectionDiffusion, FunctionSpace, assemble
    from firedrake_b200.fiat_lite import interval_element as ie
    mesh, V, cells, nodes, m0, m1, X, _ = setup(2, False, ExtrudedHexMesh(2, 2, 2))
    cases = ((dict(degree=2, cdim=3), "scalar"), (dict(degree=2, affine=True), "affine"),
             (dict(degree=5), "degree 5 outside 1..4"), (dict(degree=4, rank=2), "degree 4 outside 1..3"),
             (dict(degree=4, diagonal=True), "degree 4 outside 1..3"),
             (dict(degree=2, element=ie(2, 4)), "nq == degree\\+1"))
    for kw, msg in cases:
        gk = op2.GlobalKernel(op2.Kernel("advection_diffusion", **kw), [m0, m1], extruded=True)
        with pytest.raises(_lib.EngineError, match=msg):
            gk.compile()
    d = _lib.KernelDesc()
    d.form, d.rank, d.cell, d.degree, d.nq, d.cdim = _lib.FORM_ADVECTION_DIFFUSION, 1, _lib.CELL_TRIANGLE, 1, 2, 1
    import ctypes as C
    h = C.c_void_p()
    with pytest.raises(_lib.EngineError, match="hex cells"):
        _lib.check(_lib.lib().fdb_kernel_create(C.byref(d), C.byref(h)), "fdb_kernel_create")
    pcells = op2.ExtrudedSet(op2.Set(mesh.num_base_cells), mesh.layers, extruded_periodic=True)
    b = op2.Dat(op2.DataSet(nodes, 3))
    u, y = op2.Dat(nodes), op2.Dat(nodes)
    with pytest.raises(NotImplementedError, match="periodic"):
        op2.par_loop(op2.Kernel("advection_diffusion", degree=2), pcells, y(op2.INC, m0), X(op2.READ, m1),
                     u(op2.READ, m0), b(op2.READ, m0))
    with pytest.raises(ValueError, match="3 values per node"):
        op2.par_loop(op2.Kernel("advection_diffusion", degree=2), cells, y(op2.INC, m0), X(op2.READ, m1),
                     u(op2.READ, m0), op2.Dat(nodes)(op2.READ, m0))
    W = FunctionSpace(mesh, 2)
    with pytest.raises(ValueError, match="3 values per node"):
        AdvectionDiffusion(W, W.dat())
    A = assemble(AdvectionDiffusion(W, op2.Dat(W.vector_dset(3))), mat_type="matfree")
    with pytest.raises(NotImplementedError, match="advection-diffusion"):
        A.multTranspose(W.dat(), W.dat())


# ---- manufactured solves: u = sin(pi x) sin(pi y) sin(pi z) + x + y z, nonzero Dirichlet values on every
# side (lifted), b = (1 + y/2, 1/2 - x/4, 1/4) (divergence-free), alpha = 1, beta = 0.5: mesh Peclet
# number |b| h / (2 alpha) <= 0.6 h, far below 1
ALPHA, BETA = 1.0, 0.5


def _exact(X):
    x, y, z = X[:, 0], X[:, 1], X[:, 2]
    s, c, pi = np.sin, np.cos, np.pi
    S = s(pi * x) * s(pi * y) * s(pi * z)
    u = S + x + y * z
    grad = np.stack([pi * c(pi * x) * s(pi * y) * s(pi * z) + 1.0,
                     pi * s(pi * x) * c(pi * y) * s(pi * z) + z,
                     pi * s(pi * x) * s(pi * y) * c(pi * z) + y], axis=1)
    b = np.stack([1.0 + 0.5 * y, 0.5 - 0.25 * x, np.full_like(x, 0.25)], axis=1)
    f = ALPHA * 3.0 * pi ** 2 * S + (b * grad).sum(axis=1) + BETA * u
    return u, b, f


def manufactured_solve(V, pc, hierarchy=None, rtol=1e-10):
    """Solve on ``V``; returns (iterations, L2 error against the interpolated exact solution, u)."""
    from firedrake_b200.assemble import AdvectionDiffusion, DirichletBC, OneFormAssembler, mass, solve
    ue, bn, f = _exact(V.V.dof_coordinates())
    g = V.dat(ue)
    bcs = [DirichletBC(V, g, list(SIDES))]
    b = op2.Dat(V.vector_dset(3), bn)
    L = OneFormAssembler(mass(V), V.dat(f)).assemble()
    u = V.dat()
    its, hist = solve(AdvectionDiffusion(V, b, ALPHA, BETA), L, u, bcs=bcs, hierarchy=hierarchy,
                      solver_parameters={"pc_type": pc, "ksp_rtol": rtol, "ksp_max_it": 2000})
    e = V.dat(u.data_ro - ue)
    Me = OneFormAssembler(mass(V), e).assemble()
    return its, float(np.sqrt(e.data_ro @ Me.data_ro)), u


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
def test_advdiff_solve_matches_scipy(engine, pc):
    """Each preconditioner under GMRES gives scipy's solution of the oracle's matrix."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import FunctionSpace, OneFormAssembler, mass
    h = mg.MeshHierarchy(2, 2, 2, 2)
    V = FunctionSpace(h[2], 2)
    its, err, u = manufactured_solve(V, pc, h, rtol=1e-12)
    mesh = h[2]
    ue, bn, f = _exact(V.V.dof_coordinates())
    args = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    A = ao.csr(interval_element(2), mesh.coordinates, bn.ravel(), *args, alpha=ALPHA, beta=BETA)
    rhs = OneFormAssembler(mass(V), V.dat(f)).assemble().data_ro.copy()
    bnd = np.unique(np.concatenate([V.boundary_nodes(s) for s in SIDES]))
    us = ao.solve(A, rhs, bnd, ue)
    assert relerr(u.data_ro, us) < 1e-8, (pc, its)
    assert err < 1e-3


def test_advdiff_cg_refuses_and_gmres_is_the_default(engine):
    from firedrake_b200.assemble import AdvectionDiffusion, FunctionSpace, solve
    V = FunctionSpace(ExtrudedHexMesh(2, 2, 2), 1)
    form = AdvectionDiffusion(V, op2.Dat(V.vector_dset(3)))
    with pytest.raises(ValueError, match="symmetric"):
        solve(form, V.dat(), V.dat(), solver_parameters={"ksp_type": "cg"})


@pytest.mark.parametrize("p,n0", [(1, 8), (2, 4)])
def test_advdiff_l2_rates(engine, p, n0):
    from firedrake_b200.assemble import FunctionSpace
    errs = []
    for n in (n0, 2 * n0):
        _, err, _ = manufactured_solve(FunctionSpace(ExtrudedHexMesh(n, n, n), p), "jacobi")
        errs.append(err)
    rate = np.log2(errs[0] / errs[1])
    assert rate >= (1.8 if p == 1 else 2.8), (p, errs, rate)


def test_advdiff_mg_iterations(engine):
    """mg: a V-cycle of the symmetric part under GMRES; its iteration count stays nearly flat under
    refinement and is below Jacobi's at both sizes."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import FunctionSpace
    counts = {}
    for levels in (2, 3):
        h = mg.MeshHierarchy(2, 2, 2, levels)
        V = FunctionSpace(h[levels], 1)
        counts[levels] = {pc: manufactured_solve(V, pc, h, rtol=1e-8)[0] for pc in ("jacobi", "mg")}
    assert counts[3]["mg"] <= 1.25 * counts[2]["mg"], counts
    assert all(c["mg"] < c["jacobi"] for c in counts.values()), counts
