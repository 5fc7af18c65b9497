"""GPU checks of upwind DG transport on DQ_p hexahedra (FDB_FORM_DG_TRANSPORT: csrc/dg_transport_hex.cu and the
upwind kernel of csrc/dg_facet_hex.cu) against the NumPy oracle (tests/_dg_transport_oracle.py), the generic wrapper
path and InteriorPenalty; conservation, free-stream preservation, steady solves against scipy, the convergence rate,
SSPRK3 and the engine's refusals.  Parity meshes have their vertices moved in and out of plane.  Tolerance 1e-12
relative in the max norm."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import _boundary_oracle as bo
import _dg_oracle as do
import _dg_transport_oracle as to
from firedrake_b200 import op2
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

TOL = 1e-12


def relerr(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(b).max()


def perturbed(nx=3, ny=2, nz=3, seed=1):
    return bo.perturb(ExtrudedHexMesh(nx, ny, nz, Lx=1.2, Ly=0.9, Lz=1.1, warp=0.05, permute_seed=seed), 0.08, seed)


def dq(mesh, p):
    from firedrake_b200.assemble import FunctionSpace
    return FunctionSpace(mesh, p, family="DQ")


def velocity(V, values):
    return op2.Dat(op2.DataSet(V.vertex_set, 3), np.ascontiguousarray(values, dtype=float))


def random_b(mesh, seed):
    return np.random.default_rng(seed).standard_normal((mesh.coord_space.node_count, 3))


def values(n, seed):
    return np.random.default_rng(seed).standard_normal(n)


def run(loops):
    for loop in loops:
        loop()


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_terms_match_oracle(engine, p):
    """The cell, interior and exterior actions and diagonals separately (facets atomic, and coloured twice:
    bit-identical), then the whole action, the matrix-free mult and getDiagonal."""
    from firedrake_b200.assemble import DGTransport, ImplicitMatrixContext, _dg_transport_boundary_loops, assemble
    mesh = perturbed(seed=p)
    V = dq(mesh, p)
    el = do.element(p)
    bv = random_b(mesh, p)
    F = DGTransport(V, velocity(V, bv))
    x = V.dat(values(V.node_count, 10 + p))
    xo = x.data_ro.copy()
    Ac, Ai = to.cell_matrix(mesh, V.V, el, bv), to.interior_matrix(mesh, V.V, el, bv)
    Ae = to.exterior_matrix(mesh, V.V, el, bv, 1.0, 0.0)
    y = V.dat()
    op2.par_loop(F.kernel(1), V.cell_set, y(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                 x(op2.READ, V.cell_node_map), *F.coefficient_args())
    assert relerr(y.data_ro, Ac @ xo) < TOL
    terms = F.facet_terms()
    outs = []
    for scatter in ("atomic", "coloured", "coloured"):
        y = V.dat()
        y.zero()
        loops = terms.action_loops(y, x, scatter)
        run(loops[:2])
        assert relerr(y.data_ro, Ai @ xo) < TOL, scatter
        run(loops[2:])
        assert relerr(y.data_ro, (Ai + Ae) @ xo) < TOL, scatter
        outs.append(y.data_ro.copy())
    assert np.array_equal(outs[1], outs[2])
    A = to.operator(mesh, V.V, el, bv)
    assert relerr(assemble(F, u=x).data_ro, A @ xo) < TOL
    op = assemble(F, mat_type="matfree")
    ym = V.dat()
    op.mult(x, ym)
    assert relerr(ym.data_ro, A @ xo) < TOL
    assert relerr(op.getDiagonal(V.dat()).data_ro, A.diagonal()) < TOL
    D = V.dat()
    op2.par_loop(F.kernel(1, diagonal=True), V.cell_set, D(op2.INC, V.cell_node_map),
                 V.coordinates(op2.READ, V.coord_map), *F.coefficient_args())
    assert relerr(D.data_ro, Ac.diagonal()) < TOL
    g = V.dat(values(V.node_count, 20 + p))
    y = V.dat()
    y.zero()
    run(_dg_transport_boundary_loops(F, y, g, 0.7, -0.3))
    assert relerr(y.data_ro, to.exterior_matrix(mesh, V.V, el, bv, 0.7, -0.3) @ g.data_ro) < TOL


@pytest.mark.parametrize("p", [1, 3])
def test_native_hexes(engine, p):
    """The op2 level on native hexes: permuted full rows, one entry per interior facet ('+' row, '-' row) and per
    exterior facet; atomic and coloured; the cell term and the diagonals."""
    mesh = perturbed(3, 2, 3, seed=40 + p)
    W = mesh.dg_function_space(p)
    el = do.element(p)
    nd = W.arity
    perm = np.random.default_rng(p).permutation(mesh.num_cells)
    where = np.empty(mesh.num_cells, dtype=np.int64)
    where[perm] = np.arange(mesh.num_cells)
    full, cfull = W.full_cell_node_list()[perm], mesh.coord_space.full_cell_node_list()[perm]
    P, M, FP, FM = do.interior_facets(mesh)
    C_, Fe = do.exterior_facets(mesh, "on_boundary")
    nodes, vnodes = op2.Set(W.node_count), op2.Set(mesh.coord_space.node_count)
    X = op2.Dat(op2.DataSet(vnodes, 3), mesh.coordinates)
    bv = random_b(mesh, 3 + p)
    B = op2.Dat(op2.DataSet(vnodes, 3), bv)
    u = op2.Dat(nodes, values(W.node_count, 3))
    A = to.operator(mesh, W, el, bv)
    cset, iset, eset = op2.Set(mesh.num_cells), op2.Set(len(P)), op2.Set(len(C_))
    cm0 = op2.Map(cset, nodes, nd, np.ascontiguousarray(full))
    cm1 = op2.Map(cset, vnodes, 8, np.ascontiguousarray(cfull))
    im0 = op2.Map(iset, nodes, 2 * nd, np.ascontiguousarray(np.concatenate([full[where[P]], full[where[M]]], 1)))
    im1 = op2.Map(iset, vnodes, 16, np.ascontiguousarray(np.concatenate([cfull[where[P]], cfull[where[M]]], 1)))
    em0 = op2.Map(eset, nodes, nd, np.ascontiguousarray(full[where[C_]]))
    em1 = op2.Map(eset, vnodes, 8, np.ascontiguousarray(cfull[where[C_]]))
    pairs = op2.Dat(op2.DataSet(iset, 2), np.stack([FP, FM], 1).astype(np.uint32), dtype=np.uint32)
    fac = op2.Dat(op2.DataSet(eset, 1), Fe.astype(np.uint32), dtype=np.uint32)
    k = {i: op2.Kernel("dg_transport", degree=p, integral=i, element=el) for i in ("cell", "interior_facet",
                                                                                  "exterior_facet")}
    outs = []
    for scatter in ("atomic", "coloured", "coloured"):
        y = op2.Dat(nodes)
        op2.par_loop(k["cell"], cset, y(op2.INC, cm0), X(op2.READ, cm1), u(op2.READ, cm0), B(op2.READ, cm1),
                     scatter=scatter)
        op2.par_loop(k["interior_facet"], iset, y(op2.INC, im0), X(op2.READ, im1), u(op2.READ, im0),
                     B(op2.READ, im1), pairs(op2.READ), scatter=scatter)
        op2.par_loop(k["exterior_facet"], eset, y(op2.INC, em0), X(op2.READ, em1), u(op2.READ, em0),
                     B(op2.READ, em1), fac(op2.READ), scatter=scatter)
        assert relerr(y.data_ro, A @ u.data_ro) < TOL, scatter
        outs.append(y.data_ro.copy())
    assert np.array_equal(outs[1], outs[2])
    kd = {i: op2.Kernel("dg_transport", degree=p, integral=i, diagonal=True, element=el) for i in k}
    d = op2.Dat(nodes)
    op2.par_loop(kd["cell"], cset, d(op2.INC, cm0), X(op2.READ, cm1), B(op2.READ, cm1))
    op2.par_loop(kd["interior_facet"], iset, d(op2.INC, im0), X(op2.READ, im1), B(op2.READ, im1), pairs(op2.READ))
    op2.par_loop(kd["exterior_facet"], eset, d(op2.INC, em0), X(op2.READ, em1), B(op2.READ, em1), fac(op2.READ))
    assert relerr(d.data_ro, A.diagonal()) < TOL


@pytest.mark.parametrize("p", [1, 2, 3])
def test_generic_path(engine, p):
    from firedrake_b200.assemble import DGTransport, assemble, assemble_dg_transport_generic
    mesh = perturbed(3, 3, 2, seed=20 + p)
    V = dq(mesh, p)
    F = DGTransport(V, velocity(V, random_b(mesh, 20 + p)))
    x = V.dat(values(V.node_count, 30 + p))
    y = assemble(F, u=x).data_ro.copy()
    assert relerr(assemble_dg_transport_generic(F, x).data_ro, y) < TOL


@pytest.mark.parametrize("p", [1, 3])
def test_zero_velocity_is_interior_penalty(engine, p):
    from firedrake_b200.assemble import DGTransport, InteriorPenalty, assemble
    mesh = perturbed(seed=50 + p)
    V = dq(mesh, p)
    eta = 3.0 * (p + 1) ** 2
    x = V.dat(values(V.node_count, p))
    F = DGTransport(V, velocity(V, np.zeros((mesh.coord_space.node_count, 3))), 0.4, 1.3, eta, (1, "top"))
    y = assemble(F, u=x).data_ro.copy()
    assert relerr(y, assemble(InteriorPenalty(V, 1.3, 0.4, eta, (1, "top")), u=x).data_ro) < TOL


@pytest.mark.parametrize("p", [1, 2, 4])
def test_conservation_and_free_stream(engine, p):
    """1^T A q is the outflow flux on the device; a constant field in a constant flow on parallelepipeds gives
    A 1 = inflow_load(1)."""
    from firedrake_b200.assemble import DGTransport, assemble, inflow_load
    mesh = perturbed(seed=70 + p)
    V = dq(mesh, p)
    bv = random_b(mesh, 70 + p)
    q = V.dat(values(V.node_count, 71 + p))
    Aq = assemble(DGTransport(V, velocity(V, bv)), u=q).data_ro
    out = to.outflow_integral(mesh, V.V, do.element(p), bv, q.data_ro)
    assert abs(Aq.sum() - out) < 1e-12 * np.abs(Aq).sum()
    box = ExtrudedHexMesh(3, 2, 2, permute_seed=3)
    box.coordinates[:] = box.coordinates @ np.array([[1.0, 0.25, 0.125], [0.0, 1.25, -0.25], [0.125, 0.0, 0.75]]).T
    W = dq(box, p)
    F = DGTransport(W, velocity(W, np.tile([0.7, -0.4, 0.3], (box.coord_space.node_count, 1))))
    one = W.dat(np.ones(W.node_count))
    g = inflow_load(F, one).data_ro.copy()
    assert np.abs(assemble(F, u=one).data_ro - g).max() < 1e-12 * np.abs(g).max()


@pytest.mark.parametrize("p,pc,beta", [(1, "none", 1.0), (2, "jacobi", 1.0), (4, "none", 1.0), (4, "jacobi", 0.0)])
def test_steady_solve_matches_scipy(engine, p, pc, beta):
    """Advection(-reaction) with an inflow condition: GMRES against spsolve of the oracle matrix.  Jacobi at DQ4 is
    pure transport, whose diagonal covers DQ4 (with beta the Helmholtz diagonal stops at DQ3)."""
    from firedrake_b200.assemble import DGTransport, inflow_load, solve
    mesh = perturbed(3, 3, 3, seed=80 + p)
    V = dq(mesh, p)
    el = do.element(p)
    bv = np.tile([1.0, 0.6, -0.3], (mesh.coord_space.node_count, 1)) + 0.2 * random_b(mesh, p)
    F = DGTransport(V, velocity(V, bv), beta=beta)
    g = V.dat(values(V.node_count, 81))
    L = inflow_load(F, g)
    u = V.dat()
    its, _ = solve(F, L, u, solver_parameters={"pc_type": pc, "ksp_rtol": 1e-12, "ksp_max_it": 3000})
    ref = spla.spsolve(to.operator(mesh, V.V, el, bv, beta=beta).tocsc(), to.inflow_load(mesh, V.V, el, bv, g.data_ro))
    assert relerr(u.data_ro, ref) < 1e-8, its


def _dof_points(mesh, W, el):
    rows, Xc = do.cells(mesh, W)
    q = np.stack(np.meshgrid(el.xq, el.xq, el.xq, indexing="ij"), axis=-1).reshape(-1, 3)
    pts = np.empty((W.node_count, 3))
    pts[rows] = np.einsum("qv,cvi->cqi", to.vertex_weights(q), Xc)
    return pts


@pytest.mark.parametrize("p", [1, 2, 3])
def test_convergence_rate(engine, p):
    """b.grad u + u = f with u = exp(x/2) sin(2y) cos(z) and exact inflow values: the L2 error falls at least as
    h^(p + 0.4) from 4^3 to 8^3."""
    from firedrake_b200.assemble import DGTransport, assemble, inflow_load, mass, solve
    bvec = np.array([1.0, 0.5, 0.25])
    ue = lambda X: np.exp(X[:, 0] / 2) * np.sin(2 * X[:, 1]) * np.cos(X[:, 2])

    def f(X):
        x, y, z = X.T
        e = np.exp(x / 2)
        return (bvec[0] * 0.5 * e * np.sin(2 * y) * np.cos(z) + bvec[1] * 2 * e * np.cos(2 * y) * np.cos(z)
                - bvec[2] * e * np.sin(2 * y) * np.sin(z) + ue(X))

    errs = []
    for n in (4, 8):
        mesh = ExtrudedHexMesh(n, n, n)
        V = dq(mesh, p)
        X = _dof_points(mesh, V.V, do.element(p))
        F = DGTransport(V, velocity(V, np.tile(bvec, (mesh.coord_space.node_count, 1))), beta=1.0)
        L = assemble(mass(V), u=V.dat(f(X)))
        L.axpy(1.0, inflow_load(F, V.dat(ue(X))))
        u = V.dat()
        solve(F, L, u, solver_parameters={"ksp_rtol": 1e-12, "ksp_max_it": 3000})
        m = assemble(mass(V), u=V.dat(np.ones(V.node_count))).data_ro
        errs.append(np.sqrt(np.sum(m * (u.data_ro - ue(X)) ** 2)))
    assert np.log2(errs[0] / errs[1]) >= p + 0.4, errs


def test_advection_diffusion_with_nitsche(engine):
    from firedrake_b200.assemble import DGTransport, inflow_load, nitsche_load, solve
    p = 2
    mesh = perturbed(3, 3, 2, seed=90)
    V = dq(mesh, p)
    el = do.element(p)
    bv = np.tile([1.0, -0.5, 0.2], (mesh.coord_space.node_count, 1))
    eta = 3.0 * (p + 1) ** 2
    F = DGTransport(V, velocity(V, bv), 0.0, 0.1, eta, "on_boundary")
    g = V.dat(values(V.node_count, 91))
    L = nitsche_load(F, g)
    L.axpy(1.0, inflow_load(F, g))
    u = V.dat()
    solve(F, L, u, solver_parameters={"pc_type": "jacobi", "ksp_rtol": 1e-12, "ksp_max_it": 3000})
    A = to.operator(mesh, V.V, el, bv, 0.0, 0.1, eta, "on_boundary")
    rhs = do.nitsche_load(mesh, V.V, el, 0.1, eta, "on_boundary", g.data_ro) + \
        to.inflow_load(mesh, V.V, el, bv, g.data_ro)
    assert relerr(u.data_ro, spla.spsolve(A.tocsc(), rhs)) < 1e-8


@pytest.mark.parametrize("p", [1, 4])
def test_ssprk3_step_matches_oracle(engine, p):
    from firedrake_b200.assemble import DGTransport, inflow_load, ssprk3
    mesh = perturbed(seed=100 + p)
    V = dq(mesh, p)
    el = do.element(p)
    bv = random_b(mesh, 100 + p)
    F = DGTransport(V, velocity(V, bv))
    q0 = values(V.node_count, 101)
    g = V.dat(values(V.node_count, 102))
    load = inflow_load(F, g)
    q = ssprk3(F, V.dat(q0.copy()), 2e-3, 1, load=load)
    ref = to.ssprk3_step(to.operator(mesh, V.V, el, bv), to.mass_diagonal(mesh, V.V, el), q0, 2e-3,
                         to.inflow_load(mesh, V.V, el, bv, g.data_ro))
    assert relerr(q.data_ro, ref) < TOL


def test_ssprk3_conserves_mass_in_a_closed_flow(engine):
    """b = (sin(pi x) cos(pi y), -cos(pi x) sin(pi y), 0) has b.n = 0 on the unit cube's boundary: sum m_i q_i stays
    constant to 1e-12 relative over 100 steps."""
    from firedrake_b200.assemble import DGTransport, assemble, mass, ssprk3
    mesh = ExtrudedHexMesh(8, 8, 4)
    V = dq(mesh, 2)
    Xv = mesh.coordinates
    bv = np.stack([np.sin(np.pi * Xv[:, 0]) * np.cos(np.pi * Xv[:, 1]),
                   -np.cos(np.pi * Xv[:, 0]) * np.sin(np.pi * Xv[:, 1]), np.zeros(len(Xv))], axis=1)
    F = DGTransport(V, velocity(V, bv))
    X = _dof_points(mesh, V.V, do.element(2))
    q = V.dat(np.exp(-20 * ((X[:, 0] - 0.4) ** 2 + (X[:, 1] - 0.6) ** 2)))
    m = assemble(mass(V), u=V.dat(np.ones(V.node_count))).data_ro.copy()
    m0 = float(m @ q.data_ro)
    ssprk3(F, q, 0.01, 100)
    assert np.all(np.isfinite(q.data_ro))
    assert abs(float(m @ q.data_ro) - m0) < 1e-12 * abs(m0)


def test_refusals(engine):
    from firedrake_b200.assemble import DGTransport
    from firedrake_b200.fiat_lite import interval_element
    mesh = ExtrudedHexMesh(2, 2, 2)
    V = dq(mesh, 1)
    b = velocity(V, np.zeros((mesh.coord_space.node_count, 3)))
    maps = [V.cell_node_map, V.coord_map]
    cases = [(dict(degree=1, rank=2, element=V.element), "no assembled DG matrix"),
             (dict(degree=2, element=interval_element(2)), "collocated Gauss-Legendre"),
             (dict(degree=5, element=interval_element(5, variant="gl")), "degree 5 outside 1..4")]
    for kw, msg in cases:
        with pytest.raises(Exception, match=msg):
            op2.GlobalKernel(op2.Kernel("dg_transport", **kw), maps, extruded=True).compile()
    F = DGTransport(V, b)
    x, y = V.dat(np.ones(V.node_count)), V.dat()
    gk = op2.GlobalKernel(F.kernel(1), maps, extruded=True)
    with pytest.raises(Exception, match="device-resident Dats only"):
        op2.Parloop(gk, V.cell_set, [y(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                                     x(op2.READ, V.cell_node_map), b(op2.READ, V.coord_map)], location="host")()
    with pytest.raises(ValueError, match="3 values per vertex"):
        op2.Parloop(gk, V.cell_set, [y(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                                     x(op2.READ, V.cell_node_map), x(op2.READ, V.cell_node_map)])
