"""GPU parity of the boundary mass term gamma*inner(u, v)*ds(sub_domain) (FDB_FORM_BOUNDARY_MASS, csrc/boundary_hex.cu)
against the NumPy oracle (tests/_boundary_oracle.py) and the generic wrapper path, and the solves that use it: Robin,
Neumann and traction conditions on the Helmholtz family, elasticity, advection-diffusion, nonlinear diffusion and
hyperelasticity.  Every parity mesh has its vertices moved in and out of plane (the mesh's own warp vanishes on the
box boundary, which would leave every boundary face a flat rectangle).  Tolerance 1e-12 relative in the max norm."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import _boundary_oracle as bo
from firedrake_b200 import op2
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

TOL = 1e-12
SUBS = [1, 2, 3, 4, "bottom", "top", "on_boundary", (2, "top")]


def relerr(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(b).max()


def perturbed(nx=3, ny=2, nz=3, seed=1):
    return bo.perturb(ExtrudedHexMesh(nx, ny, nz, Lx=1.2, Ly=0.9, Lz=1.1, warp=0.05, permute_seed=seed), 0.08, seed)


def values(n, cdim, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(n) if cdim == 1 else rng.standard_normal((n, cdim))


def oracle_action(mesh, V, u, gamma, sub, cdim):
    rows, vrows, f = bo.extruded_facets(mesh, V.V, sub)
    return bo.action(interval_element(V.degree), mesh.coordinates, np.asarray(u).ravel().copy(), rows, vrows, f,
                     gamma, cdim)


def to_scipy(A, cdim):
    ro, ci, vals = A.csr()
    n = len(ro) - 1
    if cdim == 1:
        return sp.csr_matrix((vals, ci, ro), shape=(n, n))
    return sp.bsr_matrix((vals.reshape(-1, cdim, cdim), ci, ro), shape=(n * cdim, n * cdim)).tocsr()


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("cdim", [1, 3])
def test_action_matches_oracle_extruded(engine, p, cdim):
    """assemble(BoundaryMass(V, gamma, "on_boundary"), u=u), atomic and coloured; coloured is bit-identical over
    two calls."""
    from firedrake_b200.assemble import BoundaryMass, FunctionSpace, OneFormAssembler
    mesh = perturbed()
    V = FunctionSpace(mesh, p, cdim)
    u = V.dat(values(V.node_count, cdim, p))
    F = BoundaryMass(V, 1.7, "on_boundary")
    yo = oracle_action(mesh, V, u.data_ro, 1.7, "on_boundary", cdim)
    y = OneFormAssembler(F, u).assemble()
    assert relerr(y.data_ro.ravel(), yo) < TOL
    asm = OneFormAssembler(F, u, scatter="coloured")
    outs = [asm.assemble().data_ro.copy() for _ in range(2)]
    assert np.array_equal(outs[0], outs[1])
    assert relerr(outs[0].ravel(), yo) < TOL


def native_facets(mesh, V, perm):
    """Native hexes (one map row per cell, cells in the random order ``perm``): the iteration entries of every
    exterior facet, built from the cells that touch the boundary."""
    nz = mesh.nz
    where = np.empty(mesh.num_cells, dtype=np.int64)
    where[perm] = np.arange(mesh.num_cells)                 # native index of (column, layer) row col*nz + layer
    cells, local = mesh.exterior_vertical_facets()
    ent, fac = [], []
    for c, f in zip(cells, local):
        ent += [where[c * nz + l] for l in range(nz)]
        fac += [int(f)] * nz
    for c in range(mesh.num_base_cells):
        ent += [where[c * nz], where[c * nz + nz - 1]]
        fac += [4, 5]
    return np.array(ent), np.array(fac, dtype=np.uint32)


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("cdim", [1, 3])
def test_action_matches_oracle_native(engine, p, cdim):
    """The op2 level on native hexes: permuted full map rows, one iteration entry per facet; atomic and coloured."""
    mesh = perturbed(seed=4)
    W = mesh.function_space(p)
    perm = np.random.default_rng(0).permutation(mesh.num_cells)
    full, cfull = W.full_cell_node_list()[perm], mesh.coord_space.full_cell_node_list()[perm]
    ent, fac = native_facets(mesh, W, perm)
    nodes, vnodes = op2.Set(W.node_count), op2.Set(mesh.coord_space.node_count)
    fset = op2.Set(len(ent))
    m0 = op2.Map(fset, nodes, W.arity, np.ascontiguousarray(full[ent]))
    m1 = op2.Map(fset, vnodes, 8, np.ascontiguousarray(cfull[ent]))
    facet = op2.Dat(op2.DataSet(fset, 1), fac, dtype=np.uint32)
    X = op2.Dat(op2.DataSet(vnodes, 3), mesh.coordinates)
    dset = op2.DataSet(nodes, cdim)
    u = op2.Dat(dset, values(W.node_count, cdim, 10 + p))
    yo = bo.action(interval_element(p), mesh.coordinates, u.data_ro.ravel().copy(), full[ent], cfull[ent], fac,
                   0.6, cdim)
    k = op2.Kernel("boundary_mass", degree=p, alpha=0.6, cdim=cdim, integral="exterior_facet")
    outs = []
    for scatter in ("atomic", "coloured", "coloured"):
        y = op2.Dat(dset)
        op2.par_loop(k, fset, y(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), facet(op2.READ), scatter=scatter)
        assert relerr(y.data_ro.ravel(), yo) < TOL, scatter
        outs.append(y.data_ro.copy())
    assert np.array_equal(outs[1], outs[2])


@pytest.mark.parametrize("sub", SUBS, ids=str)
def test_each_sub_domain(engine, sub):
    from firedrake_b200.assemble import BoundaryMass, FunctionSpace, assemble
    mesh = perturbed(seed=2)
    V = FunctionSpace(mesh, 2)
    u = V.dat(values(V.node_count, 1, 3))
    y = assemble(BoundaryMass(V, 0.8, sub), u=u)
    assert relerr(y.data_ro, oracle_action(mesh, V, u.data_ro, 0.8, sub, 1)) < TOL


@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("cdim", [1, 3])
def test_matrix_and_diagonal_match_oracle(engine, p, cdim):
    """The aij Mat entrywise against the oracle's global matrix; the matrix-free diagonal against its diagonal and
    the assembled one; Mat.mult against the matrix-free mult."""
    from firedrake_b200.assemble import BoundaryMass, FunctionSpace, ImplicitMatrixContext, assemble
    mesh = perturbed(seed=3)
    V = FunctionSpace(mesh, p, cdim)
    F = BoundaryMass(V, 1.3, "on_boundary")
    rows, vrows, f = bo.extruded_facets(mesh, V.V, "on_boundary")
    Ao = bo.matrix(interval_element(p), mesh.coordinates, V.node_count, rows, vrows, f, 1.3, cdim)
    A = to_scipy(assemble(F), cdim)
    assert abs(A - Ao).max() < TOL * abs(Ao).max()
    d = ImplicitMatrixContext(F).getDiagonal(V.dat()).data_ro.ravel()
    assert relerr(d, Ao.diagonal()) < TOL
    assert relerr(d, A.diagonal()) < TOL
    x = V.dat(values(V.node_count, cdim, 7))
    ymf = V.dat()
    assemble(F, mat_type="matfree").mult(x, ymf)
    assert relerr(ymf.data_ro.ravel(), A @ x.data_ro.ravel()) < TOL


@pytest.mark.parametrize("cdim", [1, 3])
def test_degree5_diagonal(engine, cdim):
    from firedrake_b200.assemble import BoundaryMass, FunctionSpace, ImplicitMatrixContext
    mesh = perturbed(2, 2, 2, seed=6)
    V = FunctionSpace(mesh, 5, cdim)
    rows, vrows, f = bo.extruded_facets(mesh, V.V, (1, "top"))
    Ao = bo.matrix(interval_element(5), mesh.coordinates, V.node_count, rows, vrows, f, 0.4, cdim)
    d = ImplicitMatrixContext(BoundaryMass(V, 0.4, (1, "top"))).getDiagonal(V.dat()).data_ro.ravel()
    assert relerr(d, Ao.diagonal()) < TOL


@pytest.mark.parametrize("p", [1, 2, 3])
@pytest.mark.parametrize("cdim", [1, 3])
def test_matches_generic_path(engine, p, cdim):
    from firedrake_b200.assemble import BoundaryMass, FunctionSpace, assemble, assemble_boundary_mass_generic
    mesh = perturbed(seed=5)
    V = FunctionSpace(mesh, p, cdim)
    u = V.dat(values(V.node_count, cdim, 20 + p))
    yg = assemble_boundary_mass_generic(V, u, 0.9, "on_boundary")
    yh = assemble(BoundaryMass(V, 0.9, "on_boundary"), u=u)
    assert relerr(yh.data_ro, yg.data_ro) < TOL


def test_refusals(engine):
    import ctypes as C
    from firedrake_b200 import _lib
    from firedrake_b200.assemble import FunctionSpace, _boundary_groups
    mesh = ExtrudedHexMesh(2, 2, 2)
    V = FunctionSpace(mesh, 2)
    fset, fmap, cmap, facet = _boundary_groups(V, "on_boundary")[0]

    def refused(msg, **kw):
        kw.setdefault("integral", "exterior_facet")
        kw.setdefault("degree", 2)
        gk = op2.GlobalKernel(op2.Kernel("boundary_mass", **kw), [fmap, cmap], extruded=True)
        with pytest.raises(_lib.EngineError, match=msg):
            gk.compile()

    refused("boundary_mass has exterior-facet integrals only .*a cell integral", integral="cell")
    refused("boundary_mass has exterior-facet integrals only .*interior facets are not supported",
            integral="interior_facet")
    refused("boundary_mass action takes a scalar space or a vector space of value size 3", cdim=2)
    refused("boundary_mass action: degree 6 outside 1..5", degree=6)
    refused("boundary_mass matrix: degree 5 outside 1..4", degree=5, rank=2)
    refused("boundary_mass has no affine-cell variant", affine=True)
    refused("boundary_mass needs nq == degree\\+1", element=interval_element(2, 4))
    # extruded cells without layer offsets (the descriptor as a C caller could fill it)
    el = interval_element(1)
    d = _lib.KernelDesc()
    d.form, d.rank, d.cell, d.integral = _lib.FORM_BOUNDARY_MASS, 1, _lib.CELL_HEX_EXTRUDED, _lib.INTEGRAL_EXTERIOR_FACET
    d.degree, d.nq, d.cdim = 1, 2, 1
    for q in range(2):
        for a in range(2):
            d.B[q * 2 + a], d.D[q * 2 + a] = el.B[q, a], el.D[q, a]
    h = C.c_void_p()
    assert engine.fdb_kernel_create(C.byref(d), C.byref(h)) != 0
    assert "boundary_mass on extruded cells needs the layer offsets" in engine.fdb_last_error().decode()
    # host location and wrong argument counts, at the call
    u, y = V.dat(np.ones(V.node_count)), V.dat()
    k = op2.Kernel("boundary_mass", degree=2, integral="exterior_facet")
    with pytest.raises(_lib.EngineError, match="boundary_mass takes device-resident Dats only"):
        op2.par_loop(k, fset, y(op2.INC, fmap), V.coordinates(op2.READ, cmap), u(op2.READ, fmap), facet(op2.READ),
                     location="host")
    gk = op2.GlobalKernel(k, [fmap, cmap], extruded=True)
    with pytest.raises(_lib.EngineError, match="boundary_mass action expects 4 device args"):
        gk(0, fset.total_size, fset.layers_array.ravel(), None, [y.device_ptr, V.coordinates.device_ptr,
                                                                  u.device_ptr], None, None,
           [fmap.device_ptr, cmap.device_ptr], None, _lib.LOC_DEVICE, False, False)


# ------------------------------------------------------------------------------------------------------ solves
def _dirichlet_solve(A, b, nodes, values, cdim=1):
    """scipy: A x = b with x = values on the constrained nodes (every component)."""
    n = A.shape[0]
    fixed = np.zeros(n, dtype=bool)
    dofs = (np.asarray(nodes)[:, None] * cdim + np.arange(cdim)[None, :]).ravel()
    fixed[dofs] = True
    x = np.zeros(n)
    x[fixed] = np.asarray(values).ravel()[fixed] if np.ndim(values) else values
    free = ~fixed
    rhs = b - A @ x
    x[free] = spla.spsolve(A[free][:, free].tocsc(), rhs[free])
    return x


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
def test_helmholtz_robin_dirichlet_neumann(engine, pc):
    """Form(V, 1, 0.5, ds=((2, 2),)) with u = 1 on side 1, a Robin condition on side 2 (h = 2, u_inf = 0.3) and a
    Neumann flux g on "top": L = assemble(mass(V), u=f) + assemble(BoundaryMass(V, 2, 2), u=u_inf) +
    assemble(BoundaryMass(V, 1, "top"), u=g), against scipy on the cell matrix plus the oracle's boundary matrix."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import BoundaryMass, DirichletBC, Form, FunctionSpace, assemble, mass, solve
    h = mg.MeshHierarchy(2, 2, 2, 2)
    mesh = h[2]
    V = FunctionSpace(mesh, 2)
    Xn = V.V.dof_coordinates()
    f = V.dat(1.0 + Xn[:, 0] * Xn[:, 2])
    uinf = V.dat(np.full(V.node_count, 0.3))
    g = V.dat(np.sin(3 * Xn[:, 0]) + Xn[:, 1])
    L = assemble(mass(V), u=f)
    L.axpy(1.0, assemble(BoundaryMass(V, 2.0, 2), u=uinf))
    L.axpy(1.0, assemble(BoundaryMass(V, 1.0, "top"), u=g))
    bcs = [DirichletBC(V, 1.0, 1)]
    u = V.dat()
    its, hist = solve(Form(V, 1.0, 0.5, ds=((2.0, 2),)), L, u, bcs=bcs, hierarchy=h,
                      solver_parameters={"pc_type": pc, "ksp_rtol": 1e-12, "ksp_max_it": 3000})
    el = interval_element(2)
    rows, vrows, fc = bo.extruded_facets(mesh, V.V, 2)
    A = to_scipy(assemble(Form(V, 1.0, 0.5)), 1) + bo.matrix(el, mesh.coordinates, V.node_count, rows, vrows, fc, 2.0)
    x = _dirichlet_solve(A, L.data_ro.copy(), bcs[0].nodes, 1.0)
    assert relerr(u.data_ro, x) < 1e-8, (pc, its)
    if pc == "mg":
        assert its < 40, its


def test_elasticity_clamped_with_traction(engine):
    """Clamped on side 1, the traction t = (0.1, -0.05, 0.02) on side 2 through assemble(BoundaryMass(V, 1, 2),
    u=t), solved with the V-cycle, against scipy; the load equals the oracle's."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import BoundaryMass, DirichletBC, Elasticity, FunctionSpace, assemble, solve
    h = mg.MeshHierarchy(2, 2, 2, 1)
    mesh = h[1]
    V = FunctionSpace(mesh, 2, 3)
    t = V.dat(np.tile([0.1, -0.05, 0.02], (V.node_count, 1)))
    L = assemble(BoundaryMass(V, 1.0, 2), u=t)
    assert relerr(L.data_ro.ravel(), oracle_action(mesh, V, t.data_ro, 1.0, 2, 3)) < TOL
    F = Elasticity(V, 1.0, 1.5)
    bcs = [DirichletBC(V, 0.0, 1)]
    u = V.dat()
    its, _ = solve(F, L, u, bcs=bcs, hierarchy=h, solver_parameters={"pc_type": "mg", "ksp_rtol": 1e-12,
                                                                     "ksp_max_it": 2000})
    x = _dirichlet_solve(to_scipy(assemble(F), 3), L.data_ro.ravel().copy(), bcs[0].nodes, 0.0, 3)
    assert relerr(u.data_ro.ravel(), x) < 1e-8, its


def test_elasticity_with_elastic_support_mg(engine):
    """ds on Elasticity (an elastic support on "bottom") through the matrix-free operator, its diagonal and the
    V-cycle, against scipy on the assembled matrix with the same ds (checked against the oracle above)."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import BoundaryMass, Elasticity, FunctionSpace, assemble, solve
    h = mg.MeshHierarchy(2, 2, 2, 1)
    mesh = h[1]
    V = FunctionSpace(mesh, 1, 3)
    F = Elasticity(V, 1.0, 1.0, ds=((5.0, "bottom"),))
    L = assemble(BoundaryMass(V, 1.0, "top"), u=V.dat(np.tile([0.0, 0.0, -0.1], (V.node_count, 1))))
    el = interval_element(1)
    rows, vrows, fc = bo.extruded_facets(mesh, V.V, "bottom")
    A = to_scipy(assemble(Elasticity(V, 1.0, 1.0)), 3) + bo.matrix(el, mesh.coordinates, V.node_count, rows, vrows,
                                                                    fc, 5.0, 3)
    assert abs(to_scipy(assemble(F), 3) - A).max() < TOL * abs(A).max()
    x = spla.spsolve(A.tocsc(), L.data_ro.ravel())
    for pc in ("jacobi", "mg"):
        u = V.dat()
        its, _ = solve(F, L, u, hierarchy=h, solver_parameters={"pc_type": pc, "ksp_rtol": 1e-12, "ksp_max_it": 3000})
        assert relerr(u.data_ro.ravel(), x) < 1e-8, (pc, its)


def test_advection_diffusion_robin_outflow_gmres(engine):
    from firedrake_b200.assemble import AdvectionDiffusion, BoundaryMass, DirichletBC, FunctionSpace, assemble, solve
    mesh = perturbed(4, 3, 3, seed=7)
    V = FunctionSpace(mesh, 2)
    b = op2.Dat(V.vector_dset(3), np.tile([1.0, 0.3, 0.0], (V.node_count, 1)))
    F = AdvectionDiffusion(V, b, 0.1, 0.0, ds=((1.0, 2),))
    L = assemble(BoundaryMass(V, 1.0, 2), u=V.dat(np.full(V.node_count, 0.2)))
    bcs = [DirichletBC(V, 1.0, 1)]
    u = V.dat()
    its, _ = solve(F, L, u, bcs=bcs, solver_parameters={"pc_type": "jacobi", "ksp_rtol": 1e-12, "ksp_max_it": 3000})
    rows, vrows, fc = bo.extruded_facets(mesh, V.V, 2)
    A = to_scipy(assemble(AdvectionDiffusion(V, b, 0.1, 0.0)), 1) + \
        bo.matrix(interval_element(2), mesh.coordinates, V.node_count, rows, vrows, fc, 1.0)
    x = _dirichlet_solve(A, L.data_ro.copy(), bcs[0].nodes, 1.0)
    assert relerr(u.data_ro, x) < 1e-8, its


def test_nonlinear_diffusion_robin_cooling_newton(engine):
    """Newton on D(u) = 1 + 0.5 u + 0.2 u^2 with Robin cooling on "top" (h = 3, u_inf = 0.5) converges, and the
    residual with ds passes the Taylor test against F.jacobian(u), which carries the same ds."""
    from firedrake_b200.assemble import (BoundaryMass, DirichletBC, FunctionSpace, NonlinearDiffusion, assemble, mass,
                                         solve_nonlinear)
    mesh = perturbed(3, 3, 3, seed=8)
    V = FunctionSpace(mesh, 2)
    F = NonlinearDiffusion(V, 1.0, 0.0, (1.0, 0.5, 0.2), ds=((3.0, "top"),))
    assert F.jacobian(V.dat()).ds == F.ds
    L = assemble(mass(V), u=V.dat(np.full(V.node_count, 4.0)))
    L.axpy(1.0, assemble(BoundaryMass(V, 3.0, "top"), u=V.dat(np.full(V.node_count, 0.5))))
    u = V.dat()
    hist, kits = solve_nonlinear(F, L, u, bcs=[DirichletBC(V, 0.0, "bottom")],
                                 solver_parameters={"pc_type": "jacobi", "ksp_rtol": 1e-10, "snes_rtol": 1e-10})
    assert hist[-1] <= 1e-10 * hist[0] and len(kits) < 12, hist
    rng = np.random.default_rng(1)
    u0 = V.dat(0.3 + 0.1 * rng.standard_normal(V.node_count))
    w = V.dat(rng.standard_normal(V.node_count))
    R0 = assemble(F, u=u0).data_ro.copy()
    Jw = assemble(F.jacobian(u0), u=w).data_ro.copy()
    errs = []
    for eps in (1e-2, 5e-3):
        R1 = assemble(F, u=V.dat(u0.data_ro + eps * w.data_ro)).data_ro
        errs.append(np.abs(R1 - R0 - eps * Jw).max())
    assert 3.5 < errs[0] / errs[1] < 4.5, errs
    # the linear part: at d = (1, 0, 0) the residual with ds is the Form with the same ds
    from firedrake_b200.assemble import Form
    Fl = NonlinearDiffusion(V, 1.0, 0.0, (1.0, 0.0, 0.0), ds=((3.0, "top"),))
    assert relerr(assemble(Fl, u=u0).data_ro, assemble(Form(V, 1.0, 0.0, ds=((3.0, "top"),)), u=u0).data_ro) < TOL


def test_hyperelastic_block_under_traction(engine):
    from firedrake_b200.assemble import BoundaryMass, DirichletBC, FunctionSpace, HyperElasticity, assemble, \
        solve_nonlinear
    mesh = ExtrudedHexMesh(3, 2, 2)
    V = FunctionSpace(mesh, 2, 3)
    L = assemble(BoundaryMass(V, 1.0, 2), u=V.dat(np.tile([0.2, 0.0, -0.05], (V.node_count, 1))))
    u = V.dat()
    hist, kits = solve_nonlinear(HyperElasticity(V, 1.0, 1.0), L, u, bcs=[DirichletBC(V, 0.0, 1)],
                                 solver_parameters={"pc_type": "jacobi", "ksp_rtol": 1e-10, "snes_rtol": 1e-10})
    assert hist[-1] <= 1e-10 * hist[0] and len(kits) < 10, hist
    ux = u.data_ro[V.boundary_nodes(2), 0]
    assert ux.min() > 0.0


def _manufactured_error(n, p):
    """-div grad u + u = f on the unit cube, u = sin(x + 0.5) cos(0.7 y) exp(0.3 z): Robin on "top"
    (du/dn + 2 u = g_R) and Neumann fluxes du/dn on the other five sides, every load through BoundaryMass."""
    from firedrake_b200.assemble import BoundaryMass, Form, FunctionSpace, assemble, mass, solve
    V = FunctionSpace(ExtrudedHexMesh(n, n, n), p)
    x, y, z = V.V.dof_coordinates().T
    ue = np.sin(x + 0.5) * np.cos(0.7 * y) * np.exp(0.3 * z)
    ux = np.cos(x + 0.5) * np.cos(0.7 * y) * np.exp(0.3 * z)
    uy = -0.7 * np.sin(x + 0.5) * np.sin(0.7 * y) * np.exp(0.3 * z)
    uz = 0.3 * ue
    f = ue * (1.0 + 0.49 + 1.0 - 0.09)
    L = assemble(mass(V), u=V.dat(f))
    for sub, flux in ((1, -ux), (2, ux), (3, -uy), (4, uy), ("bottom", -uz), ("top", uz + 2.0 * ue)):
        L.axpy(1.0, assemble(BoundaryMass(V, 1.0, sub), u=V.dat(flux)))
    u = V.dat()
    solve(Form(V, 1.0, 1.0, ds=((2.0, "top"),)), L, u,
          solver_parameters={"pc_type": "jacobi", "ksp_rtol": 1e-13, "ksp_max_it": 5000})
    e = V.dat(u.data_ro - ue)
    return float(np.sqrt(np.dot(e.data_ro, assemble(mass(V), u=e).data_ro)))


@pytest.mark.parametrize("p", [1, 2, 3])
def test_robin_neumann_convergence_rate(engine, p):
    e1, e2 = _manufactured_error(3, p), _manufactured_error(6, p)
    rate = np.log2(e1 / e2)
    assert rate > p + 0.8, (p, e1, e2, rate)


def test_mg_iterations_with_robin_do_not_grow(engine):
    from firedrake_b200 import mg
    from firedrake_b200.assemble import BoundaryMass, DirichletBC, Form, FunctionSpace, assemble, solve
    its = []
    for levels in (2, 3):
        h = mg.MeshHierarchy(2, 2, 2, levels)
        V = FunctionSpace(h[levels], 2)
        L = assemble(BoundaryMass(V, 4.0, (2, 4)), u=V.dat(np.ones(V.node_count)))
        n, _ = solve(Form(V, 1.0, 0.0, ds=((4.0, (2, 4)),)), L, V.dat(), bcs=[DirichletBC(V, 0.0, "bottom")],
                     hierarchy=h, solver_parameters={"pc_type": "mg", "ksp_rtol": 1e-10})
        its.append(n)
    assert its[1] <= its[0] + 2, its
