"""GPU parity of the symmetric interior penalty discretisation on DQ_p hexahedra (FDB_FORM_INTERIOR_PENALTY and
FDB_FORM_DG_BOUNDARY, csrc/dg_facet_hex.cu; the cell term on the Helmholtz kernels with Gauss-Legendre tables)
against the NumPy oracle (tests/_dg_oracle.py) and the generic wrapper path, the engine's refusals, and the solves
that use it.  Parity meshes have their vertices moved in and out of plane.  Tolerance 1e-12 relative in the max
norm."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse.linalg as spla

import _boundary_oracle as bo
import _dg_oracle as do
from firedrake_b200 import op2
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

TOL = 1e-12


def relerr(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(b).max()


def eta_of(p):
    return 3.0 * (p + 1) ** 2


def perturbed(nx=3, ny=2, nz=3, seed=1):
    return bo.perturb(ExtrudedHexMesh(nx, ny, nz, Lx=1.2, Ly=0.9, Lz=1.1, warp=0.05, permute_seed=seed), 0.08, seed)


def values(n, seed):
    return np.random.default_rng(seed).standard_normal(n)


def parallelepipeds(nx=4, ny=2, nz=2):
    """A sheared box whose cells are parallelepipeds in floating point, not only in exact arithmetic: dyadic vertex
    positions and shear, so the four trilinear terms of every cell are exactly zero (fdb_cells_are_affine demands
    exact zeros) and Form picks the per-cell-metric variant."""
    mesh = ExtrudedHexMesh(nx, ny, nz, Lx=1.0, Ly=1.0, Lz=1.0, permute_seed=3)
    S = np.array([[1.0, 0.25, 0.125], [0.0, 1.25, -0.25], [0.125, 0.0, 0.75]])
    mesh.coordinates[:] = mesh.coordinates @ S.T + np.array([0.25, -0.125, 0.5])
    X = mesh.coordinates[mesh.coord_space.full_cell_node_list()]
    for t in (X[:, 6] - X[:, 4] - X[:, 2] + X[:, 0], X[:, 3] - X[:, 2] - X[:, 1] + X[:, 0],
              X[:, 5] - X[:, 4] - X[:, 1] + X[:, 0],
              X[:, 7] - X[:, 6] - X[:, 5] - X[:, 3] + X[:, 4] + X[:, 2] + X[:, 1] - X[:, 0]):
        assert np.all(t == 0.0)
    return mesh


def dq(mesh, p):
    from firedrake_b200.assemble import FunctionSpace
    return FunctionSpace(mesh, p, family="DQ")


# ------------------------------------------------------------------------------------------------- cell term
@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_cell_term_matches_oracle(engine, p):
    """mass(V) and poisson(V) on DQ_p (the one-thread-per-cell kernels at p = 1, 2 included) against the oracle;
    the CG kernel of the same degree runs in the same process before and after and is unchanged."""
    from firedrake_b200.assemble import FunctionSpace, ImplicitMatrixContext, assemble, mass, poisson
    mesh = perturbed(seed=p)
    Vc = FunctionSpace(mesh, p)
    xc = Vc.dat(values(Vc.node_count, 50 + p))
    yc0 = assemble(poisson(Vc), u=xc).data_ro.copy()
    V = dq(mesh, p)
    x = V.dat(values(V.node_count, p))
    el = do.element(p)
    for form, (a, b) in ((mass(V), (0.0, 1.0)), (poisson(V), (1.0, 0.0))):
        A = do.cell_matrix(mesh, V.V, el, a, b)
        assert relerr(assemble(form, u=x).data_ro, A @ x.data_ro) < TOL
        if p <= 3:
            d = ImplicitMatrixContext(form).getDiagonal(V.dat()).data_ro
            assert relerr(d, A.diagonal()) < TOL
    assert relerr(assemble(poisson(Vc), u=xc).data_ro, yc0) < TOL


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_cell_term_affine_variant(engine, monkeypatch, p):
    """On a parallelepiped mesh Form picks the per-cell-metric variant by itself (p = 1, 2: the thread-per-cell
    kernels; 3, 4: the slab kernel), and with the GL tables it matches the oracle and the per-point variant."""
    from firedrake_b200.assemble import Form, assemble
    mesh = parallelepipeds()
    V = dq(mesh, p)
    F = Form(V, 1.3, 0.7)
    assert F.kernel(1).affine
    x = V.dat(values(V.node_count, p))
    ya = assemble(F, u=x).data_ro.copy()
    assert relerr(ya, do.cell_matrix(mesh, V.V, do.element(p), 1.3, 0.7) @ x.data_ro) < TOL
    monkeypatch.setenv("FDB_AFFINE", "0")
    assert not F.kernel(1).affine
    assert relerr(ya, assemble(F, u=x).data_ro) < TOL


# ------------------------------------------------------------------------------------------------ facet terms
@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_facet_actions_and_diagonals_match_oracle(engine, p):
    """The interior-penalty loops and the Nitsche loops separately (atomic, and coloured twice: bit-identical), and
    their diagonals."""
    from firedrake_b200.assemble import InteriorPenalty
    mesh = perturbed(seed=10 + p)
    V = dq(mesh, p)
    el = do.element(p)
    alpha, eta = 1.3, eta_of(p)
    F = InteriorPenalty(V, alpha, 0.0, eta)
    terms = F.facet_terms()
    x = V.dat(values(V.node_count, p))
    Ai = do.interior_matrix(mesh, V.V, el, alpha, eta)
    Ae = do.exterior_matrix(mesh, V.V, el, "on_boundary", 0.0, alpha * eta, alpha, alpha)
    outs = []
    for scatter in ("atomic", "coloured", "coloured"):
        y = V.dat()
        y.zero()
        loops = terms.action_loops(y, x, scatter)
        nint = len(terms.interior)
        for loop in loops[:nint]:
            loop()
        assert relerr(y.data_ro, Ai @ x.data_ro) < TOL, scatter
        for loop in loops[nint:]:
            loop()
        assert relerr(y.data_ro, (Ai + Ae) @ x.data_ro) < TOL, scatter
        outs.append(y.data_ro.copy())
    assert np.array_equal(outs[1], outs[2])
    D = V.dat()
    D.zero()
    terms.diagonal(D)
    assert relerr(D.data_ro, (Ai + Ae).diagonal()) < TOL


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_whole_operator_and_generic_path(engine, p):
    """assemble(F, u=x) against A_oracle @ x, the matrix-free mult and diagonal, and the facet terms of the generic
    wrapper path."""
    from firedrake_b200.assemble import Form, InteriorPenalty, assemble, assemble_interior_penalty_generic
    mesh = perturbed(3, 3, 2, seed=20 + p)
    V = dq(mesh, p)
    el = do.element(p)
    F = InteriorPenalty(V, 0.8, 0.5, eta_of(p), weak_bcs=(1, "top", 3))
    A = do.operator(mesh, V.V, el, 0.8, 0.5, eta_of(p), weak_bcs=(1, "top", 3))
    x = V.dat(values(V.node_count, 30 + p))
    y = assemble(F, u=x).data_ro.copy()
    assert relerr(y, A @ x.data_ro) < TOL
    op = assemble(F, mat_type="matfree")
    ym = V.dat()
    op.mult(x, ym)
    assert relerr(ym.data_ro, A @ x.data_ro) < TOL
    if p <= 3:
        assert relerr(op.getDiagonal(V.dat()).data_ro, A.diagonal()) < TOL
    if p <= 3:
        yg = assemble_interior_penalty_generic(F, x).data_ro
        yc = assemble(Form(V, 0.8, 0.5), u=x).data_ro
        assert relerr(y - yc, yg) < TOL


@pytest.mark.parametrize("p", [1, 3])
def test_native_hexes(engine, p):
    """The op2 level on native hexes: permuted full rows, one entry per interior facet ('+' row, '-' row) and per
    exterior facet; atomic and coloured."""
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
    u = op2.Dat(nodes, values(W.node_count, 3))
    alpha, eta = 0.9, eta_of(p)
    A = (do.interior_matrix(mesh, W, el, alpha, eta)
         + do.exterior_matrix(mesh, W, el, "on_boundary", 0.0, alpha * eta, alpha, alpha))
    iset, eset = op2.Set(len(P)), op2.Set(len(C_))
    im0 = op2.Map(iset, nodes, 2 * nd, np.ascontiguousarray(np.concatenate([full[where[P]], full[where[M]]], 1)))
    im1 = op2.Map(iset, vnodes, 16, np.ascontiguousarray(np.concatenate([cfull[where[P]], cfull[where[M]]], 1)))
    em0 = op2.Map(eset, nodes, nd, np.ascontiguousarray(full[where[C_]]))
    em1 = op2.Map(eset, vnodes, 8, np.ascontiguousarray(cfull[where[C_]]))
    pairs = op2.Dat(op2.DataSet(iset, 2), np.stack([FP, FM], 1).astype(np.uint32), dtype=np.uint32)
    fac = op2.Dat(op2.DataSet(eset, 1), Fe.astype(np.uint32), dtype=np.uint32)
    ki = op2.Kernel("interior_penalty", degree=p, alpha=alpha, beta=eta, integral="interior_facet", element=el)
    ke = op2.Kernel("dg_boundary", degree=p, alpha=alpha, beta=alpha * eta, c_s=alpha, integral="exterior_facet",
                    element=el)
    outs = []
    for scatter in ("atomic", "coloured", "coloured"):
        y = op2.Dat(nodes)
        op2.par_loop(ki, iset, y(op2.INC, im0), X(op2.READ, im1), u(op2.READ, im0), pairs(op2.READ), scatter=scatter)
        op2.par_loop(ke, eset, y(op2.INC, em0), X(op2.READ, em1), u(op2.READ, em0), fac(op2.READ), scatter=scatter)
        assert relerr(y.data_ro, A @ u.data_ro) < TOL, scatter
        outs.append(y.data_ro.copy())
    assert np.array_equal(outs[1], outs[2])
    d = op2.Dat(nodes)
    op2.par_loop(op2.Kernel("interior_penalty", degree=p, alpha=alpha, beta=eta, diagonal=True,
                            integral="interior_facet", element=el), iset, d(op2.INC, im0), X(op2.READ, im1),
                 pairs(op2.READ))
    op2.par_loop(op2.Kernel("dg_boundary", degree=p, alpha=alpha, beta=alpha * eta, c_s=alpha, diagonal=True,
                            integral="exterior_facet", element=el), eset, d(op2.INC, em0), X(op2.READ, em1),
                 fac(op2.READ))
    assert relerr(d.data_ro, A.diagonal()) < TOL


@pytest.mark.parametrize("p", [1, 2, 4])
def test_loads_match_oracle(engine, p):
    """The three DG_BOUNDARY callers' loads: nitsche_load (0, alpha eta, alpha, 0) and dg_flux_load (1, 0, 0, 0),
    with their diagonals through the op2 level."""
    from firedrake_b200.assemble import InteriorPenalty, _boundary_groups, _dg_boundary_kernel, dg_flux_load, \
        nitsche_load
    mesh = perturbed(seed=60 + p)
    V = dq(mesh, p)
    el = do.element(p)
    g = V.dat(values(V.node_count, 7))
    F = InteriorPenalty(V, 1.1, 0.0, eta_of(p), weak_bcs=(2, "bottom"))
    yo = do.nitsche_load(mesh, V.V, el, 1.1, eta_of(p), (2, "bottom"), g.data_ro)
    assert relerr(nitsche_load(F, g).data_ro, yo) < TOL
    for sub in ("on_boundary", 4, "top"):
        assert relerr(dg_flux_load(V, g, sub).data_ro, do.flux_load(mesh, V.V, el, sub, g.data_ro)) < TOL
    for coefs in ((0.0, 1.1 * eta_of(p), 1.1, 0.0), (1.0, 0.0, 0.0, 0.0)):
        d = V.dat()
        for fset, fmap, cmap, facet in _boundary_groups(V, "on_boundary"):
            op2.par_loop(_dg_boundary_kernel(V, *coefs, diagonal=True), fset, d(op2.INC, fmap),
                         V.coordinates(op2.READ, cmap), facet(op2.READ))
        Ao = do.exterior_matrix(mesh, V.V, el, "on_boundary", *coefs)
        assert relerr(d.data_ro, Ao.diagonal()) < TOL


# --------------------------------------------------------------------------------------------------- refusals
def test_refusals(engine):
    from firedrake_b200 import _lib
    from firedrake_b200.assemble import FunctionSpace, _boundary_groups, _dg_interior_groups
    mesh = ExtrudedHexMesh(2, 2, 2)
    V = FunctionSpace(mesh, 2, family="DQ")
    el = V.element
    fset, fmap, cmap, pairs = _dg_interior_groups(V)[0]
    eset, emap, ecmap, facet = _boundary_groups(V, "on_boundary")[0]

    def refused(msg, form="interior_penalty", maps=(fmap, cmap), **kw):
        kw.setdefault("integral", "interior_facet" if form == "interior_penalty" else "exterior_facet")
        kw.setdefault("degree", 2)
        kw.setdefault("element", el if kw["degree"] == 2 else None)
        gk = op2.GlobalKernel(op2.Kernel(form, **kw), list(maps), extruded=True)
        with pytest.raises(_lib.EngineError, match=msg):
            gk.compile()

    for form, maps in (("interior_penalty", (fmap, cmap)), ("dg_boundary", (emap, ecmap))):
        refused(f"{form} has no rank-2 form: there is no assembled DG matrix", form, maps, rank=2)
        refused(f"{form} action: degree 5 outside 1..4", form, maps, degree=5)
        refused(f"{form} diagonal: degree 5 outside 1..4", form, maps, degree=5, diagonal=True)
        refused(f"{form} action takes scalar spaces only", form, maps, cdim=3)
        refused(f"{form} has no affine-cell variant", form, maps, affine=True)
        from firedrake_b200.fiat_lite import interval_element
        refused(f"{form} needs nq == degree\\+1", form, maps, element=interval_element(2, 4, "gl"))
    refused("interior_penalty has interior-facet integrals only", integral="exterior_facet")
    refused("dg_boundary has exterior-facet integrals only .*interior facets are not supported", "dg_boundary",
            (emap, ecmap), integral="interior_facet")
    refused("boundary_mass has exterior-facet integrals only .*interior facets are not supported", "boundary_mass",
            (emap, ecmap), integral="interior_facet", element=None)
    # extruded cells without layer offsets
    d = _lib.KernelDesc()
    d.form, d.rank, d.cell, d.integral = _lib.FORM_INTERIOR_PENALTY, 1, _lib.CELL_HEX_EXTRUDED, \
        _lib.INTEGRAL_INTERIOR_FACET
    d.degree, d.nq, d.cdim = 2, 3, 1
    for q in range(3):
        for a in range(3):
            d.B[q * 3 + a], d.D[q * 3 + a] = el.B[q, a], el.D[q, a]
    h = C.c_void_p()
    assert engine.fdb_kernel_create(C.byref(d), C.byref(h)) != 0
    assert "interior_penalty on extruded cells needs the layer offsets" in engine.fdb_last_error().decode()
    # host location and wrong argument counts, at the call
    u, y = V.dat(np.ones(V.node_count)), V.dat()
    k = op2.Kernel("interior_penalty", degree=2, beta=27.0, integral="interior_facet", element=el)
    with pytest.raises(_lib.EngineError, match="interior_penalty takes device-resident Dats only"):
        op2.par_loop(k, fset, y(op2.INC, fmap), V.coordinates(op2.READ, cmap), u(op2.READ, fmap), pairs(op2.READ),
                     location="host")
    gk = op2.GlobalKernel(k, [fmap, cmap], extruded=True)
    with pytest.raises(_lib.EngineError, match="interior_penalty action expects 4 device args"):
        gk(0, fset.total_size, fset.layers_array.ravel(), None, [y.device_ptr, V.coordinates.device_ptr,
                                                                  u.device_ptr], None, None,
           [fmap.device_ptr, cmap.device_ptr], None, _lib.LOC_DEVICE, False, False)


def test_dq4_diagonal_is_refused_up_front(engine):
    """The cell term's diagonal kernel covers degrees 1..3: on DQ4 getDiagonal and pc_type 'jacobi' refuse before any
    loop runs, and pc_type 'none' solves."""
    from firedrake_b200.assemble import InteriorPenalty, assemble, solve
    V = dq(perturbed(2, 2, 2, seed=3), 4)
    F = InteriorPenalty(V, 1.0, 1.0, eta_of(4))
    with pytest.raises(NotImplementedError, match="diagonal of the DQ4 cell term"):
        assemble(F, mat_type="matfree").getDiagonal(V.dat())
    with pytest.raises(NotImplementedError, match="use pc_type 'none' on DQ4"):
        solve(F, V.dat(np.ones(V.node_count)), V.dat(), solver_parameters={"pc_type": "jacobi"})
    A = do.operator(V.mesh, V.V, V.element, 1.0, 1.0, eta_of(4))
    b = V.dat(values(V.node_count, 9))
    u = V.dat()
    its, _ = solve(F, b, u, solver_parameters={"pc_type": "none", "ksp_rtol": 1e-12, "ksp_max_it": 5000})
    assert relerr(u.data_ro, spla.spsolve(A.tocsc(), b.data_ro.copy())) < 1e-8, its


# ------------------------------------------------------------------------------------------------------ solves
def _manufactured(n, p, pc="jacobi", weak="on_boundary", flux=()):
    """-div(alpha grad u) + beta u = f on the unit cube, u = sin(x + 0.5) cos(0.7 y) exp(0.3 z): Dirichlet weakly on
    ``weak``, fluxes alpha du/dn on the ``flux`` sides.  Returns (V, u, exact nodal values, iterations, F, L)."""
    from firedrake_b200.assemble import InteriorPenalty, assemble, dg_flux_load, mass, nitsche_load, solve
    alpha, beta = 1.0, 0.5
    mesh = ExtrudedHexMesh(n, n, n)
    V = dq(mesh, p)
    x, y, z = V.V.dof_coordinates().T
    ue = np.sin(x + 0.5) * np.cos(0.7 * y) * np.exp(0.3 * z)
    grads = {1: -np.cos(x + 0.5) * np.cos(0.7 * y) * np.exp(0.3 * z),
             2: np.cos(x + 0.5) * np.cos(0.7 * y) * np.exp(0.3 * z),
             3: 0.7 * np.sin(x + 0.5) * np.sin(0.7 * y) * np.exp(0.3 * z),
             4: -0.7 * np.sin(x + 0.5) * np.sin(0.7 * y) * np.exp(0.3 * z),
             "bottom": -0.3 * ue, "top": 0.3 * ue}
    f = ue * (alpha * (1.0 + 0.49 - 0.09) + beta)
    F = InteriorPenalty(V, alpha, beta, eta_of(p), weak_bcs=weak)
    L = assemble(mass(V), u=V.dat(f))
    L.axpy(1.0, nitsche_load(F, V.dat(ue)))
    for s in flux:
        L.axpy(1.0, dg_flux_load(V, V.dat(alpha * grads[s]), s))
    u = V.dat()
    its, _ = solve(F, L, u, solver_parameters={"pc_type": pc, "ksp_rtol": 1e-13, "ksp_max_it": 5000})
    return V, u, ue, its, F, L


def _l2(V, e):
    from firedrake_b200.assemble import assemble, mass
    ed = V.dat(e)
    return float(np.sqrt(np.dot(e, assemble(mass(V), u=ed).data_ro)))


@pytest.mark.parametrize("pc", ["none", "jacobi"])
def test_nitsche_solve_matches_scipy(engine, pc):
    V, u, ue, its, F, L = _manufactured(3, 2, pc)
    A = do.operator(V.mesh, V.V, V.element, 1.0, 0.5, eta_of(2))
    x = spla.spsolve(A.tocsc(), L.data_ro.copy())
    assert relerr(u.data_ro, x) < 1e-8, its


def test_jacobi_takes_fewer_iterations(engine):
    its = {pc: _manufactured(4, 2, pc)[3] for pc in ("none", "jacobi")}
    assert its["jacobi"] < its["none"], its


def test_affine_polynomial_is_reproduced(engine):
    """A total-degree-p polynomial on a sheared mesh, Dirichlet data imposed weakly everywhere: the discrete
    solution is the polynomial."""
    from firedrake_b200.assemble import InteriorPenalty, assemble, mass, nitsche_load, solve
    p = 2
    mesh = parallelepipeds(4, 4, 2)
    V = dq(mesh, p)
    x, y, z = V.V.dof_coordinates().T
    ue = 0.3 + x * y - 0.5 * z ** 2 + 0.2 * y ** 2
    f = (1.0 - 0.4) + 0.7 * ue                    # -lap(ue) = 1 - 0.4
    F = InteriorPenalty(V, 1.0, 0.7, eta_of(p))
    assert F.kernel(1).affine                       # the affine cell variant, in a solve
    L = assemble(mass(V), u=V.dat(f))
    L.axpy(1.0, nitsche_load(F, V.dat(ue)))
    u = V.dat()
    solve(F, L, u, solver_parameters={"pc_type": "jacobi", "ksp_rtol": 1e-14, "ksp_max_it": 5000})
    assert relerr(u.data_ro, ue) < 1e-9


@pytest.mark.parametrize("p", [1, 2, 3])
def test_convergence_rate(engine, p):
    errs = []
    for n in (4, 8):
        V, u, ue, its, F, L = _manufactured(n, p)
        errs.append(_l2(V, u.data_ro - ue))
    rate = np.log2(errs[0] / errs[1])
    assert rate > p + 0.8, (p, errs, rate)


def test_mixed_nitsche_and_flux(engine):
    """Dirichlet weakly on sides 1, 3 and "bottom", fluxes on the other three: against scipy and close to u."""
    V, u, ue, its, F, L = _manufactured(3, 2, "jacobi", weak=(1, 3, "bottom"), flux=(2, 4, "top"))
    A = do.operator(V.mesh, V.V, V.element, 1.0, 0.5, eta_of(2), weak_bcs=(1, 3, "bottom"))
    x = spla.spsolve(A.tocsc(), L.data_ro.copy())
    assert relerr(u.data_ro, x) < 1e-8, its
    assert _l2(V, u.data_ro - ue) < 1e-2
