"""GPU tests of Stokes flow on Taylor-Hood hexahedra (FDB_FORM_STOKES, the EL_STOKES mode of
csrc/elasticity_hex.cu): the fused saddle-point action against the NumPy oracle (tests/_stokes_oracle.py)
and the generic wrapper path, the divergence structure, the matrix-free operator with velocity conditions,
the refusals, and solves (lid-driven cavity against scipy, rates of a manufactured solution, multigrid
iteration counts).  Tolerance 1e-12 relative in the max norm for the actions."""
import numpy as np
import pytest

import _stokes_oracle as so
from firedrake_b200 import _lib, op2
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

TOL = 1e-12
MU = 1.3
ALL_FACES = (1, 2, 3, 4, "bottom", "top")


def relerr(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def setup(p, native, mesh=None):
    """op2 objects of a warped, permuted mesh for velocity CG_p and pressure CG_(p-1): extruded or native
    hexes (cells in a random order), and the oracle's view of the maps."""
    mesh = mesh or ExtrudedHexMesh(4, 3, 5, warp=0.05, permute_seed=1)
    V, Q = mesh.function_space(p), mesh.function_space(p - 1)
    nodes, qnodes = op2.Set(V.node_count), op2.Set(Q.node_count)
    vnodes = op2.Set(mesh.coord_space.node_count)
    if native:
        perm = np.random.default_rng(0).permutation(mesh.num_cells)
        full = V.full_cell_node_list()[perm]
        qfull = Q.full_cell_node_list()[perm]
        cfull = mesh.coord_space.full_cell_node_list()[perm]
        cells = op2.Set(len(perm))
        m0 = op2.Map(cells, nodes, V.arity, full)
        m1 = op2.Map(cells, vnodes, 8, cfull)
        m2 = op2.Map(cells, qnodes, Q.arity, qfull)
        geo = (np.ascontiguousarray(full), np.zeros(V.arity, dtype=np.int32), np.ascontiguousarray(cfull),
               np.zeros(8, dtype=np.int32), 1)
        geo2 = (np.ascontiguousarray(qfull), np.zeros(Q.arity, dtype=np.int32))
    else:
        cells = op2.ExtrudedSet(op2.Set(mesh.num_base_cells), mesh.layers)
        m0 = op2.Map(cells, nodes, V.arity, V.cell_node_map, offset=V.offset)
        m1 = op2.Map(cells, vnodes, 8, mesh.coord_map, offset=mesh.coord_offset)
        m2 = op2.Map(cells, qnodes, Q.arity, Q.cell_node_map, offset=Q.offset)
        geo = (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
        geo2 = (Q.cell_node_map, Q.offset)
    X = op2.Dat(op2.DataSet(vnodes, 3), mesh.coordinates)
    return mesh, V, Q, cells, nodes, qnodes, m0, m1, m2, X, geo, geo2


def _loop(k, cells, yu, yp, u, p, m0, m1, m2, X, scatter="atomic"):
    op2.par_loop(k, cells, yu(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), yp(op2.INC, m2),
                 p(op2.READ, m2), scatter=scatter)


@pytest.mark.parametrize("p", [2, 3, 4])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
@pytest.mark.parametrize("beta", [0.0, 0.7])
def test_stokes_action_matches_oracle(engine, p, native, beta):
    """Atomic and coloured scatter, both blocks; coloured is bit-identical across calls."""
    mesh, V, Q, cells, nodes, qnodes, m0, m1, m2, X, geo, geo2 = setup(p, native)
    rng = np.random.default_rng(p)
    u = op2.Dat(op2.DataSet(nodes, 3), rng.standard_normal((V.node_count, 3)))
    pr = op2.Dat(qnodes, rng.standard_normal(Q.node_count))
    wu, wp = so.action(interval_element(p), mesh.coordinates, u.data_ro.ravel().copy(), pr.data_ro.copy(),
                       geo, geo2, MU, beta)
    k = op2.Kernel("stokes", degree=p, mu=MU, beta=beta)
    yu, yp = op2.Dat(op2.DataSet(nodes, 3)), op2.Dat(qnodes)
    _loop(k, cells, yu, yp, u, pr, m0, m1, m2, X)
    assert relerr(yu.data_ro.ravel(), wu) < TOL
    assert relerr(yp.data_ro, wp) < TOL
    outs = []
    for _ in range(2):
        yu.zero()
        yp.zero()
        _loop(k, cells, yu, yp, u, pr, m0, m1, m2, X, scatter="coloured")
        outs.append((yu.data_ro.copy(), yp.data_ro.copy()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    assert relerr(outs[0][0].ravel(), wu) < TOL
    assert relerr(outs[0][1], wp) < TOL


def _spaces(p, mesh=None):
    from firedrake_b200.assemble import FunctionSpace
    mesh = mesh or ExtrudedHexMesh(4, 3, 5, warp=0.05, permute_seed=2)
    return FunctionSpace(mesh, p, 3), FunctionSpace(mesh, p - 1)


@pytest.mark.parametrize("p", [2, 3, 4])
def test_stokes_action_matches_generic_path(engine, p):
    from firedrake_b200.assemble import Stokes, assemble, assemble_stokes_generic
    V, Q = _spaces(p)
    F = Stokes(V, Q, MU, 0.4)
    rng = np.random.default_rng(3)
    up = F.dat(rng.standard_normal((V.node_count, 3)), rng.standard_normal(Q.node_count))
    y = [d.data_ro.copy() for d in assemble(F, u=up)]
    yg = [d.data_ro.copy() for d in assemble_stokes_generic(F, up)]
    assert relerr(y[0], yg[0]) < TOL
    assert relerr(y[1], yg[1]) < TOL


@pytest.mark.parametrize("p", [2, 3, 4])
def test_divergence_structure(engine, p):
    """On a warped mesh: B^T 1 vanishes on the velocity rows off the boundary, and the pressure rows vanish
    for the linear divergence-free field (x, y, -2z) (the div terms are integrated exactly)."""
    from firedrake_b200.assemble import Stokes, assemble
    V, Q = _spaces(p, ExtrudedHexMesh(3, 3, 4, warp=0.08, permute_seed=1))
    F = Stokes(V, Q, MU)
    yu, _ = assemble(F, u=F.dat(None, np.ones(Q.node_count)))
    bnd = np.unique(np.concatenate([V.boundary_nodes(s) for s in ALL_FACES]))
    inner = np.setdiff1d(np.arange(V.node_count), bnd)
    ref = np.abs(yu.data_ro).max()
    assert ref > 0.0
    assert np.abs(yu.data_ro[inner]).max() < 1e-12 * ref
    Xn = V.V.dof_coordinates()
    lin = np.stack([Xn[:, 0], Xn[:, 1], -2.0 * Xn[:, 2]], axis=1)
    _, yp = assemble(F, u=F.dat(lin, None))
    _, yp2 = assemble(F, u=F.dat(np.stack([Xn[:, 0], Xn[:, 1], Xn[:, 2]], axis=1), None))
    assert np.abs(yp.data_ro).max() < 1e-12 * np.abs(yp2.data_ro).max()


def test_matfree_mult_with_velocity_bcs_matches_oracle(engine):
    from firedrake_b200.assemble import DirichletBC, Stokes, assemble
    p = 2
    mesh = ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=3)
    V, Q = _spaces(p, mesh)
    F = Stokes(V, Q, MU, 0.3)
    bcs = [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, 0.0, 2)]
    A = assemble(F, bcs=bcs, mat_type="matfree")
    rng = np.random.default_rng(5)
    x = F.dat(rng.standard_normal((V.node_count, 3)), rng.standard_normal(Q.node_count))
    y = F.dat()
    A.mult(x, y)
    geo = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    K = so.global_matrix(interval_element(p), mesh.coordinates, geo, (Q.V.cell_node_map, Q.V.offset),
                         V.node_count, Q.node_count, MU, 0.3)
    bn = np.unique(np.concatenate([bc.nodes for bc in bcs]))
    Kc = so.constrained(K, so.velocity_dofs(bn))
    want = Kc @ np.concatenate([x[0].data_ro.ravel(), x[1].data_ro])
    got = np.concatenate([y[0].data_ro.ravel(), y[1].data_ro])
    assert relerr(got, want) < TOL
    y2 = F.dat()
    A.multTranspose(x, y2)
    assert relerr(np.concatenate([y2[0].data_ro.ravel(), y2[1].data_ro]), want) < TOL


def _desc(p, **kw):
    el = interval_element(p)
    d = _lib.KernelDesc()
    d.form, d.rank, d.cell, d.integral = _lib.FORM_STOKES, 1, _lib.CELL_HEX, _lib.INTEGRAL_CELL
    d.degree, d.nq, d.cdim, d.scatter = p, p + 1, 3, _lib.SCATTER_ATOMIC
    for q in range(el.nq):
        d.wq[q], d.xq[q] = el.wq[q], el.xq[q]
        for a in range(p + 1):
            d.B[q * (p + 1) + a], d.D[q * (p + 1) + a] = el.B[q, a], el.D[q, a]
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _space2(p, **kw):
    elq = interval_element(p - 1, p + 1)
    s2 = _lib.Space2Desc()
    s2.degree = p - 1
    for q in range(p + 1):
        for a in range(p):
            s2.B[q * p + a] = elq.B[q, a]
    for k, v in kw.items():
        setattr(s2, k, v)
    return s2


@pytest.mark.parametrize("kw,kw2,msg", [
    (dict(cdim=1), {}, "value size 3 only"),
    (dict(degree=1, nq=2), {}, "degree 1 outside 2..4"),
    (dict(degree=5, nq=6), {}, "degree 5 outside 2..4"),
    (dict(rank=2), {}, "mixed form, a rank-1 action only"),
    (dict(diagonal=1), {}, "mixed form, a rank-1 action only"),
    (dict(affine_cells=1), {}, "no affine-cell variant"),
    (dict(nq=4), {}, "nq == degree\\+1"),
    (dict(cell=_lib.CELL_HEX_EXTRUDED), {}, "needs the layer offsets of the second map"),
    ({}, dict(degree=2), "needs a second space of degree 1, got 2"),
])
def test_create_refusals(engine, kw, kw2, msg):
    import ctypes as C
    d = _desc(kw.get("degree", 2), **kw)
    keep = []
    if kw.get("cell") == _lib.CELL_HEX_EXTRUDED:
        keep = [np.zeros(27, dtype=np.int32), np.zeros(8, dtype=np.int32)]
        d.offset0 = keep[0].ctypes.data_as(C.POINTER(C.c_int32))
        d.offset1 = keep[1].ctypes.data_as(C.POINTER(C.c_int32))
    s2 = _space2(max(2, kw.get("degree", 2)), **kw2)
    h = C.c_void_p()
    with pytest.raises(_lib.EngineError, match=msg):
        _lib.check(engine.fdb_kernel_create_mixed(C.byref(d), C.byref(s2), C.byref(h)), "fdb_kernel_create_mixed")


def test_create_needs_the_matching_entry_point(engine):
    """A form on two spaces is created with its second space's descriptor, a form on one space without."""
    import ctypes as C
    h = C.c_void_p()
    d = _desc(2)
    with pytest.raises(_lib.EngineError, match="form on two spaces: create it with fdb_kernel_create_mixed"):
        _lib.check(engine.fdb_kernel_create(C.byref(d), C.byref(h)), "fdb_kernel_create")
    d.form = _lib.FORM_ELASTICITY
    s2 = _space2(2)
    with pytest.raises(_lib.EngineError, match="not a form on two spaces"):
        _lib.check(engine.fdb_kernel_create_mixed(C.byref(d), C.byref(s2), C.byref(h)), "fdb_kernel_create_mixed")


def test_call_refusals(engine):
    """Wrong argument or map counts and host-resident Dats are refused with the expected arguments named;
    op2 refuses a pressure Dat with more than one value per node."""
    mesh, V, Q, cells, nodes, qnodes, m0, m1, m2, X, _, _ = setup(2, False)
    k = op2.Kernel("stokes", degree=2, mu=MU)
    vs = op2.DataSet(nodes, 3)
    yu, u, yp, pr = op2.Dat(vs), op2.Dat(vs), op2.Dat(qnodes), op2.Dat(qnodes)
    gk = op2.GlobalKernel(k, [m0, m1, m2], extruded=True)
    with pytest.raises(_lib.EngineError, match=r"expects 5 device args \(y, coords, x, y_p, p\) and 3 maps, got 3/2"):
        gk(0, mesh.num_base_cells, cells.layers_array.ravel(), None, [yu.device_ptr, X.device_ptr, u.device_ptr],
           None, None, [m0.device_ptr, m1.device_ptr], None, _lib.LOC_DEVICE, False, False)
    loop = op2.Parloop(gk, cells, [yu(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), yp(op2.INC, m2),
                                   pr(op2.READ, m2)], location="host")
    with pytest.raises(_lib.EngineError, match="expects 5 device args"):
        loop()
    with pytest.raises(ValueError, match="pressure Dats have 1 value per node"):
        p3 = op2.Dat(op2.DataSet(qnodes, 3))
        op2.par_loop(k, cells, yu(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), p3(op2.INC, m2),
                     pr(op2.READ, m2))


def _cavity(n, p=2, mu=1.0):
    from firedrake_b200.assemble import DirichletBC, Stokes
    from firedrake_b200.assemble import FunctionSpace
    mesh = ExtrudedHexMesh(n, n, n)
    V, Q = FunctionSpace(mesh, p, 3), FunctionSpace(mesh, p - 1)
    F = Stokes(V, Q, mu)
    lid = np.zeros((V.node_count, 3))
    lid[:, 0] = 1.0
    bcs = [DirichletBC(V, 0.0, (1, 2, 3, 4, "bottom")), DirichletBC(V, V.dat(lid), "top")]
    return mesh, V, Q, F, bcs


def _fieldsplit(pc0):
    return {"ksp_type": "gmres", "ksp_rtol": 1e-12, "pc_type": "fieldsplit", "pc_fieldsplit_type": "schur",
            "pc_fieldsplit_schur_fact_type": "diag", "fieldsplit_0_pc_type": pc0,
            "fieldsplit_1_pc_type": "jacobi", "ksp_max_it": 2000}


def test_lid_driven_cavity_matches_scipy(engine):
    """Q2-Q1 on 8^3, fieldsplit + mg, constant-pressure nullspace: the velocity within 1e-8 of scipy's
    spsolve on the oracle system (one pressure pinned, then the mean removed), the pressure within 1e-7
    modulo a constant."""
    import scipy.sparse as sps
    import scipy.sparse.linalg as spla
    from firedrake_b200.assemble import solve
    from firedrake_b200.mg import MeshHierarchy
    n = 8
    mesh, V, Q, F, bcs = _cavity(n)
    hier = MeshHierarchy(2, 2, 2, 2)
    up = F.dat()
    its, _ = solve(F, F.dat(), up, bcs, _fieldsplit("mg"), hierarchy=hier, nullspace="constant")
    assert its < 1000
    geo = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    K = so.global_matrix(interval_element(2), mesh.coordinates, geo, (Q.V.cell_node_map, Q.V.offset),
                         V.node_count, Q.node_count, 1.0)
    g = np.zeros((V.node_count, 3))
    g[bcs[1].nodes, 0] = 1.0
    bn = np.unique(np.concatenate([bc.nodes for bc in bcs]))
    bd = so.velocity_dofs(bn)
    nv = 3 * V.node_count
    gfull = np.concatenate([g.ravel(), np.zeros(Q.node_count)])
    rhs = -(K @ gfull)
    rhs[bd] = 0.0
    pin = nv
    Kc = so.constrained(K, np.concatenate([bd, [pin]]))
    rhs[pin] = 0.0
    x = spla.spsolve(sps.csc_matrix(Kc), rhs) + gfull
    u_ref, p_ref = x[:nv], x[nv:] - x[nv:].mean()
    u_got = up[0].data_ro.ravel()
    p_got = up[1].data_ro - up[1].data_ro.mean()
    assert np.abs(u_got - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    assert np.abs(p_got - p_ref).max() < 1e-7 * np.abs(p_ref).max()
    assert abs(up[1].data_ro.mean()) < 1e-12 * np.abs(p_ref).max()


def test_manufactured_solution_rates(engine):
    """u = curl psi and a zero-mean p on the unit cube, Q2-Q1: L2 rates against the interpolants, velocity
    >= 2.8 and pressure >= 1.8 from 4^3 to 8^3."""
    import sympy as sp
    from firedrake_b200.assemble import DirichletBC, Form, FunctionSpace, Stokes, assemble, solve
    x, y, z = sp.symbols("x y z")
    psi = (sp.sin(sp.pi * x) * sp.sin(sp.pi * y) * sp.sin(sp.pi * z)) ** 2
    psi_v = sp.Matrix([0, psi, psi * sp.cos(x)])
    curl = lambda A: sp.Matrix([sp.diff(A[2], y) - sp.diff(A[1], z), sp.diff(A[0], z) - sp.diff(A[2], x),
                                sp.diff(A[1], x) - sp.diff(A[0], y)])
    ue = curl(psi_v)
    pe = sp.cos(sp.pi * x) * sp.cos(sp.pi * y) * sp.cos(sp.pi * z)
    mu, beta = 1.0, 0.5
    f = [-mu * sum(sp.diff(ue[i], v, 2) for v in (x, y, z)) + sp.diff(pe, (x, y, z)[i]) + beta * ue[i]
         for i in range(3)]
    fu = [sp.lambdify((x, y, z), e, "numpy") for e in ue]
    ff = [sp.lambdify((x, y, z), e, "numpy") for e in f]
    fp = sp.lambdify((x, y, z), pe, "numpy")
    errs = []
    for n in (4, 8):
        mesh = ExtrudedHexMesh(n, n, n)
        V, Q = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1)
        Vs = FunctionSpace(mesh, 2)
        Xv, Xq = V.V.dof_coordinates(), Q.V.dof_coordinates()
        ev = lambda fs, X: np.stack([np.broadcast_to(g(X[:, 0], X[:, 1], X[:, 2]), (len(X),)) for g in fs], axis=1)
        uI, pI = ev(fu, Xv), fp(Xq[:, 0], Xq[:, 1], Xq[:, 2])
        fI = ev(ff, Xv)
        F = Stokes(V, Q, mu, beta)
        L = F.dat()
        for c in range(3):
            L[0].data[:, c] = assemble(Form(Vs, 0.0, 1.0), u=Vs.dat(fI[:, c].copy())).data_ro
        bcs = [DirichletBC(V, V.dat(uI.copy()), ALL_FACES)]
        up = F.dat()
        solve(F, L, up, bcs, {**_fieldsplit("jacobi"), "ksp_rtol": 1e-11}, nullspace="constant")
        eu = up[0].data_ro - uI
        ep = up[1].data_ro - (pI - pI.mean())
        ep -= ep.mean()
        Mq = assemble(Form(Q, 0.0, 1.0), u=Q.dat(ep.copy())).data_ro
        Mu = sum(assemble(Form(Vs, 0.0, 1.0), u=Vs.dat(eu[:, c].copy())).data_ro @ eu[:, c] for c in range(3))
        errs.append((np.sqrt(Mu), np.sqrt(Mq @ ep)))
    ru = np.log2(errs[0][0] / errs[1][0])
    rp = np.log2(errs[0][1] / errs[1][1])
    assert ru >= 2.8, errs
    assert rp >= 1.8, errs


def test_multigrid_iteration_counts(engine):
    """Fieldsplit with a velocity V-cycle: the iterations at 16^3 are at most 1.25 times those at 8^3 and
    fewer than with the velocity Jacobi preconditioner at 16^3."""
    from firedrake_b200.assemble import solve
    from firedrake_b200.mg import MeshHierarchy
    its = {}
    for n, pc0 in ((8, "mg"), (16, "mg"), (16, "jacobi")):
        _, V, Q, F, bcs = _cavity(n)
        hier = MeshHierarchy(2, 2, 2, {8: 2, 16: 3}[n]) if pc0 == "mg" else None
        up = F.dat()
        sp_ = {**_fieldsplit(pc0), "ksp_rtol": 1e-8}
        its[(n, pc0)], _ = solve(F, F.dat(), up, bcs, sp_, hierarchy=hier, nullspace="constant")
    assert its[(16, "mg")] <= 1.25 * its[(8, "mg")], its
    assert its[(16, "mg")] < its[(16, "jacobi")], its


def test_solver_refusals(engine):
    from firedrake_b200.assemble import Stokes, assemble, solve
    _, V, Q, F, bcs = _cavity(2)
    up = F.dat()
    with pytest.raises(ValueError, match="indefinite"):
        solve(F, F.dat(), up, bcs, {"ksp_type": "cg"})
    with pytest.raises(NotImplementedError, match="matfree"):
        assemble(F)
    with pytest.raises(NotImplementedError, match="matfree"):
        assemble(F, mat_type="is")
    with pytest.raises(NotImplementedError, match="'schur' only"):
        solve(F, F.dat(), up, bcs, {"pc_type": "fieldsplit", "pc_fieldsplit_type": "additive"})
    with pytest.raises(NotImplementedError, match="'diag' only"):
        solve(F, F.dat(), up, bcs, {"pc_type": "fieldsplit", "pc_fieldsplit_type": "schur",
                                    "pc_fieldsplit_schur_fact_type": "full"})
    with pytest.raises(NotImplementedError, match="nullspace"):
        solve(F, F.dat(), up, bcs, nullspace="rigid")
