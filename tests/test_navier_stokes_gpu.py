"""GPU tests of steady Navier-Stokes on Taylor-Hood hexahedra (FDB_FORM_NAVIER_STOKES[_JACOBIAN], the
EL_NS_RESIDUAL / EL_NS_JACOBIAN modes of csrc/elasticity_hex.cu): the residual and the Jacobian action against
the NumPy oracle (tests/_navier_stokes_oracle.py), the generic wrapper path and the Stokes kernel, the Taylor
ratio of the device kernels, the matrix-free operator with velocity conditions, the refusals, and Newton solves
(lid-driven cavity against scipy, rates of a manufactured solution, multigrid iteration counts).  Tolerance
1e-12 relative in the max norm for the actions."""
import numpy as np
import pytest

import _navier_stokes_oracle as nso
import _stokes_oracle as so
import test_stokes_gpu as tg
from firedrake_b200 import _lib, op2
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

TOL = 1e-12
NU = 0.6
ALL_FACES = (1, 2, 3, 4, "bottom", "top")


def relerr(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def _loop(k, cells, yu, yp, x, q, m0, m1, m2, X, u=None, scatter="atomic"):
    extra = [u(op2.READ, m0)] if u is not None else []
    op2.par_loop(k, cells, yu(op2.INC, m0), X(op2.READ, m1), x(op2.READ, m0), yp(op2.INC, m2), q(op2.READ, m2),
                 *extra, scatter=scatter)


@pytest.mark.parametrize("p", [2, 3, 4])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
@pytest.mark.parametrize("beta", [0.0, 0.7])
@pytest.mark.parametrize("jac", [False, True], ids=["residual", "jacobian"])
def test_action_matches_oracle(engine, p, native, beta, jac):
    """Atomic and coloured scatter, both blocks; coloured is bit-identical across calls."""
    mesh, V, Q, cells, nodes, qnodes, m0, m1, m2, X, geo, geo2 = tg.setup(p, native)
    rng = np.random.default_rng(p)
    vs = op2.DataSet(nodes, 3)
    x = op2.Dat(vs, rng.standard_normal((V.node_count, 3)))
    q = op2.Dat(qnodes, rng.standard_normal(Q.node_count))
    u = op2.Dat(vs, rng.standard_normal((V.node_count, 3))) if jac else None
    el = interval_element(p)
    if jac:
        wu, wp = nso.jacobian_action(el, mesh.coordinates, u.data_ro.ravel().copy(), x.data_ro.ravel().copy(),
                                     q.data_ro.copy(), geo, geo2, NU, beta)
    else:
        wu, wp = nso.residual(el, mesh.coordinates, x.data_ro.ravel().copy(), q.data_ro.copy(), geo, geo2, NU, beta)
    k = op2.Kernel("navier_stokes_jacobian" if jac else "navier_stokes", degree=p, mu=NU, beta=beta)
    yu, yp = op2.Dat(vs), op2.Dat(qnodes)
    _loop(k, cells, yu, yp, x, q, m0, m1, m2, X, u)
    assert relerr(yu.data_ro.ravel(), wu) < TOL
    assert relerr(yp.data_ro, wp) < TOL
    outs = []
    for _ in range(2):
        yu.zero()
        yp.zero()
        _loop(k, cells, yu, yp, x, q, m0, m1, m2, X, u, scatter="coloured")
        outs.append((yu.data_ro.copy(), yp.data_ro.copy()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    assert relerr(outs[0][0].ravel(), wu) < TOL
    assert relerr(outs[0][1], wp) < TOL


def _form(p, mesh=None, nu=NU, beta=0.4):
    from firedrake_b200.assemble import NavierStokes
    V, Q = tg._spaces(p, mesh)
    return NavierStokes(V, Q, nu, beta)


def _random(F, seed):
    rng = np.random.default_rng(seed)
    return F.dat(rng.standard_normal((F.V.node_count, 3)), rng.standard_normal(F.Q.node_count))


def _flat(y):
    return np.concatenate([d.data_ro.ravel() for d in y])


@pytest.mark.parametrize("p", [2, 3, 4])
def test_matches_generic_path(engine, p):
    from firedrake_b200.assemble import assemble, assemble_navier_stokes_generic
    F = _form(p)
    up, wr = _random(F, 3), _random(F, 4)
    assert relerr(_flat(assemble(F, u=up)), _flat(assemble_navier_stokes_generic(F, up))) < TOL
    J = F.jacobian(up)
    assert relerr(_flat(assemble(J, u=wr)), _flat(assemble_navier_stokes_generic(F, up, wr))) < TOL


@pytest.mark.parametrize("p", [2, 3, 4])
def test_against_stokes(engine, p):
    """J(0) is the Stokes action with mu = nu, and R(0, p) is the Stokes action on (0, p)."""
    from firedrake_b200.assemble import Stokes, assemble
    F = _form(p)
    S = Stokes(F.V, F.Q, F.nu, F.beta)
    wr = _random(F, 5)
    zero = F.dat()
    assert relerr(_flat(assemble(F.jacobian(zero), u=wr)), _flat(assemble(S, u=wr))) < TOL
    z = F.dat(None, wr[1].data_ro.copy())
    assert relerr(_flat(assemble(F, u=z)), _flat(assemble(S, u=z))) < TOL


@pytest.mark.parametrize("p", [2, 3, 4])
def test_taylor_ratio(engine, p):
    """max|R(u + h w) - R(u) - h J w| falls by 4 when h is halved."""
    from firedrake_b200.assemble import assemble
    F = _form(p)
    up, wr = _random(F, 6), _random(F, 7)
    R0 = _flat(assemble(F, u=up))
    Jw = _flat(assemble(F.jacobian(up), u=wr))
    rem = []
    for h in (0.1, 0.05):
        uh = F.dat(up[0].data_ro + h * wr[0].data_ro, up[1].data_ro + h * wr[1].data_ro)
        rem.append(np.abs(_flat(assemble(F, u=uh)) - R0 - h * Jw).max())
    assert 3.5 <= rem[0] / rem[1] <= 4.5, rem


def test_matfree_mult_with_velocity_bcs_matches_oracle(engine):
    from firedrake_b200.assemble import DirichletBC, assemble
    p = 2
    mesh = ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=3)
    F = _form(p, mesh, beta=0.3)
    V, Q = F.V, F.Q
    up = _random(F, 8)
    bcs = [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, 0.0, 2)]
    A = assemble(F.jacobian(up), bcs=bcs, mat_type="matfree")
    x, y = _random(F, 9), F.dat()
    A.mult(x, y)
    geo = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    K = nso.jacobian_matrix(interval_element(p), mesh.coordinates, up[0].data_ro.ravel().copy(), geo,
                            (Q.V.cell_node_map, Q.V.offset), V.node_count, Q.node_count, NU, 0.3)
    bn = np.unique(np.concatenate([bc.nodes for bc in bcs]))
    want = so.constrained(K, so.velocity_dofs(bn)) @ _flat(x)
    assert relerr(_flat(y), want) < TOL
    with pytest.raises(NotImplementedError, match="not symmetric"):
        A.multTranspose(x, y)


_CREATE_REFUSALS = [
    (dict(cdim=1), {}, "value size 3 only"),
    (dict(degree=1, nq=2), {}, "degree 1 outside 2..4"),
    (dict(degree=5, nq=6), {}, "degree 5 outside 2..4"),
    (dict(rank=2), {}, "mixed form, a rank-1 action only"),
    (dict(diagonal=1), {}, "mixed form, a rank-1 action only"),
    (dict(affine_cells=1), {}, "no affine-cell variant"),
    (dict(nq=4), {}, "nq == degree\\+1"),
    (dict(cell=_lib.CELL_HEX_EXTRUDED), {}, "needs the layer offsets of the second map"),
    ({}, dict(degree=2), "needs a second space of degree 1, got 2"),
]


@pytest.mark.parametrize("form,name", [(_lib.FORM_NAVIER_STOKES, "navier_stokes"),
                                       (_lib.FORM_NAVIER_STOKES_JACOBIAN, "navier_stokes_jacobian")])
@pytest.mark.parametrize("kw,kw2,msg", _CREATE_REFUSALS)
def test_create_refusals(engine, form, name, kw, kw2, msg):
    import ctypes as C
    d = tg._desc(kw.get("degree", 2), **kw)
    d.form = form
    keep = []
    if kw.get("cell") == _lib.CELL_HEX_EXTRUDED:
        keep = [np.zeros(27, dtype=np.int32), np.zeros(8, dtype=np.int32)]
        d.offset0 = keep[0].ctypes.data_as(C.POINTER(C.c_int32))
        d.offset1 = keep[1].ctypes.data_as(C.POINTER(C.c_int32))
    s2 = tg._space2(max(2, kw.get("degree", 2)), **kw2)
    h = C.c_void_p()
    with pytest.raises(_lib.EngineError, match=f"{name}\\b.*{msg}"):
        _lib.check(engine.fdb_kernel_create_mixed(C.byref(d), C.byref(s2), C.byref(h)), "fdb_kernel_create_mixed")
    h = C.c_void_p()
    with pytest.raises(_lib.EngineError, match=f"{name} is a form on two spaces"):
        _lib.check(engine.fdb_kernel_create(C.byref(tg._desc(2, form=form)), C.byref(h)), "fdb_kernel_create")


def test_call_refusals(engine):
    """Wrong argument or map counts and host-resident Dats are refused with the arguments named in their
    order; op2 refuses a pressure Dat with more than one value per node."""
    mesh, V, Q, cells, nodes, qnodes, m0, m1, m2, X, _, _ = tg.setup(2, False)
    vs = op2.DataSet(nodes, 3)
    yu, w, u, yp, r = op2.Dat(vs), op2.Dat(vs), op2.Dat(vs), op2.Dat(qnodes), op2.Dat(qnodes)
    for form, want, names in (("navier_stokes", 5, r"y, coords, x, y_p, p"),
                              ("navier_stokes_jacobian", 6, r"y, coords, x, y_p, p, u")):
        k = op2.Kernel(form, degree=2, mu=NU)
        gk = op2.GlobalKernel(k, [m0, m1, m2], extruded=True)
        with pytest.raises(_lib.EngineError, match=rf"{form} action expects {want} device args \({names}\) and 3 "
                                                   rf"maps, got 3/2"):
            gk(0, mesh.num_base_cells, cells.layers_array.ravel(), None, [yu.device_ptr, X.device_ptr, w.device_ptr],
               None, None, [m0.device_ptr, m1.device_ptr], None, _lib.LOC_DEVICE, False, False)
        args = [yu(op2.INC, m0), X(op2.READ, m1), w(op2.READ, m0), yp(op2.INC, m2), r(op2.READ, m2)]
        args += [u(op2.READ, m0)] if want == 6 else []
        loop = op2.Parloop(gk, cells, args, location="host")
        with pytest.raises(_lib.EngineError, match=f"expects {want} device args"):
            loop()
        with pytest.raises(ValueError, match="pressure Dats have 1 value per node"):
            p3 = op2.Dat(op2.DataSet(qnodes, 3))
            op2.par_loop(k, cells, *(args[:3] + [p3(op2.INC, m2)] + args[4:]))


def _cavity(n, nu, p=2):
    from firedrake_b200.assemble import DirichletBC, FunctionSpace, NavierStokes
    mesh = ExtrudedHexMesh(n, n, n)
    V, Q = FunctionSpace(mesh, p, 3), FunctionSpace(mesh, p - 1)
    F = NavierStokes(V, Q, nu)
    lid = np.zeros((V.node_count, 3))
    lid[:, 0] = 1.0
    bcs = [DirichletBC(V, 0.0, (1, 2, 3, 4, "bottom")), DirichletBC(V, V.dat(lid), "top")]
    return mesh, V, Q, F, bcs


def _fieldsplit(pc0, ksp_rtol=1e-8):
    return {"snes_rtol": 1e-10, "ksp_rtol": ksp_rtol, "ksp_max_it": 2000, "pc_type": "fieldsplit",
            "pc_fieldsplit_type": "schur", "pc_fieldsplit_schur_fact_type": "diag", "fieldsplit_0_pc_type": pc0,
            "fieldsplit_1_pc_type": "jacobi"}


def _scipy_cavity(mesh, V, Q, F, bcs):
    geo = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    bd = so.velocity_dofs(np.unique(np.concatenate([bc.nodes for bc in bcs])))
    g = np.zeros((V.node_count, 3))
    g[bcs[1].nodes, 0] = 1.0
    return nso.newton(interval_element(V.degree), mesh.coordinates, geo, (Q.V.cell_node_map, Q.V.offset),
                      V.node_count, Q.node_count, F.nu, bd, g.ravel(), F.beta)


def test_lid_driven_cavity_matches_scipy(engine):
    """Q2-Q1 on 8^3 at Re = 10, Newton with fieldsplit + mg and the constant-pressure nullspace: the velocity
    within 1e-8 of scipy's Newton on the oracle system, the pressure within 1e-7 modulo a constant."""
    from firedrake_b200.assemble import solve_nonlinear
    from firedrake_b200.mg import MeshHierarchy
    mesh, V, Q, F, bcs = _cavity(8, 0.1)
    up = F.dat()
    hist, kits = solve_nonlinear(F, F.dat(), up, bcs, _fieldsplit("mg", 1e-10), hierarchy=MeshHierarchy(2, 2, 2, 2),
                                 nullspace="constant")
    assert hist[-1] <= 1e-10 * hist[0] and len(kits) < 10, (hist, kits)
    u_ref, p_ref, _ = _scipy_cavity(mesh, V, Q, F, bcs)
    assert np.abs(up[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    p = up[1].data_ro
    assert abs(p.mean()) < 1e-12 * np.abs(p_ref).max()
    assert np.abs(p - p.mean() - p_ref).max() < 1e-7 * np.abs(p_ref).max()


def test_manufactured_solution_rates(engine):
    """u = curl psi and a zero-mean p on the unit cube, f = -nu lap u + (u . grad) u + grad p + beta u, Q2-Q1:
    L2 rates against the interpolants, velocity >= 2.8 and pressure >= 1.8 from 4^3 to 8^3."""
    import sympy as sp
    from firedrake_b200.assemble import DirichletBC, Form, FunctionSpace, NavierStokes, assemble, solve_nonlinear
    x, y, z = sp.symbols("x y z")
    psi = (sp.sin(sp.pi * x) * sp.sin(sp.pi * y) * sp.sin(sp.pi * z)) ** 2
    psi_v = sp.Matrix([0, psi, psi * sp.cos(x)])
    curl = lambda A: sp.Matrix([sp.diff(A[2], y) - sp.diff(A[1], z), sp.diff(A[0], z) - sp.diff(A[2], x),
                                sp.diff(A[1], x) - sp.diff(A[0], y)])
    ue = curl(psi_v)
    pe = sp.cos(sp.pi * x) * sp.cos(sp.pi * y) * sp.cos(sp.pi * z)
    nu, beta = 0.5, 0.5
    X3 = (x, y, z)
    f = [-nu * sum(sp.diff(ue[i], v, 2) for v in X3) + sum(ue[k] * sp.diff(ue[i], X3[k]) for k in range(3))
         + sp.diff(pe, X3[i]) + beta * ue[i] for i in range(3)]
    fu = [sp.lambdify(X3, e, "numpy") for e in ue]
    ff = [sp.lambdify(X3, e, "numpy") for e in f]
    fp = sp.lambdify(X3, pe, "numpy")
    errs = []
    for n in (4, 8):
        mesh = ExtrudedHexMesh(n, n, n)
        V, Q = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1)
        Vs = FunctionSpace(mesh, 2)
        Xv, Xq = V.V.dof_coordinates(), Q.V.dof_coordinates()
        ev = lambda fs, X: np.stack([np.broadcast_to(g(X[:, 0], X[:, 1], X[:, 2]), (len(X),)) for g in fs], axis=1)
        uI, pI = ev(fu, Xv), fp(Xq[:, 0], Xq[:, 1], Xq[:, 2])
        fI = ev(ff, Xv)
        F = NavierStokes(V, Q, nu, beta)
        L = F.dat()
        for c in range(3):
            L[0].data[:, c] = assemble(Form(Vs, 0.0, 1.0), u=Vs.dat(fI[:, c].copy())).data_ro
        bcs = [DirichletBC(V, V.dat(uI.copy()), ALL_FACES)]
        up = F.dat()
        hist, _ = solve_nonlinear(F, L, up, bcs, _fieldsplit("jacobi", 1e-10), nullspace="constant")
        assert hist[-1] <= 1e-10 * hist[0], hist
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
    """Re = 10: the GMRES iterations per Newton step with the velocity V-cycle at 16^3 are at most 1.25 times
    those at 8^3, and fewer than with velocity Jacobi at 16^3."""
    from firedrake_b200.assemble import solve_nonlinear
    from firedrake_b200.mg import MeshHierarchy
    its = {}
    for n, pc0 in ((8, "mg"), (16, "mg"), (16, "jacobi")):
        _, V, Q, F, bcs = _cavity(n, 0.1)
        hier = MeshHierarchy(2, 2, 2, {8: 2, 16: 3}[n]) if pc0 == "mg" else None
        up = F.dat()
        _, kits = solve_nonlinear(F, F.dat(), up, bcs, _fieldsplit(pc0), hierarchy=hier, nullspace="constant")
        its[(n, pc0)] = np.mean(kits)
    assert its[(16, "mg")] <= 1.25 * its[(8, "mg")], its
    assert its[(16, "mg")] < its[(16, "jacobi")], its


def test_solver_refusals(engine):
    from firedrake_b200.assemble import NonlinearDiffusion, assemble, solve_nonlinear
    _, V, Q, F, bcs = _cavity(2, 0.1)
    up = F.dat()
    J = F.jacobian(up)
    with pytest.raises(ValueError, match="residual is a 1-form"):
        assemble(F)
    with pytest.raises(ValueError, match="residual is a 1-form"):
        F.kernel(2)
    for mt in ("aij", "is"):
        with pytest.raises(NotImplementedError, match="Navier-Stokes Jacobian has no assembled matrix"):
            assemble(J, mat_type=mt)
    with pytest.raises(NotImplementedError, match="action only"):
        J.kernel(2)
    fs = {"pc_type": "fieldsplit", "pc_fieldsplit_type": "schur", "pc_fieldsplit_schur_fact_type": "diag"}
    for extra, msg in (({"ksp_type": "cg"}, "gmres"), ({"mat_type": "aij"}, "matfree"),
                       ({"pc_type": "jacobi"}, "'none' or 'fieldsplit'"),
                       ({"pc_type": "fieldsplit", "pc_fieldsplit_type": "additive"}, "'schur' only"),
                       ({**fs, "pc_fieldsplit_schur_fact_type": "full"}, "'diag' only"),
                       ({**fs, "fieldsplit_0_pc_type": "ilu"}, "'jacobi' or 'mg'"),
                       ({**fs, "fieldsplit_1_pc_type": "mg"}, "fieldsplit_1_pc_type"),
                       ({**fs, "fieldsplit_0_ksp_type": "cg"}, "preonly")):
        with pytest.raises(NotImplementedError, match=msg):
            solve_nonlinear(F, F.dat(), up, bcs, extra)
    with pytest.raises(ValueError, match="hierarchy"):
        solve_nonlinear(F, F.dat(), up, bcs, {**fs, "fieldsplit_0_pc_type": "mg"})
    with pytest.raises(NotImplementedError, match="nullspace"):
        solve_nonlinear(F, F.dat(), up, bcs, nullspace="rigid")
    with pytest.raises(NotImplementedError, match="Navier-Stokes forms only"):
        solve_nonlinear(NonlinearDiffusion(Q), Q.dat(), Q.dat(), nullspace="constant")
