"""GPU tests of the Boussinesq (Rayleigh-Benard) system on Taylor-Hood hexahedra with the temperature on the
pressure numbering (FDB_FORM_BOUSSINESQ[_JACOBIAN], the EL_RB_RESIDUAL / EL_RB_JACOBIAN modes of
csrc/elasticity_hex.cu): the residual and the Jacobian action against the NumPy oracle (tests/_boussinesq_oracle.py)
on extruded and native hexes with atomic and coloured scatter, the generic wrapper path, the Navier-Stokes kernel at
Ra = 0, the Taylor ratio, the refusals, and Newton with the demo's fieldsplit on the differentially heated cavity
against scipy's Newton.  Tolerance 1e-12 relative in the max norm for the actions."""
import ctypes as C

import numpy as np
import pytest

import _boussinesq_oracle as bo
import test_stokes_gpu as tg
from firedrake_b200 import _lib, op2
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

TOL = 1e-12
BG = (0.4, -0.3, -2.1)
KT = 0.7
WALLS = (1, 2, 3, 4, "bottom", "top")


def relerr(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def _loop(k, cells, ys, xs, m0, m1, m2, X, lin=None, scatter="atomic"):
    (yu, yp, yt), (x, q, t) = ys, xs
    extra = [lin[0](op2.READ, m0), lin[1](op2.READ, m2)] if lin is not None else []
    op2.par_loop(k, cells, yu(op2.INC, m0), X(op2.READ, m1), x(op2.READ, m0), yp(op2.INC, m2), q(op2.READ, m2),
                 yt(op2.INC, m2), t(op2.READ, m2), *extra, scatter=scatter)


@pytest.mark.parametrize("p", [2, 3, 4])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
@pytest.mark.parametrize("jac", [False, True], ids=["residual", "jacobian"])
def test_action_matches_oracle(engine, p, native, jac):
    """Atomic and coloured scatter, all three blocks; coloured is bit-identical across calls."""
    mesh, V, Q, cells, nodes, qnodes, m0, m1, m2, X, geo, geo2 = tg.setup(p, native)
    rng = np.random.default_rng(p + 10 * native)
    vs = op2.DataSet(nodes, 3)
    x = op2.Dat(vs, rng.standard_normal((V.node_count, 3)))
    q = op2.Dat(qnodes, rng.standard_normal(Q.node_count))
    t = op2.Dat(qnodes, rng.standard_normal(Q.node_count))
    lin = (op2.Dat(vs, rng.standard_normal((V.node_count, 3))), op2.Dat(qnodes, rng.standard_normal(Q.node_count))) \
        if jac else None
    el = interval_element(p)
    flat = lambda d: d.data_ro.ravel().copy()
    if jac:
        want = bo.jacobian_action(el, mesh.coordinates, flat(lin[0]), flat(lin[1]), flat(x), flat(q), flat(t), geo,
                                  geo2, BG, KT)
    else:
        want = bo.residual(el, mesh.coordinates, flat(x), flat(q), flat(t), geo, geo2, BG, KT)
    k = op2.Kernel("boussinesq_jacobian" if jac else "boussinesq", degree=p, mu=1.0, bg=BG, kt=KT)
    ys = (op2.Dat(vs), op2.Dat(qnodes), op2.Dat(qnodes))
    _loop(k, cells, ys, (x, q, t), m0, m1, m2, X, lin)
    for y, w in zip(ys, want):
        assert relerr(flat(y), w) < TOL
    outs = []
    for _ in range(2):
        for y in ys:
            y.zero()
        _loop(k, cells, ys, (x, q, t), m0, m1, m2, X, lin, scatter="coloured")
        outs.append([flat(y) for y in ys])
    for a, b, w in zip(outs[0], outs[1], want):
        assert np.array_equal(a, b)
        assert relerr(a, w) < TOL


def _form(p, Ra=2.0e3, Pr=0.8, g=(0.3, 0.1, -1.0), mesh=None):
    from firedrake_b200.assemble import Boussinesq, FunctionSpace
    mesh = mesh or ExtrudedHexMesh(4, 3, 5, warp=0.05, permute_seed=2)
    return Boussinesq(FunctionSpace(mesh, p, 3), FunctionSpace(mesh, p - 1), FunctionSpace(mesh, p - 1), Ra, Pr, g)


def _random(F, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return F.dat(scale * rng.standard_normal((F.V.node_count, 3)), scale * rng.standard_normal(F.Q.node_count),
                 scale * rng.standard_normal(F.W.node_count))


def _flat(y):
    return np.concatenate([d.data_ro.ravel() for d in y])


@pytest.mark.parametrize("p", [2, 3, 4])
def test_matches_generic_path(engine, p):
    from firedrake_b200.assemble import assemble, assemble_boussinesq_generic
    F = _form(p)
    upT, wrs = _random(F, 3), _random(F, 4)
    assert relerr(_flat(assemble(F, u=upT)), _flat(assemble_boussinesq_generic(F, upT))) < TOL
    assert relerr(_flat(assemble(F.jacobian(upT), u=wrs)), _flat(assemble_boussinesq_generic(F, upT, wrs))) < TOL


@pytest.mark.parametrize("p", [2, 3, 4])
def test_ra_zero_is_navier_stokes(engine, p):
    """At Ra = 0 the (u, p) rows of the residual and of the Jacobian are NavierStokes(V, Q, nu=1)'s on the device."""
    from firedrake_b200.assemble import NavierStokes, assemble
    F = _form(p, Ra=0.0)
    N = NavierStokes(F.V, F.Q, 1.0)
    upT, wrs = _random(F, 5), _random(F, 6)
    up, wr = N.dat(upT[0].data_ro, upT[1].data_ro), N.dat(wrs[0].data_ro, wrs[1].data_ro)
    R, Rn = assemble(F, u=upT), assemble(N, u=up)
    for b in range(2):
        assert relerr(R[b].data_ro.ravel(), Rn[b].data_ro.ravel()) < TOL
    J, Jn = assemble(F.jacobian(upT), u=wrs), assemble(N.jacobian(up), u=wr)
    for b in range(2):
        assert relerr(J[b].data_ro.ravel(), Jn[b].data_ro.ravel()) < TOL


@pytest.mark.parametrize("p", [2, 3, 4])
def test_taylor_ratio(engine, p):
    """max|R(x + h d) - R(x) - h J d| falls by 4 when h is halved (R is quadratic)."""
    from firedrake_b200.assemble import assemble
    F = _form(p)
    upT, wrs = _random(F, 7), _random(F, 8)
    R0 = _flat(assemble(F, u=upT))
    Jw = _flat(assemble(F.jacobian(upT), u=wrs))
    rem = []
    for h in (0.1, 0.05):
        xh = F.dat(*[a.data_ro + h * b.data_ro for a, b in zip(upT, wrs)])
        rem.append(np.abs(_flat(assemble(F, u=xh)) - R0 - h * Jw).max())
    assert 3.5 <= rem[0] / rem[1] <= 4.5, rem


@pytest.mark.parametrize("form,name", [(_lib.FORM_BOUSSINESQ, "boussinesq"),
                                       (_lib.FORM_BOUSSINESQ_JACOBIAN, "boussinesq_jacobian")])
def test_create_refusals(engine, form, name):
    """Rank 2 and the diagonal are refused naming the form; so is creation without the second space."""
    for kw in (dict(rank=2), dict(diagonal=1)):
        d = tg._desc(2, form=form, **kw)
        h = C.c_void_p()
        with pytest.raises(_lib.EngineError, match=f"{name} is a mixed form, a rank-1 action only"):
            _lib.check(engine.fdb_kernel_create_mixed(C.byref(d), C.byref(tg._space2(2)), C.byref(h)),
                       "fdb_kernel_create_mixed")
    h = C.c_void_p()
    with pytest.raises(_lib.EngineError, match=f"{name} is a form on two spaces"):
        _lib.check(engine.fdb_kernel_create(C.byref(tg._desc(2, form=form)), C.byref(h)), "fdb_kernel_create")


def test_call_refusals(engine):
    """Wrong argument counts and host-resident Dats are refused with the arguments named in their order."""
    mesh, V, Q, cells, nodes, qnodes, m0, m1, m2, X, _, _ = tg.setup(2, False)
    vs = op2.DataSet(nodes, 3)
    yu, w, u, yp, r, yt, s, t0 = (op2.Dat(vs), op2.Dat(vs), op2.Dat(vs), op2.Dat(qnodes), op2.Dat(qnodes),
                                  op2.Dat(qnodes), op2.Dat(qnodes), op2.Dat(qnodes))
    for form, want, names in (("boussinesq", 7, r"y, coords, x, y_p, p, y_T, T"),
                              ("boussinesq_jacobian", 9, r"y, coords, x, y_p, p, y_T, s, u0, T0")):
        k = op2.Kernel(form, degree=2)
        gk = op2.GlobalKernel(k, [m0, m1, m2], extruded=True)
        with pytest.raises(_lib.EngineError, match=rf"{form} action expects {want} device args \({names}\) and 3 "
                                                   rf"maps, got 5/3"):
            gk(0, mesh.num_base_cells, cells.layers_array.ravel(), None,
               [yu.device_ptr, X.device_ptr, w.device_ptr, yp.device_ptr, r.device_ptr], None, None,
               [m0.device_ptr, m1.device_ptr, m2.device_ptr], None, _lib.LOC_DEVICE, False, False)
        args = [yu(op2.INC, m0), X(op2.READ, m1), w(op2.READ, m0), yp(op2.INC, m2), r(op2.READ, m2),
                yt(op2.INC, m2), s(op2.READ, m2)]
        args += [u(op2.READ, m0), t0(op2.READ, m2)] if want == 9 else []
        with pytest.raises(_lib.EngineError, match=f"{form} action expects {want} device args"):
            op2.Parloop(gk, cells, args, location="host")()


def _cavity(n, Ra, Pr, p=2):
    """The differentially heated cube of Firedrake's demo in 3-D: no slip on every wall, T = 1 on face 1 (x = 0),
    T = 0 on face 2 (x = 1), adiabatic elsewhere."""
    from firedrake_b200.assemble import DirichletBC
    F = _form(p, Ra, Pr, (0.0, 0.0, -1.0), ExtrudedHexMesh(n, n, n))
    bcs = [DirichletBC(F.V, 0.0, WALLS), DirichletBC(F.W, 1.0, 1), DirichletBC(F.W, 0.0, 2)]
    return F, bcs


def _demo_options(split="multiplicative", velocity_pc="jacobi", temperature_pc="jacobi"):
    """The demo's nested options with the assembled preconditioners replaced by the engine's."""
    return {"mat_type": "matfree", "snes_monitor": None, "snes_rtol": 1e-10,
            "ksp_type": "fgmres", "ksp_gmres_modifiedgramschmidt": None, "ksp_monitor_true_residual": None,
            "ksp_rtol": 1e-8, "ksp_max_it": 500,
            "pc_type": "fieldsplit", "pc_fieldsplit_type": split,
            "pc_fieldsplit_0_fields": "0,1", "pc_fieldsplit_1_fields": "2",
            "fieldsplit_0": {"ksp_type": "gmres", "ksp_gmres_modifiedgramschmidt": None, "ksp_rtol": 1e-2,
                             "pc_type": "fieldsplit", "pc_fieldsplit_type": "schur",
                             "pc_fieldsplit_schur_fact_type": "lower",
                             "fieldsplit_0": {"ksp_type": "preonly", "pc_type": velocity_pc},
                             "fieldsplit_1": {"ksp_type": "preonly", "pc_type": "jacobi"}},
            "fieldsplit_1": {"ksp_type": "gmres", "ksp_rtol": 1e-4, "pc_type": temperature_pc}}


def test_heated_cavity_matches_scipy(engine):
    """Q2-Q1-Q1 on 6^3 at Ra = 1e3, Pr = 6.8: velocity and temperature within 1e-8 of scipy's Newton on the oracle
    system, the pressure within 1e-7 modulo a constant."""
    from firedrake_b200.assemble import solve_nonlinear
    F, bcs = _cavity(6, 1e3, 6.8)
    upT = F.dat()
    hist, kits, inner = solve_nonlinear(F, F.dat(), upT, bcs, _demo_options(), nullspace="constant")
    assert hist[-1] <= 1e-10 * hist[0] and len(kits) < 10, (hist, kits)
    assert all(a > 0 and b > 0 for a, b in inner)
    mesh, V, Q = F.V.mesh, F.V, F.Q
    nv, nq = V.node_count, Q.node_count
    geo = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    walls = bcs[0].nodes
    fixed = np.concatenate([(3 * walls[:, None] + np.arange(3)).ravel(), [3 * nv], 3 * nv + nq + bcs[1].nodes,
                            3 * nv + nq + bcs[2].nodes])
    values = np.concatenate([np.zeros(3 * len(walls) + 1), np.ones(len(bcs[1].nodes)), np.zeros(len(bcs[2].nodes))])
    u_ref, p_ref, T_ref, _ = bo.newton(interval_element(2), mesh.coordinates, geo, (Q.V.cell_node_map, Q.V.offset),
                                       nv, nq, F.bg, F.kt, fixed, values)
    assert np.abs(upT[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    assert np.abs(upT[2].data_ro - T_ref).max() < 1e-8 * np.abs(T_ref).max()
    p = upT[1].data_ro
    assert abs(p.mean()) < 1e-12 * np.abs(p_ref).max()
    assert np.abs(p - p.mean() - p_ref).max() < 1e-7 * np.abs(p_ref).max()


def test_multiplicative_needs_no_more_iterations_than_additive(engine):
    """16^3 at Ra = 1e4: the block Gauss-Seidel split takes no more outer iterations than the additive one."""
    from firedrake_b200.assemble import solve_nonlinear
    its = {}
    for split in ("multiplicative", "additive"):
        F, bcs = _cavity(16, 1e4, 6.8)
        upT = F.dat()
        hist, kits, _ = solve_nonlinear(F, F.dat(), upT, bcs, dict(_demo_options(split), snes_rtol=1e-8),
                                        nullspace="constant")
        assert hist[-1] <= 1e-8 * hist[0], (split, hist)
        its[split] = sum(kits)
    assert its["multiplicative"] <= its["additive"], its


def test_solver_refusals(engine):
    from firedrake_b200.assemble import DirichletBC, solve_nonlinear
    F, bcs = _cavity(2, 1e3, 6.8)
    base = _demo_options()
    cases = [({"fieldsplit_1_pc_type": "python", "fieldsplit_1_pc_python_type": "firedrake.AssembledPC"},
              "AssembledPC"),
             ({"fieldsplit_1_assembled_pc_type": "hypre"}, "hypre"),
             ({"fieldsplit_1_pc_type": "lu"}, "no assembled matrix"),
             ({"fieldsplit_1_pc_type": "mumps"}, "no assembled matrix"),
             ({"fieldsplit_1_pc_type": "ilu"}, "no assembled matrix"),
             ({"fieldsplit_0_fieldsplit_1_pc_type": "python",
               "fieldsplit_0_fieldsplit_1_pc_python_type": "firedrake.PCDPC"}, "4.13"),
             ({"pc_fieldsplit_type": "schur"}, "'multiplicative' or 'additive'"),
             ({"pc_fieldsplit_type": "symmetric_multiplicative"}, "'multiplicative' or 'additive'"),
             ({"pc_fieldsplit_type": "full"}, "'multiplicative' or 'additive'"),
             ({"pc_fieldsplit_0_fields": "0", "pc_fieldsplit_1_fields": "1,2"}, "'0,1'"),
             ({"ksp_type": "cg"}, "'fgmres' or 'gmres'"),
             ({"fieldsplit_1_ksp_type": "cg"}, "'preonly' or 'gmres'"),
             ({"not_an_option": 1}, "unknown Boussinesq solver option 'not_an_option'")]
    for extra, msg in cases:
        flat = dict(base)
        flat.update(extra)
        with pytest.raises(NotImplementedError, match=msg):
            solve_nonlinear(F, F.dat(), F.dat(), bcs, flat)
    with pytest.raises(NotImplementedError, match="pressure space"):
        solve_nonlinear(F, F.dat(), F.dat(), [DirichletBC(F.Q, 0.0, 1)], base)
