"""Host logic of FDMPC with the vertex-star relaxation on the CPU (DESIGN.md section 4.20).

* The solver options of both demo shapes (one-level ASMExtrudedStarPC, and P1PC / PMGPC with the star smoother in
  pmg_mg_levels), nested or flattened, and every refusal by its message.
* Against a mock engine that computes fdb_fdm_star_* in NumPy from the C ABI's arrays (tests/_fdm_oracle.py) on top
  of the p-multigrid mock: the engine calls of one one-level apply and one P1PC + star cycle at p = 2 and 3, and the
  outer iterations that bound tests/test_fdm_gpu.py::test_iterations."""
import numpy as np
import pytest

import _fdm_oracle as fo
import _mock_engine as me
from firedrake_b200.assemble import (DirichletBC, Elasticity, Form, FunctionSpace, _fdm, fdm_options, mass,
                                     pmg_options, solve)
from firedrake_b200.utility_meshes import ExtrudedHexMesh
from test_pmg_host_mock import PMGEngine

STAR_INNER = {"pc_type": "python", "pc_python_type": "firedrake.ASMExtrudedStarPC", "pc_star_use_coloring": True,
              "pc_star_sub_sub_pc_type": "lu"}
LEVELS = {"ksp_type": "chebyshev", "ksp_max_it": 2, "pc_type": "python",
          "pc_python_type": "firedrake.ASMExtrudedStarPC", "pc_star_use_coloring": True,
          "pc_star_sub_sub_pc_type": "lu"}


def fdm(inner):
    return {"pc_type": "python", "pc_python_type": "firedrake.FDMPC", "fdm": inner}


def two_level(kind="firedrake.P1PC", **levels):
    return fdm({"pc_type": "python", "pc_python_type": kind, "pmg_mg_levels": dict(LEVELS, **levels)})


def test_one_level_options():
    assert fdm_options(fdm(STAR_INNER)) == ("star", None)
    assert fdm_options(fdm(dict(STAR_INNER, pc_python_type="firedrake.ASMStarPC")))[0] == "star"
    flat = {"pc_type": "python", "pc_python_type": "firedrake.FDMPC", "fdm_pc_type": "python",
            "fdm_pc_python_type": "firedrake.ASMExtrudedStarPC", "fdm_pc_star_construct_dim": 0,
            "fdm_pc_star_use_coloring": False}
    assert fdm_options(flat) == ("star", None)


@pytest.mark.parametrize("kind", ["firedrake.P1PC", "firedrake.PMGPC"])
def test_two_level_options(kind):
    k, o = fdm_options(two_level(kind, ksp_max_it=3))
    assert k == "pmg" and o["level_pc"] == "star" and o["halve"] == (kind == "firedrake.PMGPC")
    assert (o["pmg_mg_levels_ksp_type"], o["pmg_mg_levels_ksp_max_it"]) == ("chebyshev", 3)
    assert (o["pmg_mg_coarse_ksp_type"], o["pmg_mg_coarse_pc_type"]) == ("cg", "jacobi")


def test_pmg_pins_unchanged():
    with pytest.raises(NotImplementedError, match="pc_python_type 'firedrake.ASMStarPC'"):
        pmg_options({"pc_python_type": "firedrake.ASMStarPC"})
    with pytest.raises(NotImplementedError, match="pmg_mg_levels_pc_python_type"):
        pmg_options({"pc_python_type": "firedrake.PMGPC", "pmg_mg_levels": {"pc_python_type": "x"}})


@pytest.mark.parametrize("sp,msg", [
    (fdm({"pc_type": "lu"}), "fdm_pc_type 'lu': there is no direct solver"),
    (fdm({"pc_type": "cholesky"}), "fdm_pc_type 'cholesky': there is no direct solver"),
    (fdm({"pc_type": "jacobi"}), "fdm_pc_type 'jacobi'"),
    (fdm(dict(STAR_INNER, pc_python_type="firedrake.PatchPC")), "fdm_pc_python_type 'firedrake.PatchPC'"),
    (fdm(dict(STAR_INNER, pc_star_construct_dim=1)), "fdm_pc_star_construct_dim 1"),
    (fdm(dict(STAR_INNER, pc_star_sub_sub_pc_type="ilu")), "fdm_pc_star_sub_sub_pc_type 'ilu'"),
    (fdm(dict(STAR_INNER, pc_star_mat_ordering_type="nd")), "fdm_pc_star_mat_ordering_type"),
    (fdm(dict(STAR_INNER, ksp_type="gmres")), "unknown FDMPC option.*fdm_ksp_type"),
    (two_level(pc_star_sub_sub_pc_type="cholesky"), "fdm_pmg_mg_levels_pc_star_sub_sub_pc_type 'cholesky'"),
    (two_level(ksp_type="richardson"), "fdm_pmg_mg_levels_ksp_type 'richardson'"),
    (two_level(pc_python_type="firedrake.PatchPC"), "fdm_pmg_mg_levels_pc_python_type 'firedrake.ASMExtrudedStarPC'"),
    (two_level(pc_jacobi_type="rowsum"), "unknown FDMPC option.*fdm_pmg_mg_levels_pc_jacobi_type"),
    (dict(two_level(), fdm=dict(two_level()["fdm"], ksp_type="gmres")), "unknown FDMPC option.*fdm_ksp_type"),
    (dict(two_level(), fdm=dict(two_level()["fdm"], mat_type="aij")), "unknown FDMPC option.*fdm_mat_type"),
    (dict(two_level(), fdm=dict(two_level()["fdm"], pmg_foo=1)), "unknown p-multigrid option.*pmg_foo"),
])
def test_option_refusals(sp, msg):
    with pytest.raises(NotImplementedError, match=msg):
        fdm_options(sp)


def test_direct_coarse_solve_is_refused():
    """fdm_options passes the coarse options on; p-multigrid refuses a direct coarse solve when it is built."""
    V = FunctionSpace(ExtrudedHexMesh(3, 3, 3), 2)
    sp = fdm({"pc_type": "python", "pc_python_type": "firedrake.P1PC", "pmg_mg_levels": LEVELS,
              "pmg_mg_coarse": {"pc_type": "lu"}})
    assert fdm_options(sp)[1]["pmg_mg_coarse_pc_type"] == "lu"
    with pytest.raises(NotImplementedError, match="coarse solve ksp_type 'cg' with pc_type 'lu'"):
        _fdm(Form(V), (), sp)


def test_form_refusals():
    mesh = ExtrudedHexMesh(3, 3, 3)
    V = FunctionSpace(mesh, 2)
    sp = fdm(STAR_INNER)
    with pytest.raises(NotImplementedError, match="FDMPC on Elasticity"):
        _fdm(Elasticity(FunctionSpace(mesh, 2, 3), 1.0, 1.0), (), sp)
    with pytest.raises(NotImplementedError, match="ds terms"):
        _fdm(Form(V, ds=((1.0, 1),)), (), sp)
    with pytest.raises(NotImplementedError, match="scalar CG spaces only"):
        _fdm(Form(FunctionSpace(mesh, 2, family="DQ")), (), sp)
    with pytest.raises(NotImplementedError, match="scalar CG spaces only"):
        _fdm(Form(FunctionSpace(mesh, 2, 3)), (), sp)
    for p in (4, 5):
        with pytest.raises(NotImplementedError, match=f"P1PC / PMGPC at fine degree {p}"):
            _fdm(Form(FunctionSpace(mesh, p)), (), two_level())
    # the relaxation itself takes a Form without ds terms only, whoever builds it (mg.PMG's levels too)
    from firedrake_b200.patch import FDMStar
    with pytest.raises(NotImplementedError, match="FDMStar takes a Form without ds terms.*Form with ds terms"):
        FDMStar(Form(V, ds=((1.0, 1),)))
    with pytest.raises(NotImplementedError, match="FDMStar takes a Form without ds terms.*not Elasticity"):
        FDMStar(Elasticity(FunctionSpace(mesh, 2, 3), 1.0, 1.0))


class FDMEngine(fo.FDMMixin, PMGEngine):
    pass


class fdm_mock(me.install):
    def __init__(self, oracle, compute=True):
        self.engine = FDMEngine(oracle, compute)


def test_star_outside_fdmpc_is_refused(oracle):
    with fdm_mock(oracle):
        V = FunctionSpace(ExtrudedHexMesh(2, 2, 2), 2)
        for kind in ("firedrake.ASMStarPC", "firedrake.ASMExtrudedStarPC"):
            with pytest.raises(NotImplementedError, match=f"pc_python_type '{kind}' outside firedrake.FDMPC"):
                solve(Form(V), V.dat(), V.dat(), solver_parameters={"pc_type": "python", "pc_python_type": kind})


def _problem(p, nx=3, ny=2, nz=3):
    V = FunctionSpace(ExtrudedHexMesh(nx, ny, nz, warp=0.05, permute_seed=2), p)
    return V, [DirichletBC(V, 0.0, s) for s in ("bottom", "top")]


@pytest.mark.parametrize("p", [2, 3])
def test_one_level_apply_engine_calls(oracle, p):
    """One application is one fdb_fdm_star_apply, and the mock's gather from the ABI arrays is the lattice
    oracle's."""
    with fdm_mock(oracle) as eng:
        V, bcs = _problem(p)
        M = _fdm(Form(V, 1.0, 0.5), bcs, fdm(STAR_INNER))
        r = np.random.default_rng(0).standard_normal(V.node_count)
        z = V.dat()
        rd = V.dat(r)
        rd.device_ptr
        z.device_ptr
        eng.trace.clear()
        M(rd, z)
        assert eng.trace == [("fdb_fdm_star_apply", V.node_count)]
        st = next(iter(eng.stars.values()))
        from firedrake_b200.patch import StarTables
        t = StarTables(V, ("bottom", "top"))
        nodes, _ = fo.star_nodes(V, t)
        assert np.array_equal(np.sort(st["nodes"].ravel()), np.sort(nodes.ravel()))
        ref = fo.apply(t, nodes, r, 1.0, 0.5)
        assert np.abs(z.data_ro - ref).max() < 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize("p", [2, 3])
def test_p1pc_star_cycle_engine_calls(oracle, p):
    """One P1PC cycle with the star smoother, nu = 2: on the fine level per Chebyshev iteration one action, the
    residual, one star apply and one fused pass; then the residual, one restriction, the coarse Jacobi-PCG, one
    prolongation and the post-smoothing."""
    with fdm_mock(oracle) as eng:
        V, bcs = _problem(p)
        M = _fdm(Form(V), bcs, two_level())
        r = V.dat(np.sin(np.arange(V.node_count)))
        for bc in bcs:
            bc.zero(r)
        z = V.dat()
        M(r, z)
        z.zero()
        z.device_ptr
        eng.trace.clear()
        M(r, z)
        trace = list(eng.trace)
    nf = V.node_count
    A = ("helmholtz", p, "action")
    zero_bc = [("fdb_dat_zero_nodes", None)] * len(bcs)
    mult = [("fdb_memcpy_d2d", None)] + zero_bc + [("fdb_memset", None), A] + [("fdb_dat_set_nodes", None)] * len(bcs)
    it = mult + [("fdb_vec_aypx", nf), ("fdb_fdm_star_apply", nf), ("fdb_vec_chebyshev", nf)]
    i_r, i_p = trace.index(("p_restrict", p, 1)), trace.index(("p_prolong", p, 1))
    assert trace[:i_r] == it + it + mult + [("fdb_vec_aypx", nf)] + zero_bc + [("fdb_memset", None)]
    assert trace[i_p + 1:] == zero_bc + [("fdb_vec_axpy", nf)] + it + it
    assert [t[0] for t in trace].count("fdb_fdm_star_apply") == 4


def _poisson(V, sp):
    bcs = [DirichletBC(V, 0.0, s) for s in ("bottom", "top")]
    from firedrake_b200.assemble import assemble
    L = assemble(mass(V), u=V.dat(np.sin(np.arange(V.node_count) * 0.37)))
    u = V.dat()
    its, _ = solve(Form(V, 1.0, 0.0), L, u, bcs=bcs, solver_parameters=dict(sp, ksp_rtol=1e-11))
    return its


# the outer iterations of P1PC + star to rtol 1e-11 on warped 8^3 and 16^3 meshes (tests/test_fdm_gpu.py::
# test_iterations is bounded by these)
MOCK_ITS = {2: {8: 13, 16: 12}, 3: {8: 12, 16: 12}}


@pytest.mark.parametrize("p", [2, 3])
def test_iterations_on_mock(oracle, p):
    its = {}
    for n in (8, 16):
        with fdm_mock(oracle):
            its[n] = _poisson(FunctionSpace(ExtrudedHexMesh(n, n, n, warp=0.05), p), two_level())
    print(f"CG{p}: P1PC + star {its}")
    assert its == MOCK_ITS[p]


@pytest.mark.parametrize("case", ["none", "jacobi", "mg", "pmgpc", "p1pc"])
def test_solve_engine_calls_unchanged(oracle, case):
    """solve with pc_type none, jacobi, mg and the p-multigrid python options makes exactly the engine calls it made
    before FDMPC was added (recorded from that version by the same function into
    tests/golden/solve_pc_engine_calls.json)."""
    import json
    import os
    import _solve_recorder as sr
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "solve_pc_engine_calls.json")) as f:
        want = json.load(f)[case]
    names, trace = sr.solve_calls(oracle, case)
    assert trace == want["trace"]
    assert names == want["names"]
