"""The fast-diagonalisation vertex-star relaxation on the device (csrc/fdm_star_hex.cu, patch.FDMStar) and FDMPC in
solve / solve_nonlinear (DESIGN.md section 4.20)."""
import numpy as np
import pytest
import scipy.sparse as sp

import _fdm_oracle as fo
from firedrake_b200.assemble import (DirichletBC, Form, FunctionSpace, NonlinearDiffusion, assemble,
                                     mass, solve, solve_nonlinear)
from firedrake_b200.patch import FDMStar, PatchASM, vertex_star_patches
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

STAR = {"pc_type": "python", "pc_python_type": "firedrake.FDMPC",
        "fdm": {"pc_type": "python", "pc_python_type": "firedrake.ASMExtrudedStarPC", "pc_star_use_coloring": True,
                "pc_star_sub_sub_pc_type": "lu"}}


def two_level(kind):
    return {"pc_type": "python", "pc_python_type": "firedrake.FDMPC",
            "fdm": {"pc_type": "python", "pc_python_type": kind,
                    "pmg_mg_levels": {"ksp_type": "chebyshev", "ksp_max_it": 2, "pc_type": "python",
                                      "pc_python_type": "firedrake.ASMExtrudedStarPC",
                                      "pc_star_sub_sub_pc_type": "lu"}}}


def _rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def _apply(star, V, r):
    z = V.dat()
    star.apply(V.dat(r), z)
    return z.data_ro.copy()


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("warp,kappa", [(0.0, False), (0.05, False), (0.05, True)])
def test_apply_matches_oracle(engine, p, warp, kappa):
    mesh = ExtrudedHexMesh(4, 3, 5, Lx=1.0, Ly=0.8, Lz=1.2, warp=warp, permute_seed=5)
    V = FunctionSpace(mesh, p)
    domains = ("bottom", 2, 3)
    bcs = [DirichletBC(V, 0.0, s) for s in domains]
    k = 1.0 + np.random.default_rng(1).random(V.node_count) if kappa else None
    form = Form(V, 0.8, 0.3, None if k is None else V.dat(k))
    star = FDMStar(form, bcs)
    nodes, _ = fo.star_nodes(V, star.tables)
    r = np.random.default_rng(2).standard_normal(V.node_count)
    z = _apply(star, V, r)
    ref = fo.apply(star.tables, nodes, r, 0.8, 0.3, k)
    assert _rel(z, ref) < 1e-12, _rel(z, ref)
    # Dirichlet rows stay zero, two applications are bitwise equal, <P r, s> = <r, P s>
    bc = np.unique(np.concatenate([V.boundary_nodes(s) for s in domains]))
    assert not z[bc].any()
    assert np.array_equal(_apply(star, V, r), z)
    s = np.random.default_rng(3).standard_normal(V.node_count)
    Ps = _apply(star, V, s)
    assert abs(z @ s - r @ Ps) < 1e-12 * np.abs(z).max() * np.abs(s).sum()


@pytest.mark.parametrize("p", [1, 2, 3])
def test_matches_patch_asm_on_unwarped_mesh(engine, p):
    """On a Cartesian mesh the separable star operators are the assembled star blocks: the relaxation is PatchASM
    on the assembled matrix."""
    mesh = ExtrudedHexMesh(3, 4, 3, Lx=0.9, Ly=1.1, Lz=0.7, permute_seed=2)
    V = FunctionSpace(mesh, p)
    bcs = [DirichletBC(V, 0.0, s) for s in (1, "top")]
    bc = np.unique(np.concatenate([V.boundary_nodes(s) for s in (1, "top")]))
    form = Form(V, 1.0, 0.5)
    A = assemble(form)
    ptr, dofs = vertex_star_patches(V, exclude=bc)
    asm = PatchASM(A, ptr, dofs)
    r = np.random.default_rng(0).standard_normal(V.node_count)
    x = V.dat()
    asm.apply(V.dat(r), x)
    z = _apply(FDMStar(form, bcs), V, r)
    assert _rel(z, x.data_ro) < 1e-12, _rel(z, x.data_ro)


def _poisson(V, sp_, domains=("bottom", "top"), form=None):
    bcs = [DirichletBC(V, 0.0, s) for s in domains]
    L = assemble(mass(V), u=V.dat(np.sin(np.arange(V.node_count) * 0.37)))
    u = V.dat()
    its, _ = solve(form or Form(V, 1.0, 0.0), L, u, bcs=bcs, solver_parameters=dict(sp_, ksp_rtol=1e-11))
    return u.data_ro.copy(), its


@pytest.mark.parametrize("p", [2, 3, 4, 5])
def test_one_level_solve(engine, p):
    """Against Jacobi-CG, or unpreconditioned CG at degrees 4 and 5, where there is no diagonal kernel."""
    V = FunctionSpace(ExtrudedHexMesh(4, 3, 5, warp=0.05, permute_seed=0), p)
    uj, its_j = _poisson(V, {"pc_type": "jacobi" if p <= 3 else "none", "ksp_max_it": 5000})
    u, its = _poisson(V, STAR)
    print(f"CG{p}: FDMPC + star {its}, {'Jacobi' if p <= 3 else 'unpreconditioned'} CG {its_j}")
    assert _rel(u, uj) < 1e-8 and its < its_j


@pytest.mark.parametrize("p", [2, 3])
@pytest.mark.parametrize("kind", ["firedrake.P1PC", "firedrake.PMGPC"])
def test_two_level_solve(engine, p, kind):
    V = FunctionSpace(ExtrudedHexMesh(6, 5, 7, warp=0.05, permute_seed=0), p)
    uj, _ = _poisson(V, {"pc_type": "jacobi", "ksp_max_it": 5000})
    u, its = _poisson(V, two_level(kind))
    assert _rel(u, uj) < 1e-8


def test_kappa_solve(engine):
    V = FunctionSpace(ExtrudedHexMesh(5, 4, 6, warp=0.05, permute_seed=1), 3)
    X = V.V.dof_coordinates()
    form = Form(V, 1.0, 0.0, V.dat(10.0 ** (2.0 * X[:, 0])))
    uj, _ = _poisson(V, {"pc_type": "jacobi", "ksp_max_it": 5000}, form=form)
    for sp_ in (STAR, two_level("firedrake.P1PC")):
        assert _rel(_poisson(V, sp_, form=form)[0], uj) < 1e-8


# P1PC + star outer iterations on the mock engine (tests/test_fdm_host_mock.py::test_iterations_on_mock), warped 8^3
# and 16^3, Dirichlet bottom and top, rtol 1e-11
MOCK_ITS = {2: {8: 13, 16: 12}, 3: {8: 12, 16: 12}}


@pytest.mark.parametrize("p", [2, 3])
def test_iterations(engine, p):
    its = {}
    for n in (8, 16):
        V = FunctionSpace(ExtrudedHexMesh(n, n, n, warp=0.05), p)
        _, its[n] = _poisson(V, two_level("firedrake.P1PC"))
    _, its1 = _poisson(V, STAR)
    print(f"CG{p}: P1PC + star {its}, one-level star at 16^3 {its1}")
    assert all(abs(its[n] - MOCK_ITS[p][n]) <= 1 for n in its), its


def test_newton(engine, monkeypatch):
    """Newton for NonlinearDiffusion with both shapes reaches the Jacobi solution; the one-level relaxation is
    built once per solve (its coefficients are refreshed at every step), P1PC's at every step."""
    from firedrake_b200 import patch
    built = []
    init = patch.FDMStar.__init__

    def counting(self, form, bcs=()):
        built.append(form.V.degree)
        init(self, form, bcs)
    monkeypatch.setattr(patch.FDMStar, "__init__", counting)
    mesh = ExtrudedHexMesh(5, 4, 6, warp=0.05, permute_seed=1)
    V = FunctionSpace(mesh, 2)
    bcs = [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, 1.0, "top")]
    L = assemble(mass(V), u=V.dat(np.ones(V.node_count)))
    out = []
    for sp_ in ({"pc_type": "jacobi"}, STAR, two_level("firedrake.P1PC")):
        u = V.dat()
        built.clear()
        hist, kits = solve_nonlinear(NonlinearDiffusion(V, 1.0, 0.0, (1.0, 0.5, 0.2)), L, u, bcs=bcs,
                                     solver_parameters=dict(sp_, snes_rtol=1e-10, ksp_rtol=1e-8))
        assert hist[-1] <= 1e-10 * hist[0]
        assert len(built) == {0: 0, 1: 1, 2: len(kits)}[len(out)], (built, kits)
        out.append(u.data_ro.copy())
    assert _rel(out[1], out[0]) < 1e-7 and _rel(out[2], out[0]) < 1e-7
