"""The CPU oracle of nonlinear diffusion (tests/_nonlinear_oracle.py) against the coefficient-form
oracle and the constant-coefficient C oracle, a Taylor test of its Jacobian, the (non)symmetry of its
element matrices and the quadratic convergence of its Newton solve."""
import numpy as np
import pytest

import _coef_oracle as co
import _nonlinear_oracle as no
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh


def _mesh(p, seed=1):
    mesh = ExtrudedHexMesh(3, 2, 4, warp=0.06, permute_seed=seed)
    return mesh, mesh.function_space(p)


def _geo(mesh, V):
    return (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)


def rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def _u(V, seed=0):
    X = V.dof_coordinates()
    return np.sin(2.0 * X[:, 0]) * X[:, 1] + X[:, 2] + 0.2 * np.random.default_rng(seed).standard_normal(len(X))


@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("beta", [0.0, 0.6])
def test_linear_diffusivity_is_the_coefficient_form(p, beta):
    """d2 = 0: D(u_q) is exactly the interpolant of d0 + d1*u, i.e. the coefficient form's kappa."""
    mesh, V = _mesh(p)
    el = interval_element(p)
    u = _u(V, p)
    d = (1.5, 0.7, 0.0)
    y = no.residual(el, mesh.coordinates, u, *_geo(mesh, V), d, alpha=1.2, beta=beta)
    yc = co.action(el, mesh.coordinates, u, d[0] + d[1] * u, *_geo(mesh, V), alpha=1.2, beta=beta)
    assert rel(y, yc) < 1e-13


@pytest.mark.parametrize("p", [1, 2, 3])
def test_unit_diffusivity_is_the_helmholtz_oracle(oracle, p):
    mesh, V = _mesh(p, seed=2)
    el = interval_element(p)
    u = _u(V, 3)
    y = no.residual(el, mesh.coordinates, u, *_geo(mesh, V), (1.0, 0.0, 0.0), alpha=0.9, beta=0.4)
    yo = np.zeros(V.node_count)
    oracle.action_extruded(el, 0, mesh.num_base_cells, [0, mesh.layers], yo, mesh.coordinates, u,
                           V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, alpha=0.9, beta=0.4)
    assert rel(y, yo) < 1e-13


def taylor_errors(R, J, u, w, hs):
    """||(R(u + h w) - R(u - h w)) / 2h - J w||_inf for each h."""
    Jw = J(u, w)
    return np.array([np.abs((R(u + h * w) - R(u - h * w)) / (2.0 * h) - Jw).max() for h in hs])


@pytest.mark.parametrize("p", [1, 2, 3])
def test_jacobian_taylor_ratio_is_four(p):
    mesh, V = _mesh(p, seed=3)
    el = interval_element(p)
    geo = _geo(mesh, V)
    d = (1.0, 0.3, 0.25)
    u, w = _u(V, 4), np.random.default_rng(5).standard_normal(V.node_count)
    R = lambda x: no.residual(el, mesh.coordinates, x, *geo, d, alpha=1.1, beta=0.5)
    J = lambda x, v: no.jacobian_action(el, mesh.coordinates, x, v, *geo, d, alpha=1.1, beta=0.5)
    e = taylor_errors(R, J, u, w, [0.04, 0.02, 0.01])
    ratios = e[:-1] / e[1:]
    assert np.all((ratios > 3.6) & (ratios < 4.4)), (e, ratios)


@pytest.mark.parametrize("p", [1, 2, 3])
def test_element_matrices_symmetric_only_for_constant_diffusivity(p):
    mesh, V = _mesh(p, seed=4)
    el = interval_element(p)
    geo = _geo(mesh, V)
    u = _u(V, 6)
    for d, sym in (((1.3, 0.0, 0.0), True), ((1.0, 0.4, 0.0), False), ((1.0, 0.0, 0.3), False)):
        i0, A = no.jacobian_matrices(el, mesh.coordinates, u, *geo, d, alpha=1.0, beta=0.3)
        asym = np.abs(A - np.swapaxes(A, 1, 2)).max() / np.abs(A).max()
        assert (asym < 1e-14) if sym else (asym > 1e-3), (d, asym)
        # the matrices are the action's columns, their diagonal the diagonal
        w = np.random.default_rng(7).standard_normal(V.node_count)
        y = np.zeros(V.node_count)
        np.add.at(y, i0, np.einsum("cij,cj->ci", A, w[i0]))
        assert rel(y, no.jacobian_action(el, mesh.coordinates, u, w, *geo, d, alpha=1.0, beta=0.3)) < 1e-13
    dd = no.jacobian_diagonal(el, mesh.coordinates, u, *geo, d, alpha=1.0, beta=0.3)
    ref = np.zeros(V.node_count)
    np.add.at(ref, i0, np.diagonal(A, axis1=1, axis2=2))
    assert np.array_equal(dd, ref)


def test_oracle_newton_converges_quadratically():
    """Source f = 1 + x y z, Dirichlet u = 0.5 at the bottom and 2 at the top: each Newton error is
    about the square of the one before."""
    p = 2
    mesh, V = _mesh(p, seed=5)
    el = interval_element(p)
    geo = _geo(mesh, V)
    X = V.dof_coordinates()
    f = 1.0 + X[:, 0] * X[:, 1] * X[:, 2]
    L = co.action(el, mesh.coordinates, f, np.ones(V.node_count), *geo, alpha=0.0, beta=1.0)
    bot, top = V.boundary_nodes("bottom"), V.boundary_nodes("top")
    g = np.zeros(V.node_count)
    g[bot], g[top] = 0.5, 2.0
    d = (1.0, 0.5, 0.5)
    u, hist = no.newton(el, mesh.coordinates, geo, L, d, beta=0.3, bc_nodes=np.concatenate([bot, top]),
                        bc_values=g, rtol=1e-13)
    h = np.array(hist) / hist[0]
    assert len(h) <= 8 and h[-1] < 1e-13, h
    # quadratic: log(e_{k+1}) / log(e_k) -> 2 in the asymptotic steps
    k = np.flatnonzero(h < 1e-2)[0]
    assert h[k + 1] < 10.0 * h[k] ** 2 or h[k + 1] < 1e-13, h
