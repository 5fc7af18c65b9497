"""The CPU oracle of Neo-Hookean hyperelasticity (tests/_hyperelastic_oracle.py) against what the form
must satisfy: the residual is the gradient of the discrete energy, the Jacobian is the residual's
derivative (a Taylor test) and is symmetric, at u = 0 it is the linear elasticity operator, a rigid
rotation has zero residual and the rotated rigid modes span the Jacobian's kernel, and a homogeneous
deformation is reproduced by Newton with quadratic convergence.  The generic wrapper path's
``hyperelasticity_kernel`` is checked against it through its host build."""
import numpy as np
import pytest

import _elasticity_oracle as eo
import _hyperelastic_oracle as ho
import _mock_engine as me
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

MU, LMBDA = 1.3, 2.1


def _geo(mesh, V):
    return (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)


def _smooth(Xn, amp=0.1):
    """A smooth displacement with det F > 0 everywhere (flat AoS)."""
    x, y, z = Xn.T
    return amp * np.stack([np.sin(1.3 * x + 0.4 * y) * z, np.cos(0.7 * y - z) * x, x * y + 0.3 * np.sin(z)],
                          axis=1).ravel()


def _problem(p, seed=1):
    mesh = ExtrudedHexMesh(2, 2, 2, warp=0.06, permute_seed=seed)
    V = mesh.function_space(p)
    return mesh, V, interval_element(p), _geo(mesh, V)


@pytest.mark.parametrize("p", [1, 2])
def test_residual_is_the_energy_gradient(p):
    mesh, V, el, geo = _problem(p)
    u = _smooth(V.dof_coordinates())
    R = ho.residual(el, mesh.coordinates, u, *geo, MU, LMBDA, 0.3)
    rng = np.random.default_rng(2)
    h = 1e-5
    for _ in range(4):
        w = rng.standard_normal(len(u))
        dE = (ho.energy(el, mesh.coordinates, u + h * w, geo, MU, LMBDA, 0.3)
              - ho.energy(el, mesh.coordinates, u - h * w, geo, MU, LMBDA, 0.3)) / (2 * h)
        assert abs(dE - R @ w) < 1e-8 * np.abs(R).sum() * np.abs(w).max()


@pytest.mark.parametrize("p", [1, 2])
def test_taylor_rate_is_two(p):
    mesh, V, el, geo = _problem(p)
    u = _smooth(V.dof_coordinates())
    w = np.random.default_rng(3).standard_normal(len(u)) * 0.1
    res = lambda v: ho.residual(el, mesh.coordinates, v, *geo, MU, LMBDA, 0.2)
    Jw = ho.jacobian_action(el, mesh.coordinates, u, w, *geo, MU, LMBDA, 0.2)
    e = [np.abs(res(u + h * w) - res(u) - h * Jw).max() for h in (1e-2, 5e-3, 2.5e-3)]
    rates = np.log2(np.array(e[:-1]) / np.array(e[1:]))
    assert np.all(np.abs(rates - 2.0) < 0.1), (e, rates)


@pytest.mark.parametrize("p", [1, 2, 3])
def test_jacobian_at_zero_is_linear_elasticity(p):
    mesh, V, el, geo = _problem(p)
    di, A = ho.element_matrices(el, mesh.coordinates, np.zeros(3 * V.node_count), *geo, MU, LMBDA, 0.4)
    di2, A2 = eo.element_matrices(el, mesh.coordinates, *geo, MU, LMBDA, 0.4)
    assert np.array_equal(di, di2)
    assert np.abs(A - A2).max() < 1e-13 * np.abs(A2).max()


@pytest.mark.parametrize("p", [1, 2])
def test_element_jacobians_are_symmetric(p):
    mesh, V, el, geo = _problem(p)
    _, A = ho.element_matrices(el, mesh.coordinates, _smooth(V.dof_coordinates(), 0.2), *geo, MU, LMBDA, 0.0)
    for Ac in A:
        assert np.abs(Ac - Ac.T).max() < 1e-13 * np.abs(Ac).max()


@pytest.mark.parametrize("p", [1, 2])
def test_rigid_rotation(p):
    """u = (Q - I) X for a 60 degree rotation, beta = 0: zero residual, and J(u) maps the translations
    and the rotated infinitesimal rotations S Q X to zero."""
    mesh, V, el, geo = _problem(p, 3)
    Xn = V.dof_coordinates()
    Q = ho.rotation((1.0, 0.5, -0.3), np.pi / 3)
    u = (Xn @ Q.T - Xn).ravel()
    R = ho.residual(el, mesh.coordinates, u, *geo, MU, LMBDA, 0.0)
    scale = np.abs(ho.residual(el, mesh.coordinates, _smooth(Xn), *geo, MU, LMBDA, 0.0)).max() / 0.1
    assert np.abs(R).max() < 1e-13 * scale
    K = ho.global_jacobian(el, mesh.coordinates, u, geo, MU, LMBDA, 0.0)
    nK = np.abs(K).max()
    for r in ho.rotated_rigid_modes(Xn, Q):
        assert np.abs(K @ r).max() < 1e-12 * nK * np.abs(r).max()


@pytest.mark.parametrize("p", [1, 2])
def test_newton_reproduces_a_homogeneous_deformation(p):
    """u* = (A - I) X prescribed on the boundary, zero load: Newton recovers u* at every node and its
    last steps converge quadratically."""
    mesh = ExtrudedHexMesh(3, 3, 3, warp=0.05, permute_seed=4)
    V = mesh.function_space(p)
    el, geo = interval_element(p), _geo(mesh, V)
    A = ho.HOMOGENEOUS_A
    Xn = V.dof_coordinates()
    ue = (Xn @ A.T - Xn).ravel()
    bn = np.unique(np.concatenate([V.boundary_nodes(s) for s in (1, 2, 3, 4, "bottom", "top")]))
    bd = (3 * bn[:, None] + np.arange(3)).ravel()
    u0 = np.zeros_like(ue)
    u0[bd] = ue[bd]
    u, hist = ho.newton(el, mesh.coordinates, geo, MU, LMBDA, 0.0, np.zeros_like(ue), u0, bd, rtol=1e-14)
    assert np.abs(u - ue).max() < 1e-12
    assert ho.converges_quadratically(hist), hist


@pytest.mark.parametrize("p", [1, 2, 3])
@pytest.mark.parametrize("jacobian", [False, True], ids=["residual", "jacobian"])
def test_generic_path_matches_oracle(oracle, p, jacobian):
    """``assemble_hyperelasticity_generic`` (generated wrapper around ``hyperelasticity_kernel``, run
    through its host build by the mock engine) against the oracle."""
    from firedrake_b200.assemble import FunctionSpace, assemble_hyperelasticity_generic
    mesh = ExtrudedHexMesh(3, 2, 3, warp=0.06, permute_seed=2)
    V0 = mesh.function_space(p)
    u0 = _smooth(V0.dof_coordinates())
    w0 = np.random.default_rng(4).standard_normal(3 * V0.node_count)
    el, geo = interval_element(p), _geo(mesh, V0)
    if jacobian:
        y = ho.jacobian_action(el, mesh.coordinates, u0, w0, *geo, MU, LMBDA, 0.5)
    else:
        y = ho.residual(el, mesh.coordinates, u0, *geo, MU, LMBDA, 0.5)
    with me.install(oracle):
        V = FunctionSpace(mesh, p, 3)
        u = V.dat(u0.reshape(-1, 3).copy())
        w = V.dat(w0.reshape(-1, 3).copy()) if jacobian else None
        yg = assemble_hyperelasticity_generic(V, u, MU, LMBDA, 0.5, w=w).data_ro.copy()
    assert np.abs(y - yg.ravel()).max() < 1e-12 * np.abs(y).max()
