"""The CPU oracle of Stokes flow on Taylor-Hood hexahedra (tests/_stokes_oracle.py) against independent
statements of the same integrals: the coefficient oracle for the velocity block, the divergence structure
(exact quadrature of the div terms on warped cells), symmetry, a dense quadrature, the constrained system's
nullspace, and the generic wrapper path's ``stokes_kernel`` through its host build."""
import numpy as np
import pytest

import _coef_oracle as co
import _mock_engine as me
import _stokes_oracle as so
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

ALL_FACES = (1, 2, 3, 4, "bottom", "top")


def _setup(p, n=(3, 2, 4), warp=0.08, seed=1):
    mesh = ExtrudedHexMesh(*n, warp=warp, permute_seed=seed)
    V, Q = mesh.function_space(p), mesh.function_space(p - 1)
    geo = (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    return mesh, V, Q, geo, (Q.cell_node_map, Q.offset)


def _K(p, mu=1.3, beta=0.0, **kw):
    mesh, V, Q, geo, geo2 = _setup(p, **kw)
    return mesh, V, Q, so.global_matrix(interval_element(p), mesh.coordinates, geo, geo2, V.node_count,
                                        Q.node_count, mu, beta)


@pytest.mark.parametrize("p", [2, 3, 4])
def test_velocity_block_is_three_scalar_helmholtz_blocks(p):
    mesh, V, Q, geo, geo2 = _setup(p)
    K = so.global_matrix(interval_element(p), mesh.coordinates, geo, geo2, V.node_count, Q.node_count, 1.3, 0.6)
    A, _, _, _ = so.blocks(K, V.node_count)
    x = np.random.default_rng(0).standard_normal((V.node_count, 3))
    want = np.stack([co.action(interval_element(p), mesh.coordinates, x[:, c].copy(), np.ones(V.node_count),
                               *geo, alpha=1.3, beta=0.6) for c in range(3)], axis=1)
    assert np.abs(A @ x.ravel() - want.ravel()).max() < 1e-13 * np.abs(want).max()


@pytest.mark.parametrize("p", [2, 3, 4])
def test_gradient_of_a_constant_pressure_vanishes_off_the_boundary(p):
    mesh, V, Q, K = _K(p)
    _, Bt, _, _ = so.blocks(K, V.node_count)
    y = (Bt @ np.ones(Q.node_count)).reshape(-1, 3)
    bnd = np.unique(np.concatenate([V.boundary_nodes(s) for s in ALL_FACES]))
    inner = np.setdiff1d(np.arange(V.node_count), bnd)
    assert np.abs(y).max() > 0.0
    assert np.abs(y[inner]).max() < 1e-13 * np.abs(y).max()


@pytest.mark.parametrize("p", [2, 3, 4])
def test_linear_divergence_free_field_has_zero_pressure_rows(p):
    mesh, V, Q, K = _K(p)
    _, _, B, _ = so.blocks(K, V.node_count)
    X = V.dof_coordinates()
    u = np.stack([X[:, 0], X[:, 1], -2.0 * X[:, 2]], axis=1).ravel()
    ref = np.abs(B @ X.ravel()).max()
    assert np.abs(B @ u).max() < 1e-13 * ref


@pytest.mark.parametrize("p", [2, 3])
def test_saddle_matrix_is_symmetric_with_zero_pressure_block(p):
    _, V, Q, K = _K(p, beta=0.4)
    assert abs(K - K.T).max() < 1e-14 * abs(K).max()
    _, _, _, C = so.blocks(K, V.node_count)
    assert C.nnz == 0 or abs(C).max() == 0.0


@pytest.mark.parametrize("p", [2, 3])
def test_dense_quadrature(p):
    """On affine (stretched, unwarped) cells every term is a polynomial the (p+1)-point rule integrates
    exactly; on warped cells the div terms still are.  A (p+3)-point rule gives the same action."""
    for warp, full in ((0.0, True), (0.08, False)):
        mesh, V, Q, geo, geo2 = _setup(p, warp=warp)
        rng = np.random.default_rng(2)
        u, pr = rng.standard_normal(3 * V.node_count), rng.standard_normal(Q.node_count)
        mu = 1.1 if full else 0.0
        y = so.action(interval_element(p), mesh.coordinates, u, pr, geo, geo2, mu, 0.7 if full else 0.0)
        yd = so.action(interval_element(p, p + 3), mesh.coordinates, u, pr, geo, geo2, mu, 0.7 if full else 0.0)
        for a, b in zip(y, yd):
            assert np.abs(a - b).max() < 1e-12 * np.abs(b).max()


def test_constrained_nullspace_is_the_constant_pressure():
    """3^3 cells, all-Dirichlet velocity, Q2-Q1: the constrained saddle matrix has exactly one null vector,
    the constant pressure (a wrong Bq or wrong pressure offsets would add checkerboard modes)."""
    mesh, V, Q, K = _K(2, n=(3, 3, 3), warp=0.05)
    bnd = np.unique(np.concatenate([V.boundary_nodes(s) for s in ALL_FACES]))
    Kc = so.constrained(K, so.velocity_dofs(bnd)).toarray()
    s, vec = np.linalg.eigh(Kc)
    small = np.abs(s) < 1e-10 * np.abs(s).max()
    assert small.sum() == 1
    v = vec[:, np.argmin(np.abs(s))]
    nv = 3 * V.node_count
    assert np.abs(v[:nv]).max() < 1e-10
    assert np.ptp(v[nv:]) < 1e-10 * np.abs(v[nv:]).max()


@pytest.mark.parametrize("p", [2, 3])
@pytest.mark.parametrize("beta", [0.0, 0.8])
def test_generic_path_host_build_matches_the_oracle(oracle, p, beta):
    from firedrake_b200.assemble import FunctionSpace, Stokes, assemble_stokes_generic
    mesh, V0, Q0, geo, geo2 = _setup(p, seed=2)
    rng = np.random.default_rng(4)
    u0, p0 = rng.standard_normal((V0.node_count, 3)), rng.standard_normal(Q0.node_count)
    want = so.action(interval_element(p), mesh.coordinates, u0.ravel(), p0, geo, geo2, 1.2, beta)
    with me.install(oracle):
        F = Stokes(FunctionSpace(mesh, p, 3), FunctionSpace(mesh, p - 1), 1.2, beta)
        y = [d.data_ro.copy() for d in assemble_stokes_generic(F, F.dat(u0.copy(), p0.copy()))]
    assert np.abs(y[0].ravel() - want[0]).max() < 1e-12 * np.abs(want[0]).max()
    assert np.abs(y[1] - want[1]).max() < 1e-12 * np.abs(want[1]).max()


def test_stokes_form_refusals():
    from firedrake_b200.assemble import FunctionSpace, Stokes, stokes_kernel
    mesh = ExtrudedHexMesh(2, 2, 2)
    with pytest.raises(ValueError, match="3 components"):
        Stokes(FunctionSpace(mesh, 2), FunctionSpace(mesh, 1))
    with pytest.raises(ValueError, match="scalar"):
        Stokes(FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1, 3))
    with pytest.raises(ValueError, match="same mesh"):
        Stokes(FunctionSpace(mesh, 2, 3), FunctionSpace(ExtrudedHexMesh(2, 2, 2), 1))
    with pytest.raises(ValueError, match="p = 2..4"):
        Stokes(FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 2))
    with pytest.raises(ValueError, match="p = 2..4"):
        Stokes(FunctionSpace(mesh, 5, 3), FunctionSpace(mesh, 4))
    with pytest.raises(NotImplementedError, match="degrees 2..4"):
        stokes_kernel(5)
