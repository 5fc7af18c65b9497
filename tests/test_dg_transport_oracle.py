"""CPU checks of the upwind DG transport oracle (tests/_dg_transport_oracle.py) and of DGTransport's refusals:
exact conservation, free-stream preservation, the diffusion part against the interior penalty oracle, and the
diagonal."""
import numpy as np
import pytest

import _boundary_oracle as bo
import _dg_oracle as do
import _dg_transport_oracle as to
from firedrake_b200.utility_meshes import ExtrudedHexMesh


def warped(seed=0):
    return bo.perturb(ExtrudedHexMesh(3, 2, 3, Lx=1.2, Ly=0.9, Lz=1.1, warp=0.05, permute_seed=seed), 0.08, seed)


def parallelepipeds():
    mesh = ExtrudedHexMesh(3, 2, 2, permute_seed=3)
    S = np.array([[1.0, 0.25, 0.125], [0.0, 1.25, -0.25], [0.125, 0.0, 0.75]])
    mesh.coordinates[:] = mesh.coordinates @ S.T
    return mesh


@pytest.mark.parametrize("p", [1, 2, 3])
def test_conservation(p):
    """1^T A q is the outflow flux exactly, for random b and q on a warped mesh: the cell term integrates grad 1 = 0
    and every interior flux enters both sides with opposite signs."""
    mesh = warped(p)
    W = mesh.dg_function_space(p)
    el = do.element(p)
    rng = np.random.default_rng(p)
    bv = rng.standard_normal((mesh.coord_space.node_count, 3))
    q = rng.standard_normal(W.node_count)
    A = to.operator(mesh, W, el, bv)
    out = to.outflow_integral(mesh, W, el, bv, q)
    assert abs(np.ones(W.node_count) @ (A @ q) - out) < 1e-12 * np.abs(A @ q).sum()


@pytest.mark.parametrize("p", [1, 2, 3])
def test_free_stream_preservation(p):
    """A constant field in a constant flow on a parallelepiped mesh: A 1 = inflow_load(1)."""
    mesh = parallelepipeds()
    W = mesh.dg_function_space(p)
    el = do.element(p)
    bv = np.tile([0.7, -0.4, 0.3], (mesh.coord_space.node_count, 1))
    one = np.ones(W.node_count)
    r = to.operator(mesh, W, el, bv) @ one
    g = to.inflow_load(mesh, W, el, bv, one)
    assert np.abs(r - g).max() < 1e-12 * np.abs(g).max()


@pytest.mark.parametrize("p", [1, 2])
def test_diffusion_part_is_interior_penalty(p):
    mesh = warped(10 + p)
    W = mesh.dg_function_space(p)
    el = do.element(p)
    eta = 3.0 * (p + 1) ** 2
    A = to.operator(mesh, W, el, np.zeros((mesh.coord_space.node_count, 3)), 0.4, 1.3, eta, (1, "top"))
    B = do.operator(mesh, W, el, 1.3, 0.4, eta, (1, "top"))
    assert abs(A - B).max() < 1e-12 * abs(B).max()


def test_upwind_and_diagonal():
    """The interior flux takes the upwind trace, so the transport part of A is not symmetric, and its diagonal
    is max(+-b.n, 0) phi^2 W on the facets plus -w |det J| b.grad phi_i(x_i) on the cells."""
    mesh = warped(5)
    W = mesh.dg_function_space(2)
    el = do.element(2)
    bv = np.random.default_rng(5).standard_normal((mesh.coord_space.node_count, 3))
    Ai = to.interior_matrix(mesh, W, el, bv)
    assert abs(Ai - Ai.T).max() > 1e-3
    assert np.all(Ai.diagonal() >= 0.0)
    A = to.operator(mesh, W, el, bv)
    assert np.all(np.isfinite(A.diagonal()))


def test_refusals():
    from firedrake_b200 import op2
    from firedrake_b200.assemble import DGTransport, FunctionSpace
    mesh = ExtrudedHexMesh(2, 2, 2)
    V = FunctionSpace(mesh, 1, family="DQ")
    b = op2.Dat(op2.DataSet(V.vertex_set, 3), np.zeros((mesh.coord_space.node_count, 3)))
    with pytest.raises(ValueError, match="DQ space"):
        DGTransport(FunctionSpace(mesh, 1), b)
    with pytest.raises(ValueError, match="3 values per mesh vertex"):
        DGTransport(V, op2.Dat(op2.DataSet(V.vertex_set, 1), np.zeros(mesh.coord_space.node_count)))
    with pytest.raises(ValueError, match="3 values per mesh vertex"):
        DGTransport(V, op2.Dat(V.vector_dset(3), np.zeros((V.node_count, 3))))
    with pytest.raises(ValueError, match="needs the interior penalty eta"):
        DGTransport(V, b, alpha=1.0)
    with pytest.raises(ValueError, match="alpha must be >= 0"):
        DGTransport(V, b, alpha=-1.0, eta=12.0)
    with pytest.raises(ValueError, match="need alpha > 0"):
        DGTransport(V, b, weak_bcs="on_boundary")
    F = DGTransport(V, b)
    assert F.symmetric is False
    with pytest.raises(NotImplementedError, match="no assembled matrix"):
        F.kernel(2)
