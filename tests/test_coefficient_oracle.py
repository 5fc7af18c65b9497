"""The CPU oracle of the coefficient form alpha*inner(kappa*grad u, grad v)*dx + beta*inner(u, v)*dx
(tests/_coef_oracle.py) against three independent statements of the same integrals: the
constant-coefficient oracle (oracle/hex_kernels.inc) for a constant kappa, the generic wrapper path's
``variable_coefficient_kernel`` through its host build for a varying kappa, and a dense quadrature."""
import numpy as np
import pytest

import _coef_oracle as co
import _mock_engine as me
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh


def _mesh(p, seed=1):
    mesh = ExtrudedHexMesh(3, 2, 4, warp=0.06, permute_seed=seed)
    return mesh, mesh.function_space(p)


def _kappa(V, seed=0):
    """A smooth positive field through the node coordinates, plus noise (kappa need not be smooth)."""
    X = V.dof_coordinates()
    rng = np.random.default_rng(seed)
    return 2.0 + np.sin(3.0 * X[:, 0]) * X[:, 1] + 0.3 * X[:, 2] + 0.1 * rng.random(len(X))


def _args(mesh, V):
    return (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)


def rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (0.7, 1.3)])
def test_constant_kappa_is_the_scaled_helmholtz_oracle(oracle, p, alpha, beta):
    mesh, V = _mesh(p)
    el = interval_element(p)
    u = np.random.default_rng(3).standard_normal(V.node_count)
    c = 2.5
    y = co.action(el, mesh.coordinates, u, np.full(V.node_count, c), *_args(mesh, V), alpha=alpha, beta=beta)
    yo = np.zeros(V.node_count)
    oracle.action_extruded(el, 0, mesh.num_base_cells, [0, mesh.layers], yo, mesh.coordinates, u,
                           V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, alpha=alpha * c, beta=beta)
    assert rel(y, yo) < 1e-13


@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("beta", [0.0, 0.8])
def test_varying_kappa_matches_the_generic_path(oracle, p, beta):
    """``assemble_variable_coefficient`` (generated wrapper around ``variable_coefficient_kernel``,
    run through its host build by the mock engine) is the generic-path statement of the same form."""
    from firedrake_b200.assemble import FunctionSpace, assemble_variable_coefficient
    mesh, V0 = _mesh(p, seed=2)
    el = interval_element(p)
    u0 = np.random.default_rng(4).standard_normal(V0.node_count)
    k0 = _kappa(V0)
    y = co.action(el, mesh.coordinates, u0, k0, *_args(mesh, V0), beta=beta)
    with me.install(oracle):
        V = FunctionSpace(mesh, p)
        yg = assemble_variable_coefficient(V, V.dat(k0.copy()), V.dat(u0.copy()), beta=beta).data_ro.copy()
    assert rel(y, yg) < 1e-12


def test_dense_quadrature_on_one_warped_cell():
    """One trilinear cell, the bilinear form by brute force: every basis function tabulated at every
    quadrature point (no sum factorisation), Jacobian from the vertex formula."""
    p = 3
    el = interval_element(p)
    n = p + 1
    rng = np.random.default_rng(7)
    X = np.array([[bx, by, bz] for bx in (0, 1) for by in (0, 1) for bz in (0, 1)], dtype=float)
    X = X * [1.0, 0.8, 1.2] + 0.12 * rng.standard_normal((8, 3))
    kap = 1.0 + rng.random(n ** 3)
    alpha, beta = 1.3, 0.6
    B, D, w, xq = el.B, el.D, el.wq, el.xq
    A = np.zeros((n ** 3, n ** 3))
    for qx in range(n):
        for qy in range(n):
            for qz in range(n):
                xi = (xq[qx], xq[qy], xq[qz])
                J = np.zeros((3, 3))
                for v in range(8):
                    b = ((v >> 2) & 1, (v >> 1) & 1, v & 1)
                    for d in range(3):
                        g = 1.0 if b[d] else -1.0
                        for e in range(3):
                            if e != d:
                                g *= xi[e] if b[e] else 1.0 - xi[e]
                        J[:, d] += X[v] * g
                phi = np.einsum("a,b,c->abc", B[qx], B[qy], B[qz]).ravel()
                gref = np.stack([np.einsum("a,b,c->abc", D[qx], B[qy], B[qz]).ravel(),
                                 np.einsum("a,b,c->abc", B[qx], D[qy], B[qz]).ravel(),
                                 np.einsum("a,b,c->abc", B[qx], B[qy], D[qz]).ravel()], axis=1)
                gphys = gref @ np.linalg.inv(J)                  # rows: grad phi_i
                wq = w[qx] * w[qy] * w[qz] * abs(np.linalg.det(J))
                A += wq * (alpha * (phi @ kap) * gphys @ gphys.T + beta * np.outer(phi, phi))
    Ao = co.cell_matrices(el, X[None], kap[None], alpha, beta)[0]
    assert np.abs(Ao - A).max() < 1e-13 * np.abs(A).max()


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_element_matrix_symmetry_action_and_diagonal(p):
    mesh, V = _mesh(p, seed=5)
    el = interval_element(p)
    k = _kappa(V, seed=1)
    i0, A = co.element_matrices(el, mesh.coordinates, k, *_args(mesh, V), alpha=1.0, beta=0.4)
    assert np.abs(A - np.swapaxes(A, 1, 2)).max() < 1e-14 * np.abs(A).max()
    u = np.random.default_rng(6).standard_normal(V.node_count)
    y = np.zeros(V.node_count)
    np.add.at(y, i0, np.einsum("cij,cj->ci", A, u[i0]))
    assert rel(y, co.action(el, mesh.coordinates, u, k, *_args(mesh, V), alpha=1.0, beta=0.4)) < 1e-13
    d = co.diagonal(el, mesh.coordinates, k, *_args(mesh, V), alpha=1.0, beta=0.4)
    dd = np.zeros(V.node_count)
    np.add.at(dd, i0, np.diagonal(A, axis1=1, axis2=2))
    assert np.array_equal(d, dd)
