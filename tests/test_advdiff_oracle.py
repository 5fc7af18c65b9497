"""The CPU oracle of advection-diffusion alpha*inner(grad u, grad v)*dx + inner(dot(b, grad u), v)*dx +
beta*inner(u, v)*dx (tests/_advdiff_oracle.py) against independent statements of the same integrals: the
coefficient oracle at kappa = 1 for b = 0, the structure of the convective term (it annihilates constants;
for a divergence-free b tangent to the boundary it is skew on the interior), a dense quadrature, and the
generic wrapper path's ``advection_diffusion_kernel`` through its host build."""
import numpy as np
import pytest

import _advdiff_oracle as ao
import _coef_oracle as co
import _mock_engine as me
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh


def _mesh(p, seed=1, warp=0.06):
    mesh = ExtrudedHexMesh(3, 2, 4, warp=warp, permute_seed=seed)
    return mesh, mesh.function_space(p)


def _args(mesh, V):
    return (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)


def _b(V, seed=0):
    """A varying velocity with noise (b need not be smooth or divergence-free), 3 values per node."""
    X = V.dof_coordinates()
    rng = np.random.default_rng(seed)
    b = np.stack([1.0 + np.sin(2.0 * X[:, 1]), X[:, 0] * X[:, 2] - 0.5, 0.7 * np.cos(X[:, 0])], axis=1)
    return (b + 0.1 * rng.standard_normal(b.shape)).ravel()


def rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_zero_velocity_is_the_coefficient_oracle_at_kappa_one(p):
    mesh, V = _mesh(p)
    el = interval_element(p)
    u = np.random.default_rng(3).standard_normal(V.node_count)
    y = ao.action(el, mesh.coordinates, u, np.zeros(3 * V.node_count), *_args(mesh, V), alpha=0.7, beta=1.3)
    yc = co.action(el, mesh.coordinates, u, np.ones(V.node_count), *_args(mesh, V), alpha=0.7, beta=1.3)
    assert rel(y, yc) < 1e-14


@pytest.mark.parametrize("p", [1, 2, 3])
def test_convective_element_matrices_annihilate_constants(p):
    mesh, V = _mesh(p, seed=2)
    el = interval_element(p)
    _, C = ao.element_matrices(el, mesh.coordinates, _b(V), *_args(mesh, V), convective_only=True)
    assert np.abs(C.sum(axis=2)).max() < 1e-13 * np.abs(C).max()
    # and the full operator minus its symmetric part is the convective part
    _, A = ao.element_matrices(el, mesh.coordinates, _b(V), *_args(mesh, V), alpha=1.1, beta=0.4)
    _, S = ao.element_matrices(el, mesh.coordinates, np.zeros(3 * V.node_count), *_args(mesh, V),
                               alpha=1.1, beta=0.4)
    assert np.abs(A - S - C).max() < 1e-13 * np.abs(A).max()


@pytest.mark.parametrize("p", [1, 2])
def test_divergence_free_velocity_gives_a_skew_interior_block(p):
    """b = (-(y - 1/2), x - 1/2, 0) on the unit cube is divergence-free and exactly representable, and the
    Gauss rule integrates the convective term exactly on an unwarped mesh.  Integration by parts:
    (C + C^T)_ij = -int div(b) phi_i phi_j + int_boundary (b.n) phi_i phi_j, and both vanish when neither
    dof lies on the boundary."""
    mesh = ExtrudedHexMesh(3, 3, 3)
    V = mesh.function_space(p)
    X = V.dof_coordinates()
    b = np.stack([-(X[:, 1] - 0.5), X[:, 0] - 0.5, np.zeros(len(X))], axis=1).ravel()
    C = ao.csr(interval_element(p), mesh.coordinates, b, *_args(mesh, V), convective_only=True).toarray()
    bnd = np.unique(np.concatenate([V.boundary_nodes(s) for s in (1, 2, 3, 4, "bottom", "top")]))
    inner = np.setdiff1d(np.arange(V.node_count), bnd)
    S = (C + C.T)[np.ix_(inner, inner)]
    assert np.abs(C).max() > 1e-3
    assert np.abs(S).max() < 1e-14 * np.abs(C).max()


def test_dense_quadrature_on_one_warped_cell():
    """One trilinear cell, the bilinear form by brute force: every basis function tabulated at every
    quadrature point (no sum factorisation), Jacobian from the vertex formula."""
    p = 3
    el = interval_element(p)
    n = p + 1
    rng = np.random.default_rng(7)
    X = np.array([[bx, by, bz] for bx in (0, 1) for by in (0, 1) for bz in (0, 1)], dtype=float)
    X = X * [1.0, 0.8, 1.2] + 0.12 * rng.standard_normal((8, 3))
    bn = rng.standard_normal((n ** 3, 3))
    alpha, beta = 1.3, 0.6
    B, D, w, xq = el.B, el.D, el.wq, el.xq
    A = np.zeros((n ** 3, n ** 3))
    for qx in range(n):
        for qy in range(n):
            for qz in range(n):
                xi = (xq[qx], xq[qy], xq[qz])
                J = np.zeros((3, 3))
                for v in range(8):
                    bv = ((v >> 2) & 1, (v >> 1) & 1, v & 1)
                    for d in range(3):
                        g = 1.0 if bv[d] else -1.0
                        for e in range(3):
                            if e != d:
                                g *= xi[e] if bv[e] else 1.0 - xi[e]
                        J[:, d] += X[v] * g
                phi = np.einsum("a,b,c->abc", B[qx], B[qy], B[qz]).ravel()
                gref = np.stack([np.einsum("a,b,c->abc", D[qx], B[qy], B[qz]).ravel(),
                                 np.einsum("a,b,c->abc", B[qx], D[qy], B[qz]).ravel(),
                                 np.einsum("a,b,c->abc", B[qx], B[qy], D[qz]).ravel()], axis=1)
                gphys = gref @ np.linalg.inv(J)                  # rows: grad phi_j
                wq = w[qx] * w[qy] * w[qz] * abs(np.linalg.det(J))
                bq = phi @ bn
                # row = test i, column = trial j
                A += wq * (alpha * gphys @ gphys.T + np.outer(phi, gphys @ bq) + beta * np.outer(phi, phi))
    Ao = ao.cell_matrices(el, X[None], bn[None], alpha, beta)[0]
    assert np.abs(Ao - A).max() < 1e-13 * np.abs(A).max()
    assert np.abs(A - A.T).max() > 1e-3 * np.abs(A).max()          # not symmetric


@pytest.mark.parametrize("p", [1, 2, 3])
def test_matrix_diagonal_and_csr_agree_with_the_action(p):
    mesh, V = _mesh(p, seed=5)
    el = interval_element(p)
    b = _b(V, seed=1)
    u = np.random.default_rng(6).standard_normal(V.node_count)
    A = ao.csr(el, mesh.coordinates, b, *_args(mesh, V), alpha=0.9, beta=0.3)
    y = ao.action(el, mesh.coordinates, u, b, *_args(mesh, V), alpha=0.9, beta=0.3)
    assert rel(A @ u, y) < 1e-13
    d = ao.diagonal(el, mesh.coordinates, b, *_args(mesh, V), alpha=0.9, beta=0.3)
    assert rel(d, A.diagonal()) < 1e-14


def test_generic_statement_refuses_degree_4():
    from firedrake_b200.assemble import advection_diffusion_kernel
    with pytest.raises(NotImplementedError, match="degree 4 outside 1..3"):
        advection_diffusion_kernel(4)


@pytest.mark.parametrize("p", [1, 2, 3])
@pytest.mark.parametrize("beta", [0.0, 0.8])
def test_generic_path_host_build_matches_the_oracle(oracle, p, beta):
    """``assemble_advection_diffusion_generic`` (the generated wrapper around ``advection_diffusion_kernel``,
    run through its host build by the mock engine) is the generic-path statement of the same form."""
    from firedrake_b200.assemble import FunctionSpace, assemble_advection_diffusion_generic
    mesh, V0 = _mesh(p, seed=2)
    el = interval_element(p)
    u0 = np.random.default_rng(4).standard_normal(V0.node_count)
    b0 = _b(V0, seed=3)
    y = ao.action(el, mesh.coordinates, u0, b0, *_args(mesh, V0), alpha=1.2, beta=beta)
    with me.install(oracle):
        V = FunctionSpace(mesh, p)
        b = V.vector_dset(3)
        from firedrake_b200 import op2
        yg = assemble_advection_diffusion_generic(V, V.dat(u0.copy()), op2.Dat(b, b0.copy()), alpha=1.2,
                                                  beta=beta).data_ro.copy()
    assert rel(y, yg) < 1e-12


def test_scipy_solve_of_a_manufactured_problem_converges():
    """-div grad u + b.grad u = f with u = sin(pi x) sin(pi y) sin(pi z) and b = (1, 0.5, 0.25): the
    oracle's matrix and scipy's LU give the L2 interpolation error's second-order rate at CG1."""
    errs = []
    for nx in (8, 16):
        mesh = ExtrudedHexMesh(nx, nx, nx)
        V = mesh.function_space(1)
        X = V.dof_coordinates()
        el = interval_element(1)
        s = lambda t: np.sin(np.pi * t)
        c = lambda t: np.cos(np.pi * t)
        ue = s(X[:, 0]) * s(X[:, 1]) * s(X[:, 2])
        f = (3 * np.pi ** 2 * ue + np.pi * (1.0 * c(X[:, 0]) * s(X[:, 1]) * s(X[:, 2])
                                            + 0.5 * s(X[:, 0]) * c(X[:, 1]) * s(X[:, 2])
                                            + 0.25 * s(X[:, 0]) * s(X[:, 1]) * c(X[:, 2])))
        b = np.tile([1.0, 0.5, 0.25], V.node_count)
        args = _args(mesh, V)
        A = ao.csr(el, mesh.coordinates, b, *args)
        rhs = co.action(el, mesh.coordinates, f, np.zeros(V.node_count), *args, alpha=0.0, beta=1.0)
        bnd = np.unique(np.concatenate([V.boundary_nodes(s_) for s_ in (1, 2, 3, 4, "bottom", "top")]))
        u = ao.solve(A, rhs, bnd, 0.0)
        e = u - ue
        Me = co.action(el, mesh.coordinates, e, np.zeros(V.node_count), *args, alpha=0.0, beta=1.0)
        errs.append(np.sqrt(e @ Me))
    assert np.log2(errs[0] / errs[1]) > 1.8, errs
