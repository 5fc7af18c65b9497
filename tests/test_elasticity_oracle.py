"""The CPU oracle of linear elasticity (tests/_elasticity_oracle.py) against independent statements of
the same integrals: a dense strain-displacement (B^T D B, Voigt notation) quadrature, the structure every
elasticity stiffness matrix has (symmetry, semidefiniteness, exactly the six rigid-body modes in its
kernel), the closed form of its diagonal, the generic wrapper path's ``elasticity_kernel`` through its
host build, and the patch test: a linear displacement field is reproduced exactly on a warped mesh."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import _elasticity_oracle as eo
import _mock_engine as me
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

MU, LMBDA = 1.3, 2.1


def _cell(seed=7):
    rng = np.random.default_rng(seed)
    X = np.array([[bx, by, bz] for bx in (0, 1) for by in (0, 1) for bz in (0, 1)], dtype=float)
    return X * [1.0, 0.8, 1.2] + 0.12 * rng.standard_normal((8, 3))


def _geo(mesh, V):
    return (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)


def _jacobian(X, xi):
    J = np.zeros((3, 3))
    for v in range(8):
        b = ((v >> 2) & 1, (v >> 1) & 1, v & 1)
        for d in range(3):
            g = 1.0 if b[d] else -1.0
            for e in range(3):
                if e != d:
                    g *= xi[e] if b[e] else 1.0 - xi[e]
            J[:, d] += X[v] * g
    return J


def dense_element_matrix(el, X, mu, lmbda, beta):
    """K = sum_q w |det J| (B^T D B + beta N^T N): every basis function tabulated at every point."""
    n = el.ndof
    nd = n ** 3
    Bt, Dt, w, xq = el.B, el.D, el.wq, el.xq
    Dm = lmbda * np.outer([1, 1, 1, 0, 0, 0], [1, 1, 1, 0, 0, 0]) + mu * np.diag([2, 2, 2, 1, 1, 1])
    K = np.zeros((3 * nd, 3 * nd))
    for qx in range(n):
        for qy in range(n):
            for qz in range(n):
                J = _jacobian(X, (xq[qx], xq[qy], xq[qz]))
                phi = np.einsum("a,b,c->abc", Bt[qx], Bt[qy], Bt[qz]).ravel()
                gref = np.stack([np.einsum("a,b,c->abc", Dt[qx], Bt[qy], Bt[qz]).ravel(),
                                 np.einsum("a,b,c->abc", Bt[qx], Dt[qy], Bt[qz]).ravel(),
                                 np.einsum("a,b,c->abc", Bt[qx], Bt[qy], Dt[qz]).ravel()], axis=1)
                g = gref @ np.linalg.inv(J)                      # (nd, 3) physical gradients
                Bm = np.zeros((6, 3 * nd))                       # strains (xx, yy, zz, 2yz, 2xz, 2xy)
                for i in range(nd):
                    gx, gy, gz = g[i]
                    Bm[:, 3 * i + 0] = [gx, 0, 0, 0, gz, gy]
                    Bm[:, 3 * i + 1] = [0, gy, 0, gz, 0, gx]
                    Bm[:, 3 * i + 2] = [0, 0, gz, gy, gx, 0]
                Nm = np.kron(phi[None, :], np.eye(3))            # (3, 3 nd)
                wq = w[qx] * w[qy] * w[qz] * abs(np.linalg.det(J))
                K += wq * (Bm.T @ Dm @ Bm + beta * Nm.T @ Nm)
    return K


@pytest.mark.parametrize("p", [1, 2, 3])
def test_element_matrix_equals_dense_btdb(p):
    el = interval_element(p)
    X = _cell()
    A = eo.cell_matrices(el, X[None], MU, LMBDA, 0.7)[0]
    K = dense_element_matrix(el, X, MU, LMBDA, 0.7)
    assert np.abs(A - K).max() < 1e-13 * np.abs(K).max()


@pytest.mark.parametrize("p", [1, 2, 3])
def test_element_matrices_symmetric_semidefinite_with_rigid_body_kernel(p):
    mesh = ExtrudedHexMesh(2, 2, 2, warp=0.08, permute_seed=1)
    V = mesh.function_space(p)
    el = interval_element(p)
    di, A = eo.element_matrices(el, mesh.coordinates, *_geo(mesh, V), MU, LMBDA, 0.0)
    R = eo.rigid_body_modes(V.dof_coordinates())
    nd = 3 * el.ndof ** 3
    for c in range(A.shape[0]):
        Ac = A[c]
        s = np.abs(Ac).max()
        assert np.abs(Ac - Ac.T).max() < 1e-14 * s
        ev = np.linalg.eigvalsh(Ac)
        assert ev.min() > -1e-12 * ev.max()
        r = R[:, di[c]]                                        # the modes restricted to the cell
        assert np.linalg.norm(Ac @ r.T, axis=0).max() <= 1e-12 * np.linalg.norm(Ac, 2)
        assert np.linalg.matrix_rank(Ac, tol=1e-10 * ev.max()) == nd - 6
    # with beta > 0 the mass term removes the kernel
    _, Ab = eo.element_matrices(el, mesh.coordinates, *_geo(mesh, V), MU, LMBDA, 0.5)
    assert np.linalg.eigvalsh(Ab[0]).min() > 0.0


@pytest.mark.parametrize("p", [1, 2, 3])
def test_diagonal_identity(p):
    """diag(j, b) = int mu |grad phi_j|^2 + (mu + lmbda) (d_b phi_j)^2 + beta phi_j^2."""
    el = interval_element(p)
    X = _cell(3)
    beta = 0.4
    A = eo.cell_matrices(el, X[None], MU, LMBDA, beta)[0]
    n = el.ndof
    d = np.zeros((n ** 3, 3))
    for qx in range(n):
        for qy in range(n):
            for qz in range(n):
                J = _jacobian(X, (el.xq[qx], el.xq[qy], el.xq[qz]))
                phi = np.einsum("a,b,c->abc", el.B[qx], el.B[qy], el.B[qz]).ravel()
                gref = np.stack([np.einsum("a,b,c->abc", el.D[qx], el.B[qy], el.B[qz]).ravel(),
                                 np.einsum("a,b,c->abc", el.B[qx], el.D[qy], el.B[qz]).ravel(),
                                 np.einsum("a,b,c->abc", el.B[qx], el.B[qy], el.D[qz]).ravel()], axis=1)
                g = gref @ np.linalg.inv(J)
                wq = el.wq[qx] * el.wq[qy] * el.wq[qz] * abs(np.linalg.det(J))
                d += wq * (MU * (g ** 2).sum(axis=1)[:, None] + (MU + LMBDA) * g ** 2 + beta * phi[:, None] ** 2)
    assert np.abs(np.diagonal(A) - d.ravel()).max() < 1e-13 * np.abs(d).max()


@pytest.mark.parametrize("p", [1, 2, 3])
@pytest.mark.parametrize("beta", [0.0, 0.8])
def test_generic_path_matches_oracle(oracle, p, beta):
    """``assemble_elasticity_generic`` (generated wrapper around ``elasticity_kernel``, run through its
    host build by the mock engine) against the oracle."""
    from firedrake_b200.assemble import FunctionSpace, assemble_elasticity_generic
    mesh = ExtrudedHexMesh(3, 2, 3, warp=0.06, permute_seed=2)
    V0 = mesh.function_space(p)
    u0 = np.random.default_rng(4).standard_normal(3 * V0.node_count)
    y = eo.action(interval_element(p), mesh.coordinates, u0, *_geo(mesh, V0), MU, LMBDA, beta)
    with me.install(oracle):
        V = FunctionSpace(mesh, p, 3)
        yg = assemble_elasticity_generic(V, V.dat(u0.reshape(-1, 3).copy()), MU, LMBDA, beta).data_ro.copy()
    assert np.abs(y - yg.ravel()).max() < 1e-12 * np.abs(y).max()


def boundary_nodes(V):
    return np.unique(np.concatenate([V.boundary_nodes(s) for s in (1, 2, 3, 4, "bottom", "top")]))


PATCH_M = np.array([[0.3, -0.2, 0.5], [0.1, 0.4, -0.3], [-0.6, 0.2, 0.1]])     # not symmetric
PATCH_C = np.array([0.1, -0.2, 0.3])


@pytest.mark.parametrize("p", [1, 2])
def test_patch_test_reproduces_a_linear_field(p):
    """Dirichlet data u = M x + c on all six faces, zero load, beta = 0: the solve reproduces the linear
    field at every node of a warped mesh."""
    mesh = ExtrudedHexMesh(3, 3, 3, warp=0.08, permute_seed=4)
    V = mesh.function_space(p)
    K = eo.global_matrix(interval_element(p), mesh.coordinates, _geo(mesh, V), V.node_count, MU, LMBDA).tocsr()
    ue = (V.dof_coordinates() @ PATCH_M.T + PATCH_C).ravel()
    bn = boundary_nodes(V)
    bd = (3 * bn[:, None] + np.arange(3)).ravel()
    free = np.setdiff1d(np.arange(3 * V.node_count), bd)
    u = np.zeros_like(ue)
    u[bd] = ue[bd]
    u[free] = spla.spsolve(K[free][:, free].tocsc(), -K[free][:, bd] @ ue[bd])
    assert np.abs(u - ue).max() < 1e-10
