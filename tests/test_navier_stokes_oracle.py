"""The CPU oracle of steady Navier-Stokes on Taylor-Hood hexahedra (tests/_navier_stokes_oracle.py) against
independent statements: the Jacobian against central differences of the residual and its Taylor remainder,
J(0) and R(0, p) against the Stokes oracle, the quadratic scaling of the convective term, a point-by-point
evaluation of the convective term on warped cells, and the generic wrapper path's ``navier_stokes_kernel``
through its host build."""
import numpy as np
import pytest

import _mock_engine as me
import _navier_stokes_oracle as nso
import _stokes_oracle as so
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

NU = 0.7


def _setup(p, n=(3, 2, 3), warp=0.08, seed=1):
    mesh = ExtrudedHexMesh(*n, warp=warp, permute_seed=seed)
    V, Q = mesh.function_space(p), mesh.function_space(p - 1)
    geo = (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    return mesh, V, Q, geo, (Q.cell_node_map, Q.offset)


def _fields(V, Q, seed=0):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(3 * V.node_count), rng.standard_normal(Q.node_count)


def _cat(y):
    return np.concatenate(y)


@pytest.mark.parametrize("p", [2, 3, 4])
def test_jacobian_is_the_derivative_of_the_residual(p):
    """Central differences of R match J w, and the Taylor remainder R(u + h w) - R(u) - h J w falls by 4 when h
    is halved (R is quadratic in u, so the remainder is h^2 times a fixed vector)."""
    mesh, V, Q, geo, geo2 = _setup(p)
    el = interval_element(p)
    u, pr = _fields(V, Q, 1)
    w, r = _fields(V, Q, 2)
    R = lambda a, b: _cat(nso.residual(el, mesh.coordinates, a, b, geo, geo2, NU, 0.3))
    Jw = _cat(nso.jacobian_action(el, mesh.coordinates, u, w, r, geo, geo2, NU, 0.3))
    h = 1e-3
    fd = (R(u + h * w, pr + h * r) - R(u - h * w, pr - h * r)) / (2 * h)
    assert np.abs(fd - Jw).max() < 1e-9 * np.abs(Jw).max()
    rem = [np.abs(R(u + t * w, pr + t * r) - R(u, pr) - t * Jw).max() for t in (0.1, 0.05)]
    assert 3.9 < rem[0] / rem[1] < 4.1


@pytest.mark.parametrize("p", [2, 3])
def test_jacobian_matrix_matches_its_action(p):
    mesh, V, Q, geo, geo2 = _setup(p)
    el = interval_element(p)
    u, _ = _fields(V, Q, 3)
    w, r = _fields(V, Q, 4)
    K = nso.jacobian_matrix(el, mesh.coordinates, u, geo, geo2, V.node_count, Q.node_count, NU, 0.2)
    want = _cat(nso.jacobian_action(el, mesh.coordinates, u, w, r, geo, geo2, NU, 0.2))
    assert np.abs(K @ np.concatenate([w, r]) - want).max() < 1e-12 * np.abs(want).max()
    assert abs(K - K.T).max() > 1e-3 * abs(K).max()          # the convective term is not symmetric


@pytest.mark.parametrize("p", [2, 3, 4])
def test_jacobian_at_zero_is_stokes(p):
    mesh, V, Q, geo, geo2 = _setup(p)
    el = interval_element(p)
    K = nso.jacobian_matrix(el, mesh.coordinates, np.zeros(3 * V.node_count), geo, geo2, V.node_count,
                            Q.node_count, NU, 0.4)
    S = so.global_matrix(el, mesh.coordinates, geo, geo2, V.node_count, Q.node_count, NU, 0.4)
    assert abs(K - S).max() < 1e-13 * abs(S).max()


@pytest.mark.parametrize("p", [2, 3, 4])
def test_residual_at_zero_velocity_and_quadratic_scaling(p):
    """R(0, p) is the Stokes action on (0, p), and R(2u, p) - S(2u, p) = 4 (R(u, p) - S(u, p))."""
    mesh, V, Q, geo, geo2 = _setup(p)
    el = interval_element(p)
    u, pr = _fields(V, Q, 5)
    z = np.zeros_like(u)
    R0 = _cat(nso.residual(el, mesh.coordinates, z, pr, geo, geo2, NU, 0.6))
    S0 = _cat(so.action(el, mesh.coordinates, z, pr, geo, geo2, NU, 0.6))
    assert np.abs(R0 - S0).max() < 1e-14 * np.abs(S0).max()
    C = lambda a: (_cat(nso.residual(el, mesh.coordinates, a, pr, geo, geo2, NU, 0.6))
                   - _cat(so.action(el, mesh.coordinates, a, pr, geo, geo2, NU, 0.6)))
    c1, c2 = C(u), C(2 * u)
    assert np.abs(c1).max() > 0.0
    assert np.abs(c2 - 4 * c1).max() < 1e-12 * np.abs(c2).max()


def _pointwise_convective(el, X, a, b):
    """inner(dot(grad a, b), v)*dx on one cell, point by point: the trilinear map's Jacobian from its vertices,
    the basis and its reference gradient from the 1-D tables, G = (reference gradient) J^{-1}."""
    B, D, xq, wq = (np.asarray(t) for t in (el.B, el.D, el.xq, el.wq))
    n = B.shape[1]
    y = np.zeros((n ** 3, 3))
    for qx in range(n):
        for qy in range(n):
            for qz in range(n):
                xi = (xq[qx], xq[qy], xq[qz])
                J = np.zeros((3, 3))
                for v in range(8):
                    bits = ((v >> 2) & 1, (v >> 1) & 1, v & 1)
                    for r in range(3):
                        g = 1.0 if bits[r] else -1.0
                        for e in range(3):
                            if e != r:
                                g *= xi[e] if bits[e] else 1.0 - xi[e]
                        J[:, r] += X[v] * g
                phi = np.zeros(n ** 3)
                dphi = np.zeros((n ** 3, 3))
                for i in range(n):
                    for j in range(n):
                        for k in range(n):
                            idx = (i * n + j) * n + k
                            phi[idx] = B[qx, i] * B[qy, j] * B[qz, k]
                            dphi[idx] = (D[qx, i] * B[qy, j] * B[qz, k], B[qx, i] * D[qy, j] * B[qz, k],
                                         B[qx, i] * B[qy, j] * D[qz, k])
                G = (a.T @ dphi) @ np.linalg.inv(J)          # G[d, e] = d a_d / d x_e
                val = G @ (b.T @ phi)
                y += wq[qx] * wq[qy] * wq[qz] * abs(np.linalg.det(J)) * np.outer(phi, val)
    return y


@pytest.mark.parametrize("p", [2, 3])
def test_convective_term_point_by_point(p):
    mesh, V, Q, geo, geo2 = _setup(p, warp=0.1)
    el = interval_element(p)
    u, _ = _fields(V, Q, 6)
    w, _ = _fields(V, Q, 7)
    i0, i1, _, Xc, uc = nso._gather(el, mesh.coordinates, u, geo, geo2)
    wc = w.reshape(-1, 3)[i0]
    got = nso.convective(el, Xc, uc, wc)
    for c in (0, 5, len(Xc) - 1):
        want = _pointwise_convective(el, Xc[c], uc[c], wc[c])
        assert np.abs(got[c] - want).max() < 1e-13 * np.abs(want).max()


@pytest.mark.parametrize("p", [2, 3])
@pytest.mark.parametrize("beta", [0.0, 0.8])
def test_generic_path_host_build_matches_the_oracle(oracle, p, beta):
    from firedrake_b200.assemble import FunctionSpace, NavierStokes, assemble_navier_stokes_generic
    mesh, V0, Q0, geo, geo2 = _setup(p, seed=2)
    el = interval_element(p)
    u0, p0 = _fields(V0, Q0, 8)
    w0, r0 = _fields(V0, Q0, 9)
    want_r = nso.residual(el, mesh.coordinates, u0, p0, geo, geo2, 1.2, beta)
    want_j = nso.jacobian_action(el, mesh.coordinates, u0, w0, r0, geo, geo2, 1.2, beta)
    with me.install(oracle):
        F = NavierStokes(FunctionSpace(mesh, p, 3), FunctionSpace(mesh, p - 1), 1.2, beta)
        up = F.dat(u0.reshape(-1, 3).copy(), p0.copy())
        yr = [d.data_ro.copy() for d in assemble_navier_stokes_generic(F, up)]
        yj = [d.data_ro.copy() for d in assemble_navier_stokes_generic(F, up, F.dat(w0.reshape(-1, 3).copy(),
                                                                                      r0.copy()))]
    for y, want in ((yr, want_r), (yj, want_j)):
        assert np.abs(y[0].ravel() - want[0]).max() < 1e-12 * np.abs(want[0]).max()
        assert np.abs(y[1] - want[1]).max() < 1e-12 * np.abs(want[1]).max()


def test_navier_stokes_form_refusals():
    from firedrake_b200.assemble import FunctionSpace, NavierStokes, navier_stokes_kernel
    mesh = ExtrudedHexMesh(2, 2, 2)
    with pytest.raises(ValueError, match="Navier-Stokes velocity space is a vector space with 3 components"):
        NavierStokes(FunctionSpace(mesh, 2), FunctionSpace(mesh, 1))
    with pytest.raises(ValueError, match="Navier-Stokes pressure space is scalar"):
        NavierStokes(FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1, 3))
    with pytest.raises(ValueError, match="same mesh"):
        NavierStokes(FunctionSpace(mesh, 2, 3), FunctionSpace(ExtrudedHexMesh(2, 2, 2), 1))
    with pytest.raises(ValueError, match="p = 2..4"):
        NavierStokes(FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 2))
    with pytest.raises(ValueError, match="p = 2..4"):
        NavierStokes(FunctionSpace(mesh, 5, 3), FunctionSpace(mesh, 4))
    for jac in (False, True):
        with pytest.raises(NotImplementedError, match="degrees 2..4"):
            navier_stokes_kernel(5, jacobian=jac)
        with pytest.raises(NotImplementedError, match="degrees 2..4"):
            navier_stokes_kernel(1, jacobian=jac)
