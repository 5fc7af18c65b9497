"""The eigensolver on the H100: fdb_bv_dot and fdb_bv_mult against NumPy, their repeatability and refusals, and LOBPCG
against scipy's eigh of the oracle matrices for every form the solver takes, the rigid-body modes of a free body, the
preconditioners' iteration counts and the unit cube's convergence rates."""
import ctypes as C

import numpy as np
import pytest

import _eigen_oracle as eo
from firedrake_b200 import _lib, mg
from firedrake_b200.assemble import (DirichletBC, Elasticity, Form, FunctionSpace, InteriorPenalty, SpectralForm,
                                     mass)
from firedrake_b200.eigensolver import LinearEigenproblem, LinearEigensolver
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ block-vector kernels
class _Cols:
    """``count`` device columns of n doubles (one allocation, columns 256 B apart) and their pointer array."""

    def __init__(self, host):
        L = _lib.lib()
        self.count, self.n = host.shape
        self.ld = (self.n + 31) // 32 * 32
        self.base = L.fdb_malloc(max(self.count * self.ld, 1) * 8)
        assert self.base
        for i in range(self.count):
            _lib.check(L.fdb_memcpy_h2d(self.ptr(i), np.ascontiguousarray(host[i]).ctypes.data, self.n * 8))
        self.ptrs = (C.c_void_p * self.count)(*[self.ptr(i) for i in range(self.count)])

    def ptr(self, i):
        return self.base + i * self.ld * 8

    def get(self):
        out = np.empty((self.count, self.n))
        for i in range(self.count):
            _lib.check(_lib.lib().fdb_memcpy_d2h(out[i].ctypes.data, self.ptr(i), self.n * 8))
        return out

    def free(self):
        _lib.lib().fdb_free(self.base)


def _dot(n, x, y):
    g = np.empty((x.count, y.count))
    _lib.check(_lib.lib().fdb_bv_dot(n, x.count, x.ptrs, y.count, y.ptrs, g.ctypes.data_as(C.POINTER(C.c_double))))
    return g


def _mult(n, y, beta, alpha, x, Q):
    Q = np.ascontiguousarray(Q)
    return _lib.lib().fdb_bv_mult(n, y.count, y.ptrs, beta, alpha, x.count, x.ptrs,
                                  Q.ctypes.data_as(C.POINTER(C.c_double)))


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("n", [1, 255, 1_000_003])
@pytest.mark.parametrize("m", [1, 7, 48, 64])
@pytest.mark.parametrize("k", [1, 7, 48, 64])
def test_bv_kernels_match_numpy(engine, n, m, k):
    rng = np.random.default_rng(n + 100 * m + k)
    X, Y = rng.standard_normal((m, n)), rng.standard_normal((k, n))
    Q = rng.standard_normal((m, k))
    x, y = _Cols(X), _Cols(Y)
    try:
        G = _dot(n, x, y)
        # the entries are sums of n products of unit normals: relative to the sum of |products|, not to |G|
        scale = np.abs(X) @ np.abs(Y).T
        assert np.all(np.abs(G - X @ Y.T) <= 1e-13 * scale + 1e-300)
        assert np.array_equal(G, _dot(n, x, y))                      # bitwise repeatable
        _lib.check(_mult(n, y, 0.5, -2.0, x, Q))
        want = 0.5 * Y - 2.0 * (Q.T @ X)
        tol = 1e-13 * (0.5 * np.abs(Y) + 2.0 * (np.abs(Q).T @ np.abs(X)))
        assert np.all(np.abs(y.get() - want) <= tol)
        # beta = 0 does not read y: NaNs there do not propagate
        _lib.check(_lib.lib().fdb_memset(y.base, 0xFF, y.count * y.ld * 8))
        _lib.check(_mult(n, y, 0.0, 1.0, x, Q))
        assert np.all(np.abs(y.get() - Q.T @ X) <= 1e-13 * (np.abs(Q).T @ np.abs(X)))
    finally:
        x.free()
        y.free()


def test_bv_n_zero(engine):
    x, y = _Cols(np.ones((3, 4))), _Cols(np.full((2, 4), 7.0))
    try:
        assert not _dot(0, x, y).any()
        _lib.check(_mult(0, y, 0.0, 1.0, x, np.ones((3, 2))))
        assert np.all(y.get() == 7.0)
    finally:
        x.free()
        y.free()


def test_bv_refusals(engine):
    L = _lib.lib()
    x, y = _Cols(np.ones((65, 8))), _Cols(np.ones((2, 8)))
    g = np.empty(65 * 2)
    gp = g.ctypes.data_as(C.POINTER(C.c_double))
    Q = np.ones(65 * 2)
    qp = Q.ctypes.data_as(C.POINTER(C.c_double))

    def err(rc):
        assert rc != 0
        return L.fdb_last_error().decode()

    try:
        assert "x (m) = 0 columns; 1..64" in err(L.fdb_bv_dot(8, 0, x.ptrs, 2, y.ptrs, gp))
        assert "x (m) = 65 columns; 1..64" in err(L.fdb_bv_dot(8, 65, x.ptrs, 2, y.ptrs, gp))
        assert "y (k) = 65 columns" in err(L.fdb_bv_mult(8, 65, x.ptrs, 0.0, 1.0, 2, y.ptrs, qp))
        assert "NULL column array for y (k)" in err(L.fdb_bv_dot(8, 2, x.ptrs, 2, None, gp))
        nul = (C.c_void_p * 2)(y.ptr(0), None)
        assert "column 1 of y (k) is NULL" in err(L.fdb_bv_dot(8, 2, x.ptrs, 2, nul, gp))
        assert "NULL host pointer for G" in err(L.fdb_bv_dot(8, 2, x.ptrs, 2, y.ptrs, None))
        assert "NULL host pointer for Q" in err(L.fdb_bv_mult(8, 2, y.ptrs, 0.0, 1.0, 2, x.ptrs, None))
        alias = (C.c_void_p * 2)(x.ptr(5), y.ptr(1))
        assert "y column 1 is x column 1" in err(L.fdb_bv_mult(8, 2, y.ptrs, 0.0, 1.0, 2, alias, qp))
        assert "not in place" in L.fdb_last_error().decode()
        assert "y column 0 is x column 1" in err(L.fdb_bv_mult(8, 2, alias, 0.0, 1.0, 2, (C.c_void_p * 2)(
            x.ptr(0), x.ptr(5)), qp))
    finally:
        x.free()
        y.free()


# ------------------------------------------------------------------ LOBPCG against the oracle
TOL = 1e-10     # the default eps_tol (Firedrake's)


def _solve(A, M, bcs, n, sp=None, hierarchy=None, seed=0):
    es = LinearEigensolver(LinearEigenproblem(A, M, bcs), n, solver_parameters=sp, hierarchy=hierarchy, seed=seed)
    assert es.options["eps_tol"] == TOL
    assert es.solve() == n
    lam = np.array([es.eigenvalue(i) for i in range(n)])
    X = np.stack([es.eigenfunction(i)[0].data_ro.reshape(-1).copy() for i in range(n)], axis=1)
    assert not es.eigenfunction(0)[1].data_ro.any()
    return es, lam, X


def _check(es, lam, X, K, Mm, constrained, ref, tol=TOL):
    assert np.abs(lam - ref).max() <= 1e-9 * np.abs(ref).max(), (lam, ref)
    assert np.abs(X.T @ (Mm @ X) - np.eye(len(lam))).max() < 1e-10
    if len(constrained):
        assert np.abs(X[constrained]).max() == 0.0
    free = np.setdiff1d(np.arange(K.shape[0]), constrained)
    R = (K @ X - (Mm @ X) * lam)[free]
    MX = (Mm @ X)[free]
    scale = np.maximum(np.abs(lam), es.theta)
    assert np.all(np.linalg.norm(R, axis=0) <= tol * scale * np.linalg.norm(MX, axis=0) * (1 + 1e-6))


def _kappa(W, seed=0):
    X = W.dof_coordinates()
    return 1.0 + 0.5 * np.sin(3.0 * X[:, 0]) * X[:, 1] + 0.2 * np.random.default_rng(seed).random(len(X))


@pytest.mark.parametrize("p", [1, 2, 3])
def test_form_with_kappa(engine, p):
    mesh = ExtrudedHexMesh(4, 4, 3, warp=0.05, permute_seed=1)
    V = FunctionSpace(mesh, p)
    kap = _kappa(V.V)
    bc = DirichletBC(V, 0.0, list(eo.WALLS))
    es, lam, X = _solve(Form(V, 1.0, 0.0, V.dat(kap)), mass(V), [bc], 6, {"st_pc_type": "jacobi"})
    K, Mm = eo.helmholtz(mesh, V.V, p, 1.0, 0.0, kap), eo.helmholtz(mesh, V.V, p, 0.0, 1.0)
    ref, _ = eo.restricted_eigh(K, Mm, bc.nodes, 6)
    _check(es, lam, X, K, Mm, bc.nodes, ref)


@pytest.mark.parametrize("p,seed", [(3, 0), (3, 1), (5, 0), (5, 1), (5, 2), (5, 3)])
def test_spectral_form_lumped_mass(engine, p, seed):
    # a square base makes clusters of nearly equal eigenvalues (two and three within 1e-3); several random starts
    mesh = ExtrudedHexMesh(3, 3, 2, warp=0.05, permute_seed=2)
    V = FunctionSpace(mesh, p)
    bc = DirichletBC(V, 0.0, list(eo.WALLS))
    es, lam, X = _solve(SpectralForm(V, 1.0, 0.0), SpectralForm(V, 0.0, 1.0), [bc], 5, {"st_pc_type": "jacobi"},
                        seed=seed)
    K, Mm = eo.spectral(mesh, V.V, p, 1.0, 0.0), eo.spectral(mesh, V.V, p, 0.0, 1.0)
    ref, _ = eo.restricted_eigh(K, Mm, bc.nodes, 5)
    _check(es, lam, X, K, Mm, bc.nodes, ref)


def test_interior_penalty_dq2(engine):
    mesh = ExtrudedHexMesh(3, 3, 3, warp=0.05, permute_seed=3)
    D = FunctionSpace(mesh, 2, family="DQ")
    eta = 3.0 * 9
    es, lam, X = _solve(InteriorPenalty(D, 1.0, 0.0, eta, "on_boundary"), mass(D), [], 5, {"st_pc_type": "jacobi"})
    K, Mm = eo.interior_penalty(mesh, D.V, 2, 1.0, 0.0, eta), eo.dg_mass(mesh, D.V, 2)
    ref, _ = eo.restricted_eigh(K, Mm, [], 5)
    _check(es, lam, X, K, Mm, np.zeros(0, dtype=np.int64), ref)


MU, LMBDA = 1.0, 1.5


def _vector_dofs(nodes):
    return (3 * np.asarray(nodes, dtype=np.int64)[:, None] + np.arange(3)).ravel()


def test_clamped_cantilever_cg2(engine):
    mesh = ExtrudedHexMesh(6, 2, 2, Lx=3.0, warp=0.03, permute_seed=4)
    V = FunctionSpace(mesh, 2, cdim=3)
    bc = DirichletBC(V, 0.0, 1)
    es, lam, X = _solve(Elasticity(V, MU, LMBDA), mass(V), [bc], 6, {"st_pc_type": "jacobi"})
    K, Mm = eo.elasticity(mesh, V.V, 2, MU, LMBDA), eo.vector_mass(mesh, V.V, 2)
    cons = _vector_dofs(bc.nodes)
    ref, _ = eo.restricted_eigh(K, Mm, cons, 6)
    _check(es, lam, X, K, Mm, cons, ref)


def test_free_free_elasticity_rigid_modes(engine):
    """No conditions, Jacobi: the six rigid-body modes come out with |lambda| <= 1e-8 lambda_7 and lambda_7 matches."""
    mesh = ExtrudedHexMesh(3, 2, 2, Lx=1.5, warp=0.03, permute_seed=5)
    V = FunctionSpace(mesh, 1, cdim=3)
    es, lam, X = _solve(Elasticity(V, MU, LMBDA), mass(V), [], 7, {"st_pc_type": "jacobi"})
    K, Mm = eo.elasticity(mesh, V.V, 1, MU, LMBDA), eo.vector_mass(mesh, V.V, 1)
    ref, _ = eo.restricted_eigh(K, Mm, [], 7)
    assert np.all(np.abs(lam[:6]) <= 1e-8 * lam[6])
    assert abs(lam[6] - ref[6]) <= 1e-9 * ref[6]
    assert np.abs(X.T @ (Mm @ X) - np.eye(7)).max() < 1e-10


def _iterations(h, pc):
    V = FunctionSpace(h[len(h) - 1], 2)
    bc = DirichletBC(V, 0.0, list(eo.WALLS))
    es = LinearEigensolver(LinearEigenproblem(Form(V, 1.0, 0.0), mass(V), [bc]), 4,
                           solver_parameters={"st_pc_type": pc, "eps_tol": 1e-8, "eps_max_it": 2000}, hierarchy=h)
    es.solve()
    return es.iterations


def test_mg_iterations_mesh_independent(engine):
    """With a V-cycle on CG2 the iteration count on 16^3 is at most 1.3 times that on 8^3, and below Jacobi's."""
    h8, h16 = mg.MeshHierarchy(2, 2, 2, 2, warp=0.03), mg.MeshHierarchy(2, 2, 2, 3, warp=0.03)
    m8, m16 = _iterations(h8, "mg"), _iterations(h16, "mg")
    j8, j16 = _iterations(h8, "jacobi"), _iterations(h16, "jacobi")
    print(f"LOBPCG iterations, CG2: mg {m8} (8^3) {m16} (16^3); jacobi {j8} (8^3) {j16} (16^3)")
    assert m16 <= 1.3 * m8
    assert m8 < j8 and m16 < j16


def test_p1pc_cg3_converges(engine):
    mesh = ExtrudedHexMesh(4, 4, 4, warp=0.05, permute_seed=6)
    V = FunctionSpace(mesh, 3)
    bc = DirichletBC(V, 0.0, list(eo.WALLS))
    es, lam, X = _solve(Form(V, 1.0, 0.0), mass(V), [bc], 4,
                        {"st_pc_type": "python", "st_pc_python_type": "firedrake.P1PC"})
    K, Mm = eo.helmholtz(mesh, V.V, 3), eo.helmholtz(mesh, V.V, 3, 0.0, 1.0)
    ref, _ = eo.restricted_eigh(K, Mm, bc.nodes, 4)
    _check(es, lam, X, K, Mm, bc.nodes, ref)


def test_unit_cube_cg3_rates(engine):
    """The first 7 Dirichlet eigenvalues at CG3 on 4^3 and 8^3 converge to pi^2 (l^2 + m^2 + n^2) at rates in
    [2p - 0.3, 2p + 0.5], as the oracle's do."""
    lams = []
    for n in (4, 8):
        V = FunctionSpace(ExtrudedHexMesh(n, n, n), 3)
        bc = DirichletBC(V, 0.0, list(eo.WALLS))
        _, lam, _ = _solve(Form(V, 1.0, 0.0), mass(V), [bc], 7, {"st_pc_type": "jacobi"})
        lams.append(lam)
    exact = eo.exact_cube(7)
    rates = np.log2((lams[0] - exact) / (lams[1] - exact))
    print("CG3 rates", rates)
    assert np.all(rates >= 5.7) and np.all(rates <= 6.5), rates
