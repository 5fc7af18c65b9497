"""Host logic of the eigensolver on the CPU, against a recording stand-in for the engine that runs the Helmholtz family
as products with the oracle's global matrices and fdb_bv_dot / fdb_bv_mult in NumPy: the engine calls of one LOBPCG
iteration, no device-to-host copy but the Gram matrices, the result against scipy's eigh, every refusal, and the
engine calls of ``solve`` (whose preconditioner construction the eigensolver shares) against those recorded before
that code moved into ``assemble._preconditioner``."""
import json
import os

import numpy as np
import pytest

import _eigen_oracle as eo
import _mock_engine as me
from firedrake_b200 import _lib
from firedrake_b200.utility_meshes import ExtrudedHexMesh

HERE = os.path.dirname(os.path.abspath(__file__))
SOLVE_CALLS = os.path.join(HERE, "golden", "solve_engine_calls.json")


class EigenRecorder(me.MockEngine):
    """The Helmholtz kernels as (alpha K + beta M) products, the block-vector kernels in NumPy; records those calls,
    the preconditioner's pointwise products, the Dirichlet zeroing and every device-to-host copy.  With ``names``, also
    the name of every engine entry point called, in order."""

    def __init__(self, K, Mm):
        super().__init__(None)
        self.K, self.Mm, self.calls, self.names = K, Mm, [], None

    def __getattribute__(self, name):
        if name.startswith("fdb_"):
            names = object.__getattribute__(self, "names")
            if names is not None:
                names.append(name)
        return object.__getattribute__(self, name)

    def fdb_kernel_create(self, desc, out):
        d = me._obj(desc)
        if d.form != _lib.FORM_HELMHOLTZ:
            return super().fdb_kernel_create(desc, out)
        self._next += 1
        self.kernels[self._next] = dict(kind="mat", alpha=d.alpha, beta=d.beta, diagonal=bool(d.diagonal),
                                        rank=d.rank)
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        k = self.kernels[me._addr(h)]
        if k["kind"] != "mat":
            self.calls.append(("jit",) if k["kind"] == "jit" else ("kernel", k["kind"]))
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        n = self.K.shape[0]
        A = k["alpha"] * self.K + k["beta"] * self.Mm
        y = me._view(a.args[0], n)
        if k["diagonal"]:
            self.calls.append(("diagonal", k["alpha"], k["beta"]))
            y += A.diagonal()
        else:
            self.calls.append(("action", k["alpha"], k["beta"]))
            y += A @ me._view(a.args[2], n)
        return 0

    def _cols(self, p, count, n):
        return np.stack([me._view(p[i], n) for i in range(count)])

    def fdb_bv_dot(self, n, m, x, k, y, g):
        self.calls.append(("bv_dot", m, k))
        me._view(g, m * k)[:] = (self._cols(x, m, n) @ self._cols(y, k, n).T).ravel()
        return 0

    def fdb_bv_mult(self, n, k, y, beta, alpha, m, x, q):
        self.calls.append(("bv_mult", k, m))
        if {y[j] for j in range(k)} & {x[i] for i in range(m)}:
            return self._fail("fdb_bv_mult: in place")
        X = self._cols(x, m, n).copy()
        Q = me._view(q, m * k).reshape(m, k)
        for j in range(k):
            yj = me._view(y[j], n)
            yj[:] = (beta * yj if beta != 0.0 else 0.0) + alpha * (Q[:, j] @ X)
        return 0

    def fdb_vec_pointwise_mult(self, n, x, y, w):
        self.calls.append(("pointwise",))
        return super().fdb_vec_pointwise_mult(n, x, y, w)

    def fdb_dat_zero_nodes(self, dat, cdim, nodes, n):
        self.calls.append(("zero_nodes", n))
        return super().fdb_dat_zero_nodes(dat, cdim, nodes, n)

    def fdb_memcpy_d2h(self, dst, src, n):
        self.calls.append(("d2h", n))
        return self._copy(dst, src, n)


class recording(me.install):
    def __init__(self, K, Mm):
        self.engine = EigenRecorder(K, Mm)


def _poisson(p=2, n=(3, 3, 2)):
    from firedrake_b200.assemble import FunctionSpace
    mesh = ExtrudedHexMesh(*n, warp=0.05, permute_seed=3)
    V = FunctionSpace(mesh, p)
    return mesh, V, eo.helmholtz(mesh, V.V, p), eo.helmholtz(mesh, V.V, p, 0.0, 1.0)


def _problem(V):
    from firedrake_b200.assemble import DirichletBC, Form, mass
    from firedrake_b200.eigensolver import LinearEigenproblem
    bc = DirichletBC(V, 0.0, list(eo.WALLS))
    return LinearEigenproblem(Form(V, 1.0, 0.0), mass(V), bcs=[bc]), bc


def test_one_iteration_calls():
    """One LOBPCG iteration (the first: no P yet, every column active), in order: the residuals R = AX - MX diag(lam)
    by one fdb_bv_mult, their norms and ||M x_i|| from one fdb_bv_dot of [R, MX]; per column one Jacobi product and
    the Dirichlet zeroing; (MX)^T W by one fdb_bv_dot and W made M-orthogonal to X by one fdb_bv_mult; per column a
    fresh A action and M action, each followed by the Dirichlet zeroing; the Grams S^T(AS) and S^T(MS) of S = [X, W];
    then fdb_bv_mult for P, AP, MP from W and for X, AX, MX from [X, P].  No device-to-host copy in the loop."""
    from firedrake_b200.eigensolver import LinearEigensolver
    mesh, V, K, Mm = _poisson()
    nb = None
    with recording(K, Mm) as eng:
        prob, bc = _problem(V)
        nb = len(bc.nodes)
        es = LinearEigensolver(prob, 4, solver_parameters={"st_pc_type": "jacobi", "eps_tol": 1e-8})
        es.solve()
        calls = list(eng.calls)
    bs = 5                                              # 4 + ceil(4 / 4)
    keep = ("bv_dot", "bv_mult", "pointwise", "zero_nodes", "action", "diagonal", "d2h")
    calls = [c for c in calls if c[0] in keep]
    start = next(i for i, c in enumerate(calls) if c == ("bv_mult", bs, 2 * bs))     # the first residual
    pc = [("pointwise",), ("zero_nodes", nb)]
    act = [("action", 1.0, 0.0), ("zero_nodes", nb), ("action", 0.0, 1.0), ("zero_nodes", nb)]
    want = ([("bv_mult", bs, 2 * bs), ("bv_dot", 2 * bs, 2 * bs)] + pc * bs
            + [("bv_dot", bs, bs), ("bv_mult", bs, bs)]                          # W M-orthogonal to X
            + act * bs + [("bv_dot", 2 * bs, 2 * bs)] * 2
            + [("bv_mult", bs, bs)] * 3 + [("bv_mult", bs, 2 * bs)] * 3)
    assert calls[start:start + len(want)] == want
    # the second iteration has P, made M-orthogonal to X as W is and given fresh products: S = [X, W, P] has up to
    # 3 bs columns
    nxt = calls[start + len(want):]
    dots = [c for c in nxt if c[0] == "bv_dot"]
    grams = [c for c in dots if c[1] == c[2] and c[1] > 2 * bs]
    assert grams[:2] == [grams[0]] * 2 and dots[1:3] == [("bv_dot", bs, bs)] * 2   # (MX)^T W, (MX)^T P
    assert not any(c[0] == "d2h" for c in calls[start:])
    # before the loop: the initial block's A and M actions and one Rayleigh-Ritz, no other host copy
    assert not any(c[0] == "d2h" for c in calls[:start])
    assert es.iterations > 1


@pytest.mark.parametrize("pc", ["none", "jacobi"])
def test_result_matches_oracle(pc):
    """The 4 smallest eigenvalues to 1e-9 relative, M-orthonormal eigenvectors to 1e-10, zero on the Dirichlet nodes,
    and every residual within eps_tol."""
    from firedrake_b200.eigensolver import LinearEigensolver
    mesh, V, K, Mm = _poisson()
    with recording(K, Mm):
        prob, bc = _problem(V)
        es = LinearEigensolver(prob, 4, solver_parameters={"st_pc_type": pc, "eps_max_it": 2000})
        assert es.solve() == 4
        lam = np.array([es.eigenvalue(i) for i in range(4)])
        X = np.stack([es.eigenfunction(i)[0].data_ro.copy() for i in range(4)], axis=1)
        im = es.eigenfunction(0)[1].data_ro.copy()
        nodes = bc.nodes
    ref, _ = eo.restricted_eigh(K, Mm, nodes, 4)
    assert np.abs(lam - ref).max() <= 1e-9 * np.abs(ref).max()
    assert np.abs(X.T @ (Mm @ X) - np.eye(4)).max() < 1e-10
    assert np.abs(X[nodes]).max() == 0.0 and not im.any()
    assert np.all(es.residuals[:4] <= 1e-10)
    # the residuals recomputed here, on the scale of the block's largest Ritz value (at least lambda_4)
    # (on the free rows: the restricted problem has no constrained rows)
    free = np.setdiff1d(np.arange(K.shape[0]), nodes)
    R = (K @ X - (Mm @ X) * lam)[free]
    MX = (Mm @ X)[free]
    assert np.all(np.linalg.norm(R, axis=0) <= 1e-10 * es.theta * np.linalg.norm(MX, axis=0) * (1 + 1e-6))


def test_convergence_error_names_iterations_and_residual():
    from firedrake_b200.assemble import ConvergenceError
    from firedrake_b200.eigensolver import LinearEigensolver
    mesh, V, K, Mm = _poisson()
    with recording(K, Mm):
        prob, _ = _problem(V)
        es = LinearEigensolver(prob, 4, solver_parameters={"eps_max_it": 2})
        with pytest.raises(ConvergenceError, match=r"in 2 iterations: the worst relative residual .* is"):
            es.solve()


def test_refusals():
    from firedrake_b200.assemble import (AdvectionDiffusion, DGTransport, DirichletBC, Elasticity, Form,
                                         FunctionSpace, HyperElasticity, HyperElasticityJacobian, InteriorPenalty,
                                         NavierStokes, NavierStokesJacobian, NonlinearDiffusion,
                                         NonlinearDiffusionJacobian, SpectralForm, Stokes, mass)
    from firedrake_b200.eigensolver import LinearEigenproblem, LinearEigensolver
    mesh, V, K, Mm = _poisson(1)
    with recording(K, Mm):
        A = Form(V, 1.0, 0.0)
        W = FunctionSpace(mesh, 1, cdim=3)
        D = FunctionSpace(mesh, 2, family="DQ")
        # the refusals look at the form's type only
        for cls in (AdvectionDiffusion, DGTransport, NonlinearDiffusion, NonlinearDiffusionJacobian, HyperElasticity,
                    HyperElasticityJacobian):
            with pytest.raises(NotImplementedError, match=f"{cls.__name__} is nonsymmetric"):
                LinearEigenproblem(object.__new__(cls))
        for cls in (Stokes, NavierStokes, NavierStokesJacobian):
            with pytest.raises(NotImplementedError, match="Taylor-Hood and mixed"):
                LinearEigenproblem(object.__new__(cls))
        with pytest.raises(TypeError, match="not one of Form"):
            LinearEigenproblem(object())
        with pytest.raises(ValueError, match="another function space"):
            LinearEigenproblem(A, mass(FunctionSpace(mesh, 1)))
        with pytest.raises(NotImplementedError, match="restrict=False"):
            LinearEigenproblem(A, restrict=False)
        with pytest.raises(NotImplementedError, match="lumped mass"):
            LinearEigenproblem(A, SpectralForm(V, 1.0, 1.0))
        with pytest.raises(TypeError, match="not a Form"):
            LinearEigenproblem(A, Elasticity(W, 1.0, 1.0))
        Vp = FunctionSpace(mesh, 1)
        Vp.dof_dset.halo = object()                    # stands for the halo of a partitioned space
        with pytest.raises(NotImplementedError, match="partitioned space"):
            LinearEigenproblem(Form(Vp, 1.0, 0.0))
        prob = LinearEigenproblem(A, bcs=[DirichletBC(V, 0.0, list(eo.WALLS))])
        for sp, exc, match in (
                ({"eps_type": "krylovschur"}, NotImplementedError, "eps_type 'krylovschur'"),
                ({"eps_largest_real": None}, NotImplementedError, "eps_largest_real"),
                ({"eps_largest_magnitude": None}, NotImplementedError, "eps_largest_magnitude"),
                ({"eps_target": 1.0}, NotImplementedError, "eps_target"),
                ({"eps_target_real": None}, NotImplementedError, "eps_target_real"),
                ({"st_type": "sinvert"}, NotImplementedError, "st_type 'sinvert'"),
                ({"eps_gen_non_hermitian": None}, NotImplementedError, "eps_gen_non_hermitian"),
                ({"eps_lobpcg_blocksize": 22}, NotImplementedError, "eps_lobpcg_blocksize 22"),
                ({"eps_lobpcg_blocksize": 3}, ValueError, "smaller than n_evals"),
                ({"eps_bogus": 1}, NotImplementedError, "eps_bogus"),
                ({"st": {"bogus": 1}}, NotImplementedError, "st_bogus"),
                ({"st_ksp_type": "cg"}, NotImplementedError, "st_ksp_type 'cg'"),
                ({"st_pc_type": "ilu"}, NotImplementedError, "st_pc_type 'ilu'"),
                ({"st_pc_type": "mg"}, ValueError, "hierarchy")):
            with pytest.raises(exc, match=match):
                LinearEigensolver(prob, 4, solver_parameters=sp)
        with pytest.raises(NotImplementedError, match="n_evals = 22"):
            LinearEigensolver(prob, 22)
        # the accepted flags and nested dicts
        es = LinearEigensolver(prob, 20, solver_parameters={"eps_smallest_real": None, "eps_gen_hermitian": None,
                                                            "eps": {"tol": 1e-6}, "st": {"pc_type": "jacobi"}})
        assert es.options["eps_lobpcg_blocksize"] == 21 and es.options["eps_tol"] == 1e-6
        assert LinearEigensolver(prob, 8).options["eps_lobpcg_blocksize"] == 10
        # mg and p-multigrid on a singular A, the SEM operator and DQ
        free = LinearEigenproblem(A)
        for pc in ("mg", "python"):
            with pytest.raises(NotImplementedError, match="singular A"):
                LinearEigensolver(free, 2, solver_parameters={"st_pc_type": pc}, hierarchy=object())
            with pytest.raises(NotImplementedError, match="SpectralForm"):
                LinearEigensolver(LinearEigenproblem(SpectralForm(V), SpectralForm(V, 0.0, 1.0)), 2,
                                  solver_parameters={"st_pc_type": pc})
            with pytest.raises(NotImplementedError, match="DQ space"):
                LinearEigensolver(LinearEigenproblem(InteriorPenalty(D, 1.0, 0.0, 27.0)), 2,
                                  solver_parameters={"st_pc_type": pc})
        # unknown p-multigrid options are refused by pmg_options when the preconditioner is built
        with pytest.raises(NotImplementedError, match="pmg_bogus"):
            LinearEigensolver(prob, 2, solver_parameters={"st_pc_type": "python",
                                                          "st_pc_python_type": "firedrake.P1PC",
                                                          "st_pmg_bogus": 1}).solve()


def _solve_calls(pc):
    """The engine entry points a Poisson solve calls, in order, on the recording engine."""
    from firedrake_b200.assemble import DirichletBC, Form, FunctionSpace, assemble, mass, solve
    mesh = ExtrudedHexMesh(3, 3, 2, warp=0.05, permute_seed=3)
    Vh = mesh.function_space(2)
    K, Mm = eo.helmholtz(mesh, Vh, 2), eo.helmholtz(mesh, Vh, 2, 0.0, 1.0)
    with recording(K, Mm) as eng:
        V = FunctionSpace(mesh, 2)
        bc = DirichletBC(V, 0.0, list(eo.WALLS))
        L = assemble(mass(V), u=V.dat(np.ones(V.node_count)))
        u = V.dat()
        eng.names = []
        solve(Form(V, 1.0, 0.0), L, u, bcs=[bc], solver_parameters={"pc_type": pc, "ksp_rtol": 1e-10})
        return list(eng.names)


@pytest.mark.parametrize("pc", ["none", "jacobi"])
def test_solve_engine_calls_unchanged(pc):
    """solve makes exactly the engine calls it made before its preconditioner construction moved into
    assemble._preconditioner (recorded from that version into tests/golden/solve_engine_calls.json)."""
    with open(SOLVE_CALLS) as f:
        want = json.load(f)[pc]
    assert _solve_calls(pc) == want


class _CorruptAX:
    """Adds 1e-6 x to the carried A x of the first column, once, when the third update of X writes AX: AX then no longer
    equals A X, and a residual or Gram matrix from the carried products alone points at a wrong lambda."""

    def __init__(self, es):
        self.es, self.seen, self.done = es, 0, False
        orig = es._setup

        def setup():
            orig()
            mult = es._bv.mult

            def wrapped(ys, xs, Q, beta=0.0, alpha=1.0):
                mult(ys, xs, Q, beta, alpha)
                v = es._v
                if not self.done and len(xs) == 2 * len(ys) and ys[0] is v["AW"][0] and xs[0] in v["AX"]:
                    self.seen += 1
                    if self.seen == 3:
                        L = _lib.lib()
                        _lib.check(L.fdb_vec_axpy(ys[0]._data.size, 1e-6, v["W"][0].device_ptr, ys[0].device_ptr))
                        ys[0]._device_written()
                        self.done = True
            es._bv.mult = wrapped
        es._setup = setup


def test_lock_needs_fresh_products():
    """With the carried AX of one column corrupted, the pairs are locked on fresh A and M actions only: the result
    still matches scipy to 1e-9, where trusting the carried products would report a lambda off by about 1e-6."""
    from firedrake_b200.eigensolver import LinearEigensolver
    mesh, V, K, Mm = _poisson()
    with recording(K, Mm):
        prob, bc = _problem(V)
        es = LinearEigensolver(prob, 4, solver_parameters={"st_pc_type": "jacobi", "eps_max_it": 2000})
        bad = _CorruptAX(es)
        es.solve()
        lam = np.array([es.eigenvalue(i) for i in range(4)])
        X = np.stack([es.eigenfunction(i)[0].data_ro.copy() for i in range(4)], axis=1)
        nodes = bc.nodes
    assert bad.done and es.refreshed >= 4
    ref, _ = eo.restricted_eigh(K, Mm, nodes, 4)
    assert np.abs(lam - ref).max() <= 1e-9 * np.abs(ref).max()
    free = np.setdiff1d(np.arange(K.shape[0]), nodes)
    R = (K @ X - (Mm @ X) * lam)[free]
    assert np.all(np.linalg.norm(R, axis=0) <= 1e-10 * es.theta * np.linalg.norm((Mm @ X)[free], axis=0) * 1.000001)


def test_rank_deficient_start_and_indefinite_mass():
    """More block columns than free rows ends in ConvergenceError, not a LinAlgError; an M that is not positive
    definite is refused by name."""
    from firedrake_b200.assemble import ConvergenceError, DirichletBC, Form, FunctionSpace, mass
    from firedrake_b200.eigensolver import LinearEigenproblem, LinearEigensolver
    mesh = ExtrudedHexMesh(1, 1, 1)
    Vh = mesh.function_space(2)
    K, Mm = eo.helmholtz(mesh, Vh, 2), eo.helmholtz(mesh, Vh, 2, 0.0, 1.0)
    with recording(K, Mm):
        V = FunctionSpace(mesh, 2)
        bc = DirichletBC(V, 0.0, list(eo.WALLS))                  # one free node
        es = LinearEigensolver(LinearEigenproblem(Form(V, 1.0, 0.0), mass(V), [bc]), 2)
        with pytest.raises(ConvergenceError, match="rank-deficient"):
            es.solve()
        for M in (Form(V, 1.0, 0.0), Form(V, 0.0, -1.0), Form(V, -1.0, 1.0)):
            with pytest.raises(ValueError, match="not positive definite"):
                LinearEigenproblem(Form(V, 1.0, 0.0), M)
