"""Symmetric generalised eigenproblems ``A x = lambda M x`` on the device: Firedrake's ``LinearEigenproblem`` and
``LinearEigensolver`` (firedrake/eigensolver.py), solved by preconditioned block LOBPCG (Knyazev), which is SLEPc's
``eps_type lobpcg`` with ``st_type precond``.

The operator half of an iteration runs on the existing kernels: block-size actions of A and M through
:class:`assemble.OneFormAssembler` (a lumped M is a pointwise multiply by its diagonal) and preconditioner
applications.  The subspace half runs on ``fdb_bv_dot`` (the Gram matrices) and ``fdb_bv_mult`` (the basis updates,
csrc/bv.cu), whose columns are the block's own Dats.  Only the Gram matrices come back to the host, where the
Rayleigh-Ritz problem of at most 63 x 63 is solved with ``scipy.linalg.eigh``."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .assemble import (AdvectionDiffusion, ConvergenceError, DGTransport, Elasticity, Form, HyperElasticity,
                       HyperElasticityJacobian, ImplicitMatrixContext, InteriorPenalty, NavierStokes,
                       NavierStokesJacobian, NonlinearDiffusion, NonlinearDiffusionJacobian, OneFormAssembler,
                       SpectralForm, Stokes, _preconditioner, mass)

__all__ = ["LinearEigenproblem", "LinearEigensolver"]

_NONSYMMETRIC = (AdvectionDiffusion, DGTransport, NonlinearDiffusion, NonlinearDiffusionJacobian, HyperElasticity,
                 HyperElasticityJacobian)
_MIXED = (Stokes, NavierStokes, NavierStokesJacobian)
_OPERATORS = (Form, Elasticity, SpectralForm, InteriorPenalty)

# the largest block: S = [X, W, P] has at most 3 * bs <= FDB_BV_MAX_COLUMNS columns
MAX_BLOCKSIZE = _lib.BV_MAX_COLUMNS // 3

REFRESH_EVERY = 20

_DEFAULTS = {"eps_type": "lobpcg", "eps_tol": 1e-10, "eps_max_it": 500, "eps_lobpcg_blocksize": None,
             "st_type": "precond", "st_ksp_type": "preonly", "st_pc_type": "none", "st_pc_python_type": None}
_FLAGS = ("eps_smallest_real", "eps_gen_hermitian", "eps_hermitian")
_REFUSED = {
    "eps_largest_real": "only the smallest eigenvalues (eps_smallest_real) are computed",
    "eps_largest_magnitude": "only the smallest eigenvalues (eps_smallest_real) are computed",
    "eps_largest_imaginary": "only the smallest eigenvalues (eps_smallest_real) are computed",
    "eps_smallest_magnitude": "only the smallest eigenvalues (eps_smallest_real) are computed",
    "eps_smallest_imaginary": "only the smallest eigenvalues (eps_smallest_real) are computed",
    "eps_target": "targets and shift-and-invert are not implemented",
    "eps_target_magnitude": "targets and shift-and-invert are not implemented",
    "eps_target_real": "targets and shift-and-invert are not implemented",
    "eps_target_imaginary": "targets and shift-and-invert are not implemented",
    "eps_gen_non_hermitian": "the problems here are symmetric (A symmetric, M symmetric positive definite)",
    "eps_non_hermitian": "the problems here are symmetric (A symmetric, M symmetric positive definite)",
    "eps_pos_gen_non_hermitian": "the problems here are symmetric (A symmetric, M symmetric positive definite)",
}


class LinearEigenproblem:
    """The generalised eigenproblem ``A x = lambda M x`` (firedrake.LinearEigenproblem).

    ``A``: a symmetric form -- :class:`Form` (with ``kappa`` and ``ds``), :class:`Elasticity`, :class:`SpectralForm` or
    :class:`InteriorPenalty`.  ``M``: a :class:`Form` on the same space (default ``mass(V)``) or the lumped mass
    ``SpectralForm(V, 0.0, 1.0)``.  ``bcs``: DirichletBCs; only the restricted problem is built (``restrict=True``, the
    reference's default): the constrained rows are zeroed in the initial block and after every action and
    preconditioner application, so every iterate lies in the restricted space, no spurious boundary eigenvalue appears
    and the eigenfunctions vanish on the Dirichlet nodes.  ``bc_shift`` is ignored there, as in Firedrake.

    Refused by name: nonsymmetric forms, Taylor-Hood and mixed forms, an M on another space, partitioned spaces and
    ``restrict=False``."""

    def __init__(self, A, M=None, bcs=(), bc_shift=0.0, restrict=True):
        if any(getattr(getattr(F, "V", None), "family", "CG") == "NCF" for F in (A, M)):
            raise NotImplementedError("the eigensolver does not take NCF (H(div)) spaces: MixedPoisson, the only "
                                      "form on NCF, is indefinite")
        if isinstance(A, _MIXED) or isinstance(M, _MIXED):
            raise NotImplementedError(f"{type(A if isinstance(A, _MIXED) else M).__name__}: Taylor-Hood and mixed "
                                      f"forms are not implemented in the eigensolver")
        if isinstance(A, _NONSYMMETRIC):
            raise NotImplementedError(f"{type(A).__name__} is nonsymmetric: the eigensolver takes symmetric forms "
                                      f"(Form, Elasticity, SpectralForm, InteriorPenalty)")
        if not isinstance(A, _OPERATORS):
            raise TypeError(f"A: {type(A).__name__} is not one of Form, Elasticity, SpectralForm, InteriorPenalty")
        V = A.V
        if M is None:
            M = mass(V)
        if isinstance(M, _NONSYMMETRIC):
            raise NotImplementedError(f"{type(M).__name__} is nonsymmetric: M must be symmetric positive definite")
        if isinstance(M, SpectralForm):
            if M.alpha != 0.0 or M.beta <= 0.0:
                raise NotImplementedError("M as a SpectralForm is the lumped mass SpectralForm(V, 0.0, beta > 0)")
        elif not isinstance(M, Form):
            raise TypeError(f"M: {type(M).__name__} is not a Form (e.g. mass(V)) or the lumped mass "
                            f"SpectralForm(V, 0.0, 1.0)")
        elif M.alpha < 0.0 or M.beta <= 0.0:
            raise ValueError(f"M = Form(V, alpha={M.alpha}, beta={M.beta}) is not positive definite: M needs "
                             f"beta > 0 and alpha >= 0 (e.g. mass(V))")
        if M.V is not V:
            raise ValueError("M is on another function space than A: both forms must be on the same space")
        if V.dof_dset.halo is not None:
            raise NotImplementedError("the eigensolver on a partitioned space is not implemented")
        if not restrict:
            raise NotImplementedError("restrict=False is not implemented: only the restricted problem is built "
                                      "(the constrained rows are removed, bc_shift does not apply)")
        self.A, self.M, self.bcs = A, M, tuple(bcs)
        self.bc_shift, self.restrict = bc_shift, True
        self.output_space = V

    @property
    def singular(self):
        """True when A has a null space a multigrid preconditioner cannot handle: no Dirichlet rows, no mass term
        (beta == 0) and no ds terms."""
        return not self.bcs and getattr(self.A, "beta", 0.0) == 0.0 and not getattr(self.A, "ds", ())


def _flatten(sp):
    out = {}
    for k, v in (sp or {}).items():
        if isinstance(v, dict):
            out.update({f"{k}_{kk}": vv for kk, vv in _flatten(v).items()})
        else:
            out[k] = v
    return out


def eigensolver_options(sp, n_evals):
    """The LOBPCG settings of ``solver_parameters`` (PETSc / SLEPc names, nested dicts flattened): a dict with the keys
    of ``_DEFAULTS``, the blocksize resolved, and the ``st_pmg_*`` keys as the ``pmg_*`` options of
    :func:`assemble.pmg_options`.  Anything this solver does not do is refused by name."""
    flat = _flatten(sp)
    o = dict(_DEFAULTS)
    pmg = {}
    for k, v in flat.items():
        if k in _REFUSED:
            raise NotImplementedError(f"{k}: {_REFUSED[k]}")
        if k in _FLAGS:
            continue
        if k.startswith("st_pmg_"):
            pmg[k[3:]] = v
        elif k in _DEFAULTS:
            o[k] = v
        else:
            raise NotImplementedError(f"unknown eigensolver option {k}: the supported ones are "
                                      f"{', '.join(list(_DEFAULTS) + list(_FLAGS))} and st_pmg_*")
    if o["eps_type"] != "lobpcg":
        raise NotImplementedError(f"eps_type {o['eps_type']!r}: only 'lobpcg' (preconditioned LOBPCG) is implemented; "
                                  f"Krylov-Schur and the other SLEPc solvers are not")
    if o["st_type"] != "precond":
        raise NotImplementedError(f"st_type {o['st_type']!r}: only 'precond' (shift-and-invert, Cayley and shift "
                                  f"transforms are not implemented)")
    if o["st_ksp_type"] != "preonly":
        raise NotImplementedError(f"st_ksp_type {o['st_ksp_type']!r}: only 'preonly' (one preconditioner "
                                  f"application, no inner solve)")
    if o["st_pc_type"] not in ("none", "jacobi", "mg", "python"):
        raise NotImplementedError(f"st_pc_type {o['st_pc_type']!r}: 'none', 'jacobi', 'mg' or 'python' "
                                  f"(firedrake.PMGPC / firedrake.P1PC)")
    n_evals = int(n_evals)
    if not 1 <= n_evals <= MAX_BLOCKSIZE:
        raise NotImplementedError(f"n_evals = {n_evals}: 1..{MAX_BLOCKSIZE} (the LOBPCG block holds at most "
                                  f"{MAX_BLOCKSIZE} columns, so that 3 * blocksize <= {_lib.BV_MAX_COLUMNS})")
    bs = o["eps_lobpcg_blocksize"]
    if bs is None:
        bs = min(n_evals + -(-n_evals // 4), MAX_BLOCKSIZE)
    bs = int(bs)
    if bs > MAX_BLOCKSIZE:
        raise NotImplementedError(f"eps_lobpcg_blocksize {bs}: at most {MAX_BLOCKSIZE} (3 * blocksize <= "
                                  f"{_lib.BV_MAX_COLUMNS})")
    if bs < n_evals:
        raise ValueError(f"eps_lobpcg_blocksize {bs} is smaller than n_evals = {n_evals}")
    o["eps_lobpcg_blocksize"] = bs
    o["eps_tol"], o["eps_max_it"] = float(o["eps_tol"]), int(o["eps_max_it"])
    o["pmg"] = pmg
    return o


def _ptrs(dats):
    return (C.c_void_p * len(dats))(*[d.device_ptr for d in dats])


class _Block:
    """Dats as the columns of a block vector (the operands of fdb_bv_dot / fdb_bv_mult)."""

    def __init__(self, n):
        self.n = n

    def dot(self, xs, ys):
        """G[i, j] = x_i . y_j on the device; G (m x k) comes back to the host."""
        g = np.empty((len(xs), len(ys)))
        _lib.check(_lib.lib().fdb_bv_dot(self.n, len(xs), _ptrs(xs), len(ys), _ptrs(ys),
                                         g.ctypes.data_as(C.POINTER(C.c_double))), "fdb_bv_dot")
        return g

    def mult(self, ys, xs, Q, beta=0.0, alpha=1.0):
        """y_j = beta y_j + alpha sum_i x_i Q[i, j]."""
        Q = np.ascontiguousarray(Q, dtype=np.float64)
        assert Q.shape == (len(xs), len(ys))
        _lib.check(_lib.lib().fdb_bv_mult(self.n, len(ys), _ptrs(ys), float(beta), float(alpha), len(xs), _ptrs(xs),
                                          Q.ctypes.data_as(C.POINTER(C.c_double))), "fdb_bv_mult")
        for y in ys:
            y._device_written()


class LinearEigensolver:
    """The ``n_evals`` smallest eigenpairs of a :class:`LinearEigenproblem` (firedrake.LinearEigensolver) by
    preconditioned block LOBPCG on the device.  ``solve()`` returns the number of converged pairs;
    ``eigenvalue(i)`` the i-th smallest eigenvalue and ``eigenfunction(i)`` (real Dat, zero imaginary Dat), the
    eigenvectors M-orthonormal.

    ``solver_parameters`` (PETSc / SLEPc names; nested dicts are flattened):

    - ``eps_type`` "lobpcg", the default and the only type.  Firedrake's own default is Krylov-Schur, which needs a
      sparse LU for the shift-and-invert that finds the smallest eigenvalues; LOBPCG needs none and reuses the
      preconditioners of :func:`assemble.solve`.
    - ``eps_smallest_real`` (the only target), ``eps_gen_hermitian`` / ``eps_hermitian`` (flags).
    - ``eps_tol`` (1e-10), ``eps_max_it`` (500), ``eps_lobpcg_blocksize`` (n_evals + ceil(n_evals / 4), at most
      ``MAX_BLOCKSIZE`` = 21; the extra columns are guard vectors, not reported).
    - ``st_type`` "precond", ``st_ksp_type`` "preonly" and ``st_pc_type``: "none", "jacobi" (the diagonal of A), "mg"
      (a V-cycle on ``hierarchy``) or "python" with ``st_pc_python_type`` "firedrake.PMGPC" / "firedrake.P1PC" and
      the ``st_pmg_*`` options; built on A as :func:`assemble.solve` builds them, with the same refusals.  mg and
      p-multigrid on a singular A (no Dirichlet rows, beta == 0, no ds) are refused.

    Convergence of pair i: ||A x_i - lambda_i M x_i||_2 <= eps_tol * max(|lambda_i|, theta) * ||M x_i||_2, with theta
    the largest Ritz value of the block, so that a zero eigenvalue (a rigid-body mode) is measured on the block's
    scale.  This is not SLEPc's exact normalisation.  A converged pair is locked: frozen and left out of the search (hard
    locking; soft locking, which keeps converged columns in the Rayleigh-Ritz, let them drift off near the attainable
    accuracy).  A pair is locked only on the residual of fresh A and M actions on its column, as the carried AX and MX
    only nominate it, and the active columns' products are recomputed every ``REFRESH_EVERY`` iterations; the run ends when the ``n_evals`` smallest Ritz values of the block are all locked, otherwise ``ConvergenceError``
    after ``eps_max_it`` iterations.  ``seed`` seeds the random initial block."""

    def __init__(self, problem: LinearEigenproblem, n_evals, *, solver_parameters=None, hierarchy=None, seed=0):
        self._problem = problem
        self.n_evals = int(n_evals)
        self.options = o = eigensolver_options(solver_parameters, n_evals)
        self.hierarchy, self.seed = hierarchy, seed
        A, V = problem.A, problem.output_space
        pc = o["st_pc_type"]
        if pc in ("mg", "python"):
            which = "geometric multigrid" if pc == "mg" else "p-multigrid (PMGPC / P1PC)"
            if isinstance(A, SpectralForm):
                raise NotImplementedError(f"st_pc_type {pc!r} on a SpectralForm: 'none' or 'jacobi' ({which} is not "
                                          f"implemented for the SEM operator)")
            if getattr(V, "family", "CG") == "DQ":
                raise NotImplementedError(f"st_pc_type {pc!r} on a DQ space: 'none' or 'jacobi' (there is no DQ "
                                          f"multigrid)")
            if problem.singular:
                raise NotImplementedError(f"st_pc_type {pc!r} on a singular A (no Dirichlet rows, beta == 0 and no "
                                          f"ds terms): {which} needs an invertible operator; use 'jacobi'")
            if pc == "mg" and hierarchy is None:
                raise ValueError("st_pc_type mg needs the mesh hierarchy")
        self.nconv = 0
        self.iterations = 0
        self.residuals = None          # the relative residuals of the block's columns at the last iteration
        self.theta = None              # the largest |Ritz value| of the block, the scale of the criterion
        self._values = None
        self._vectors = None

    # ------------------------------------------------------------------ the operators
    def _setup(self):
        prob, o = self._problem, self.options
        A, M, V, bcs = prob.A, prob.M, prob.output_space, prob.bcs
        bs = o["eps_lobpcg_blocksize"]
        self._bv = _Block(V.node_set.size * V.cdim)
        # the block vectors: X, W, P, their images under A and M, and a spare set for the new P (which first holds
        # the residuals)
        names = ("X", "AX", "MX", "W", "AW", "MW", "P", "AP", "MP", "Q", "AQ", "MQ")
        self._v = {k: [V.dat() for _ in range(bs)] for k in names}
        # one assembler per input column, keyed by the Dat and made on first use.  X and W (and AX and AW, MX and
        # MW) trade places together, as P and Q do, so each assembler keeps one output Dat and its parloop is built
        # once
        self._aA, self._aM = {}, {}
        self._lumped = None
        if isinstance(M, SpectralForm):
            self._lumped = ImplicitMatrixContext(M).getDiagonal(V.dat())
        sp = {"pc_type": o["st_pc_type"]}
        if o["st_pc_type"] == "python":
            sp["pc_python_type"] = o["st_pc_python_type"]
            sp.update(o["pmg"])
        self._pc = _preconditioner(A, None, bcs, sp, self.hierarchy)

    def _restrict(self, dat):
        for bc in self._problem.bcs:
            bc.zero(dat)

    def _apply(self, op, x, out):
        """out = A x (op "A") or M x (op "M") for a block column x, zero on the constrained rows."""
        if op == "A":
            if id(x) not in self._aA:
                self._aA[id(x)] = OneFormAssembler(self._problem.A, x, ())
            self._aA[id(x)].assemble(tensor=out)
        elif self._lumped is not None:
            _lib.check(_lib.lib().fdb_vec_pointwise_mult(self._lumped._data.size, x.device_ptr,
                                                         self._lumped.device_ptr, out.device_ptr))
            out._device_written()
        else:
            if id(x) not in self._aM:
                self._aM[id(x)] = OneFormAssembler(self._problem.M, x, ())
            self._aM[id(x)].assemble(tensor=out)
        self._restrict(out)

    def _precondition(self, r, z):
        """z = P^-1 r on the free rows; a multigrid cycle starts from the z passed in, so z starts at zero."""
        if self._pc is None:
            _lib.check(_lib.lib().fdb_memcpy_d2d(z.device_ptr, r.device_ptr, r.nbytes))
            z._device_written()
        else:
            z.zero()
            z.device_ptr
            self._pc(r, z)
        self._restrict(z)

    # ------------------------------------------------------------------ Rayleigh-Ritz
    @staticmethod
    def _normaliser(G):
        """R^-1 of the Cholesky factor G = R^T R, or None when the Cholesky fails or R's condition number (estimated
        from the 2-norm condition of G) exceeds 1e14."""
        import scipy.linalg as sl
        try:
            R = sl.cholesky(G, lower=False)
        except (np.linalg.LinAlgError, ValueError):
            return None
        if not np.all(np.isfinite(R)) or np.linalg.cond(R) > 1e14:
            return None
        return sl.solve_triangular(R, np.eye(len(G)), lower=False)

    @staticmethod
    def _ritz(gA, gB, D, nev, strict=False):
        """The nev smallest Ritz pairs of (gA, gB) in the basis S D: eigh of D^T gA D, D^T gB D restricted to the
        numerically nonsingular part of D^T gB D.  Returns (theta, C) with S C the M-orthonormal Ritz vectors.
        ``strict``: raise LinAlgError instead when D^T gB D has a condition number above 1e10 (the caller then drops
        P, which near convergence becomes nearly parallel to W)."""
        import scipy.linalg as sl
        a = D.T @ gA @ D
        b = D.T @ gB @ D
        a, b = (a + a.T) / 2, (b + b.T) / 2
        s, U = sl.eigh(b)
        if strict and s.min() < 1e-10 * s.max():
            raise np.linalg.LinAlgError("the basis [X, W, P] is ill-conditioned")
        keep = s > 1e-14 * s.max()
        T = U[:, keep] / np.sqrt(s[keep])
        if T.shape[1] < nev:
            raise np.linalg.LinAlgError("the LOBPCG basis lost rank")
        theta, c = sl.eigh(T.T @ a @ T)
        return theta[:nev], D @ T @ c[:, :nev]

    # ------------------------------------------------------------------ LOBPCG
    def solve(self):
        """Run LOBPCG; returns nconv, the number of the first ``n_evals`` pairs that converged (all of them, or a
        ConvergenceError is raised)."""
        o = self.options
        self._setup()
        V = self._problem.output_space
        bs, nev, tol = o["eps_lobpcg_blocksize"], self.n_evals, o["eps_tol"]
        v, bv = self._v, self._bv
        # the random initial block, zero on the constrained rows, uploaded once
        rng = np.random.default_rng(self.seed)
        constrained = np.unique(np.concatenate([bc.nodes for bc in self._problem.bcs])) if self._problem.bcs else \
            np.zeros(0, dtype=np.int32)
        for j in range(bs):
            x0 = rng.standard_normal((V.node_count, V.cdim) if V.cdim > 1 else V.node_count)
            x0[constrained] = 0.0
            x = v["X"][j]
            x.data_wo[...] = x0
            x.device_ptr
        for j in range(bs):
            self._apply("A", v["X"][j], v["AX"][j])
            self._apply("M", v["X"][j], v["MX"][j])
        # Rayleigh-Ritz on the initial block
        gA, gB = bv.dot(v["X"], v["AX"]), bv.dot(v["X"], v["MX"])
        try:
            lam, Cx = self._ritz(gA, gB, np.eye(bs), bs)
        except np.linalg.LinAlgError:
            raise ConvergenceError(f"LOBPCG cannot start: the initial block of {bs} columns is rank-deficient in the "
                                   f"M inner product (more columns than free rows?)", "DIVERGED_BREAKDOWN") from None
        for k in ("", "A", "M"):
            bv.mult(v[k + "W"], v[k + "X"], Cx)
        self._swap("X", "W")
        # hard locking: a pair whose residual meets eps_tol is frozen (X, AX and MX columns and lambda); the others
        # are searched for in the M-orthogonal complement of every X column.  Rotating converged columns again, as
        # soft locking does, lets them drift off at the edge of the attainable accuracy.  AX and MX are carried by
        # combination, so a pair is locked only on the residual of fresh A and M actions on its column
        locked = np.zeros(bs, dtype=bool)
        have_p, pcol = False, []                         # pcol[c]: the X column whose P is P[c]
        worst = np.inf
        self.refreshed = 0                               # columns whose AX, MX were recomputed to confirm a lock
        for it in range(o["eps_max_it"] + 1):
            res = self._residuals(lam)
            # every REFRESH_EVERY iterations every active column is refreshed too: a carried residual that drifted
            # above eps_tol would otherwise never be corrected
            due = it > 0 and it % REFRESH_EVERY == 0
            cand = np.flatnonzero(~locked & ((res <= tol) | due))
            if len(cand):
                for j in cand:
                    self._apply("A", v["X"][j], v["AX"][j])
                    self._apply("M", v["X"][j], v["MX"][j])
                self.refreshed += len(cand)
                res = self._residuals(lam)
                locked[cand] = res[cand] <= tol
            self.residuals = res.copy()
            first = np.argsort(lam, kind="stable")[:nev]
            worst = res[first].max()
            self.iterations = it
            if locked[first].all():
                break
            if it == o["eps_max_it"]:
                raise ConvergenceError(f"LOBPCG did not converge in {it} iterations: the worst relative residual of "
                                       f"the first {nev} pairs is {worst:.3e} (eps_tol {tol:.1e})",
                                       "DIVERGED_ITS")
            act = np.flatnonzero(~locked)
            na = len(act)
            for a, j in enumerate(act):
                self._precondition(v["Q"][j], v["W"][a])
            W, AW, MW = v["W"][:na], v["AW"][:na], v["MW"][:na]
            cols = lambda k, idx: [v[k][j] for j in idx]
            pidx = [pcol.index(j) for j in act] if have_p else []
            # W <- W - X (X^T M W) and P <- P - X (X^T M P), with X^T M = (MX)^T: the search directions M-orthogonal
            # to every X column (W's component along X dominates as X converges; P mixes columns locked since it was
            # formed).  Then their A and M products by fresh actions: carried through the projection, they would keep
            # the absolute error of the large terms that cancel in it
            blocks_wp = [W] + ([cols("P", pidx)] if have_p else [])
            for blk in blocks_wp:
                bv.mult(blk, v["X"], bv.dot(v["MX"], blk), beta=1.0, alpha=-1.0)
            for a in range(na):
                self._apply("A", W[a], AW[a])
                self._apply("M", W[a], MW[a])
            if have_p:
                for c in pidx:
                    self._apply("A", v["P"][c], v["AP"][c])
                    self._apply("M", v["P"][c], v["MP"][c])
            S, AS, MS = cols("X", act) + W, cols("AX", act) + AW, cols("MX", act) + MW
            if have_p:
                S, AS, MS = S + cols("P", pidx), AS + cols("AP", pidx), MS + cols("MP", pidx)
            gA, gB = bv.dot(S, AS), bv.dot(S, MS)
            # Cholesky-QR of W and P in the M inner product, applied through the coefficients (no extra pass); P is
            # dropped for this iteration when its factor fails or is ill-conditioned (Hetmaniuk-Lehoucq)
            nw = 2 * na
            Dw = self._normaliser(gB[na:nw, na:nw])
            if Dw is None:                              # W nearly dependent: let the rank filter of _ritz handle it
                Dw = np.diag(1.0 / np.sqrt(np.maximum(np.diag(gB)[na:nw], 1e-300)))
            Dp = self._normaliser(gB[nw:, nw:]) if have_p else None
            if have_p and Dp is None:
                have_p = False
            ns = nw + (na if have_p else 0)
            gA, gB = gA[:ns, :ns], gB[:ns, :ns]
            blocks = [np.eye(na), Dw] + ([Dp] if have_p else [])
            try:
                theta, Cs = self._ritz(gA, gB, _blockdiag(blocks), na, strict=have_p)
            except np.linalg.LinAlgError:
                if not have_p:
                    raise ConvergenceError(f"LOBPCG broke down at iteration {it}: the Rayleigh-Ritz basis lost rank "
                                           f"(worst relative residual {worst:.3e})", "DIVERGED_BREAKDOWN")
                have_p, ns = False, nw
                theta, Cs = self._ritz(gA[:nw, :nw], gB[:nw, :nw], _blockdiag(blocks[:2]), na)
            lam[act] = theta
            # new P = [W, P] C_{W,P} into Q; new X = X C_X + P into W's columns, which then take the active columns'
            # places in X; the same combinations give AX, MX, AP and MP
            Cx, Cwp = Cs[:na], Cs[na:ns]
            for k in ("", "A", "M"):
                src = v[k + "W"][:na] + (cols(k + "P", pidx) if have_p else [])
                bv.mult(v[k + "Q"][:na], src, Cwp)
            for k in ("", "A", "M"):
                bv.mult(v[k + "W"][:na], cols(k + "X", act) + v[k + "Q"][:na], np.vstack([Cx, np.eye(na)]))
            for a, j in enumerate(act):
                for k in ("", "A", "M"):
                    v[k + "X"][j], v[k + "W"][a] = v[k + "W"][a], v[k + "X"][j]
            self._swap("P", "Q")
            have_p, pcol = True, list(act)
        first = np.argsort(lam, kind="stable")[:nev]
        self._values = np.asarray(lam[first], dtype=float)
        self._vectors = [v["X"][j] for j in first]
        self.nconv = nev
        return self.nconv

    def _residuals(self, lam):
        """||A x_i - lam_i M x_i||_2 / (max(|lam_i|, theta) ||M x_i||_2) from the carried AX and MX: R into Q by one
        fdb_bv_mult, the norms from the diagonal of one fdb_bv_dot of [R, MX]."""
        v, bs = self._v, len(lam)
        self._bv.mult(v["Q"], v["AX"] + v["MX"], np.vstack([np.eye(bs), -np.diag(lam)]))
        RM = v["Q"] + v["MX"]
        g = np.diag(self._bv.dot(RM, RM))
        rn, mn = np.sqrt(np.maximum(g[:bs], 0.0)), np.sqrt(np.maximum(g[bs:], 0.0))
        self.theta = np.abs(lam).max()
        return rn / (np.maximum(np.abs(lam), self.theta) * np.where(mn > 0, mn, 1.0))

    def _swap(self, a, b):
        v = self._v
        for k in ("", "A", "M"):
            v[k + a], v[k + b] = v[k + b], v[k + a]

    # ------------------------------------------------------------------ results
    def eigenvalue(self, i):
        """The i-th smallest eigenvalue (0 <= i < nconv)."""
        if not 0 <= i < self.nconv:
            raise IndexError(f"eigenvalue {i}: {self.nconv} converged")
        return float(self._values[i])

    def eigenfunction(self, i):
        """(real part, imaginary part) of the i-th eigenvector, M-orthonormal; the imaginary part is zero."""
        if not 0 <= i < self.nconv:
            raise IndexError(f"eigenfunction {i}: {self.nconv} converged")
        V = self._problem.output_space
        re = V.dat()
        src = self._vectors[i]
        _lib.check(_lib.lib().fdb_memcpy_d2d(re.device_ptr, src.device_ptr, src.nbytes))
        re._device_written()
        return re, V.dat()


def _blockdiag(blocks):
    n = sum(len(b) for b in blocks)
    D = np.zeros((n, n))
    o = 0
    for b in blocks:
        D[o:o + len(b), o:o + len(b)] = b
        o += len(b)
    return D
