"""Host logic of the spectral-element wave equation on the CPU, against a recording stand-in for the engine: the exact
engine calls of a leapfrog step (one SEM action, one point load into its output, one fused leapfrog pass and one point
evaluation into the device trace, and no device-to-host copy until the traces come back), wave_dt_bound's use of the
SEM action and 1/m, and the refusals of SpectralForm, assemble and solve."""
import numpy as np
import pytest

import _mock_engine as me
import _sem_oracle as so
from firedrake_b200 import _lib
from firedrake_b200.utility_meshes import ExtrudedHexMesh

SEM = (_lib.FORM_SPECTRAL_HELMHOLTZ, _lib.FORM_SPECTRAL_HELMHOLTZ_COEF)


class SemRecorder(me.MockEngine):
    """Runs the spectral kernels as products with a given matrix A (the oracle's), the point kernels and
    fdb_vec_leapfrog in NumPy, and records every one of those calls and every device-to-host copy."""

    def __init__(self, A):
        super().__init__(None)
        self.A, self.calls = A, []

    def fdb_kernel_create(self, desc, out):
        d = me._obj(desc)
        if d.form not in SEM:
            return super().fdb_kernel_create(desc, out)
        self._next += 1
        self.kernels[self._next] = dict(kind="sem", form=d.form, diagonal=bool(d.diagonal), alpha=d.alpha,
                                        beta=d.beta)
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        k = self.kernels[me._addr(h)]
        if k["kind"] != "sem":
            self.calls.append(("jit",) if k["kind"] == "jit" else ("kernel", k["kind"]))
            return super().fdb_kernel_call(h, ca)
        a = me._obj(ca)
        n = self.A.shape[0]
        y = me._view(a.args[0], n)
        if k["diagonal"]:
            self.calls.append(("diagonal", k["form"], a.nargs))
            y += self.A.diagonal()
        else:
            self.calls.append(("action", k["form"], a.nargs))
            y += self.A @ me._view(a.args[2], n)
        return 0

    def fdb_vec_leapfrog(self, n, dt2, minv, r, u, up):
        self.calls.append(("leapfrog", n, dt2))
        upv = me._view(up, n)
        upv[:] = 2.0 * me._view(u, n) - upv - dt2 * me._view(minv, n) * me._view(r, n)
        return 0

    def _pw(self, npts, nper, idx, w):
        return (me._view(idx, npts * nper, np.int32).reshape(npts, nper).copy(),
                me._view(w, npts * nper).reshape(npts, nper).copy())

    def fdb_point_eval(self, npts, nper, idx, w, u, out):
        self.calls.append(("eval", npts))
        n = self.A.shape[0]
        me._view(out, npts)[:] = so.evaluate(self._pw(npts, nper, idx, w), me._view(u, n))
        return 0

    def fdb_point_load(self, npts, nper, idx, w, a, scale, y):
        self.calls.append(("load", npts, scale))
        n = self.A.shape[0]
        me._view(y, n)[:] += scale * so.adjoint(self._pw(npts, nper, idx, w), me._view(a, npts), n)
        return 0

    def fdb_memcpy_d2h(self, dst, src, n):
        self.calls.append(("d2h", n))
        return self._copy(dst, src, n)


class recording(me.install):
    def __init__(self, A):
        self.engine = SemRecorder(A)


def _setup(p=2):
    from firedrake_b200.assemble import FunctionSpace
    mesh = ExtrudedHexMesh(3, 3, 3, warp=0.05, permute_seed=1)
    V = FunctionSpace(mesh, p)
    kap = np.where(V.V.dof_coordinates()[:, 2] > 0.5, 2.0, 1.0)
    return mesh, V, kap, so.operator(mesh, V.V, p, 1.0, 0.0, kap)


@pytest.mark.parametrize("steps", [4, 5])
def test_leapfrog_step_calls(steps):
    """Per step exactly: the SEM action [y, coords, u, kappa], the point load (scale -1) into its output, one
    fdb_vec_leapfrog over every node with dt^2, one point evaluation; one device-to-host copy (the traces) after the
    loop.  The traces and the final (u, u_prev) are the oracle recurrence's, for an even and an odd step count."""
    from firedrake_b200.assemble import PointEvaluator, SpectralForm, leapfrog, ricker
    mesh, V, kap, A = _setup()
    m = so.operator(mesh, V.V, 2, 0.0, 1.0).diagonal()
    dt = 0.01
    amp = ricker(np.arange(steps) * dt, 5.0, 0.02)[:, None]
    with recording(A) as eng:
        F = SpectralForm(V, 1.0, 0.0, V.dat(kap))
        src = PointEvaluator(V, [[0.5, 0.5, 0.5]])
        rec = PointEvaluator(V, [[0.2, 0.3, 0.4], [0.7, 0.6, 0.5]])
        u0 = np.random.default_rng(0).standard_normal(V.node_count)
        u, up = V.dat(u0.copy()), V.dat(u0.copy())      # (a Dat wraps its array)
        md = V.dat(m)
        eng.calls.clear()
        tr = leapfrog(F, u, up, dt, steps, md, sources=(src, amp), receivers=rec)
        calls = list(eng.calls)
        uo, upo = u.data_ro.copy(), up.data_ro.copy()
    first = next(i for i, c in enumerate(calls) if c[0] == "action")
    loop = [c for c in calls[first:] if c[0] in ("action", "load", "leapfrog", "eval", "d2h", "kernel", "diagonal")]
    n = V.node_count
    step = [("action", _lib.FORM_SPECTRAL_HELMHOLTZ_COEF, 4), ("load", 1, -1.0), ("leapfrog", n, dt * dt),
            ("eval", 2)]
    assert loop[:4 * steps] == step * steps
    assert [c[0] for c in loop[4 * steps:]][:1] == ["d2h"]             # the traces, once
    assert not any(c[0] == "d2h" for c in calls[first:first + len(step) * steps])
    want_u, want_up, want_tr = so.leapfrog(A, m, u0, u0, dt, steps, src=(src.idx, src.w), amp=amp,
                                           rec=(rec.idx, rec.w))
    assert np.allclose(tr, want_tr, rtol=1e-13, atol=1e-13 * np.abs(want_tr).max())
    assert np.allclose(uo, want_u, rtol=1e-13, atol=1e-13) and np.allclose(upo, want_up, rtol=1e-13, atol=1e-13)


def test_wave_dt_bound_uses_sem_action_and_inverse_mass():
    """Only SEM actions (no diagonal, no other form) and the reciprocal of m: the bound is 2/sqrt(1.1 lambda_max) of
    M^-1 K to the accuracy of 30 Lanczos steps."""
    from firedrake_b200.assemble import SpectralForm, wave_dt_bound
    mesh, V, kap, A = _setup()
    m = so.operator(mesh, V.V, 2, 0.0, 1.0).diagonal()
    with recording(A) as eng:
        F = SpectralForm(V, 1.0, 0.0, V.dat(kap))
        dt = wave_dt_bound(F, V.dat(m), steps=30)
        calls = list(eng.calls)
    acts = [c for c in calls if c[0] in ("action", "diagonal", "kernel")]
    assert acts and all(c == ("action", _lib.FORM_SPECTRAL_HELMHOLTZ_COEF, 4) for c in acts)
    assert len(acts) <= 30
    lmax = np.linalg.eigvalsh((A.toarray() / np.sqrt(m)[:, None]) / np.sqrt(m)[None, :]).max()
    assert abs(dt - 2.0 / np.sqrt(1.1 * lmax)) < 1e-3 * dt


def test_refusals():
    from firedrake_b200.assemble import FunctionSpace, SpectralForm, assemble, leapfrog, solve
    mesh = ExtrudedHexMesh(2, 2, 2)
    V = FunctionSpace(mesh, 2)
    F = SpectralForm(V)
    with pytest.raises(NotImplementedError, match="no assembled SEM matrix"):
        assemble(F)
    with pytest.raises(NotImplementedError, match="no assembled SEM matrix"):
        F.kernel(2)
    for sp, match in ((dict(mat_type="aij"), "no assembled SEM matrix"), (dict(mat_type="is"), "no assembled"),
                      (dict(pc_type="mg"), "geometric multigrid"),
                      (dict(pc_type="python", pc_python_type="firedrake.PMGPC"), "p-multigrid")):
        with pytest.raises(NotImplementedError, match=match):
            solve(F, V.dat(), V.dat(), solver_parameters=sp)
    with pytest.raises(NotImplementedError, match="DQ"):
        SpectralForm(FunctionSpace(mesh, 2, family="DQ"))
    with pytest.raises(NotImplementedError, match="scalar"):
        SpectralForm(FunctionSpace(mesh, 2, cdim=3))
    with pytest.raises(NotImplementedError, match="ds terms"):
        SpectralForm(V, ds=((1.0, "bottom"),))
    with pytest.raises(NotImplementedError, match="degree 6"):
        SpectralForm(FunctionSpace(mesh, 6))
    with pytest.raises(TypeError, match="SpectralForm"):
        leapfrog(object(), V.dat(), V.dat(), 0.1, 1, V.dat())
