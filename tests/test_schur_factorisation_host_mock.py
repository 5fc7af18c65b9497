"""Host logic of the "lower" and "upper" Schur factorisations of the Taylor-Hood fieldsplit on the CPU, with the
mock engine of tests/test_navier_stokes_host_mock.py (Stokes and Navier-Stokes through the NumPy oracles): the
signs with exact inner inverses injected, Stokes solves and Newton on the cavity against scipy, and the option
refusals.  The device runs are tests/test_schur_factorisation_gpu.py."""
import numpy as np
import pytest

import _stokes_oracle as so
import test_navier_stokes_gpu as tn
import test_navier_stokes_host_mock as nm
import test_stokes_gpu as tg
import test_stokes_host_mock as sm
from firedrake_b200.fiat_lite import interval_element


@pytest.fixture()
def mock(oracle):
    with nm.install(oracle) as eng:
        yield eng


def _exact_inverses(mesh, V, Q, F, bcs):
    """Dense F^-1 of the constrained velocity block and (B F^-1 B^T)^-1 of the oracle's Stokes system."""
    geo = (V.V.cell_node_map, V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    K = so.global_matrix(interval_element(V.degree), mesh.coordinates, geo, (Q.V.cell_node_map, Q.V.offset),
                         V.node_count, Q.node_count, F.mu, F.beta)
    bd = so.velocity_dofs(np.unique(np.concatenate([bc.nodes for bc in bcs])))
    A, Bt, B, _ = so.blocks(so.constrained(K, bd), V.node_count)
    Finv = np.linalg.inv(A.toarray())
    return Finv, np.linalg.pinv(B.toarray() @ Finv @ Bt.toarray())


@pytest.mark.parametrize("fact", ["lower", "upper"])
def test_signs_with_exact_inverses(mock, fact):
    """With P_0 = F^-1 and P_1 = (B F^-1 B^T)^-1 injected, A M - I is nilpotent on the mean-free pressures
    ((A M - I)^2 = 0, so GMRES converges in 2 iterations); with P_1 negated it is not."""
    from firedrake_b200.assemble import (StokesMatrixContext, _pressure_mean_remover, _schur_factorisation,
                                         gmres)
    mesh, V, Q, F, bcs = tg._cavity(3)
    Finv, Sinv = _exact_inverses(mesh, V, Q, F, bcs)
    A = StokesMatrixContext(F, bcs)
    remove = _pressure_mean_remover(Q)

    def Mu(r, z):
        z.data[:] = (Finv @ r.data_ro.ravel()).reshape(-1, 3)

    rng = np.random.default_rng(1)
    b = F.dat(rng.standard_normal((V.node_count, 3)), rng.standard_normal(Q.node_count))
    for bc in bcs:
        bc.zero(b[0])
    remove(b)
    for sign in (1.0, -1.0):
        def Mp(r, z, sign=sign):
            z.data[:] = sign * (Sinv @ r.data_ro)

        M = _schur_factorisation(fact, Mu, Mp, A, F.dat, remove)

        def T(v):
            z, y = F.dat(), F.dat()
            M(v, z)
            A.mult(z, y)
            y.axpy(-1.0, v)
            return y

        rest = T(T(b)).norm() / b.norm()
        if sign > 0:
            assert rest < 1e-9, rest
            x = F.dat()
            for d in x:
                d.device_ptr
            its, hist = gmres(A, b, x, M, rtol=1e-10, restart=30, maxit=10)
            assert its <= 2 and hist[-1] <= 1e-10 * hist[0], (its, hist)
        else:
            assert rest > 0.1, rest


@pytest.mark.parametrize("fact", ["lower", "upper"])
@pytest.mark.parametrize("pc0", ["jacobi", "mg"])
def test_stokes_solve_matches_scipy(mock, fact, pc0):
    from firedrake_b200.assemble import solve
    from firedrake_b200.mg import MeshHierarchy
    mesh, V, Q, F, bcs = tg._cavity(4)
    g = np.zeros((V.node_count, 3))
    g[bcs[1].nodes, 0] = 1.0
    up = F.dat()
    its, hist = solve(F, F.dat(), up, bcs, {**tg._fieldsplit(pc0), "pc_fieldsplit_schur_fact_type": fact},
                      hierarchy=MeshHierarchy(2, 2, 2, 1) if pc0 == "mg" else None, nullspace="constant")
    assert hist[-1] <= 1e-12 * hist[0]
    _, u_ref, p_ref = sm._reference(mesh, V, Q, bcs, g)
    assert np.abs(up[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    assert np.abs(up[1].data_ro - p_ref).max() < 1e-7 * np.abs(p_ref).max()


@pytest.mark.parametrize("fact", ["lower", "upper"])
def test_newton_matches_scipy(mock, fact):
    """The 4^3 cavity at Re = 10 with the factorised fieldsplit and the velocity V-cycle: scipy's Newton."""
    from firedrake_b200.assemble import solve_nonlinear
    from firedrake_b200.mg import MeshHierarchy
    mesh, V, Q, F, bcs = tn._cavity(4, 0.1)
    up = F.dat()
    hist, kits = solve_nonlinear(F, F.dat(), up, bcs,
                                 {**tn._fieldsplit("mg", 1e-10), "pc_fieldsplit_schur_fact_type": fact},
                                 hierarchy=MeshHierarchy(2, 2, 2, 1), nullspace="constant")
    assert hist[-1] <= 1e-10 * hist[0] and 2 <= len(kits) < 10, (hist, kits)
    u_ref, p_ref, _ = tn._scipy_cavity(mesh, V, Q, F, bcs)
    assert np.abs(up[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    assert np.abs(up[1].data_ro - p_ref).max() < 1e-7 * np.abs(p_ref).max()


def test_lower_takes_fewer_iterations_than_diag(mock):
    """Stokes on the 4^3 cavity with velocity Jacobi: "lower" and "upper" need fewer GMRES iterations than
    "diag"."""
    from firedrake_b200.assemble import solve
    _, V, Q, F, bcs = tg._cavity(4)
    its = {}
    for fact in ("diag", "lower", "upper"):
        its[fact], _ = solve(F, F.dat(), F.dat(), bcs,
                             {**tg._fieldsplit("jacobi"), "ksp_rtol": 1e-8, "pc_fieldsplit_schur_fact_type": fact},
                             nullspace="constant")
    assert its["lower"] < its["diag"] and its["upper"] < its["diag"], its


def test_refusals(mock):
    from firedrake_b200.assemble import solve, solve_nonlinear
    fs = {"pc_type": "fieldsplit", "pc_fieldsplit_type": "schur"}
    _, V, Q, F, bcs = tg._cavity(2)
    _, _, _, Fn, bcn = tn._cavity(2, 0.1)
    for fact in ("full", "self"):
        for run in (lambda sp: solve(F, F.dat(), F.dat(), bcs, sp),
                    lambda sp: solve_nonlinear(Fn, Fn.dat(), Fn.dat(), bcn, sp)):
            with pytest.raises(NotImplementedError, match=f"'{fact}': not built \\('diag' only, or 'lower' / "
                                                          f"'upper'\\)"):
                run({**fs, "pc_fieldsplit_schur_fact_type": fact})
    for extra, msg in (({"fieldsplit_0_ksp_type": "gmres"}, "preonly"),
                       ({"fieldsplit_1_pc_type": "python"}, "fieldsplit_1_pc_type"),
                       ({"fieldsplit_0_pc_type": "lu"}, "'jacobi' or 'mg'")):
        with pytest.raises(NotImplementedError, match=msg):
            solve(F, F.dat(), F.dat(), bcs, {**fs, "pc_fieldsplit_schur_fact_type": "lower", **extra})
