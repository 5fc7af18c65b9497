"""GPU tests of the "lower" and "upper" Schur factorisations of the Taylor-Hood fieldsplit (Stokes solves and
Newton for Navier-Stokes): the lid-driven cavity against scipy, and fewer GMRES iterations than the diagonal
factorisation with the same inner preconditioners."""
import numpy as np
import pytest

import test_navier_stokes_gpu as tn
import test_stokes_gpu as tg
import test_stokes_host_mock as sm

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fact", ["lower", "upper"])
def test_stokes_cavity_matches_scipy(engine, fact):
    """Q2-Q1 on 8^3, velocity V-cycle, constant nullspace: velocity within 1e-8 of scipy's solve, pressure within
    1e-7, and fewer iterations than "diag"."""
    from firedrake_b200.assemble import solve
    from firedrake_b200.mg import MeshHierarchy
    mesh, V, Q, F, bcs = tg._cavity(8)
    hier = MeshHierarchy(2, 2, 2, 2)
    its = {}
    for f in ("diag", fact):
        up = F.dat()
        its[f], hist = solve(F, F.dat(), up, bcs, {**tg._fieldsplit("mg"), "pc_fieldsplit_schur_fact_type": f},
                             hierarchy=hier, nullspace="constant")
        assert hist[-1] <= 1e-12 * hist[0]
    g = np.zeros((V.node_count, 3))
    g[bcs[1].nodes, 0] = 1.0
    _, u_ref, p_ref = sm._reference(mesh, V, Q, bcs, g)
    assert np.abs(up[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    assert np.abs(up[1].data_ro - p_ref).max() < 1e-7 * np.abs(p_ref).max()
    assert its[fact] < its["diag"], its


def test_navier_stokes_cavity_matches_scipy(engine):
    """Q2-Q1 on 8^3 at Re = 10, "lower" with the velocity V-cycle: scipy's Newton (velocity 1e-8, pressure 1e-7
    modulo a constant)."""
    from firedrake_b200.assemble import solve_nonlinear
    from firedrake_b200.mg import MeshHierarchy
    mesh, V, Q, F, bcs = tn._cavity(8, 0.1)
    up = F.dat()
    hist, kits = solve_nonlinear(F, F.dat(), up, bcs,
                                 {**tn._fieldsplit("mg", 1e-10), "pc_fieldsplit_schur_fact_type": "lower"},
                                 hierarchy=MeshHierarchy(2, 2, 2, 2), nullspace="constant")
    assert hist[-1] <= 1e-10 * hist[0] and len(kits) < 10, (hist, kits)
    u_ref, p_ref, _ = tn._scipy_cavity(mesh, V, Q, F, bcs)
    assert np.abs(up[0].data_ro.ravel() - u_ref).max() < 1e-8 * np.abs(u_ref).max()
    p = up[1].data_ro
    assert np.abs(p - p.mean() - p_ref).max() < 1e-7 * np.abs(p_ref).max()


def test_re100_iterations_below_diag(engine):
    """The 8^3 cavity at Re = 100 with the velocity V-cycle: the mean GMRES iterations per Newton step after the
    first are less than half as many with "lower" as with "diag"."""
    from firedrake_b200.assemble import solve_nonlinear
    from firedrake_b200.mg import MeshHierarchy
    its = {}
    for fact in ("diag", "lower"):
        _, V, Q, F, bcs = tn._cavity(8, 0.01)
        sp = {**tn._fieldsplit("mg", 1e-6), "snes_rtol": 1e-8, "ksp_max_it": 3000,
              "pc_fieldsplit_schur_fact_type": fact}
        hist, kits = solve_nonlinear(F, F.dat(), F.dat(), bcs, sp, hierarchy=MeshHierarchy(2, 2, 2, 2),
                                     nullspace="constant")
        assert hist[-1] <= 1e-8 * hist[0], (fact, hist, kits)
        its[fact] = (np.mean(kits[1:]), kits)
    # measured on an H100: 110.5 ("lower") against 691.5 ("diag") iterations per step
    assert its["lower"][0] < 0.5 * its["diag"][0], its
