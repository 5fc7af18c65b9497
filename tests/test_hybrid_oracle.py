"""The hybridisation of mixed Poisson on the CPU: the HDiv-trace numbering, and the dense oracle
(tests/_hybrid_oracle.py) against the dense mixed solve of tests/_mixed_poisson_oracle.py."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import _hybrid_oracle as ho
import _mixed_poisson_oracle as mo
from firedrake_b200 import _lib
from firedrake_b200.utility_meshes import ExtrudedHexMesh


def _spaces(k=2, n=(2, 3, 2), warp=0.06, permute_seed=2):
    mesh = ExtrudedHexMesh(*n, warp=warp, permute_seed=permute_seed)
    return mesh, mesh.hdiv_function_space(k), mesh.dg_function_space(k - 1), mesh.trace_function_space(k - 1)


def _load(mesh, S, Q, seed=0):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(S.node_count), rng.standard_normal(Q.node_count)


def _mixed(mesh, S, Q, alpha, L0, L1, flux_subs=(), nullspace=False):
    """The dense mixed solve with the flux-condition rows as identity rows (as MixedPoisson's solve)."""
    M, B = mo.global_matrices(mesh, S, Q, alpha)
    rows = np.unique(np.concatenate([S.boundary_nodes(s) for s in flux_subs])) if flux_subs else np.zeros(0, int)
    rhs = np.concatenate([L0, L1])
    rhs[rows] = 0.0
    pin = []
    if nullspace:
        rhs[S.node_count:] -= rhs[S.node_count:].mean()
        pin = [S.node_count]
        rhs[pin] = 0.0
    x = spla.spsolve(mo.constrained(mo.saddle(M, B), np.concatenate([rows, pin]).astype(int)).tocsc(), rhs)
    if nullspace:
        x[S.node_count:] -= x[S.node_count:].mean()
    return x[:S.node_count], x[S.node_count:]


@pytest.mark.parametrize("k", [2, 3])
def test_trace_numbering(k):
    """Counts, arity and offsets; every face's k^2 dofs are shared by at most two cells, and a trace dof sits on
    the same face as the NCF face dof of the same local position."""
    mesh, S, Q, T = _spaces(k, n=(3, 2, 3))
    nx, ny, nz = mesh.nx, mesh.ny, mesh.nz
    nfaces = (nx + 1) * ny * nz + nx * (ny + 1) * nz + nx * ny * (nz + 1)
    assert T.node_count == nfaces * k * k
    assert T.arity == 6 * k * k and np.all(T.offset == k * k)
    full = T.full_cell_node_list()
    counts = np.bincount(full.ravel(), minlength=T.node_count)
    assert counts.min() >= 1 and counts.max() == 2
    # interior faces: 2 cells; boundary faces: 1
    bnd = np.unique(np.concatenate([T.boundary_nodes(s) for s in ho.SUBS]))
    assert np.all(counts[bnd] == 1)
    assert np.sum(counts == 1) == len(bnd)
    # the NCF face dof of the same local position: same pairing across the mesh (a bijection)
    fs = S.full_cell_node_list()
    loc = np.array([ho.face_dof(k, t)[0] for t in range(6 * k * k)])
    pair = {}
    for c in range(full.shape[0]):
        for t in range(6 * k * k):
            assert pair.setdefault(full[c, t], fs[c, loc[t]]) == fs[c, loc[t]]
    assert len(set(pair.values())) == T.node_count
    for s in ho.SUBS:
        assert sorted(pair[t] for t in T.boundary_nodes(s)) == sorted(S.boundary_nodes(s))


@pytest.mark.parametrize("k", [2, 3])
def test_trace_matrix_symmetric_psd(k):
    mesh, S, Q, T = _spaces(k)
    H = ho.trace_matrix(mesh, S, Q, T, 1.3)
    assert np.abs(H - H.T).max() < 1e-13 * np.abs(H).max()
    ev = np.linalg.eigvalsh(H)
    assert ev.min() > -1e-12 * ev.max()


@pytest.mark.parametrize("k", [2, 3])
def test_kernel_of_h_is_the_constants(k):
    """Every cell's C^ K_K^-1 C^^T annihilates the constants (B^T 1 = C^T 1 cell by cell), so H 1 = 0 and, with
    flux conditions on the whole boundary (no rows replaced), the kernel is exactly the constants."""
    mesh, S, Q, T = _spaces(k)
    H = ho.trace_matrix(mesh, S, Q, T, 0.7)
    assert np.abs(H @ np.ones(T.node_count)).max() < 1e-12 * np.abs(H).max()
    ev = np.linalg.eigvalsh(H)
    assert ev[1] > 1e-8 * ev[-1]


@pytest.mark.parametrize("k", [2, 3])
def test_hybrid_solve_equals_mixed_with_natural_data(k):
    mesh, S, Q, T = _spaces(k)
    L0, L1 = _load(mesh, S, Q, k)
    s_h, u_h, _ = ho.hybrid_solve(mesh, S, Q, T, 1.3, L0, L1)
    s_m, u_m = _mixed(mesh, S, Q, 1.3, L0, L1)
    assert np.abs(s_h - s_m).max() < 1e-12 * np.abs(s_m).max()
    assert np.abs(u_h - u_m).max() < 1e-12 * np.abs(u_m).max()


@pytest.mark.parametrize("flux_subs, nullspace", [((1, "top"), False), (ho.SUBS, True)])
def test_hybrid_solve_equals_mixed_with_flux_conditions(flux_subs, nullspace):
    mesh, S, Q, T = _spaces(2)
    L0, L1 = _load(mesh, S, Q, 5)
    s_h, u_h, _ = ho.hybrid_solve(mesh, S, Q, T, 1.3, L0, L1, flux_subs, nullspace)
    s_m, u_m = _mixed(mesh, S, Q, 1.3, L0, L1, flux_subs, nullspace)
    assert np.abs(s_h - s_m).max() < 1e-11 * np.abs(s_m).max()
    assert np.abs(u_h - u_m).max() < 1e-11 * np.abs(u_m).max()
    for s in flux_subs:
        assert np.abs(s_h[S.boundary_nodes(s)]).max() < 1e-12 * np.abs(s_m).max()


def test_any_split_of_the_load_gives_the_same_solution():
    """A split w' != w of L[0] over the cells (w'_K summing to 1 on every dof) shifts lambda only."""
    mesh, S, Q, T = _spaces(2)
    L0, L1 = _load(mesh, S, Q, 9)
    s_ref, u_ref, lam_ref = ho.hybrid_solve(mesh, S, Q, T, 1.1, L0, L1)
    # the '-' cell takes 0.8 of an interior face load, the '+' cell 0.2: per-cell weights, summing to 1
    fs = S.full_cell_node_list()
    seen = np.zeros(S.node_count, dtype=bool)
    wcell = np.ones(fs.shape)
    counts = np.bincount(fs.ravel(), minlength=S.node_count)
    for c in range(fs.shape[0]):
        for j, g in enumerate(fs[c]):
            if counts[g] == 2:
                wcell[c, j] = 0.2 if seen[g] else 0.8
                seen[g] = True
    k = S.degree
    C = ho.trace_coupling(k)
    H = ho.trace_matrix(mesh, S, Q, T, 1.1)
    r = np.zeros(T.node_count)
    cells = ho.cell_data(mesh, S, Q, T)
    for c, (rs, rq, rt, Xv) in enumerate(cells):
        x = np.linalg.solve(ho.local_saddle(k, Xv, 1.1), np.concatenate([wcell[c] * L0[rs], L1[rq]]))
        r[rt] += C @ x[:len(rs)]
    nat = ho.natural_nodes(T, ())
    H[nat, :] = 0.0
    H[:, nat] = 0.0
    H[nat, nat] = 1.0
    r[nat] = 0.0
    lam = np.linalg.solve(H, r)
    u = np.zeros(Q.node_count)
    sig = np.zeros(S.node_count)
    for c, (rs, rq, rt, Xv) in enumerate(cells):
        g = np.concatenate([wcell[c] * L0[rs], L1[rq]])
        g[:len(rs)] -= C.T @ lam[rt]
        x = np.linalg.solve(ho.local_saddle(k, Xv, 1.1), g)
        sig[rs] += x[:len(rs)] / counts[rs]
        u[rq] = x[len(rs):]
    assert np.abs(sig - s_ref).max() < 1e-12 * np.abs(s_ref).max()
    assert np.abs(u - u_ref).max() < 1e-12 * np.abs(u_ref).max()
    assert np.abs(lam - lam_ref).max() > 1e-6 * np.abs(lam_ref).max()


def test_both_sides_agree_on_interior_faces():
    mesh, S, Q, T = _spaces(3)
    L0, L1 = _load(mesh, S, Q, 4)
    _, _, lam = ho.hybrid_solve(mesh, S, Q, T, 1.0, L0, L1)
    _, _, cells = ho.reconstruct(mesh, S, Q, T, 1.0, lam, L0, L1, per_cell=True)
    vals = {}
    for rs, sk in cells:
        for g, v in zip(rs, sk):
            vals.setdefault(g, []).append(v)
    scale = max(abs(v) for vs in vals.values() for v in vs)
    shared = [vs for vs in vals.values() if len(vs) == 2]
    assert shared and max(abs(a - b) for a, b in shared) < 1e-11 * scale


def test_abi_enum_matches_lib():
    import re
    import pathlib
    h = (pathlib.Path(__file__).resolve().parents[1] / "include" / "fdb200.h").read_text()
    for name, val in [("FDB_FORM_MIXED_POISSON_HYBRID", 26), ("FDB_FORM_MIXED_POISSON_RECONSTRUCT", 27)]:
        assert re.search(rf"\b{name}\s*=\s*{val}\b", h), name
    assert _lib.FORM_MIXED_POISSON_HYBRID == 26 and _lib.FORM_MIXED_POISSON_RECONSTRUCT == 27
