"""The fast-diagonalisation vertex-star relaxation on the CPU (DESIGN.md section 4.20).

* On unwarped meshes with constant coefficients the separable star operator A_v equals the star block of the
  assembled operator, for p = 1..5, anisotropic and permuted meshes, Dirichlet conditions on several face sets,
  beta = 0 and beta > 0; the star dof sets are those of patch.vertex_star_patches.
* The tables diagonalise the 1-D pencils: S^T M S = I and S^T K S = diag(lam).
* The relaxation is SPD, and its two-level error propagation under P1PC contracts (pinned radii)."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as sla

import _eigen_oracle as eo
import _fdm_oracle as fo
from firedrake_b200 import mg
from firedrake_b200.assemble import FunctionSpace
from firedrake_b200.patch import StarTables, star_matrices, vertex_star_patches
from firedrake_b200.utility_meshes import ExtrudedHexMesh

FACE_SETS = [(), (1,), (1, 2, 3, 4, "bottom", "top"), (2, 3, "top")]


def _setup(p, domains, permute_seed=None, warp=0.0, dims=(5, 4, 6), L=(1.0, 0.7, 1.3)):
    mesh = ExtrudedHexMesh(*dims, Lx=L[0], Ly=L[1], Lz=L[2], warp=warp, permute_seed=permute_seed)
    V = FunctionSpace(mesh, p)
    t = StarTables(V, domains)
    nodes, ijk = fo.star_nodes(V, t)
    return mesh, V, t, nodes, ijk


def _bc_nodes(V, domains):
    return np.unique(np.concatenate([V.boundary_nodes(s) for s in domains])) if domains else np.zeros(0, int)


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("domains", FACE_SETS)
def test_separable_star_operator_is_the_assembled_block(p, domains):
    mesh, V, t, nodes, (I, J, K) = _setup(p, domains, permute_seed=3)
    excl = _bc_nodes(V, domains)
    ptr, dofs = vertex_star_patches(V, exclude=excl)
    patches = [set(dofs[ptr[k]:ptr[k + 1]].tolist()) for k in range(len(ptr) - 1)]
    act = fo._outer(*fo._dirs(t, "act")) != 0
    # vertex_star_patches lists the non-empty stars in lattice order (I, J, K)
    lex = np.lexsort((K, J, I))
    nonempty = [s for s in lex if act[s].any()]
    assert len(nonempty) == len(patches)
    assert all(set(nodes[s][act[s]].tolist()) == patches[k] for k, s in enumerate(nonempty))
    for alpha, beta in ((1.0, 0.0), (0.7, 2.5)):
        A = eo.helmholtz(mesh, V.V, p, alpha, beta).tocsr()
        for s in nonempty[::max(1, len(nonempty) // 40)]:
            d = nodes[s][act[s]]
            blk = A[d][:, d].toarray()
            sep = fo.separable_operator(t, s, alpha, beta)
            assert np.abs(sep - blk).max() <= 1e-13 * np.abs(blk).max(), (s, np.abs(sep - blk).max())


def test_pool_is_small_on_unwarped_meshes():
    _, _, t, _, _ = _setup(3, (1, 2, 3, 4, "bottom", "top"), dims=(8, 8, 8), L=(1.0, 1.0, 1.0))
    # per direction: interior, the two boundary ends with and without the Dirichlet node removed
    assert len(t.pool) <= 5
    _, _, tw, _, _ = _setup(3, (), dims=(8, 8, 8), warp=0.05)
    assert len(tw.pool) > 100


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
def test_tables_diagonalise_the_pencils(p):
    _, _, t, _, _ = _setup(p, ("bottom", 2), warp=0.04)
    K, M, act, _ = star_matrices(p, t.flags, t.hl, t.hr)
    for e in range(len(t.pool)):
        a = np.nonzero(act[e])[0]
        if not len(a):                              # p = 1 at a Dirichlet vertex: an empty patch
            assert not t.S[e].any() and np.all(t.lam[e] == 1.0)
            continue
        S = t.S[e][np.ix_(a, np.arange(len(a)))]
        assert np.abs(S.T @ M[e][np.ix_(a, a)] @ S - np.eye(len(a))).max() < 1e-12
        L = S.T @ K[e][np.ix_(a, a)] @ S
        assert np.abs(L - np.diag(t.lam[e][:len(a)])).max() < 1e-12 * max(1.0, t.lam[e].max())
        # padded and removed nodes: zero rows and columns, eigenvalue 1
        assert not t.S[e][act[e] == 0].any() and not t.S[e][:, len(a):].any()
        assert np.all(t.lam[e][len(a):] == 1.0)


@pytest.mark.parametrize("p,warp,kappa", [(2, 0.0, False), (3, 0.05, True)])
def test_relaxation_is_spd(p, warp, kappa):
    mesh, V, t, nodes, _ = _setup(p, (1, "top"), warp=warp, dims=(3, 4, 3))
    n = V.node_count
    k = 1.0 + np.random.default_rng(0).random(n) if kappa else None
    P = np.stack([fo.apply(t, nodes, e, 1.0, 0.3, k) for e in np.eye(n)], axis=1)
    free = np.setdiff1d(np.arange(n), _bc_nodes(V, (1, "top")))
    Pf = P[np.ix_(free, free)]
    assert np.abs(Pf - Pf.T).max() < 1e-12 * np.abs(Pf).max()
    assert np.linalg.eigvalsh(Pf).min() > 0.0
    assert not P[_bc_nodes(V, (1, "top"))].any()


def _stiffness(V, p):
    return eo.helmholtz(V.mesh, V, p, 1.0, 0.0).tocsr()


def two_level_radius_star(p, n, nu=2):
    """The spectral radius of E = S (I - P Ac^-1 P^T A) S of two-level P1PC (CG_p over a rediscretised CG1,
    Dirichlet bottom and top, n^3 unit cubes) with S = nu Chebyshev iterations preconditioned by the star
    relaxation, bounds (0.1, 1.1) x lmax(P_star^-1 A): the setting of tests/test_pmg_oracle.py with the Jacobi
    smoother replaced."""
    import _pmg_oracle as po
    mesh = ExtrudedHexMesh(n, n, n)
    Wf = FunctionSpace(mesh, p)
    Vf, Vc = mesh.function_space(p), mesh.function_space(1)
    t = StarTables(Wf, ("bottom", "top"))
    nodes, _ = fo.star_nodes(Wf, t)

    def free(V):
        return np.setdiff1d(np.arange(V.node_count), np.union1d(V.boundary_nodes("bottom"), V.boundary_nodes("top")))
    ff, fc = free(Vf), free(Vc)
    A = _stiffness(Vf, p)[ff][:, ff].tocsc()
    Ac = sla.splu(_stiffness(Vc, 1)[fc][:, fc].tocsc())
    P = sp.csr_matrix(po.global_prolongation(Vf, Vc)[np.ix_(ff, fc)])

    def prec(r):
        full = np.zeros(Vf.node_count)
        full[ff] = r
        return fo.apply(t, nodes, full)[ff]
    PA = sla.LinearOperator((len(ff),) * 2, matvec=lambda e: prec(A @ e), dtype=float)
    lmax = float(np.abs(sla.eigs(PA, k=1, which="LM", return_eigenvectors=False, tol=1e-8)[0]))
    coef = mg.chebyshev_coefficients(0.1 * lmax, 1.1 * lmax, nu)

    def smooth(e):
        d = np.zeros_like(e)
        for cd, cz in coef:
            d = cz * prec(-(A @ e)) + (cd * d if cd else 0.0)
            e = e + d
        return e

    def E(e):
        e = smooth(np.array(e, dtype=float).ravel())
        e = e - P @ Ac.solve(P.T @ (A @ e))
        return smooth(e)
    op = sla.LinearOperator((len(ff),) * 2, matvec=E, dtype=float)
    return float(np.abs(sla.eigs(op, k=1, which="LM", return_eigenvectors=False, tol=1e-6)[0]))


# two-level radii with the star smoother at 4^3 and 8^3 (tests/test_pmg_oracle.py: 0.282 / 0.283 at CG2 and
# 0.324 / 0.326 at CG3 with Chebyshev-Jacobi)
STAR_RADII = {2: (0.359, 0.382), 3: (0.293, 0.297)}


@pytest.mark.parametrize("p", [2, 3])
def test_two_level_spectral_radius_with_star_smoother(p):
    r4, r8 = two_level_radius_star(p, 4), two_level_radius_star(p, 8)
    print(f"CG{p} star: rho(4^3) = {r4:.3f}, rho(8^3) = {r8:.3f}")
    e4, e8 = STAR_RADII[p]
    assert abs(r4 - e4) < 5e-3 and abs(r8 - e8) < 5e-3
