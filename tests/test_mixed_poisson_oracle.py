"""Mixed Poisson on NCF_k x DQ_{k-1} on the CPU: the NCF numbering of ExtrudedHDivFunctionSpace, the element
(orientation, Piola map, divergence), the convergence of the discretisation with scipy, the ABI, and the refusals of
the Python layer.  The kernels themselves are checked on the GPU (tests/test_mixed_poisson_gpu.py)."""
import itertools
import os
import re

import numpy as np
import pytest
import scipy.sparse.linalg as spla

import _mixed_poisson_oracle as mo
from firedrake_b200.fiat_lite import gauss_legendre
from firedrake_b200.utility_meshes import ExtrudedHexMesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MESHES = [dict(), dict(warp=0.06, permute_seed=4)]


@pytest.mark.parametrize("k", [2, 3, 4])
def test_counts_offsets_and_sharing(k):
    """Counts follow the face / interior census, the layer offsets are constant per local dof, and every face dof
    is shared by exactly the cells that touch its face (two inside, one on the boundary); interior dofs by one."""
    nx, ny, nz = 3, 2, 4
    mesh = ExtrudedHexMesh(nx, ny, nz, permute_seed=2)
    S = mesh.hdiv_function_space(k)
    k2 = k * k
    assert S.arity == 3 * k2 * (k + 1)
    assert S.node_count == ((nx + 1) * ny * nz + nx * (ny + 1) * nz + nx * ny * (nz + 1)) * k2 \
        + nx * ny * nz * 3 * (k - 1) * k2
    full = S.full_cell_node_list().astype(np.int64)
    assert np.array_equal(full.reshape(mesh.num_base_cells, nz, -1)[:, 1:] -
                          full.reshape(mesh.num_base_cells, nz, -1)[:, :-1],
                          np.broadcast_to(S.offset, (mesh.num_base_cells, nz - 1, S.arity)))
    assert len(np.unique(full)) == S.node_count and full.max() == S.node_count - 1
    count = np.bincount(full.ravel(), minlength=S.node_count)
    assert (count == 1).sum() == nx * ny * nz * 3 * (k - 1) * k2 + 2 * (ny * nz + nx * nz + nx * ny) * k2
    assert count.max() == 2
    for sub in (1, 2, 3, 4, "bottom", "top"):
        b = S.boundary_nodes(sub)
        assert np.all(count[b] == 1)
    nb = sum(len(S.boundary_nodes(s)) for s in (1, 2, 3, 4, "bottom", "top"))
    assert nb == 2 * (ny * nz + nx * nz + nx * ny) * k2


@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("opts", MESHES)
def test_interior_faces_agree_on_flux(k, opts):
    """On every interior face, the two cells reach the same dofs and, from their own Jacobians, the same physical
    normal flux sigma.n dS at every face point: one reference orientation, no sign flips (warped, permuted)."""
    mesh = ExtrudedHexMesh(3, 3, 2, **opts)
    S = mesh.hdiv_function_space(k)
    full = S.full_cell_node_list().astype(np.int64)
    fc = mesh.coord_space.full_cell_node_list()
    nz = mesh.nz
    cell = {}
    for c in range(mesh.num_base_cells):
        for l in range(nz):
            cell[(mesh.cell_ix[c], mesh.cell_iy[c], l)] = c * nz + l
    sigma = np.random.default_rng(k).standard_normal(S.node_count)
    x, _ = gauss_legendre(k + 1)
    fp = np.array(list(itertools.product(x, x)))
    for (i, j, l), a in cell.items():
        for d, step in enumerate([(1, 0, 0), (0, 1, 0), (0, 0, 1)]):
            b = cell.get((i + step[0], j + step[1], l + step[2]))
            if b is None:
                continue
            pa, pb = np.insert(fp, d, 1.0, axis=1), np.insert(fp, d, 0.0, axis=1)
            flux = []
            for c, pts in ((a, pa), (b, pb)):
                Xv = mesh.coordinates[fc[c]]
                J = mo.jacobians(Xv, pts)
                val, _, _ = mo.tabulate(k, pts)
                sh = np.einsum("j,jqa->qa", sigma[full[c]], val)
                sp = np.einsum("qab,qb->qa", J, sh) / np.linalg.det(J)[:, None]
                e0, e1 = [e for e in range(3) if e != d]
                area = np.cross(J[:, :, e0], J[:, :, e1])            # n dS / ds^ (orientation of +x_d)
                flux.append(np.sum(sp * area, axis=1))
                assert np.allclose(mo.trilinear(Xv, pts), mo.trilinear(mesh.coordinates[fc[a]], pa))
            assert np.allclose(flux[0], flux[1], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("opts", MESHES)
def test_jacobian_determinant_is_positive(opts):
    mesh = ExtrudedHexMesh(4, 4, 4, **opts)
    P, _ = mo.points(5)
    for Xv in mesh.coordinates[mesh.coord_space.full_cell_node_list()]:
        assert np.linalg.det(mo.jacobians(Xv, P)).min() > 0


@pytest.mark.parametrize("k", [2, 3, 4])
def test_divergence_maps_onto_q_k_minus_1(k):
    """div^ of every NCF_k basis function is a polynomial of Q_{k-1} (its least-squares fit in DQ_{k-1} at
    (k+2)^3 points is exact) and the reference B has full rank k^3 (onto)."""
    P, W = mo.points(k + 2)
    _, div, psi = mo.tabulate(k, P)
    coef, *_ = np.linalg.lstsq(psi.T, div.T, rcond=None)
    assert np.abs(psi.T @ coef - div.T).max() < 1e-11 * np.abs(div).max()
    assert np.linalg.matrix_rank(coef) == k ** 3


@pytest.mark.parametrize("k", [2, 3])
def test_cell_divergence_is_net_face_flux(k):
    """1^T B_K sigma = the net outward flux of sigma through the six faces of K (divergence theorem)."""
    mesh = ExtrudedHexMesh(1, 1, 1, warp=0.08)
    S = mesh.hdiv_function_space(k)
    Q = mesh.dg_function_space(k - 1)
    _, B = mo.global_matrices(mesh, S, Q)
    sigma = np.random.default_rng(3).standard_normal(S.node_count)
    ones = np.ones(Q.node_count)
    total = sum(mo.dirichlet_load(mesh, S, np.ones(len(mesh.coordinates)), s) @ sigma
                for s in (1, 2, 3, 4, "bottom", "top"))
    assert abs(ones @ (B @ sigma) - total) < 1e-12 * np.abs(sigma).sum()


@pytest.mark.parametrize("k", [2, 3])
def test_saddle_symmetric_and_constant_kernel(k):
    mesh = ExtrudedHexMesh(2, 2, 2, warp=0.05, permute_seed=1)
    S, Q = mesh.hdiv_function_space(k), mesh.dg_function_space(k - 1)
    M, B = mo.global_matrices(mesh, S, Q, 1.5)
    K = mo.saddle(M, B)
    assert abs(K - K.T).max() < 1e-14 * abs(K).max()
    rows = np.unique(np.concatenate([S.boundary_nodes(s) for s in (1, 2, 3, 4, "bottom", "top")]))
    Kc = mo.constrained(K, rows).toarray()
    w, v = np.linalg.eigh(Kc)
    small = np.abs(w) < 1e-10 * np.abs(w).max()
    assert small.sum() == 1
    null = v[:, np.argmin(np.abs(w))]
    assert np.abs(null[:S.node_count]).max() < 1e-10
    assert np.ptp(null[S.node_count:]) < 1e-10


@pytest.mark.parametrize("k", [2, 3])
def test_convergence_rates(k):
    """u = sin(pi x) sin(pi y) sin(pi z), sigma = grad u, -div sigma = f = 3 pi^2 u, u = 0 (natural): the L2 errors
    of u and sigma fall at rate >= k - 0.3 from 4^3 to 8^3."""
    pi = np.pi
    ue = lambda X: np.sin(pi * X[:, 0]) * np.sin(pi * X[:, 1]) * np.sin(pi * X[:, 2])
    ge = lambda X: pi * np.stack([np.cos(pi * X[:, 0]) * np.sin(pi * X[:, 1]) * np.sin(pi * X[:, 2]),
                                  np.sin(pi * X[:, 0]) * np.cos(pi * X[:, 1]) * np.sin(pi * X[:, 2]),
                                  np.sin(pi * X[:, 0]) * np.sin(pi * X[:, 1]) * np.cos(pi * X[:, 2])], axis=1)
    errs = []
    for n in (4, 8):
        mesh = ExtrudedHexMesh(n, n, n)
        S, Q = mesh.hdiv_function_space(k), mesh.dg_function_space(k - 1)
        M, B = mo.global_matrices(mesh, S, Q)
        f = 3 * pi ** 2 * ue(Q.dof_coordinates())
        rhs = np.concatenate([np.zeros(S.node_count), -(mo.dq_mass(mesh, Q) @ f)])
        x = spla.spsolve(mo.saddle(M, B).tocsc(), rhs)
        errs.append(mo.field_errors(mesh, S, Q, x[:S.node_count], x[S.node_count:], ue, ge))
    rates = np.log2(np.array(errs[0]) / np.array(errs[1]))
    assert np.all(rates >= k - 0.3), rates


def test_abi_enum_matches_lib():
    from firedrake_b200 import _lib
    h = open(os.path.join(ROOT, "include", "fdb200.h")).read()
    for name, val in (("MIXED_POISSON", 22), ("MIXED_POISSON_SCHUR", 23)):
        assert re.search(rf"FDB_FORM_{name} = {val}\b", h)
        assert getattr(_lib, f"FORM_{name}") == val


def test_unknown_family_still_refused():
    from firedrake_b200.assemble import FunctionSpace
    with pytest.raises(ValueError, match="family"):
        FunctionSpace(ExtrudedHexMesh(2, 2, 2), 2, family="RT")


def test_ncf_space_refusals():
    from firedrake_b200 import assemble as A
    mesh = ExtrudedHexMesh(2, 2, 2)
    with pytest.raises(ValueError, match="NCF degree 5"):
        mesh.hdiv_function_space(5)
    with pytest.raises(NotImplementedError, match="cdim 1"):
        A.FunctionSpace(mesh, 2, cdim=3, family="NCF")
    S = A.FunctionSpace(mesh, 2, family="NCF")
    Q = A.FunctionSpace(mesh, 1, family="DQ")
    V3 = A.FunctionSpace(mesh, 2, 3)
    for make in (lambda: A.Form(S), lambda: A.NonlinearDiffusion(S), lambda: A.Elasticity(S, 1.0, 1.0),
                 lambda: A.HyperElasticity(S, 1.0, 1.0), lambda: A.AdvectionDiffusion(S, None),
                 lambda: A.Stokes(S, Q), lambda: A.Stokes(V3, S), lambda: A.NavierStokes(S, Q),
                 lambda: A.SpectralForm(S), lambda: A.PointEvaluator(S, np.zeros((1, 3))),
                 lambda: A.interpolate(S, "x[0]"), lambda: A.interpolate_q1(S, S.coordinates),
                 lambda: A.InteriorPenalty(S), lambda: A.DGTransport(S, None), lambda: A.BoundaryMass(S),
                 lambda: A.dg_flux_load(S, None), lambda: A.assemble_functional(S, None)):
        with pytest.raises(NotImplementedError, match="NCF"):
            make()
    with pytest.raises(NotImplementedError, match="NCF"):
        A.DirichletBC(S, 1.0, 1)
    from firedrake_b200 import eigensolver, mg, patch
    with pytest.raises(NotImplementedError, match="NCF"):
        mg.PMG(S, lambda W: None)
    with pytest.raises(NotImplementedError, match="NCF"):
        mg.PTransfer(S, S)
    with pytest.raises(NotImplementedError, match="NCF"):
        eigensolver.LinearEigenproblem(A.MixedPoisson(S, Q))
    fdm = A.Form(A.FunctionSpace(mesh, 2))
    fdm.V = S                          # a Form that reached FDMStar with an NCF space
    with pytest.raises(NotImplementedError, match="NCF"):
        patch.FDMStar(fdm)
    with pytest.raises(ValueError, match="DQ_\\(k-1\\)"):
        A.MixedPoisson(S, A.FunctionSpace(mesh, 2, family="DQ"))
    A.MixedPoisson(S, Q)
    assert len(A.DirichletBC(S, 0.0, "top").nodes) == 4 * 4
