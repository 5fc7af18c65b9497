"""CPU checks of the SIPG oracle (tests/_dg_oracle.py), the DQ space and the interior-facet sets the assembler builds:
symmetry, the constant null space of the pure Neumann operator, Galerkin consistency on an affine mesh, positive
definiteness at the penalty the GPU tests use, the DQ numbering and node positions, facet counts and the pairing of
the two sides' face points."""
import numpy as np
import pytest

import _boundary_oracle as bo
import _dg_oracle as do
from firedrake_b200.utility_meshes import ExtrudedHexMesh


def eta_of(p):
    return 3.0 * (p + 1) ** 2


def warped(n=3, seed=0):
    return bo.perturb(ExtrudedHexMesh(n, n, n, Lx=1.1, Ly=0.9, Lz=1.0, warp=0.04, permute_seed=seed), 0.06, seed)


def sheared(nx=2, ny=3, nz=2):
    """An affine image of a box (every cell a parallelepiped)."""
    mesh = ExtrudedHexMesh(nx, ny, nz, Lx=1.0, Ly=1.2, Lz=0.8, permute_seed=3)
    S = np.array([[1.0, 0.3, 0.1], [0.0, 1.1, -0.2], [0.15, 0.0, 0.9]])
    mesh.coordinates[:] = mesh.coordinates @ S.T + np.array([0.2, -0.1, 0.3])
    return mesh


@pytest.mark.parametrize("p", [1, 2, 3])
def test_symmetric(p):
    mesh = warped(2, seed=p)
    W = mesh.dg_function_space(p)
    A = do.operator(mesh, W, do.element(p), 1.3, 0.4, eta_of(p))
    assert abs(A - A.T).max() < 1e-12 * abs(A).max()


@pytest.mark.parametrize("p", [1, 2, 3])
def test_constants_in_the_kernel_without_weak_conditions(p):
    mesh = warped(2, seed=5 + p)
    W = mesh.dg_function_space(p)
    A = do.operator(mesh, W, do.element(p), 0.7, 0.0, eta_of(p), weak_bcs=())
    assert np.abs(A @ np.ones(W.node_count)).max() < 1e-12 * abs(A).max()


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_galerkin_consistency_on_an_affine_mesh(p):
    """u a total-degree-p polynomial, f = -alpha lap u + beta u: A u = M f + nitsche_load(u) to roundoff."""
    mesh = sheared()
    W = mesh.dg_function_space(p)
    el = do.element(p)
    alpha, beta, eta = 1.4, 0.6, eta_of(p)
    x, y, z = W.dof_coordinates().T
    c = np.random.default_rng(p).standard_normal(6)
    if p == 1:
        u = c[0] + c[1] * x + c[2] * y + c[3] * z
        lap = 0.0 * x
    else:
        u = c[0] + c[1] * x * y + c[2] * z ** 2 + c[3] * y ** p + c[4] * x ** (p - 1) * z + c[5] * x ** p
        lap = 2 * c[2] + c[3] * p * (p - 1) * y ** (p - 2) + (c[4] * (p - 1) * (p - 2) * x ** max(p - 3, 0) * z
                                                           if p > 2 else 0.0) + c[5] * p * (p - 1) * x ** (p - 2)
    f = -alpha * lap + beta * u
    A = do.operator(mesh, W, el, alpha, beta, eta)
    M = do.cell_matrix(mesh, W, el, 0.0, 1.0)
    r = A @ u - M @ f - do.nitsche_load(mesh, W, el, alpha, eta, "on_boundary", u)
    assert np.abs(r).max() < 1e-11 * max(1.0, np.abs(A @ u).max()), np.abs(r).max()


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_positive_definite_at_the_test_penalty(p):
    """eta = 3 (p+1)^2 gives an SPD operator on a warped 3^3 mesh, with and without the Nitsche terms."""
    mesh = warped(3, seed=11)
    W = mesh.dg_function_space(p)
    for weak, beta in (("on_boundary", 0.0), ((), 0.3)):
        A = do.operator(mesh, W, do.element(p), 1.0, beta, eta_of(p), weak_bcs=weak).toarray()
        assert np.linalg.eigvalsh(0.5 * (A + A.T))[0] > 0.0, (p, weak)


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_dq_numbering_and_nodes(p):
    mesh = ExtrudedHexMesh(3, 2, 4, permute_seed=2)
    W = mesh.dg_function_space(p)
    n = p + 1
    full = W.full_cell_node_list()
    assert np.array_equal(np.sort(full.ravel()), np.arange(W.node_count))
    assert np.all(W.offset == n ** 3)
    assert np.array_equal(W.cell_node_map[:, 1:] - W.cell_node_map[:, :-1], np.ones((mesh.num_base_cells, n ** 3 - 1)))
    assert np.array_equal(np.sort(W.cell_node_map[:, 0]), np.arange(mesh.num_base_cells) * mesh.nz * n ** 3)
    # the dofs sit at the Gauss-Legendre points of each cell (ascending, local (ax*n + ay)*n + az)
    X = W.dof_coordinates()
    rows, Xc = do.cells(mesh, W)
    el = do.element(p)
    pts = np.stack(np.meshgrid(el.nodes, el.nodes, el.nodes, indexing="ij"), axis=-1).reshape(-1, 3)
    b = np.array([[(v >> 2) & 1, (v >> 1) & 1, v & 1] for v in range(8)])
    wts = np.prod(np.where(b[None] > 0, pts[:, None, :], 1 - pts[:, None, :]), axis=-1)   # (N^3, 8)
    assert np.allclose(X[rows], np.einsum("qv,cvi->cqi", wts, Xc), atol=1e-14)
    assert np.all(np.diff(el.nodes) > 0)
    with pytest.raises(ValueError, match="no boundary nodes"):
        W.boundary_nodes(1)
    with pytest.raises(ValueError, match="outside 1..4"):
        mesh.dg_function_space(5)


@pytest.mark.parametrize("shape", [(3, 2, 4), (1, 3, 1), (4, 4, 2)])
def test_facet_counts(shape):
    nx, ny, nz = shape
    mesh = ExtrudedHexMesh(nx, ny, nz, permute_seed=1)
    P, M, FP, FM = do.interior_facets(mesh)
    assert len(P) == ((nx - 1) * ny + nx * (ny - 1)) * nz + nx * ny * (nz - 1)
    from firedrake_b200.assemble import FunctionSpace, _dg_interior_groups
    V = FunctionSpace(mesh, 1, family="DQ")
    groups = _dg_interior_groups(V)
    sizes = [(g[0].total_size, g[0].layers - 1) for g in groups]
    want = []
    if (nx - 1) * ny + nx * (ny - 1):
        want.append(((nx - 1) * ny + nx * (ny - 1), nz))
    if nz > 1:
        want.append((nx * ny, nz - 1))
    assert sizes == want
    assert _dg_interior_groups(V) is groups                           # cached on the space


@pytest.mark.parametrize("p", [1, 3])
def test_assembler_facet_sets_pair_the_same_points(p):
    """Every facet of the assembler's interior sets, in every layer: face point (a, b) of '+' is face point (a, b)
    of '-' (physically), the rows are the two cells' rows and the pairs are (1, 0), (3, 2) or (5, 4)."""
    from firedrake_b200.assemble import FunctionSpace, _dg_interior_groups
    mesh = warped(3, seed=4)
    V = FunctionSpace(mesh, p, family="DQ")
    el = do.element(p)
    nd = (p + 1) ** 3
    seen = 0
    for fset, fmap, cmap, pairs in _dg_interior_groups(V):
        pr = pairs.data_ro.reshape(-1, 2)
        assert {tuple(r) for r in pr} <= {(1, 0), (3, 2), (5, 4)}
        assert fmap.arity == 2 * nd and cmap.arity == 16
        for layer in range(fset.layers - 1):
            rows = fmap.values.astype(np.int64) + layer * np.asarray(fmap.offset, dtype=np.int64)
            xrows = cmap.values.astype(np.int64) + layer * np.asarray(cmap.offset, dtype=np.int64)
            Xp, Xm = mesh.coordinates[xrows[:, :8]], mesh.coordinates[xrows[:, 8:]]
            for fv in {tuple(r) for r in pr}:
                sel = (pr[:, 0] == fv[0]) & (pr[:, 1] == fv[1])
                qp, qm = do.face_points(el, fv[0]), do.face_points(el, fv[1])
                b = np.array([[(v >> 2) & 1, (v >> 1) & 1, v & 1] for v in range(8)])
                wp = np.prod(np.where(b[None] > 0, qp[:, None, :], 1 - qp[:, None, :]), axis=-1)
                wm = np.prod(np.where(b[None] > 0, qm[:, None, :], 1 - qm[:, None, :]), axis=-1)
                assert np.allclose(np.einsum("qv,cvi->cqi", wp, Xp[sel]), np.einsum("qv,cvi->cqi", wm, Xm[sel]),
                                   atol=1e-14)
            # the '-' row is the '-' cell's full DQ row: contiguous dofs
            assert np.all(np.diff(rows[:, nd:], axis=1) == 1) and np.all(np.diff(rows[:, :nd], axis=1) == 1)
            seen += len(pr)
    P, _, _, _ = do.interior_facets(mesh)
    assert seen == len(P)


def test_orientation_check_refuses_a_mismatched_face():
    from firedrake_b200.assemble import _check_facet_orientation
    xrows = np.tile(np.arange(16), (1, 1))
    with pytest.raises(ValueError, match="parametrise the face differently"):
        _check_facet_orientation(xrows, np.ones(16), np.array([[1, 0]]))


def test_space_and_form_refusals():
    from firedrake_b200 import assemble as A
    mesh = ExtrudedHexMesh(2, 2, 2)
    V = A.FunctionSpace(mesh, 2, family="DQ")
    assert V.element.variant == "gl" and A.FunctionSpace(mesh, 2).element is None
    with pytest.raises(NotImplementedError, match="vector DQ"):
        A.FunctionSpace(mesh, 2, 3, family="DQ")
    with pytest.raises(ValueError, match="family"):
        A.FunctionSpace(mesh, 2, family="RT")
    with pytest.raises(ValueError, match="needs the penalty eta"):
        A.InteriorPenalty(V, 1.0, 0.0)
    with pytest.raises(ValueError, match="takes a DQ space"):
        A.InteriorPenalty(A.FunctionSpace(mesh, 2), 1.0, 0.0, 27.0)
    with pytest.raises(NotImplementedError, match="DirichletBC does not take DQ spaces.*weak_bcs"):
        A.DirichletBC(V, 0.0, 1)
    b = V.dat()
    for make, name in ((lambda: A.Elasticity(V, 1.0, 1.0), "Elasticity"),
                       (lambda: A.HyperElasticity(V, 1.0, 1.0), "HyperElasticity"),
                       (lambda: A.NonlinearDiffusion(V), "NonlinearDiffusion"),
                       (lambda: A.AdvectionDiffusion(V, b), "AdvectionDiffusion"),
                       (lambda: A.Stokes(V, V, 1.0), "Stokes"),
                       (lambda: A.NavierStokes(V, V, 1.0), "NavierStokes"),
                       (lambda: A.BoundaryMass(V, 1.0), "BoundaryMass"),
                       (lambda: A.Form(V, 1.0, 0.0, ds=((1.0, 1),)), "Form's ds terms"),
                       (lambda: A.interpolate(V, "x[0]"), "interpolate"),
                       (lambda: A.interpolate_q1(V, b), "interpolate_q1"),
                       (lambda: A.assemble_functional(V, b), "assemble_functional")):
        with pytest.raises(NotImplementedError, match=f"{name} does not take DQ spaces"):
            make()
    with pytest.raises(NotImplementedError, match="no assembled matrix"):
        A.Form(V, 1.0, 0.0).kernel(2)
    F = A.InteriorPenalty(V, 1.0, 0.0, 27.0)
    for mt in ("aij", "is"):
        with pytest.raises(NotImplementedError, match="no assembled matrix on a DQ space"):
            A.assemble(F, mat_type=mt)
    with pytest.raises(NotImplementedError, match="'none' or 'jacobi'"):
        A.solve(F, V.dat(), V.dat(), solver_parameters={"pc_type": "mg"})
    with pytest.raises(ValueError, match="no weakly imposed"):
        A.nitsche_load(A.InteriorPenalty(V, 1.0, 0.0, 27.0, weak_bcs=()), V.dat())
    with pytest.raises(ValueError, match="takes a DQ space"):
        A.dg_flux_load(A.FunctionSpace(mesh, 2), V.dat())
