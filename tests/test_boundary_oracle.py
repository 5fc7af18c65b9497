"""CPU checks of the boundary mass oracle (tests/_boundary_oracle.py) and of the facet sets the assembler builds
for ``ds(sub_domain)``: areas, first moments, an independent fine quadrature of non-planar bilinear faces,
symmetry, the tensor-product structure on flat faces, and the facet sets and shifted top maps of
firedrake_b200.assemble against the oracle's own facet lists."""
import numpy as np
import pytest

import _boundary_oracle as bo
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

L = (1.5, 0.8, 1.2)


def box(nx=3, ny=4, nz=2, warp=0.05, seed=None):
    return ExtrudedHexMesh(nx, ny, nz, Lx=L[0], Ly=L[1], Lz=L[2], warp=warp, permute_seed=seed)


def ones_integral(mesh, p, sub, u=None, nq=None):
    V = mesh.function_space(p)
    el = interval_element(p, nq)
    rows, vrows, f = bo.extruded_facets(mesh, V, sub)
    A = bo.matrix(el, mesh.coordinates, V.node_count, rows, vrows, f)
    one = np.ones(V.node_count)
    return one @ (A @ (one if u is None else u))


AREAS = {1: L[1] * L[2], 2: L[1] * L[2], 3: L[0] * L[2], 4: L[0] * L[2], "bottom": L[0] * L[1],
         "top": L[0] * L[1]}


@pytest.mark.parametrize("p", [1, 2, 3])
@pytest.mark.parametrize("sub", [1, 2, 3, 4, "bottom", "top"])
def test_area_of_each_side(p, sub):
    """1^T M 1 is the area of the side (the warp vanishes on the box boundary, so the faces are flat)."""
    assert abs(ones_integral(box(seed=1), p, sub) - AREAS[sub]) < 1e-13
    assert abs(ones_integral(box(seed=1), p, "on_boundary") - sum(AREAS.values())) < 1e-12


@pytest.mark.parametrize("p", [1, 2])
def test_first_moments_match_closed_forms(p):
    """int x_i ds over each side: the coordinate is exact in CG_p, the side is a rectangle."""
    mesh = box(seed=0)
    Xn = mesh.function_space(p).dof_coordinates()
    lo = {1: (0, 0.0), 2: (0, L[0]), 3: (1, 0.0), 4: (1, L[1]), "bottom": (2, 0.0), "top": (2, L[2])}
    for sub, (axis, val) in lo.items():
        for i in range(3):
            want = AREAS[sub] * (val if i == axis else L[i] / 2)
            assert abs(ones_integral(mesh, p, sub, Xn[:, i]) - want) < 1e-12, (sub, i)


def _fine_surface_integral(mesh, p, sub, u, nfine=16, h=1e-5):
    """int u_h ds by a 16^2-point Gauss rule on every face, the surface measure from central differences of the
    cell's full trilinear map, u_h from the cell's full Q_p basis: a second, independent statement."""
    V = mesh.function_space(p)
    el = interval_element(p)
    rows, vrows, facets = bo.extruded_facets(mesh, V, sub)
    X = mesh.coordinates
    x, w = np.polynomial.legendre.leggauss(nfine)
    x, w = (x + 1) / 2, w / 2
    n = p + 1
    total = 0.0

    def trilinear(Xc, xi):
        out = np.zeros(3)
        for v in range(8):
            b = ((v >> 2) & 1, (v >> 1) & 1, v & 1)
            out += Xc[v] * np.prod([xi[k] if b[k] else 1 - xi[k] for k in range(3)])
        return out

    for r, vr, f in zip(rows, vrows, facets):
        Xc = X[vr]
        d, side = f // 2, f % 2
        t1, t2 = [k for k in range(3) if k != d]
        for i, s in enumerate(x):
            for j, t in enumerate(x):
                xi = np.zeros(3)
                xi[d], xi[t1], xi[t2] = side, s, t
                ds_, dt_ = np.zeros(3), np.zeros(3)
                ds_[t1], dt_[t2] = h, h
                gs = (trilinear(Xc, xi + ds_) - trilinear(Xc, xi - ds_)) / (2 * h)
                gt = (trilinear(Xc, xi + dt_) - trilinear(Xc, xi - dt_)) / (2 * h)
                tabs = [el.tabulate([xi[k]])[0][0] for k in range(3)]
                phi = np.einsum("a,b,c->abc", *tabs).ravel()
                total += w[i] * w[j] * np.linalg.norm(np.cross(gs, gt)) * (phi @ u[r])
    return total


@pytest.mark.parametrize("p", [1, 2])
def test_non_planar_faces_match_fine_quadrature(p):
    """Vertices moved in and out of plane: the oracle with a 12-point rule agrees with the independent 16-point
    rule on finite-difference surface measures."""
    mesh = bo.perturb(box(2, 2, 2, warp=0.0), 0.1, seed=3)
    V = mesh.function_space(p)
    Xn = V.dof_coordinates()
    u = 1.0 + Xn[:, 0] * Xn[:, 1] - 0.5 * Xn[:, 2] ** 2
    for sub in (1, "top"):
        got = ones_integral(mesh, p, sub, u, nq=12)
        want = _fine_surface_integral(mesh, p, sub, u)
        assert abs(got - want) < 1e-9 * abs(want), (sub, got, want)


def test_symmetry_and_flat_tensor_product():
    mesh = bo.perturb(box(2, 3, 2), 0.08, seed=5)
    V = mesh.function_space(3)
    el = interval_element(3)
    rows, vrows, f = bo.extruded_facets(mesh, V, "on_boundary")
    A = bo.matrix(el, mesh.coordinates, V.node_count, rows, vrows, f, gamma=0.7)
    assert abs(A - A.T).max() < 1e-15 * abs(A).max()
    # a flat rectangular face of size hs x ht: hs ht (M1 (x) M1)
    Xf = np.array([[[0, 0, 0], [0, 0, 0.3], [0.5, 0, 0], [0.5, 0, 0.3]]], dtype=float)
    M = bo.facet_matrices(el, Xf, gamma=2.0)[0]
    B, w = np.asarray(el.B), np.asarray(el.wq)
    M1 = B.T @ np.diag(w) @ B
    assert np.abs(M - 2.0 * 0.5 * 0.3 * np.kron(M1, M1)).max() < 1e-15


@pytest.mark.parametrize("sub", [1, 3, "bottom", "top", (2, "top"), "on_boundary"])
def test_assembler_facet_sets_match_oracle(sub):
    """The facet groups of assemble.BoundaryMass (one vertical set over all layers, one horizontal set with one
    cell layer whose top rows are shifted by (nz - 1) * offset) cover exactly the oracle's facets."""
    from firedrake_b200.assemble import FunctionSpace, _boundary_groups
    mesh = box(3, 2, 3, seed=2)
    V = FunctionSpace(mesh, 2)
    got = set()
    for fset, fmap, cmap, facet in _boundary_groups(V, sub):
        nlay = fset.layers - 1
        for c in range(fset.total_size):
            for lay in range(nlay):
                got.add((tuple(fmap.values[c] + fmap.offset * lay), tuple(cmap.values[c] + cmap.offset * lay),
                         int(facet.data_ro[c])))
    rows, vrows, f = bo.extruded_facets(mesh, V.V, sub)
    want = {(tuple(r), tuple(v), int(k)) for r, v, k in zip(rows, vrows, f)}
    assert got == want and len(want) == len(f)
    assert _boundary_groups(V, sub) is _boundary_groups(V, sub)          # cached on the space


def test_sub_domain_names_are_checked():
    from firedrake_b200.assemble import BoundaryMass, FunctionSpace
    V = FunctionSpace(box(2, 2, 2), 1)
    with pytest.raises(ValueError, match="unknown sub_domain"):
        BoundaryMass(V, 1.0, 5)
    with pytest.raises(ValueError, match="unknown sub_domain"):
        BoundaryMass(V, 1.0, "left")


def test_forms_that_refuse_boundary_terms():
    """Taylor-Hood forms and partitioned spaces refuse ds with the reason; ds=() keeps every form as it was."""
    from firedrake_b200.assemble import Elasticity, Form, FunctionSpace, NavierStokes, Stokes
    mesh = box(2, 2, 2)
    V, Q = FunctionSpace(mesh, 2, 3), FunctionSpace(mesh, 1)
    for cls in (Stokes, NavierStokes):
        with pytest.raises(NotImplementedError, match="boundary terms on the .*Stokes form"):
            cls(V, Q, 1.0, 0.0, ds=((1.0, 2),))
    assert Form(Q, 1.0, 0.0).ds == () and Elasticity(V, 1.0, 1.0).ds == ()
    W = FunctionSpace(box(2, 2, 2), 1)
    W.cell_set.owner_computes = True               # as on an exec-halo partition
    with pytest.raises(NotImplementedError, match="partitioned space"):
        Form(W, 1.0, 0.0, ds=((1.0, "top"),))
    with pytest.raises(ValueError, match="pairs"):
        Form(Q, 1.0, 0.0, ds=(1.0,))
