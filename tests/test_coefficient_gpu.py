"""GPU parity of the coefficient form alpha*inner(kappa*grad u, grad v)*dx + beta*inner(u, v)*dx
(FDB_FORM_HELMHOLTZ_COEF, the slab-thread kernel's COEF mode): action, element matrix, diagonal,
matrix-free operator and solvers, against the NumPy oracle (tests/_coef_oracle.py), the generic
wrapper path and the constant-coefficient kernels.  Tolerance 1e-12 relative in the max norm.

Every test takes the engine as its first argument, so tests/test_coefficient_host_mock.py runs the
same host logic on the CPU against a mock engine."""
import numpy as np
import pytest

import _coef_oracle as co
from firedrake_b200 import op2
from firedrake_b200.fiat_lite import interval_element
from firedrake_b200.utility_meshes import ExtrudedHexMesh

pytestmark = pytest.mark.gpu

TOL = 1e-12
KAPPA = "2.0 + sin(3.0 * x[0]) * x[1]"


def relerr(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def kappa_values(V, seed=0):
    """Positive, varying in every direction, not smooth (per-node noise)."""
    X = V.dof_coordinates()
    return 2.0 + np.sin(3.0 * X[:, 0]) * X[:, 1] + 0.5 * X[:, 2] + 0.2 * np.random.default_rng(seed).random(len(X))


def setup(p, native, mesh=None):
    """op2 objects of a warped, permuted mesh: extruded (column map + offsets) or native hexes (one map row
    per cell, cells in a random order), and the oracle's view of the same maps."""
    mesh = mesh or ExtrudedHexMesh(4, 3, 6, warp=0.05, permute_seed=1)
    V = mesh.function_space(p)
    nodes = op2.Set(V.node_count)
    vnodes = op2.Set(mesh.coord_space.node_count)
    if native:
        perm = np.random.default_rng(0).permutation(mesh.num_cells)
        full, cfull = V.full_cell_node_list()[perm], mesh.coord_space.full_cell_node_list()[perm]
        cells = op2.Set(len(perm))
        m0 = op2.Map(cells, nodes, V.arity, full)
        m1 = op2.Map(cells, vnodes, 8, cfull)
        omaps = (np.ascontiguousarray(full), np.zeros(V.arity, dtype=np.int32), np.ascontiguousarray(cfull),
                 np.zeros(8, dtype=np.int32), 1)
    else:
        cells = op2.ExtrudedSet(op2.Set(mesh.num_base_cells), mesh.layers)
        m0 = op2.Map(cells, nodes, V.arity, V.cell_node_map, offset=V.offset)
        m1 = op2.Map(cells, vnodes, 8, mesh.coord_map, offset=mesh.coord_offset)
        omaps = (V.cell_node_map, V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz)
    X = op2.Dat(op2.DataSet(vnodes, 3), mesh.coordinates)
    return mesh, V, cells, nodes, m0, m1, X, omaps


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("native", [False, True], ids=["extruded", "native"])
@pytest.mark.parametrize("beta", [0.0, 0.6])
def test_coef_action_matches_oracle(engine, p, native, beta):
    """Atomic and coloured scatter; coloured is bit-identical across calls.  Degree 5 on 6 layers takes
    the slim staging with atomics and the full one with colours (3 layers per launch)."""
    mesh, V, cells, nodes, m0, m1, X, omaps = setup(p, native)
    rng = np.random.default_rng(p)
    u = op2.Dat(nodes, rng.standard_normal(V.node_count))
    kap = op2.Dat(nodes, kappa_values(V, p))
    alpha = 1.3
    yo = co.action(interval_element(p), mesh.coordinates, u.data_ro.copy(), kap.data_ro.copy(), *omaps,
                   alpha=alpha, beta=beta)
    k = op2.Kernel("helmholtz_coef", degree=p, alpha=alpha, beta=beta)
    y = op2.Dat(nodes)
    op2.par_loop(k, cells, y(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), kap(op2.READ, m0))
    assert relerr(y.data_ro, yo) < TOL
    outs = []
    for _ in range(2):
        y.zero()
        op2.par_loop(k, cells, y(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), kap(op2.READ, m0),
                     scatter="coloured")
        outs.append(y.data_ro.copy())
    assert np.array_equal(outs[0], outs[1])
    assert relerr(outs[0], yo) < TOL


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5])
def test_coef_action_matches_generic_path_and_constant_form(engine, p):
    """The hand-written kernel against ``assemble_variable_coefficient`` (the generic wrapper path), and
    kappa == 1 against the constant-coefficient ``Form``."""
    from firedrake_b200.assemble import (Form, FunctionSpace, OneFormAssembler, assemble_variable_coefficient,
                                         interpolate)
    mesh = ExtrudedHexMesh(4, 3, 5, warp=0.05, permute_seed=2)
    V = FunctionSpace(mesh, p)
    u = V.dat(np.random.default_rng(1).standard_normal(V.node_count))
    kap = interpolate(V, KAPPA)
    yg = assemble_variable_coefficient(V, kap, u, beta=0.5)
    yc = OneFormAssembler(Form(V, 1.0, 0.5, kap), u).assemble()
    assert relerr(yc.data_ro, yg.data_ro) < TOL
    one = interpolate(V, "1.0")
    y1 = OneFormAssembler(Form(V, 0.8, 0.5, one), u).assemble()
    yf = OneFormAssembler(Form(V, 0.8, 0.5), u).assemble()
    assert relerr(y1.data_ro, yf.data_ro) < TOL


def _bcs(V):
    from firedrake_b200.assemble import DirichletBC
    return [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, 0.0, "top")]


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_coef_matrix_matches_oracle(engine, p):
    """Entrywise against the oracle's element matrices added through the BC-masked lgmaps, unit
    diagonal on the constrained rows; Mat.mult equals the matrix-free operator's mult."""
    from firedrake_b200.assemble import Form, FunctionSpace, assemble
    mesh = ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=2) if p < 4 else \
        ExtrudedHexMesh(2, 2, 3, warp=0.05, permute_seed=2)
    V = FunctionSpace(mesh, p)
    kap = V.dat(kappa_values(V.V, 3))
    bcs = _bcs(V)
    form = Form(V, 1.1, 0.7, kap)
    A = assemble(form, bcs=bcs)
    ro, ci, vals = A.csr()
    lg = np.arange(V.node_count, dtype=np.int32)
    bn = np.unique(np.concatenate([bc.nodes for bc in bcs]))
    lg[bn] = -1
    i0, Ae = co.element_matrices(interval_element(p), mesh.coordinates, kap.data_ro.copy(), V.V.cell_node_map,
                                 V.V.offset, mesh.coord_map, mesh.coord_offset, mesh.nz, alpha=1.1, beta=0.7)
    vo = co.add_to_csr(ro, ci, np.zeros(len(ci)), i0, Ae, lg, lg)
    diag = ro[bn] + np.array([np.searchsorted(ci[ro[r]:ro[r + 1]], r) for r in bn], dtype=np.int64)
    vo[diag] = 1.0
    assert np.abs(vals - vo).max() < TOL * np.abs(vo).max()
    x = V.dat(np.random.default_rng(4).standard_normal(V.node_count))
    y, ymf = V.dat(), V.dat()
    A.mult(x, y)
    assemble(form, bcs=bcs, mat_type="matfree").mult(x, ymf)
    assert relerr(y.data_ro, ymf.data_ro) < TOL


@pytest.mark.parametrize("p", [1, 2, 3])
def test_coef_diagonal_equals_assembled_diagonal(engine, p):
    from firedrake_b200.assemble import Form, FunctionSpace, ImplicitMatrixContext, assemble
    mesh = ExtrudedHexMesh(3, 2, 4, warp=0.05, permute_seed=3)
    V = FunctionSpace(mesh, p)
    kap = V.dat(kappa_values(V.V, 5))
    form = Form(V, 1.0, 0.3, kap)
    bcs = _bcs(V)
    d = ImplicitMatrixContext(form, bcs).getDiagonal(V.dat()).data_ro.copy()
    ro, ci, vals = assemble(form, bcs=bcs).csr()
    dA = np.array([vals[ro[r] + np.searchsorted(ci[ro[r]:ro[r + 1]], r)] for r in range(V.node_count)])
    assert relerr(d, dA) < TOL


def test_coef_host_pointer_mode_equals_device_mode(engine):
    """Host-resident Dats through the mirror cache (monolithic path, kappa acquired like the other
    READ arguments); a host write to kappa bumps its version and is picked up by the next call."""
    p = 3
    mesh, V, cells, nodes, m0, m1, X, _ = setup(p, False, ExtrudedHexMesh(4, 4, 6, warp=0.05))
    rng = np.random.default_rng(9)
    u = op2.Dat(nodes, rng.standard_normal(V.node_count))
    kap = op2.Dat(nodes, kappa_values(V, 9))
    k = op2.Kernel("helmholtz_coef", degree=p, alpha=1.0, beta=0.0)
    yd = op2.Dat(nodes)
    op2.par_loop(k, cells, yd(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), kap(op2.READ, m0))
    ref = yd.data_ro.copy()
    yh = op2.Dat(nodes)
    gk = op2.GlobalKernel(k, [m0, m1], extruded=True)
    loop = op2.Parloop(gk, cells, [yh(op2.INC, m0), X(op2.READ, m1), u(op2.READ, m0), kap(op2.READ, m0)],
                       location="host")
    loop()
    assert relerr(yh.data_ro, ref) < TOL
    kap.data[:] *= 2.0
    yh.zero()
    loop()
    assert relerr(yh.data_ro, 2.0 * ref) < TOL


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
def test_coef_solve(engine, pc):
    """kappa = 2 + sin(3x) y does not depend on z: with u = 0 at the bottom and 42 at the top, u = 42 z
    is exact (the side fluxes vanish), for every preconditioner; mg coarsens kappa by injection."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import DirichletBC, Form, FunctionSpace, interpolate, solve
    h = mg.MeshHierarchy(2, 2, 2, 2)
    V = FunctionSpace(h[2], 2)
    kap = interpolate(V, KAPPA)
    bcs = [DirichletBC(V, 0.0, "bottom"), DirichletBC(V, 42.0, "top")]
    u = V.dat()
    its, hist = solve(Form(V, 1.0, 0.0, kap), V.dat(), u, bcs=bcs, hierarchy=h,
                      solver_parameters={"pc_type": pc, "ksp_rtol": 1e-12})
    z = V.V.dof_coordinates()[:, 2]
    assert np.abs(u.data_ro - 42.0 * z).max() < 1e-7, (pc, its, hist[-1])
    # bounds from the mock-engine run of this test (164 / 86 / 9 iterations) with some margin
    assert its < {"none": 200, "jacobi": 120, "mg": 15}[pc], (pc, its)


def test_coef_kernel_refuses_what_it_does_not_cover(engine):
    """Vector spaces, the affine variant, degrees outside the instantiated ranges: a clear error from
    fdb_kernel_create, never a silent fall-back."""
    from firedrake_b200 import _lib
    mesh, V, cells, nodes, m0, m1, X, _ = setup(2, False, ExtrudedHexMesh(2, 2, 2))
    for kw, msg in ((dict(degree=2, cdim=3), "scalar"), (dict(degree=2, affine=True), "affine"),
                    (dict(degree=5, rank=2), "degree 5"), (dict(degree=4, diagonal=True), "degree 4")):
        gk = op2.GlobalKernel(op2.Kernel("helmholtz_coef", **kw), [m0, m1], extruded=True)
        with pytest.raises(_lib.EngineError, match=msg):
            gk.compile()
