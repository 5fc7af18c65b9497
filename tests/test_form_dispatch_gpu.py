"""The hex-form argument path of fdb_kernel_call (csrc/global_kernel.cu): every form with an element matrix
assembles the same matrix from host pointers (through the mirror cache) as from device pointers, and a
host-mode matrix call without the byte sizes of its buffers is an error.  Tolerance 1e-12 relative in the
max norm."""
import numpy as np
import pytest

from firedrake_b200 import _lib, op2
from firedrake_b200.utility_meshes import ExtrudedHexMesh
from test_coefficient_gpu import kappa_values, relerr, setup
from test_hyperelastic_oracle import _smooth

pytestmark = pytest.mark.gpu

TOL = 1e-12
P = 2
HELM = dict(alpha=1.0, beta=0.5)
ELAS = dict(mu=1.3, lmbda=2.1, beta=0.3)

# form, value size, kernel parameters, trailing coefficient (None: the form has none)
CASES = {
    "helmholtz": ("helmholtz", 1, HELM, None),
    "helmholtz_vector": ("helmholtz", 3, HELM, None),
    "helmholtz_coef": ("helmholtz_coef", 1, HELM, "kappa"),
    "nonlinear_diffusion_jacobian": ("nonlinear_diffusion_jacobian", 1, dict(HELM, d=(1.0, 0.5, 0.5)), "u"),
    "elasticity": ("elasticity", 3, ELAS, None),
    "hyperelasticity_jacobian": ("hyperelasticity_jacobian", 3, ELAS, "u"),
}


def _problem(case):
    form, cdim, kw, coef = CASES[case]
    mesh, V, cells, nodes, m0, m1, X, _ = setup(P, False, ExtrudedHexMesh(3, 3, 4, warp=0.05, permute_seed=1))
    ins = [X]
    if coef == "kappa":
        ins.append(op2.Dat(nodes, kappa_values(V)))
    elif coef == "u" and cdim == 1:
        ins.append(op2.Dat(nodes, 0.5 + 0.3 * np.sin(3.0 * V.dof_coordinates()[:, 0])))
    elif coef == "u":
        ins.append(op2.Dat(op2.DataSet(nodes, 3), _smooth(V.dof_coordinates()).reshape(-1, 3)))
    k = op2.Kernel(form, degree=P, rank=2, cdim=cdim, **kw)
    sparsity = op2.Sparsity((op2.DataSet(nodes, cdim),) * 2, [(m0, m0, None)])
    return mesh, cells, m0, m1, k, sparsity, ins


def _host_call(gk, mesh, m0, m1, mat, ins, arg_bytes=True):
    """The matrix call with host pointers for every Dat and map (the Mat handle stays in args[0])."""
    layers = np.array([0, mesh.layers], dtype=np.int32)
    maps = (m0, m1)
    gk(0, mesh.num_base_cells, layers, None, [mat.handle.value] + [d._data.ctypes.data for d in ins],
       [0] + [d.nbytes for d in ins] if arg_bytes else None,
       [0] + [d.dat_version for d in ins] if arg_bytes else None,
       [m.values_with_halo.ctypes.data for m in maps], [m.values_with_halo.nbytes for m in maps],
       _lib.LOC_HOST, False, False, map_versions=[m._generation for m in maps])


@pytest.mark.parametrize("case", list(CASES))
def test_host_matrix_equals_device_matrix(engine, case):
    mesh, cells, m0, m1, k, sparsity, ins = _problem(case)
    md = op2.Mat(sparsity)
    op2.par_loop(k, cells, md(op2.INC, (m0, m0)), ins[0](op2.READ, m1), *[d(op2.READ, m0) for d in ins[1:]])
    mh = op2.Mat(sparsity)
    _host_call(op2.GlobalKernel(k, [m0, m1], extruded=True), mesh, m0, m1, mh, ins)
    want = md.values
    assert np.abs(want).max() > 0
    assert relerr(mh.values, want) < TOL


@pytest.mark.parametrize("case", list(CASES))
def test_host_matrix_without_byte_sizes_is_an_error(engine, case):
    mesh, cells, m0, m1, k, sparsity, ins = _problem(case)
    with pytest.raises(_lib.EngineError, match="host mode needs arg_bytes"):
        _host_call(op2.GlobalKernel(k, [m0, m1], extruded=True), mesh, m0, m1, op2.Mat(sparsity), ins,
                   arg_bytes=False)
