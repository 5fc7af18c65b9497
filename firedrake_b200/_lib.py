"""ctypes binding of ``libfdb200.so`` (the C ABI declared in ``include/fdb200.h``).

There is NO CPU fallback: if the shared library is missing, or no sm_90 device
is present when a compute entry point is used, this module raises.  The oracle
under ``oracle/`` is test infrastructure and is never imported from here.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FDB200_LIB", os.path.join(HERE, "lib", "libfdb200.so"))

MAX_1D = 8
BV_MAX_COLUMNS = 64                    # FDB_BV_MAX_COLUMNS: columns of one fdb_bv_dot / fdb_bv_mult operand

FORM_HELMHOLTZ = 1
FORM_DG_ADVECTION = 2
FORM_HELMHOLTZ_COEF = 3
FORM_NONLINEAR_DIFFUSION = 4
FORM_NONLINEAR_DIFFUSION_JACOBIAN = 5
FORM_ELASTICITY = 6
FORM_HYPERELASTICITY = 7
FORM_HYPERELASTICITY_JACOBIAN = 8
FORM_ADVECTION_DIFFUSION = 9
FORM_STOKES = 10
FORM_NAVIER_STOKES = 11
FORM_NAVIER_STOKES_JACOBIAN = 12
FORM_BOUNDARY_MASS = 13
FORM_INTERIOR_PENALTY = 14
FORM_DG_BOUNDARY = 15
FORM_DG_TRANSPORT = 16
FORM_P_PROLONG = 17
FORM_P_RESTRICT = 18
FORM_P_INJECT = 19
FORM_SPECTRAL_HELMHOLTZ = 20           # alpha*inner(grad u, grad v)*dx(GLL) + beta*inner(u, v)*dx(GLL)
FORM_SPECTRAL_HELMHOLTZ_COEF = 21      # the same with a trailing nodal kappa in the stiffness term
FORM_MIXED_POISSON = 22                # alpha*dot(sigma, tau)*dx + div(tau)*u*dx + div(sigma)*v*dx on NCF_k x DQ_{k-1}
FORM_MIXED_POISSON_SCHUR = 23          # its selfp Schur complement B W B^T (metric-free)
FORM_BOUSSINESQ = 24                   # Navier-Stokes + buoyancy + temperature advection-diffusion (Rayleigh-Benard)
FORM_BOUSSINESQ_JACOBIAN = 25          # its exact Gateaux derivative at (u0, T0)
FORM_MIXED_POISSON_HYBRID = 26         # mixed Poisson hybridised: the condensed trace matrix (rank 2), its load (rank 1)
FORM_MIXED_POISSON_RECONSTRUCT = 27    # (sigma, u) cell by cell from the trace multiplier lambda
FORM_TRACE_PROLONG = 28                # CG1 vertex values -> HDiv-trace face points (GTMG)
FORM_TRACE_RESTRICT = 29               # its transpose, HDiv trace -> CG1
CELL_HEX_EXTRUDED = 1
CELL_HEX = 2
CELL_TRIANGLE = 3
CELL_QUAD = 4
INTEGRAL_CELL = 0
INTEGRAL_EXTERIOR_FACET = 1
INTEGRAL_INTERIOR_FACET = 2
INTEGRAL_FUSED = 3
SCATTER_ATOMIC = 0
SCATTER_COLOURED = 1
LOC_HOST = 0
LOC_DEVICE = 1


class EngineError(RuntimeError):
    pass


class KernelDesc(C.Structure):
    _fields_ = [
        ("form", C.c_int32), ("rank", C.c_int32), ("cell", C.c_int32),
        ("integral", C.c_int32), ("degree", C.c_int32), ("nq", C.c_int32),
        ("cdim", C.c_int32), ("scatter", C.c_int32),
        ("alpha", C.c_double), ("beta", C.c_double),
        ("B", C.c_double * (MAX_1D * MAX_1D)), ("D", C.c_double * (MAX_1D * MAX_1D)),
        ("wq", C.c_double * MAX_1D), ("xq", C.c_double * MAX_1D),
        ("offset0", C.POINTER(C.c_int32)), ("offset1", C.POINTER(C.c_int32)),
        ("diagonal", C.c_int32), ("affine_cells", C.c_int32),
        ("dcoef", C.c_double * 3),
        ("lmbda", C.c_double),
    ]


class Space2Desc(C.Structure):
    """fdb_space2_desc: the second space of a form on two spaces (fdb_kernel_create_mixed)."""
    _fields_ = [
        ("degree", C.c_int32),
        ("B", C.c_double * (MAX_1D * MAX_1D)),
        ("offset", C.POINTER(C.c_int32)),
    ]


class CallArgs(C.Structure):
    _fields_ = [
        ("start", C.c_int32), ("end", C.c_int32),
        ("layers", C.POINTER(C.c_int32)), ("subset", C.c_void_p),
        ("nargs", C.c_int32), ("args", C.POINTER(C.c_void_p)),
        ("arg_bytes", C.POINTER(C.c_size_t)), ("arg_versions", C.POINTER(C.c_uint64)),
        ("nmaps", C.c_int32), ("maps", C.POINTER(C.c_void_p)),
        ("map_bytes", C.POINTER(C.c_size_t)),
        ("location", C.c_int32), ("writeback", C.c_int32), ("output_is_zero", C.c_int32),
        ("map_versions", C.POINTER(C.c_uint64)), ("subset_version", C.c_uint64),
        ("layers_count", C.c_int32), ("layers_version", C.c_uint64),
    ]


# generic wrapper builder (fdb_wrapper_*)
READ, WRITE, RW, INC, MIN, MAX = 1, 2, 3, 4, 5, 6
ARG_DAT, ARG_GLOBAL, ARG_MAT = 1, 2, 3
F64, F32, I32, U32, I64 = 1, 2, 3, 4, 5
REGION_ALL, REGION_ON_BOTTOM, REGION_ON_TOP, REGION_ON_INTERIOR_FACETS = 0, 1, 2, 3
WRAP_MAX_ARGS, WRAP_MAX_MAPS, WRAP_MAX_MATS = 16, 8, 4


class WrapperArg(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("access", C.c_int32), ("dtype", C.c_int32),
        ("dim", C.c_int32), ("dim2", C.c_int32), ("map", C.c_int32), ("map2", C.c_int32),
        ("arity", C.c_int32), ("arity2", C.c_int32),
        ("offset", C.POINTER(C.c_int32)), ("offset2", C.POINTER(C.c_int32)),
        ("permutation", C.POINTER(C.c_int32)),
        ("interior_horizontal", C.c_int32),
        ("offset_quotient", C.POINTER(C.c_int32)), ("offset_quotient2", C.POINTER(C.c_int32)),
        ("mixed_continuation", C.c_int32),
    ]


class WrapperDesc(C.Structure):
    _fields_ = [
        ("kernel_source", C.c_char_p), ("kernel_name", C.c_char_p),
        ("nargs", C.c_int32), ("args", C.POINTER(WrapperArg)),
        ("extruded", C.c_int32), ("subset", C.c_int32), ("iteration_region", C.c_int32),
        ("pass_layer_arg", C.c_int32), ("extruded_periodic", C.c_int32), ("variable_layers", C.c_int32),
    ]


# name -> (restype, argtypes); every symbol include/fdb200.h declares
SIGNATURES = {
    "fdb_init": (C.c_int, [C.c_int]),
    "fdb_finalize": (C.c_int, []),
    "fdb_last_error": (C.c_char_p, []),
    "fdb_synchronize": (C.c_int, []),
    "fdb_device_info": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_size_t)]),
    "fdb_launch_count": (C.c_uint64, []),
    "fdb_set_option": (C.c_int, [C.c_char_p, C.c_int]),
    "fdb_get_option": (C.c_int, [C.c_char_p, C.POINTER(C.c_int)]),
    "fdb_malloc": (C.c_void_p, [C.c_size_t]),
    "fdb_free": (C.c_int, [C.c_void_p]),
    "fdb_memset": (C.c_int, [C.c_void_p, C.c_int, C.c_size_t]),
    "fdb_memcpy_h2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fdb_memcpy_d2h": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fdb_memcpy_d2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fdb_zero_background": (C.c_int, [C.c_void_p, C.c_size_t]),
    "fdb_background_barrier": (C.c_int, []),
    "fdb_host_alloc": (C.c_void_p, [C.c_size_t]),
    "fdb_host_free": (C.c_int, [C.c_void_p]),
    "fdb_host_register": (C.c_int, [C.c_void_p, C.c_size_t]),
    "fdb_host_unregister": (C.c_int, [C.c_void_p]),
    "fdb_mirror_acquire": (C.c_int, [C.c_void_p, C.c_size_t, C.c_uint64, C.c_int, C.POINTER(C.c_void_p)]),
    "fdb_mirror_writeback": (C.c_int, [C.c_void_p]),
    "fdb_mirror_upload_range": (C.c_int, [C.c_void_p, C.c_size_t, C.c_size_t]),
    "fdb_mirror_download_range": (C.c_int, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int]),
    "fdb_mirror_set_version": (C.c_int, [C.c_void_p, C.c_uint64]),
    "fdb_mirror_drop": (C.c_int, [C.c_void_p]),
    "fdb_mirror_drop_all": (C.c_int, []),
    "fdb_kernel_create": (C.c_int, [C.POINTER(KernelDesc), C.POINTER(C.c_void_p)]),
    "fdb_kernel_create_mixed": (C.c_int, [C.POINTER(KernelDesc), C.POINTER(Space2Desc), C.POINTER(C.c_void_p)]),
    "fdb_kernel_destroy": (C.c_int, [C.c_void_p]),
    "fdb_cells_are_affine": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int,
                                       C.POINTER(C.c_int)]),
    "fdb_kernel_call": (C.c_int, [C.c_void_p, C.POINTER(CallArgs)]),
    "fdb_wrapper_source": (C.c_int, [C.POINTER(WrapperDesc), C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "fdb_wrapper_compile": (C.c_int, [C.POINTER(WrapperDesc), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "fdb_wrapper_create": (C.c_int, [C.POINTER(WrapperDesc), C.POINTER(C.c_void_p)]),
    "fdb_mat_create_blocked": (C.c_int, [C.c_int32, C.c_void_p, C.c_int32, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                         C.POINTER(C.c_void_p)]),
    "fdb_mat_set_diagonal_blocked": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_int]),
    "fdb_mat_create": (C.c_int, [C.c_int32, C.c_void_p, C.c_int32, C.c_int, C.c_void_p, C.c_int,
                                 C.POINTER(C.c_void_p)]),
    "fdb_mat_destroy": (C.c_int, [C.c_void_p]),
    "fdb_mat_nnz": (C.c_int, [C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_int32)]),
    "fdb_mat_zero": (C.c_int, [C.c_void_p]),
    "fdb_mat_set_lgmaps": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "fdb_mat_set_diagonal": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_double]),
    "fdb_mat_mult": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "fdb_mat_get_diagonal": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fdb_mat_get_csr": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "fdb_dat_zero_nodes": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int32]),
    "fdb_dat_set_nodes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int32]),
    "fdb_dat_set_nodes_scalar": (C.c_int, [C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_int32]),
    "fdb_vec_axpy": (C.c_int, [C.c_size_t, C.c_double, C.c_void_p, C.c_void_p]),
    "fdb_vec_aypx": (C.c_int, [C.c_size_t, C.c_double, C.c_void_p, C.c_void_p]),
    "fdb_vec_scale": (C.c_int, [C.c_size_t, C.c_double, C.c_void_p]),
    "fdb_vec_fill": (C.c_int, [C.c_size_t, C.c_double, C.c_void_p]),
    "fdb_vec_leapfrog": (C.c_int, [C.c_size_t, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "fdb_point_eval": (C.c_int, [C.c_int32, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "fdb_point_load": (C.c_int, [C.c_int32, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]),
    "fdb_vec_gather": (C.c_int, [C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    "fdb_vec_scatter": (C.c_int, [C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    "fdb_asm_create": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "fdb_asm_destroy": (C.c_int, [C.c_void_p]),
    "fdb_asm_update": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]),
    "fdb_asm_apply": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "fdb_asm_get_blocks": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fdb_fdm_star_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int32, C.c_int,
                                      C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_void_p, C.POINTER(C.c_void_p)]),
    "fdb_fdm_star_update": (C.c_int, [C.c_void_p, C.c_double, C.c_double, C.c_void_p]),
    "fdb_fdm_star_apply": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "fdb_fdm_star_destroy": (C.c_int, [C.c_void_p]),
    "fdb_vec_dot": (C.c_int, [C.c_size_t, C.c_void_p, C.c_void_p, C.POINTER(C.c_double)]),
    "fdb_bv_dot": (C.c_int, [C.c_size_t, C.c_int, C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_void_p),
                             C.POINTER(C.c_double)]),
    "fdb_bv_mult": (C.c_int, [C.c_size_t, C.c_int, C.POINTER(C.c_void_p), C.c_double, C.c_double, C.c_int,
                              C.POINTER(C.c_void_p), C.POINTER(C.c_double)]),
    "fdb_vec_pointwise_mult": (C.c_int, [C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    "fdb_vec_chebyshev": (C.c_int, [C.c_size_t, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p]),
    "fdb_interpolate_q1": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_int32, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "fdb_comm_get_unique_id": (C.c_int, [C.c_char_p]),
    "fdb_comm_init": (C.c_int, [C.c_int, C.c_int, C.c_char_p]),
    "fdb_comm_finalize": (C.c_int, []),
    "fdb_comm_rank": (C.c_int, []),
    "fdb_comm_size": (C.c_int, []),
    "fdb_halo_create": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_int, C.POINTER(C.c_void_p)]),
    "fdb_halo_destroy": (C.c_int, [C.c_void_p]),
    "fdb_halo_global_to_local_begin": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "fdb_halo_global_to_local_end": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "fdb_halo_local_to_global_begin": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "fdb_halo_local_to_global_end": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "fdb_allreduce": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "fdb_timer_create": (C.c_int, [C.POINTER(C.c_void_p)]),
    "fdb_timer_start": (C.c_int, [C.c_void_p]),
    "fdb_timer_stop": (C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
    "fdb_timer_destroy": (C.c_int, [C.c_void_p]),
    "fdb_flush_l2": (C.c_int, []),
}

_lib = None


def load():
    """Load the shared library (no GPU needed for this step)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EngineError(
            f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  firedrake_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().fdb_last_error().decode(errors="replace")
        raise EngineError(f"{what}: {msg}" if what else msg)


_initialised = None


def init(device=None):
    """Initialise the engine on ``device`` (default: LOCAL_RANK or 0)."""
    global _initialised
    lib = load()
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    if _initialised is not None:
        if _initialised != device:
            raise EngineError(f"engine already initialised on device {_initialised}")
        return lib
    check(lib.fdb_init(device), "fdb_init")
    _initialised = device
    return lib


def lib():
    """The initialised library; raises if there is no usable GPU."""
    if _initialised is None:
        return init()
    return _lib
