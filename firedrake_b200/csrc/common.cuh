// Shared internals of libfdb200 (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>

#include "../../include/fdb200.h"

namespace fdb {

struct Context {
    bool ready = false;
    int device = -1;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    uint64_t launches = 0;
    void *flush_buf = nullptr;
    size_t flush_bytes = 0;
    double *reduce_scratch = nullptr;   // device scratch for reductions
    double *reduce_host = nullptr;      // pinned
    int *work_counter = nullptr;        // device work-queue counter of the persistent kernels
};

Context &ctx();
void set_error(const char *fmt, ...);
int require_init();

#define FDB_CUDA(call)                                                              \
    do {                                                                            \
        cudaError_t e_ = (call);                                                    \
        if (e_ != cudaSuccess) {                                                    \
            fdb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call,            \
                           cudaGetErrorString(e_));                                 \
            return 1;                                                               \
        }                                                                           \
    } while (0)

#define FDB_LAUNCH_CHECK()                                                          \
    do {                                                                            \
        fdb::ctx().launches++;                                                      \
        cudaError_t e_ = cudaGetLastError();                                        \
        if (e_ != cudaSuccess) {                                                    \
            fdb::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__,        \
                           cudaGetErrorString(e_));                                 \
            return 1;                                                               \
        }                                                                           \
    } while (0)

}  // namespace fdb

extern int fdb_opt_matrix_kernel;   // fdb_set_option("matrix_kernel", ...)

struct fdb_jit_s;   // NVRTC-compiled generic wrapper (wrapper_jit.cu)
struct fdb_hex_form;   // a form of the hand-written hex kernels (global_kernel.cu)

// kernel object behind fdb_kernel_t
struct fdb_kernel_s {
    fdb_kernel_desc desc;
    int n1d;                 // p + 1
    int arity;               // dofs per cell of the argument map
    fdb_int *d_off0 = nullptr;   // device copies of the layer offsets
    fdb_int *d_off1 = nullptr;
    fdb_int h_off0[512];
    fdb_int h_off1[16];          // 8 vertices per cell, 16 on an interior facet (both cells)
    fdb_int *d_off2 = nullptr;   // a form on two spaces (FDB_FORM_STOKES): the second map's layer offsets
    fdb_int h_off2[512];
    double B2[FDB_MAX_1D * FDB_MAX_1D];   // and the second space's basis at the points, (nq, degree2 + 1)
    double Dt[FDB_MAX_1D * FDB_MAX_1D];   // collocated derivative D * B^{-1}
    // the DG facet forms: phi_a(0), phi_a(1), phi_a'(0), phi_a'(1), rows of FDB_MAX_1D
    double Bend[4 * FDB_MAX_1D];
    // colouring plan for FDB_SCATTER_COLOURED, built lazily per map
    const void *colour_map_key = nullptr;   // plan is valid for (map pointer, generation, end)
    uint64_t colour_map_gen = 0;
    fdb_int colour_end = 0;
    fdb_int *d_colour_cols = nullptr;     // columns sorted by colour
    int ncolours = 0;
    fdb_int colour_start[65];
    // dense B^T D B path (bdb_matrix.cu): tabulated reference gradients / values, built lazily
    double *d_bdb_table = nullptr;
    // non-NULL: this handle is a generated wrapper around an arbitrary local kernel
    fdb_jit_s *jit = nullptr;
    // the form's row for the hex kernels; NULL for DG advection, P1 triangles and generated wrappers
    const fdb_hex_form *hex = nullptr;
};

int fdb_jit_call(fdb_kernel_s *k, const fdb_call_args *a);
void fdb_jit_destroy(fdb_jit_s *j);

extern "C" int fdb_mirror_set_version(const void *host, uint64_t version);
bool fdb_mirror_is_current(const void *host, size_t nbytes, uint64_t version);
void fdb_mirror_new_epoch();   // start of a kernel call: mirrors touched from now on are pinned

typedef struct fdb_mat_s *fdb_mat_t;
int fdb_mat_device_view(fdb_mat_t m, const long long **rowptr, const fdb_int **colidx, double **vals,
                        const fdb_int **row_lg, const fdb_int **col_lg);
int fdb_mat_rank_table(fdb_mat_t m, const unsigned short **rank, int *nvar);
int fdb_mat_block_size(fdb_mat_t m, int *bs);
int fdb_mat_rows(fdb_mat_t m, fdb_int *nrows);      // node rows (block rows if blocked)
int fdb_mat_scalar_view_begin(fdb_mat_t blocked, fdb_mat_t *view);
int fdb_mat_scalar_view_end(fdb_mat_t blocked, fdb_mat_t view);
int fdb_launch_helmholtz_matrix(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay,
                                const fdb_int *subset, fdb_mat_t mat, const double *coords,
                                const fdb_int *map0, const fdb_int *map1, double *diag_out);

int fdb_launch_helmholtz_matrix_dmma(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay,
                                     const fdb_int *subset, fdb_mat_t mat, const double *coords,
                                     const fdb_int *map0, const fdb_int *map1);

int fdb_launch_tri_p1(fdb_kernel_s *k, fdb_int start, fdb_int end, const fdb_int *subset, double *y,
                      const double *coords, const double *x, const fdb_int *map, fdb_mat_t mat);
int fdb_launch_dg_advection(fdb_kernel_s *k, fdb_int start, fdb_int end, const fdb_int *subset,
                            double *out, const double *coords, const double *q, const double *u,
                            const double *consts_host, const unsigned *facet, const fdb_int *dgmap,
                            const fdb_int *cgmap, const fdb_int *nbr);

int fdb_launch_q1_action(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                         double *y, const double *coords, const double *x, const fdb_int *map0,
                         const fdb_int *map1);

int fdb_launch_q2_action(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                         double *y, const double *coords, const double *x, const fdb_int *map0,
                         const fdb_int *map1);

// launchers implemented in the kernel translation units
int fdb_launch_helmholtz_action(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay,
                                const fdb_int *subset, double *y, const double *coords,
                                const double *x, const fdb_int *map0, const fdb_int *map1);
// FDB_FORM_HELMHOLTZ_COEF (action_hex.cu): kappa is a device pointer gathered through map0
int fdb_launch_helmholtz_coef_action(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay,
                                     const fdb_int *subset, double *y, const double *coords,
                                     const double *x, const double *kappa, const fdb_int *map0,
                                     const fdb_int *map1);
int fdb_launch_helmholtz_coef_matrix(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay,
                                     const fdb_int *subset, fdb_mat_t mat, const double *coords,
                                     const double *kappa, const fdb_int *map0, const fdb_int *map1,
                                     double *diag_out);
// FDB_FORM_ELASTICITY and FDB_FORM_HYPERELASTICITY[_JACOBIAN] (elasticity_hex.cu): x, y, u and diag_out are
// AoS with 3 values per node; mat has block size 3 (diag_out is used when mat is NULL).  u is the
// Jacobian's linearisation point (NULL for the other forms; the residual's u is x)
int fdb_launch_elasticity_action(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                                 double *y, const double *coords, const double *x, const double *u,
                                 const fdb_int *map0, const fdb_int *map1);
int fdb_launch_elasticity_matrix(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                                 fdb_mat_t mat, const double *coords, const double *u, const fdb_int *map0,
                                 const fdb_int *map1, double *diag_out);
// FDB_FORM_STOKES (elasticity_hex.cu): yu and u AoS with 3 values per node of map0, yp and p one value per
// node of map2 (the pressure map).  FDB_FORM_NAVIER_STOKES[_JACOBIAN] run through it too: ulin is the
// Jacobian's linearisation velocity (AoS through map0), NULL for the other two forms
int fdb_launch_stokes_action(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                             double *yu, const double *coords, const double *u, double *yp, const double *p,
                             const double *ulin, const fdb_int *map0, const fdb_int *map1, const fdb_int *map2);
// FDB_FORM_BOUNDARY_MASS (boundary_hex.cu): one exterior facet per iteration entry, facet[col] its local facet
// number.  mat != NULL: the element matrices into mat; else x != NULL: the action into y; else the diagonal
// into y (cdim values per node, the same in each component)
int fdb_launch_boundary_mass(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                             fdb_mat_t mat, double *y, const double *coords, const double *x, const unsigned *facet,
                             const fdb_int *map0, const fdb_int *map1);
// FDB_FORM_INTERIOR_PENALTY and FDB_FORM_DG_BOUNDARY (dg_facet_hex.cu): one facet per iteration entry, facet[col *
// sides + side] its local facet numbers ('+' first).  x != NULL: the action into y; else the diagonal into y
int fdb_launch_dg_facet(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
                        const double *coords, const double *x, const unsigned *facet, const fdb_int *map0,
                        const fdb_int *map1);
// FDB_FORM_DG_TRANSPORT: the cell term (dg_transport_hex.cu, facet == NULL) or the upwind facet terms
// (dg_facet_hex.cu); b holds 3 values per vertex, read through map1.  x != NULL: the action; else the diagonal
int fdb_launch_dg_transport(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
                            const double *coords, const double *x, const double *b, const unsigned *facet,
                            const fdb_int *map0, const fdb_int *map1);
int fdb_launch_dg_upwind(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
                         const double *coords, const double *x, const double *b, const unsigned *facet,
                         const fdb_int *map0, const fdb_int *map1);
// FDB_FORM_P_PROLONG / P_RESTRICT / P_INJECT (p_transfer_hex.cu): mapf the fine rows ((degree+1)^3), mapc the coarse
// rows ((nq)^3); w the restriction's fine-node weights (NULL for the other two)
int fdb_launch_p_transfer(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *out,
                          const double *in, const double *w, const fdb_int *mapf, const fdb_int *mapc);
// FDB_FORM_SPECTRAL_HELMHOLTZ[_COEF] (sem_hex.cu): the collocated GLL kernel; kappa (nodal, through map0) or NULL.
// x != NULL: the action into y; else the diagonal into y.  Atomic or coloured scatter (the colouring of map0)
int fdb_launch_spectral_helmholtz(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                                  double *y, const double *coords, const double *x, const double *kappa,
                                  const fdb_int *map0, const fdb_int *map1);
