// "Compile" and call of a global kernel: the replacement for
// pyop2.global_kernel.compile_global_kernel + GlobalKernel.__call__
// (reference pyop2/global_kernel.py:327-335, 426-456).  fdb_kernel_create compiles
// nothing: it validates the descriptor against the set of hand-written sm_90a
// kernels and precomputes the tables they need.  Handles made by
// fdb_wrapper_create (wrapper_jit.cu: NVRTC wrapper around an arbitrary local
// kernel) are dispatched from fdb_kernel_call as well.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

using namespace fdb;

namespace {

// Dt = D * B^{-1}  (collocated derivative on the quadrature points).
// Solves X B = D by Gaussian elimination with partial pivoting on B^T X^T = D^T.
int collocated_derivative(int n, const double *B, const double *D, double *Dt)
{
    double A[FDB_MAX_1D][FDB_MAX_1D], R[FDB_MAX_1D][FDB_MAX_1D];
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) {
            A[i][j] = B[j * n + i];   // B^T
            R[i][j] = D[j * n + i];   // D^T
        }
    for (int c = 0; c < n; c++) {
        int piv = c;
        for (int r = c + 1; r < n; r++)
            if (fabs(A[r][c]) > fabs(A[piv][c])) piv = r;
        if (fabs(A[piv][c]) < 1e-14) return 1;
        if (piv != c)
            for (int j = 0; j < n; j++) {
                std::swap(A[piv][j], A[c][j]);
                std::swap(R[piv][j], R[c][j]);
            }
        for (int r = 0; r < n; r++) {
            if (r == c) continue;
            double f = A[r][c] / A[c][c];
            for (int j = 0; j < n; j++) {
                A[r][j] -= f * A[c][j];
                R[r][j] -= f * R[c][j];
            }
        }
    }
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) Dt[j * n + i] = R[i][j] / A[i][i];   // X = (X^T)^T
    return 0;
}

// The basis and its derivative at the ends of the interval, Bend[e * FDB_MAX_1D + a] = phi_a(0), phi_a(1),
// phi_a'(0), phi_a'(1) for e = 0..3, from the basis at the n Gauss points: a degree-(n-1) polynomial is its
// Lagrange interpolant through them, phi_a(x) = sum_q B[q][a] L_q(x), exactly.
void endpoint_tables(int n, const double *B, const double *xq, double *Bend)
{
    for (int e = 0; e < 2; e++) {
        const double x = (double)e;
        for (int q = 0; q < n; q++) {
            double den = 1.0, val = 1.0, der = 0.0;
            for (int r = 0; r < n; r++) {
                if (r == q) continue;
                den *= xq[q] - xq[r];
                der = der * (x - xq[r]) + val;      // (prod_r (x - x_r))' by the product rule
                val *= x - xq[r];
            }
            for (int a = 0; a < n; a++) {
                Bend[e * FDB_MAX_1D + a] += B[q * n + a] * val / den;
                Bend[(2 + e) * FDB_MAX_1D + a] += B[q * n + a] * der / den;
            }
        }
    }
}

// Greedy colouring of columns (base cells) so that no two columns of one
// colour share a dof column: the deterministic fallback of the north_star
// ("warp-aggregated atomic kernel with a colouring fallback").  Host side,
// once per map.
int build_colouring(fdb_kernel_s *k, const fdb_int *h_map, fdb_int ncols, int arity)
{
    fdb_int maxnode = 0;
    for (long long i = 0; i < (long long)ncols * arity; i++) maxnode = std::max(maxnode, h_map[i]);
    // node -> bitmask of colours already used by a column touching it
    std::vector<uint64_t> used((size_t)maxnode + 1, 0);
    std::vector<int> colour(ncols);
    int ncolours = 0;
    for (fdb_int c = 0; c < ncols; c++) {
        uint64_t m = 0;
        for (int i = 0; i < arity; i++) m |= used[h_map[(size_t)c * arity + i]];
        int col = 0;
        while (col < 64 && (m >> col) & 1) col++;
        if (col >= 64) {
            set_error("colouring needs more than 64 colours");
            return 1;
        }
        colour[c] = col;
        ncolours = std::max(ncolours, col + 1);
        for (int i = 0; i < arity; i++) used[h_map[(size_t)c * arity + i]] |= (uint64_t)1 << col;
    }
    std::vector<fdb_int> sorted(ncols);
    int pos = 0;
    for (int col = 0; col < ncolours; col++) {
        k->colour_start[col] = pos;
        for (fdb_int c = 0; c < ncols; c++)
            if (colour[c] == col) sorted[pos++] = c;
    }
    k->colour_start[ncolours] = pos;
    k->ncolours = ncolours;
    if (k->d_colour_cols) cudaFree(k->d_colour_cols);
    FDB_CUDA(cudaMalloc(&k->d_colour_cols, sizeof(fdb_int) * std::max(ncols, 1)));
    FDB_CUDA(cudaMemcpyAsync(k->d_colour_cols, sorted.data(), sizeof(fdb_int) * ncols,
                             cudaMemcpyHostToDevice, ctx().stream));
    FDB_CUDA(cudaStreamSynchronize(ctx().stream));
    return 0;
}

// Drop-in (host pointer) call of a 1-form with the output just zeroed by the
// assembler: instead of "upload x, compute, download y" back to back, the
// iteration range is cut into chunks of columns and three streams overlap
//     H2D of the x rows chunk k+1 needs  |  kernel on chunk k  |  D2H of the
//     y rows no later chunk can touch
// (PCIe is full duplex, so the end-to-end time tends to max(H2D, D2H) instead
// of their sum).  Which rows a chunk touches is read off the map on the host:
// with Firedrake's cell-closure numbering the touched range grows monotonically
// with the chunk index; for an arbitrary numbering the schedule degenerates to
// the monolithic one by construction (everything uploaded before chunk 0,
// downloaded after the last), never to a wrong one.
static inline uint64_t map_ver(const fdb_call_args *a, int i)
{
    return a->map_versions ? a->map_versions[i] : 0;
}

struct PipelinePlan {
    const void *map_key = nullptr;
    uint64_t map_gen = 0;
    fdb_int start = 0, end = 0;
    int nlay = 0;
    std::vector<fdb_int> c0, c1;          // column range of each chunk
    std::vector<long long> upto;          // rows [0, upto[k]) must be resident before chunk k
    std::vector<long long> final_below;   // rows [0, final_below[k]) are final after chunk k
};
static PipelinePlan g_plan;
static cudaStream_t g_h2d = nullptr, g_d2h = nullptr;
static std::vector<cudaEvent_t> g_ev_up, g_ev_done;

static int pipelined_host_action(fdb_kernel_s *k, const fdb_call_args *a, int nlay)
{
    static const int nchunks_env = getenv("FDB_PIPELINE_CHUNKS") ? atoi(getenv("FDB_PIPELINE_CHUNKS")) : 32;
    const fdb_int ncols = a->end - a->start;
    int K = nchunks_env;
    if (K <= 1 || ncols < 64 * K) return -1;
    const int arity = k->arity;
    const size_t nrows = a->arg_bytes[0] / (sizeof(double) * k->desc.cdim);
    cudaStream_t st = ctx().stream;
    if (!g_h2d) {
        FDB_CUDA(cudaStreamCreateWithFlags(&g_h2d, cudaStreamNonBlocking));
        FDB_CUDA(cudaStreamCreateWithFlags(&g_d2h, cudaStreamNonBlocking));
    }
    while ((int)g_ev_up.size() < K) {
        cudaEvent_t e1, e2;
        FDB_CUDA(cudaEventCreateWithFlags(&e1, cudaEventDisableTiming));
        FDB_CUDA(cudaEventCreateWithFlags(&e2, cudaEventDisableTiming));
        g_ev_up.push_back(e1);
        g_ev_done.push_back(e2);
    }
    PipelinePlan &pl = g_plan;
    if (pl.map_key != (const void *)a->maps[0] || pl.map_gen != map_ver(a, 0) || pl.start != a->start ||
        pl.end != a->end ||
        pl.nlay != nlay || (int)pl.c0.size() != K) {
        // host analysis of the map (cached while the same map is passed)
        const fdb_int *map = a->maps[0];
        pl = PipelinePlan();
        pl.map_key = a->maps[0];
        pl.map_gen = map_ver(a, 0);
        pl.start = a->start;
        pl.end = a->end;
        pl.nlay = nlay;
        std::vector<long long> lo(K), hi(K);
        for (int c = 0; c < K; c++) {
            fdb_int b0 = a->start + (fdb_int)((long long)ncols * c / K);
            fdb_int b1 = a->start + (fdb_int)((long long)ncols * (c + 1) / K);
            pl.c0.push_back(b0);
            pl.c1.push_back(b1);
            long long l = (long long)nrows, h = 0;
            for (fdb_int col = b0; col < b1; col++)
                for (int i = 0; i < arity; i++) {
                    long long v = map[(size_t)col * arity + i];
                    long long top = v + (long long)k->h_off0[i] * (nlay - 1);
                    if (v < l) l = v;
                    if (top + 1 > h) h = top + 1;
                }
            lo[c] = l;
            hi[c] = h;
        }
        pl.upto.resize(K);
        pl.final_below.resize(K);
        long long m = 0;
        for (int c = 0; c < K; c++) {
            if (hi[c] > m) m = hi[c];
            pl.upto[c] = m;
        }
        long long mn = (long long)nrows;
        for (int c = K - 1; c >= 0; c--) {
            pl.final_below[c] = mn;          // min over later chunks of their lowest row
            if (lo[c] < mn) mn = lo[c];
        }
        pl.final_below[K - 1] = (long long)nrows;
    }
    void *dy, *dx, *dc, *dm0, *dm1;
    // static inputs through the mirror cache (uploaded once)
    if (fdb_mirror_acquire(a->args[1], a->arg_bytes[1], a->arg_versions[1], 1, &dc)) return 1;
    if (fdb_mirror_acquire(a->maps[0], a->map_bytes[0], map_ver(a, 0), 1, &dm0)) return 1;
    if (fdb_mirror_acquire(a->maps[1], a->map_bytes[1], map_ver(a, 1), 1, &dm1)) return 1;
    if (fdb_mirror_acquire(a->args[0], a->arg_bytes[0], a->arg_versions[0], 0, &dy)) return 1;
    bool x_current = fdb_mirror_is_current(a->args[2], a->arg_bytes[2], a->arg_versions[2]);
    if (fdb_mirror_acquire(a->args[2], a->arg_bytes[2], a->arg_versions[2], 0, &dx)) return 1;
    const size_t rowb = sizeof(double) * k->desc.cdim;
    // uploads wait for whatever the engine stream was doing with these buffers
    FDB_CUDA(cudaEventRecord(g_ev_done[0], st));
    FDB_CUDA(cudaStreamWaitEvent(g_h2d, g_ev_done[0], 0));
    FDB_CUDA(cudaStreamWaitEvent(g_d2h, g_ev_done[0], 0));
    // rows above the highest touched one: never gathered, must still read as zero
    if (pl.upto[K - 1] < (long long)nrows)
        FDB_CUDA(cudaMemsetAsync((char *)dy + pl.upto[K - 1] * rowb, 0,
                                 (size_t)((long long)nrows - pl.upto[K - 1]) * rowb, st));
    long long up_done = 0, down_done = 0;
    for (int c = 0; c < K; c++) {
        if (pl.upto[c] > up_done) {
            if (!x_current)
                FDB_CUDA(cudaMemcpyAsync((char *)dx + up_done * rowb, (const char *)a->args[2] + up_done * rowb,
                                         (size_t)(pl.upto[c] - up_done) * rowb, cudaMemcpyHostToDevice, g_h2d));
            FDB_CUDA(cudaMemsetAsync((char *)dy + up_done * rowb, 0, (size_t)(pl.upto[c] - up_done) * rowb, st));
            up_done = pl.upto[c];
        }
        FDB_CUDA(cudaEventRecord(g_ev_up[c], g_h2d));
        FDB_CUDA(cudaStreamWaitEvent(st, g_ev_up[c], 0));
        if (fdb_launch_helmholtz_action(k, pl.c0[c], pl.c1[c], nlay, nullptr, (double *)dy, (const double *)dc,
                                        (const double *)dx, (const fdb_int *)dm0, (const fdb_int *)dm1))
            return 1;
        FDB_CUDA(cudaEventRecord(g_ev_done[c], st));
        if (pl.final_below[c] > down_done) {
            FDB_CUDA(cudaStreamWaitEvent(g_d2h, g_ev_done[c], 0));
            FDB_CUDA(cudaMemcpyAsync((char *)a->args[0] + down_done * rowb, (const char *)dy + down_done * rowb,
                                     (size_t)(pl.final_below[c] - down_done) * rowb, cudaMemcpyDeviceToHost, g_d2h));
            down_done = pl.final_below[c];
        }
    }
    FDB_CUDA(cudaStreamSynchronize(g_d2h));
    FDB_CUDA(cudaStreamSynchronize(st));
    if (up_done == (long long)nrows) fdb_mirror_set_version(a->args[2], a->arg_versions[2]);
    fdb_mirror_set_version(a->args[0], a->arg_versions[0] + 1);
    return 0;
}

// The call's pointers on the device.  Device mode passes them through.  Host mode mirrors every Dat
// argument (not the Mat handle in args[0] of a matrix call), both maps and the subset; an output the
// caller has just zeroed is zero-filled on the device instead of uploaded.
static int device_pointers(const fdb_call_args *a, bool mat, void **args, const fdb_int **maps,
                           const fdb_int **subset)
{
    for (int i = 0; i < a->nargs; i++) args[i] = a->args[i];
    for (int i = 0; i < a->nmaps; i++) maps[i] = a->maps[i];
    *subset = a->subset;
    if (a->location != FDB_LOC_HOST) return 0;
    if (!a->arg_bytes || !a->map_bytes) {
        set_error("fdb_kernel_call: host mode needs arg_bytes and map_bytes");
        return 1;
    }
    for (int i = mat ? 1 : 0; i < a->nargs; i++) {
        // without versions every call re-uploads (drop-in default: the
        // reference hands over live NumPy buffers)
        if (!a->arg_versions) fdb_mirror_drop(a->args[i]);
        const bool zero_out = (i == 0 && a->output_is_zero);
        if (fdb_mirror_acquire(a->args[i], a->arg_bytes[i], a->arg_versions ? a->arg_versions[i] : 0,
                               zero_out ? 0 : 1, &args[i]))
            return 1;
        if (zero_out) FDB_CUDA(cudaMemsetAsync(args[i], 0, a->arg_bytes[i], ctx().stream));
    }
    void *p;
    for (int i = 0; i < 2; i++) {
        if (fdb_mirror_acquire(a->maps[i], a->map_bytes[i], map_ver(a, i), 1, &p)) return 1;
        maps[i] = (const fdb_int *)p;
    }
    if (a->subset) {
        if (fdb_mirror_acquire(a->subset, sizeof(fdb_int) * (size_t)a->end, a->subset_version, 1, &p)) return 1;
        *subset = (const fdb_int *)p;
    }
    return 0;
}

}  // namespace

// The forms of the hand-written hex kernels: what fdb_kernel_create accepts for each and how
// fdb_kernel_call hands its arguments to the launchers.
enum { MODE_ACTION, MODE_MATRIX, MODE_DIAGONAL };
enum { LAUNCH_HELMHOLTZ, LAUNCH_HELMHOLTZ_COEF, LAUNCH_ELASTICITY, LAUNCH_STOKES, LAUNCH_BOUNDARY, LAUNCH_DG_FACET,
       LAUNCH_DG_TRANSPORT, LAUNCH_P_TRANSFER, LAUNCH_SPECTRAL, LAUNCH_HDIV, LAUNCH_HYBRID, LAUNCH_TRACE_TRANSFER };
// the degree of the second space of a form on two spaces: the descriptor's degree - 1 (Stokes' pressure, the
// default of a row that does not name one), or any lower degree of an instantiated (fine, coarse) pair (the
// p-multigrid transfers), or CG1 (the trace transfers)
enum { SPACE2_PRESSURE = 0, SPACE2_COARSER };
enum { SPACE2_CG1 = SPACE2_COARSER + 1 };

struct fdb_hex_form {
    int form;                 // enum fdb_form
    const char *name;
    int cdim;                 // value size of the argument space; 0: any of 1..3, the diagonal scalar only;
                              // -1: 1 or 3 in every mode
    bool affine;              // has the affine_cells variant
    const char *coef;         // the trailing coefficient argument (an exterior-facet form: the uint32 local
                              // facet number of each entry), or NULL
    int coef_cdim;            // its values per node (0 without one): the argument space's, or 3 for b
    bool residual;            // a 1-form action only
    int launcher;             // fdb_launch_helmholtz_*, fdb_launch_helmholtz_coef_* (which also run the
                              // nonlinear diffusion and advection-diffusion forms), fdb_launch_elasticity_*
                              // fdb_launch_stokes_action (which also runs the Navier-Stokes and Boussinesq forms),
                              // fdb_launch_boundary_mass, fdb_launch_dg_facet (the DG facet forms),
                              // fdb_launch_dg_transport or fdb_launch_spectral_helmholtz
    int max_degree[3];        // per mode: action, matrix, diagonal
    int min_degree;
    const char *space2;       // the arguments on a second space (output and input, through a third map), or
                              // NULL: such a form is an action only, in device mode
    int integral;             // enum fdb_integral: facet forms run in device mode only; -1: the descriptor's
                              // integral (cell, exterior or interior facet) selects the term
    int space2_degree;        // SPACE2_*: the degree the second space must have (read when space2 is set)
    const char *field3;       // the arguments of a third field on the second space's map (output and input, after
                              // the second space's: Boussinesq's temperature), or NULL
    int ncoef;                // the number of trailing coefficient arguments when coef names more than one
                              // (Boussinesq's Jacobian: u0, T0), 0: one
};

static const fdb_hex_form hex_forms[] = {
    {FDB_FORM_HELMHOLTZ, "helmholtz", 0, true, nullptr, 0, false, LAUNCH_HELMHOLTZ, {5, 4, 3}, 1, nullptr, FDB_INTEGRAL_CELL},
    {FDB_FORM_HELMHOLTZ_COEF, "helmholtz_coef", 1, false, "kappa", 1, false, LAUNCH_HELMHOLTZ_COEF, {5, 4, 3}, 1,
     nullptr, FDB_INTEGRAL_CELL},
    {FDB_FORM_NONLINEAR_DIFFUSION, "nonlinear_diffusion", 1, false, nullptr, 0, true, LAUNCH_HELMHOLTZ_COEF,
     {5, 0, 0}, 1, nullptr, FDB_INTEGRAL_CELL},
    {FDB_FORM_NONLINEAR_DIFFUSION_JACOBIAN, "nonlinear_diffusion_jacobian", 1, false, "u", 1, false,
     LAUNCH_HELMHOLTZ_COEF, {5, 4, 3}, 1, nullptr, FDB_INTEGRAL_CELL},
    {FDB_FORM_ELASTICITY, "elasticity", 3, false, nullptr, 0, false, LAUNCH_ELASTICITY, {4, 3, 3}, 1, nullptr, FDB_INTEGRAL_CELL},
    {FDB_FORM_HYPERELASTICITY, "hyperelasticity", 3, false, nullptr, 0, true, LAUNCH_ELASTICITY, {4, 0, 0}, 1,
     nullptr, FDB_INTEGRAL_CELL},
    {FDB_FORM_HYPERELASTICITY_JACOBIAN, "hyperelasticity_jacobian", 3, false, "u", 3, false, LAUNCH_ELASTICITY,
     {4, 3, 3}, 1, nullptr, FDB_INTEGRAL_CELL},
    {FDB_FORM_ADVECTION_DIFFUSION, "advection_diffusion", 1, false, "b", 3, false, LAUNCH_HELMHOLTZ_COEF,
     {4, 3, 3}, 1, nullptr, FDB_INTEGRAL_CELL},
    // velocity CG_p with pressure CG_{p-1}: p >= 2
    {FDB_FORM_STOKES, "stokes", 3, false, nullptr, 0, false, LAUNCH_STOKES, {4, 0, 0}, 2, "y_p, p", FDB_INTEGRAL_CELL},
    {FDB_FORM_NAVIER_STOKES, "navier_stokes", 3, false, nullptr, 0, true, LAUNCH_STOKES, {4, 0, 0}, 2, "y_p, p", FDB_INTEGRAL_CELL},
    {FDB_FORM_NAVIER_STOKES_JACOBIAN, "navier_stokes_jacobian", 3, false, "u", 3, false, LAUNCH_STOKES, {4, 0, 0}, 2,
     "y_p, p", FDB_INTEGRAL_CELL},
    // Navier-Stokes coupled to a temperature in CG_{p-1} on the pressure map: [y_u, coords, u, y_p, p, y_T, T]; the
    // Jacobian reads its linearisation point (u0 through the velocity map, T0 through the pressure map) last
    {FDB_FORM_BOUSSINESQ, "boussinesq", 3, false, nullptr, 0, true, LAUNCH_STOKES, {4, 0, 0}, 2, "y_p, p",
     FDB_INTEGRAL_CELL, SPACE2_PRESSURE, "y_T, T"},
    {FDB_FORM_BOUSSINESQ_JACOBIAN, "boussinesq_jacobian", 3, false, "u0, T0", 3, false, LAUNCH_STOKES, {4, 0, 0}, 2,
     "y_p, p", FDB_INTEGRAL_CELL, SPACE2_PRESSURE, "y_T, s", 2},
    // gamma*inner(u, v)*ds: one exterior facet of one cell per entry, its local facet number last
    {FDB_FORM_BOUNDARY_MASS, "boundary_mass", -1, false, "facet", 1, false, LAUNCH_BOUNDARY, {5, 4, 5}, 1, nullptr,
     FDB_INTEGRAL_EXTERIOR_FACET},
    // the SIPG facet terms on DQ_p: one interior facet ('+' row, '-' row) per entry, the two local facet numbers
    // last; and the Nitsche / load terms on exterior facets.  No rank 2 (no assembled DG matrix)
    {FDB_FORM_INTERIOR_PENALTY, "interior_penalty", 1, false, "facets", 1, false, LAUNCH_DG_FACET, {4, 0, 4}, 1,
     nullptr, FDB_INTEGRAL_INTERIOR_FACET},
    {FDB_FORM_DG_BOUNDARY, "dg_boundary", 1, false, "facet", 1, false, LAUNCH_DG_FACET, {4, 0, 4}, 1, nullptr,
     FDB_INTEGRAL_EXTERIOR_FACET},
    // upwind DG transport on DQ_p: b (3 values per vertex, through the vertex map), then on facets the local
    // facet numbers.  Device mode only, no rank 2
    {FDB_FORM_DG_TRANSPORT, "dg_transport", 1, false, "b", 3, false, LAUNCH_DG_TRANSPORT, {4, 0, 4}, 1, nullptr, -1},
    // the p-multigrid degree transfers: the descriptor is the fine space CG_p, the second space the coarse CG_q, and
    // R (desc.B, nq = q+1) and P (space2.B) their 1-D tables.  Device mode only, rank 1, no diagonal
    {FDB_FORM_P_PROLONG, "p_prolong", -1, false, nullptr, 0, false, LAUNCH_P_TRANSFER, {3, 0, 0}, 2, "coarse",
     FDB_INTEGRAL_CELL, SPACE2_COARSER},
    {FDB_FORM_P_RESTRICT, "p_restrict", -1, false, nullptr, 0, false, LAUNCH_P_TRANSFER, {3, 0, 0}, 2, "fine, w",
     FDB_INTEGRAL_CELL, SPACE2_COARSER},
    {FDB_FORM_P_INJECT, "p_inject", -1, false, nullptr, 0, false, LAUNCH_P_TRANSFER, {3, 0, 0}, 2, "fine",
     FDB_INTEGRAL_CELL, SPACE2_COARSER},
    // the spectral-element Helmholtz operator on the collocated GLL rule, without and with a nodal kappa (one kernel
    // template).  Device mode only, action and diagonal, no rank 2; no second space (space2_degree is the default)
    {FDB_FORM_SPECTRAL_HELMHOLTZ, "spectral_helmholtz", 1, false, nullptr, 0, false, LAUNCH_SPECTRAL, {5, 0, 5}, 1,
     nullptr, FDB_INTEGRAL_CELL, SPACE2_PRESSURE},
    {FDB_FORM_SPECTRAL_HELMHOLTZ_COEF, "spectral_helmholtz_coef", 1, false, "kappa", 1, false, LAUNCH_SPECTRAL,
     {5, 0, 5}, 1, nullptr, FDB_INTEGRAL_CELL, SPACE2_PRESSURE},
    // mixed Poisson on NCF_k x DQ_{k-1} (the descriptor is the flux space, the second space the DQ one), and its
    // metric-free selfp Schur complement.  Device mode only, action and diagonal, no rank 2 (hdiv_call)
    {FDB_FORM_MIXED_POISSON, "mixed_poisson", 1, false, nullptr, 0, false, LAUNCH_HDIV, {4, 0, 4}, 2, "y_u, u",
     FDB_INTEGRAL_CELL, SPACE2_PRESSURE},
    {FDB_FORM_MIXED_POISSON_SCHUR, "mixed_poisson_schur", 1, false, nullptr, 0, false, LAUNCH_HDIV, {4, 0, 4}, 2,
     "w, t", FDB_INTEGRAL_CELL, SPACE2_PRESSURE},
    // its hybridisation on the HDiv-trace space: the condensed trace matrix (rank 2) and the elimination of the load
    // (rank 1), and the reconstruction of (sigma, u) from lambda.  Device mode, atomic scatter, k = 2..3 (hybrid_call)
    {FDB_FORM_MIXED_POISSON_HYBRID, "mixed_poisson_hybrid", 1, false, nullptr, 0, false, LAUNCH_HYBRID, {3, 3, 0}, 2,
     "f_sigma, w, f_u", FDB_INTEGRAL_CELL, SPACE2_PRESSURE},
    {FDB_FORM_MIXED_POISSON_RECONSTRUCT, "mixed_poisson_reconstruct", 1, false, nullptr, 0, false, LAUNCH_HYBRID,
     {3, 0, 0}, 2, "lambda, f_sigma, w, y_u, f_u", FDB_INTEGRAL_CELL, SPACE2_PRESSURE},
    // the GTMG transfers between CG1 and that trace space: the descriptor is the trace space (degree k - 1), the
    // second space CG1.  Device mode only, rank 1, no diagonal (trace_transfer_call)
    {FDB_FORM_TRACE_PROLONG, "trace_prolong", 1, false, nullptr, 0, false, LAUNCH_TRACE_TRANSFER, {2, 0, 0}, 1, "c",
     FDB_INTEGRAL_CELL, SPACE2_CG1},
    {FDB_FORM_TRACE_RESTRICT, "trace_restrict", 1, false, nullptr, 0, false, LAUNCH_TRACE_TRANSFER, {2, 0, 0}, 1,
     "lambda, w", FDB_INTEGRAL_CELL, SPACE2_CG1},
};

// the (fine, coarse) degree pairs the transfer kernels instantiate (p_transfer_hex.cu)
static bool p_transfer_pair(int p, int q)
{
    return (p == 2 && q == 1) || (p == 3 && q == 1) || (p == 3 && q == 2);
}

static const char *const mode_name[] = {"action", "matrix", "diagonal"};

// rank 2 is the matrix whatever the diagonal flag says
static int hex_mode(const fdb_kernel_desc *d)
{
    return d->rank == 2 ? MODE_MATRIX : (d->diagonal ? MODE_DIAGONAL : MODE_ACTION);
}

// fdb_kernel_create (s2 == NULL) and fdb_kernel_create_mixed (s2: the second space of a form on two spaces)
static int kernel_create(const fdb_kernel_desc *d, const fdb_space2_desc *s2, fdb_kernel_t *out)
{
    if (require_init()) return 1;
    if (!d || !out) {
        set_error("fdb_kernel_create: NULL argument");
        return 1;
    }
    if (d->form == FDB_FORM_DG_ADVECTION) {
        if (d->cell != FDB_CELL_QUAD || d->rank != 1 || d->degree != 1 || d->cdim != 1 ||
            d->nq < 1 || d->nq > FDB_MAX_1D || d->integral < 0 || d->integral > FDB_INTEGRAL_FUSED) {
            set_error("fdb_kernel_create: DG advection is DQ1 on quads, rank 1, nq <= %d", FDB_MAX_1D);
            return 1;
        }
        fdb_kernel_s *k = new fdb_kernel_s;
        k->desc = *d;
        k->n1d = 2;
        k->arity = d->integral == FDB_INTEGRAL_INTERIOR_FACET ? 8 : 4;
        k->desc.offset0 = k->desc.offset1 = nullptr;
        *out = k;
        return 0;
    }
    if (d->form == FDB_FORM_HELMHOLTZ && d->cell == FDB_CELL_TRIANGLE) {
        // affine P1 triangles: B = basis table (3, nq), D = reference gradients (3, 2)
        if (d->degree != 1 || d->cdim != 1 || d->nq < 1 || d->nq > FDB_MAX_1D ||
            (d->rank != 1 && d->rank != 2) || d->integral != FDB_INTEGRAL_CELL) {
            set_error("fdb_kernel_create: triangle kernels are P1, scalar, nq <= %d", FDB_MAX_1D);
            return 1;
        }
        fdb_kernel_s *k = new fdb_kernel_s;
        k->desc = *d;
        k->n1d = 2;
        k->arity = 3;
        k->desc.offset0 = k->desc.offset1 = nullptr;
        *out = k;
        return 0;
    }
    const fdb_hex_form *f = nullptr;
    for (const fdb_hex_form &row : hex_forms)
        if (row.form == d->form) f = &row;
    if (!f) {
        set_error("fdb_kernel_create: form %d is not in the supported set", d->form);
        return 1;
    }
    if (f->space2 && !s2) {
        set_error("fdb_kernel_create: %s is a form on two spaces: create it with fdb_kernel_create_mixed and the "
                  "second space's fdb_space2_desc", f->name);
        return 1;
    }
    const int mode = hex_mode(d);
    if (d->cell != FDB_CELL_HEX_EXTRUDED && d->cell != FDB_CELL_HEX) {
        set_error("fdb_kernel_create: %s needs hex cells (extruded or native), got cell %d", f->name, d->cell);
        return 1;
    }
    if (f->cdim < 0 && d->cdim != 1 && d->cdim != 3) {
        set_error("fdb_kernel_create: %s %s takes a scalar space or a vector space of value size 3 (cdim %d)",
                  f->name, mode_name[mode], d->cdim);
        return 1;
    }
    const int cdim = f->cdim ? f->cdim : (mode == MODE_DIAGONAL ? 1 : 0);
    if (cdim > 0 ? d->cdim != cdim : (cdim == 0 && (d->cdim < 1 || d->cdim > 3))) {
        set_error("fdb_kernel_create: %s %s takes %s (cdim %d)", f->name, mode_name[mode],
                  cdim == 1 ? "scalar spaces only"
                            : (cdim == 3 ? "a vector space of value size 3 only" : "value sizes 1..3"),
                  d->cdim);
        return 1;
    }
    if (d->affine_cells && !f->affine) {
        set_error("fdb_kernel_create: %s has no affine-cell variant (affine_cells must be 0)", f->name);
        return 1;
    }
    const bool transfer = f->launcher == LAUNCH_P_TRANSFER;
    const bool trace = f->launcher == LAUNCH_TRACE_TRANSFER;
    if (trace) {
        if (d->degree < 1 || d->degree > 2) {
            set_error("fdb_kernel_create_mixed: %s: trace degree %d not instantiated: the hybridised trace spaces of "
                      "k = 2, 3 (trace degrees 1, 2)", f->name, d->degree);
            return 1;
        }
        if (mode != MODE_ACTION) {
            set_error("fdb_kernel_create_mixed: %s is a transfer, a rank-1 map between CG1 and the trace space: it "
                      "has no rank-2 or diagonal form", f->name);
            return 1;
        }
        if (s2->degree != 1) {
            set_error("fdb_kernel_create_mixed: %s: the second space must be CG1, the vertex values (degree 1), got "
                      "degree %d", f->name, s2->degree);
            return 1;
        }
    }
    if (f->launcher == LAUNCH_SPECTRAL) {
        // the GLL rule in dof order: the points are the nodes (dof 0 at 0, dof 1 at 1), so B is the identity
        if (d->rank == 2) {
            set_error("fdb_kernel_create: %s has no rank-2 form: there is no assembled SEM matrix; use the action "
                      "and the diagonal", f->name);
            return 1;
        }
        if (d->nq != d->degree + 1) {
            set_error("fdb_kernel_create: %s needs the GLL rule at the nodes: nq == degree+1 (got nq=%d for degree "
                      "%d)", f->name, d->nq, d->degree);
            return 1;
        }
        if (d->nq >= 2 && (d->xq[0] != 0.0 || d->xq[1] != 1.0)) {
            set_error("fdb_kernel_create: %s needs the GLL rule in dof order: xq[0] == 0 and xq[1] == 1 exactly "
                      "(got %.17g, %.17g)", f->name, d->xq[0], d->xq[1]);
            return 1;
        }
        const int n = d->degree + 1;
        if (n <= FDB_MAX_1D)
            for (int q = 0; q < n; q++)
                for (int a = 0; a < n; a++)
                    if (d->B[q * n + a] != (q == a ? 1.0 : 0.0)) {
                        set_error("fdb_kernel_create: %s needs the collocated GLL element: B must be exactly the "
                                  "identity (B[%d][%d] = %.17g)", f->name, q, a, d->B[q * n + a]);
                        return 1;
                    }
    }
    if (transfer && s2->degree + 1 != d->nq) {
        set_error("fdb_kernel_create_mixed: %s: R (desc.B) has nq = q+1 rows, got nq=%d for the coarse degree %d",
                  f->name, d->nq, s2->degree);
        return 1;
    }
    if (!transfer && d->nq != d->degree + 1) {
        set_error("fdb_kernel_create: %s needs nq == degree+1 Gauss points per axis (got nq=%d for degree %d); "
                  "pin the rule with dx(degree=2*p)", f->name, d->nq, d->degree);
        return 1;
    }
    if (f->launcher == LAUNCH_HDIV && mode == MODE_MATRIX) {
        set_error("fdb_kernel_create: %s has no rank-2 form: there is no assembled mixed matrix; use the action and "
                  "the diagonal", f->name);
        return 1;
    }
    if (f->launcher == LAUNCH_HYBRID) {
        if (d->degree == 4) {
            set_error("fdb_kernel_create: %s: degree 4 is not built: its local flux mass matrix alone (240^2 doubles, "
                      "460 KB) exceeds the 227 KB of shared memory of an SM; degrees 2..3", f->name);
            return 1;
        }
        if (mode == MODE_DIAGONAL) {
            set_error("fdb_kernel_create: %s has no diagonal form: the trace matrix is assembled (rank 2)", f->name);
            return 1;
        }
        if (mode == MODE_MATRIX && d->form != FDB_FORM_MIXED_POISSON_HYBRID) {
            set_error("fdb_kernel_create: %s has no rank-2 form: it is the rank-1 reconstruction of (sigma, u); the "
                      "trace matrix is mixed_poisson_hybrid at rank 2", f->name);
            return 1;
        }
        if (d->scatter != FDB_SCATTER_ATOMIC) {
            set_error("fdb_kernel_create: %s takes atomic scatter only: every entry receives at most two cell "
                      "contributions, so the atomic sums are already bit-reproducible", f->name);
            return 1;
        }
    }
    // (a mixed residual has no matrix or diagonal, nor has its Jacobian: the mixed-form message comes first)
    if (f->space2 && mode != MODE_ACTION && f->launcher != LAUNCH_HDIV && f->launcher != LAUNCH_HYBRID) {
        set_error("fdb_kernel_create: %s is a mixed form, a rank-1 action only: it has no assembled matrix or "
                  "diagonal", f->name);
        return 1;
    }
    if (f->residual && mode != MODE_ACTION) {
        set_error("fdb_kernel_create: %s is the residual, a 1-form action only: its matrix and diagonal are those "
                  "of %s_jacobian", f->name, f->name);
        return 1;
    }
    if ((f->launcher == LAUNCH_DG_FACET || f->launcher == LAUNCH_DG_TRANSPORT) && mode == MODE_MATRIX) {
        set_error("fdb_kernel_create: %s has no rank-2 form: there is no assembled DG matrix (the facet terms couple "
                  "neighbouring cells outside the cell sparsity); use the action and the diagonal", f->name);
        return 1;
    }
    if (d->degree < f->min_degree || d->degree > f->max_degree[mode]) {
        set_error("fdb_kernel_create: %s %s: degree %d outside %d..%d", f->name, mode_name[mode], d->degree,
                  f->min_degree, f->max_degree[mode]);
        return 1;
    }
    if (f->integral == FDB_INTEGRAL_CELL && d->integral != FDB_INTEGRAL_CELL) {
        set_error("fdb_kernel_create: %s has cell integrals only", f->name);
        return 1;
    }
    if (f->integral == FDB_INTEGRAL_EXTERIOR_FACET && d->integral != FDB_INTEGRAL_EXTERIOR_FACET) {
        set_error("fdb_kernel_create: %s has exterior-facet integrals only (integral %d: %s)", f->name, d->integral,
                  d->integral == FDB_INTEGRAL_CELL ? "a cell integral"
                  : (d->integral == FDB_INTEGRAL_INTERIOR_FACET ? "interior facets are not supported" : "unknown"));
        return 1;
    }
    if (f->integral == FDB_INTEGRAL_INTERIOR_FACET && d->integral != FDB_INTEGRAL_INTERIOR_FACET) {
        set_error("fdb_kernel_create: %s has interior-facet integrals only (integral %d)", f->name, d->integral);
        return 1;
    }
    if (f->integral < 0 && (d->integral < FDB_INTEGRAL_CELL || d->integral > FDB_INTEGRAL_INTERIOR_FACET)) {
        set_error("fdb_kernel_create: %s takes a cell, exterior-facet or interior-facet integral (integral %d)",
                  f->name, d->integral);
        return 1;
    }
    if (f->launcher == LAUNCH_DG_TRANSPORT) {
        // the form is stated on the collocated GL element: u at Gauss point q is the dof u[q]
        for (int q = 0; q < d->nq; q++)
            for (int a = 0; a <= d->degree; a++)
                if (d->B[q * (d->degree + 1) + a] != (q == a ? 1.0 : 0.0)) {
                    set_error("fdb_kernel_create: %s needs the collocated Gauss-Legendre element (B must be the "
                              "identity: B[%d][%d] = %g)", f->name, q, a, d->B[q * (d->degree + 1) + a]);
                    return 1;
                }
    }
    if (f->integral != FDB_INTEGRAL_CELL && d->cell == FDB_CELL_HEX_EXTRUDED && (!d->offset0 || !d->offset1)) {
        set_error("fdb_kernel_create: %s on extruded cells needs the layer offsets offset0/offset1", f->name);
        return 1;
    }
    if (d->rank != 1 && d->rank != 2) {
        set_error("fdb_kernel_create: rank must be 1 or 2");
        return 1;
    }
    // (a transfer and the Schur complement of mixed Poisson read no coordinates: offset1 is not used)
    const bool no_coords = transfer || trace || d->form == FDB_FORM_MIXED_POISSON_SCHUR;
    if (d->cell == FDB_CELL_HEX_EXTRUDED && (!d->offset0 || (!d->offset1 && !no_coords))) {
        set_error("fdb_kernel_create: extruded cells need offset0/offset1");
        return 1;
    }
    // the second space: CG_{p-1} with p^3 dofs per cell (Stokes' pressure)
    if (f->space2 && f->space2_degree == SPACE2_PRESSURE && s2->degree != d->degree - 1) {
        set_error("fdb_kernel_create_mixed: %s of degree %d needs a second space of degree %d, got %d", f->name,
                  d->degree, d->degree - 1, s2->degree);
        return 1;
    }
    // or a coarser CG_q of an instantiated pair, with exact unit endpoint rows in P and R (GLL nodes at both ends)
    if (f->space2_degree == SPACE2_COARSER) {
        if (!p_transfer_pair(d->degree, s2->degree)) {
            set_error("fdb_kernel_create_mixed: %s: degree pair (fine %d, coarse %d) not instantiated: (2, 1), "
                      "(3, 1), (3, 2)", f->name, d->degree, s2->degree);
            return 1;
        }
        const int nf = d->degree + 1, nc = s2->degree + 1;
        for (int e = 0; e < 2; e++) {
            for (int a = 0; a < nc; a++)
                if (s2->B[e * nc + a] != (a == e ? 1.0 : 0.0)) {
                    set_error("fdb_kernel_create_mixed: %s needs GLL elements: row %d of P (space2.B) must be the "
                              "exact unit vector e_%d (P[%d][%d] = %.17g); a Gauss-Legendre (DQ) element has no "
                              "nodes at the ends", f->name, e, e, e, a, s2->B[e * nc + a]);
                    return 1;
                }
            for (int i = 0; i < nf; i++)
                if (d->B[e * nf + i] != (i == e ? 1.0 : 0.0)) {
                    set_error("fdb_kernel_create_mixed: %s needs GLL elements: row %d of R (desc.B) must be the "
                              "exact unit vector e_%d (R[%d][%d] = %.17g); a Gauss-Legendre (DQ) element has no "
                              "nodes at the ends", f->name, e, e, e, i, d->B[e * nf + i]);
                    return 1;
                }
        }
    }
    if (f->space2 && d->cell == FDB_CELL_HEX_EXTRUDED && !s2->offset) {
        set_error("fdb_kernel_create_mixed: %s on extruded cells needs the layer offsets of the second map "
                  "(fdb_space2_desc.offset)", f->name);
        return 1;
    }
    fdb_kernel_s *k = new fdb_kernel_s;
    k->desc = *d;
    k->hex = f;
    k->n1d = d->degree + 1;
    // an interior-facet entry reads both cells: 2 (p+1)^3 dofs and 16 vertices
    const int sides = d->integral == FDB_INTEGRAL_INTERIOR_FACET ? 2 : 1;
    k->arity = sides * k->n1d * k->n1d * k->n1d;
    if (f->launcher == LAUNCH_HDIV) k->arity = 3 * d->degree * d->degree * (d->degree + 1);    // NCF_k
    // the hybrid forms: offset0 holds the trace map's 6k^2 layer offsets, then the NCF map's 3k^2(k+1)
    if (f->launcher == LAUNCH_HYBRID) k->arity = 6 * d->degree * d->degree + 3 * d->degree * d->degree * (d->degree + 1);
    if (trace) k->arity = 6 * k->n1d * k->n1d;                                      // the trace map: 6k^2
    const int arity1 = sides * 8;
    memset(k->h_off0, 0, sizeof(k->h_off0));
    memset(k->h_off1, 0, sizeof(k->h_off1));
    if (d->offset0) memcpy(k->h_off0, d->offset0, sizeof(fdb_int) * k->arity);
    if (d->offset1) memcpy(k->h_off1, d->offset1, sizeof(fdb_int) * arity1);
    k->desc.offset0 = k->h_off0;
    k->desc.offset1 = k->h_off1;
    // the second space's map: (degree2 + 1)^3 dofs per cell
    const int arity2 = f->space2 ? (s2->degree + 1) * (s2->degree + 1) * (s2->degree + 1) : 0;
    memset(k->h_off2, 0, sizeof(k->h_off2));
    memset(k->B2, 0, sizeof(k->B2));
    if (f->space2) {
        if (s2->offset) memcpy(k->h_off2, s2->offset, sizeof(fdb_int) * arity2);
        memcpy(k->B2, s2->B, sizeof(k->B2));
    }
    if (!transfer && !trace && collocated_derivative(k->n1d, d->B, d->D, k->Dt)) {
        set_error("fdb_kernel_create: basis table B is singular");
        delete k;
        return 1;
    }
    memset(k->Bend, 0, sizeof(k->Bend));
    if (f->launcher == LAUNCH_DG_FACET || f->launcher == LAUNCH_DG_TRANSPORT) endpoint_tables(k->n1d, d->B, d->xq, k->Bend);
    FDB_CUDA(cudaMalloc(&k->d_off0, sizeof(fdb_int) * k->arity));
    FDB_CUDA(cudaMalloc(&k->d_off1, sizeof(fdb_int) * arity1));
    FDB_CUDA(cudaMemcpyAsync(k->d_off0, k->h_off0, sizeof(fdb_int) * k->arity,
                             cudaMemcpyHostToDevice, ctx().stream));
    FDB_CUDA(cudaMemcpyAsync(k->d_off1, k->h_off1, sizeof(fdb_int) * arity1, cudaMemcpyHostToDevice,
                             ctx().stream));
    if (f->space2) {
        FDB_CUDA(cudaMalloc(&k->d_off2, sizeof(fdb_int) * arity2));
        FDB_CUDA(cudaMemcpyAsync(k->d_off2, k->h_off2, sizeof(fdb_int) * arity2, cudaMemcpyHostToDevice,
                                 ctx().stream));
    }
    FDB_CUDA(cudaStreamSynchronize(ctx().stream));
    *out = k;
    return 0;
}

// the colouring plan of the call's map m (arity k->arity), rebuilt when the map, its generation or the range
// changes.  It covers columns [0, end): the map is copied to the host if needed
static int colouring_for(fdb_kernel_s *k, const fdb_call_args *a, int m, int arity = 0)
{
    if (!arity) arity = k->arity;
    if (k->colour_map_key == (const void *)a->maps[m] && k->colour_map_gen == map_ver(a, m) &&
        k->colour_end == a->end)
        return 0;
    std::vector<fdb_int> hmap;
    const fdb_int *src = a->maps[m];
    if (a->location == FDB_LOC_DEVICE) {
        hmap.resize((size_t)a->end * arity);
        FDB_CUDA(cudaMemcpy(hmap.data(), a->maps[m], sizeof(fdb_int) * hmap.size(), cudaMemcpyDeviceToHost));
        src = hmap.data();
    }
    if (build_colouring(k, src, a->end, arity)) return 1;
    k->colour_map_key = (const void *)a->maps[m];
    k->colour_map_gen = map_ver(a, m);
    k->colour_end = a->end;
    return 0;
}

// the p-multigrid transfers: args and maps in first-use order (include/fdb200.h), device mode only.  A coloured
// restriction is coloured on the fine map: two cells that share a coarse node share a fine node too
static int p_transfer_call(fdb_kernel_s *k, const fdb_call_args *a, int nlay)
{
    const int form = k->desc.form;
    const fdb_hex_form *f = k->hex;
    const int want = form == FDB_FORM_P_RESTRICT ? 3 : 2;
    if (a->nargs != want || a->nmaps != 2 || a->location != FDB_LOC_DEVICE) {
        set_error("fdb_kernel_call: %s expects %d device args (%s, %s) and 2 maps (%s), got %d/%d", f->name, want,
                  form == FDB_FORM_P_PROLONG ? "fine" : "coarse", f->space2,
                  form == FDB_FORM_P_PROLONG ? "fine map, coarse map" : "coarse map, fine map", a->nargs, a->nmaps);
        return 1;
    }
    const int fm = form == FDB_FORM_P_PROLONG ? 0 : 1;      // the fine map's slot
    if (form == FDB_FORM_P_RESTRICT && k->desc.scatter == FDB_SCATTER_COLOURED) {
        if (a->start != 0) {
            set_error("fdb_kernel_call: coloured scatter needs start == 0");
            return 1;
        }
        if (colouring_for(k, a, fm)) return 1;
    }
    return fdb_launch_p_transfer(k, a->start, a->end, nlay, a->subset, (double *)a->args[0],
                                 (const double *)a->args[1],
                                 form == FDB_FORM_P_RESTRICT ? (const double *)a->args[2] : nullptr,
                                 a->maps[fm], a->maps[1 - fm]);
}

// the GTMG trace transfers: args and maps in first-use order (include/fdb200.h), device mode only.  A coloured
// restriction is coloured on the CG1 map (8 vertices per cell): cells that share a vertex must not run together
static int trace_transfer_call(fdb_kernel_s *k, const fdb_call_args *a, int nlay)
{
    const bool prolong = k->desc.form == FDB_FORM_TRACE_PROLONG;
    const fdb_hex_form *f = k->hex;
    const int want = prolong ? 2 : 3;
    if (a->location != FDB_LOC_DEVICE) {
        set_error("fdb_kernel_call: %s takes device-resident Dats only (no host-pointer mode)", f->name);
        return 1;
    }
    if (a->nargs != want || a->nmaps != 2) {
        set_error("fdb_kernel_call: %s expects %d device args (%s) and 2 maps (%s), got %d/%d", f->name, want,
                  prolong ? "lambda, c" : "c, lambda, w", prolong ? "trace map, CG1 map" : "CG1 map, trace map",
                  a->nargs, a->nmaps);
        return 1;
    }
    const int tm = prolong ? 0 : 1;      // the trace map's slot
    if (!prolong && k->desc.scatter == FDB_SCATTER_COLOURED) {
        if (a->start != 0) {
            set_error("fdb_kernel_call: coloured scatter needs start == 0");
            return 1;
        }
        if (colouring_for(k, a, 1 - tm, 8)) return 1;
    }
    return fdb_launch_trace_transfer(k, a->start, a->end, nlay, a->subset, (double *)a->args[0],
                                     (const double *)a->args[1], prolong ? nullptr : (const double *)a->args[2],
                                     a->maps[tm], a->maps[1 - tm]);
}

// mixed Poisson (FDB_FORM_MIXED_POISSON[_SCHUR]): args and maps as include/fdb200.h lists them, device mode only.
// The flux scatters (the action, the diagonal of alpha M and the Schur form's B^T pass) are coloured on the NCF map
static int hdiv_call(fdb_kernel_s *k, const fdb_call_args *a, int nlay)
{
    const fdb_hex_form *f = k->hex;
    const bool schur = k->desc.form == FDB_FORM_MIXED_POISSON_SCHUR;
    const int mode = hex_mode(&k->desc);
    static const char *const sig[2][2] = {{"y_sigma, coords, sigma, y_u, u", "d, coords"}, {"y_u, u, w, t", "d, w"}};
    static const char *const mapsig[2][2] = {{"NCF map, coord map, DQ map", "NCF map, coord map"},
                                             {"DQ map, NCF map", "DQ map, NCF map"}};
    const int m = mode == MODE_ACTION ? 0 : 1;
    const int want = schur ? (m ? 2 : 4) : (m ? 2 : 5);
    const int want_maps = !schur && !m ? 3 : 2;
    if (a->location != FDB_LOC_DEVICE) {
        set_error("fdb_kernel_call: %s takes device-resident Dats only (no host-pointer mode)", f->name);
        return 1;
    }
    if (a->nargs != want || a->nmaps != want_maps) {
        set_error("fdb_kernel_call: %s %s expects %d device args (%s) and %d maps (%s), got %d/%d", f->name,
                  mode_name[mode], want, sig[schur][m], want_maps, mapsig[schur][m], a->nargs, a->nmaps);
        return 1;
    }
    if (k->desc.scatter == FDB_SCATTER_COLOURED && !(schur && m)) {
        if (a->start != 0) {
            set_error("fdb_kernel_call: coloured scatter needs start == 0");
            return 1;
        }
        if (colouring_for(k, a, schur ? 1 : 0)) return 1;
    }
    return fdb_launch_hdiv(k, a->start, a->end, nlay, a->subset, a->args, a->maps);
}

// the hybridised mixed Poisson forms (FDB_FORM_MIXED_POISSON_HYBRID / _RECONSTRUCT): args and maps as include/fdb200.h
// lists them, device mode only, atomic scatter
static int hybrid_call(fdb_kernel_s *k, const fdb_call_args *a, int nlay)
{
    const fdb_hex_form *f = k->hex;
    const int mode = hex_mode(&k->desc);
    const bool reconstruct = k->desc.form == FDB_FORM_MIXED_POISSON_RECONSTRUCT;
    const char *sig = mode == MODE_MATRIX ? "H mat, coords"
                      : (reconstruct ? "y_sigma, coords, lambda, f_sigma, w, y_u, f_u" : "r, coords, f_sigma, w, f_u");
    const char *mapsig = mode == MODE_MATRIX ? "trace map, coord map"
                         : (reconstruct ? "NCF map, coord map, trace map, DQ map"
                                        : "trace map, coord map, NCF map, DQ map");
    const int want = mode == MODE_MATRIX ? 2 : (reconstruct ? 7 : 5);
    const int want_maps = mode == MODE_MATRIX ? 2 : 4;
    if (a->location != FDB_LOC_DEVICE) {
        set_error("fdb_kernel_call: %s takes device-resident Dats only (no host-pointer mode)", f->name);
        return 1;
    }
    if (a->nargs != want || a->nmaps != want_maps) {
        set_error("fdb_kernel_call: %s %s expects %d device args (%s) and %d maps (%s), got %d/%d", f->name,
                  mode_name[mode], want, sig, want_maps, mapsig, a->nargs, a->nmaps);
        return 1;
    }
    return fdb_launch_hybrid(k, a->start, a->end, nlay, a->subset, a->args, a->maps);
}

extern "C" {

int fdb_kernel_create(const fdb_kernel_desc *d, fdb_kernel_t *out)
{
    return kernel_create(d, nullptr, out);
}

int fdb_kernel_create_mixed(const fdb_kernel_desc *d, const fdb_space2_desc *s2, fdb_kernel_t *out)
{
    if (require_init()) return 1;
    if (!d || !s2 || !out) {
        set_error("fdb_kernel_create_mixed: NULL argument");
        return 1;
    }
    for (const fdb_hex_form &row : hex_forms)
        if (row.form == d->form && row.space2) return kernel_create(d, s2, out);
    set_error("fdb_kernel_create_mixed: form %d is not a form on two spaces: create it with fdb_kernel_create",
              d->form);
    return 1;
}

int fdb_kernel_destroy(fdb_kernel_t k)
{
    if (!k) return 0;
    if (ctx().ready) cudaStreamSynchronize(ctx().stream);
    if (k->jit) fdb_jit_destroy(k->jit);
    if (ctx().ready) {
        if (k->d_off0) cudaFree(k->d_off0);
        if (k->d_off1) cudaFree(k->d_off1);
        if (k->d_off2) cudaFree(k->d_off2);
        if (k->d_colour_cols) cudaFree(k->d_colour_cols);
        if (k->d_bdb_table) cudaFree(k->d_bdb_table);
    }
    delete k;
    return 0;
}

int fdb_kernel_call(fdb_kernel_t k, const fdb_call_args *a)
{
    if (require_init()) return 1;
    if (!k || !a) {
        set_error("fdb_kernel_call: NULL argument");
        return 1;
    }
    fdb_mirror_new_epoch();
    if (k->jit) return fdb_jit_call(k, a);      // generated wrapper (wrapper_jit.cu)
    if (k->desc.form == FDB_FORM_DG_ADVECTION) {
        // args = [out (INC), coords, q, u, consts (HOST double[2] {dtc, q_in}), facet numbers]
        // maps = [DQ1 (facet-)node map, CG1 (facet-)node map]
        const bool facets = k->desc.integral != FDB_INTEGRAL_CELL;
        const bool fused = k->desc.integral == FDB_INTEGRAL_FUSED;
        const int want = fused ? 7 : (facets ? 6 : 5);
        if (a->nargs != want || a->nmaps != 2) {
            set_error("fdb_kernel_call: DG advection expects %d args and 2 maps", want);
            return 1;
        }
        if (a->location != FDB_LOC_DEVICE) {
            set_error("fdb_kernel_call: DG advection kernels take device-resident Dats");
            return 1;
        }
        return fdb_launch_dg_advection(k, a->start, a->end, a->subset, (double *)a->args[0],
                                       (const double *)a->args[1], (const double *)a->args[2],
                                       (const double *)a->args[3], (const double *)a->args[4],
                                       facets ? (const unsigned *)a->args[5] : nullptr, a->maps[0],
                                       a->maps[1], fused ? (const fdb_int *)a->args[6] : nullptr);
    }
    if (k->desc.cell == FDB_CELL_TRIANGLE) {
        // rank 1: args = [y, coords, x]; rank 2: args = [mat, coords]; maps[0] = cell->vertex map
        // (V and the P1 coordinate space share it; a second identical map is accepted)
        const int want = k->desc.rank == 1 ? 3 : 2;
        if (a->nargs != want || a->nmaps < 1 || a->location != FDB_LOC_DEVICE) {
            set_error("fdb_kernel_call: P1 triangle kernel expects %d device args and 1-2 maps", want);
            return 1;
        }
        if (k->desc.rank == 1)
            return fdb_launch_tri_p1(k, a->start, a->end, a->subset, (double *)a->args[0],
                                     (const double *)a->args[1], (const double *)a->args[2], a->maps[0],
                                     nullptr);
        return fdb_launch_tri_p1(k, a->start, a->end, a->subset, nullptr, (const double *)a->args[1],
                                 nullptr, a->maps[0], (fdb_mat_t)a->args[0]);
    }
    const bool extruded = k->desc.cell == FDB_CELL_HEX_EXTRUDED;
    if (extruded && !a->layers) {
        set_error("fdb_kernel_call: extruded kernel called without layers");
        return 1;
    }
    if (a->end < a->start) {
        set_error("fdb_kernel_call: end < start");
        return 1;
    }
    const int nlay = extruded ? (a->layers[1] - a->layers[0] - 1) : 1;
    if (extruded && a->layers[0] != 0) {
        set_error("fdb_kernel_call: nonzero bottom layer not supported");
        return 1;
    }
    if ((long long)(a->end - a->start) * nlay >= (1ll << 31) - 64) {
        set_error("fdb_kernel_call: iteration set too large for IntType");
        return 1;
    }
    // args = [y (INC), coords, x] (action), [Mat handle (INC), coords] (matrix: the reference passes the
    // PETSc Mat handle in the same slot, pyop2/types/mat.py:621-623) or [d (INC), coords] (diagonal), then
    // the form's trailing coefficient; maps = [V map, coord map].  A form on two spaces (Stokes) has the
    // output and input of the second space after x and a third map: [y, coords, x, y2, x2], [V map, coord
    // map, second map]; with a trailing coefficient as well (the Navier-Stokes Jacobian's u) the coefficient
    // comes last: [y, coords, x, y2, x2, coef]; a third field on the second map (Boussinesq's temperature) comes
    // after the second space's arguments, and its coefficients (several: u0, T0) last: [y, coords, x, y2, x2, y3,
    // x3, coef...]
    // an exterior-facet form (boundary_mass): the trailing argument is the uint32 local facet number of each
    // entry, [y, coords, x, facet] / [mat, coords, facet] / [d, coords, facet]; an interior-facet form
    // (interior_penalty): the two local facet numbers ('+', '-') of each entry, [y, coords, x, facets]; dg_transport
    // reads b before them: [y, coords, x, b], [d, coords, b] on cells, [y, coords, x, b, facets], [d, coords, b,
    // facets] on facets
    const fdb_hex_form *f = k->hex;
    if (f->launcher == LAUNCH_P_TRANSFER) return p_transfer_call(k, a, nlay);
    if (f->launcher == LAUNCH_HDIV) return hdiv_call(k, a, nlay);
    if (f->launcher == LAUNCH_HYBRID) return hybrid_call(k, a, nlay);
    if (f->launcher == LAUNCH_TRACE_TRANSFER) return trace_transfer_call(k, a, nlay);
    const int mode = hex_mode(&k->desc);
    const bool transport_facets = f->launcher == LAUNCH_DG_TRANSPORT && k->desc.integral != FDB_INTEGRAL_CELL;
    if (f->integral != FDB_INTEGRAL_CELL && a->location != FDB_LOC_DEVICE) {
        set_error("fdb_kernel_call: %s takes device-resident Dats only (no host-pointer mode for facet integrals)",
                  f->name);
        return 1;
    }
    const int ncoef = f->coef ? (f->ncoef ? f->ncoef : 1) : 0;
    const int want = (mode == MODE_ACTION ? 3 : 2) + ncoef + (f->space2 ? 2 : 0) + (f->field3 ? 2 : 0) +
                     (transport_facets ? 1 : 0);
    const int want_maps = f->space2 ? 3 : 2;
    const bool device_only = mode == MODE_DIAGONAL || f->space2 || f->integral != FDB_INTEGRAL_CELL;
    if (f->launcher == LAUNCH_SPECTRAL && a->location != FDB_LOC_DEVICE) {
        set_error("fdb_kernel_call: %s takes device-resident Dats only (no host-pointer mode)", f->name);
        return 1;
    }
    if (a->nargs != want || a->nmaps != want_maps || (device_only && a->location != FDB_LOC_DEVICE)) {
        static const char *const args[] = {"y, coords, x", "mat, coords", "d, coords"};
        set_error("fdb_kernel_call: %s %s expects %d %sargs (%s%s%s%s%s%s%s) and %d maps, got %d/%d", f->name,
                  mode_name[mode], want, device_only ? "device " : "", args[mode], f->space2 ? ", " : "",
                  f->space2 ? f->space2 : "", f->field3 ? ", " : "", f->field3 ? f->field3 : "", f->coef ? ", " : "",
                  transport_facets ? "b, facets" : (f->coef ? f->coef : ""), want_maps, a->nargs,
                  a->nmaps);
        return 1;
    }
    const fdb_mat_t mat = mode == MODE_MATRIX ? (fdb_mat_t)a->args[0] : nullptr;
    if (mat) {
        int mat_bs = 1;
        fdb_mat_block_size(mat, &mat_bs);
        if (mat_bs != k->desc.cdim) {
            set_error("fdb_kernel_call: Mat block size %d != value size %d of the argument space", mat_bs,
                      k->desc.cdim);
            return 1;
        }
        if (k->desc.scatter != FDB_SCATTER_ATOMIC) {
            set_error("fdb_kernel_call: coloured scatter is not implemented for matrices");
            return 1;
        }
    }
    if (f->coef && f->coef_cdim != k->desc.cdim && a->location == FDB_LOC_HOST && a->arg_bytes && mode != MODE_DIAGONAL) {
        // a coefficient with another value size than the argument space (advection-diffusion's b): host mode
        // mirrors it by its byte size, which must cover every node that x (action) or the Mat's rows (matrix)
        // cover.  Device mode has no sizes to check; op2.Parloop checks the Dat's value size there.
        size_t nodes;
        if (mat) {
            fdb_int rows = 0;
            fdb_mat_rows(mat, &rows);
            nodes = (size_t)rows;
        } else {
            nodes = a->arg_bytes[2] / (sizeof(double) * k->desc.cdim);
        }
        if (a->arg_bytes[want - 1] < nodes * f->coef_cdim * sizeof(double)) {
            set_error("fdb_kernel_call: %s %s: %s has %d values per node, %zu bytes are too few for %zu nodes",
                      f->name, mode_name[mode], f->coef, f->coef_cdim, a->arg_bytes[want - 1], nodes);
            return 1;
        }
    }
    // the pipelined host action moves x and y only and runs the constant-coefficient kernels: the
    // coefficient, nonlinear and elasticity-kernel forms take the monolithic path
    if (f->launcher == LAUNCH_HELMHOLTZ && mode == MODE_ACTION && a->location == FDB_LOC_HOST && a->arg_versions &&
        a->arg_bytes && a->map_bytes && a->writeback && a->output_is_zero && !a->subset && extruded &&
        k->desc.scatter == FDB_SCATTER_ATOMIC) {
        int rc = pipelined_host_action(k, a, nlay);
        if (rc >= 0) return rc;      // -1: not applicable, fall through to the monolithic path
    }
    void *dargs[9];
    const fdb_int *dmaps[3];
    const fdb_int *dsubset;
    if (device_pointers(a, mat != nullptr, dargs, dmaps, &dsubset)) return 1;
    const double *coords = (const double *)dargs[1];
    const double *coef = f->coef ? (const double *)dargs[want - ncoef] : nullptr;
    // dg_transport: b, and on facets the local facet numbers after it
    const double *vel = f->launcher == LAUNCH_DG_TRANSPORT ? (const double *)dargs[mode == MODE_ACTION ? 3 : 2] : nullptr;
    const unsigned *tfacets = transport_facets ? (const unsigned *)dargs[want - 1] : nullptr;
    double *out = mat ? nullptr : (double *)dargs[0];     // the action's y or the diagonal
    if (mode != MODE_ACTION) {
        switch (f->launcher) {
        case LAUNCH_HELMHOLTZ:
            if (mat && k->desc.cdim > 1) {
                // vector-valued space: the element tensor of the Helmholtz family is A_scalar (x) I_cdim
                // (off-diagonal component blocks vanish identically), so the scalar kernel assembles into
                // a scalar view of the blocked pattern, which is then added to the block diagonals
                fdb_mat_t view = nullptr;
                if (fdb_mat_scalar_view_begin(mat, &view)) return 1;
                int rc = fdb_launch_helmholtz_matrix(k, a->start, a->end, nlay, dsubset, view, coords, dmaps[0],
                                                     dmaps[1], nullptr);
                int rc2 = fdb_mat_scalar_view_end(mat, view);
                return rc ? rc : rc2;
            }
            return fdb_launch_helmholtz_matrix(k, a->start, a->end, nlay, dsubset, mat, coords, dmaps[0], dmaps[1],
                                               out);
        case LAUNCH_HELMHOLTZ_COEF:
            return fdb_launch_helmholtz_coef_matrix(k, a->start, a->end, nlay, dsubset, mat, coords, coef, dmaps[0],
                                                    dmaps[1], out);
        case LAUNCH_BOUNDARY:
            return fdb_launch_boundary_mass(k, a->start, a->end, nlay, dsubset, mat, out, coords, nullptr,
                                            (const unsigned *)coef, dmaps[0], dmaps[1]);
        case LAUNCH_DG_FACET:
            return fdb_launch_dg_facet(k, a->start, a->end, nlay, dsubset, out, coords, nullptr,
                                       (const unsigned *)coef, dmaps[0], dmaps[1]);
        case LAUNCH_DG_TRANSPORT:
            return fdb_launch_dg_transport(k, a->start, a->end, nlay, dsubset, out, coords, nullptr, vel, tfacets,
                                           dmaps[0], dmaps[1]);
        case LAUNCH_SPECTRAL:
            // the diagonal's scatter is coloured like the action's
            if (k->desc.scatter == FDB_SCATTER_COLOURED) {
                if (a->start != 0) {
                    set_error("fdb_kernel_call: coloured scatter needs start == 0");
                    return 1;
                }
                if (colouring_for(k, a, 0)) return 1;
            }
            return fdb_launch_spectral_helmholtz(k, a->start, a->end, nlay, dsubset, out, coords, nullptr, coef,
                                                 dmaps[0], dmaps[1]);
        default:
            return fdb_launch_elasticity_matrix(k, a->start, a->end, nlay, dsubset, mat, coords, coef, dmaps[0],
                                                dmaps[1], out);
        }
    }
    // (the dg_transport cell term needs no colours: a DQ cell owns its dofs)
    if (k->desc.scatter == FDB_SCATTER_COLOURED && !(f->launcher == LAUNCH_DG_TRANSPORT && !transport_facets) &&
        colouring_for(k, a, 0))
        return 1;
    if (k->desc.scatter == FDB_SCATTER_COLOURED && a->start != 0) {
        set_error("fdb_kernel_call: coloured scatter needs start == 0");
        return 1;
    }
    // (a residual's coefficient is NULL: its u is x, see action_hex.cu and elasticity_hex.cu)
    const double *x = (const double *)dargs[2];
    int rc;
    switch (f->launcher) {
    case LAUNCH_HELMHOLTZ:
        rc = fdb_launch_helmholtz_action(k, a->start, a->end, nlay, dsubset, out, coords, x, dmaps[0], dmaps[1]);
        break;
    case LAUNCH_HELMHOLTZ_COEF:
        rc = fdb_launch_helmholtz_coef_action(k, a->start, a->end, nlay, dsubset, out, coords, x, coef, dmaps[0],
                                              dmaps[1]);
        break;
    case LAUNCH_ELASTICITY:
        rc = fdb_launch_elasticity_action(k, a->start, a->end, nlay, dsubset, out, coords, x, coef, dmaps[0],
                                          dmaps[1]);
        break;
    case LAUNCH_BOUNDARY:
        rc = fdb_launch_boundary_mass(k, a->start, a->end, nlay, dsubset, nullptr, out, coords, x,
                                      (const unsigned *)coef, dmaps[0], dmaps[1]);
        break;
    case LAUNCH_DG_FACET:
        rc = fdb_launch_dg_facet(k, a->start, a->end, nlay, dsubset, out, coords, x, (const unsigned *)coef,
                                 dmaps[0], dmaps[1]);
        break;
    case LAUNCH_DG_TRANSPORT:
        rc = fdb_launch_dg_transport(k, a->start, a->end, nlay, dsubset, out, coords, x, vel, tfacets, dmaps[0],
                                     dmaps[1]);
        break;
    case LAUNCH_SPECTRAL:
        rc = fdb_launch_spectral_helmholtz(k, a->start, a->end, nlay, dsubset, out, coords, x, coef, dmaps[0],
                                           dmaps[1]);
        break;
    default:
        rc = fdb_launch_stokes_action(k, a->start, a->end, nlay, dsubset, out, coords, x, (double *)dargs[3],
                                      (const double *)dargs[4], coef, dmaps[0], dmaps[1], dmaps[2],
                                      f->field3 ? (double *)dargs[5] : nullptr,
                                      f->field3 ? (const double *)dargs[6] : nullptr,
                                      ncoef > 1 ? (const double *)dargs[want - 1] : nullptr);
    }
    if (rc) return rc;
    if (a->location == FDB_LOC_HOST && a->writeback) {
        // the output mirror now differs from the host copy: write it back
        if (fdb_mirror_writeback(a->args[0])) return 1;
        if (a->arg_versions) fdb_mirror_set_version(a->args[0], a->arg_versions[0] + 1);
    }
    return 0;
}

}  // extern "C"
