// Matrix-free action of  alpha*inner(grad u, grad v)*dx + beta*inner(u, v)*dx
// on Q_p (x) P_p hexahedra (extruded or native), fp64, sm_90a.
//
// One launch = gather through the cell->node map + element kernel + scatter-add,
// i.e. the whole PyOP2 wrapper of SURVEY.md section 9.1 (reference
// pyop2/codegen/builder.py:80-128, 352-429, 730-812) fused with the TSFC kernel
// it calls (reference tsfc/kernel_interface/common.py:139-239).
//
// Thread mapping ("slab threads"): N = p+1 lanes cooperate on one cell, each
// lane owning one N x N slab of the N^3 tensor; a warp holds 32/N cells, which
// are CONSECUTIVE LAYERS of one column so that a warp-wide gather instruction
// walks a contiguous run of each dof column.  Two slab orientations are used:
//   layout Z: lane t owns index t along z, holds [x][y]   (gather / scatter)
//   layout Y: lane t owns index t along y, holds [x][z]   (quadrature points)
// Contractions along in-slab axes run in registers (N^2 x N FMAs against a
// constant-bank table); the two orientation changes go through a per-warp
// shared-memory tile with __syncwarp only -- no block-level barrier in the work
// loop.
//
// Data movement: a three-stage cp.async pipeline per warp (map rows -> indices
// and values -> compute) with chunks of columns handed out by an atomic counter;
// the quadrature (zeta) loop is rolled, with U / Vp kept column-rotated, so that
// the loop body fits the instruction cache and 168 registers (12 warps per SM at
// p = 3).  Template flags: MASS (beta != 0), ATOMIC vs coloured scatter, MATRIX
// (rank 2: columns of the element tensor as actions on unit vectors, also the
// diagonal), SLIM (p = 5: one staged map row per column, indices recomputed).
// DESIGN.md section 4.1 has the measurements behind each of these choices.
// helmholtz_coef_kernel is the same body (action_hex_body.cuh) with COEF set: a coefficient field
// kappa scales the stiffness term (FDB_FORM_HELMHOLTZ_COEF, DESIGN.md section 4.5).
// nonlinear_residual_kernel and nonlinear_jacobian_kernel are the same body with NL = 1 / 2: the
// residual and the exact Newton Jacobian of alpha*inner(D(u) grad u, grad v)*dx + beta*inner(u, v)*dx
// (FDB_FORM_NONLINEAR_DIFFUSION[_JACOBIAN], DESIGN.md section 4.6).
// advection_diffusion_kernel is the same body with ADV set: the velocity b (3 values per node) in three
// kappa buffers adds inner(dot(b, grad u), v)*dx (FDB_FORM_ADVECTION_DIFFUSION, DESIGN.md section 4.10).
//
// Arithmetic: the basis is first interpolated to the N Gauss points per axis
// (B (x) B (x) B), gradients are then taken with the collocated derivative
// matrix Dt = D B^{-1}; the transpose path mirrors it.  6 N^4 FMAs each way
// instead of 8 N^4 for the textbook form; identical in exact arithmetic.
// Geometry (trilinear Q1 coordinate field) is recomputed at every quadrature
// point, as TSFC does (reference tsfc/ufl_utils.py:41-85), from the 8 vertex
// coordinates: cofactor rows r_k of J, det = a.(b x c), and the flux in
// reference coordinates is  (alpha w / |det|) r_k . (sum_m r_m ghat_m).
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace {

template <int N>
struct HelmParams {
    double *y;
    const double *x;
    const double *coords;
    const int *map0;
    const int *map1;
    const int *collist;      // column indirection (subset / colour list) or NULL
    const int *off0;         // device, N^3 entries (zeros for non-extruded)
    const int *off1;         // device, 8 entries
    int ncols;               // number of columns to process
    int col0;                // first column (when collist == NULL)
    int nlay_items;          // layers to process per column
    int lay_first, lay_step; // layer = lay_first + lay_step * k
    unsigned nlay_rcp;       // floor(2^32 / nlay_items)
    int cdim;
    // matrix mode (rank 2): CSR destination; each unit computes one column j of
    // the element tensor as the action on the unit vector e_j
    const long long *rowptr;
    const int *colidx;
    double *vals;
    const int *row_lg;       // -1 = row dropped (Dirichlet), NULL = identity
    const int *col_lg;
    const unsigned short *rank_tab;   // within-row positions per (column, layer class, j, i) or NULL
    int nvar, nlay_total;
    int chunk;               // items per work chunk
    int ws_flags;            // warp-specialised kernel: timing probes (0 in production)
    int *counter;            // device work counter (zeroed before the launch)
    double alpha, beta;
    double B[N * N];         // B[q][a]
    double Dt[N * N];        // Dt[q][q']
    double DtR[N * N];       // DtR[q][j] = Dt[q][(j + q) % N]  (rolled zeta loop)
    double DB[N * N];        // DB[q][a] = sum_j Dt[q][j] B[j][a] = d phi_a / d x at point q (the collocated pair's product)
    double wq[N];
    double xq[N];
};

// FDB_FORM_HELMHOLTZ_COEF: the coefficient field kappa, gathered through map0 like x.  A derived
// struct, so that the parameter layout of the constant-coefficient kernels stays as it is.
template <int N>
struct HelmCoefParams : HelmParams<N> {
    const double *kappa;
};

// FDB_FORM_NONLINEAR_DIFFUSION[_JACOBIAN]: D(s) = dcoef[0] + dcoef[1] s + dcoef[2] s^2; the Jacobian
// passes the linearisation point u as kappa
template <int N>
struct HelmNlParams : HelmCoefParams<N> {
    double dcoef[3];
};

// the quadrature weight of the stiffness flux, times kappa at the point (COEF: s_kap[q])
template <bool COEF>
__device__ __forceinline__ double coef_weight(double w, const double *s_kap, int q)
{
    if constexpr (COEF) return w * s_kap[q];
    else return w;
}

// the same for every mode of the slab-thread body: NL == 1 (residual) scales by D(u_q), u_q = x at the
// point; NL == 2 (Jacobian) applies D and D' to the gradient instead and keeps w
template <bool COEF, int NL>
__device__ __forceinline__ double stiff_weight(double w, const double *s_kap, int q, double uq, const double *dcoef)
{
    if constexpr (NL == 1) return w * fma(fma(dcoef[2], uq, dcoef[1]), uq, dcoef[0]);
    else if constexpr (NL == 2) return w;
    else return coef_weight<COEF>(w, s_kap, q);
}

__device__ __forceinline__ double fast_rcp(double x)
{
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    // one third-order step r (1 + e + e^2), e = 1 - x r: |e| <= 2^-20 after MUFU.RCP64H -> 2^-60;
    // three dependent FMAs (two Newton steps are four)
    const double e = fma(-x, r, 1.0);
    const double t = fma(e, e, e);
    return fma(r, t, r);
}

// out[i][j] = sum_k M(i,k) in[k][j];  M(i,k) = T ? M[k*N+i] : M[i*N+k]
template <int N, bool T>
__device__ __forceinline__ void apply_first(const double *M, const double (&in)[N][N],
                                            double (&out)[N][N])
{
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < N; k++) s = fma(T ? M[k * N + i] : M[i * N + k], in[k][j], s);
            out[i][j] = s;
        }
}

// out[i][j] = sum_k M(j,k) in[i][k]
template <int N, bool T>
__device__ __forceinline__ void apply_second(const double *M, const double (&in)[N][N],
                                             double (&out)[N][N])
{
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < N; k++) s = fma(T ? M[k * N + j] : M[j * N + k], in[i][k], s);
            out[i][j] = s;
        }
}

// A field's dof values in a cell-strided buffer (this lane's layout-Z slots) to its values at the
// quadrature points (B (x) B (x) B, this lane's layout-Y slots), in place: the kappa interpolation of
// action_hex_body.cuh, for the second and third components of the advection velocity
template <int N>
__device__ __forceinline__ void to_points_in_place(const double *B, double *sk, bool valid, int t)
{
    double kz[N][N], kt[N][N];
#pragma unroll
    for (int x = 0; x < N; x++)
#pragma unroll
        for (int yy = 0; yy < N; yy++) kz[x][yy] = valid ? sk[(x * N + yy) * N + t] : 0.0;
    apply_first<N, false>(B, kz, kt);
    apply_second<N, false>(B, kt, kz);
#pragma unroll
    for (int x = 0; x < N; x++)
#pragma unroll
        for (int yy = 0; yy < N; yy++) sk[(x * N + yy) * N + t] = kz[x][yy];
    __syncwarp();
#pragma unroll
    for (int x = 0; x < N; x++)
#pragma unroll
        for (int z = 0; z < N; z++) kt[x][z] = sk[(x * N + t) * N + z];
    apply_second<N, false>(B, kt, kz);
#pragma unroll
    for (int x = 0; x < N; x++)
#pragma unroll
        for (int z = 0; z < N; z++) sk[(x * N + t) * N + z] = kz[x][z];
}

// Shared-memory tile used to re-orient slabs.  For N == 4 the (y, z) position
// is rotated by the cell's index in the warp so that both the layout-Z and the
// layout-Y access patterns touch all 32 banks exactly once per half-warp.
template <int N>
struct Tile {
    static constexpr int PAD = (N == 4) ? 0 : ((N * N * N) % 2 == 0 ? 2 : 1);
    static constexpr int STRIDE = N * N * N + PAD;
    double *base;
    int t, r, k[N], cwrot;
    __device__ __forceinline__ Tile(double *warp_smem, int cw, int t_) : t(t_)
    {
        base = warp_smem + cw * STRIDE;
        cwrot = cw;
        if (N == 4) {
            r = (t_ + cw) & 3;
#pragma unroll
            for (int j = 0; j < N; j++) k[j] = (j + cw) & 3;
        } else {
            r = t_;
#pragma unroll
            for (int j = 0; j < N; j++) k[j] = j;
        }
    }
    // lane t == z holds a[x][y]
    __device__ __forceinline__ void store_Z(const double (&a)[N][N]) const
    {
#pragma unroll
        for (int x = 0; x < N; x++)
#pragma unroll
            for (int y = 0; y < N; y++) base[(x * N + k[y]) * N + r] = a[x][y];
    }
    __device__ __forceinline__ void load_Z(double (&a)[N][N]) const
    {
#pragma unroll
        for (int x = 0; x < N; x++)
#pragma unroll
            for (int y = 0; y < N; y++) a[x][y] = base[(x * N + k[y]) * N + r];
    }
    // pointer to element (x = 0, lane's y, z) for a RUN-TIME z; (x, y, z) is N*N further per x
    __device__ __forceinline__ double *row_Y(int z) const
    {
        const int kz = (N == 4) ? ((z + cwrot) & 3) : z;
        return base + r * N + kz;
    }
    __device__ __forceinline__ double get_Y(int x, int z) const { return base[(x * N + r) * N + k[z]]; }
    __device__ __forceinline__ void put_Y(int x, int z, double v) const { base[(x * N + r) * N + k[z]] = v; }
    // lane t == y holds a[x][z]
    __device__ __forceinline__ void store_Y(const double (&a)[N][N]) const
    {
#pragma unroll
        for (int x = 0; x < N; x++)
#pragma unroll
            for (int z = 0; z < N; z++) base[(x * N + r) * N + k[z]] = a[x][z];
    }
    __device__ __forceinline__ void load_Y(double (&a)[N][N]) const
    {
#pragma unroll
        for (int x = 0; x < N; x++)
#pragma unroll
            for (int z = 0; z < N; z++) a[x][z] = base[(x * N + r) * N + k[z]];
    }
};

#ifndef FDB_WARPS
#define FDB_WARPS 4
#endif
// degree 3: the geometry coefficients that are needed once per zeta plane only (c2, c4, c5, c7 of the
// cell, A1 of the lane) are parked in shared memory: 30 registers less in the quadrature loop;
// -DFDB_NO_STASH builds without
#ifdef FDB_NO_STASH
constexpr bool OPT_STASH = false;
#else
constexpr bool OPT_STASH = true;
#endif
// warps per CTA: 4 everywhere except degree 5 (N = 6), whose per-warp staging is 38 KB:
// one CTA of 5 warps fills the 227 KB of shared memory better than one of 4
template <int N, bool SLIM = false, bool COEF = false>
struct WPC {
    // degree 5 (N = 6): 38 KB of staging per warp -> 5 warps; 27.5 KB when SLIM -> 8 warps
    // (255 registers x 256 threads = the whole register file).  The coefficient kernel stages
    // 10.4 KB more per warp at degree 5: 4 warps (5 when SLIM) fit the 227 KB.
    static constexpr int value = (N == 6) ? (COEF ? (SLIM ? 5 : 4) : (SLIM ? 8 : 5)) : FDB_WARPS;
};

__device__ __forceinline__ void cp_async8(void *smem, const void *gmem)
{
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(sa), "l"(gmem));
}
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem)
{
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int K>
__device__ __forceinline__ void cp_async_wait()
{
    asm volatile("cp.async.wait_group %0;" ::"n"(K) : "memory");
}

__device__ __forceinline__ void cp_async4(void *smem, const void *gmem)
{
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(sa), "l"(gmem));
}

// per-warp shared-memory footprint.  Cell strides are padded so that the
// 16 (64-bit) / 32 (32-bit) lanes of an access phase hit distinct banks.
// SLIM (used for p >= 4, where the staging buffers limit occupancy): no per-cell
// index buffer -- gather and scatter indices are recomputed from the staged map
// row -- and one staged row per distinct COLUMN of the warp (at most two when a
// column has at least 32/N layers) instead of one per cell, triple-buffered over
// the three items in flight (compute / value prefetch / row prefetch).
// COEF: one more cell-strided buffer for kappa, first its gathered dof values (layout Z), then,
// overwritten in place, its values at the quadrature points (layout Y: [qx][qy][qz] at qy = lane);
// NKAP such buffers (3 for the advection velocity b, one per component)
template <int N, bool SLIM = false, bool COEF = false, int NKAP = 1>
struct WarpSmem {
    static constexpr int CW = 32 / N;
    static constexpr int CWS = (32 % N == 0) ? CW : CW + 1;   // idle lanes get a scratch slot
    static constexpr int ND = N * N * N;
    static constexpr int US = (N == 4) ? ND + 4 : ((ND % 2) ? ND : ND + 1);   // cell stride
    static constexpr int CS = 26;                              // coord stride (24 used)
    static constexpr int TILE = CWS * Tile<N>::STRIDE;         // doubles
    static constexpr int UBUF = CWS * US;                      // doubles: gathered values (single buffer)
    static constexpr int COORD = CWS * CS;                     // doubles: vertex coordinates (single buffer)
#ifndef FDB_STASH_STRIDE
#define FDB_STASH_STRIDE 28
#endif
    static constexpr int GS = FDB_STASH_STRIDE;                // stash stride: c2 c4 c5 c7 (12) + A1 of 4 lanes (4 apart)
    static constexpr int STASH = (OPT_STASH && N == 4 && !SLIM) ? CWS * GS : 0;   // doubles
    static constexpr int KAPPA = COEF ? NKAP * CWS * US : 0;   // doubles: kappa (single buffer)
    static constexpr int IDX = SLIM ? 0 : 2 * CWS * US;        // ints: global dof index per local dof
    static constexpr int MAPRAW = SLIM ? 3 * 2 * US : CWS * US;   // ints: bottom-cell map row(s)
    static constexpr int VIDX = SLIM ? 3 * 2 * 8 : 2 * CWS * 8;   // ints: bottom-cell vertex row(s)
    static constexpr int BYTES =
        (((TILE + UBUF + COORD + STASH + KAPPA) * 8 + (IDX + MAPRAW + VIDX) * 4) + 15) / 16 * 16;
    static constexpr int CTA_BYTES = WPC<N, SLIM, COEF>::value * BYTES + ND * 4 + 32;
};

// One pipeline unit = (item, component): the cells a warp works on next.
struct Unit {
    int item;     // -1: none
    int comp;
    int ib;       // item-buffer index (advances when the item changes: mod 2, mod 3 if SLIM)
    int cur, end; // chunk bookkeeping (warp uniform)
    bool valid;   // per lane: this lane's cell exists
    int col, layer;
    int src;      // slot holding this column's staged map rows (leader cell, or 0/1 if SLIM)
    bool lead;    // this lane's cell copies the rows of its column
};

// AFFINE: the caller promises that every cell is a parallelepiped (fdb_kernel_desc.affine_cells):
// the trilinear terms of the coordinate field vanish, the Jacobian is constant per cell and the
// metric G = (alpha / |det|) K K^T (K = cofactor rows) is formed once per cell instead of at
// each of the N^3 quadrature points (DESIGN.md section 8b).
// COEF: alpha*inner(kappa*grad u, grad v)*dx + beta*inner(u, v)*dx with kappa in the argument space
// (FDB_FORM_HELMHOLTZ_COEF): kappa's dof values are gathered with x's indices, interpolated to the
// quadrature points once per cell and scale the stiffness flux (DESIGN.md section 4.5).
template <int N, bool MASS, bool ATOMIC, int MINB, bool MATRIX = false, bool SLIM = false, bool AFFINE = false>
__global__ void __launch_bounds__(WPC<N, SLIM>::value * 32, MINB)
helmholtz_action_kernel(const __grid_constant__ HelmParams<N> P)
{
    constexpr bool COEF = false, ADV = false;
    constexpr int NL = 0;
    [[maybe_unused]] const double *kappa = nullptr;
    [[maybe_unused]] const double *dcoef = nullptr;
#include "action_hex_body.cuh"
}

// FDB_FORM_HELMHOLTZ_COEF (action, element matrix, diagonal): the same body with COEF set
template <int N, bool MASS, bool ATOMIC, int MINB, bool MATRIX = false, bool SLIM = false>
__global__ void __launch_bounds__(WPC<N, SLIM, true>::value * 32, MINB)
helmholtz_coef_kernel(const __grid_constant__ HelmCoefParams<N> P)
{
    constexpr bool COEF = true, AFFINE = false, ADV = false;
    constexpr int NL = 0;
    const double *kappa = P.kappa;
    [[maybe_unused]] const double *dcoef = nullptr;
#include "action_hex_body.cuh"
}

// FDB_FORM_NONLINEAR_DIFFUSION (action only): the constant-coefficient layout, D(u_q) from the
// gathered values themselves
template <int N, bool MASS, bool ATOMIC, int MINB, bool SLIM = false>
__global__ void __launch_bounds__(WPC<N, SLIM>::value * 32, MINB)
nonlinear_residual_kernel(const __grid_constant__ HelmNlParams<N> P)
{
    constexpr bool COEF = false, MATRIX = false, AFFINE = false, ADV = false;
    constexpr int NL = 1;
    [[maybe_unused]] const double *kappa = nullptr;
    const double *dcoef = P.dcoef;
#include "action_hex_body.cuh"
}

// FDB_FORM_NONLINEAR_DIFFUSION_JACOBIAN (action, element matrix, diagonal): the coefficient layout,
// u in the kappa buffer
template <int N, bool MASS, bool ATOMIC, int MINB, bool MATRIX = false, bool SLIM = false>
__global__ void __launch_bounds__(WPC<N, SLIM, true>::value * 32, MINB)
nonlinear_jacobian_kernel(const __grid_constant__ HelmNlParams<N> P)
{
    constexpr bool COEF = true, AFFINE = false, ADV = false;
    constexpr int NL = 2;
    const double *kappa = P.kappa;
    const double *dcoef = P.dcoef;
#include "action_hex_body.cuh"
}

// FDB_FORM_ADVECTION_DIFFUSION (action, element matrix, diagonal): the coefficient layout with three
// kappa buffers, b's components, reused across the N^3 units of a cell in matrix mode
template <int N, bool MASS, bool ATOMIC, int MINB, bool MATRIX = false>
__global__ void __launch_bounds__(WPC<N, false, true>::value * 32, MINB)
advection_diffusion_kernel(const __grid_constant__ HelmCoefParams<N> P)
{
    constexpr bool COEF = true, AFFINE = false, SLIM = false, ADV = true;
    constexpr int NL = 0;
    const double *kappa = P.kappa;   // b, 3 values per node
    [[maybe_unused]] const double *dcoef = nullptr;
#include "action_hex_body.cuh"
}

#include "action_hex_ws.cuh"

template <int N, bool MASS, bool ATOMIC, int MINB, bool MATRIX = false, bool SLIM = false, bool AFFINE = false,
          bool COEF = false, int NL = 0, bool ADV = false>
int launch_one(int grid_cap_per_sm, cudaStream_t st, HelmNlParams<N> &P, int sm_count)
{
    static_assert(NL == 0 || COEF == (NL == 2), "the Jacobian takes the coefficient layout, the residual not");
    static_assert(!ADV || (COEF && NL == 0 && !SLIM), "advection-diffusion takes the coefficient layout");
    using WS = WarpSmem<N, SLIM, COEF, ADV ? 3 : 1>;
    constexpr int WARPS_PER_CTA = WPC<N, SLIM, COEF>::value;
    constexpr int T = WARPS_PER_CTA * 32;
    auto kern = [] {
        if constexpr (ADV) return advection_diffusion_kernel<N, MASS, ATOMIC, MINB, MATRIX>;
        else if constexpr (NL == 1) return nonlinear_residual_kernel<N, MASS, ATOMIC, MINB, SLIM>;
        else if constexpr (NL == 2) return nonlinear_jacobian_kernel<N, MASS, ATOMIC, MINB, MATRIX, SLIM>;
        else if constexpr (COEF) return helmholtz_coef_kernel<N, MASS, ATOMIC, MINB, MATRIX, SLIM>;
        else return helmholtz_action_kernel<N, MASS, ATOMIC, MINB, MATRIX, SLIM, AFFINE>;
    }();
    static bool configured = false;
    static int occ = 1;
    if (!configured) {
        FDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, WS::CTA_BYTES));
        FDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, T, WS::CTA_BYTES));
        if (occ < 1) occ = 1;
        configured = true;
    }
    const int ncells = P.ncols * P.nlay_items;
    const int nitems = (ncells + WS::CW - 1) / WS::CW;
    int per_sm = occ;
    if (grid_cap_per_sm > 0 && grid_cap_per_sm < per_sm) per_sm = grid_cap_per_sm;
    long long grid = (long long)sm_count * per_sm;
    long long need = (nitems + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
    if (grid > need) grid = need;
    if (grid < 1) grid = 1;
    // chunk: one column's worth of items, bounded so that every resident warp
    // gets several chunks
    int chunk = P.nlay_items / WS::CW;
    if (chunk < 8) chunk = 8;
    if (chunk > 64) chunk = 64;
    long long per_warp = nitems / (grid * WARPS_PER_CTA) + 1;
    // at least ~32 chunks per warp: the tail of the persistent grid is then < 3 % of the launch
    // (2.1 M cells on one GPU = the per-rank load of an 8-GPU run: 1.237 ms with 4-item chunks
    // against 1.278 ms with 16; no effect at 256^3, where a column's 32 items stay one chunk)
    if (chunk > per_warp / 32 + 1) chunk = (int)(per_warp / 32 + 1);
    static const int chunk_env = getenv("FDB_CHUNK") ? atoi(getenv("FDB_CHUNK")) : 0;
    if (chunk_env > 0) chunk = chunk_env;
    P.chunk = chunk;
    P.nlay_rcp = (unsigned)(0x100000000ull / (unsigned long long)P.nlay_items);
    if (P.nlay_items == 1) P.nlay_rcp = 0xffffffffu;
    FDB_CUDA(cudaMemsetAsync(P.counter, 0, sizeof(int), st));
    if constexpr (NL != 0) kern<<<(int)grid, T, WS::CTA_BYTES, st>>>(P);
    else if constexpr (COEF) kern<<<(int)grid, T, WS::CTA_BYTES, st>>>(static_cast<const HelmCoefParams<N> &>(P));
    else kern<<<(int)grid, T, WS::CTA_BYTES, st>>>(static_cast<const HelmParams<N> &>(P));
    FDB_LAUNCH_CHECK();
    return 0;
}

// register bound of the coefficient kernel (-Xptxas -v, DESIGN.md section 4.5): shared memory holds
// two CTAs of 4 warps at degree 3 either way, so it gets the whole 255 registers there
template <int N>
struct CoefMinB {
    static constexpr int value = (N >= 5) ? 1 : 2;
};

// coefficient form (action): the slab-thread kernel for every degree -- no thread-per-cell,
// warp-specialised or affine variant
template <int N, bool ATOMIC>
int launch_coef(bool mass, int cap, cudaStream_t st, HelmNlParams<N> &P, int sm_count)
{
    constexpr int MB = CoefMinB<N>::value;
    if (N == 6 && P.nlay_items >= 32 / N) {
        if (mass) return launch_one<N, true, ATOMIC, MB, false, (N == 6), false, true>(cap, st, P, sm_count);
        return launch_one<N, false, ATOMIC, MB, false, (N == 6), false, true>(cap, st, P, sm_count);
    }
    if (mass) return launch_one<N, true, ATOMIC, MB, false, false, false, true>(cap, st, P, sm_count);
    return launch_one<N, false, ATOMIC, MB, false, false, false, true>(cap, st, P, sm_count);
}

// register bound of the residual kernel (-Xptxas -v, DESIGN.md section 4.6): as the constant-coefficient
// kernel, 3 CTAs x 4 warps x 168 registers at degree 3
template <int N>
struct NlResMinB {
    static constexpr int value = (N == 4) ? 3 : ((N >= 5) ? 1 : 2);
};

// nonlinear diffusion (nl = 1 residual, 2 Jacobian action): the slab-thread kernel for every degree,
// slim staging at degree 5 as for the other forms -- no thread-per-cell, warp-specialised or affine
// variant
template <int N, bool ATOMIC>
int launch_nl(int nl, bool mass, int cap, cudaStream_t st, HelmNlParams<N> &P, int sm_count)
{
    constexpr bool SL = (N == 6);
    const bool slim = SL && P.nlay_items >= 32 / N;
    if (nl == 1) {
        constexpr int MB = NlResMinB<N>::value;
        if (slim) {
            if (mass) return launch_one<N, true, ATOMIC, MB, false, SL, false, false, 1>(cap, st, P, sm_count);
            return launch_one<N, false, ATOMIC, MB, false, SL, false, false, 1>(cap, st, P, sm_count);
        }
        if (mass) return launch_one<N, true, ATOMIC, MB, false, false, false, false, 1>(cap, st, P, sm_count);
        return launch_one<N, false, ATOMIC, MB, false, false, false, false, 1>(cap, st, P, sm_count);
    }
    constexpr int MB = CoefMinB<N>::value;
    if (slim) {
        if (mass) return launch_one<N, true, ATOMIC, MB, false, SL, false, true, 2>(cap, st, P, sm_count);
        return launch_one<N, false, ATOMIC, MB, false, SL, false, true, 2>(cap, st, P, sm_count);
    }
    if (mass) return launch_one<N, true, ATOMIC, MB, false, false, false, true, 2>(cap, st, P, sm_count);
    return launch_one<N, false, ATOMIC, MB, false, false, false, true, 2>(cap, st, P, sm_count);
}

// advection-diffusion (action, element matrix or diagonal: MATRIX): the slab-thread kernel with b in three
// kappa buffers, degrees 1..4 (no slim staging, no thread-per-cell, warp-specialised, affine or DMMA variant);
// the register bound is the coefficient kernel's
template <int N, bool ATOMIC, bool MATRIX = false>
int launch_adv(bool mass, int cap, cudaStream_t st, HelmNlParams<N> &P, int sm_count)
{
    if constexpr (N <= (MATRIX ? 4 : 5)) {
        constexpr int MB = CoefMinB<N>::value;
        if (mass) return launch_one<N, true, ATOMIC, MB, MATRIX, false, false, true, 0, true>(cap, st, P, sm_count);
        return launch_one<N, false, ATOMIC, MB, MATRIX, false, false, true, 0, true>(cap, st, P, sm_count);
    }
    fdb::set_error("advection_diffusion %s: degree %d not instantiated", MATRIX ? "matrix" : "action", N - 1);
    return 1;
}

inline bool is_adv(const fdb_kernel_s *k) { return k->desc.form == FDB_FORM_ADVECTION_DIFFUSION; }

// nonlinear mode of a kernel: 1 residual, 2 Jacobian, 0 any other form
inline int nl_mode(const fdb_kernel_s *k)
{
    if (k->desc.form == FDB_FORM_NONLINEAR_DIFFUSION) return 1;
    if (k->desc.form == FDB_FORM_NONLINEAR_DIFFUSION_JACOBIAN) return 2;
    return 0;
}

template <int N>
void set_dcoef(const fdb_kernel_s *k, HelmNlParams<N> &P)
{
    for (int i = 0; i < 3; i++) P.dcoef[i] = nl_mode(k) ? k->desc.dcoef[i] : 0.0;
}

template <int N, bool ATOMIC>
int launch_variant(bool mass, int minb, int cap, cudaStream_t st, HelmNlParams<N> &P, int sm_count,
                   bool affine = false)
{
    if (affine && ATOMIC) {
        // affine cells (caller's promise): per-cell metric; same staging / occupancy choices
        constexpr int AB = (N == 4) ? 3 : ((N >= 5) ? 1 : 2);
        constexpr bool ASL = (N == 6);
        if (!ASL || P.nlay_items >= 32 / N) {
            if (mass) return launch_one<N, true, true, AB, false, ASL, true>(cap, st, P, sm_count);
            return launch_one<N, false, true, AB, false, ASL, true>(cap, st, P, sm_count);
        }
    }
    if (N == 4 && minb == 3) {
        if (mass) return launch_one<N, true, ATOMIC, (N == 4 ? 3 : 2)>(cap, st, P, sm_count);
        return launch_one<N, false, ATOMIC, (N == 4 ? 3 : 2)>(cap, st, P, sm_count);
    }
    if (N == 4 && minb == 4) {
        if (mass) return launch_one<N, true, ATOMIC, (N == 4 ? 4 : 2)>(cap, st, P, sm_count);
        return launch_one<N, false, ATOMIC, (N == 4 ? 4 : 2)>(cap, st, P, sm_count);
    }
    if (N == 4 && minb == 1) {
        if (mass) return launch_one<N, true, ATOMIC, 1>(cap, st, P, sm_count);
        return launch_one<N, false, ATOMIC, 1>(cap, st, P, sm_count);
    }
    constexpr int DEF = (N >= 5) ? 1 : 2;
    if (N == 6) {
        // degree 5: the slim staging lifts occupancy from 5 to 8 warps per SM (12.9 -> 9.0 ms at
        // 128^3); for degree 4 occupancy is register-bound either way and it measured 6 % slower
        static const bool slim_on = !(getenv("FDB_NO_SLIM") && atoi(getenv("FDB_NO_SLIM")));
        if (slim_on && P.nlay_items >= 32 / N) {
            if (mass) return launch_one<N, true, ATOMIC, DEF, false, (N == 6)>(cap, st, P, sm_count);
            return launch_one<N, false, ATOMIC, DEF, false, (N == 6)>(cap, st, P, sm_count);
        }
    }
    if (mass) return launch_one<N, true, ATOMIC, DEF>(cap, st, P, sm_count);
    return launch_one<N, false, ATOMIC, DEF>(cap, st, P, sm_count);
}

template <int N>
int launch_n(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
             double *y, const double *coords, const double *x, const fdb_int *map0,
             const fdb_int *map1, const double *kappa)
{
    fdb::Context &c = fdb::ctx();
    HelmNlParams<N> P;
    P.kappa = kappa;             // NULL: constant-coefficient form and residual
    set_dcoef(k, P);
    const int nl = nl_mode(k);
    P.y = y;
    P.x = x;
    P.coords = coords;
    P.map0 = map0;
    P.map1 = map1;
    P.off0 = k->d_off0;
    P.off1 = k->d_off1;
    P.cdim = k->desc.cdim;
    P.alpha = k->desc.alpha;
    P.beta = k->desc.beta;
    for (int i = 0; i < N * N; i++) {
        P.B[i] = k->desc.B[i];
        P.Dt[i] = k->Dt[i];
    }
    for (int q = 0; q < N; q++)
        for (int j = 0; j < N; j++) {
            P.DtR[q * N + j] = k->Dt[q * N + (j + q) % N];
            double d = 0.0;
            for (int i = 0; i < N; i++) d += k->Dt[q * N + i] * k->desc.B[i * N + j];
            P.DB[q * N + j] = d;
        }
    for (int i = 0; i < N; i++) {
        P.wq[i] = k->desc.wq[i];
        P.xq[i] = k->desc.xq[i];
    }
    const bool mass = k->desc.beta != 0.0;
    static const int minb = getenv("FDB_MINB") ? atoi(getenv("FDB_MINB")) : 3;   // N == 4: 3 CTAs x 4 warps, 168 registers (DESIGN.md 4.1)
    static const int cap = getenv("FDB_CTAS_PER_SM") ? atoi(getenv("FDB_CTAS_PER_SM")) : 0;
    P.counter = c.work_counter;
    if (k->desc.scatter == FDB_SCATTER_ATOMIC) {
        P.collist = subset;
        P.col0 = start;
        P.ncols = end - start;
        P.nlay_items = nlay;
        P.lay_first = 0;
        P.lay_step = 1;
        if (P.ncols <= 0 || nlay <= 0) return 0;
        if (is_adv(k)) return launch_adv<N, true>(mass, cap, c.stream, P, c.sm_count);
        if (kappa && !nl) return launch_coef<N, true>(mass, cap, c.stream, P, c.sm_count);
        if (nl) return launch_nl<N, true>(nl, mass, cap, c.stream, P, c.sm_count);
        if constexpr (N == 4) {
            // degree 3, scalar: warp-specialised kernel (action_hex_ws.cuh)
            static const int ws = getenv("FDB_WS") ? atoi(getenv("FDB_WS")) : 0;
            if (ws && P.cdim == 1 && nlay >= 8 && !k->desc.affine_cells) {
#define FDB_WS_CASE(id, NC, NM, NS, ST)                                                            \
    if (ws == id)                                                                              \
        return mass ? launch_ws<true, NC, NM, NS, ST>(c.stream, P, c.sm_count)                 \
                    : launch_ws<false, NC, NM, NS, ST>(c.stream, P, c.sm_count);
                FDB_WS_CASE(1, 12, 4, 2, true)     // 12 compute warps x 160 registers, 4 movers x 32, 2 stages
                FDB_WS_CASE(2, 8, 4, 3, true)      // 8 x 224, 4 movers x 56, 3 stages
                FDB_WS_CASE(3, 8, 4, 3, false)     // ... geometry coefficients kept in registers
                FDB_WS_CASE(4, 8, 8, 3, false)     // 8 x 208, one mover (48) per compute warp
#undef FDB_WS_CASE
            }
        }
        return launch_variant<N, true>(mass, minb, cap, c.stream, P, c.sm_count, k->desc.affine_cells != 0);
    }
    // deterministic: one launch per (colour, layer parity); within a launch no
    // two cells share a dof, so plain read-modify-write is race free and the
    // summation order is fixed.
    if (subset) {
        fdb::set_error("coloured scatter does not support subsets yet");
        return 1;
    }
    for (int col = 0; col < k->ncolours; col++) {
        int cbeg = k->colour_start[col], cend = k->colour_start[col + 1];
        for (int par = 0; par < (nlay > 1 ? 2 : 1); par++) {
            P.collist = k->d_colour_cols + cbeg;
            P.col0 = 0;
            P.ncols = cend - cbeg;
            P.lay_first = par;
            P.lay_step = 2;
            P.nlay_items = (nlay - par + 1) / 2;
            if (P.ncols <= 0 || P.nlay_items <= 0) continue;
            if (is_adv(k)      ? launch_adv<N, false>(mass, cap, c.stream, P, c.sm_count)
                : kappa && !nl ? launch_coef<N, false>(mass, cap, c.stream, P, c.sm_count)
                : nl         ? launch_nl<N, false>(nl, mass, cap, c.stream, P, c.sm_count)
                             : launch_variant<N, false>(mass, minb, cap, c.stream, P, c.sm_count))
                return 1;
        }
    }
    return 0;
}

template <int N>
int launch_matrix_n(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                    fdb_mat_t mat, const double *coords, const fdb_int *map0, const fdb_int *map1,
                    double *diag_out, const double *kappa)
{
    fdb::Context &c = fdb::ctx();
    HelmNlParams<N> P;
    memset(&P, 0, sizeof(P));
    P.kappa = kappa;             // NULL: constant-coefficient form
    set_dcoef(k, P);
    P.coords = coords;
    P.map0 = map0;
    P.map1 = map1;
    P.off0 = k->d_off0;
    P.off1 = k->d_off1;
    P.cdim = N * N * N;          // one pipeline unit per trial dof
    P.alpha = k->desc.alpha;
    P.beta = k->desc.beta;
    for (int i = 0; i < N * N; i++) {
        P.B[i] = k->desc.B[i];
        P.Dt[i] = k->Dt[i];
    }
    for (int q = 0; q < N; q++)
        for (int j = 0; j < N; j++) {
            P.DtR[q * N + j] = k->Dt[q * N + (j + q) % N];
            double d = 0.0;
            for (int i = 0; i < N; i++) d += k->Dt[q * N + i] * k->desc.B[i * N + j];
            P.DB[q * N + j] = d;
        }
    for (int i = 0; i < N; i++) {
        P.wq[i] = k->desc.wq[i];
        P.xq[i] = k->desc.xq[i];
    }
    if (mat) {
        fdb_mat_device_view(mat, &P.rowptr, &P.colidx, &P.vals, &P.row_lg, &P.col_lg);
        fdb_mat_rank_table(mat, &P.rank_tab, &P.nvar);
    } else {
        P.y = diag_out;          // diagonal mode
    }
    P.nlay_total = nlay;
    if (subset || k->desc.cell != FDB_CELL_HEX_EXTRUDED) P.rank_tab = nullptr;   // table is per column of the full set
    P.counter = c.work_counter;
    P.collist = subset;
    P.col0 = start;
    P.ncols = end - start;
    P.nlay_items = nlay;
    P.lay_first = 0;
    P.lay_step = 1;
    if (P.ncols <= 0 || nlay <= 0) return 0;
    if (is_adv(k)) return launch_adv<N, true, true>(k->desc.beta != 0.0, 0, c.stream, P, c.sm_count);
    if (kappa && nl_mode(k) == 0) {
        constexpr int MB = CoefMinB<N>::value;
        if (k->desc.beta != 0.0)
            return launch_one<N, true, true, MB, true, false, false, true>(0, c.stream, P, c.sm_count);
        return launch_one<N, false, true, MB, true, false, false, true>(0, c.stream, P, c.sm_count);
    }
    if (nl_mode(k) == 2) {
        // the Jacobian's element matrix / diagonal: u in the kappa buffer, reused across the N^3 units
        constexpr int MB = CoefMinB<N>::value;
        if (k->desc.beta != 0.0)
            return launch_one<N, true, true, MB, true, false, false, true, 2>(0, c.stream, P, c.sm_count);
        return launch_one<N, false, true, MB, true, false, false, true, 2>(0, c.stream, P, c.sm_count);
    }
    constexpr int DEF = (N >= 5) ? 1 : 2;
    if (k->desc.beta != 0.0) return launch_one<N, true, true, DEF, true>(0, c.stream, P, c.sm_count);
    return launch_one<N, false, true, DEF, true>(0, c.stream, P, c.sm_count);
}

}  // namespace

int fdb_launch_helmholtz_matrix(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay,
                                const fdb_int *subset, fdb_mat_t mat, const double *coords,
                                const fdb_int *map0, const fdb_int *map1, double *diag_out)
{
    // explicit matrices: dense B^T D B on the fp64 tensor pipe (bdb_matrix.cu) where it is the
    // faster kernel -- degrees 3 and 4 (symmetric tilings: CG3 64^3 15.4 against 23.3 ms, config 4 at
    // 32^3 11.9 against 18.2 ms; at degree 2 the sum-factorised kernel wins, 1.26 against 1.73 ms);
    // option "matrix_kernel": 0 keeps the sum-factorised column-by-column kernel everywhere, 1 takes
    // the DMMA kernel for every instantiated degree (2..4)
    const int dmma = fdb_opt_matrix_kernel;
    if (mat && dmma != 0 && k->n1d <= 5 && k->n1d >= (dmma == 1 ? 3 : 4))
        return fdb_launch_helmholtz_matrix_dmma(k, start, end, nlay, subset, mat, coords, map0, map1);
    switch (k->n1d) {
    case 2: return launch_matrix_n<2>(k, start, end, nlay, subset, mat, coords, map0, map1, diag_out, nullptr);
    case 3: return launch_matrix_n<3>(k, start, end, nlay, subset, mat, coords, map0, map1, diag_out, nullptr);
    case 4: return launch_matrix_n<4>(k, start, end, nlay, subset, mat, coords, map0, map1, diag_out, nullptr);
    case 5: return launch_matrix_n<5>(k, start, end, nlay, subset, mat, coords, map0, map1, diag_out, nullptr);
    }
    fdb::set_error("helmholtz matrix: degree %d not instantiated (1..4)", k->n1d - 1);
    return 1;
}

int fdb_launch_helmholtz_action(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay,
                                const fdb_int *subset, double *y, const double *coords,
                                const double *x, const fdb_int *map0, const fdb_int *map1)
{
    // degree 1 on extruded columns: one thread per cell (q1_action.cu); FDB_Q1_THREAD=0 opts out
    static const bool q1_thread = !(getenv("FDB_Q1_THREAD") && atoi(getenv("FDB_Q1_THREAD")) == 0);
    if (q1_thread && k->n1d == 2 && k->desc.cdim == 1 && k->desc.scatter == FDB_SCATTER_ATOMIC &&
        k->desc.cell == FDB_CELL_HEX_EXTRUDED && nlay >= 16)
        return fdb_launch_q1_action(k, start, end, nlay, subset, y, coords, x, map0, map1);
    // degree 2 likewise (q2_action.cu); FDB_Q2_THREAD=0 opts out
    static const bool q2_thread = !(getenv("FDB_Q2_THREAD") && atoi(getenv("FDB_Q2_THREAD")) == 0);
    if (q2_thread && k->n1d == 3 && k->desc.cdim == 1 && k->desc.scatter == FDB_SCATTER_ATOMIC &&
        k->desc.cell == FDB_CELL_HEX_EXTRUDED && nlay >= 16)
        return fdb_launch_q2_action(k, start, end, nlay, subset, y, coords, x, map0, map1);
    switch (k->n1d) {
    case 2: return launch_n<2>(k, start, end, nlay, subset, y, coords, x, map0, map1, nullptr);
    case 3: return launch_n<3>(k, start, end, nlay, subset, y, coords, x, map0, map1, nullptr);
    case 4: return launch_n<4>(k, start, end, nlay, subset, y, coords, x, map0, map1, nullptr);
    case 5: return launch_n<5>(k, start, end, nlay, subset, y, coords, x, map0, map1, nullptr);
    case 6: return launch_n<6>(k, start, end, nlay, subset, y, coords, x, map0, map1, nullptr);
    }
    fdb::set_error("helmholtz action: degree %d not instantiated (1..5)", k->n1d - 1);
    return 1;
}

// FDB_FORM_HELMHOLTZ_COEF: the slab-thread kernel for every degree (1..5 action, 1..4 matrix and
// diagonal); never the thread-per-cell, warp-specialised, affine or DMMA kernels.  The nonlinear
// diffusion and advection-diffusion forms take the same entry points (launch_n / launch_matrix_n pick
// the mode from the form): the residual with kappa = NULL, the Jacobian with kappa = the linearisation
// point u, advection-diffusion with kappa = b (3 values per node).
int fdb_launch_helmholtz_coef_action(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay,
                                     const fdb_int *subset, double *y, const double *coords,
                                     const double *x, const double *kappa, const fdb_int *map0,
                                     const fdb_int *map1)
{
    switch (k->n1d) {
    case 2: return launch_n<2>(k, start, end, nlay, subset, y, coords, x, map0, map1, kappa);
    case 3: return launch_n<3>(k, start, end, nlay, subset, y, coords, x, map0, map1, kappa);
    case 4: return launch_n<4>(k, start, end, nlay, subset, y, coords, x, map0, map1, kappa);
    case 5: return launch_n<5>(k, start, end, nlay, subset, y, coords, x, map0, map1, kappa);
    case 6: return launch_n<6>(k, start, end, nlay, subset, y, coords, x, map0, map1, kappa);
    }
    fdb::set_error("helmholtz_coef action: degree %d not instantiated (1..5)", k->n1d - 1);
    return 1;
}

int fdb_launch_helmholtz_coef_matrix(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay,
                                     const fdb_int *subset, fdb_mat_t mat, const double *coords,
                                     const double *kappa, const fdb_int *map0, const fdb_int *map1,
                                     double *diag_out)
{
    switch (k->n1d) {
    case 2: return launch_matrix_n<2>(k, start, end, nlay, subset, mat, coords, map0, map1, diag_out, kappa);
    case 3: return launch_matrix_n<3>(k, start, end, nlay, subset, mat, coords, map0, map1, diag_out, kappa);
    case 4: return launch_matrix_n<4>(k, start, end, nlay, subset, mat, coords, map0, map1, diag_out, kappa);
    case 5: return launch_matrix_n<5>(k, start, end, nlay, subset, mat, coords, map0, map1, diag_out, kappa);
    }
    fdb::set_error("helmholtz_coef matrix: degree %d not instantiated (1..4)", k->n1d - 1);
    return 1;
}
