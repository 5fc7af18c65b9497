// Block-vector operations over columns that are ordinary device Dats (SLEPc's BVDot and BVMult): the subspace half
// of LOBPCG (firedrake_b200/eigensolver.py).  The column pointers travel in the kernel's parameter struct, so no
// device-side pointer array is built or copied.
//
// fdb_bv_dot: each CTA stages chunks of BV_ROWS rows of every x and y column in shared memory and each thread
// accumulates a T x T tile of G over a slice of the chunk's rows; the slices are summed in a fixed order, one partial
// G per CTA goes to a scratch buffer, and a second pass sums the partials in CTA order.  The grid depends only on n,
// so G is bitwise repeatable for the same inputs.
// fdb_bv_mult: Q is staged to the device once per call, through a ring of pinned slots, and into shared memory once per
// CTA; each thread owns rows and forms all k outputs of a row from one read of its m inputs, so every x column is read
// once per call.
#include "common.cuh"

#include <algorithm>

using namespace fdb;

namespace {

constexpr int BV_MAX = FDB_BV_MAX_COLUMNS;
constexpr int BV_THREADS = 256;
constexpr int BV_ROWS = 32;                 // rows per staged chunk
constexpr int BV_LD = BV_MAX + 1;           // odd row stride of the staged chunks (no bank conflicts on the stores)
constexpr int BV_SLACK = 8;                 // a T x T tile of the last row may read past column m
constexpr int BV_DOT_BLOCKS = 528;          // 132 SMs x 4 (H100 SXM); fixed, so the grid depends only on n
constexpr int BV_MULT_THREADS = 128;

struct BvCols {
    const double *p[BV_MAX];
};

struct BvOut {
    double *p[BV_MAX];
};

// one partial G per CTA: partial[blockIdx.x * m * k + i * k + j]
template <int T>
__global__ void __launch_bounds__(BV_THREADS)
k_bv_dot_partial(size_t n, int m, int k, int tiles_j, int ntiles, int nslices, const __grid_constant__ BvCols x,
                 const __grid_constant__ BvCols y, double *__restrict__ partial)
{
    __shared__ double sh[2 * BV_ROWS * BV_LD + BV_SLACK];
    double *sx = sh, *sy = sh + BV_ROWS * BV_LD;
    const int t = threadIdx.x;
    const int tile = t % ntiles, slice = t / ntiles;
    const bool active = slice < nslices;
    const int i0 = (tile / tiles_j) * T, j0 = (tile % tiles_j) * T;
    double acc[T][T];
#pragma unroll
    for (int a = 0; a < T; ++a)
#pragma unroll
        for (int b = 0; b < T; ++b) acc[a][b] = 0.0;
    const size_t nchunks = (n + BV_ROWS - 1) / BV_ROWS;
    for (size_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const size_t base = c * BV_ROWS;
        __syncthreads();
        for (int e = t; e < m * BV_ROWS; e += BV_THREADS) {
            const int i = e / BV_ROWS, r = e % BV_ROWS;
            const size_t row = base + r;
            sx[r * BV_LD + i] = row < n ? x.p[i][row] : 0.0;
        }
        for (int e = t; e < k * BV_ROWS; e += BV_THREADS) {
            const int j = e / BV_ROWS, r = e % BV_ROWS;
            const size_t row = base + r;
            sy[r * BV_LD + j] = row < n ? y.p[j][row] : 0.0;
        }
        __syncthreads();
        if (active) {
            for (int r = slice; r < BV_ROWS; r += nslices) {
                double xa[T], yb[T];
#pragma unroll
                for (int a = 0; a < T; ++a) xa[a] = sx[r * BV_LD + i0 + a];
#pragma unroll
                for (int b = 0; b < T; ++b) yb[b] = sy[r * BV_LD + j0 + b];
#pragma unroll
                for (int a = 0; a < T; ++a)
#pragma unroll
                    for (int b = 0; b < T; ++b) acc[a][b] = fma(xa[a], yb[b], acc[a][b]);
            }
        }
    }
    // the slices of each tile, summed in slice order
    __syncthreads();
    if (active) {
#pragma unroll
        for (int a = 0; a < T; ++a)
#pragma unroll
            for (int b = 0; b < T; ++b) sh[(t * T + a) * T + b] = acc[a][b];
    }
    __syncthreads();
    if (t < ntiles) {
        double *out = partial + (size_t)blockIdx.x * m * k;
#pragma unroll
        for (int a = 0; a < T; ++a)
#pragma unroll
            for (int b = 0; b < T; ++b) {
                double s = 0.0;
                for (int q = 0; q < nslices; ++q) s += sh[((q * ntiles + t) * T + a) * T + b];
                const int i = i0 + a, j = j0 + b;
                if (i < m && j < k) out[i * k + j] = s;
            }
    }
}

// G[e] = sum over CTAs b, in order, of partial[b * mk + e]
__global__ void __launch_bounds__(BV_THREADS)
k_bv_dot_final(int nb, int mk, const double *__restrict__ partial, double *__restrict__ g)
{
    const int e = blockIdx.x * BV_THREADS + threadIdx.x;
    if (e >= mk) return;
    double s = 0.0;
    for (int b = 0; b < nb; ++b) s += partial[(size_t)b * mk + e];
    g[e] = s;
}

// y_j = beta y_j + alpha sum_i x_i Q[i, j] for j < k <= KMAX; beta == 0 does not read y
template <int KMAX>
__global__ void __launch_bounds__(BV_MULT_THREADS)
k_bv_mult(size_t n, int k, int m, double beta, double alpha, const __grid_constant__ BvOut y,
          const __grid_constant__ BvCols x, const double *__restrict__ q)
{
    __shared__ __align__(16) double sq[BV_MAX * KMAX];
    for (int e = threadIdx.x; e < m * KMAX; e += BV_MULT_THREADS) {
        const int i = e / KMAX, j = e % KMAX;
        sq[e] = j < k ? q[i * k + j] : 0.0;
    }
    __syncthreads();
    const size_t stride = (size_t)gridDim.x * BV_MULT_THREADS;
    for (size_t row = (size_t)blockIdx.x * BV_MULT_THREADS + threadIdx.x; row < n; row += stride) {
        double acc[KMAX];
#pragma unroll
        for (int j = 0; j < KMAX; ++j) acc[j] = 0.0;
        for (int i = 0; i < m; ++i) {
            const double xi = x.p[i][row];
            const double2 *qi = reinterpret_cast<const double2 *>(sq + i * KMAX);
#pragma unroll
            for (int j = 0; j < KMAX / 2; ++j) {
                const double2 qv = qi[j];
                acc[2 * j] = fma(xi, qv.x, acc[2 * j]);
                acc[2 * j + 1] = fma(xi, qv.y, acc[2 * j + 1]);
            }
        }
#pragma unroll
        for (int j = 0; j < KMAX; ++j) {
            if (j < k) {
                double *yj = y.p[j];
                yj[row] = beta == 0.0 ? alpha * acc[j] : fma(beta, yj[row], alpha * acc[j]);
            }
        }
    }
}

// the kernels' own buffers: grown to the largest request, released by fdb_finalize
double *g_partial = nullptr;
size_t g_partial_count = 0;
double *g_dev_small = nullptr;              // G of fdb_bv_dot on the device (BV_MAX^2)
double *g_host_small = nullptr;             // pinned G
// Q of fdb_bv_mult: a ring of pinned and device slots, so that the H2D copy is asynchronous and the host only waits
// for the copy of the call BV_Q_SLOTS calls back
constexpr int BV_Q_SLOTS = 32;
double *g_q_host = nullptr, *g_q_dev = nullptr;
cudaEvent_t g_q_done[BV_Q_SLOTS];
bool g_q_used[BV_Q_SLOTS] = {};
int g_q_next = 0;

int ensure_buffers(size_t partial_count)
{
    if (!g_dev_small) FDB_CUDA(cudaMalloc(&g_dev_small, BV_MAX * BV_MAX * sizeof(double)));
    if (!g_host_small)
        FDB_CUDA(cudaHostAlloc((void **)&g_host_small, BV_MAX * BV_MAX * sizeof(double), cudaHostAllocDefault));
    if (!g_q_host) {
        FDB_CUDA(cudaHostAlloc((void **)&g_q_host, BV_Q_SLOTS * BV_MAX * BV_MAX * sizeof(double),
                               cudaHostAllocDefault));
        FDB_CUDA(cudaMalloc(&g_q_dev, BV_Q_SLOTS * BV_MAX * BV_MAX * sizeof(double)));
        for (int i = 0; i < BV_Q_SLOTS; ++i) FDB_CUDA(cudaEventCreateWithFlags(&g_q_done[i], cudaEventDisableTiming));
    }
    if (partial_count > g_partial_count) {
        if (g_partial) {
            FDB_CUDA(cudaStreamSynchronize(ctx().stream));
            cudaFree(g_partial);
            g_partial = nullptr;
            g_partial_count = 0;
        }
        FDB_CUDA(cudaMalloc(&g_partial, partial_count * sizeof(double)));
        g_partial_count = partial_count;
    }
    return 0;
}

int check_columns(const char *fn, const char *what, int count, const double *const *cols)
{
    if (count < 1 || count > BV_MAX) {
        set_error("%s: %s = %d columns; 1..%d (FDB_BV_MAX_COLUMNS)", fn, what, count, BV_MAX);
        return 1;
    }
    if (!cols) {
        set_error("%s: NULL column array for %s", fn, what);
        return 1;
    }
    for (int i = 0; i < count; ++i)
        if (!cols[i]) {
            set_error("%s: column %d of %s is NULL", fn, i, what);
            return 1;
        }
    return 0;
}

// the tile edge T in 1..4 that keeps the most of the CTA's threads busy (ties: the larger T, fewer shared-memory
// reads per FMA); a tile's row slices never outnumber the chunk's rows
void dot_shape(int m, int k, int *T, int *tiles_j, int *ntiles, int *nslices)
{
    int best = -1;
    for (int t = 4; t >= 1; --t) {
        const int tj = (k + t - 1) / t, nt = ((m + t - 1) / t) * tj;
        if (nt > BV_THREADS) continue;
        const int ns = std::min(BV_THREADS / nt, BV_ROWS);
        if (ns * nt > best) {
            best = ns * nt;
            *T = t, *tiles_j = tj, *ntiles = nt, *nslices = ns;
        }
    }
}

}  // namespace

void fdb::fdb_bv_release()
{
    cudaFree(g_partial);
    cudaFree(g_dev_small);
    cudaFreeHost(g_host_small);
    if (g_q_host) {
        for (int i = 0; i < BV_Q_SLOTS; ++i) cudaEventDestroy(g_q_done[i]);
        cudaFreeHost(g_q_host);
        cudaFree(g_q_dev);
    }
    for (int i = 0; i < BV_Q_SLOTS; ++i) g_q_used[i] = false;
    g_q_host = g_q_dev = nullptr;
    g_q_next = 0;
    g_partial = g_dev_small = g_host_small = nullptr;
    g_partial_count = 0;
}

extern "C" {

int fdb_bv_dot(size_t n, int m, const double *const *x, int k, const double *const *y, double *g_host)
{
    if (require_init()) return 1;
    if (check_columns("fdb_bv_dot", "x (m)", m, x) || check_columns("fdb_bv_dot", "y (k)", k, y)) return 1;
    if (!g_host) {
        set_error("fdb_bv_dot: NULL host pointer for G");
        return 1;
    }
    if (n == 0) {
        memset(g_host, 0, (size_t)m * k * sizeof(double));
        return 0;
    }
    Context &c = ctx();
    const int nb = (int)std::min<size_t>((n + BV_ROWS - 1) / BV_ROWS, BV_DOT_BLOCKS);
    if (ensure_buffers((size_t)nb * m * k)) return 1;
    BvCols xs{}, ys{};
    for (int i = 0; i < m; ++i) xs.p[i] = x[i];
    for (int j = 0; j < k; ++j) ys.p[j] = y[j];
    int T = 1, tiles_j = 1, ntiles = 1, nslices = 1;
    dot_shape(m, k, &T, &tiles_j, &ntiles, &nslices);
    switch (T) {
    case 4: k_bv_dot_partial<4><<<nb, BV_THREADS, 0, c.stream>>>(n, m, k, tiles_j, ntiles, nslices, xs, ys, g_partial);
        break;
    case 3: k_bv_dot_partial<3><<<nb, BV_THREADS, 0, c.stream>>>(n, m, k, tiles_j, ntiles, nslices, xs, ys, g_partial);
        break;
    case 2: k_bv_dot_partial<2><<<nb, BV_THREADS, 0, c.stream>>>(n, m, k, tiles_j, ntiles, nslices, xs, ys, g_partial);
        break;
    default: k_bv_dot_partial<1><<<nb, BV_THREADS, 0, c.stream>>>(n, m, k, tiles_j, ntiles, nslices, xs, ys, g_partial);
    }
    FDB_LAUNCH_CHECK();
    const int mk = m * k;
    k_bv_dot_final<<<(mk + BV_THREADS - 1) / BV_THREADS, BV_THREADS, 0, c.stream>>>(nb, mk, g_partial, g_dev_small);
    FDB_LAUNCH_CHECK();
    FDB_CUDA(cudaMemcpyAsync(g_host_small, g_dev_small, mk * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
    FDB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(g_host, g_host_small, mk * sizeof(double));
    return 0;
}

int fdb_bv_mult(size_t n, int k, double *const *y, double beta, double alpha, int m, const double *const *x,
                const double *q_host)
{
    if (require_init()) return 1;
    if (check_columns("fdb_bv_mult", "y (k)", k, (const double *const *)y) ||
        check_columns("fdb_bv_mult", "x (m)", m, x))
        return 1;
    if (!q_host) {
        set_error("fdb_bv_mult: NULL host pointer for Q");
        return 1;
    }
    for (int j = 0; j < k; ++j)
        for (int i = 0; i < m; ++i)
            if (y[j] == x[i]) {
                set_error("fdb_bv_mult: y column %d is x column %d; the update is not in place", j, i);
                return 1;
            }
    if (n == 0) return 0;
    Context &c = ctx();
    if (ensure_buffers(0)) return 1;
    // Q through the next pinned slot: its previous copy (BV_Q_SLOTS calls back) has to be done before it is
    // overwritten; the device slot is then read only by this call's kernel, which the stream orders after the copy
    const int slot = g_q_next;
    g_q_next = (g_q_next + 1) % BV_Q_SLOTS;
    double *qh = g_q_host + (size_t)slot * BV_MAX * BV_MAX, *qd = g_q_dev + (size_t)slot * BV_MAX * BV_MAX;
    if (g_q_used[slot]) FDB_CUDA(cudaEventSynchronize(g_q_done[slot]));
    memcpy(qh, q_host, (size_t)m * k * sizeof(double));
    FDB_CUDA(cudaMemcpyAsync(qd, qh, (size_t)m * k * sizeof(double), cudaMemcpyHostToDevice, c.stream));
    FDB_CUDA(cudaEventRecord(g_q_done[slot], c.stream));
    g_q_used[slot] = true;
    BvOut ys{};
    BvCols xs{};
    for (int j = 0; j < k; ++j) ys.p[j] = y[j];
    for (int i = 0; i < m; ++i) xs.p[i] = x[i];
    const int blocks = (int)std::min<size_t>((n + BV_MULT_THREADS - 1) / BV_MULT_THREADS, (size_t)c.sm_count * 8);
    if (k <= 8)
        k_bv_mult<8><<<blocks, BV_MULT_THREADS, 0, c.stream>>>(n, k, m, beta, alpha, ys, xs, qd);
    else if (k <= 16)
        k_bv_mult<16><<<blocks, BV_MULT_THREADS, 0, c.stream>>>(n, k, m, beta, alpha, ys, xs, qd);
    else if (k <= 32)
        k_bv_mult<32><<<blocks, BV_MULT_THREADS, 0, c.stream>>>(n, k, m, beta, alpha, ys, xs, qd);
    else if (k <= 48)
        k_bv_mult<48><<<blocks, BV_MULT_THREADS, 0, c.stream>>>(n, k, m, beta, alpha, ys, xs, qd);
    else
        k_bv_mult<64><<<blocks, BV_MULT_THREADS, 0, c.stream>>>(n, k, m, beta, alpha, ys, xs, qd);
    FDB_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
