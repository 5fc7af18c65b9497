// Dat subset operations (K5) and vector algebra (K6) on device buffers.
// Reference semantics: firedrake/bcs.py:192-221 (DirichletBC.zero/set),
// pyop2/types/dat.py:297-311 (zero(subset)), :354-540 (_op/_iop/inner/axpy).
// All are single-pass HBM-bound streams: 128-bit vectorised where the layout
// allows, grid sized to a multiple of the SM count.
#include "common.cuh"

using namespace fdb;

namespace {

__global__ void k_zero_nodes(double *dat, int cdim, const fdb_int *nodes, fdb_int n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long tot = (long long)n * cdim;
    for (; i < tot; i += (long long)gridDim.x * blockDim.x) {
        fdb_int k = (fdb_int)(i / cdim);
        int c = (int)(i - (long long)k * cdim);
        dat[(long long)nodes[k] * cdim + c] = 0.0;
    }
}

__global__ void k_set_nodes(double *dat, const double *src, double value, int cdim,
                            const fdb_int *nodes, fdb_int n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long tot = (long long)n * cdim;
    for (; i < tot; i += (long long)gridDim.x * blockDim.x) {
        fdb_int k = (fdb_int)(i / cdim);
        int c = (int)(i - (long long)k * cdim);
        long long j = (long long)nodes[k] * cdim + c;
        dat[j] = src ? src[j] : value;
    }
}

template <int OP>   // 0: y += a x   1: y = x + a y   2: x *= a   3: w = x*y
__global__ void k_stream(size_t n, double a, const double *__restrict__ x,
                         double *__restrict__ y, double *__restrict__ w)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t n2 = n / 2;
    // all buffers come from cudaMalloc (256 B aligned): double2 is safe
    for (size_t j = i; j < n2; j += stride) {
        if (OP == 0) {
            double2 xv = reinterpret_cast<const double2 *>(x)[j];
            double2 yv = reinterpret_cast<double2 *>(y)[j];
            yv.x = fma(a, xv.x, yv.x);
            yv.y = fma(a, xv.y, yv.y);
            reinterpret_cast<double2 *>(y)[j] = yv;
        } else if (OP == 1) {
            double2 xv = reinterpret_cast<const double2 *>(x)[j];
            double2 yv = reinterpret_cast<double2 *>(y)[j];
            yv.x = fma(a, yv.x, xv.x);
            yv.y = fma(a, yv.y, xv.y);
            reinterpret_cast<double2 *>(y)[j] = yv;
        } else if (OP == 2) {
            double2 yv = reinterpret_cast<double2 *>(y)[j];
            yv.x *= a;
            yv.y *= a;
            reinterpret_cast<double2 *>(y)[j] = yv;
        } else {
            double2 xv = reinterpret_cast<const double2 *>(x)[j];
            double2 yv = reinterpret_cast<const double2 *>(y)[j];
            reinterpret_cast<double2 *>(w)[j] = make_double2(xv.x * yv.x, xv.y * yv.y);
        }
    }
    if (i == 0 && (n & 1)) {
        size_t j = n - 1;
        if (OP == 0) y[j] = fma(a, x[j], y[j]);
        else if (OP == 1) y[j] = fma(a, y[j], x[j]);
        else if (OP == 2) y[j] *= a;
        else w[j] = x[j] * y[j];
    }
}

// x[:] = a (no alignment assumption: used on the ghost tail of a Dat)
__global__ void k_fill(size_t n, double a, double *__restrict__ x)
{
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) x[j] = a;
}

// compact gather / scatter through an index list (virtual sub-matrices of a matrix-free operator)
__global__ void k_gather(size_t n, const fdb_int *__restrict__ idx, const double *__restrict__ src,
                         double *__restrict__ dst)
{
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) dst[j] = src[idx[j]];
}

__global__ void k_scatter(size_t n, const fdb_int *__restrict__ idx, const double *__restrict__ src,
                          double *__restrict__ dst)
{
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) dst[idx[j]] = src[j];
}

// one Chebyshev iteration's vector work, d = c_d d + c_z dinv o (b - ax), x += d, in a single pass (c_d == 0: the
// first iteration, d is not read)
__global__ void k_chebyshev(size_t n, double cd, double cz, const double *__restrict__ b, const double *__restrict__ ax,
                            const double *__restrict__ dinv, double *__restrict__ d, double *__restrict__ x)
{
    size_t stride = (size_t)gridDim.x * blockDim.x;
    const bool first = cd == 0.0;
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        const double z = cz * (dinv[j] * (b[j] - ax[j]));
        const double dj = first ? z : fma(cd, d[j], z);
        d[j] = dj;
        x[j] += dj;
    }
}

constexpr int DOT_BLOCKS_MAX = 1056;   // 132 SMs x 8 (H100 SXM)

__global__ void __launch_bounds__(256)
k_dot_partial(size_t n, const double *__restrict__ x, const double *__restrict__ y,
              double *__restrict__ partial)
{
    double s = 0.0;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t n2 = n / 2;
    for (size_t j = i; j < n2; j += stride) {
        double2 xv = reinterpret_cast<const double2 *>(x)[j];
        double2 yv = reinterpret_cast<const double2 *>(y)[j];
        s = fma(xv.x, yv.x, s);
        s = fma(xv.y, yv.y, s);
    }
    if (i == 0 && (n & 1)) s = fma(x[n - 1], y[n - 1], s);
    __shared__ double sh[8];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 8) {
        s = sh[threadIdx.x];
        for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffu, s, o);
        if (threadIdx.x == 0) partial[blockIdx.x] = s;
    }
}

__global__ void __launch_bounds__(256) k_dot_final(int nb, const double *partial, double *out)
{
    // fixed-order tree: deterministic for a given grid
    double s = 0.0;
    for (int j = threadIdx.x; j < nb; j += 256) s += partial[j];
    __shared__ double sh[8];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 8) {
        s = sh[threadIdx.x];
        for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffu, s, o);
        if (threadIdx.x == 0) out[0] = s;
    }
}

int stream_grid(size_t n)
{
    size_t blocks = (n / 2 + 255) / 256;
    size_t cap = (size_t)ctx().sm_count * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

}  // namespace

// device-side dot whose result stays on the device (used by the CG driver)
int fdb_vec_dot_device(size_t n, const double *x, const double *y, double *d_out)
{
    Context &c = ctx();
    int nb = stream_grid(n);
    if (nb > DOT_BLOCKS_MAX) nb = DOT_BLOCKS_MAX;
    k_dot_partial<<<nb, 256, 0, c.stream>>>(n, x, y, c.reduce_scratch);
    FDB_LAUNCH_CHECK();
    k_dot_final<<<1, 256, 0, c.stream>>>(nb, c.reduce_scratch, d_out);
    FDB_LAUNCH_CHECK();
    return 0;
}

extern "C" {

int fdb_dat_zero_nodes(double *dat, int cdim, const fdb_int *nodes, fdb_int n)
{
    if (require_init()) return 1;
    if (n <= 0) return 0;
    int blocks = (int)std::min<long long>(((long long)n * cdim + 255) / 256, ctx().sm_count * 8);
    k_zero_nodes<<<blocks, 256, 0, ctx().stream>>>(dat, cdim, nodes, n);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_dat_set_nodes(double *dat, const double *src, int cdim, const fdb_int *nodes, fdb_int n)
{
    if (require_init()) return 1;
    if (n <= 0) return 0;
    int blocks = (int)std::min<long long>(((long long)n * cdim + 255) / 256, ctx().sm_count * 8);
    k_set_nodes<<<blocks, 256, 0, ctx().stream>>>(dat, src, 0.0, cdim, nodes, n);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_dat_set_nodes_scalar(double *dat, double value, int cdim, const fdb_int *nodes, fdb_int n)
{
    if (require_init()) return 1;
    if (n <= 0) return 0;
    int blocks = (int)std::min<long long>(((long long)n * cdim + 255) / 256, ctx().sm_count * 8);
    k_set_nodes<<<blocks, 256, 0, ctx().stream>>>(dat, nullptr, value, cdim, nodes, n);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_vec_axpy(size_t n, double a, const double *x, double *y)
{
    if (require_init()) return 1;
    k_stream<0><<<stream_grid(n), 256, 0, ctx().stream>>>(n, a, x, y, nullptr);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_vec_aypx(size_t n, double a, const double *x, double *y)
{
    if (require_init()) return 1;
    k_stream<1><<<stream_grid(n), 256, 0, ctx().stream>>>(n, a, x, y, nullptr);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_vec_scale(size_t n, double a, double *x)
{
    if (require_init()) return 1;
    k_stream<2><<<stream_grid(n), 256, 0, ctx().stream>>>(n, a, nullptr, x, nullptr);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_vec_fill(size_t n, double a, double *x)
{
    if (require_init()) return 1;
    if (n == 0) return 0;
    k_fill<<<stream_grid(n), 256, 0, ctx().stream>>>(n, a, x);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_vec_gather(size_t n, const fdb_int *idx, const double *src, double *dst)    /* dst[j] = src[idx[j]] */
{
    if (require_init()) return 1;
    if (n == 0) return 0;
    k_gather<<<stream_grid(n), 256, 0, ctx().stream>>>(n, idx, src, dst);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_vec_scatter(size_t n, const fdb_int *idx, const double *src, double *dst)   /* dst[idx[j]] = src[j] */
{
    if (require_init()) return 1;
    if (n == 0) return 0;
    k_scatter<<<stream_grid(n), 256, 0, ctx().stream>>>(n, idx, src, dst);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_vec_pointwise_mult(size_t n, const double *x, const double *y, double *w)
{
    if (require_init()) return 1;
    k_stream<3><<<stream_grid(n), 256, 0, ctx().stream>>>(n, 0.0, x, const_cast<double *>(y), w);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_vec_chebyshev(size_t n, double c_d, double c_z, const double *b, const double *ax, const double *dinv,
                      double *d, double *x)
{
    if (require_init()) return 1;
    if (n == 0) return 0;
    k_chebyshev<<<stream_grid(2 * n), 256, 0, ctx().stream>>>(n, c_d, c_z, b, ax, dinv, d, x);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_vec_dot(size_t n, const double *x, const double *y, double *out)
{
    if (require_init()) return 1;
    Context &c = ctx();
    double *d_out = c.reduce_scratch + 2048;
    if (fdb_vec_dot_device(n, x, y, d_out)) return 1;
    FDB_CUDA(cudaMemcpyAsync(c.reduce_host, d_out, sizeof(double), cudaMemcpyDeviceToHost, c.stream));
    FDB_CUDA(cudaStreamSynchronize(c.stream));
    *out = c.reduce_host[0];
    return 0;
}

}  // extern "C"
