// Device CSR matrices: sparsity construction (K7 / A8), zero, BC lgmaps and
// diagonal (A6 / A10), SpMV, export.
//
// Reference semantics:
//   * pattern = union over cells (and layers) of rowmap x colmap, the diagonal is
//     always allocated, all entries zero-filled so later adds never allocate
//     (pyop2/sparsity.pyx:106-160, 198-204, 347-373; pyop2/types/mat.py:741-804)
//   * Dirichlet rows/columns are removed by local-to-global maps whose entries
//     are -1: MatSetValuesLocal drops negative indices
//     (firedrake/functionspaceimpl.py:854-926, pyop2/parloop.py:279-314)
//   * afterwards the diagonal of constrained rows is set
//     (pyop2/types/mat.py:897-937 set_local_diagonal_entries)
// Construction: (row, col) keys of every cell -> thrust sort + unique -> CSR
// with sorted columns per row.  The element-tensor scatter finds a position by
// binary search inside the row (the cost model of PETSc's MatSetValues, here
// in parallel and hitting L2).
#include <stdlib.h>

#include <thrust/device_ptr.h>
#include <thrust/execution_policy.h>
#include <thrust/scan.h>
#include <thrust/sort.h>
#include <thrust/unique.h>

#include "common.cuh"

using namespace fdb;

struct fdb_mat_s {
    fdb_int nrows = 0;
    long long nnz = 0;
    long long *d_rowptr = nullptr;
    fdb_int *d_colidx = nullptr;
    double *d_vals = nullptr;
    fdb_int *d_row_lgmap = nullptr, *d_col_lgmap = nullptr;   // NULL = identity
    // within-row position of every (test dof i, trial dof j) pair of a cell,
    // per column and layer class (bottom / interior / top): extruded numbering
    // is translation invariant along a column, so interior layers share one
    // table.  rank[((col*nvar + v)*arity + j)*arity + i].  NULL: binary search.
    unsigned short *d_rank = nullptr;
    int nvar = 0, arity = 0, nlay = 0;
    // block size (BAIJ-like): rowptr/colidx address NODES, vals holds bs*bs doubles
    // per stored block, row-major inside the block; lgmaps are dof-level (nrows*bs)
    int bs = 1;
    bool shallow = false;      // scalar view sharing the pattern of a blocked matrix
    // blocked matrices zero LAZILY: MatZeroEntries followed by the A (x) I assembly of the Helmholtz
    // family then costs one streaming WRITE of the blocks (fdb_mat_scalar_view_end) instead of a
    // memset plus a read-modify-write pass over them (35 GB each for config 4 at 32^3)
    bool zero_pending = false;
    // scratch of the A (x) I assembly (fdb_mat_scalar_view_*), kept across assemblies: allocating and
    // freeing 3.6 GB per assembly cost several ms of the 26 ms config-4 assembly
    double *d_view_vals = nullptr;
    fdb_int *d_view_rlg = nullptr, *d_view_clg = nullptr;
};

static int materialise_zero(fdb_mat_s *m)
{
    if (m->zero_pending) {
        FDB_CUDA(cudaMemsetAsync(m->d_vals, 0, sizeof(double) * (size_t)m->nnz * m->bs * m->bs, ctx().stream));
        m->zero_pending = false;
    }
    return 0;
}

namespace {

__global__ void k_gen_keys(const fdb_int *__restrict__ map, const fdb_int *__restrict__ off,
                           fdb_int ncols, int arity, int nlay, fdb_int nrows,
                           unsigned long long *__restrict__ keys)
{
    const long long per_cell = (long long)arity * arity;
    const long long total = (long long)ncols * nlay * per_cell;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i < total; i += (long long)gridDim.x * blockDim.x) {
        long long cell = i / per_cell;
        int e = (int)(i - cell * per_cell);
        int a = e / arity, b = e - a * arity;
        fdb_int c = (fdb_int)(cell / nlay);
        int l = (int)(cell - (long long)c * nlay);
        unsigned long long r = map[(long long)c * arity + a] + (off ? off[a] * l : 0);
        unsigned long long cc = map[(long long)c * arity + b] + (off ? off[b] * l : 0);
        keys[i] = r * (unsigned long long)nrows + cc;
    }
    // diagonal entries
    long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; j < nrows; j += (long long)gridDim.x * blockDim.x)
        keys[total + j] = (unsigned long long)j * nrows + j;
}

__global__ void k_count_rows(const unsigned long long *__restrict__ keys, long long n, fdb_int nrows,
                             long long *__restrict__ counts, fdb_int *__restrict__ colidx)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i < n; i += (long long)gridDim.x * blockDim.x) {
        unsigned long long k = keys[i];
        unsigned long long r = k / (unsigned long long)nrows;
        colidx[i] = (fdb_int)(k - r * nrows);
        atomicAdd((unsigned long long *)&counts[r], 1ull);
    }
}

__global__ void k_build_rank(const fdb_int *__restrict__ map, const fdb_int *__restrict__ off,
                             fdb_int ncols, int arity, int nlay, int nvar,
                             const long long *__restrict__ rowptr, const fdb_int *__restrict__ colidx,
                             unsigned short *__restrict__ rank)
{
    const long long per_col = (long long)nvar * arity * arity;
    const long long total = (long long)ncols * per_col;
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; t < total; t += (long long)gridDim.x * blockDim.x) {
        const fdb_int c = (fdb_int)(t / per_col);
        int e = (int)(t - (long long)c * per_col);
        const int v = e / (arity * arity);
        e -= v * arity * arity;
        const int j = e / arity, i = e - j * arity;
        // representative layer of the class
        const int layer = nlay < 3 ? v : (v == 0 ? 0 : (v == 1 ? 1 : nlay - 1));
        const fdb_int r = map[(long long)c * arity + i] + (off ? off[i] * layer : 0);
        const fdb_int cc = map[(long long)c * arity + j] + (off ? off[j] * layer : 0);
        long long lo = rowptr[r], hi = rowptr[r + 1];
        const long long base = lo;
        while (hi - lo > 1) {
            long long mid = (lo + hi) >> 1;
            if (colidx[mid] <= cc) lo = mid; else hi = mid;
        }
        rank[t] = (unsigned short)(lo - base);
    }
}

__global__ void k_spmv(fdb_int nrows, const long long *__restrict__ rowptr,
                       const fdb_int *__restrict__ colidx, const double *__restrict__ vals,
                       const double *__restrict__ x, double *__restrict__ y)
{
    // one warp per row
    long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long r = w; r < nrows; r += nw) {
        double s = 0.0;
        for (long long k = rowptr[r] + lane; k < rowptr[r + 1]; k += 32) s = fma(vals[k], x[colidx[k]], s);
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) y[r] = s;
    }
}

// d[r] = A[r][r] (0 where the pattern has no diagonal entry), scalar matrices
__global__ void k_get_diag(const long long *__restrict__ rowptr, const fdb_int *__restrict__ colidx,
                           const double *__restrict__ vals, fdb_int n, double *__restrict__ d)
{
    for (fdb_int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        long long lo = rowptr[r], hi = rowptr[r + 1];
        if (hi == lo) {
            d[r] = 0.0;
            continue;
        }
        while (hi - lo > 1) {
            long long mid = (lo + hi) >> 1;
            if (colidx[mid] <= r) lo = mid; else hi = mid;
        }
        d[r] = colidx[lo] == r ? vals[lo] : 0.0;
    }
}

__global__ void k_set_diag(const long long *__restrict__ rowptr, const fdb_int *__restrict__ colidx,
                           double *__restrict__ vals, const fdb_int *__restrict__ rows, fdb_int n,
                           double value)
{
    fdb_int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fdb_int r = rows[i];
    long long lo = rowptr[r], hi = rowptr[r + 1];
    while (hi - lo > 1) {
        long long mid = (lo + hi) >> 1;
        if (colidx[mid] <= r) lo = mid; else hi = mid;
    }
    if (colidx[lo] == r) vals[lo] = value;
}

// blocked SpMV: one warp per node row, bs partial sums per lane
template <int BS>
__global__ void k_spmv_blocked(fdb_int nrows, const long long *__restrict__ rowptr,
                               const fdb_int *__restrict__ colidx, const double *__restrict__ vals,
                               const double *__restrict__ x, double *__restrict__ y)
{
    long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long r = w; r < nrows; r += nw) {
        double s[BS];
#pragma unroll
        for (int a = 0; a < BS; a++) s[a] = 0.0;
        for (long long k = rowptr[r] + lane; k < rowptr[r + 1]; k += 32) {
            const double *blk = vals + k * (BS * BS);
            const double *xc = x + (long long)colidx[k] * BS;
#pragma unroll
            for (int a = 0; a < BS; a++)
#pragma unroll
                for (int b = 0; b < BS; b++) s[a] = fma(blk[a * BS + b], xc[b], s[a]);
        }
#pragma unroll
        for (int a = 0; a < BS; a++) {
            for (int o = 16; o > 0; o >>= 1) s[a] += __shfl_xor_sync(0xffffffffu, s[a], o);
            if (lane == 0) y[r * BS + a] = s[a];
        }
    }
}

// diagonal of constrained node rows: component idx, or every component when idx < 0
__global__ void k_set_diag_blocked(const long long *__restrict__ rowptr, const fdb_int *__restrict__ colidx,
                                   double *__restrict__ vals, const fdb_int *__restrict__ rows, fdb_int n,
                                   double value, int bs, int idx)
{
    fdb_int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fdb_int r = rows[i];
    long long lo = rowptr[r], hi = rowptr[r + 1];
    while (hi - lo > 1) {
        long long mid = (lo + hi) >> 1;
        if (colidx[mid] <= r) lo = mid; else hi = mid;
    }
    if (colidx[lo] != r) return;
    double *blk = vals + lo * bs * bs;
    for (int a = 0; a < bs; a++)
        if (idx < 0 || idx == a) blk[a * bs + a] = value;
}

// node-level lgmap of a dof-level one: a node is masked when ALL its components are;
// *mixed is raised when only some are (component BC: not expressible per node)
__global__ void k_node_lgmap(const fdb_int *__restrict__ dof_lg, fdb_int nnodes, int bs,
                             fdb_int *__restrict__ node_lg, int *__restrict__ mixed)
{
    fdb_int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nnodes) return;
    int masked = 0;
    for (int a = 0; a < bs; a++) masked += dof_lg[(long long)r * bs + a] < 0;
    node_lg[r] = masked == bs ? -1 : r;
    if (masked != 0 && masked != bs) *mixed = 1;
}

// blocked = scalar (x) I_bs (the blocked matrix was zero: plain coalesced stores, no read).
// 16-byte stores, block size folded at compile time (a 35 GB stream for config 4 at 32^3).
template <int BS>
__global__ void __launch_bounds__(256) k_store_scalar_blocks(long long n2, const double *__restrict__ sv,
                                                             double2 *__restrict__ bv)
{
    constexpr int BB = BS * BS;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i < n2; i += (long long)gridDim.x * blockDim.x) {
        const long long e0 = 2 * i, e1 = e0 + 1;
        const long long k0 = e0 / BB, k1 = e1 / BB;
        const int r0 = (int)(e0 - k0 * BB), r1 = (int)(e1 - k1 * BB);
        double2 v;
        v.x = (r0 % (BS + 1) == 0) ? __ldg(sv + k0) : 0.0;
        v.y = (r1 % (BS + 1) == 0) ? __ldg(sv + k1) : 0.0;
        bv[i] = v;
    }
}

// blocked += scalar (x) I_bs on an identical node pattern
__global__ void k_add_scalar_blocks(long long nnz, int bs, const double *__restrict__ sv, double *__restrict__ bv)
{
    long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; k < nnz; k += (long long)gridDim.x * blockDim.x) {
        const double v = sv[k];
        if (v == 0.0) continue;
        double *blk = bv + k * bs * bs;
        for (int a = 0; a < bs; a++) blk[a * bs + a] += v;
    }
}

int grid1d(long long n)
{
    long long b = (n + 255) / 256;
    long long cap = (long long)ctx().sm_count * 16;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
}

}  // namespace

// used by the element-tensor scatter in action_hex.cu / tri_p1.cu
int fdb_mat_rank_table(fdb_mat_t m, const unsigned short **rank, int *nvar)
{
    *rank = m->d_rank;
    *nvar = m->nvar;
    return 0;
}

int fdb_mat_block_size(fdb_mat_t m, int *bs)
{
    *bs = m->bs;
    return 0;
}

int fdb_mat_rows(fdb_mat_t m, fdb_int *nrows)
{
    *nrows = m->nrows;
    return 0;
}

// Scalar view of a blocked matrix for forms whose element tensor is A_scalar (x) I
// (inner(grad u, grad v) + inner(u, v) on a vector space: the off-diagonal
// component blocks vanish identically, SURVEY.md section 8d).  The view shares the
// pattern and the rank table, owns a zeroed value array and node-level lgmaps;
// ..._end adds it into the diagonal of every block and releases it.
int fdb_mat_scalar_view_begin(fdb_mat_t mb, fdb_mat_t *view)
{
    if (require_init()) return 1;
    cudaStream_t st = ctx().stream;
    fdb_mat_s *v = new fdb_mat_s(*mb);
    v->shallow = true;
    v->zero_pending = false;
    v->bs = 1;
    v->d_row_lgmap = v->d_col_lgmap = nullptr;
    v->d_view_vals = nullptr;
    v->d_view_rlg = v->d_view_clg = nullptr;
    if (!mb->d_view_vals) FDB_CUDA(cudaMalloc(&mb->d_view_vals, sizeof(double) * (size_t)mb->nnz));
    v->d_vals = mb->d_view_vals;
    FDB_CUDA(cudaMemsetAsync(v->d_vals, 0, sizeof(double) * (size_t)mb->nnz, st));
    int *d_mixed = nullptr;
    FDB_CUDA(cudaMalloc(&d_mixed, sizeof(int)));
    FDB_CUDA(cudaMemsetAsync(d_mixed, 0, sizeof(int), st));
    const fdb_int *src[2] = {mb->d_row_lgmap, mb->d_col_lgmap};
    fdb_int **dst[2] = {&v->d_row_lgmap, &v->d_col_lgmap};
    fdb_int **keep[2] = {&mb->d_view_rlg, &mb->d_view_clg};
    for (int i = 0; i < 2; i++) {
        if (!src[i]) continue;
        if (!*keep[i]) FDB_CUDA(cudaMalloc(keep[i], sizeof(fdb_int) * (size_t)mb->nrows));
        *dst[i] = *keep[i];
        k_node_lgmap<<<(mb->nrows + 255) / 256, 256, 0, st>>>(src[i], mb->nrows, mb->bs, *dst[i], d_mixed);
        FDB_LAUNCH_CHECK();
    }
    int mixed = 0;
    FDB_CUDA(cudaMemcpyAsync(&mixed, d_mixed, sizeof(int), cudaMemcpyDeviceToHost, st));
    FDB_CUDA(cudaStreamSynchronize(st));
    cudaFree(d_mixed);
    if (mixed) {
        set_error("blocked matrix assembly: Dirichlet conditions on single components are not supported "
                  "by the A (x) I fast path (use the generic wrapper)");
        delete v;
        return 1;
    }
    *view = v;
    return 0;
}

int fdb_mat_scalar_view_end(fdb_mat_t mb, fdb_mat_t view)
{
    cudaStream_t st = ctx().stream;
    if (mb->zero_pending) {
        const long long n = mb->nnz * mb->bs * mb->bs;
        const long long n2 = n / 2;
        double2 *out2 = reinterpret_cast<double2 *>(mb->d_vals);
        const int g = grid1d(n2);
        switch (mb->bs) {
        case 2: k_store_scalar_blocks<2><<<g, 256, 0, st>>>(n2, view->d_vals, out2); break;
        case 3: k_store_scalar_blocks<3><<<g, 256, 0, st>>>(n2, view->d_vals, out2); break;
        case 4: k_store_scalar_blocks<4><<<g, 256, 0, st>>>(n2, view->d_vals, out2); break;
        default:
            // other block sizes: zero, then add
            FDB_CUDA(cudaMemsetAsync(mb->d_vals, 0, sizeof(double) * (size_t)n, st));
            k_add_scalar_blocks<<<grid1d(mb->nnz), 256, 0, st>>>(mb->nnz, mb->bs, view->d_vals, mb->d_vals);
        }
        if (mb->bs >= 2 && mb->bs <= 4 && (n & 1)) {
            // odd total (bs = 3, odd nnz): the last entry is the (bs-1, bs-1) diagonal of the last block
            FDB_CUDA(cudaMemcpyAsync(mb->d_vals + (n - 1), view->d_vals + (mb->nnz - 1), sizeof(double),
                                     cudaMemcpyDeviceToDevice, st));
        }
        mb->zero_pending = false;
    } else {
        k_add_scalar_blocks<<<grid1d(mb->nnz), 256, 0, st>>>(mb->nnz, mb->bs, view->d_vals, mb->d_vals);
    }
    FDB_LAUNCH_CHECK();
    delete view;          // its buffers belong to the blocked matrix (kept for the next assembly)
    return 0;
}

int fdb_mat_device_view(fdb_mat_t m, const long long **rowptr, const fdb_int **colidx, double **vals,
                        const fdb_int **row_lg, const fdb_int **col_lg)
{
    if (materialise_zero(m)) return 1;
    *rowptr = m->d_rowptr;
    *colidx = m->d_colidx;
    *vals = m->d_vals;
    *row_lg = m->d_row_lgmap;
    *col_lg = m->d_col_lgmap;
    return 0;
}

extern "C" {

int fdb_mat_create(fdb_int nrows, const fdb_int *map_host, fdb_int ncolumns, int arity,
                   const fdb_int *offset_host, int nlayers, fdb_mat_t *out)
{
    return fdb_mat_create_blocked(nrows, map_host, ncolumns, arity, offset_host, nlayers, 1, out);
}

int fdb_mat_create_blocked(fdb_int nrows, const fdb_int *map_host, fdb_int ncolumns, int arity,
                           const fdb_int *offset_host, int nlayers, int bs, fdb_mat_t *out)
{
    if (require_init()) return 1;
    if (bs < 1 || bs > 8) {
        set_error("fdb_mat_create_blocked: block size %d outside 1..8", bs);
        return 1;
    }
    if (nlayers < 1 || arity < 1 || nrows < 1) {
        set_error("fdb_mat_create: bad sizes");
        return 1;
    }
    cudaStream_t st = ctx().stream;
    const long long npairs = (long long)ncolumns * nlayers * arity * arity + nrows;
    size_t free_b = 0, total_b = 0;
    FDB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    // keys + radix-sort scratch + CSR
    if ((double)npairs * 8.0 * 2.3 > (double)free_b * 0.9) {
        set_error("fdb_mat_create: %lld (row,col) pairs need %.1f GB to sort, %.1f GB free: assemble "
                  "matrix-free instead (SURVEY.md fact 5)",
                  npairs, npairs * 8.0 * 2.3 / 1e9, free_b / 1e9);
        return 1;
    }
    fdb_int *d_map = nullptr, *d_off = nullptr;
    unsigned long long *keys = nullptr;
    FDB_CUDA(cudaMalloc(&d_map, sizeof(fdb_int) * (size_t)ncolumns * arity));
    FDB_CUDA(cudaMemcpyAsync(d_map, map_host, sizeof(fdb_int) * (size_t)ncolumns * arity,
                             cudaMemcpyHostToDevice, st));
    if (offset_host) {
        FDB_CUDA(cudaMalloc(&d_off, sizeof(fdb_int) * arity));
        FDB_CUDA(cudaMemcpyAsync(d_off, offset_host, sizeof(fdb_int) * arity, cudaMemcpyHostToDevice, st));
    }
    FDB_CUDA(cudaMalloc(&keys, sizeof(unsigned long long) * (size_t)npairs));
    k_gen_keys<<<grid1d(npairs), 256, 0, st>>>(d_map, d_off, ncolumns, arity, nlayers, nrows, keys);
    FDB_LAUNCH_CHECK();
    long long nnz = 0;
    try {
        thrust::device_ptr<unsigned long long> kp(keys);
        thrust::sort(thrust::cuda::par.on(st), kp, kp + npairs);
        nnz = thrust::unique(thrust::cuda::par.on(st), kp, kp + npairs) - kp;
    } catch (const std::exception &e) {
        set_error("fdb_mat_create: thrust failed: %s", e.what());
        cudaFree(keys);
        cudaFree(d_map);
        cudaFree(d_off);
        return 1;
    }
    fdb_mat_s *m = new fdb_mat_s;
    m->nrows = nrows;
    m->nnz = nnz;
    m->bs = bs;
    const size_t bb = (size_t)bs * bs;
    FDB_CUDA(cudaMalloc(&m->d_rowptr, sizeof(long long) * ((size_t)nrows + 1)));
    FDB_CUDA(cudaMalloc(&m->d_colidx, sizeof(fdb_int) * (size_t)nnz));
    if (cudaMalloc(&m->d_vals, sizeof(double) * (size_t)nnz * bb) != cudaSuccess) {
        set_error("fdb_mat_create: %.1f GB of values do not fit (nnz %lld, block size %d)",
                  (double)nnz * bb * 8.0 / 1e9, nnz, bs);
        cudaFree(m->d_rowptr);
        cudaFree(m->d_colidx);
        cudaFree(keys);
        cudaFree(d_map);
        cudaFree(d_off);
        delete m;
        return 1;
    }
    FDB_CUDA(cudaMemsetAsync(m->d_rowptr, 0, sizeof(long long) * ((size_t)nrows + 1), st));
    k_count_rows<<<grid1d(nnz), 256, 0, st>>>(keys, nnz, nrows, m->d_rowptr + 1, m->d_colidx);
    FDB_LAUNCH_CHECK();
    try {
        thrust::device_ptr<long long> rp(m->d_rowptr);
        thrust::inclusive_scan(thrust::cuda::par.on(st), rp, rp + nrows + 1, rp);
    } catch (const std::exception &e) {
        set_error("fdb_mat_create: scan failed: %s", e.what());
        return 1;
    }
    FDB_CUDA(cudaMemsetAsync(m->d_vals, 0, sizeof(double) * (size_t)nnz * bb, st));
    FDB_CUDA(cudaStreamSynchronize(st));
    cudaFree(keys);
    keys = nullptr;
    // position table for the element-tensor scatter (skipped when it would not fit)
    const int nlay = nlayers;
    m->arity = arity;
    m->nlay = nlay;
    m->nvar = nlay < 3 ? nlay : 3;
    {
        const double tab_bytes = (double)ncolumns * m->nvar * arity * arity * 2.0;
        FDB_CUDA(cudaMemGetInfo(&free_b, &total_b));
        static const bool use_rank = !(getenv("FDB_MAT_NO_RANK") && atoi(getenv("FDB_MAT_NO_RANK")));
        if (use_rank && tab_bytes < 0.25 * (double)free_b && tab_bytes < 8e9) {
            FDB_CUDA(cudaMalloc(&m->d_rank, (size_t)tab_bytes));
            k_build_rank<<<grid1d((long long)(tab_bytes / 2)), 256, 0, st>>>(
                d_map, d_off, ncolumns, arity, nlay, m->nvar, m->d_rowptr, m->d_colidx, m->d_rank);
            FDB_LAUNCH_CHECK();
            FDB_CUDA(cudaStreamSynchronize(st));
        }
    }
    cudaFree(d_map);
    if (d_off) cudaFree(d_off);
    *out = m;
    return 0;
}

int fdb_mat_destroy(fdb_mat_t m)
{
    if (!m) return 0;
    if (ctx().ready) {
        cudaStreamSynchronize(ctx().stream);
        cudaFree(m->d_rowptr);
        cudaFree(m->d_colidx);
        cudaFree(m->d_vals);
        cudaFree(m->d_row_lgmap);
        cudaFree(m->d_col_lgmap);
        if (m->d_rank) cudaFree(m->d_rank);
        if (m->d_view_vals) cudaFree(m->d_view_vals);
        if (m->d_view_rlg) cudaFree(m->d_view_rlg);
        if (m->d_view_clg) cudaFree(m->d_view_clg);
    }
    delete m;
    return 0;
}

int fdb_mat_nnz(fdb_mat_t m, long long *nnz, fdb_int *nrows)
{
    if (nnz) *nnz = m->nnz;
    if (nrows) *nrows = m->nrows;
    return 0;
}

int fdb_mat_zero(fdb_mat_t m)
{
    if (require_init()) return 1;
    if (m->bs > 1) {
        m->zero_pending = true;      // materialised by the next reader, or overwritten by the assembly
        return 0;
    }
    FDB_CUDA(cudaMemsetAsync(m->d_vals, 0, sizeof(double) * (size_t)m->nnz * m->bs * m->bs, ctx().stream));
    return 0;
}

int fdb_mat_get_csr(fdb_mat_t m, long long *rowptr, fdb_int *colidx, double *vals)
{
    if (require_init()) return 1;
    if (materialise_zero(m)) return 1;
    cudaStream_t st = ctx().stream;
    if (rowptr)
        FDB_CUDA(cudaMemcpyAsync(rowptr, m->d_rowptr, sizeof(long long) * ((size_t)m->nrows + 1),
                                 cudaMemcpyDeviceToHost, st));
    if (colidx)
        FDB_CUDA(cudaMemcpyAsync(colidx, m->d_colidx, sizeof(fdb_int) * (size_t)m->nnz,
                                 cudaMemcpyDeviceToHost, st));
    if (vals)
        FDB_CUDA(cudaMemcpyAsync(vals, m->d_vals, sizeof(double) * (size_t)m->nnz * m->bs * m->bs,
                                 cudaMemcpyDeviceToHost, st));
    FDB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int fdb_mat_set_lgmaps(fdb_mat_t m, const fdb_int *row_lgmap_host, const fdb_int *col_lgmap_host)
{
    if (require_init()) return 1;
    cudaStream_t st = ctx().stream;
    const fdb_int *src[2] = {row_lgmap_host, col_lgmap_host};
    fdb_int **dst[2] = {&m->d_row_lgmap, &m->d_col_lgmap};
    for (int i = 0; i < 2; i++) {
        if (!src[i]) {
            if (*dst[i]) {
                FDB_CUDA(cudaStreamSynchronize(st));
                cudaFree(*dst[i]);
                *dst[i] = nullptr;
            }
            continue;
        }
        const size_t nlg = (size_t)m->nrows * m->bs;      // dof-level for blocked matrices
        if (!*dst[i]) FDB_CUDA(cudaMalloc(dst[i], sizeof(fdb_int) * nlg));
        FDB_CUDA(cudaMemcpyAsync(*dst[i], src[i], sizeof(fdb_int) * nlg, cudaMemcpyHostToDevice, st));
    }
    FDB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int fdb_mat_set_diagonal(fdb_mat_t m, const fdb_int *rows_host, fdb_int n, double value)
{
    return fdb_mat_set_diagonal_blocked(m, rows_host, n, value, -1);
}

int fdb_mat_set_diagonal_blocked(fdb_mat_t m, const fdb_int *rows_host, fdb_int n, double value, int idx)
{
    if (require_init()) return 1;
    if (n <= 0) return 0;
    if (idx >= m->bs) {
        set_error("fdb_mat_set_diagonal_blocked: component %d >= block size %d", idx, m->bs);
        return 1;
    }
    if (materialise_zero(m)) return 1;
    cudaStream_t st = ctx().stream;
    fdb_int *d_rows = nullptr;
    FDB_CUDA(cudaMalloc(&d_rows, sizeof(fdb_int) * (size_t)n));
    FDB_CUDA(cudaMemcpyAsync(d_rows, rows_host, sizeof(fdb_int) * (size_t)n, cudaMemcpyHostToDevice, st));
    if (m->bs == 1)
        k_set_diag<<<(n + 255) / 256, 256, 0, st>>>(m->d_rowptr, m->d_colidx, m->d_vals, d_rows, n, value);
    else
        k_set_diag_blocked<<<(n + 255) / 256, 256, 0, st>>>(m->d_rowptr, m->d_colidx, m->d_vals, d_rows, n,
                                                           value, m->bs, idx);
    FDB_LAUNCH_CHECK();
    FDB_CUDA(cudaStreamSynchronize(st));
    cudaFree(d_rows);
    return 0;
}

int fdb_mat_get_diagonal(fdb_mat_t m, double *d)
{
    if (require_init()) return 1;
    if (m->bs != 1) {
        set_error("fdb_mat_get_diagonal: scalar matrices only (block size %d)", m->bs);
        return 1;
    }
    if (materialise_zero(m)) return 1;
    if (m->nrows <= 0) return 0;
    k_get_diag<<<grid1d(m->nrows), 256, 0, ctx().stream>>>(m->d_rowptr, m->d_colidx, m->d_vals, m->nrows, d);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_mat_mult(fdb_mat_t m, const double *x, double *y)
{
    if (require_init()) return 1;
    if (materialise_zero(m)) return 1;
    long long threads = (long long)m->nrows * 32;
    cudaStream_t st = ctx().stream;
    const int g = grid1d(threads);
    switch (m->bs) {
    case 1: k_spmv<<<g, 256, 0, st>>>(m->nrows, m->d_rowptr, m->d_colidx, m->d_vals, x, y); break;
    case 2: k_spmv_blocked<2><<<g, 256, 0, st>>>(m->nrows, m->d_rowptr, m->d_colidx, m->d_vals, x, y); break;
    case 3: k_spmv_blocked<3><<<g, 256, 0, st>>>(m->nrows, m->d_rowptr, m->d_colidx, m->d_vals, x, y); break;
    case 4: k_spmv_blocked<4><<<g, 256, 0, st>>>(m->nrows, m->d_rowptr, m->d_colidx, m->d_vals, x, y); break;
    default:
        set_error("fdb_mat_mult: block size %d not instantiated (1..4)", m->bs);
        return 1;
    }
    FDB_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
