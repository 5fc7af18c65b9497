// Transfers between CG1 (vertex values) and the HDiv-trace space of degree k - 1 (k = 2, 3) on the same hex cells:
// FDB_FORM_TRACE_PROLONG and FDB_FORM_TRACE_RESTRICT, the level transfers of the two-level GTMG cycle for the
// hybridised mixed Poisson trace system (DESIGN.md section 4.24).
//
//   prolong   lambda  = P c                 WRITE into the trace space
//   restrict  c      += P^T (w o lambda)    INC into CG1 (atomic or coloured)
//
// Trace dof t of a cell (face 2d + s, GL indices t0, t1 along the two tangential axes e0 < e1) is the value at its
// face point of the trilinear interpolant of the cell's 8 vertex values: the 4 vertices with a_d = s, weighted by
// P1[t0][a_e0] * P1[t1][a_e1], P1 (k, 2) the CG1 basis at the k Gauss-Legendre points.  Metric-free.
// w = 1 / (cells holding the trace dof), so that the restriction is exactly P^T.
//
// A shared face is written by both of its cells.  Each cell computes the four products weight * c_v and sums them in
// ascending order of the GLOBAL vertex number, so both sides store bitwise the same value whatever the local vertex
// order of either cell, and the result does not depend on which write lands last.
//
// Layout: prolong runs one thread per (cell, trace dof), restrict one thread per (cell, vertex), which sums its 3k^2
// trace dofs in a fixed order.  No shared memory: the operations per byte are few and these kernels are judged on
// bandwidth.
#include "common.cuh"

namespace {

enum { TT_PROLONG = 0, TT_RESTRICT = 1 };

template <int K>
struct TraceParams {
    double *out;
    const double *in, *w;             // w: restrict only, one value per trace dof
    const fdb_int *mapt, *mapv;       // trace (6K^2) and CG1 (8) rows per column
    const fdb_int *offt, *offv;       // their layer offsets (zeros on native hexes)
    const fdb_int *collist;           // columns to visit (subset or colour) or NULL = col0 + i
    int col0, ncols;
    int nlay_items, lay_first, lay_step;   // layers lay_first + i * lay_step, i < nlay_items
    double P[K * 2];                  // CG1 basis at the GL points: P[q * 2 + a]
};

constexpr int THREADS = 256;

template <int K, int KIND, bool ATOMIC>
__global__ void __launch_bounds__(THREADS)
trace_transfer_kernel(const __grid_constant__ TraceParams<K> T)
{
    constexpr int NT = 6 * K * K;
    constexpr int PER = KIND == TT_PROLONG ? NT : 8;          // threads per cell
    const long long nunits = (long long)T.ncols * T.nlay_items;
    const long long nthr = nunits * PER;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nthr;
         i += (long long)gridDim.x * blockDim.x) {
        const long long unit = i / PER;
        const int l = (int)(i - unit * PER);
        const int ci = (int)(unit / T.nlay_items);
        const int layer = T.lay_first + (int)(unit - (long long)ci * T.nlay_items) * T.lay_step;
        const int col = T.collist ? __ldg(T.collist + ci) : T.col0 + ci;
        const fdb_int *rowt = T.mapt + (long long)col * NT;
        const fdb_int *rowv = T.mapv + (long long)col * 8;
        if (KIND == TT_PROLONG) {
            const int f = l / (K * K), r = l - f * K * K;
            const int d = f >> 1, s = f & 1;
            const int t0 = r / K, t1 = r - t0 * K;
            const int e0 = d == 0 ? 1 : 0, e1 = d == 2 ? 1 : 2;
            long long g[4];
            double v[4];
#pragma unroll
            for (int b = 0; b < 4; b++) {
                // local vertex (a0 * 2 + a1) * 2 + a2: axis e holds bit 2 - e
                const int lv = (s << (2 - d)) | ((b >> 1) << (2 - e0)) | ((b & 1) << (2 - e1));
                g[b] = __ldg(rowv + lv) + (long long)__ldg(T.offv + lv) * layer;
                v[b] = (T.P[t0 * 2 + (b >> 1)] * T.P[t1 * 2 + (b & 1)]) * __ldg(T.in + g[b]);
            }
            // a sorting network on the global vertex numbers: the canonical summation order
#define FDB_TT_SWAP(x, y)                                                                                      \
    if (g[y] < g[x]) {                                                                                       \
        const long long tg = g[x]; g[x] = g[y]; g[y] = tg;                                                   \
        const double tv = v[x]; v[x] = v[y]; v[y] = tv;                                                      \
    }
            FDB_TT_SWAP(0, 1)
            FDB_TT_SWAP(2, 3)
            FDB_TT_SWAP(0, 2)
            FDB_TT_SWAP(1, 3)
            FDB_TT_SWAP(1, 2)
#undef FDB_TT_SWAP
            const long long gt = __ldg(rowt + l) + (long long)__ldg(T.offt + l) * layer;
            T.out[gt] = ((v[0] + v[1]) + v[2]) + v[3];
        } else {
            auto a = [l](int e) { return (l >> (2 - e)) & 1; };     // the vertex's index along axis e
            double acc = 0.0;
#pragma unroll
            for (int d = 0; d < 3; d++) {
                const int e0 = d == 0 ? 1 : 0, e1 = d == 2 ? 1 : 2;
                const int f = 2 * d + a(d);
#pragma unroll
                for (int t0 = 0; t0 < K; t0++)
#pragma unroll
                    for (int t1 = 0; t1 < K; t1++) {
                        const int t = f * K * K + t0 * K + t1;
                        const long long gt = __ldg(rowt + t) + (long long)__ldg(T.offt + t) * layer;
                        acc = fma(T.P[t0 * 2 + a(e0)] * T.P[t1 * 2 + a(e1)], __ldg(T.w + gt) * __ldg(T.in + gt), acc);
                    }
            }
            const long long gv = __ldg(rowv + l) + (long long)__ldg(T.offv + l) * layer;
            if (ATOMIC) atomicAdd(T.out + gv, acc);
            else T.out[gv] += acc;                                  // colour and layer parity: no other writer
        }
    }
}

template <int K, int KIND, bool ATOMIC>
int launch(const TraceParams<K> &T)
{
    fdb::Context &c = fdb::ctx();
    auto kern = trace_transfer_kernel<K, KIND, ATOMIC>;
    int per_sm = 0;
    FDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, THREADS, 0));
    const long long nthr = (long long)T.ncols * T.nlay_items * (KIND == TT_PROLONG ? 6 * K * K : 8);
    long long grid = (nthr + THREADS - 1) / THREADS;
    const long long cap = (long long)c.sm_count * (per_sm > 0 ? per_sm : 1);
    if (grid > cap) grid = cap;
    if (grid < 1) return 0;
    kern<<<(int)grid, THREADS, 0, c.stream>>>(T);
    FDB_LAUNCH_CHECK();
    return 0;
}

template <int K>
int run(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *out, const double *in,
        const double *w, const fdb_int *mapt, const fdb_int *mapv)
{
    TraceParams<K> T;
    memset(&T, 0, sizeof(T));
    T.out = out;
    T.in = in;
    T.w = w;
    T.mapt = mapt;
    T.mapv = mapv;
    T.offt = k->d_off0;
    T.offv = k->d_off2;
    for (int i = 0; i < K * 2; i++) T.P[i] = k->B2[i];
    const bool prolong = k->desc.form == FDB_FORM_TRACE_PROLONG;
    if (prolong || k->desc.scatter == FDB_SCATTER_ATOMIC) {
        T.collist = subset;
        T.col0 = start;
        T.ncols = end - start;
        T.nlay_items = nlay;
        T.lay_step = 1;
        if (T.ncols <= 0 || nlay <= 0) return 0;
        if (prolong) return launch<K, TT_PROLONG, false>(T);
        return launch<K, TT_RESTRICT, true>(T);
    }
    // deterministic restrict: one launch per (colour, layer parity), no two cells of a launch share a vertex
    if (subset) {
        fdb::set_error("trace_restrict: coloured scatter does not support subsets");
        return 1;
    }
    for (int col = 0; col < k->ncolours; col++) {
        T.collist = k->d_colour_cols + k->colour_start[col];
        T.ncols = k->colour_start[col + 1] - k->colour_start[col];
        for (int par = 0; par < (nlay > 1 ? 2 : 1); par++) {
            T.lay_first = par;
            T.lay_step = 2;
            T.nlay_items = (nlay - par + 1) / 2;
            if (T.ncols <= 0 || T.nlay_items <= 0) continue;
            if (launch<K, TT_RESTRICT, false>(T)) return 1;
        }
    }
    return 0;
}

}  // namespace

int fdb_launch_trace_transfer(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                              double *out, const double *in, const double *w, const fdb_int *mapt,
                              const fdb_int *mapv)
{
    if (k->desc.degree == 1) return run<2>(k, start, end, nlay, subset, out, in, w, mapt, mapv);
    if (k->desc.degree == 2) return run<3>(k, start, end, nlay, subset, out, in, w, mapt, mapv);
    fdb::set_error("trace transfer: trace degree %d not instantiated: 1, 2 (k = 2, 3)", k->desc.degree);
    return 1;
}
