// FDB_FORM_BOUNDARY_MASS: the boundary mass term on scalar (cdim = 1) and vector (cdim = 3) Q_p (x) P_p
// hexahedra,
//     a_G(u, v) = gamma * inner(u, v) * ds(sub_domain)      (gamma = desc.alpha),
// an exterior-facet integral: the Robin operator term, and through its action every boundary load
// (inner(g, v)*ds is the action of a_G with gamma = 1 on g).  DESIGN.md section 4.14.
//
// An iteration entry is one exterior facet of one cell: a column of the facet set (one map row of the cell
// that owns the facet, plus offset * layer on extruded cells) and its local facet number f (a uint32 per
// column, read like a direct Dat of the column).  f = 2*direction + side: the facet is the face of the cell
// where the 1-D dof index along axis `direction` (x, y, z of the local numbering (ax*N + ay)*N + v) is
// `side` -- dof index 0 is the 0 end of the reference interval, 1 the 1 end.  Only the N^2 face nodes are
// gathered; the face's tangential axes s, t are the other two axes in increasing order.
//
// Layout: one thread per face node, which is also one face quadrature point (nq = N), FPB facets ("slots")
// per CTA, everything in static shared memory.  Per slot: the face's 4 vertices (from the Q1 coordinate
// map row, vertex (bx*2 + by)*2 + bz), the gathered values and one work buffer per component, and the
// weights W = gamma w_s w_t |dX/ds x dX/dt| at the points of the bilinear face X(s, t).
//   ACTION    B along s, B along t, times W, B^T along t, B^T along s, scatter (atomic or coloured)
//   DIAGONAL  d[a][b] = sum_st B[s][a]^2 B[t][b]^2 W[s][t], two passes, the same value added to every
//             component of the node (atomic)
//   MATRIX    each thread (test node i) forms its row of the element matrix M[i][j] = sum_st B[s][i_s]
//             B[s][j_s] B[t][i_t] B[t][j_t] W[s][t] and adds it into the CSR (block diagonals of a
//             blocked Mat: the form does not couple components); entries whose dof-level lgmap index is
//             negative are dropped (atomic)
#include "common.cuh"

namespace {

enum { BM_ACTION = 0, BM_DIAGONAL = 1, BM_MATRIX = 2 };

template <int N>
struct BoundaryParams {
    double *y;                   // action / diagonal output (cdim values per node)
    const double *x;             // action input
    const double *coords;        // AoS, 3 per vertex
    const fdb_int *map0, *map1;  // node map (N^3 per column / cell), vertex map (8)
    const fdb_int *off0, *off1;  // layer offsets (zeros for native hexes)
    const unsigned *facet;       // local facet number of each column of the iteration set
    const fdb_int *collist;      // columns to visit (subset / colour) or NULL = col0 + i
    int col0, ncols;
    int nlay_items, lay_first, lay_step;   // layers lay_first + lay_step * k, k < nlay_items
    double gamma;
    double B[N * N], wq[N], xq[N];
    // MATRIX
    const long long *rowptr;
    const fdb_int *colidx;
    double *vals;
    const fdb_int *row_lg, *col_lg;   // dof-level, NULL = identity
};

template <int N>
struct BoundaryShape {
    static constexpr int NF = N * N;                                   // face nodes = face points
    static constexpr int FPB = 256 / NF;                               // facets (slots) per CTA
    static constexpr int THREADS = ((FPB * NF + 31) / 32) * 32;
};

template <int N, int CDIM, int MODE, bool ATOMIC>
__global__ void __launch_bounds__(BoundaryShape<N>::THREADS)
boundary_mass_kernel(const __grid_constant__ BoundaryParams<N> P)
{
    using S = BoundaryShape<N>;
    constexpr int NF = S::NF;
    constexpr int FPB = S::FPB;
    constexpr int ND = N * N * N;
    constexpr int NB = MODE == BM_ACTION ? CDIM : 1;       // value / work buffers per slot
    __shared__ double s_x[FPB][12];                        // face vertex (sa*2 + sb), component
    __shared__ double s_u[FPB][NB * NF];
    __shared__ double s_t[FPB][NB * NF];
    __shared__ double s_w[FPB][NF];
    __shared__ int s_idx[FPB][MODE == BM_MATRIX ? NF : 1];
    const int slot = threadIdx.x / NF;
    const int l = threadIdx.x - slot * NF;
    const bool in_cta = slot < FPB;
    const int sl = in_cta ? slot : 0;
    const int a = l / N, b = l - (l / N) * N;              // face node (a along s, b along t) = point (a, b)

    const long long nunits = (long long)P.ncols * P.nlay_items;
    for (long long base = (long long)blockIdx.x * FPB; base < nunits; base += (long long)gridDim.x * FPB) {
        const long long unit = base + slot;
        const bool valid = in_cta && unit < nunits;
        int col = 0, layer = 0;
        unsigned f = 0;
        if (valid) {
            const int ci = (int)(unit / P.nlay_items);
            layer = P.lay_first + P.lay_step * (int)(unit - (long long)ci * P.nlay_items);
            col = P.collist ? __ldg(P.collist + ci) : P.col0 + ci;
            f = __ldg(P.facet + col);
        }
        const int dir = (int)(f >> 1), side = (int)(f & 1u);
        // ---- gather: the face node's cell-local dof, its values, the face's vertices
        const int lc = dir == 0 ? (side * N + a) * N + b : (dir == 1 ? (a * N + side) * N + b : (a * N + b) * N + side);
        int g = 0;
        if (valid) {
            g = __ldg(P.map0 + (long long)col * ND + lc) + __ldg(P.off0 + lc) * layer;
            if (MODE == BM_ACTION) {
#pragma unroll
                for (int c = 0; c < CDIM; c++) s_u[sl][c * NF + l] = __ldg(P.x + (long long)g * CDIM + c);
            }
            if (MODE == BM_MATRIX) s_idx[sl][l] = g;
            for (int i = l; i < 12; i += NF) {
                const int v = i / 3, c = i - 3 * v;
                const int sa = v >> 1, sb = v & 1;
                const int bx = dir == 0 ? side : sa;
                const int by = dir == 0 ? sa : (dir == 1 ? side : sb);
                const int bz = dir == 2 ? side : sb;
                const int vc = (bx * 2 + by) * 2 + bz;
                const int gv = __ldg(P.map1 + (long long)col * 8 + vc) + __ldg(P.off1 + vc) * layer;
                s_x[sl][i] = __ldg(P.coords + (long long)gv * 3 + c);
            }
        } else if (in_cta) {
            // idle slot: a degenerate face (zero weights) with zero values
            if (MODE == BM_ACTION) {
#pragma unroll
                for (int c = 0; c < CDIM; c++) s_u[sl][c * NF + l] = 0.0;
            }
            if (MODE == BM_MATRIX) s_idx[sl][l] = 0;
            for (int i = l; i < 12; i += NF) s_x[sl][i] = 0.0;
        }
        __syncthreads();
        // ---- weight at point (a, b): gamma w_s w_t |dX/ds x dX/dt|
        double W = 0.0;
        if (in_cta) {
            const double s = P.xq[a], t = P.xq[b];
            const double *X = s_x[sl];
            double xs[3], xt[3];
#pragma unroll
            for (int c = 0; c < 3; c++) {
                xs[c] = (1.0 - t) * (X[6 + c] - X[c]) + t * (X[9 + c] - X[3 + c]);
                xt[c] = (1.0 - s) * (X[3 + c] - X[c]) + s * (X[9 + c] - X[6 + c]);
            }
            const double n0 = xs[1] * xt[2] - xs[2] * xt[1];
            const double n1 = xs[2] * xt[0] - xs[0] * xt[2];
            const double n2 = xs[0] * xt[1] - xs[1] * xt[0];
            W = P.gamma * P.wq[a] * P.wq[b] * sqrt(n0 * n0 + n1 * n1 + n2 * n2);
            if (MODE != BM_ACTION) s_w[sl][l] = W;
        }
        if (MODE == BM_ACTION) {
            // B along s: t[q][b] = sum_k B[q][k] u[k][b]
            if (in_cta) {
#pragma unroll
                for (int c = 0; c < CDIM; c++) {
                    double acc = 0.0;
#pragma unroll
                    for (int k = 0; k < N; k++) acc = fma(P.B[a * N + k], s_u[sl][c * NF + k * N + b], acc);
                    s_t[sl][c * NF + l] = acc;
                }
            }
            __syncthreads();
            // B along t, times W: u[q][r] = W[q][r] sum_k B[r][k] t[q][k]
            if (in_cta) {
#pragma unroll
                for (int c = 0; c < CDIM; c++) {
                    double acc = 0.0;
#pragma unroll
                    for (int k = 0; k < N; k++) acc = fma(P.B[b * N + k], s_t[sl][c * NF + a * N + k], acc);
                    s_u[sl][c * NF + l] = W * acc;
                }
            }
            __syncthreads();
            // B^T along t: t[q][b] = sum_r B[r][b] u[q][r]
            if (in_cta) {
#pragma unroll
                for (int c = 0; c < CDIM; c++) {
                    double acc = 0.0;
#pragma unroll
                    for (int r = 0; r < N; r++) acc = fma(P.B[r * N + b], s_u[sl][c * NF + a * N + r], acc);
                    s_t[sl][c * NF + l] = acc;
                }
            }
            __syncthreads();
            // B^T along s and the scatter: y[a][b] += sum_q B[q][a] t[q][b]
            if (valid) {
                double *dst = P.y + (long long)g * CDIM;
#pragma unroll
                for (int c = 0; c < CDIM; c++) {
                    double acc = 0.0;
#pragma unroll
                    for (int q = 0; q < N; q++) acc = fma(P.B[q * N + a], s_t[sl][c * NF + q * N + b], acc);
                    if (ATOMIC) atomicAdd(dst + c, acc);
                    else dst[c] += acc;
                }
            }
        } else if (MODE == BM_DIAGONAL) {
            __syncthreads();
            // t[q][b] = sum_r B[r][b]^2 W[q][r]
            if (in_cta) {
                double acc = 0.0;
#pragma unroll
                for (int r = 0; r < N; r++) {
                    const double br = P.B[r * N + b];
                    acc = fma(br * br, s_w[sl][a * N + r], acc);
                }
                s_t[sl][l] = acc;
            }
            __syncthreads();
            if (valid) {
                double acc = 0.0;
#pragma unroll
                for (int q = 0; q < N; q++) {
                    const double bq = P.B[q * N + a];
                    acc = fma(bq * bq, s_t[sl][q * N + b], acc);
                }
#pragma unroll
                for (int c = 0; c < CDIM; c++) atomicAdd(P.y + (long long)g * CDIM + c, acc);
            }
        } else {
            __syncthreads();
            // this thread's row (test node (a, b)): M[(a, b)][(c, d)] = sum_q B[q][a] B[q][c] T_d[q],
            // T_d[q] = sum_r B[r][b] B[r][d] W[q][r]
            if (valid) {
                const long long lo0 = __ldg(P.rowptr + g), hi0 = __ldg(P.rowptr + g + 1);
                for (int d = 0; d < N; d++) {
                    double T[N];
#pragma unroll
                    for (int q = 0; q < N; q++) {
                        double acc = 0.0;
#pragma unroll
                        for (int r = 0; r < N; r++) acc = fma(P.B[r * N + b] * P.B[r * N + d], s_w[sl][q * N + r], acc);
                        T[q] = acc;
                    }
#pragma unroll
                    for (int c = 0; c < N; c++) {
                        double m = 0.0;
#pragma unroll
                        for (int q = 0; q < N; q++) m = fma(P.B[q * N + a] * P.B[q * N + c], T[q], m);
                        const int gj = s_idx[sl][c * N + d];
                        long long lo = lo0, hi = hi0;
                        while (hi - lo > 1) {
                            const long long mid = (lo + hi) >> 1;
                            if (__ldg(P.colidx + mid) <= gj) lo = mid; else hi = mid;
                        }
#pragma unroll
                        for (int e = 0; e < CDIM; e++) {
                            if (P.row_lg && __ldg(P.row_lg + (long long)g * CDIM + e) < 0) continue;
                            if (P.col_lg && __ldg(P.col_lg + (long long)gj * CDIM + e) < 0) continue;
                            atomicAdd(P.vals + (lo * CDIM + e) * CDIM + e, m);
                        }
                    }
                }
            }
        }
        __syncthreads();          // the slot's buffers are refilled by the next facet
    }
}

template <int N, int CDIM, int MODE, bool ATOMIC>
int launch(cudaStream_t st, const BoundaryParams<N> &P, int sm_count)
{
    using S = BoundaryShape<N>;
    auto kern = boundary_mass_kernel<N, CDIM, MODE, ATOMIC>;
    int per_sm = 0;
    FDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, S::THREADS, 0));
    const long long nunits = (long long)P.ncols * P.nlay_items;
    long long grid = (nunits + S::FPB - 1) / S::FPB;
    const long long cap = (long long)sm_count * (per_sm > 0 ? per_sm : 1);
    if (grid > cap) grid = cap;
    if (grid < 1) return 0;
    kern<<<(int)grid, S::THREADS, 0, st>>>(P);
    FDB_LAUNCH_CHECK();
    return 0;
}

template <int N, int CDIM>
int run_n(fdb_kernel_s *k, int mode, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
          const double *coords, const double *x, const unsigned *facet, const fdb_int *map0, const fdb_int *map1,
          fdb_mat_t mat)
{
    fdb::Context &c = fdb::ctx();
    BoundaryParams<N> P;
    memset(&P, 0, sizeof(P));
    P.off0 = k->d_off0;
    P.off1 = k->d_off1;
    P.gamma = k->desc.alpha;
    for (int i = 0; i < N * N; i++) P.B[i] = k->desc.B[i];
    for (int i = 0; i < N; i++) {
        P.wq[i] = k->desc.wq[i];
        P.xq[i] = k->desc.xq[i];
    }
    P.y = y;
    P.x = x;
    P.coords = coords;
    P.facet = facet;
    P.map0 = map0;
    P.map1 = map1;
    if (mat && fdb_mat_device_view(mat, &P.rowptr, &P.colidx, &P.vals, &P.row_lg, &P.col_lg)) return 1;
    if (mode != BM_ACTION || k->desc.scatter == FDB_SCATTER_ATOMIC) {
        P.collist = subset;
        P.col0 = start;
        P.ncols = end - start;
        P.nlay_items = nlay;
        P.lay_first = 0;
        P.lay_step = 1;
        if (P.ncols <= 0 || nlay <= 0) return 0;
        if (mode == BM_MATRIX) {
            if constexpr (N <= 5) return launch<N, CDIM, BM_MATRIX, true>(c.stream, P, c.sm_count);
            fdb::set_error("boundary_mass matrix: degree %d not instantiated (1..4)", N - 1);
            return 1;
        }
        if (mode == BM_DIAGONAL) return launch<N, CDIM, BM_DIAGONAL, true>(c.stream, P, c.sm_count);
        return launch<N, CDIM, BM_ACTION, true>(c.stream, P, c.sm_count);
    }
    // deterministic: one launch per (colour, layer parity), no two facets of a launch share a node
    if (subset) {
        fdb::set_error("coloured scatter does not support subsets yet");
        return 1;
    }
    for (int col = 0; col < k->ncolours; col++) {
        P.collist = k->d_colour_cols + k->colour_start[col];
        P.col0 = 0;
        P.ncols = k->colour_start[col + 1] - k->colour_start[col];
        for (int par = 0; par < (nlay > 1 ? 2 : 1); par++) {
            P.lay_first = par;
            P.lay_step = 2;
            P.nlay_items = (nlay - par + 1) / 2;
            if (P.ncols <= 0 || P.nlay_items <= 0) continue;
            if (launch<N, CDIM, BM_ACTION, false>(c.stream, P, c.sm_count)) return 1;
        }
    }
    return 0;
}

template <int CDIM>
int run_cdim(fdb_kernel_s *k, int mode, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
             const double *coords, const double *x, const unsigned *facet, const fdb_int *map0,
             const fdb_int *map1, fdb_mat_t mat)
{
    switch (k->n1d) {
    case 2: return run_n<2, CDIM>(k, mode, start, end, nlay, subset, y, coords, x, facet, map0, map1, mat);
    case 3: return run_n<3, CDIM>(k, mode, start, end, nlay, subset, y, coords, x, facet, map0, map1, mat);
    case 4: return run_n<4, CDIM>(k, mode, start, end, nlay, subset, y, coords, x, facet, map0, map1, mat);
    case 5: return run_n<5, CDIM>(k, mode, start, end, nlay, subset, y, coords, x, facet, map0, map1, mat);
    case 6: return run_n<6, CDIM>(k, mode, start, end, nlay, subset, y, coords, x, facet, map0, map1, mat);
    }
    fdb::set_error("boundary_mass: degree %d not instantiated (1..5)", k->n1d - 1);
    return 1;
}

}  // namespace

int fdb_launch_boundary_mass(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                             fdb_mat_t mat, double *y, const double *coords, const double *x, const unsigned *facet,
                             const fdb_int *map0, const fdb_int *map1)
{
    const int mode = mat ? BM_MATRIX : (x ? BM_ACTION : BM_DIAGONAL);
    if (k->desc.cdim == 1)
        return run_cdim<1>(k, mode, start, end, nlay, subset, y, coords, x, facet, map0, map1, mat);
    if (k->desc.cdim == 3)
        return run_cdim<3>(k, mode, start, end, nlay, subset, y, coords, x, facet, map0, map1, mat);
    fdb::set_error("boundary_mass: cdim %d (1 or 3)", k->desc.cdim);
    return 1;
}
