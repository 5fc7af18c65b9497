// The cell term of FDB_FORM_DG_TRANSPORT, upwind DG transport on scalar DQ_p hexahedra (DESIGN.md section 4.16):
//
//   - u*dot(b, grad v)*dx
//
// on the collocated Gauss-Legendre element (B = I, nq = p+1), with b given at the 8 vertices and interpolated
// trilinearly.  u at point q is the dof u[q], so the trial side needs no contraction; the test side is one D^T
// contraction per reference axis of the point coefficients c_d = -w |det J| u (J^-1 b)_d.
//
// Layout: one thread per Gauss point, CPB cells per CTA, static shared memory (per cell: 8 vertices, b at them and
// the 3 N^3 point coefficients).  A DQ cell owns its dofs, so no two cells of a launch write the same entry of y:
// the scatter is a plain read-add-write, without atomics, colours or layer parity, and is deterministic.
//   ACTION    gather, point stage, D^T contractions along the three axes + scatter
//   DIAGONAL  -w_i |det J_i| (J^-1 b)_i . (D_ii, D_jj, D_kk) at the point alone (no contraction)
// The facet terms are dg_upwind_kernel (dg_facet_hex.cu).
#include "common.cuh"
#include "dg_hex.cuh"

namespace {

enum { TR_ACTION = 0, TR_DIAGONAL = 1 };

template <int N>
struct TransportCellParams {
    double *y;                   // action / diagonal output
    const double *x;             // action input
    const double *coords, *b;    // AoS, 3 per vertex
    const fdb_int *map0, *map1;  // dof map (N^3 per column), vertex map (8)
    const fdb_int *off0, *off1;  // layer offsets (zeros for native hexes)
    const fdb_int *collist;      // columns to visit (subset) or NULL = col0 + i
    int col0, ncols, nlay;
    double D[N * N], wq[N], xq[N];
};

template <int N>
struct TransportCellShape {
    static constexpr int ND = N * N * N;                                // points = dofs
    static constexpr int CPB = 256 / ND < 32 ? 256 / ND : 32;           // cells (slots) per CTA
    static constexpr int THREADS = ((CPB * ND + 31) / 32) * 32;
};

template <int N, int MODE>
__global__ void __launch_bounds__(TransportCellShape<N>::THREADS)
dg_transport_cell_kernel(const __grid_constant__ TransportCellParams<N> P)
{
    using S = TransportCellShape<N>;
    constexpr int ND = S::ND;
    constexpr int CPB = S::CPB;
    __shared__ double s_x[CPB][24];
    __shared__ double s_b[CPB][24];
    __shared__ double s_c[CPB][MODE == TR_ACTION ? 3 * ND : 1];   // c_0, c_1, c_2 at every point
    const int slot = threadIdx.x / ND;
    const int l = threadIdx.x - slot * ND;
    const bool in_cta = slot < CPB;
    const int sl = in_cta ? slot : 0;
    const int i0 = l / (N * N), i1 = (l / N) % N, i2 = l % N;   // point = dof (i0*N + i1)*N + i2

    const long long nunits = (long long)P.ncols * P.nlay;
    for (long long base = (long long)blockIdx.x * CPB; base < nunits; base += (long long)gridDim.x * CPB) {
        const long long unit = base + slot;
        const bool valid = in_cta && unit < nunits;
        int g = 0;
        double u = 0.0;
        if (valid) {
            const int ci = (int)(unit / P.nlay);
            const int layer = (int)(unit - (long long)ci * P.nlay);
            const int col = P.collist ? __ldg(P.collist + ci) : P.col0 + ci;
            g = __ldg(P.map0 + (long long)col * ND + l) + __ldg(P.off0 + l) * layer;
            if (MODE == TR_ACTION) u = __ldg(P.x + g);
#pragma unroll 1          // unrolled, the DQ1 diagonal spills 4 bytes under ptxas's register target
            for (int i = l; i < 24; i += ND) {
                const int v = i / 3, c = i - 3 * v;
                const long long gv = (long long)(__ldg(P.map1 + (long long)col * 8 + v) + __ldg(P.off1 + v) * layer);
                s_x[sl][i] = __ldg(P.coords + gv * 3 + c);
                s_b[sl][i] = __ldg(P.b + gv * 3 + c);
            }
        } else if (in_cta) {
            // idle slot: the unit cube at rest (finite geometry), nothing scattered
            for (int i = l; i < 24; i += ND) {
                const int v = i / 3, c = i % 3;
                s_x[sl][i] = (double)((v >> (2 - c)) & 1);
                s_b[sl][i] = 0.0;
            }
        }
        __syncthreads();
        double val = 0.0;
        if (in_cta) {
            const double xi[3] = {P.xq[i0], P.xq[i1], P.xq[i2]};
            double K[3][3], bq[3];
            const double detJ = trilinear_inverse_jacobian(&s_x[sl][0], xi, K);
            trilinear_interpolate(&s_b[sl][0], xi, bq);
            const double w = P.wq[i0] * P.wq[i1] * P.wq[i2] * detJ;
            double kb[3];                                          // J^-1 b: b in reference components
#pragma unroll
            for (int d = 0; d < 3; d++) kb[d] = K[d][0] * bq[0] + K[d][1] * bq[1] + K[d][2] * bq[2];
            if (MODE == TR_ACTION) {
                const double c = -w * u;
#pragma unroll
                for (int d = 0; d < 3; d++) s_c[sl][d * ND + l] = c * kb[d];
            } else {
                val = -w * (kb[0] * P.D[i0 * N + i0] + kb[1] * P.D[i1 * N + i1] + kb[2] * P.D[i2 * N + i2]);
            }
        }
        if (MODE == TR_ACTION) {
            __syncthreads();
            // y[i0, i1, i2] = sum_q D[q][i0] c_0[q, i1, i2] + D[q][i1] c_1[i0, q, i2] + D[q][i2] c_2[i0, i1, q]
            if (valid) {
#pragma unroll
                for (int q = 0; q < N; q++) {
                    val = fma(P.D[q * N + i0], s_c[sl][(q * N + i1) * N + i2], val);
                    val = fma(P.D[q * N + i1], s_c[sl][ND + (i0 * N + q) * N + i2], val);
                    val = fma(P.D[q * N + i2], s_c[sl][2 * ND + (i0 * N + i1) * N + q], val);
                }
            }
        }
        if (valid) P.y[g] += val;                                  // the cell owns dof g: no other writer
        __syncthreads();                                           // the slot's buffers are refilled next
    }
}

template <int N, int MODE>
int launch_cell(const TransportCellParams<N> &P)
{
    using S = TransportCellShape<N>;
    fdb::Context &c = fdb::ctx();
    auto kern = dg_transport_cell_kernel<N, MODE>;
    int per_sm = 0;
    FDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, S::THREADS, 0));
    const long long nunits = (long long)P.ncols * P.nlay;
    long long grid = (nunits + S::CPB - 1) / S::CPB;
    const long long cap = (long long)c.sm_count * (per_sm > 0 ? per_sm : 1);
    if (grid > cap) grid = cap;
    if (grid < 1) return 0;
    kern<<<(int)grid, S::THREADS, 0, c.stream>>>(P);
    FDB_LAUNCH_CHECK();
    return 0;
}

template <int N>
int run_cell_n(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
               const double *coords, const double *x, const double *b, const fdb_int *map0, const fdb_int *map1)
{
    TransportCellParams<N> P;
    memset(&P, 0, sizeof(P));
    P.y = y;
    P.x = x;
    P.coords = coords;
    P.b = b;
    P.map0 = map0;
    P.map1 = map1;
    P.off0 = k->d_off0;
    P.off1 = k->d_off1;
    P.collist = subset;
    P.col0 = start;
    P.ncols = end - start;
    P.nlay = nlay;
    for (int i = 0; i < N * N; i++) P.D[i] = k->desc.D[i];
    for (int i = 0; i < N; i++) {
        P.wq[i] = k->desc.wq[i];
        P.xq[i] = k->desc.xq[i];
    }
    if (P.ncols <= 0 || nlay <= 0) return 0;
    return x ? launch_cell<N, TR_ACTION>(P) : launch_cell<N, TR_DIAGONAL>(P);
}

}  // namespace

int fdb_launch_dg_transport(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
                            const double *coords, const double *x, const double *b, const unsigned *facet,
                            const fdb_int *map0, const fdb_int *map1)
{
    if (k->desc.integral != FDB_INTEGRAL_CELL)
        return fdb_launch_dg_upwind(k, start, end, nlay, subset, y, coords, x, b, facet, map0, map1);
    switch (k->n1d) {
    case 2: return run_cell_n<2>(k, start, end, nlay, subset, y, coords, x, b, map0, map1);
    case 3: return run_cell_n<3>(k, start, end, nlay, subset, y, coords, x, b, map0, map1);
    case 4: return run_cell_n<4>(k, start, end, nlay, subset, y, coords, x, b, map0, map1);
    case 5: return run_cell_n<5>(k, start, end, nlay, subset, y, coords, x, b, map0, map1);
    }
    fdb::set_error("dg transport cell kernel: degree %d not instantiated (1..4)", k->n1d - 1);
    return 1;
}
