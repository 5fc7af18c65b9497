// FDB_FORM_SPECTRAL_HELMHOLTZ and FDB_FORM_SPECTRAL_HELMHOLTZ_COEF: the spectral-element (collocated GLL) Helmholtz
// operator on scalar CG_p hexahedra, p = 1..5 (DESIGN.md section 4.18):
//
//   alpha*inner(kappa*grad u, grad v)*dx(GLL) + beta*inner(u, v)*dx(GLL)
//
// integrated with the (p+1)^3-point GLL rule at the nodes themselves, so that B = I: u and kappa at point q are the
// dofs u[q], kappa[q], and the mass term is diagonal.  Per cell:
//   ACTION    the reference gradient is one D contraction per axis (3 N^4 FMAs), the point metric
//             G = alpha kappa w |det J| J^-1 J^-T (the trilinear geometry of dg_hex.cuh), one D^T contraction per
//             axis (3 N^4) and the mass term beta w |det J| u at the point alone.
//   DIAGONAL  d phi_i / d xi_a vanishes at every point off the a-line through node i, so
//             diag_i = sum_a sum_q G_aa(q on i's a-line) D[q][i_a]^2 + sum_{a != b} G_ab(i) D[i_a][i_a] D[i_b][i_b]
//                      + beta w_i |det J_i|      (O(N^4) per cell at every degree)
//
// Layout: one thread per node, CPB cells per CTA, static shared memory (per cell: 8 vertices, the N^3 values and the
// 3 N^3 point fluxes).  The gather and scatter go through the CG cell-node map: atomicAdd, or the colour / layer-
// parity schedule of the other CG kernels, under which no two cells of a launch share a node and every node's sum is
// taken in launch order (bit-reproducible).
#include "common.cuh"
#include "dg_hex.cuh"

namespace {

enum { SEM_ACTION = 0, SEM_DIAGONAL = 1 };

template <int N>
struct SemParams {
    double *y;                   // action / diagonal output
    const double *x;             // action input
    const double *kappa;         // COEF: nodal kappa, through map0
    const double *coords;        // AoS, 3 per vertex
    const fdb_int *map0, *map1;  // dof map (N^3 per column), vertex map (8)
    const fdb_int *off0, *off1;  // layer offsets (zeros for native hexes)
    const fdb_int *collist;      // columns to visit (subset or colour) or NULL = col0 + i
    int col0, ncols;
    int nlay_items, lay_first, lay_step;   // layers lay_first + i * lay_step, i < nlay_items
    double alpha, beta;
    double D[N * N], wq[N], xq[N];         // D[q * N + a] = l_a'(x_q), all in dof order
};

template <int N>
struct SemShape {
    static constexpr int ND = N * N * N;                                // nodes = points
    static constexpr int CPB = 256 / ND < 32 ? (256 / ND > 0 ? 256 / ND : 1) : 32;
    static constexpr int THREADS = ((CPB * ND + 31) / 32) * 32;
};

template <int N, int MODE, bool COEF, bool ATOMIC>
__global__ void __launch_bounds__(SemShape<N>::THREADS)
sem_helmholtz_kernel(const __grid_constant__ SemParams<N> P)
{
    using S = SemShape<N>;
    constexpr int ND = S::ND;
    constexpr int CPB = S::CPB;
    __shared__ double s_x[CPB][24];
    __shared__ double s_u[CPB][MODE == SEM_ACTION ? ND : 1];
    __shared__ double s_c[CPB][3 * ND];            // action: the fluxes c_a; diagonal: G_aa
    const int slot = threadIdx.x / ND;
    const int l = threadIdx.x - slot * ND;
    const bool in_cta = slot < CPB;
    const int sl = in_cta ? slot : 0;
    const int i0 = l / (N * N), i1 = (l / N) % N, i2 = l % N;   // node (i0*N + i1)*N + i2 at (xq[i0], xq[i1], xq[i2])

    const long long nunits = (long long)P.ncols * P.nlay_items;
    for (long long base = (long long)blockIdx.x * CPB; base < nunits; base += (long long)gridDim.x * CPB) {
        const long long unit = base + slot;
        const bool valid = in_cta && unit < nunits;
        long long g = 0;
        double u = 0.0, kap = 1.0;
        if (valid) {
            const int ci = (int)(unit / P.nlay_items);
            const int layer = P.lay_first + (int)(unit - (long long)ci * P.nlay_items) * P.lay_step;
            const int col = P.collist ? __ldg(P.collist + ci) : P.col0 + ci;
            g = __ldg(P.map0 + (long long)col * ND + l) + (long long)__ldg(P.off0 + l) * layer;
            if (MODE == SEM_ACTION) {
                u = __ldg(P.x + g);
                s_u[sl][l] = u;
            }
            if (COEF) kap = __ldg(P.kappa + g);
#pragma unroll 1
            for (int i = l; i < 24; i += ND) {
                const int v = i / 3, c = i - 3 * v;
                const long long gv = __ldg(P.map1 + (long long)col * 8 + v) + (long long)__ldg(P.off1 + v) * layer;
                s_x[sl][i] = __ldg(P.coords + gv * 3 + c);
            }
        } else if (in_cta) {
            // idle slot: the unit cube (finite geometry), nothing scattered
            if (MODE == SEM_ACTION) s_u[sl][l] = 0.0;
            for (int i = l; i < 24; i += ND) {
                const int v = i / 3, c = i % 3;
                s_x[sl][i] = (double)((v >> (2 - c)) & 1);
            }
        }
        __syncthreads();
        double val = 0.0;
        if (in_cta) {
            const double xi[3] = {P.xq[i0], P.xq[i1], P.xq[i2]};
            double K[3][3];
            const double detJ = trilinear_inverse_jacobian(&s_x[sl][0], xi, K);
            const double w = P.wq[i0] * P.wq[i1] * P.wq[i2] * detJ;
            const double s = P.alpha * kap * w;
            double G[3][3];                                        // s K K^T (symmetric)
#pragma unroll
            for (int a = 0; a < 3; a++)
#pragma unroll
                for (int b = a; b < 3; b++) G[a][b] = s * (K[a][0] * K[b][0] + K[a][1] * K[b][1] + K[a][2] * K[b][2]);
            if (MODE == SEM_ACTION) {
                // the reference gradient at the point: one D contraction per axis
                double r0 = 0.0, r1 = 0.0, r2 = 0.0;
#pragma unroll
                for (int q = 0; q < N; q++) {
                    r0 = fma(P.D[i0 * N + q], s_u[sl][(q * N + i1) * N + i2], r0);
                    r1 = fma(P.D[i1 * N + q], s_u[sl][(i0 * N + q) * N + i2], r1);
                    r2 = fma(P.D[i2 * N + q], s_u[sl][(i0 * N + i1) * N + q], r2);
                }
                s_c[sl][l] = G[0][0] * r0 + G[0][1] * r1 + G[0][2] * r2;
                s_c[sl][ND + l] = G[0][1] * r0 + G[1][1] * r1 + G[1][2] * r2;
                s_c[sl][2 * ND + l] = G[0][2] * r0 + G[1][2] * r1 + G[2][2] * r2;
                val = P.beta * w * u;
            } else {
                s_c[sl][l] = G[0][0];
                s_c[sl][ND + l] = G[1][1];
                s_c[sl][2 * ND + l] = G[2][2];
                const double d0 = P.D[i0 * N + i0], d1 = P.D[i1 * N + i1], d2 = P.D[i2 * N + i2];
                val = P.beta * w + 2.0 * (G[0][1] * d0 * d1 + G[0][2] * d0 * d2 + G[1][2] * d1 * d2);
            }
        }
        __syncthreads();
        if (valid) {
            if (MODE == SEM_ACTION) {
                // y[i0, i1, i2] += sum_q D[q][i0] c_0[q, i1, i2] + D[q][i1] c_1[i0, q, i2] + D[q][i2] c_2[i0, i1, q]
#pragma unroll
                for (int q = 0; q < N; q++) {
                    val = fma(P.D[q * N + i0], s_c[sl][(q * N + i1) * N + i2], val);
                    val = fma(P.D[q * N + i1], s_c[sl][ND + (i0 * N + q) * N + i2], val);
                    val = fma(P.D[q * N + i2], s_c[sl][2 * ND + (i0 * N + i1) * N + q], val);
                }
            } else {
#pragma unroll
                for (int q = 0; q < N; q++) {
                    const double e0 = P.D[q * N + i0], e1 = P.D[q * N + i1], e2 = P.D[q * N + i2];
                    val = fma(e0 * e0, s_c[sl][(q * N + i1) * N + i2], val);
                    val = fma(e1 * e1, s_c[sl][ND + (i0 * N + q) * N + i2], val);
                    val = fma(e2 * e2, s_c[sl][2 * ND + (i0 * N + i1) * N + q], val);
                }
            }
            if (ATOMIC) atomicAdd(P.y + g, val);
            else P.y[g] += val;                                    // colour and layer parity: no other writer
        }
        __syncthreads();                                           // the slot's buffers are refilled next
    }
}

template <int N, int MODE, bool COEF, bool ATOMIC>
int launch(const SemParams<N> &P)
{
    using S = SemShape<N>;
    fdb::Context &c = fdb::ctx();
    auto kern = sem_helmholtz_kernel<N, MODE, COEF, ATOMIC>;
    int per_sm = 0;
    FDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, S::THREADS, 0));
    const long long nunits = (long long)P.ncols * P.nlay_items;
    long long grid = (nunits + S::CPB - 1) / S::CPB;
    const long long cap = (long long)c.sm_count * (per_sm > 0 ? per_sm : 1);
    if (grid > cap) grid = cap;
    if (grid < 1) return 0;
    kern<<<(int)grid, S::THREADS, 0, c.stream>>>(P);
    FDB_LAUNCH_CHECK();
    return 0;
}

template <int N, int MODE, bool COEF>
int run_mode(fdb_kernel_s *k, SemParams<N> &P, fdb_int start, fdb_int end, int nlay, const fdb_int *subset)
{
    if (k->desc.scatter == FDB_SCATTER_ATOMIC) {
        P.collist = subset;
        P.col0 = start;
        P.ncols = end - start;
        P.nlay_items = nlay;
        P.lay_first = 0;
        P.lay_step = 1;
        if (P.ncols <= 0 || nlay <= 0) return 0;
        return launch<N, MODE, COEF, true>(P);
    }
    // deterministic: one launch per (colour, layer parity); within a launch no two cells share a node
    if (subset) {
        fdb::set_error("%s: coloured scatter does not support subsets", COEF ? "spectral_helmholtz_coef"
                                                                              : "spectral_helmholtz");
        return 1;
    }
    for (int col = 0; col < k->ncolours; col++) {
        P.collist = k->d_colour_cols + k->colour_start[col];
        P.ncols = k->colour_start[col + 1] - k->colour_start[col];
        for (int par = 0; par < (nlay > 1 ? 2 : 1); par++) {
            P.lay_first = par;
            P.lay_step = nlay > 1 ? 2 : 1;
            P.nlay_items = nlay > 1 ? (nlay - par + 1) / 2 : nlay;
            if (P.ncols <= 0 || P.nlay_items <= 0) continue;
            if (launch<N, MODE, COEF, false>(P)) return 1;
        }
    }
    return 0;
}

template <int N>
int run_n(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
          const double *coords, const double *x, const double *kappa, const fdb_int *map0, const fdb_int *map1)
{
    SemParams<N> P;
    memset(&P, 0, sizeof(P));
    P.y = y;
    P.x = x;
    P.kappa = kappa;
    P.coords = coords;
    P.map0 = map0;
    P.map1 = map1;
    P.off0 = k->d_off0;
    P.off1 = k->d_off1;
    P.alpha = k->desc.alpha;
    P.beta = k->desc.beta;
    for (int i = 0; i < N * N; i++) P.D[i] = k->desc.D[i];
    for (int i = 0; i < N; i++) {
        P.wq[i] = k->desc.wq[i];
        P.xq[i] = k->desc.xq[i];
    }
    const bool coef = k->desc.form == FDB_FORM_SPECTRAL_HELMHOLTZ_COEF;
    if (x) return coef ? run_mode<N, SEM_ACTION, true>(k, P, start, end, nlay, subset)
                       : run_mode<N, SEM_ACTION, false>(k, P, start, end, nlay, subset);
    return coef ? run_mode<N, SEM_DIAGONAL, true>(k, P, start, end, nlay, subset)
                : run_mode<N, SEM_DIAGONAL, false>(k, P, start, end, nlay, subset);
}

}  // namespace

int fdb_launch_spectral_helmholtz(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                                  double *y, const double *coords, const double *x, const double *kappa,
                                  const fdb_int *map0, const fdb_int *map1)
{
    switch (k->n1d) {
    case 2: return run_n<2>(k, start, end, nlay, subset, y, coords, x, kappa, map0, map1);
    case 3: return run_n<3>(k, start, end, nlay, subset, y, coords, x, kappa, map0, map1);
    case 4: return run_n<4>(k, start, end, nlay, subset, y, coords, x, kappa, map0, map1);
    case 5: return run_n<5>(k, start, end, nlay, subset, y, coords, x, kappa, map0, map1);
    case 6: return run_n<6>(k, start, end, nlay, subset, y, coords, x, kappa, map0, map1);
    }
    fdb::set_error("spectral helmholtz kernel: degree %d not instantiated (1..5)", k->n1d - 1);
    return 1;
}
