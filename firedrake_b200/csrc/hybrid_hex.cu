// FDB_FORM_MIXED_POISSON_HYBRID and FDB_FORM_MIXED_POISSON_RECONSTRUCT: hybridisation (static condensation) of mixed
// Poisson on NCF_k x DQ_{k-1} hexahedra, k = 2 and 3 (DESIGN.md section 4.23).  The flux space is broken cell by
// cell and normal continuity is enforced by a Lagrange multiplier lambda in the HDiv-trace space (Q_{k-1} on every
// face, its k^2 dofs at the Gauss-Legendre points of the face).  Per cell K, with A = alpha M and B the cell blocks
// of FDB_FORM_MIXED_POISSON and C the (diagonal, metric-free) trace coupling C[t][sigma-dof(t)] = o_t w_t:
//
//   K_K = [[A, B^T], [B, 0]],   C^ = [C 0],   H = sum_K C^ K_K^-1 C^^T,   r = sum_K C^ K_K^-1 f_K
//   (sigma_K, u_K) = K_K^-1 (f_K - C^^T lambda)
//
// All three are one symmetric Gaussian elimination (no pivoting: the pivots of A are positive, those of the Schur
// complement -B A^-1 B^T negative) of a bordered matrix held as a packed lower triangle in shared memory, rebuilt
// for every cell (no per-cell factors are stored):
//
//   HY_CONDENSE     [[A, B^T, C^T], [B, 0, 0], [C, 0, 0]]: after eliminating the NS + NU local unknowns the trailing
//                   6k^2 x 6k^2 block is -C^ K_K^-1 C^^T, scattered (negated) into the trace CSR through the masked
//                   lgmaps.
//   HY_ELIMINATE    [[K_K, g], [g^T, 0]] with g = f_K: the last row becomes L^-1 g, a back substitution gives
//   HY_RECONSTRUCT  x = K_K^-1 g (g = f_K - C^^T lambda for the reconstruction); r += C x_sigma, or y_sigma += w o
//                   x_sigma and y_u += x_u.
//
// f_K = (w o sigma-load, u-load) gathered through the NCF and DQ maps, w one value per flux dof (1 / the number of
// cells that hold it).  Every output entry receives at most two cell contributions onto zero (two faces share at
// most one cell; a face has at most two cells), so the atomic scatter is bit-reproducible.
//
// Layout: one cell per CTA (one warp at k = 2, eight at k = 3), grid-stride over (column, layer) units.  The
// elimination gives each warp whole rows of the trailing triangle and its lanes the columns of a row: one barrier
// per eliminated column.
#include "common.cuh"

namespace {

enum { HY_CONDENSE = 0, HY_ELIMINATE, HY_RECONSTRUCT };

template <int K>
struct HybridShape {
    static constexpr int Q = K + 1;                       // Gauss points per axis
    static constexpr int NP = Q * Q * Q;
    static constexpr int NB = K * K * (K + 1);            // flux dofs per component block
    static constexpr int NS = 3 * NB;                     // flux dofs per cell
    static constexpr int NU = K * K * K;                  // DQ_{k-1} dofs per cell
    static constexpr int NF = 6 * K * K;                  // trace dofs per cell
    static constexpr int NL = NS + NU;                    // eliminated unknowns
    static constexpr int THREADS = K == 2 ? 32 : 256;
    static constexpr int NWARPS = THREADS / 32;
};

template <int K>
struct HybridParams {
    double *out;                 // CONDENSE: unused (the CSR); ELIMINATE: r; RECONSTRUCT: y_sigma
    double *yu;                  // RECONSTRUCT: y_u
    const double *lam;           // RECONSTRUCT: lambda
    const double *fs, *w, *fu;   // sigma load, flux weights, u load
    const double *coords;
    const fdb_int *map_t, *map_c, *map_s, *map_u;   // trace (6k^2), vertex (8), NCF (3k^2(k+1)), DQ (k^3)
    const fdb_int *off_t, *off_c, *off_s, *off_u;   // layer offsets (zeros for native hexes)
    const fdb_int *collist;
    int col0, ncols, nlay;
    // the trace CSR (CONDENSE)
    const long long *rowptr;
    const fdb_int *colidx;
    double *vals;
    const fdb_int *row_lg, *col_lg;   // -1 = masked (natural-condition faces), NULL = identity
    double alpha;
    double Bc[(K + 1) * (K + 1)];   // CG_k at the points, [q][a]
    double Bg[(K + 1) * K];         // DQ_{k-1} (GL) at the points, [q][b]
    double wq[K + 1], xq[K + 1];
    double Dx[K * (K + 1)];         // B: [v][a] = sum_q w_q psi_v(x_q) phi_a'(x_q)
    double Mg[K * K];               // B: [v][b] = sum_q w_q psi_v(x_q) psi_b(x_q)
    double wg[K];                   // the k-point Gauss-Legendre weights: C = o w_t0 w_t1
};

__device__ __forceinline__ int tri(int i) { return i * (i + 1) / 2; }

template <int K, int MODE>
__host__ __device__ constexpr int hybrid_n()
{
    using S = HybridShape<K>;
    return MODE == HY_CONDENSE ? S::NL + S::NF : S::NL + 1;
}

template <int K, int MODE>
constexpr size_t hybrid_smem()
{
    constexpr int N = hybrid_n<K, MODE>();
    return sizeof(double) * ((size_t)N * (N + 1) / 2 + 6 * HybridShape<K>::NP + HybridShape<K>::NL);
}

// the local flux dof of trace dof t: face 2d + s, (t0, t1) the GL indices of the other two axes in axis order
template <int K>
__device__ __forceinline__ int face_dof(int t, int *d_out, int *s_out, int *t0_out, int *t1_out)
{
    const int f = t / (K * K), r = t % (K * K), d = f >> 1, s = f & 1, t0 = r / K, t1 = r % K;
    int idx[3];
    idx[d] = s;
    idx[d == 0 ? 1 : 0] = t0;
    idx[d == 2 ? 1 : 2] = t1;
    const int n1 = d == 1 ? K + 1 : K, n2 = d == 2 ? K + 1 : K;
    *d_out = d;
    *s_out = s;
    *t0_out = t0;
    *t1_out = t1;
    return d * HybridShape<K>::NB + (idx[0] * n1 + idx[1]) * n2 + idx[2];
}

template <int K, int MODE>
__global__ void __launch_bounds__(HybridShape<K>::THREADS)
hybrid_kernel(const __grid_constant__ HybridParams<K> P)
{
    using S = HybridShape<K>;
    constexpr int Q = S::Q, NP = S::NP, NB = S::NB, NS = S::NS, NU = S::NU, NF = S::NF, NL = S::NL;
    constexpr int NT = S::THREADS, NW = S::NWARPS;
    constexpr int N = hybrid_n<K, MODE>();
    extern __shared__ double smem[];
    double *T = smem;                                  // packed lower triangle, row i at tri(i)
    double *Gw = T + N * (N + 1) / 2;                  // alpha w G at the points: 00 01 02 11 12 22
    double *X = Gw + 6 * NP;                           // the solution of the solve modes
    __shared__ double tBc[Q * Q], tBg[Q * K], tDx[K * (K + 1)], tMg[K * K];
    __shared__ double sX[24];
    __shared__ int dofd[NS], dofi[NS];                 // component and packed (i0, i1, i2) of a flux dof

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < Q * Q; i += NT) tBc[i] = P.Bc[i];
    for (int i = threadIdx.x; i < Q * K; i += NT) tBg[i] = P.Bg[i];
    for (int i = threadIdx.x; i < K * (K + 1); i += NT) tDx[i] = P.Dx[i];
    for (int i = threadIdx.x; i < K * K; i += NT) tMg[i] = P.Mg[i];
    for (int i = threadIdx.x; i < NS; i += NT) {
        const int d = i / NB, r = i % NB;
        const int n1 = d == 1 ? K + 1 : K, n2 = d == 2 ? K + 1 : K;
        dofd[i] = d;
        dofi[i] = ((r / (n1 * n2)) << 8) | (((r / n2) % n1) << 4) | (r % n2);
    }
    __syncthreads();

    const long long nunits = (long long)P.ncols * P.nlay;
    for (long long unit = blockIdx.x; unit < nunits; unit += gridDim.x) {
        const int ci = (int)(unit / P.nlay);
        const int layer = (int)(unit - (long long)ci * P.nlay);
        const int col = P.collist ? __ldg(P.collist + ci) : P.col0 + ci;
        for (int i = threadIdx.x; i < N * (N + 1) / 2; i += NT) T[i] = 0.0;
        for (int i = threadIdx.x; i < 24; i += NT) {
            const int v = i / 3, c = i - 3 * v;
            const long long gv = __ldg(P.map_c + (long long)col * 8 + v) + (long long)__ldg(P.off_c + v) * layer;
            sX[i] = __ldg(P.coords + gv * 3 + c);
        }
        __syncthreads();
        // the metric at the points (as FDB_FORM_MIXED_POISSON)
        for (int q = threadIdx.x; q < NP; q += NT) {
            const int qx = q / (Q * Q), qy = (q / Q) % Q, qz = q % Q;
            const double xi[3] = {P.xq[qx], P.xq[qy], P.xq[qz]};
            double J[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
#pragma unroll
            for (int v = 0; v < 8; v++) {
                const int b0 = (v >> 2) & 1, b1 = (v >> 1) & 1, b2 = v & 1;
                const double f0 = b0 ? xi[0] : 1.0 - xi[0], f1 = b1 ? xi[1] : 1.0 - xi[1];
                const double f2 = b2 ? xi[2] : 1.0 - xi[2];
                const double g0 = (b0 ? 1.0 : -1.0) * f1 * f2, g1 = (b1 ? 1.0 : -1.0) * f0 * f2;
                const double g2 = (b2 ? 1.0 : -1.0) * f0 * f1;
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    const double xc = sX[v * 3 + c];
                    J[c][0] = fma(xc, g0, J[c][0]);
                    J[c][1] = fma(xc, g1, J[c][1]);
                    J[c][2] = fma(xc, g2, J[c][2]);
                }
            }
            const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1]) -
                               J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0]) +
                               J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
            const double s = P.alpha * P.wq[qx] * P.wq[qy] * P.wq[qz] / det;
            int e = 0;
#pragma unroll
            for (int a = 0; a < 3; a++)
#pragma unroll
                for (int b = a; b < 3; b++, e++)
                    Gw[e * NP + q] = s * (J[0][a] * J[0][b] + J[1][a] * J[1][b] + J[2][a] * J[2][b]);
        }
        // B (metric-free Kronecker products), C or the right-hand side
        for (int e = threadIdx.x; e < NU * NS; e += NT) {
            const int v = e / NS, j = e % NS;
            const int d = dofd[j], ji = dofi[j];
            const int jx[3] = {ji >> 8, (ji >> 4) & 15, ji & 15}, vx[3] = {v / (K * K), (v / K) % K, v % K};
            double b = 1.0;
#pragma unroll
            for (int a = 0; a < 3; a++) b *= a == d ? tDx[vx[a] * (K + 1) + jx[a]] : tMg[vx[a] * K + jx[a]];
            T[tri(NS + v) + j] = b;
        }
        if (MODE == HY_CONDENSE) {
            for (int t = threadIdx.x; t < NF; t += NT) {
                int d, s, t0, t1;
                const int i = face_dof<K>(t, &d, &s, &t0, &t1);
                T[tri(NL + t) + i] = (s ? 1.0 : -1.0) * P.wg[t0] * P.wg[t1];
            }
        } else {
            // g = f_K (- C^T lambda): the last row
            double *g = T + tri(NL);
            for (int i = threadIdx.x; i < NS; i += NT) {
                const long long gs = __ldg(P.map_s + (long long)col * NS + i) + (long long)__ldg(P.off_s + i) * layer;
                g[i] = __ldg(P.w + gs) * __ldg(P.fs + gs);
            }
            for (int v = threadIdx.x; v < NU; v += NT)
                g[NS + v] = __ldg(P.fu + __ldg(P.map_u + (long long)col * NU + v) + (long long)__ldg(P.off_u + v) * layer);
            if (MODE == HY_RECONSTRUCT) {
                __syncthreads();
                for (int t = threadIdx.x; t < NF; t += NT) {
                    int d, s, t0, t1;
                    const int i = face_dof<K>(t, &d, &s, &t0, &t1);
                    const long long gt =
                        __ldg(P.map_t + (long long)col * NF + t) + (long long)__ldg(P.off_t + t) * layer;
                    g[i] -= (s ? 1.0 : -1.0) * P.wg[t0] * P.wg[t1] * __ldg(P.lam + gt);
                }
            }
        }
        __syncthreads();
        // A = alpha M entry by entry: sum over the points of G[d_i][d_j] phi_i phi_j
        for (int e = threadIdx.x; e < NS * (NS + 1) / 2; e += NT) {
            int i = (int)((sqrt(8.0 * e + 1.0) - 1.0) * 0.5);
            if (tri(i + 1) <= e) i++;
            if (tri(i) > e) i--;
            const int j = e - tri(i);
            const int di = dofd[i], dj = dofd[j], ii = dofi[i], jj = dofi[j];
            const int a = di < dj ? di : dj, b = di < dj ? dj : di;
            const double *G = Gw + (a == 0 ? b : (a == 1 ? 2 + b : 5)) * NP;
            const int i0 = ii >> 8, i1 = (ii >> 4) & 15, i2 = ii & 15;
            const int j0 = jj >> 8, j1 = (jj >> 4) & 15, j2 = jj & 15;
            double acc = 0.0;
            for (int q0 = 0; q0 < Q; q0++) {
                const double a0 = (di == 0 ? tBc[q0 * Q + i0] : tBg[q0 * K + i0]) *
                                  (dj == 0 ? tBc[q0 * Q + j0] : tBg[q0 * K + j0]);
                for (int q1 = 0; q1 < Q; q1++) {
                    const double a1 = a0 * (di == 1 ? tBc[q1 * Q + i1] : tBg[q1 * K + i1]) *
                                      (dj == 1 ? tBc[q1 * Q + j1] : tBg[q1 * K + j1]);
#pragma unroll
                    for (int q2 = 0; q2 < Q; q2++)
                        acc = fma(G[(q0 * Q + q1) * Q + q2] * a1,
                                  (di == 2 ? tBc[q2 * Q + i2] : tBg[q2 * K + i2]) *
                                      (dj == 2 ? tBc[q2 * Q + j2] : tBg[q2 * K + j2]),
                                  acc);
                }
            }
            T[e] = acc;
        }
        __syncthreads();
        // symmetric elimination of the NL local unknowns: row i -= (T[i][j] / T[j][j]) row j on the lower triangle
        for (int j = 0; j < NL; j++) {
            const double inv = 1.0 / T[tri(j) + j];
            for (int i = j + 1 + warp; i < N; i += NW) {
                const double m = T[tri(i) + j] * inv;
                double *Ti = T + tri(i);
                if (m != 0.0)
                    for (int l = j + 1 + lane; l <= i; l += 32) Ti[l] = fma(-m, T[tri(l) + j], Ti[l]);
            }
            __syncthreads();
        }
        if (MODE == HY_CONDENSE) {
            // H_K = -(trailing block): both triangles into the CSR
            for (int e = threadIdx.x; e < NF * NF; e += NT) {
                const int a = e / NF, b = e % NF;
                const double h = -T[tri(NL + (a > b ? a : b)) + NL + (a > b ? b : a)];
                const long long ga = __ldg(P.map_t + (long long)col * NF + a) + (long long)__ldg(P.off_t + a) * layer;
                const long long gb = __ldg(P.map_t + (long long)col * NF + b) + (long long)__ldg(P.off_t + b) * layer;
                const int r = P.row_lg ? __ldg(P.row_lg + ga) : (int)ga;
                const int c = P.col_lg ? __ldg(P.col_lg + gb) : (int)gb;
                if (r < 0 || c < 0) continue;
                long long lo = __ldg(P.rowptr + r), hi = __ldg(P.rowptr + r + 1);
                while (hi - lo > 1) {
                    const long long mid = (lo + hi) >> 1;
                    if (__ldg(P.colidx + mid) <= c) lo = mid;
                    else hi = mid;
                }
                atomicAdd(P.vals + lo, h);
            }
        } else {
            // back substitution x = L^-T D^-1 (L^-1 g) by one warp; the last row holds L^-1 g
            double *y = T + tri(NL);
            if (warp == 0)
                for (int i = NL - 1; i >= 0; i--) {
                    const double xi = y[i] / T[tri(i) + i];
                    const double *Ti = T + tri(i);
                    for (int j = lane; j < i; j += 32) y[j] = fma(-Ti[j], xi, y[j]);
                    if (lane == 0) X[i] = xi;
                    __syncwarp();
                }
            __syncthreads();
            if (MODE == HY_ELIMINATE) {
                for (int t = threadIdx.x; t < NF; t += NT) {
                    int d, s, t0, t1;
                    const int i = face_dof<K>(t, &d, &s, &t0, &t1);
                    const long long gt =
                        __ldg(P.map_t + (long long)col * NF + t) + (long long)__ldg(P.off_t + t) * layer;
                    atomicAdd(P.out + gt, (s ? 1.0 : -1.0) * P.wg[t0] * P.wg[t1] * X[i]);
                }
            } else {
                for (int i = threadIdx.x; i < NS; i += NT) {
                    const long long gs =
                        __ldg(P.map_s + (long long)col * NS + i) + (long long)__ldg(P.off_s + i) * layer;
                    atomicAdd(P.out + gs, __ldg(P.w + gs) * X[i]);
                }
                for (int v = threadIdx.x; v < NU; v += NT)
                    P.yu[__ldg(P.map_u + (long long)col * NU + v) + (long long)__ldg(P.off_u + v) * layer] += X[NS + v];
            }
        }
        __syncthreads();                                 // T is rebuilt for the next cell
    }
}

template <int K, int MODE>
int launch(const HybridParams<K> &P)
{
    using S = HybridShape<K>;
    fdb::Context &c = fdb::ctx();
    auto kern = hybrid_kernel<K, MODE>;
    constexpr size_t smem = hybrid_smem<K, MODE>();
    static bool attr = false;
    if (!attr) {
        FDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = true;
    }
    int per_sm = 0;
    FDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, S::THREADS, smem));
    long long grid = (long long)P.ncols * P.nlay;
    const long long cap = (long long)c.sm_count * (per_sm > 0 ? per_sm : 1);
    if (grid > cap) grid = cap;
    if (grid < 1) return 0;
    kern<<<(int)grid, S::THREADS, smem, c.stream>>>(P);
    FDB_LAUNCH_CHECK();
    return 0;
}

template <int K>
int run_k(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, void *const *args,
          const fdb_int *const *maps)
{
    constexpr int Q = K + 1;
    HybridParams<K> P;
    memset(&P, 0, sizeof(P));
    P.alpha = k->desc.alpha;
    for (int i = 0; i < Q * Q; i++) P.Bc[i] = k->desc.B[i];
    for (int i = 0; i < Q * K; i++) P.Bg[i] = k->B2[i];
    for (int q = 0; q < Q; q++) {
        P.wq[q] = k->desc.wq[q];
        P.xq[q] = k->desc.xq[q];
    }
    // the 1-D tables of B, exact with the k+1 point rule (as hdiv_hex.cu), and the GL weights int psi_b
    for (int v = 0; v < K; v++) {
        double sw = 0.0;
        for (int q = 0; q < Q; q++) sw += P.wq[q] * P.Bg[q * K + v];
        P.wg[v] = sw;
        for (int a = 0; a < K + 1; a++) {
            double s = 0.0;
            for (int q = 0; q < Q; q++) s += P.wq[q] * P.Bg[q * K + v] * k->desc.D[q * Q + a];
            P.Dx[v * (K + 1) + a] = s;
        }
        for (int b = 0; b < K; b++) {
            double s = 0.0;
            for (int q = 0; q < Q; q++) s += P.wq[q] * P.Bg[q * K + v] * P.Bg[q * K + b];
            P.Mg[v * K + b] = s;
        }
    }
    // offset0: the trace map's 6k^2 layer offsets, then the NCF map's 3k^2(k+1)
    P.off_t = k->d_off0;
    P.off_s = k->d_off0 + HybridShape<K>::NF;
    P.off_c = k->d_off1;
    P.off_u = k->d_off2;
    P.collist = subset;
    P.col0 = start;
    P.ncols = end - start;
    P.nlay = nlay;
    if (P.ncols <= 0 || nlay <= 0) return 0;
    P.coords = (const double *)args[1];
    P.map_c = maps[1];
    if (k->desc.rank == 2) {
        P.map_t = maps[0];
        fdb_mat_t mat = (fdb_mat_t)args[0];
        if (fdb_mat_device_view(mat, &P.rowptr, &P.colidx, &P.vals, &P.row_lg, &P.col_lg)) return 1;
        return launch<K, HY_CONDENSE>(P);
    }
    if (k->desc.form == FDB_FORM_MIXED_POISSON_HYBRID) {
        // [r, coords, f_sigma, w, f_u], maps [trace, coord, NCF, DQ]
        P.out = (double *)args[0];
        P.fs = (const double *)args[2];
        P.w = (const double *)args[3];
        P.fu = (const double *)args[4];
        P.map_t = maps[0];
        P.map_s = maps[2];
        P.map_u = maps[3];
        return launch<K, HY_ELIMINATE>(P);
    }
    // [y_sigma, coords, lambda, f_sigma, w, y_u, f_u], maps [NCF, coord, trace, DQ]
    P.out = (double *)args[0];
    P.lam = (const double *)args[2];
    P.fs = (const double *)args[3];
    P.w = (const double *)args[4];
    P.yu = (double *)args[5];
    P.fu = (const double *)args[6];
    P.map_s = maps[0];
    P.map_t = maps[2];
    P.map_u = maps[3];
    return launch<K, HY_RECONSTRUCT>(P);
}

}  // namespace

int fdb_launch_hybrid(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, void *const *args,
                      const fdb_int *const *maps)
{
    switch (k->desc.degree) {
    case 2: return run_k<2>(k, start, end, nlay, subset, args, maps);
    case 3: return run_k<3>(k, start, end, nlay, subset, args, maps);
    }
    fdb::set_error("mixed_poisson_hybrid kernel: degree %d not instantiated (2..3)", k->desc.degree);
    return 1;
}
