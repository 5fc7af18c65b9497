// FDB_FORM_MIXED_POISSON and FDB_FORM_MIXED_POISSON_SCHUR: mixed Poisson / Darcy on H(div) hexahedra, the flux
// sigma in NCF_k (k = 2..4, the "spectral" variant) and the scalar u in DQ_{k-1}, both on Gauss-Legendre points
// along their discontinuous axes (DESIGN.md section 4.21):
//
//   a((sigma, u), (tau, v)) = alpha*dot(sigma, tau)*dx + div(tau)*u*dx + div(sigma)*v*dx
//
// A flux dof is one component of the contravariant pull-back sigma^ = det J J^-1 sigma at its node.  Component d of
// sigma^ has k+1 CG_k (GLL) factors along axis d and k DG_{k-1} (GL) factors along the other two; its block of the
// local numbering is (i0 * n1 + i1) * n2 + i2 with n_d = k+1, n_e = k, blocks x, y, z one after the other.  With
// det J > 0 the Piola identities give
//   dot(sigma, tau) dx = sigma^T (J^T J / det J) tau^ dx^,    div(sigma) v dx = div^(sigma^) v dx^,
// so only the mass term needs the point metric G = J^T J / det J (6 entries); B is the same on every cell.
//
//   MIXED_POISSON  action     y_s = alpha M s + B^T u, y_u = B s at the (k+1)^3 Gauss points: six forward
//                             contractions of s (values and the axis-d derivative of component d), one of u; the
//                             metric at each point; seven transposed contractions
//                  diagonal   diag(alpha M): alpha w G_dd at the points contracted with the squared tables
//   MIXED_POISSON_SCHUR (metric-free, on the dofs, no points)
//                  action     t += B^T u, then y_u += B (w o t): the selfp Schur complement S_p = B W B^T when t is
//                             zero on entry and w = diag(alpha M)^-1.  Per component B is the Kronecker product
//                             Dx (x) Mg (x) Mg with Dx[v][a] = int psi_v phi_a', Mg[v][b] = int psi_v psi_b
//                  diagonal   y_u += diag(B W B^T) = sum_d (Dx^2 (x) Mg^2 (x) Mg^2) w_d, cell by cell
//
// Layout: one cell per CTA at a time (grid-stride over (column, layer) units), every contraction a three-stage
// sum-factorised pass over shared memory with all threads of the CTA.  The flux scatter goes through the NCF map:
// atomicAdd, or the colour / layer-parity schedule of the CG kernels (no two cells of a launch share a face);
// the DQ outputs belong to one cell each and are added without atomics.
#include "common.cuh"

namespace {

enum { HD_ACTION = 0, HD_DIAGONAL, HD_SCHUR_BT, HD_SCHUR_B, HD_SCHUR_DIAG };

template <int K>
struct HdivShape {
    static constexpr int Q = K + 1;                       // Gauss points per axis
    static constexpr int NP = Q * Q * Q;                  // points per cell
    static constexpr int NB = K * K * (K + 1);            // flux dofs per component block
    static constexpr int NS = 3 * NB;                     // flux dofs per cell
    static constexpr int NU = K * K * K;                  // DQ_{k-1} dofs per cell
    static constexpr int THREADS = K == 2 ? 32 : 128;   // k = 2: at most 27 elements per stage, one warp
};

template <int K>
struct HdivParams {
    double *ys;                  // flux output (action / diagonal / t of the Schur action)
    const double *s;             // flux input
    double *yu;                  // DQ output
    const double *u;             // DQ input
    const double *w;             // Schur forms: W, one value per flux dof
    const double *coords;        // AoS, 3 per vertex
    const fdb_int *map_s, *map_c, *map_u;   // NCF (3k^2(k+1)), vertex (8) and DQ (k^3) rows per column
    const fdb_int *off_s, *off_c, *off_u;   // layer offsets (zeros for native hexes)
    const fdb_int *collist;      // columns to visit (subset or colour) or NULL = col0 + i
    int col0, ncols;
    int nlay_items, lay_first, lay_step;
    double alpha;
    double Bc[(K + 1) * (K + 1)];   // CG_k at the points, [q][a]
    double Dc[(K + 1) * (K + 1)];   // its derivative, [q][a]
    double Bg[(K + 1) * K];         // DQ_{k-1} (GL) at the points, [q][b]
    double wq[K + 1], xq[K + 1];
    double Dx[K * (K + 1)];         // Schur: [v][a] = sum_q w_q psi_v(x_q) phi_a'(x_q)
    double Mg[K * K];               // Schur: [v][b] = sum_q w_q psi_v(x_q) psi_b(x_q)
};

// out[o0][o1][o2] (+)= sum A0[o0][i0] A1[o1][i1] A2[o2][i2] in[i0][i1][i2], all row-major, by the CTA's NT threads;
// t1, t2 hold the two intermediates.  Ends with a barrier.
template <int NT, int I0, int I1, int I2, int O0, int O1, int O2>
__device__ __forceinline__ void contract3(const double *A0, const double *A1, const double *A2, const double *in,
                                          double *out, double *t1, double *t2, bool acc)
{
    for (int e = threadIdx.x; e < I0 * I1 * O2; e += NT) {
        const int o2 = e % O2, r = e / O2;               // r = i0 * I1 + i1
        double v = 0.0;
#pragma unroll
        for (int i = 0; i < I2; i++) v = fma(A2[o2 * I2 + i], in[r * I2 + i], v);
        t1[e] = v;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < I0 * O1 * O2; e += NT) {
        const int o2 = e % O2, o1 = (e / O2) % O1, i0 = e / (O1 * O2);
        double v = 0.0;
#pragma unroll
        for (int i = 0; i < I1; i++) v = fma(A1[o1 * I1 + i], t1[(i0 * I1 + i) * O2 + o2], v);
        t2[e] = v;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < O0 * O1 * O2; e += NT) {
        const int r = e % (O1 * O2), o0 = e / (O1 * O2);
        double v = acc ? out[e] : 0.0;
#pragma unroll
        for (int i = 0; i < I0; i++) v = fma(A0[o0 * I0 + i], t2[i * O1 * O2 + r], v);
        out[e] = v;
    }
    __syncthreads();
}

// the tables of component block d: axis d carries the CG (or derivative) table C, the other axes G
template <int NT, int K, int D, bool FWD>
__device__ __forceinline__ void block(const double *C, const double *G, const double *in, double *out, double *t1,
                                      double *t2, bool acc)
{
    constexpr int Q = K + 1;
    constexpr int N0 = D == 0 ? K + 1 : K, N1 = D == 1 ? K + 1 : K, N2 = D == 2 ? K + 1 : K;
    const double *A0 = D == 0 ? C : G, *A1 = D == 1 ? C : G, *A2 = D == 2 ? C : G;
    if (FWD) contract3<NT, N0, N1, N2, Q, Q, Q>(A0, A1, A2, in, out, t1, t2, acc);
    else contract3<NT, Q, Q, Q, N0, N1, N2>(A0, A1, A2, in, out, t1, t2, acc);
}

// the same between the flux block d and the DQ dofs (the Schur forms: square K-tables on the GL axes)
template <int NT, int K, int D, bool TO_U>
__device__ __forceinline__ void dof_block(const double *C, const double *G, const double *in, double *out,
                                          double *t1, double *t2, bool acc)
{
    constexpr int N0 = D == 0 ? K + 1 : K, N1 = D == 1 ? K + 1 : K, N2 = D == 2 ? K + 1 : K;
    const double *A0 = D == 0 ? C : G, *A1 = D == 1 ? C : G, *A2 = D == 2 ? C : G;
    if (TO_U) contract3<NT, N0, N1, N2, K, K, K>(A0, A1, A2, in, out, t1, t2, acc);
    else contract3<NT, K, K, K, N0, N1, N2>(A0, A1, A2, in, out, t1, t2, acc);
}

template <int K, int MODE, bool ATOMIC>
__global__ void __launch_bounds__(HdivShape<K>::THREADS)
hdiv_kernel(const __grid_constant__ HdivParams<K> P)
{
    using S = HdivShape<K>;
    constexpr int Q = S::Q, NP = S::NP, NB = S::NB, NS = S::NS, NU = S::NU, NT = S::THREADS;
    constexpr int NC = (K + 1) * (K + 1), NG = (K + 1) * K, NX = K * (K + 1);
    constexpr bool POINTS = MODE == HD_ACTION || MODE == HD_DIAGONAL;
    // tables: forward [q][i] and transposed [i][q] (squared for the diagonals)
    __shared__ double tBc[NC], tDc[NC], tBg[NG], tBcT[NC], tDcT[NC], tBgT[NG];
    __shared__ double tDx[NX], tDxT[NX], tMg[K * K];
    __shared__ double sX[24];
    __shared__ double sS[NS], sU[NU];                 // gathered flux / DQ values (or W for the Schur diagonal)
    __shared__ double sP[POINTS ? 5 * NP : 1];         // at the points: 3 flux components, div, u
    __shared__ double sT1[NP], sT2[NP];               // every intermediate of a contraction fits (k+1)^3
    __shared__ double sYs[NS], sYu[NU];

    const bool square = MODE == HD_DIAGONAL || MODE == HD_SCHUR_DIAG;
    for (int i = threadIdx.x; i < NC; i += NT) {
        const int q = i / (K + 1), a = i % (K + 1);
        const double b = P.Bc[i], d = P.Dc[i];
        tBc[i] = b;
        tDc[i] = d;
        tBcT[a * Q + q] = square ? b * b : b;
        tDcT[a * Q + q] = d;
    }
    for (int i = threadIdx.x; i < NG; i += NT) {
        const int q = i / K, b = i % K;
        const double g = P.Bg[i];
        tBg[i] = g;
        tBgT[b * Q + q] = square ? g * g : g;
    }
    for (int i = threadIdx.x; i < NX; i += NT) {
        const int v = i / (K + 1), a = i % (K + 1);
        const double d = P.Dx[i];
        tDx[i] = square ? d * d : d;
        tDxT[a * K + v] = d;
    }
    for (int i = threadIdx.x; i < K * K; i += NT) tMg[i] = square ? P.Mg[i] * P.Mg[i] : P.Mg[i];
    __syncthreads();

    const long long nunits = (long long)P.ncols * P.nlay_items;
    for (long long unit = blockIdx.x; unit < nunits; unit += gridDim.x) {
        const int ci = (int)(unit / P.nlay_items);
        const int layer = P.lay_first + (int)(unit - (long long)ci * P.nlay_items) * P.lay_step;
        const int col = P.collist ? __ldg(P.collist + ci) : P.col0 + ci;
        // gather
        if (MODE == HD_ACTION || MODE == HD_SCHUR_B || MODE == HD_SCHUR_DIAG)
            for (int i = threadIdx.x; i < NS; i += NT) {
                const long long g = __ldg(P.map_s + (long long)col * NS + i) + (long long)__ldg(P.off_s + i) * layer;
                sS[i] = MODE == HD_ACTION ? __ldg(P.s + g)
                        : (MODE == HD_SCHUR_B ? __ldg(P.w + g) * P.ys[g] : __ldg(P.w + g));
            }
        if (MODE == HD_ACTION || MODE == HD_SCHUR_BT)
            for (int i = threadIdx.x; i < NU; i += NT)
                sU[i] = __ldg(P.u + __ldg(P.map_u + (long long)col * NU + i) + (long long)__ldg(P.off_u + i) * layer);
        if (POINTS)
            for (int i = threadIdx.x; i < 24; i += NT) {
                const int v = i / 3, c = i - 3 * v;
                const long long gv = __ldg(P.map_c + (long long)col * 8 + v) + (long long)__ldg(P.off_c + v) * layer;
                sX[i] = __ldg(P.coords + gv * 3 + c);
            }
        __syncthreads();

        if (MODE == HD_ACTION) {
            // the three components, the reference divergence and u at the points
            block<NT, K, 0, true>(tBc, tBg, sS, sP, sT1, sT2, false);
            block<NT, K, 1, true>(tBc, tBg, sS + NB, sP + NP, sT1, sT2, false);
            block<NT, K, 2, true>(tBc, tBg, sS + 2 * NB, sP + 2 * NP, sT1, sT2, false);
            block<NT, K, 0, true>(tDc, tBg, sS, sP + 3 * NP, sT1, sT2, false);
            block<NT, K, 1, true>(tDc, tBg, sS + NB, sP + 3 * NP, sT1, sT2, true);
            block<NT, K, 2, true>(tDc, tBg, sS + 2 * NB, sP + 3 * NP, sT1, sT2, true);
            contract3<NT, K, K, K, Q, Q, Q>(tBg, tBg, tBg, sU, sP + 4 * NP, sT1, sT2, false);
        }
        if (POINTS) {
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
                const double w = P.wq[qx] * P.wq[qy] * P.wq[qz];
                const double s = P.alpha * w / det;          // alpha w G = alpha w J^T J / det J
                double G[3][3];
#pragma unroll
                for (int a = 0; a < 3; a++)
#pragma unroll
                    for (int b = a; b < 3; b++) G[a][b] = s * (J[0][a] * J[0][b] + J[1][a] * J[1][b] + J[2][a] * J[2][b]);
                if (MODE == HD_ACTION) {
                    const double s0 = sP[q], s1 = sP[NP + q], s2 = sP[2 * NP + q];
                    sP[q] = G[0][0] * s0 + G[0][1] * s1 + G[0][2] * s2;
                    sP[NP + q] = G[0][1] * s0 + G[1][1] * s1 + G[1][2] * s2;
                    sP[2 * NP + q] = G[0][2] * s0 + G[1][2] * s1 + G[2][2] * s2;
                    sP[3 * NP + q] *= w;
                    sP[4 * NP + q] *= w;
                } else {
                    sP[q] = G[0][0];
                    sP[NP + q] = G[1][1];
                    sP[2 * NP + q] = G[2][2];
                }
            }
            __syncthreads();
            // test side: y_s,d = (values)^T alpha w G s + (axis-d derivative)^T w u;  y_u = (values)^T w div s
            block<NT, K, 0, false>(tBcT, tBgT, sP, sYs, sT1, sT2, false);
            block<NT, K, 1, false>(tBcT, tBgT, sP + NP, sYs + NB, sT1, sT2, false);
            block<NT, K, 2, false>(tBcT, tBgT, sP + 2 * NP, sYs + 2 * NB, sT1, sT2, false);
            if (MODE == HD_ACTION) {
                block<NT, K, 0, false>(tDcT, tBgT, sP + 4 * NP, sYs, sT1, sT2, true);
                block<NT, K, 1, false>(tDcT, tBgT, sP + 4 * NP, sYs + NB, sT1, sT2, true);
                block<NT, K, 2, false>(tDcT, tBgT, sP + 4 * NP, sYs + 2 * NB, sT1, sT2, true);
                contract3<NT, Q, Q, Q, K, K, K>(tBgT, tBgT, tBgT, sP + 3 * NP, sYu, sT1, sT2, false);
            }
        }
        if (MODE == HD_SCHUR_BT) {
            dof_block<NT, K, 0, false>(tDxT, tMg, sU, sYs, sT1, sT2, false);
            dof_block<NT, K, 1, false>(tDxT, tMg, sU, sYs + NB, sT1, sT2, false);
            dof_block<NT, K, 2, false>(tDxT, tMg, sU, sYs + 2 * NB, sT1, sT2, false);
        }
        if (MODE == HD_SCHUR_B || MODE == HD_SCHUR_DIAG) {
            dof_block<NT, K, 0, true>(tDx, tMg, sS, sYu, sT1, sT2, false);
            dof_block<NT, K, 1, true>(tDx, tMg, sS + NB, sYu, sT1, sT2, true);
            dof_block<NT, K, 2, true>(tDx, tMg, sS + 2 * NB, sYu, sT1, sT2, true);
        }
        // scatter
        if (MODE == HD_ACTION || MODE == HD_DIAGONAL || MODE == HD_SCHUR_BT)
            for (int i = threadIdx.x; i < NS; i += NT) {
                const long long g = __ldg(P.map_s + (long long)col * NS + i) + (long long)__ldg(P.off_s + i) * layer;
                if (ATOMIC) atomicAdd(P.ys + g, sYs[i]);
                else P.ys[g] += sYs[i];                 // colour and layer parity: no other writer
            }
        if (MODE != HD_DIAGONAL && MODE != HD_SCHUR_BT)
            for (int i = threadIdx.x; i < NU; i += NT) {
                const long long g = __ldg(P.map_u + (long long)col * NU + i) + (long long)__ldg(P.off_u + i) * layer;
                P.yu[g] += sYu[i];                       // a DQ dof belongs to this cell alone
            }
        __syncthreads();                                 // the buffers are refilled for the next cell
    }
}

template <int K, int MODE, bool ATOMIC>
int launch(const HdivParams<K> &P)
{
    using S = HdivShape<K>;
    fdb::Context &c = fdb::ctx();
    auto kern = hdiv_kernel<K, MODE, ATOMIC>;
    int per_sm = 0;
    FDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, S::THREADS, 0));
    long long grid = (long long)P.ncols * P.nlay_items;
    const long long cap = (long long)c.sm_count * (per_sm > 0 ? per_sm : 1);
    if (grid > cap) grid = cap;
    if (grid < 1) return 0;
    kern<<<(int)grid, S::THREADS, 0, c.stream>>>(P);
    FDB_LAUNCH_CHECK();
    return 0;
}

// every unit at once (a DQ output: no conflicts) or, for a flux scatter, atomic or the colour / parity schedule
template <int K, int MODE>
int run_mode(fdb_kernel_s *k, HdivParams<K> &P, fdb_int start, fdb_int end, int nlay, const fdb_int *subset)
{
    constexpr bool flux_out = MODE == HD_ACTION || MODE == HD_DIAGONAL || MODE == HD_SCHUR_BT;
    if (!flux_out || k->desc.scatter == FDB_SCATTER_ATOMIC) {
        P.collist = subset;
        P.col0 = start;
        P.ncols = end - start;
        P.nlay_items = nlay;
        P.lay_first = 0;
        P.lay_step = 1;
        if (P.ncols <= 0 || nlay <= 0) return 0;
        if constexpr (MODE == HD_ACTION || MODE == HD_DIAGONAL || MODE == HD_SCHUR_BT) return launch<K, MODE, true>(P);
        else return launch<K, MODE, false>(P);
    }
    if (subset) {
        fdb::set_error("mixed_poisson: coloured scatter does not support subsets");
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
            if (launch<K, MODE, false>(P)) return 1;
        }
    }
    return 0;
}

template <int K>
int run_k(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, void *const *args,
          const fdb_int *const *maps)
{
    constexpr int Q = K + 1;
    HdivParams<K> P;
    memset(&P, 0, sizeof(P));
    P.alpha = k->desc.alpha;
    for (int i = 0; i < Q * Q; i++) {
        P.Bc[i] = k->desc.B[i];
        P.Dc[i] = k->desc.D[i];
    }
    for (int i = 0; i < Q * K; i++) P.Bg[i] = k->B2[i];
    for (int q = 0; q < Q; q++) {
        P.wq[q] = k->desc.wq[q];
        P.xq[q] = k->desc.xq[q];
    }
    // the metric-free 1-D tables of B, exact with the k+1 point rule (polynomial degree 2k-1 at most)
    for (int v = 0; v < K; v++) {
        for (int a = 0; a < K + 1; a++) {
            double s = 0.0;
            for (int q = 0; q < Q; q++) s += P.wq[q] * P.Bg[q * K + v] * P.Dc[q * Q + a];
            P.Dx[v * (K + 1) + a] = s;
        }
        for (int b = 0; b < K; b++) {
            double s = 0.0;
            for (int q = 0; q < Q; q++) s += P.wq[q] * P.Bg[q * K + v] * P.Bg[q * K + b];
            P.Mg[v * K + b] = s;
        }
    }
    const bool schur = k->desc.form == FDB_FORM_MIXED_POISSON_SCHUR;
    const bool diag = k->desc.diagonal != 0;
    P.off_s = k->d_off0;
    P.off_c = k->d_off1;
    P.off_u = k->d_off2;
    if (!schur) {
        P.ys = (double *)args[0];
        P.coords = (const double *)args[1];
        P.map_s = maps[0];
        P.map_c = maps[1];
        if (diag) return run_mode<K, HD_DIAGONAL>(k, P, start, end, nlay, subset);
        P.s = (const double *)args[2];
        P.yu = (double *)args[3];
        P.u = (const double *)args[4];
        P.map_u = maps[2];
        return run_mode<K, HD_ACTION>(k, P, start, end, nlay, subset);
    }
    P.yu = (double *)args[0];
    P.map_u = maps[0];
    P.map_s = maps[1];
    if (diag) {
        P.w = (const double *)args[1];
        return run_mode<K, HD_SCHUR_DIAG>(k, P, start, end, nlay, subset);
    }
    P.u = (const double *)args[1];
    P.w = (const double *)args[2];
    P.ys = (double *)args[3];
    if (run_mode<K, HD_SCHUR_BT>(k, P, start, end, nlay, subset)) return 1;
    return run_mode<K, HD_SCHUR_B>(k, P, start, end, nlay, subset);
}

}  // namespace

int fdb_launch_hdiv(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, void *const *args,
                    const fdb_int *const *maps)
{
    switch (k->desc.degree) {
    case 2: return run_k<2>(k, start, end, nlay, subset, args, maps);
    case 3: return run_k<3>(k, start, end, nlay, subset, args, maps);
    case 4: return run_k<4>(k, start, end, nlay, subset, args, maps);
    }
    fdb::set_error("mixed_poisson kernel: degree %d not instantiated (2..4)", k->desc.degree);
    return 1;
}
