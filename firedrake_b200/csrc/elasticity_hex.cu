// FDB_FORM_ELASTICITY: linear elasticity on vector (cdim = 3) Q_p (x) P_p hexahedra,
//     a(u, v) = inner(sigma(u), grad v)*dx + beta*inner(u, v)*dx,
//     sigma(u) = mu (grad u + grad u^T) + lmbda tr(grad u) I
// (mu = desc.alpha, lmbda = desc.lmbda).  The first form of the engine whose element tensor couples
// the components: the stress at a Gauss point needs the full 3 x 3 physical gradient, so the three
// components cannot run through the slab-thread pipeline of action_hex.cu one after the other.
//
// Layout (DESIGN.md section 4.8): one thread per Gauss point, CPB cells ("slots") per CTA.  Per slot the
// CTA keeps in shared memory the 8 vertices, the three components' values at the points (S_U), a work
// buffer (S_T) and the nine reference fluxes (S_F, also the second work buffer of the sum-factorised
// passes).  Per unit:
//   gather u (AoS, three components)  ->  B (x) B (x) B, one axis per pass (three passes through S_T/S_F)
//   point: reference gradients of the three components by collocated differentiation (Dt = D B^{-1})
//          of S_U, geometry from the trilinear vertex field, G = ghat J^{-1}, sigma, the fluxes
//          fhat_d = w |det J| J^{-1} sigma_d into S_F and the mass term beta w |det J| u_d
//   Dt^T of the fluxes plus the mass term at the points, then B^T along each axis, and the scatter.
// The point stage holds the geometry once for the three components.
//
// MATRIX: one unit per trial dof (node j, component b) of a cell (3 N^3 units per cell); its gathered
// values are the unit vector e_(j,b), and the thread of test node i scatters entries (i, a; j, b),
// a = 0..2, into the 3 x 3 block at the node pair's CSR position (row-major inside the block).  Entries
// whose dof-level lgmap index is negative are dropped.  With vals == NULL the kernel adds the
// diagonal entry (j, b; j, b) into diag[3 j + b] instead.
//
// FDB_FORM_HYPERELASTICITY[_JACOBIAN] (DESIGN.md section 4.9) run through the same kernel with MODE
// EL_RESIDUAL / EL_JACOBIAN: the compressible Neo-Hookean residual and its exact Gateaux derivative,
//     F = I + grad u,  J = det F,  P(F) = mu (F - F^{-T}) + lmbda ln(J) F^{-T}
//     R(u; v)    = inner(P(F(u)), grad v)*dx + beta*inner(u, v)*dx
//     J(u)[w; v] = inner(dP[grad w], grad v)*dx + beta*inner(w, v)*dx,
//     dP[H] = mu H + (mu - lmbda ln J) F^{-T} H^T F^{-T} + lmbda tr(F^{-1} H) F^{-T}.
// Only the point stage differs: P (or dP) goes into the nine fluxes where sigma goes.  The residual's
// gathered values are u itself.  The Jacobian also gathers u (through the same node map, again for every
// trial-dof unit in MATRIX mode) into a fourth per-slot buffer S_V; its forward passes share S_T/S_F
// with those of w, and F comes from the collocated derivative of S_V.  J <= 0 at a point gives NaN
// (ln of a negative number), as in Firedrake: the kernel does not guard it.
//
// FDB_FORM_STOKES (DESIGN.md section 4.11) runs with MODE EL_STOKES: the Taylor-Hood saddle-point action
// on velocity u (vector CG_p, the node map) and pressure p (scalar CG_{p-1}, a second map map2),
//     a((u, p), (v, q)) = mu inner(grad u, grad v)*dx + beta inner(u, v)*dx - p div(v)*dx - q div(u)*dx.
// p's (N-1)^3 values are gathered into a fifth per-slot buffer laid out as an N^3 block whose entries
// with a dof index N-1 along any axis are zero, so the rectangular (N, N-1) table Bq runs through the
// same square passes as B: Bq is padded with a zero last column.  The point stage puts mu G - p I into
// the fluxes where sigma goes and replaces p by its test value -w |det J| tr G, which goes back through
// Bq^T along z, y, x; the threads of the (N-1)^3 pressure dofs scatter it into yp.
//
// FDB_FORM_NAVIER_STOKES[_JACOBIAN] (DESIGN.md section 4.12) run with MODE EL_NS_RESIDUAL / EL_NS_JACOBIAN:
// steady incompressible Navier-Stokes on the same spaces and its exact Newton Jacobian at u,
//     R((u, p); (v, q))      = Stokes((u, p); (v, q)) + inner(dot(grad u, u), v)*dx
//     J(u)[(w, r); (v, q)]   = Stokes((w, r); (v, q)) + inner(dot(grad w, u), v)*dx + inner(dot(grad u, w), v)*dx
// (mu = nu).  Gather, passes and scatter are those of EL_STOKES; only the value slot of the point stage
// gains the convective term, w |det J| sum_k G[d][k] u_k (residual) or w |det J| sum_k (G_w[d][k] u_k +
// G_u[d][k] w_k) (Jacobian).  The Jacobian gathers u into S_V as EL_JACOBIAN does (its forward passes share
// S_F[3..9)), takes G_u from the collocated derivative of S_V, and keeps S_P / S_Q after S_V.
//
// FDB_FORM_BOUSSINESQ[_JACOBIAN] (DESIGN.md section 4.22) run with MODE EL_RB_RESIDUAL / EL_RB_JACOBIAN: the
// Boussinesq (Rayleigh-Benard) system, Navier-Stokes coupled to a temperature T in CG_{p-1} on the pressure
// numbering, with bg = (Ra/Pr) g and kT = 1/Pr,
//     R((u, p, T); (v, q, S)) = NS((u, p); (v, q)) - T inner(bg, v)*dx + dot(grad T, u) S*dx
//                               + kT inner(grad T, grad S)*dx
//     J(u, T)[(w, r, s); ...]  = NS-Jacobian(u)[(w, r); (v, q)] - s inner(bg, v)*dx
//                               + (dot(grad s, u) + dot(grad T, w)) S*dx + kT inner(grad s, grad S)*dx.
// T (s, and the Jacobian's T) is gathered through map2 into a padded N^3 block like p and runs through the
// Bq passes in two more per-slot buffers S_A / S_B (the Jacobian's T through S_TF as work, into S_T0); its
// physical gradient comes from the collocated derivative Dt of the point values (exact: degree p-1 <= N-1).
// The point stage subtracts bg T from the velocity value slot, and gives T's test function a value
// u . grad T and three reference fluxes kT w |det J| J^{-1} J^{-T} grad^ T in S_TF; Dt^T and Bq^T take them
// back, and the threads of the pressure dofs scatter into y_T.
#include "common.cuh"

namespace {

template <int N>
struct ElasParams {
    double *y;                   // action / diagonal output (AoS, 3 per node)
    const double *x;             // action input (AoS)
    const double *coords;        // AoS, 3 per vertex
    const fdb_int *map0, *map1;  // node map (ND per column / cell), vertex map (8)
    const fdb_int *off0, *off1;  // layer offsets (zeros for native hexes)
    const fdb_int *collist;      // columns to visit (subset / colour) or NULL = col0 + i
    int col0, ncols;
    int nlay_items, lay_first, lay_step;   // layers lay_first + lay_step * k, k < nlay_items
    double mu, lmbda, beta;
    double B[N * N], Dt[N * N], wq[N];
    double xq[N];
    // MATRIX
    const long long *rowptr;
    const fdb_int *colidx;
    double *vals;                // NULL: diagonal into y
    const fdb_int *row_lg, *col_lg;   // dof-level, NULL = identity
    const unsigned short *rank_tab;
    int nvar, nlay_total;
    const double *u;             // EL_JACOBIAN, EL_NS_JACOBIAN, EL_RB_JACOBIAN: the linearisation point (AoS, node map)
    // EL_STOKES, EL_NS_*: the pressure action output and input (one value per node of map2, (N-1)^3 per cell)
    double *yp;
    const double *xp;
    const fdb_int *map2, *off2;
    double Bq[N * N];            // pressure basis at the points, (N, N-1) padded with a zero last column
    // EL_RB_*: the temperature output and input (through map2), the Jacobian's linearisation temperature, and
    // the buoyancy vector (Ra/Pr) g; 1/Pr is lmbda
    double *yt;
    const double *xt, *t0;
    double bg[3];
};

enum { EL_LINEAR = 0, EL_RESIDUAL = 1, EL_JACOBIAN = 2, EL_STOKES = 3, EL_NS_RESIDUAL = 4, EL_NS_JACOBIAN = 5,
       EL_RB_RESIDUAL = 6, EL_RB_JACOBIAN = 7 };

// the modes that also gather u into S_V (a Jacobian's linearisation point), those on the Taylor-Hood pair, and
// those with a temperature on the pressure numbering
__host__ __device__ constexpr bool el_holds_u(int mode)
{
    return mode == EL_JACOBIAN || mode == EL_NS_JACOBIAN || mode == EL_RB_JACOBIAN;
}
__host__ __device__ constexpr bool el_pressure(int mode)
{
    return mode == EL_STOKES || mode == EL_NS_RESIDUAL || mode == EL_NS_JACOBIAN || mode == EL_RB_RESIDUAL ||
           mode == EL_RB_JACOBIAN;
}
__host__ __device__ constexpr bool el_temperature(int mode) { return mode == EL_RB_RESIDUAL || mode == EL_RB_JACOBIAN; }

template <int N, int MODE = EL_LINEAR>
struct ElasShape {
    static constexpr int ND = N * N * N;
    static constexpr int CPB = (256 / ND) > 0 ? 256 / ND : 1;          // cells (slots) per CTA
    static constexpr int THREADS = ((CPB * ND + 31) / 32) * 32;
    // doubles per slot: vertices, values at the points, work buffer, fluxes (9 per point); the Jacobians
    // also hold u's values (S_V), the Taylor-Hood modes the pressure and its work buffer (S_P, S_Q, after S_V),
    // the Boussinesq modes the temperature's two buffers and three fluxes (S_A, S_B, S_TF) and the Jacobian's
    // linearisation temperature (S_T0)
    static constexpr int SLOT = 24 + 3 * ND + 3 * ND + 9 * ND + (el_holds_u(MODE) ? 3 * ND : 0) +
                                (el_pressure(MODE) ? 2 * ND : 0) + (el_temperature(MODE) ? 5 * ND : 0) +
                                (MODE == EL_RB_JACOBIAN ? ND : 0);
    static constexpr size_t SMEM = (size_t)CPB * SLOT * sizeof(double) + (size_t)CPB * ND * sizeof(int);
};

// out[i][j][k] (one value per thread, the thread's (i, j, k)) = sum_a T[a-index along `axis`] in[...]:
// tr = false: T[q][a] applied to the a-index (dofs -> points); tr = true: T^T (points -> dofs)
template <int N, int AXIS, bool TR>
__device__ __forceinline__ double pass1(const double *__restrict__ T, const double *in, int i, int j, int k)
{
    constexpr int ST = AXIS == 0 ? N * N : (AXIS == 1 ? N : 1);
    const int o = AXIS == 0 ? i : (AXIS == 1 ? j : k);
    const int base = (i * N + j) * N + k - o * ST;
    double s = 0.0;
#pragma unroll
    for (int a = 0; a < N; a++) s = fma(TR ? T[a * N + o] : T[o * N + a], in[base + a * ST], s);
    return s;
}

// cof[i][j] = cofactor of F[i][j]: F^{-T} = cof / det F, F^{-1}[i][j] = cof[j][i] / det F; returns det F
__device__ __forceinline__ double cofactors(const double F[3][3], double cof[3][3])
{
    cof[0][0] = F[1][1] * F[2][2] - F[1][2] * F[2][1];
    cof[0][1] = F[1][2] * F[2][0] - F[1][0] * F[2][2];
    cof[0][2] = F[1][0] * F[2][1] - F[1][1] * F[2][0];
    cof[1][0] = F[0][2] * F[2][1] - F[0][1] * F[2][2];
    cof[1][1] = F[0][0] * F[2][2] - F[0][2] * F[2][0];
    cof[1][2] = F[0][1] * F[2][0] - F[0][0] * F[2][1];
    cof[2][0] = F[0][1] * F[1][2] - F[0][2] * F[1][1];
    cof[2][1] = F[0][2] * F[1][0] - F[0][0] * F[1][2];
    cof[2][2] = F[0][0] * F[1][1] - F[0][1] * F[1][0];
    return F[0][0] * cof[0][0] + F[0][1] * cof[0][1] + F[0][2] * cof[0][2];
}

template <int N, bool MATRIX, bool ATOMIC, int MODE = EL_LINEAR>
__global__ void __launch_bounds__(ElasShape<N>::THREADS)
elasticity_kernel(const __grid_constant__ ElasParams<N> P)
{
    using S = ElasShape<N, MODE>;
    constexpr int ND = S::ND;
    constexpr int CPB = S::CPB;
    constexpr bool JAC = el_holds_u(MODE);                 // EL_JACOBIAN, EL_NS_JACOBIAN: u in S_V
    constexpr bool STK = el_pressure(MODE);                // EL_STOKES, EL_NS_*, EL_RB_*: the pressure space
    constexpr bool TMP = el_temperature(MODE);             // EL_RB_*: the temperature on the pressure numbering
    constexpr bool RBJ = MODE == EL_RB_JACOBIAN;
    constexpr int NP = N - 1;                              // pressure dofs per axis (EL_STOKES, EL_NS_*)
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int slot = threadIdx.x / ND;
    const int l = threadIdx.x - slot * ND;                 // this thread's dof / point in the cell
    const bool in_cta = slot < CPB;
    const int sl = in_cta ? slot : 0;
    double *sb = reinterpret_cast<double *>(smem_raw) + (size_t)sl * S::SLOT;
    double *s_x = sb;                                      // [8][3]
    double *s_u = s_x + 24;                                // [3][ND]
    double *s_t = s_u + 3 * ND;                            // [3][ND]
    double *s_f = s_t + 3 * ND;                            // [3 d][3 m][ND]
    double *s_v = s_f + 9 * ND;                            // [3][ND], the modes that hold u only
    double *s_p = s_f + 9 * ND + (MODE == EL_NS_JACOBIAN || RBJ ? 3 * ND : 0);   // [ND], pressure modes: pressure
    double *s_q = s_p + ND;                                // [ND], pressure modes: its work buffer
    double *s_a = s_q + ND;                                // [ND], EL_RB_*: the temperature (s) and
    double *s_b = s_a + ND;                                // [ND]  its work buffer
    double *s_tf = s_b + ND;                               // [3 m][ND], EL_RB_*: its reference fluxes
    double *s_t0 = s_tf + 3 * ND;                          // [ND], EL_RB_JACOBIAN: the linearisation temperature
    int *s_idx = reinterpret_cast<int *>(reinterpret_cast<double *>(smem_raw) + (size_t)CPB * S::SLOT) + sl * ND;
    const int qi = l / (N * N), qj = (l / N) % N, qk = l % N;
    // pressure modes: this thread's pressure dof, if its (i, j, k) is one
    const bool pdof = STK && qi < NP && qj < NP && qk < NP;
    const int lp = (qi * NP + qj) * NP + qk;

    const long long ncells = (long long)P.ncols * P.nlay_items;
    const long long nunits = MATRIX ? ncells * 3 * ND : ncells;
    for (long long base = (long long)blockIdx.x * CPB; base < nunits; base += (long long)gridDim.x * CPB) {
        const long long unit = base + slot;
        const bool valid = in_cta && unit < nunits;
        const long long cell = MATRIX ? unit / (3 * ND) : unit;
        const int jb = MATRIX ? (int)(unit - cell * 3 * ND) : 0;   // trial dof: node jb / 3, component jb % 3
        int col = 0, layer = 0;
        if (valid) {
            const int ci = (int)(cell / P.nlay_items);
            layer = P.lay_first + P.lay_step * (int)(cell - (long long)ci * P.nlay_items);
            col = P.collist ? __ldg(P.collist + ci) : P.col0 + ci;
        }
        // ---- gather: node index, values (or the unit vector), vertices
        int g = 0, gp = 0;
        if (valid) {
            g = __ldg(P.map0 + (long long)col * ND + l) + __ldg(P.off0 + l) * layer;
            s_idx[l] = g;
#pragma unroll
            for (int d = 0; d < 3; d++)
                s_u[d * ND + l] = MATRIX ? ((jb == 3 * l + d) ? 1.0 : 0.0) : __ldg(P.x + (long long)g * 3 + d);
            if (JAC) {
#pragma unroll
                for (int d = 0; d < 3; d++) s_v[d * ND + l] = __ldg(P.u + (long long)g * 3 + d);
            }
            if (STK) {
                if (pdof) gp = __ldg(P.map2 + (long long)col * (NP * NP * NP) + lp) + __ldg(P.off2 + lp) * layer;
                s_p[l] = pdof ? __ldg(P.xp + gp) : 0.0;
            }
            if (TMP) s_a[l] = pdof ? __ldg(P.xt + gp) : 0.0;
            if (RBJ) s_t0[l] = pdof ? __ldg(P.t0 + gp) : 0.0;
            for (int i = l; i < 24; i += ND) {
                const int v = i / 3, a = i - 3 * v;
                const int gv = __ldg(P.map1 + (long long)col * 8 + v) + __ldg(P.off1 + v) * layer;
                s_x[i] = __ldg(P.coords + (long long)gv * 3 + a);
            }
        } else if (in_cta) {
            // idle slot: the unit cube with zero values keeps the point stage finite
#pragma unroll
            for (int d = 0; d < 3; d++) s_u[d * ND + l] = 0.0;
            if (JAC) {
#pragma unroll
                for (int d = 0; d < 3; d++) s_v[d * ND + l] = 0.0;
            }
            if (STK) s_p[l] = 0.0;
            if (TMP) s_a[l] = 0.0;
            if (RBJ) s_t0[l] = 0.0;
            for (int i = l; i < 24; i += ND) s_x[i] = (double)(((i / 3) >> (2 - i % 3)) & 1);
        }
        __syncthreads();
        // ---- forward: values at the points, x then y then z (S_U -> S_T -> S_F -> S_U; the Jacobian's u:
        //      S_V -> S_F[3..6) -> S_F[6..9) -> S_V)
        if (in_cta) {
#pragma unroll
            for (int d = 0; d < 3; d++) s_t[d * ND + l] = pass1<N, 0, false>(P.B, s_u + d * ND, qi, qj, qk);
            if (JAC) {
#pragma unroll
                for (int d = 0; d < 3; d++)
                    s_f[(3 + d) * ND + l] = pass1<N, 0, false>(P.B, s_v + d * ND, qi, qj, qk);
            }
            if (STK) s_q[l] = pass1<N, 0, false>(P.Bq, s_p, qi, qj, qk);
            if (TMP) s_b[l] = pass1<N, 0, false>(P.Bq, s_a, qi, qj, qk);
            if (RBJ) s_tf[l] = pass1<N, 0, false>(P.Bq, s_t0, qi, qj, qk);
        }
        __syncthreads();
        if (in_cta) {
#pragma unroll
            for (int d = 0; d < 3; d++) s_f[d * ND + l] = pass1<N, 1, false>(P.B, s_t + d * ND, qi, qj, qk);
            if (JAC) {
#pragma unroll
                for (int d = 0; d < 3; d++)
                    s_f[(6 + d) * ND + l] = pass1<N, 1, false>(P.B, s_f + (3 + d) * ND, qi, qj, qk);
            }
            if (STK) s_p[l] = pass1<N, 1, false>(P.Bq, s_q, qi, qj, qk);
            if (TMP) s_a[l] = pass1<N, 1, false>(P.Bq, s_b, qi, qj, qk);
            if (RBJ) s_tf[ND + l] = pass1<N, 1, false>(P.Bq, s_tf, qi, qj, qk);
        }
        __syncthreads();
        if (in_cta) {
#pragma unroll
            for (int d = 0; d < 3; d++) s_u[d * ND + l] = pass1<N, 2, false>(P.B, s_f + d * ND, qi, qj, qk);
            if (JAC) {
#pragma unroll
                for (int d = 0; d < 3; d++)
                    s_v[d * ND + l] = pass1<N, 2, false>(P.B, s_f + (6 + d) * ND, qi, qj, qk);
            }
            if (STK) s_q[l] = pass1<N, 2, false>(P.Bq, s_p, qi, qj, qk);
            if (TMP) s_b[l] = pass1<N, 2, false>(P.Bq, s_a, qi, qj, qk);
            if (RBJ) s_t0[l] = pass1<N, 2, false>(P.Bq, s_tf + ND, qi, qj, qk);
        }
        __syncthreads();
        // ---- point stage
        double mres[3] = {0.0, 0.0, 0.0};
        double tres = 0.0;                                 // EL_RB_*: the temperature's test value
        if (in_cta) {
            double gh[3][3];                               // gh[d][m] = d u_d / d xi_m
#pragma unroll
            for (int d = 0; d < 3; d++) {
                gh[d][0] = pass1<N, 0, false>(P.Dt, s_u + d * ND, qi, qj, qk);
                gh[d][1] = pass1<N, 1, false>(P.Dt, s_u + d * ND, qi, qj, qk);
                gh[d][2] = pass1<N, 2, false>(P.Dt, s_u + d * ND, qi, qj, qk);
            }
            // J[c][r] = d x_c / d xi_r of the trilinear vertex field (vertex (bx*2 + by)*2 + bz)
            const double xi[3] = {P.xq[qi], P.xq[qj], P.xq[qk]};
            double J[3][3];
#pragma unroll
            for (int c = 0; c < 3; c++)
#pragma unroll
                for (int r = 0; r < 3; r++) J[c][r] = 0.0;
#pragma unroll
            for (int v = 0; v < 8; v++) {
                const int b[3] = {(v >> 2) & 1, (v >> 1) & 1, v & 1};
                double dphi[3];
#pragma unroll
                for (int r = 0; r < 3; r++) {
                    double s = b[r] ? 1.0 : -1.0;
#pragma unroll
                    for (int e = 0; e < 3; e++)
                        if (e != r) s *= b[e] ? xi[e] : 1.0 - xi[e];
                    dphi[r] = s;
                }
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    const double X = s_x[v * 3 + c];
#pragma unroll
                    for (int r = 0; r < 3; r++) J[c][r] = fma(X, dphi[r], J[c][r]);
                }
            }
            // cofactor rows: R[m] . J[:, r] = det * delta_mr, so J^{-1}[m][c] = R[m][c] / det
            double R[3][3];
            R[0][0] = J[1][1] * J[2][2] - J[2][1] * J[1][2];
            R[0][1] = J[2][1] * J[0][2] - J[0][1] * J[2][2];
            R[0][2] = J[0][1] * J[1][2] - J[1][1] * J[0][2];
            R[1][0] = J[1][2] * J[2][0] - J[2][2] * J[1][0];
            R[1][1] = J[2][2] * J[0][0] - J[0][2] * J[2][0];
            R[1][2] = J[0][2] * J[1][0] - J[1][2] * J[0][0];
            R[2][0] = J[1][0] * J[2][1] - J[2][0] * J[1][1];
            R[2][1] = J[2][0] * J[0][1] - J[0][0] * J[2][1];
            R[2][2] = J[0][0] * J[1][1] - J[1][0] * J[0][1];
            const double det = J[0][0] * R[0][0] + J[1][0] * R[0][1] + J[2][0] * R[0][2];
            const double rdet = 1.0 / det;
            const double w = P.wq[qi] * P.wq[qj] * P.wq[qk];
            // physical gradient G[d][k] = sum_m gh[d][m] J^{-1}[m][k]
            double G[3][3];
#pragma unroll
            for (int d = 0; d < 3; d++)
#pragma unroll
                for (int k = 0; k < 3; k++)
                    G[d][k] = (gh[d][0] * R[0][k] + gh[d][1] * R[1][k] + gh[d][2] * R[2][k]) * rdet;
            if (MODE == EL_LINEAR) {
            const double ltr = P.lmbda * (G[0][0] + G[1][1] + G[2][2]);
            // fhat_d[m] = w |det| sum_k J^{-1}[m][k] sigma[d][k] = (w |det| / det) sum_k R[m][k] sigma[d][k]
            const double sw = w * fabs(det) * rdet;
#pragma unroll
            for (int d = 0; d < 3; d++) {
                double sg[3];
#pragma unroll
                for (int k = 0; k < 3; k++) sg[k] = P.mu * (G[d][k] + G[k][d]) + (k == d ? ltr : 0.0);
#pragma unroll
                for (int m = 0; m < 3; m++)
                    s_f[(d * 3 + m) * ND + l] = sw * (R[m][0] * sg[0] + R[m][1] * sg[1] + R[m][2] * sg[2]);
                mres[d] = P.beta * w * fabs(det) * s_u[d * ND + l];
            }
            } else if (MODE == EL_STOKES) {
                // flux mu G - p I; the pressure's test value -w |det| div u replaces p in S_P
                const double pv = s_q[l];
                const double sw = w * fabs(det) * rdet;
#pragma unroll
                for (int d = 0; d < 3; d++) {
                    double sg[3];
#pragma unroll
                    for (int k = 0; k < 3; k++) sg[k] = P.mu * G[d][k] - (k == d ? pv : 0.0);
#pragma unroll
                    for (int m = 0; m < 3; m++)
                        s_f[(d * 3 + m) * ND + l] = sw * (R[m][0] * sg[0] + R[m][1] * sg[1] + R[m][2] * sg[2]);
                    mres[d] = P.beta * w * fabs(det) * s_u[d * ND + l];
                }
                s_p[l] = -w * fabs(det) * (G[0][0] + G[1][1] + G[2][2]);
            } else if (STK) {
                // Navier-Stokes: the Stokes flux and pressure test value; the value slot adds the convective
                // term, (grad u) u (residual: G is grad u) or (grad w) u + (grad u) w (Jacobian: G is grad w,
                // u and its gradient come from S_V)
                const double pv = s_q[l];
                const double wd = w * fabs(det);
                const double sw = wd * rdet;
                double uq[3], cv[3];
#pragma unroll
                for (int k = 0; k < 3; k++) uq[k] = JAC ? s_v[k * ND + l] : s_u[k * ND + l];
#pragma unroll
                for (int d = 0; d < 3; d++) cv[d] = G[d][0] * uq[0] + G[d][1] * uq[1] + G[d][2] * uq[2];
                if (JAC) {
#pragma unroll
                    for (int d = 0; d < 3; d++) {
                        const double g0 = pass1<N, 0, false>(P.Dt, s_v + d * ND, qi, qj, qk);
                        const double g1 = pass1<N, 1, false>(P.Dt, s_v + d * ND, qi, qj, qk);
                        const double g2 = pass1<N, 2, false>(P.Dt, s_v + d * ND, qi, qj, qk);
#pragma unroll
                        for (int k = 0; k < 3; k++)
                            cv[d] = fma((g0 * R[0][k] + g1 * R[1][k] + g2 * R[2][k]) * rdet, s_u[k * ND + l], cv[d]);
                    }
                }
                if (TMP) {
                    // Boussinesq: buoyancy -bg T in the value slot; T's test value u . grad T (Jacobian: u0 . grad s
                    // + w . grad T0) and fluxes kT w |det| J^{-1} grad T (grad s) in S_TF
                    const double tv = s_b[l];
                    double gt[3];
                    {
                        const double h0 = pass1<N, 0, false>(P.Dt, s_b, qi, qj, qk);
                        const double h1 = pass1<N, 1, false>(P.Dt, s_b, qi, qj, qk);
                        const double h2 = pass1<N, 2, false>(P.Dt, s_b, qi, qj, qk);
#pragma unroll
                        for (int k = 0; k < 3; k++) gt[k] = (h0 * R[0][k] + h1 * R[1][k] + h2 * R[2][k]) * rdet;
                    }
                    double tr = uq[0] * gt[0] + uq[1] * gt[1] + uq[2] * gt[2];
                    if (RBJ) {
                        const double h0 = pass1<N, 0, false>(P.Dt, s_t0, qi, qj, qk);
                        const double h1 = pass1<N, 1, false>(P.Dt, s_t0, qi, qj, qk);
                        const double h2 = pass1<N, 2, false>(P.Dt, s_t0, qi, qj, qk);
#pragma unroll
                        for (int k = 0; k < 3; k++)
                            tr = fma((h0 * R[0][k] + h1 * R[1][k] + h2 * R[2][k]) * rdet, s_u[k * ND + l], tr);
                    }
                    tres = wd * tr;
                    const double kw = P.lmbda * sw;
#pragma unroll
                    for (int m = 0; m < 3; m++)
                        s_tf[m * ND + l] = kw * (R[m][0] * gt[0] + R[m][1] * gt[1] + R[m][2] * gt[2]);
#pragma unroll
                    for (int d = 0; d < 3; d++) cv[d] = fma(-P.bg[d], tv, cv[d]);
                }
#pragma unroll
                for (int d = 0; d < 3; d++) {
                    double sg[3];
#pragma unroll
                    for (int k = 0; k < 3; k++) sg[k] = P.mu * G[d][k] - (k == d ? pv : 0.0);
#pragma unroll
                    for (int m = 0; m < 3; m++)
                        s_f[(d * 3 + m) * ND + l] = sw * (R[m][0] * sg[0] + R[m][1] * sg[1] + R[m][2] * sg[2]);
                    mres[d] = wd * (P.beta * s_u[d * ND + l] + cv[d]);
                }
                s_p[l] = -wd * (G[0][0] + G[1][1] + G[2][2]);
            } else {
                // deformation gradient Fd = I + grad u: u's gradient is G (residual) or comes from S_V
                double Fd[3][3];
                if (JAC) {
#pragma unroll
                    for (int d = 0; d < 3; d++) {
                        const double g0 = pass1<N, 0, false>(P.Dt, s_v + d * ND, qi, qj, qk);
                        const double g1 = pass1<N, 1, false>(P.Dt, s_v + d * ND, qi, qj, qk);
                        const double g2 = pass1<N, 2, false>(P.Dt, s_v + d * ND, qi, qj, qk);
#pragma unroll
                        for (int k = 0; k < 3; k++)
                            Fd[d][k] = (k == d ? 1.0 : 0.0) + (g0 * R[0][k] + g1 * R[1][k] + g2 * R[2][k]) * rdet;
                    }
                } else {
#pragma unroll
                    for (int d = 0; d < 3; d++)
#pragma unroll
                        for (int k = 0; k < 3; k++) Fd[d][k] = (k == d ? 1.0 : 0.0) + G[d][k];
                }
                double cof[3][3];
                const double detF = cofactors(Fd, cof);
                const double rJ = 1.0 / detF;
                const double lnJ = log(detF);
                // Pk[d][k]: the first Piola-Kirchhoff stress (residual) or dP[H] with H = G (Jacobian)
                double Pk[3][3];
                if (JAC) {
                    // tr(F^{-1} H) = cof : H / J;  C = F^{-1} H F^{-1}, C^T = F^{-T} H^T F^{-T}
                    double trA = 0.0;
#pragma unroll
                    for (int a = 0; a < 3; a++)
#pragma unroll
                        for (int b = 0; b < 3; b++) trA = fma(cof[a][b], G[a][b], trA);
                    trA *= rJ;
                    double T[3][3];                        // T = H F^{-1} * J
#pragma unroll
                    for (int a = 0; a < 3; a++)
#pragma unroll
                        for (int d = 0; d < 3; d++)
                            T[a][d] = G[a][0] * cof[d][0] + G[a][1] * cof[d][1] + G[a][2] * cof[d][2];
                    const double c1 = (P.mu - P.lmbda * lnJ) * rJ * rJ;
                    const double c2 = P.lmbda * trA * rJ;
#pragma unroll
                    for (int d = 0; d < 3; d++)
#pragma unroll
                        for (int k = 0; k < 3; k++)   // C[k][d] = sum_a F^{-1}[k][a] T[a][d] / J
                            Pk[d][k] = P.mu * G[d][k] +
                                       c1 * (cof[0][k] * T[0][d] + cof[1][k] * T[1][d] + cof[2][k] * T[2][d]) +
                                       c2 * cof[d][k];
                } else {
                    const double c = (P.lmbda * lnJ - P.mu) * rJ;
#pragma unroll
                    for (int d = 0; d < 3; d++)
#pragma unroll
                        for (int k = 0; k < 3; k++) Pk[d][k] = P.mu * Fd[d][k] + c * cof[d][k];
                }
                const double sw = w * fabs(det) * rdet;
#pragma unroll
                for (int d = 0; d < 3; d++) {
#pragma unroll
                    for (int m = 0; m < 3; m++)
                        s_f[(d * 3 + m) * ND + l] = sw * (R[m][0] * Pk[d][0] + R[m][1] * Pk[d][1] + R[m][2] * Pk[d][2]);
                    mres[d] = P.beta * w * fabs(det) * s_u[d * ND + l];
                }
            }
        }
        __syncthreads();
        // ---- backward: Dt^T of the fluxes plus the mass term at the points, then B^T along z, y, x
        if (in_cta) {
#pragma unroll
            for (int d = 0; d < 3; d++) {
                const double *f = s_f + d * 3 * ND;
                s_t[d * ND + l] = mres[d] + pass1<N, 0, true>(P.Dt, f, qi, qj, qk) +
                                  pass1<N, 1, true>(P.Dt, f + ND, qi, qj, qk) +
                                  pass1<N, 2, true>(P.Dt, f + 2 * ND, qi, qj, qk);
            }
            if (STK) s_q[l] = pass1<N, 2, true>(P.Bq, s_p, qi, qj, qk);
            if (TMP)
                s_a[l] = tres + pass1<N, 0, true>(P.Dt, s_tf, qi, qj, qk) +
                         pass1<N, 1, true>(P.Dt, s_tf + ND, qi, qj, qk) +
                         pass1<N, 2, true>(P.Dt, s_tf + 2 * ND, qi, qj, qk);
        }
        __syncthreads();
        if (in_cta) {
#pragma unroll
            for (int d = 0; d < 3; d++) s_u[d * ND + l] = pass1<N, 2, true>(P.B, s_t + d * ND, qi, qj, qk);
            if (STK) s_p[l] = pass1<N, 1, true>(P.Bq, s_q, qi, qj, qk);
            if (TMP) s_b[l] = pass1<N, 2, true>(P.Bq, s_a, qi, qj, qk);
        }
        __syncthreads();
        if (in_cta) {
#pragma unroll
            for (int d = 0; d < 3; d++) s_t[d * ND + l] = pass1<N, 1, true>(P.B, s_u + d * ND, qi, qj, qk);
            if (TMP) s_a[l] = pass1<N, 1, true>(P.Bq, s_b, qi, qj, qk);
        }
        __syncthreads();
        double out[3], outp = 0.0, outt = 0.0;
        if (in_cta) {
#pragma unroll
            for (int d = 0; d < 3; d++) out[d] = pass1<N, 0, true>(P.B, s_t + d * ND, qi, qj, qk);
            if (STK) outp = pass1<N, 0, true>(P.Bq, s_p, qi, qj, qk);
            if (TMP) outt = pass1<N, 0, true>(P.Bq, s_a, qi, qj, qk);
        }
        // ---- scatter (this thread's node, three components)
        if (valid) {
            if (!MATRIX) {
                double *dst = P.y + (long long)g * 3;
#pragma unroll
                for (int a = 0; a < 3; a++) {
                    if (ATOMIC) atomicAdd(dst + a, out[a]);
                    else dst[a] += out[a];
                }
                if (pdof) {
                    if (ATOMIC) atomicAdd(P.yp + gp, outp);
                    else P.yp[gp] += outp;
                }
                if (TMP && pdof) {
                    if (ATOMIC) atomicAdd(P.yt + gp, outt);
                    else P.yt[gp] += outt;
                }
            } else {
                const int j = jb / 3, b = jb - 3 * (jb / 3);
                if (P.vals == nullptr) {
                    if (l == j) atomicAdd(P.y + (long long)g * 3 + b, b == 0 ? out[0] : (b == 1 ? out[1] : out[2]));
                } else {
                    const int gj = s_idx[j];
                    if (!P.col_lg || __ldg(P.col_lg + (long long)gj * 3 + b) >= 0) {
                        long long lo = __ldg(P.rowptr + g);
                        if (P.rank_tab) {
                            const int v = P.nlay_total < 3 ? layer
                                                           : (layer == 0 ? 0 : (layer == P.nlay_total - 1 ? 2 : 1));
                            lo += __ldg(P.rank_tab + (((long long)col * P.nvar + v) * ND + j) * ND + l);
                        } else {
                            long long hi = __ldg(P.rowptr + g + 1);
                            while (hi - lo > 1) {
                                const long long mid = (lo + hi) >> 1;
                                if (__ldg(P.colidx + mid) <= gj) lo = mid; else hi = mid;
                            }
                        }
#pragma unroll
                        for (int a = 0; a < 3; a++) {
                            if (P.row_lg && __ldg(P.row_lg + (long long)g * 3 + a) < 0) continue;
                            atomicAdd(P.vals + (lo * 3 + a) * 3 + b, out[a]);
                        }
                    }
                }
            }
        }
        __syncthreads();          // the slot's buffers are refilled by the next unit
    }
}

template <int N, bool MATRIX, bool ATOMIC, int MODE>
int launch(cudaStream_t st, const ElasParams<N> &P, int sm_count)
{
    using S = ElasShape<N, MODE>;
    auto kern = elasticity_kernel<N, MATRIX, ATOMIC, MODE>;
    static bool attr = false;
    if (!attr) {
        FDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S::SMEM));
        attr = true;
    }
    int per_sm = 0;
    FDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, S::THREADS, S::SMEM));
    const long long ncells = (long long)P.ncols * P.nlay_items;
    const long long nunits = MATRIX ? ncells * 3 * S::ND : ncells;
    long long grid = (nunits + S::CPB - 1) / S::CPB;
    const long long cap = (long long)sm_count * (per_sm > 0 ? per_sm : 1);
    if (grid > cap) grid = cap;
    if (grid < 1) return 0;
    kern<<<(int)grid, S::THREADS, S::SMEM, st>>>(P);
    FDB_LAUNCH_CHECK();
    return 0;
}

template <int N>
void fill_tables(const fdb_kernel_s *k, ElasParams<N> &P)
{
    P.off0 = k->d_off0;
    P.off1 = k->d_off1;
    P.mu = k->desc.alpha;
    P.lmbda = k->desc.lmbda;
    P.beta = k->desc.beta;
    for (int i = 0; i < N * N; i++) {
        P.B[i] = k->desc.B[i];
        P.Dt[i] = k->Dt[i];
    }
    for (int i = 0; i < N; i++) {
        P.wq[i] = k->desc.wq[i];
        P.xq[i] = k->desc.xq[i];
    }
    if (k->desc.form == FDB_FORM_STOKES || k->desc.form == FDB_FORM_NAVIER_STOKES ||
        k->desc.form == FDB_FORM_NAVIER_STOKES_JACOBIAN || k->desc.form == FDB_FORM_BOUSSINESQ ||
        k->desc.form == FDB_FORM_BOUSSINESQ_JACOBIAN) {
        P.off2 = k->d_off2;
        for (int d = 0; d < 3; d++) P.bg[d] = k->desc.dcoef[d];
        for (int q = 0; q < N; q++)
            for (int a = 0; a < N; a++) P.Bq[q * N + a] = a < N - 1 ? k->B2[q * (N - 1) + a] : 0.0;
    }
}

template <int N, int MODE>
int action_n(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
             const double *coords, const double *x, const double *u, const fdb_int *map0, const fdb_int *map1,
             double *yp, const double *xp, const fdb_int *map2, double *yt, const double *xt, const double *t0)
{
    fdb::Context &c = fdb::ctx();
    ElasParams<N> P;
    memset(&P, 0, sizeof(P));
    fill_tables(k, P);
    P.y = y;
    P.x = x;
    P.u = u;
    P.coords = coords;
    P.map0 = map0;
    P.map1 = map1;
    P.yp = yp;
    P.xp = xp;
    P.map2 = map2;
    P.yt = yt;
    P.xt = xt;
    P.t0 = t0;
    if (k->desc.scatter == FDB_SCATTER_ATOMIC) {
        P.collist = subset;
        P.col0 = start;
        P.ncols = end - start;
        P.nlay_items = nlay;
        P.lay_first = 0;
        P.lay_step = 1;
        if (P.ncols <= 0 || nlay <= 0) return 0;
        return launch<N, false, true, MODE>(c.stream, P, c.sm_count);
    }
    // deterministic: one launch per (colour, layer parity), no two cells of a launch share a node
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
            if (launch<N, false, false, MODE>(c.stream, P, c.sm_count)) return 1;
        }
    }
    return 0;
}

template <int N, int MODE>
int matrix_n(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, fdb_mat_t mat,
             const double *coords, const double *u, const fdb_int *map0, const fdb_int *map1, double *diag_out)
{
    fdb::Context &c = fdb::ctx();
    ElasParams<N> P;
    memset(&P, 0, sizeof(P));
    fill_tables(k, P);
    P.coords = coords;
    P.u = u;
    P.map0 = map0;
    P.map1 = map1;
    if (mat) {
        if (fdb_mat_device_view(mat, &P.rowptr, &P.colidx, &P.vals, &P.row_lg, &P.col_lg)) return 1;
        fdb_mat_rank_table(mat, &P.rank_tab, &P.nvar);
    } else {
        P.y = diag_out;
    }
    P.nlay_total = nlay;
    if (subset || k->desc.cell != FDB_CELL_HEX_EXTRUDED) P.rank_tab = nullptr;   // table is per column of the full set
    P.collist = subset;
    P.col0 = start;
    P.ncols = end - start;
    P.nlay_items = nlay;
    P.lay_first = 0;
    P.lay_step = 1;
    if (P.ncols <= 0 || nlay <= 0) return 0;
    return launch<N, true, true, MODE>(c.stream, P, c.sm_count);
}

template <int MODE>
int action_mode(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
                const double *coords, const double *x, const double *u, const fdb_int *map0, const fdb_int *map1,
                double *yp = nullptr, const double *xp = nullptr, const fdb_int *map2 = nullptr, double *yt = nullptr,
                const double *xt = nullptr, const double *t0 = nullptr)
{
    // the Taylor-Hood modes have no degree-1 instantiation (their pressure space would be CG_0)
    switch (k->n1d) {
    case 2:
        if constexpr (!el_pressure(MODE))
            return action_n<2, MODE>(k, start, end, nlay, subset, y, coords, x, u, map0, map1, yp, xp, map2, yt, xt,
                                     t0);
        break;
    case 3:
        return action_n<3, MODE>(k, start, end, nlay, subset, y, coords, x, u, map0, map1, yp, xp, map2, yt, xt, t0);
    case 4:
        return action_n<4, MODE>(k, start, end, nlay, subset, y, coords, x, u, map0, map1, yp, xp, map2, yt, xt, t0);
    case 5:
        return action_n<5, MODE>(k, start, end, nlay, subset, y, coords, x, u, map0, map1, yp, xp, map2, yt, xt, t0);
    }
    fdb::set_error("elasticity action: degree %d not instantiated (1..4)", k->n1d - 1);
    return 1;
}

template <int MODE>
int matrix_mode(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, fdb_mat_t mat,
                const double *coords, const double *u, const fdb_int *map0, const fdb_int *map1, double *diag_out)
{
    switch (k->n1d) {
    case 2: return matrix_n<2, MODE>(k, start, end, nlay, subset, mat, coords, u, map0, map1, diag_out);
    case 3: return matrix_n<3, MODE>(k, start, end, nlay, subset, mat, coords, u, map0, map1, diag_out);
    case 4: return matrix_n<4, MODE>(k, start, end, nlay, subset, mat, coords, u, map0, map1, diag_out);
    }
    fdb::set_error("elasticity matrix: degree %d not instantiated (1..3)", k->n1d - 1);
    return 1;
}

}  // namespace

int fdb_launch_elasticity_action(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                                 double *y, const double *coords, const double *x, const double *u,
                                 const fdb_int *map0, const fdb_int *map1)
{
    switch (k->desc.form) {
    case FDB_FORM_ELASTICITY:
        return action_mode<EL_LINEAR>(k, start, end, nlay, subset, y, coords, x, nullptr, map0, map1);
    case FDB_FORM_HYPERELASTICITY:
        return action_mode<EL_RESIDUAL>(k, start, end, nlay, subset, y, coords, x, nullptr, map0, map1);
    case FDB_FORM_HYPERELASTICITY_JACOBIAN:
        return action_mode<EL_JACOBIAN>(k, start, end, nlay, subset, y, coords, x, u, map0, map1);
    }
    fdb::set_error("elasticity action: form %d is not an elasticity form", k->desc.form);
    return 1;
}

int fdb_launch_stokes_action(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                             double *yu, const double *coords, const double *u, double *yp, const double *p,
                             const double *ulin, const fdb_int *map0, const fdb_int *map1, const fdb_int *map2,
                             double *yt, const double *t, const double *tlin)
{
    switch (k->desc.form) {
    case FDB_FORM_STOKES:
        return action_mode<EL_STOKES>(k, start, end, nlay, subset, yu, coords, u, nullptr, map0, map1, yp, p, map2);
    case FDB_FORM_NAVIER_STOKES:
        return action_mode<EL_NS_RESIDUAL>(k, start, end, nlay, subset, yu, coords, u, nullptr, map0, map1, yp, p,
                                           map2);
    case FDB_FORM_NAVIER_STOKES_JACOBIAN:
        return action_mode<EL_NS_JACOBIAN>(k, start, end, nlay, subset, yu, coords, u, ulin, map0, map1, yp, p,
                                           map2);
    case FDB_FORM_BOUSSINESQ:
        return action_mode<EL_RB_RESIDUAL>(k, start, end, nlay, subset, yu, coords, u, nullptr, map0, map1, yp, p,
                                           map2, yt, t);
    case FDB_FORM_BOUSSINESQ_JACOBIAN:
        return action_mode<EL_RB_JACOBIAN>(k, start, end, nlay, subset, yu, coords, u, ulin, map0, map1, yp, p,
                                           map2, yt, t, tlin);
    }
    fdb::set_error("stokes action: form %d is not a Taylor-Hood form", k->desc.form);
    return 1;
}

int fdb_launch_elasticity_matrix(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset,
                                 fdb_mat_t mat, const double *coords, const double *u, const fdb_int *map0,
                                 const fdb_int *map1, double *diag_out)
{
    switch (k->desc.form) {
    case FDB_FORM_ELASTICITY:
        return matrix_mode<EL_LINEAR>(k, start, end, nlay, subset, mat, coords, nullptr, map0, map1, diag_out);
    case FDB_FORM_HYPERELASTICITY_JACOBIAN:
        return matrix_mode<EL_JACOBIAN>(k, start, end, nlay, subset, mat, coords, u, map0, map1, diag_out);
    }
    fdb::set_error("elasticity matrix: form %d has no element matrix", k->desc.form);
    return 1;
}
