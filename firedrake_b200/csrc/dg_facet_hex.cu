// The facet terms of the symmetric interior penalty (SIPG) discretisation of -div(alpha grad u) + beta u = f on
// scalar DQ_p hexahedra (Gauss-Legendre nodes), DESIGN.md section 4.15:
//
//   FDB_FORM_INTERIOR_PENALTY (an interior-facet integral, alpha = desc.alpha, eta = desc.beta)
//       alpha*( -inner(avg(grad u), jump(v, n)) - inner(jump(u, n), avg(grad v))
//               + (eta/avg(h))*inner(jump(u, n), jump(v, n)) )*dS
//   FDB_FORM_DG_BOUNDARY (an exterior-facet integral, c_f = desc.alpha, c_p = desc.beta, c_m = desc.dcoef[0],
//   c_s = desc.dcoef[1])
//       ( c_m*u*v + (c_p/h)*u*v - c_s*u*dot(grad v, n) - c_f*dot(grad u, n)*v )*ds
//
// h is the cell diameter (the largest distance between two of the cell's 8 vertices), n the unit normal,
// outward from '+' (interior) or from the cell (exterior).
//
// An iteration entry is one facet: an interior entry's maps are the '+' cell's row followed by the '-' cell's
// (2 N^3 dofs, 16 vertices), an exterior entry's the cell's row (N^3, 8), plus offset * layer on extruded cells;
// the local facet numbers f = 2*direction + side (one per side, '+' first) are read like a direct Dat of the
// column.  The face's tangential axes s, t are the other two reference axes in increasing order; face point
// (a, b) of '+' and of '-' are the same physical point (the mesh orients both sides of a face alike, which the
// facet-set builder checks).
//
// Layout: one thread per face Gauss point (a, b) (nq = N per axis), FPB facets ("slots") per CTA, static shared
// memory.  Per slot and side: the cell's N^3 values (one block of contiguous dofs for a DQ cell) and its 8
// vertices.  The trace and normal reference derivative come from contracting each normal line with the endpoint
// tables phi(side), phi'(side) (computed in fdb_kernel_create); B and D along s and t then give u and the
// reference gradient at the points, J^-T the physical gradient.  The test-side coefficients of v and grad v
// at each point are mapped back with J^-1 and the transposed contractions, and expanded along the normal line:
//   ACTION    gather, normal contraction, s pass, t pass + point stage, t^T pass, s^T pass + scatter (atomic or
//             coloured)
//   DIAGONAL  the self-terms of each side: point stage, t^T pass and s^T pass on squared tables (atomic)
#include "common.cuh"
#include "dg_hex.cuh"

namespace {

enum { DG_ACTION = 0, DG_DIAGONAL = 1 };

template <int N>
struct DGFacetParams {
    double *y;                   // action / diagonal output
    const double *x;             // action input
    const double *coords;        // AoS, 3 per vertex
    const fdb_int *map0, *map1;  // dof map (NS * N^3 per column), vertex map (NS * 8)
    const fdb_int *off0, *off1;  // layer offsets (zeros for native hexes)
    const unsigned *facet;       // NS local facet numbers per column of the iteration set
    const fdb_int *collist;      // columns to visit (subset / colour) or NULL = col0 + i
    int col0, ncols;
    int nlay_items, lay_first, lay_step;   // layers lay_first + lay_step * k, k < nlay_items
    double c_f, c_p, c_m, c_s;   // interior: alpha, eta (c_m, c_s unused)
    double B[N * N], D[N * N], wq[N], xq[N];
    double E[4][N];              // phi_k(0), phi_k(1), phi_k'(0), phi_k'(1)
};

template <int N>
struct DGFacetShape {
    static constexpr int NF = N * N;                                    // face points
    static constexpr int FPB = 256 / NF < 32 ? 256 / NF : 32;           // facets (slots) per CTA
    static constexpr int THREADS = ((FPB * NF + 31) / 32) * 32;
};

// the cell-local dof of (i_s, i_t, k) on a facet of direction dir: k along the normal axis
template <int N>
__device__ __forceinline__ int cell_dof(int dir, int is, int it, int k)
{
    return dir == 0 ? (k * N + is) * N + it : (dir == 1 ? (is * N + k) * N + it : (is * N + it) * N + k);
}

// the largest distance between two of a cell's 8 vertices (UFL's CellDiameter)
__device__ __forceinline__ double cell_diameter(const double *X)
{
    double m = 0.0;
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = i + 1; j < 8; j++) {
            const double dx = X[i * 3] - X[j * 3], dy = X[i * 3 + 1] - X[j * 3 + 1], dz = X[i * 3 + 2] - X[j * 3 + 2];
            m = fmax(m, dx * dx + dy * dy + dz * dz);
        }
    return sqrt(m);
}

// a reference-axis vector in the face axes (s, t, n) of a facet of direction dir, and back (selects, no dynamic
// indexing: the arrays stay in registers)
__device__ __forceinline__ void to_face_axes(int dir, const double v[3], double &vs, double &vt, double &vn)
{
    vs = dir == 0 ? v[1] : v[0];
    vt = dir == 2 ? v[1] : v[2];
    vn = dir == 0 ? v[0] : (dir == 1 ? v[1] : v[2]);
}

__device__ __forceinline__ void from_face_axes(int dir, double vs, double vt, double vn, double v[3])
{
    v[0] = dir == 0 ? vn : vs;
    v[1] = dir == 1 ? vn : (dir == 0 ? vs : vt);
    v[2] = dir == 2 ? vn : vt;
}

// the inverse Jacobian and |det J| of a cell's trilinear map at the face point (s, t) of facet (dir, side)
__device__ __forceinline__ double face_inverse_jacobian(const double *X, int dir, int side, double s, double t,
                                                        double K[3][3])
{
    double xi[3];
    from_face_axes(dir, s, t, (double)side, xi);
    return trilinear_inverse_jacobian(X, xi, K);
}

template <int N, bool INTERIOR, int MODE, bool ATOMIC>
__global__ void __launch_bounds__(DGFacetShape<N>::THREADS)
dg_facet_kernel(const __grid_constant__ DGFacetParams<N> P)
{
    using S = DGFacetShape<N>;
    constexpr int NF = S::NF;
    constexpr int FPB = S::FPB;
    constexpr int ND = N * N * N;
    constexpr int NS = INTERIOR ? 2 : 1;                          // sides
    constexpr int NU = MODE == DG_ACTION ? (NS * ND > NS * 4 * NF ? NS * ND : NS * 4 * NF) : NS * 4 * NF;
    __shared__ double s_x[FPB][NS * 24];                          // vertex v of side sd: [sd * 24 + v * 3 + c]
    __shared__ double s_u[FPB][NU];                               // gathered values, then the point coefficients
    __shared__ double s_t[FPB][MODE == DG_ACTION ? NS * 2 * NF : 1];   // normal-line contractions
    __shared__ double s_s[FPB][NS * 3 * NF];                      // one-axis contractions
    __shared__ double s_h[FPB][NS];
    const int slot = threadIdx.x / NF;
    const int l = threadIdx.x - slot * NF;
    const bool in_cta = slot < FPB;
    const int sl = in_cta ? slot : 0;
    const int a = l / N, b = l - (l / N) * N;                    // point (a along s, b along t) = face node

    const long long nunits = (long long)P.ncols * P.nlay_items;
    for (long long base = (long long)blockIdx.x * FPB; base < nunits; base += (long long)gridDim.x * FPB) {
        const long long unit = base + slot;
        const bool valid = in_cta && unit < nunits;
        int col = 0, layer = 0;
        unsigned f[NS];
#pragma unroll
        for (int sd = 0; sd < NS; sd++) f[sd] = sd == 0 ? 5u : 4u;   // idle slot: any valid facet pair
        if (valid) {
            const int ci = (int)(unit / P.nlay_items);
            layer = P.lay_first + P.lay_step * (int)(unit - (long long)ci * P.nlay_items);
            col = P.collist ? __ldg(P.collist + ci) : P.col0 + ci;
#pragma unroll
            for (int sd = 0; sd < NS; sd++) f[sd] = __ldg(P.facet + (long long)col * NS + sd);
        }
        // ---- gather: both cells' values and vertices
        if (valid) {
            if (MODE == DG_ACTION) {
                for (int i = l; i < NS * ND; i += NF) {
                    const int g = __ldg(P.map0 + (long long)col * NS * ND + i) + __ldg(P.off0 + i) * layer;
                    s_u[sl][i] = __ldg(P.x + g);
                }
            }
            for (int i = l; i < NS * 24; i += NF) {
                const int v = i / 3, c = i - 3 * v;               // v: vertex of the NS * 8 map entries
                const int gv = __ldg(P.map1 + (long long)col * NS * 8 + v) + __ldg(P.off1 + v) * layer;
                s_x[sl][i] = __ldg(P.coords + (long long)gv * 3 + c);
            }
        } else if (in_cta) {
            // idle slot: the unit cube on both sides (finite geometry) with zero values, nothing scattered
            if (MODE == DG_ACTION)
                for (int i = l; i < NS * ND; i += NF) s_u[sl][i] = 0.0;
            for (int i = l; i < NS * 24; i += NF) {
                const int v = (i / 3) & 7, c = i % 3;
                s_x[sl][i] = (double)((v >> (2 - c)) & 1);
            }
        }
        __syncthreads();
        if (in_cta && l < NS) s_h[sl][l] = cell_diameter(&s_x[sl][l * 24]);
        if (MODE == DG_ACTION) {
            // normal lines: T0[is][it] = sum_k phi_k(side) u[is, it, k], T1 the same with phi'
            if (in_cta) {
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    const int dir = (int)(f[sd] >> 1), side = (int)(f[sd] & 1u);
                    double t0 = 0.0, t1 = 0.0;
#pragma unroll
                    for (int k = 0; k < N; k++) {
                        const double u = s_u[sl][sd * ND + cell_dof<N>(dir, a, b, k)];
                        t0 = fma(P.E[side][k], u, t0);
                        t1 = fma(P.E[2 + side][k], u, t1);
                    }
                    s_t[sl][(sd * 2) * NF + l] = t0;
                    s_t[sl][(sd * 2 + 1) * NF + l] = t1;
                }
            }
            __syncthreads();
            // along s (thread (q = a, it = b)): S0 = B T0, S1 = D T0, S2 = B T1
            if (in_cta) {
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
#pragma unroll
                    for (int k = 0; k < N; k++) {
                        const double t0 = s_t[sl][(sd * 2) * NF + k * N + b];
                        s0 = fma(P.B[a * N + k], t0, s0);
                        s1 = fma(P.D[a * N + k], t0, s1);
                        s2 = fma(P.B[a * N + k], s_t[sl][(sd * 2 + 1) * NF + k * N + b], s2);
                    }
                    s_s[sl][(sd * 3) * NF + l] = s0;
                    s_s[sl][(sd * 3 + 1) * NF + l] = s1;
                    s_s[sl][(sd * 3 + 2) * NF + l] = s2;
                }
            }
            __syncthreads();
            // along t, and the point stage at (a, b)
            if (in_cta) {
                double gr[NS][3], K[NS][3][3], u[NS], detJ[NS];
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    double v0 = 0.0, vs = 0.0, vt = 0.0, vn = 0.0;
#pragma unroll
                    for (int k = 0; k < N; k++) {
                        const double s0 = s_s[sl][(sd * 3) * NF + a * N + k];
                        v0 = fma(P.B[b * N + k], s0, v0);
                        vt = fma(P.D[b * N + k], s0, vt);
                        vs = fma(P.B[b * N + k], s_s[sl][(sd * 3 + 1) * NF + a * N + k], vs);
                        vn = fma(P.B[b * N + k], s_s[sl][(sd * 3 + 2) * NF + a * N + k], vn);
                    }
                    const int dir = (int)(f[sd] >> 1), side = (int)(f[sd] & 1u);
                    detJ[sd] = face_inverse_jacobian(&s_x[sl][sd * 24], dir, side, P.xq[a], P.xq[b], K[sd]);
                    double rg[3];
                    from_face_axes(dir, vs, vt, vn, rg);
                    u[sd] = v0;
#pragma unroll
                    for (int c = 0; c < 3; c++) gr[sd][c] = K[sd][0][c] * rg[0] + K[sd][1][c] * rg[1] + K[sd][2][c] * rg[2];
                }
                // unit normal and surface weight from '+': n ~ grad xi_dir = row dir of J^-1,
                // |dX/ds x dX/dt| = |det J| |grad xi_dir|
                const int dir0 = (int)(f[0] >> 1), side0 = (int)(f[0] & 1u);
                const double detJ0 = detJ[0];
                const double n0 = dir0 == 0 ? K[0][0][0] : (dir0 == 1 ? K[0][1][0] : K[0][2][0]);
                const double n1 = dir0 == 0 ? K[0][0][1] : (dir0 == 1 ? K[0][1][1] : K[0][2][1]);
                const double n2 = dir0 == 0 ? K[0][0][2] : (dir0 == 1 ? K[0][1][2] : K[0][2][2]);
                const double gn = sqrt(n0 * n0 + n1 * n1 + n2 * n2);
                const double sgn = side0 ? 1.0 / gn : -1.0 / gn;
                const double n[3] = {n0 * sgn, n1 * sgn, n2 * sgn};
                const double W = P.wq[a] * P.wq[b] * detJ0 * gn;
                double cv[NS], gc;
                if (INTERIOR) {
                    const double ju = u[0] - u[NS - 1];
                    const double fu = 0.5 * (n[0] * (gr[0][0] + gr[NS - 1][0]) + n[1] * (gr[0][1] + gr[NS - 1][1]) +
                                             n[2] * (gr[0][2] + gr[NS - 1][2]));
                    const double sig = P.c_p / (0.5 * (s_h[sl][0] + s_h[sl][NS - 1]));
                    cv[0] = P.c_f * W * (sig * ju - fu);
                    cv[NS - 1] = -cv[0];
                    gc = -0.5 * P.c_f * W * ju;
                } else {
                    const double dn = n[0] * gr[0][0] + n[1] * gr[0][1] + n[2] * gr[0][2];
                    cv[0] = W * ((P.c_m + P.c_p / s_h[sl][0]) * u[0] - P.c_f * dn);
                    gc = -P.c_s * W * u[0];
                }
                // test-side coefficients in each side's reference axes: cv (v), J^-1 (gc n) (grad^ v)
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    const int dir = (int)(f[sd] >> 1);
                    double gh[3];
#pragma unroll
                    for (int d = 0; d < 3; d++) gh[d] = gc * (K[sd][d][0] * n[0] + K[sd][d][1] * n[1] + K[sd][d][2] * n[2]);
                    double gs, gt, gn2;
                    to_face_axes(dir, gh, gs, gt, gn2);
                    s_u[sl][(sd * 4) * NF + l] = cv[sd];
                    s_u[sl][(sd * 4 + 1) * NF + l] = gs;
                    s_u[sl][(sd * 4 + 2) * NF + l] = gt;
                    s_u[sl][(sd * 4 + 3) * NF + l] = gn2;
                }
            }
            __syncthreads();
            // t^T (thread (q = a, it = b)): X0 = B^T cv + D^T g_t, X1 = B^T g_s, X2 = B^T g_n
            if (in_cta) {
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    double x0 = 0.0, x1 = 0.0, x2 = 0.0;
#pragma unroll
                    for (int r = 0; r < N; r++) {
                        const double br = P.B[r * N + b];
                        const double *R = &s_u[sl][(sd * 4) * NF + a * N + r];
                        x0 = fma(br, R[0], x0);
                        x0 = fma(P.D[r * N + b], R[2 * NF], x0);
                        x1 = fma(br, R[NF], x1);
                        x2 = fma(br, R[3 * NF], x2);
                    }
                    s_s[sl][(sd * 3) * NF + l] = x0;
                    s_s[sl][(sd * 3 + 1) * NF + l] = x1;
                    s_s[sl][(sd * 3 + 2) * NF + l] = x2;
                }
            }
            __syncthreads();
            // s^T (thread (is = a, it = b)) and the expansion along the normal line: the scatter
            if (valid) {
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    double q0 = 0.0, q1 = 0.0;
#pragma unroll
                    for (int q = 0; q < N; q++) {
                        q0 = fma(P.B[q * N + a], s_s[sl][(sd * 3) * NF + q * N + b], q0);
                        q0 = fma(P.D[q * N + a], s_s[sl][(sd * 3 + 1) * NF + q * N + b], q0);
                        q1 = fma(P.B[q * N + a], s_s[sl][(sd * 3 + 2) * NF + q * N + b], q1);
                    }
                    const int dir = (int)(f[sd] >> 1), side = (int)(f[sd] & 1u);
#pragma unroll
                    for (int k = 0; k < N; k++) {
                        const int i = sd * ND + cell_dof<N>(dir, a, b, k);
                        const int g = __ldg(P.map0 + (long long)col * NS * ND + i) + __ldg(P.off0 + i) * layer;
                        const double val = fma(P.E[side][k], q0, P.E[2 + side][k] * q1);
                        if (ATOMIC) atomicAdd(P.y + g, val);
                        else P.y[g] += val;
                    }
                }
            }
        } else {
            __syncthreads();                                       // s_h
            // the point stage of the self-terms: P1 (v v), and the (s, t, n) components of the flux weight
            if (in_cta) {
                double K[NS][3][3], detJ[NS];
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    const int dir = (int)(f[sd] >> 1), side = (int)(f[sd] & 1u);
                    detJ[sd] = face_inverse_jacobian(&s_x[sl][sd * 24], dir, side, P.xq[a], P.xq[b], K[sd]);
                }
                const int dir0 = (int)(f[0] >> 1), side0 = (int)(f[0] & 1u);
                const double detJ0 = detJ[0];
                const double n0 = dir0 == 0 ? K[0][0][0] : (dir0 == 1 ? K[0][1][0] : K[0][2][0]);
                const double n1 = dir0 == 0 ? K[0][0][1] : (dir0 == 1 ? K[0][1][1] : K[0][2][1]);
                const double n2 = dir0 == 0 ? K[0][0][2] : (dir0 == 1 ? K[0][1][2] : K[0][2][2]);
                const double gn = sqrt(n0 * n0 + n1 * n1 + n2 * n2);
                const double sgn = side0 ? 1.0 / gn : -1.0 / gn;
                const double n[3] = {n0 * sgn, n1 * sgn, n2 * sgn};
                const double W = P.wq[a] * P.wq[b] * detJ0 * gn;
                double p1, pf[NS];
                if (INTERIOR) {
                    p1 = P.c_f * W * P.c_p / (0.5 * (s_h[sl][0] + s_h[sl][NS - 1]));
                    pf[0] = -P.c_f * W;
                    pf[NS - 1] = P.c_f * W;                            // the '-' side's outward normal is -n
                } else {
                    p1 = W * (P.c_m + P.c_p / s_h[sl][0]);
                    pf[0] = -(P.c_f + P.c_s) * W;
                }
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    const int dir = (int)(f[sd] >> 1);
                    double m[3];
#pragma unroll
                    for (int d = 0; d < 3; d++) m[d] = pf[sd] * (K[sd][d][0] * n[0] + K[sd][d][1] * n[1] + K[sd][d][2] * n[2]);
                    double ms, mt, mn;
                    to_face_axes(dir, m, ms, mt, mn);
                    s_u[sl][(sd * 4) * NF + l] = p1;
                    s_u[sl][(sd * 4 + 1) * NF + l] = ms;
                    s_u[sl][(sd * 4 + 2) * NF + l] = mt;
                    s_u[sl][(sd * 4 + 3) * NF + l] = mn;
                }
            }
            __syncthreads();
            // t^T on squared tables: Y0 = B^2 P1 + (B D) P_t, Y1 = B^2 P_s, Y2 = B^2 P_n
            if (in_cta) {
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    double y0 = 0.0, y1 = 0.0, y2 = 0.0;
#pragma unroll
                    for (int r = 0; r < N; r++) {
                        const double br = P.B[r * N + b], bb = br * br;
                        const double *R = &s_u[sl][(sd * 4) * NF + a * N + r];
                        y0 = fma(bb, R[0], y0);
                        y0 = fma(br * P.D[r * N + b], R[2 * NF], y0);
                        y1 = fma(bb, R[NF], y1);
                        y2 = fma(bb, R[3 * NF], y2);
                    }
                    s_s[sl][(sd * 3) * NF + l] = y0;
                    s_s[sl][(sd * 3 + 1) * NF + l] = y1;
                    s_s[sl][(sd * 3 + 2) * NF + l] = y2;
                }
            }
            __syncthreads();
            // s^T: d[is, it, k] += phi_k^2 E + phi_k phi_k' G
            if (valid) {
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    double e = 0.0, g2 = 0.0;
#pragma unroll
                    for (int q = 0; q < N; q++) {
                        const double bq = P.B[q * N + a], bb = bq * bq;
                        e = fma(bb, s_s[sl][(sd * 3) * NF + q * N + b], e);
                        e = fma(bq * P.D[q * N + a], s_s[sl][(sd * 3 + 1) * NF + q * N + b], e);
                        g2 = fma(bb, s_s[sl][(sd * 3 + 2) * NF + q * N + b], g2);
                    }
                    const int dir = (int)(f[sd] >> 1), side = (int)(f[sd] & 1u);
#pragma unroll
                    for (int k = 0; k < N; k++) {
                        const int i = sd * ND + cell_dof<N>(dir, a, b, k);
                        const int g = __ldg(P.map0 + (long long)col * NS * ND + i) + __ldg(P.off0 + i) * layer;
                        const double pk = P.E[side][k];
                        atomicAdd(P.y + g, pk * fma(pk, e, P.E[2 + side][k] * g2));
                    }
                }
            }
        }
        __syncthreads();          // the slot's buffers are refilled by the next facet
    }
}

// The upwind facet terms of FDB_FORM_DG_TRANSPORT on the collocated GL element (B = I): the trace of side sd at face
// point (a, b) is the phi(side) contraction of its normal line (a, b), b.n comes from b interpolated trilinearly
// from the '+' cell's vertices and n from the '+' Jacobian, and the flux times the weight goes back along the
// normal line of each side with opposite signs.  Only values are read: no tangential contractions, no '-' geometry.
//   ACTION    gather ('+' vertices and b, both cells' values), point stage + scatter (atomic or coloured)
//   DIAGONAL  the self-terms: max(+-b.n, 0) phi_k(side)^2 W per side, or (c_out max + c_in min)(b.n) phi_k^2 W (atomic)
template <int N>
struct DGUpwindParams {
    double *y;                   // action / diagonal output
    const double *x;             // action input
    const double *coords, *b;    // AoS, 3 per vertex
    const fdb_int *map0, *map1;  // dof map (NS * N^3 per column), vertex map (NS * 8; the '+' 8 are read)
    const fdb_int *off0, *off1;  // layer offsets (zeros for native hexes)
    const unsigned *facet;       // NS local facet numbers per column of the iteration set
    const fdb_int *collist;      // columns to visit (subset / colour) or NULL = col0 + i
    int col0, ncols;
    int nlay_items, lay_first, lay_step;   // layers lay_first + lay_step * k, k < nlay_items
    double c_out, c_in;          // exterior: the max(b.n, 0) and min(b.n, 0) coefficients
    double wq[N], xq[N];
    double E[2][N];              // phi_k(0), phi_k(1)
};

template <int N, bool INTERIOR, int MODE, bool ATOMIC>
__global__ void __launch_bounds__(DGFacetShape<N>::THREADS)
dg_upwind_kernel(const __grid_constant__ DGUpwindParams<N> P)
{
    using S = DGFacetShape<N>;
    constexpr int NF = S::NF;
    constexpr int FPB = S::FPB;
    constexpr int ND = N * N * N;
    constexpr int NS = INTERIOR ? 2 : 1;                          // sides
    __shared__ double s_x[FPB][24];                               // the '+' cell's vertices
    __shared__ double s_b[FPB][24];                               // and b at them
    __shared__ double s_u[FPB][MODE == DG_ACTION ? NS * ND : 1];  // both cells' values
    const int slot = threadIdx.x / NF;
    const int l = threadIdx.x - slot * NF;
    const bool in_cta = slot < FPB;
    const int sl = in_cta ? slot : 0;
    const int a = l / N, b = l - (l / N) * N;                    // point (a along s, b along t) = face node

    const long long nunits = (long long)P.ncols * P.nlay_items;
    for (long long base = (long long)blockIdx.x * FPB; base < nunits; base += (long long)gridDim.x * FPB) {
        const long long unit = base + slot;
        const bool valid = in_cta && unit < nunits;
        int col = 0, layer = 0;
        unsigned f[NS];
#pragma unroll
        for (int sd = 0; sd < NS; sd++) f[sd] = sd == 0 ? 5u : 4u;   // idle slot: any valid facet pair
        if (valid) {
            const int ci = (int)(unit / P.nlay_items);
            layer = P.lay_first + P.lay_step * (int)(unit - (long long)ci * P.nlay_items);
            col = P.collist ? __ldg(P.collist + ci) : P.col0 + ci;
#pragma unroll
            for (int sd = 0; sd < NS; sd++) f[sd] = __ldg(P.facet + (long long)col * NS + sd);
        }
        if (valid) {
            if (MODE == DG_ACTION) {
                for (int i = l; i < NS * ND; i += NF) {
                    const int g = __ldg(P.map0 + (long long)col * NS * ND + i) + __ldg(P.off0 + i) * layer;
                    s_u[sl][i] = __ldg(P.x + g);
                }
            }
            for (int i = l; i < 24; i += NF) {
                const int v = i / 3, c = i - 3 * v;
                const long long gv = (long long)(__ldg(P.map1 + (long long)col * NS * 8 + v) + __ldg(P.off1 + v) * layer);
                s_x[sl][i] = __ldg(P.coords + gv * 3 + c);
                s_b[sl][i] = __ldg(P.b + gv * 3 + c);
            }
        } else if (in_cta) {
            // idle slot: the unit cube at rest with zero values, nothing scattered
            if (MODE == DG_ACTION)
                for (int i = l; i < NS * ND; i += NF) s_u[sl][i] = 0.0;
            for (int i = l; i < 24; i += NF) {
                const int v = i / 3, c = i % 3;
                s_x[sl][i] = (double)((v >> (2 - c)) & 1);
                s_b[sl][i] = 0.0;
            }
        }
        __syncthreads();
        if (valid) {
            // unit normal, surface weight and b.n from '+' (as in dg_facet_kernel)
            const int dir0 = (int)(f[0] >> 1), side0 = (int)(f[0] & 1u);
            double xi[3], K[3][3], bq[3];
            from_face_axes(dir0, P.xq[a], P.xq[b], (double)side0, xi);
            const double detJ0 = trilinear_inverse_jacobian(&s_x[sl][0], xi, K);
            trilinear_interpolate(&s_b[sl][0], xi, bq);
            const double n0 = dir0 == 0 ? K[0][0] : (dir0 == 1 ? K[1][0] : K[2][0]);
            const double n1 = dir0 == 0 ? K[0][1] : (dir0 == 1 ? K[1][1] : K[2][1]);
            const double n2 = dir0 == 0 ? K[0][2] : (dir0 == 1 ? K[1][2] : K[2][2]);
            const double gn = sqrt(n0 * n0 + n1 * n1 + n2 * n2);
            const double W = P.wq[a] * P.wq[b] * detJ0 * gn;
            const double bn = (side0 ? 1.0 : -1.0) * (n0 * bq[0] + n1 * bq[1] + n2 * bq[2]) / gn;
            double cv[NS];                                     // the coefficient of phi_k(side) on each side
            if (MODE == DG_ACTION) {
                double tr[NS];
#pragma unroll
                for (int sd = 0; sd < NS; sd++) {
                    const int dir = (int)(f[sd] >> 1), side = (int)(f[sd] & 1u);
                    double t0 = 0.0;
#pragma unroll
                    for (int k = 0; k < N; k++) t0 = fma(P.E[side][k], s_u[sl][sd * ND + cell_dof<N>(dir, a, b, k)], t0);
                    tr[sd] = t0;
                }
                if (INTERIOR) {
                    cv[0] = W * bn * (bn >= 0.0 ? tr[0] : tr[NS - 1]);
                    cv[NS - 1] = -cv[0];
                } else {
                    cv[0] = W * (P.c_out * fmax(bn, 0.0) + P.c_in * fmin(bn, 0.0)) * tr[0];
                }
            } else {
                if (INTERIOR) {
                    cv[0] = W * fmax(bn, 0.0);
                    cv[NS - 1] = W * fmax(-bn, 0.0);
                } else {
                    cv[0] = W * (P.c_out * fmax(bn, 0.0) + P.c_in * fmin(bn, 0.0));
                }
            }
#pragma unroll
            for (int sd = 0; sd < NS; sd++) {
                const int dir = (int)(f[sd] >> 1), side = (int)(f[sd] & 1u);
#pragma unroll
                for (int k = 0; k < N; k++) {
                    const int i = sd * ND + cell_dof<N>(dir, a, b, k);
                    const int g = __ldg(P.map0 + (long long)col * NS * ND + i) + __ldg(P.off0 + i) * layer;
                    const double pk = P.E[side][k];
                    const double val = MODE == DG_ACTION ? pk * cv[sd] : pk * pk * cv[sd];
                    if (ATOMIC) atomicAdd(P.y + g, val);
                    else P.y[g] += val;
                }
            }
        }
        __syncthreads();          // the slot's buffers are refilled by the next facet
    }
}

template <class Kern, class Params>
int launch_facets(Kern kern, int threads, int fpb, cudaStream_t st, const Params &P, int sm_count)
{
    int per_sm = 0;
    FDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, 0));
    const long long nunits = (long long)P.ncols * P.nlay_items;
    long long grid = (nunits + fpb - 1) / fpb;
    const long long cap = (long long)sm_count * (per_sm > 0 ? per_sm : 1);
    if (grid > cap) grid = cap;
    if (grid < 1) return 0;
    kern<<<(int)grid, threads, 0, st>>>(P);
    FDB_LAUNCH_CHECK();
    return 0;
}

// The launches of one facet call: one atomic launch (the diagonal, or FDB_SCATTER_ATOMIC), or one launch per
// (colour, layer parity), in which no two facets share a dof.  run(P, diagonal, atomic) launches the kernel.
template <class Params, class Run>
int schedule_facets(const fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, bool diagonal,
                    Params &P, Run run)
{
    if (diagonal || k->desc.scatter == FDB_SCATTER_ATOMIC) {
        P.collist = subset;
        P.col0 = start;
        P.ncols = end - start;
        P.nlay_items = nlay;
        P.lay_first = 0;
        P.lay_step = 1;
        if (P.ncols <= 0 || nlay <= 0) return 0;
        return run(P, diagonal, true);
    }
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
            if (run(P, false, false)) return 1;
        }
    }
    return 0;
}

template <int N, bool INTERIOR>
int run_n(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
          const double *coords, const double *x, const unsigned *facet, const fdb_int *map0, const fdb_int *map1)
{
    fdb::Context &c = fdb::ctx();
    DGFacetParams<N> P;
    memset(&P, 0, sizeof(P));
    P.off0 = k->d_off0;
    P.off1 = k->d_off1;
    P.c_f = k->desc.alpha;
    P.c_p = k->desc.beta;
    P.c_m = k->desc.dcoef[0];
    P.c_s = k->desc.dcoef[1];
    for (int i = 0; i < N * N; i++) {
        P.B[i] = k->desc.B[i];
        P.D[i] = k->desc.D[i];
    }
    for (int i = 0; i < N; i++) {
        P.wq[i] = k->desc.wq[i];
        P.xq[i] = k->desc.xq[i];
        for (int e = 0; e < 4; e++) P.E[e][i] = k->Bend[e * FDB_MAX_1D + i];
    }
    P.y = y;
    P.x = x;
    P.coords = coords;
    P.facet = facet;
    P.map0 = map0;
    P.map1 = map1;
    using S = DGFacetShape<N>;
    return schedule_facets(k, start, end, nlay, subset, !x, P, [&](const DGFacetParams<N> &Q, bool diag, bool atomic) {
        if (diag) return launch_facets(dg_facet_kernel<N, INTERIOR, DG_DIAGONAL, true>, S::THREADS, S::FPB, c.stream, Q, c.sm_count);
        if (atomic) return launch_facets(dg_facet_kernel<N, INTERIOR, DG_ACTION, true>, S::THREADS, S::FPB, c.stream, Q, c.sm_count);
        return launch_facets(dg_facet_kernel<N, INTERIOR, DG_ACTION, false>, S::THREADS, S::FPB, c.stream, Q, c.sm_count);
    });
}

template <int N, bool INTERIOR>
int run_upwind_n(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
                 const double *coords, const double *x, const double *b, const unsigned *facet, const fdb_int *map0,
                 const fdb_int *map1)
{
    fdb::Context &c = fdb::ctx();
    DGUpwindParams<N> P;
    memset(&P, 0, sizeof(P));
    P.off0 = k->d_off0;
    P.off1 = k->d_off1;
    P.c_out = k->desc.dcoef[0];
    P.c_in = k->desc.dcoef[1];
    for (int i = 0; i < N; i++) {
        P.wq[i] = k->desc.wq[i];
        P.xq[i] = k->desc.xq[i];
        for (int e = 0; e < 2; e++) P.E[e][i] = k->Bend[e * FDB_MAX_1D + i];
    }
    P.y = y;
    P.x = x;
    P.coords = coords;
    P.b = b;
    P.facet = facet;
    P.map0 = map0;
    P.map1 = map1;
    using S = DGFacetShape<N>;
    return schedule_facets(k, start, end, nlay, subset, !x, P, [&](const DGUpwindParams<N> &Q, bool diag, bool atomic) {
        if (diag) return launch_facets(dg_upwind_kernel<N, INTERIOR, DG_DIAGONAL, true>, S::THREADS, S::FPB, c.stream, Q, c.sm_count);
        if (atomic) return launch_facets(dg_upwind_kernel<N, INTERIOR, DG_ACTION, true>, S::THREADS, S::FPB, c.stream, Q, c.sm_count);
        return launch_facets(dg_upwind_kernel<N, INTERIOR, DG_ACTION, false>, S::THREADS, S::FPB, c.stream, Q, c.sm_count);
    });
}

template <bool INTERIOR>
int run_interior(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
                 const double *coords, const double *x, const unsigned *facet, const fdb_int *map0,
                 const fdb_int *map1)
{
    switch (k->n1d) {
    case 2: return run_n<2, INTERIOR>(k, start, end, nlay, subset, y, coords, x, facet, map0, map1);
    case 3: return run_n<3, INTERIOR>(k, start, end, nlay, subset, y, coords, x, facet, map0, map1);
    case 4: return run_n<4, INTERIOR>(k, start, end, nlay, subset, y, coords, x, facet, map0, map1);
    case 5: return run_n<5, INTERIOR>(k, start, end, nlay, subset, y, coords, x, facet, map0, map1);
    }
    fdb::set_error("dg facet kernel: degree %d not instantiated (1..4)", k->n1d - 1);
    return 1;
}

template <bool INTERIOR>
int run_upwind(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
               const double *coords, const double *x, const double *b, const unsigned *facet, const fdb_int *map0,
               const fdb_int *map1)
{
    switch (k->n1d) {
    case 2: return run_upwind_n<2, INTERIOR>(k, start, end, nlay, subset, y, coords, x, b, facet, map0, map1);
    case 3: return run_upwind_n<3, INTERIOR>(k, start, end, nlay, subset, y, coords, x, b, facet, map0, map1);
    case 4: return run_upwind_n<4, INTERIOR>(k, start, end, nlay, subset, y, coords, x, b, facet, map0, map1);
    case 5: return run_upwind_n<5, INTERIOR>(k, start, end, nlay, subset, y, coords, x, b, facet, map0, map1);
    }
    fdb::set_error("dg upwind kernel: degree %d not instantiated (1..4)", k->n1d - 1);
    return 1;
}

}  // namespace

int fdb_launch_dg_facet(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
                        const double *coords, const double *x, const unsigned *facet, const fdb_int *map0,
                        const fdb_int *map1)
{
    if (k->desc.integral == FDB_INTEGRAL_INTERIOR_FACET)
        return run_interior<true>(k, start, end, nlay, subset, y, coords, x, facet, map0, map1);
    return run_interior<false>(k, start, end, nlay, subset, y, coords, x, facet, map0, map1);
}

int fdb_launch_dg_upwind(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *y,
                         const double *coords, const double *x, const double *b, const unsigned *facet,
                         const fdb_int *map0, const fdb_int *map1)
{
    if (k->desc.integral == FDB_INTEGRAL_INTERIOR_FACET)
        return run_upwind<true>(k, start, end, nlay, subset, y, coords, x, b, facet, map0, map1);
    return run_upwind<false>(k, start, end, nlay, subset, y, coords, x, b, facet, map0, map1);
}
