// Degree transfers between CG_p and CG_q (q < p) on the same hex mesh, both on GLL nodes: FDB_FORM_P_PROLONG,
// FDB_FORM_P_RESTRICT and FDB_FORM_P_INJECT, the level transfers of p-multigrid (DESIGN.md section 4.17).
//
//   prolong   fine  = (P (x) P (x) P) coarse                   WRITE into fine
//   restrict  coarse += (P (x) P (x) P)^T (w o fine)           INC into coarse (atomic or coloured)
//   inject    coarse = (R (x) R (x) R) fine                    WRITE into coarse
//
// P (p+1, q+1) is the coarse 1-D basis at the fine nodes, R (q+1, p+1) the fine basis at the coarse nodes, both in
// 1-D dof numbering (dof 0 at x = 0, dof 1 at x = 1, then the interior).  w = 1 / (cells containing the fine node),
// so that the restriction is exactly P^T.
//
// Every cell sharing a fine node writes it in prolong (and every cell sharing a coarse node writes it in inject).
// fdb_kernel_create checks that the endpoint rows of P and R are exact unit vectors, and the contraction runs over
// the axes in one fixed order (first axis outermost): a node on a shared face then takes the face plane's values
// exactly along the normal axis and the same products in the same order along the tangential ones, so every writer
// stores bitwise the same value and the result does not depend on which write lands last.  This needs neighbouring
// cells to share the orientation of their local axes, so that the tangential contractions of a shared face run over
// the same nodes in the same order from both sides: true of ExtrudedHexMesh, whose cells all have their local x, y,
// z along the mesh's.
//
// Layout: one thread per fine node of a cell, CPB cells per CTA, the cell's input in static shared memory.  The
// operations per byte are few: these kernels are judged on bandwidth.
#include "common.cuh"

namespace {

enum { PT_PROLONG = 0, PT_RESTRICT = 1, PT_INJECT = 2 };

template <int NF, int NC>
struct TransferParams {
    double *out;
    const double *in, *w;             // w: restrict only, one value per fine node
    const fdb_int *mapf, *mapc;       // fine (NF^3) and coarse (NC^3) rows per column
    const fdb_int *offf, *offc;       // their layer offsets (zeros on native hexes)
    const fdb_int *collist;           // columns to visit (subset or colour) or NULL = col0 + i
    int col0, ncols;
    int nlay_items, lay_first, lay_step;   // layers lay_first + i * lay_step, i < nlay_items
    double P[NF * NC];                // P[i * NC + a]
    double R[NC * NF];                // R[a * NF + i]
};

template <int NF>
struct TransferShape {
    static constexpr int ND = NF * NF * NF;                   // threads per cell: one per fine node
    static constexpr int CPB = 256 / ND;
    static constexpr int THREADS = ((CPB * ND + 31) / 32) * 32;
};

template <int NF, int NC, int CDIM, int KIND, bool ATOMIC>
__global__ void __launch_bounds__(TransferShape<NF>::THREADS)
p_transfer_kernel(const __grid_constant__ TransferParams<NF, NC> T)
{
    using S = TransferShape<NF>;
    constexpr int ND = S::ND, CPB = S::CPB, NC3 = NC * NC * NC;
    constexpr int NIN = KIND == PT_PROLONG ? NC3 : ND;        // input nodes per cell
    __shared__ double s_in[CPB][NIN * CDIM];
    const int slot = threadIdx.x / ND;
    const int l = threadIdx.x - slot * ND;
    const bool in_cta = slot < CPB;
    const int sl = in_cta ? slot : 0;

    const long long nunits = (long long)T.ncols * T.nlay_items;
    for (long long base = (long long)blockIdx.x * CPB; base < nunits; base += (long long)gridDim.x * CPB) {
        const long long unit = base + slot;
        const bool valid = in_cta && unit < nunits;
        int col = 0, layer = 0;
        if (valid) {
            const int ci = (int)(unit / T.nlay_items);
            layer = T.lay_first + (int)(unit - (long long)ci * T.nlay_items) * T.lay_step;
            col = T.collist ? __ldg(T.collist + ci) : T.col0 + ci;
            if (KIND == PT_PROLONG) {
                if (l < NC3) {
                    const long long g = __ldg(T.mapc + (long long)col * NC3 + l) + (long long)__ldg(T.offc + l) * layer;
#pragma unroll
                    for (int c = 0; c < CDIM; c++) s_in[sl][l * CDIM + c] = __ldg(T.in + g * CDIM + c);
                }
            } else {
                const long long g = __ldg(T.mapf + (long long)col * ND + l) + (long long)__ldg(T.offf + l) * layer;
                const double wt = KIND == PT_RESTRICT ? __ldg(T.w + g) : 1.0;
#pragma unroll
                for (int c = 0; c < CDIM; c++) s_in[sl][l * CDIM + c] = wt * __ldg(T.in + g * CDIM + c);
            }
        }
        __syncthreads();
        if (valid && KIND == PT_PROLONG) {
            const int i0 = l / (NF * NF), i1 = (l / NF) % NF, i2 = l % NF;
            const long long g = __ldg(T.mapf + (long long)col * ND + l) + (long long)__ldg(T.offf + l) * layer;
#pragma unroll
            for (int c = 0; c < CDIM; c++) {
                double v = 0.0;
#pragma unroll
                for (int a = 0; a < NC; a++) {
                    double va = 0.0;
#pragma unroll
                    for (int b = 0; b < NC; b++) {
                        double vb = 0.0;
#pragma unroll
                        for (int d = 0; d < NC; d++) vb = fma(T.P[i2 * NC + d], s_in[sl][((a * NC + b) * NC + d) * CDIM + c], vb);
                        va = fma(T.P[i1 * NC + b], vb, va);
                    }
                    v = fma(T.P[i0 * NC + a], va, v);
                }
                T.out[g * CDIM + c] = v;
            }
        }
        if (valid && KIND != PT_PROLONG && l < NC3) {
            const int a0 = l / (NC * NC), a1 = (l / NC) % NC, a2 = l % NC;
            const long long g = __ldg(T.mapc + (long long)col * NC3 + l) + (long long)__ldg(T.offc + l) * layer;
            // restrict: the columns of P; inject: the rows of R
            auto t = [&](int a, int i) { return KIND == PT_RESTRICT ? T.P[i * NC + a] : T.R[a * NF + i]; };
#pragma unroll 1          // unrolled over the components as well, the NF = 4 vector kernels spill
            for (int c = 0; c < CDIM; c++) {
                double v = 0.0;
#pragma unroll
                for (int i = 0; i < NF; i++) {
                    double vi = 0.0;
#pragma unroll
                    for (int j = 0; j < NF; j++) {
                        double vj = 0.0;
#pragma unroll
                        for (int k = 0; k < NF; k++) vj = fma(t(a2, k), s_in[sl][((i * NF + j) * NF + k) * CDIM + c], vj);
                        vi = fma(t(a1, j), vj, vi);
                    }
                    v = fma(t(a0, i), vi, v);
                }
                if (KIND == PT_INJECT) T.out[g * CDIM + c] = v;
                else if (ATOMIC) atomicAdd(T.out + g * CDIM + c, v);
                else T.out[g * CDIM + c] += v;                    // colour and layer parity: no other writer
            }
        }
        __syncthreads();                                            // the slot's buffer is refilled next
    }
}

template <int NF, int NC, int CDIM, int KIND, bool ATOMIC>
int launch(const TransferParams<NF, NC> &T)
{
    using S = TransferShape<NF>;
    fdb::Context &c = fdb::ctx();
    auto kern = p_transfer_kernel<NF, NC, CDIM, KIND, ATOMIC>;
    int per_sm = 0;
    FDB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, S::THREADS, 0));
    const long long nunits = (long long)T.ncols * T.nlay_items;
    long long grid = (nunits + S::CPB - 1) / S::CPB;
    const long long cap = (long long)c.sm_count * (per_sm > 0 ? per_sm : 1);
    if (grid > cap) grid = cap;
    if (grid < 1) return 0;
    kern<<<(int)grid, S::THREADS, 0, c.stream>>>(T);
    FDB_LAUNCH_CHECK();
    return 0;
}

template <int NF, int NC, int CDIM>
int run(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *out, const double *in,
        const double *w, const fdb_int *mapf, const fdb_int *mapc)
{
    TransferParams<NF, NC> T;
    memset(&T, 0, sizeof(T));
    T.out = out;
    T.in = in;
    T.w = w;
    T.mapf = mapf;
    T.mapc = mapc;
    T.offf = k->d_off0;
    T.offc = k->d_off2;
    for (int i = 0; i < NF * NC; i++) {
        T.P[i] = k->B2[i];
        T.R[i] = k->desc.B[i];
    }
    const int form = k->desc.form;
    if (form != FDB_FORM_P_RESTRICT || k->desc.scatter == FDB_SCATTER_ATOMIC) {
        T.collist = subset;
        T.col0 = start;
        T.ncols = end - start;
        T.nlay_items = nlay;
        T.lay_step = 1;
        if (T.ncols <= 0 || nlay <= 0) return 0;
        if (form == FDB_FORM_P_PROLONG) return launch<NF, NC, CDIM, PT_PROLONG, false>(T);
        if (form == FDB_FORM_P_INJECT) return launch<NF, NC, CDIM, PT_INJECT, false>(T);
        return launch<NF, NC, CDIM, PT_RESTRICT, true>(T);
    }
    // deterministic restrict: one launch per (colour, layer parity), no two cells of a launch share a node
    if (subset) {
        fdb::set_error("p_restrict: coloured scatter does not support subsets");
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
            if (launch<NF, NC, CDIM, PT_RESTRICT, false>(T)) return 1;
        }
    }
    return 0;
}

template <int CDIM>
int run_cdim(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *out,
             const double *in, const double *w, const fdb_int *mapf, const fdb_int *mapc)
{
    const int p = k->desc.degree, q = k->desc.nq - 1;
    if (p == 2 && q == 1) return run<3, 2, CDIM>(k, start, end, nlay, subset, out, in, w, mapf, mapc);
    if (p == 3 && q == 1) return run<4, 2, CDIM>(k, start, end, nlay, subset, out, in, w, mapf, mapc);
    if (p == 3 && q == 2) return run<4, 3, CDIM>(k, start, end, nlay, subset, out, in, w, mapf, mapc);
    fdb::set_error("p transfer: degree pair (%d, %d) not instantiated: (2, 1), (3, 1), (3, 2)", p, q);
    return 1;
}

}  // namespace

int fdb_launch_p_transfer(fdb_kernel_s *k, fdb_int start, fdb_int end, int nlay, const fdb_int *subset, double *out,
                          const double *in, const double *w, const fdb_int *mapf, const fdb_int *mapc)
{
    if (k->desc.cdim == 1) return run_cdim<1>(k, start, end, nlay, subset, out, in, w, mapf, mapc);
    if (k->desc.cdim == 3) return run_cdim<3>(k, start, end, nlay, subset, out, in, w, mapf, mapc);
    fdb::set_error("p transfer: cdim %d (1 or 3)", k->desc.cdim);
    return 1;
}
