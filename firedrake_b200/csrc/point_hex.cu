// Point evaluation and point loads (receivers and sources of the wave equation, DESIGN.md section 4.18).  A point k
// lies in one cell: idx[k*nper + j] are that cell's nper = (p+1)^3 global nodes and w[k*nper + j] = phi_j(x_k) their
// basis weights, located once on the host (assemble.PointEvaluator).  Both kernels fix the order of every sum, so
// their results are bit-reproducible:
//   eval  one thread per point sums its nper terms in j order;
//   load  one CTA walks the points in k order, one thread per node of the point's cell, with a barrier between two
//         points: a cell's nodes are distinct, so no two threads write one entry at once, and a node shared by
//         several points takes their terms in k order.  The point counts here are small (sources of a survey).
// A point with idx[k*nper] < 0 was not found: it evaluates to NaN and loads nothing.
#include "common.cuh"

using namespace fdb;

namespace {

__global__ void k_point_eval(fdb_int npts, int nper, const fdb_int *__restrict__ idx, const double *__restrict__ w,
                             const double *__restrict__ u, double *__restrict__ out)
{
    const fdb_int k = (fdb_int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (k >= npts) return;
    const long long b = (long long)k * nper;
    if (idx[b] < 0) {
        out[k] = __longlong_as_double(0x7ff8000000000000ll);      // quiet NaN
        return;
    }
    double s = 0.0;
    for (int j = 0; j < nper; j++) s = fma(w[b + j], u[idx[b + j]], s);
    out[k] = s;
}

__global__ void k_point_load(fdb_int npts, int nper, const fdb_int *__restrict__ idx, const double *__restrict__ w,
                             const double *__restrict__ a, double scale, double *y)
{
    for (fdb_int k = 0; k < npts; k++) {
        const long long b = (long long)k * nper;
        if (idx[b] >= 0)                                            // uniform over the CTA
            for (int j = threadIdx.x; j < nper; j += blockDim.x) y[idx[b + j]] += scale * a[k] * w[b + j];
        __syncthreads();                                            // point k's writes land before point k+1's
    }
}

}  // namespace

extern "C" {

int fdb_point_eval(fdb_int npts, int nper, const fdb_int *idx, const double *w, const double *u, double *out)
{
    if (require_init()) return 1;
    if (npts <= 0) return 0;
    if (nper < 1) {
        set_error("fdb_point_eval: nper = %d (>= 1)", nper);
        return 1;
    }
    k_point_eval<<<(npts + 127) / 128, 128, 0, ctx().stream>>>(npts, nper, idx, w, u, out);
    FDB_LAUNCH_CHECK();
    return 0;
}

int fdb_point_load(fdb_int npts, int nper, const fdb_int *idx, const double *w, const double *a, double scale,
                   double *y)
{
    if (require_init()) return 1;
    if (npts <= 0) return 0;
    if (nper < 1) {
        set_error("fdb_point_load: nper = %d (>= 1)", nper);
        return 1;
    }
    const int threads = nper < 256 ? ((nper + 31) / 32) * 32 : 256;
    k_point_load<<<1, threads, 0, ctx().stream>>>(npts, nper, idx, w, a, scale, y);
    FDB_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
