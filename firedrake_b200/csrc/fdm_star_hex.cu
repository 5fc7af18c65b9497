// Fast-diagonalisation vertex-star relaxation on extruded CG_p hexahedra (DESIGN.md section 4.20).
//
// For every mesh vertex v the patch is the open star of v: on the p-refined node lattice, the nodes closer than p to
// v in every direction, m = 2p - 1 per direction.  Its operator is replaced by the Kronecker sum
//   A_v = a_v (K_x (x) M_y (x) M_z + M_x (x) K_y (x) M_z + M_x (x) M_y (x) K_z) + beta M_x (x) M_y (x) M_z,
// a_v = alpha * mean(kappa over the star), whose inverse is (S_x (x) S_y (x) S_z) diag(1 / (a_v (lx + ly + lz) +
// beta)) (S_x (x) S_y (x) S_z)^T with the generalised eigenpairs K_d S_d = M_d S_d L_d, S_d^T M_d S_d = I (built on
// the host, patch.FDMStar).  The relaxation is additive: z = sum_v R_v^T A_v^-1 R_v r.
//
// Every star has one shape: each direction is padded to m nodes; a padded node (no cell on that side) or a node
// removed by a Dirichlet condition has a zero row in S, eigenvalue 1 and the gathered value 0.  The 1-D tables live
// in a deduplicated pool, an entry of m*m + 3m doubles: S (row = star node, column = mode), the eigenvalues, the
// active mask (1: in the patch) and the existence mask (1: some cell of the star holds the node).
//
// One group of m^2 threads per star, several stars per CTA.  Thread (j, k) gathers the x-line (., j, k) of the star
// into registers and contracts it with S_x^T; the y- and z-contractions, the scaling and the z- and y-expansions run
// on lines of shared memory; the same thread expands its x-line and adds it into z.  The scatter is not atomic:
// the stars are launched in the 8 colours of the vertex lattice (parities of i, j and layer), and stars of one colour
// share no node, so the result is bitwise repeatable.
//
// The cells of a star are found through the vertex -> base-column table (quadrant sx*2 + sy, -1 where there is no
// cell) and the extruded cell-node map (base-cell map + layer * offset).  The mesh's cells share their local axes
// with the vertex lattice (ExtrudedHexMesh), so the star's x-offset o of a node is its local position in the cell on
// side sx: o + p on the left (sx = 0), o on the right.
#include <vector>

#include "common.cuh"

using namespace fdb;

struct fdb_fdm_star_s {
    int degree = 0, nz = 0, ncols = 0, nvert = 0, nstar = 0, npool = 0;
    fdb_int node_count = 0;
    long long colour_ptr[9] = {0};
    const fdb_int *d_cmap = nullptr, *d_off = nullptr;   // the caller's device cell map and offsets, not owned
    fdb_int *d_vcols = nullptr;
    fdb_int *d_svert = nullptr, *d_slay = nullptr, *d_stab = nullptr;
    double *d_pool = nullptr;
    double *d_ak = nullptr;          // alpha * mean kappa per star
    double beta = 0.0;
};

namespace {

struct StarArgs {
    int nz;
    const fdb_int *__restrict__ cmap;    // [ncols][N^3] base-cell map
    const fdb_int *__restrict__ off;     // [N^3] layer offsets
    const fdb_int *__restrict__ vcols;   // [nvert][4] base column of quadrant sx*2 + sy, -1 where there is none
    const fdb_int *__restrict__ svert;   // per star: base vertex,
    const fdb_int *__restrict__ slay;    //           node layer K (the cells below and above are K-1 and K),
    const fdb_int *__restrict__ stab;    //           [3] pool entries of the x, y and z tables
    const double *__restrict__ pool;
};

template <int P>
struct Shape {
    static constexpr int M = 2 * P - 1, M2 = M * M, M3 = M2 * M, E = M2 + 3 * M;
    static constexpr int G = 256 / M2;   // stars per CTA
    static constexpr int T = G * M2;     // threads per CTA
};

// entity-ordered 1-D dof number of the local position a (0 = left vertex, 1 = right vertex, 2.. interior)
template <int P>
__device__ __forceinline__ int pos2dof(int a)
{
    return a == 0 ? 0 : (a == P ? 1 : a + 1);
}

// the global nodes of the x-line (., j, k) of a star, -1 where the node does not exist
template <int P>
__device__ __forceinline__ void line_nodes(const StarArgs &a, int vert, int K, int j, int k, int node[2 * P - 1])
{
    constexpr int N = P + 1, M = 2 * P - 1;
    const fdb_int *vc = a.vcols + 4 * (size_t)vert;
    const int rx = (vc[2] >= 0) | (vc[3] >= 0), ry = (vc[1] >= 0) | (vc[3] >= 0), rz = K < a.nz;
    const int oy = j - (P - 1), oz = k - (P - 1);
    const int sy = oy < 0 ? 0 : (oy > 0 ? 1 : ry), sz = oz < 0 ? 0 : (oz > 0 ? 1 : rz);
    const int dy = pos2dof<P>(sy ? oy : oy + P), dz = pos2dof<P>(sz ? oz : oz + P);
    const int layer = K - 1 + sz;
    const bool zok = layer >= 0 && layer < a.nz;
#pragma unroll
    for (int i = 0; i < M; i++) {
        const int ox = i - (P - 1);
        const int sx = ox < 0 ? 0 : (ox > 0 ? 1 : rx);
        const int col = vc[sx * 2 + sy];
        const int loc = (pos2dof<P>(sx ? ox : ox + P) * N + dy) * N + dz;
        node[i] = (col >= 0 && zok) ? a.cmap[(size_t)col * (N * N * N) + loc] + layer * a.off[loc] : -1;
    }
}

template <int P>
__device__ __forceinline__ void load_tables(const StarArgs &a, int s, bool live, int t, double *tab)
{
    using S = Shape<P>;
    if (live)
        for (int e = t; e < 3 * S::E; e += S::M2) {
            const int d = e / S::E, r = e - d * S::E;
            tab[e] = a.pool[(size_t)a.stab[3 * (size_t)s + d] * S::E + r];
        }
}

// out[c] = sum_i T[i][c] in[i] (transpose: the S^T contraction) or out[i] = sum_c T[i][c] in[c]
template <int M, bool TRANSPOSE>
__device__ __forceinline__ void contract(const double *__restrict__ T, const double in[M], double out[M])
{
#pragma unroll
    for (int c = 0; c < M; c++) {
        double acc = 0.0;
#pragma unroll
        for (int i = 0; i < M; i++) acc = fma(TRANSPOSE ? T[i * M + c] : T[c * M + i], in[i], acc);
        out[c] = acc;
    }
}

// one colour of stars [first, first + count): z[R_v^T A_v^-1 R_v r] += for every star
template <int P>
__global__ void __launch_bounds__(Shape<P>::T) k_fdm_star_apply(StarArgs a, int first, int count,
                                                                  const double *__restrict__ ak, double beta,
                                                                  const double *__restrict__ r, double *__restrict__ z)
{
    using S = Shape<P>;
    constexpr int M = S::M, M2 = S::M2, E = S::E;
    __shared__ double sh_u[S::G][S::M3];
    __shared__ double sh_tab[S::G][3 * E];
    const int g = threadIdx.x / M2, t = threadIdx.x - g * M2;
    const int sl = blockIdx.x * S::G + g;
    const bool live = g < S::G && sl < count;
    const int s = first + sl;
    double *u = sh_u[g < S::G ? g : 0];
    const double *tab = sh_tab[g < S::G ? g : 0];
    const double *Sx = tab, *Sy = tab + E, *Sz = tab + 2 * E;
    load_tables<P>(a, s, live, t, sh_tab[g < S::G ? g : 0]);
    __syncthreads();

    // gather the x-line (., j, k) and contract it with S_x^T
    int node[M];
    double v[M], w[M];
    const int j0 = t / M, k0 = t - j0 * M;
    if (live) {
        line_nodes<P>(a, a.svert[s], a.slay[s], j0, k0, node);
        const double act = Sy[M2 + M + j0] * Sz[M2 + M + k0];
#pragma unroll
        for (int i = 0; i < M; i++) v[i] = (act * Sx[M2 + M + i] != 0.0) ? r[node[i]] : 0.0;
        contract<M, true>(Sx, v, w);
#pragma unroll
        for (int c = 0; c < M; c++) u[(c * M + j0) * M + k0] = w[c];
    }
    __syncthreads();
    // y: thread (c, k) contracts the line u[c][.][k] with S_y^T
    const int c0 = t / M, kk = t - c0 * M;
    if (live) {
#pragma unroll
        for (int j = 0; j < M; j++) v[j] = u[(c0 * M + j) * M + kk];
        contract<M, true>(Sy, v, w);
#pragma unroll
        for (int j = 0; j < M; j++) u[(c0 * M + j) * M + kk] = w[j];
    }
    __syncthreads();
    // z: thread (a, b) contracts u[a][b][.] with S_z^T, scales by the reciprocal eigenvalue sum, expands with S_z
    const int ax = t / M, by = t - ax * M;
    if (live) {
        const double av = ak[s];
        const double lxy = Sx[M2 + ax] + Sy[M2 + by];
#pragma unroll
        for (int k = 0; k < M; k++) v[k] = u[(ax * M + by) * M + k];
        contract<M, true>(Sz, v, w);
#pragma unroll
        for (int k = 0; k < M; k++) w[k] = w[k] / fma(av, lxy + Sz[M2 + k], beta);
        contract<M, false>(Sz, w, v);
#pragma unroll
        for (int k = 0; k < M; k++) u[(ax * M + by) * M + k] = v[k];
    }
    __syncthreads();
    // y expansion
    if (live) {
#pragma unroll
        for (int j = 0; j < M; j++) v[j] = u[(c0 * M + j) * M + kk];
        contract<M, false>(Sy, v, w);
#pragma unroll
        for (int j = 0; j < M; j++) u[(c0 * M + j) * M + kk] = w[j];
    }
    __syncthreads();
    // x expansion of this thread's line and the scatter: no other star of this colour holds these nodes
    if (live) {
        const double act = Sy[M2 + M + j0] * Sz[M2 + M + k0];
#pragma unroll
        for (int c = 0; c < M; c++) v[c] = u[(c * M + j0) * M + k0];
        contract<M, false>(Sx, v, w);
#pragma unroll
        for (int i = 0; i < M; i++)
            if (act * Sx[M2 + M + i] != 0.0) z[node[i]] += w[i];
    }
}

// ak[s] = alpha * (mean of kappa over the existing nodes of star s), or alpha without kappa
template <int P>
__global__ void __launch_bounds__(Shape<P>::T) k_fdm_star_mean(StarArgs a, int nstar, double alpha,
                                                                 const double *__restrict__ kappa,
                                                                 double *__restrict__ ak)
{
    using S = Shape<P>;
    constexpr int M = S::M, M2 = S::M2, E = S::E;
    __shared__ double sh_sum[S::G][M2];
    __shared__ double sh_cnt[S::G][M2];
    __shared__ double sh_tab[S::G][3 * E];
    const int g = threadIdx.x / M2, t = threadIdx.x - g * M2;
    const int s = blockIdx.x * S::G + g;
    const bool live = g < S::G && s < nstar;
    const int gg = g < S::G ? g : 0;
    load_tables<P>(a, s, live, t, sh_tab[gg]);
    __syncthreads();
    if (live) {
        const double *tab = sh_tab[gg];
        int node[M];
        const int j0 = t / M, k0 = t - j0 * M;
        line_nodes<P>(a, a.svert[s], a.slay[s], j0, k0, node);
        const double has = tab[E + M2 + 2 * M + j0] * tab[2 * E + M2 + 2 * M + k0];
        double sum = 0.0, cnt = 0.0;
#pragma unroll
        for (int i = 0; i < M; i++)
            if (has * tab[M2 + 2 * M + i] != 0.0) {
                sum += kappa ? kappa[node[i]] : 1.0;
                cnt += 1.0;
            }
        sh_sum[gg][t] = sum;
        sh_cnt[gg][t] = cnt;
    }
    __syncthreads();
    if (live && t == 0) {
        double sum = 0.0, cnt = 0.0;
        for (int e = 0; e < M2; e++) {
            sum += sh_sum[gg][e];
            cnt += sh_cnt[gg][e];
        }
        ak[s] = alpha * (sum / cnt);
    }
}

StarArgs args_of(const fdb_fdm_star_s *h)
{
    return StarArgs{h->nz, h->d_cmap, h->d_off, h->d_vcols, h->d_svert, h->d_slay, h->d_stab, h->d_pool};
}

template <int P>
int launch_apply(const fdb_fdm_star_s *h, const double *r, double *z)
{
    using S = Shape<P>;
    const StarArgs a = args_of(h);
    for (int c = 0; c < 8; c++) {
        const int first = (int)h->colour_ptr[c], count = (int)(h->colour_ptr[c + 1] - h->colour_ptr[c]);
        if (count == 0) continue;
        k_fdm_star_apply<P><<<(count + S::G - 1) / S::G, S::T, 0, ctx().stream>>>(a, first, count, h->d_ak, h->beta,
                                                                                  r, z);
        FDB_LAUNCH_CHECK();
    }
    return 0;
}

template <int P>
int launch_mean(const fdb_fdm_star_s *h, double alpha, const double *kappa)
{
    using S = Shape<P>;
    if (h->nstar == 0) return 0;
    k_fdm_star_mean<P><<<(h->nstar + S::G - 1) / S::G, S::T, 0, ctx().stream>>>(args_of(h), h->nstar, alpha, kappa,
                                                                                 h->d_ak);
    FDB_LAUNCH_CHECK();
    return 0;
}

template <typename T>
int upload(T **dst, const T *src, size_t n)
{
    FDB_CUDA(cudaMalloc(dst, sizeof(T) * (n ? n : 1)));
    if (n) FDB_CUDA(cudaMemcpyAsync(*dst, src, sizeof(T) * n, cudaMemcpyHostToDevice, ctx().stream));
    return 0;
}

}  // namespace

extern "C" {

int fdb_fdm_star_destroy(fdb_fdm_star_t h)
{
    if (!h) return 0;
    if (ctx().ready) {
        cudaStreamSynchronize(ctx().stream);
        cudaFree(h->d_vcols);
        cudaFree(h->d_svert);
        cudaFree(h->d_slay);
        cudaFree(h->d_stab);
        cudaFree(h->d_pool);
        cudaFree(h->d_ak);
    }
    delete h;
    return 0;
}

int fdb_fdm_star_create(int degree, int nz, int ncols, const fdb_int *cell_node_map, const fdb_int *offset,
                        fdb_int node_count, int nvert, const fdb_int *vert_cols, int nstar, const fdb_int *star_vert,
                        const fdb_int *star_layer, const fdb_int *star_table, const long long *colour_ptr, int npool,
                        const double *pool, fdb_fdm_star_t *out)
{
    if (require_init()) return 1;
    if (degree < 1 || degree > 5) {
        set_error("fdb_fdm_star_create: degree %d outside 1..5", degree);
        return 1;
    }
    if (nz < 1 || ncols < 0 || nvert < 0 || nstar < 0 || npool < 0 || node_count < 0 || !out || !colour_ptr ||
        (ncols && (!cell_node_map || !offset)) || (nvert && !vert_cols) ||
        (nstar && (!star_vert || !star_layer || !star_table || !pool))) {
        set_error("fdb_fdm_star_create: bad arguments");
        return 1;
    }
    if (colour_ptr[0] != 0 || colour_ptr[8] != nstar) {
        set_error("fdb_fdm_star_create: colour offsets must run from 0 to nstar");
        return 1;
    }
    for (int c = 0; c < 8; c++)
        if (colour_ptr[c + 1] < colour_ptr[c]) {
            set_error("fdb_fdm_star_create: colour offsets must be non-decreasing");
            return 1;
        }
    for (long long e = 0; e < 4LL * nvert; e++)
        if (vert_cols[e] < -1 || vert_cols[e] >= ncols) {
            set_error("fdb_fdm_star_create: vertex %lld names base column %d of %d", e / 4, vert_cols[e], ncols);
            return 1;
        }
    for (int s = 0; s < nstar; s++) {
        if (star_vert[s] < 0 || star_vert[s] >= nvert || star_layer[s] < 0 || star_layer[s] > nz) {
            set_error("fdb_fdm_star_create: star %d at vertex %d, layer %d is outside the mesh", s, star_vert[s],
                      star_layer[s]);
            return 1;
        }
        for (int d = 0; d < 3; d++)
            if (star_table[3 * s + d] < 0 || star_table[3 * s + d] >= npool) {
                set_error("fdb_fdm_star_create: star %d names table %d of %d", s, star_table[3 * s + d], npool);
                return 1;
            }
    }
    const int m = 2 * degree - 1;
    const size_t entry = (size_t)m * m + 3 * m;
    fdb_fdm_star_s *h = new fdb_fdm_star_s;
    h->degree = degree;
    h->nz = nz;
    h->ncols = ncols;
    h->nvert = nvert;
    h->nstar = nstar;
    h->npool = npool;
    h->node_count = node_count;
    for (int c = 0; c < 9; c++) h->colour_ptr[c] = colour_ptr[c];
    h->d_cmap = cell_node_map;
    h->d_off = offset;
    if (upload(&h->d_vcols, vert_cols, 4 * (size_t)nvert) || upload(&h->d_svert, star_vert, (size_t)nstar) ||
        upload(&h->d_slay, star_layer, (size_t)nstar) || upload(&h->d_stab, star_table, 3 * (size_t)nstar) ||
        upload(&h->d_pool, pool, (size_t)npool * entry)) {
        fdb_fdm_star_destroy(h);
        return 1;
    }
    if (cudaMalloc(&h->d_ak, sizeof(double) * (nstar ? nstar : 1)) != cudaSuccess ||
        cudaStreamSynchronize(ctx().stream) != cudaSuccess) {
        set_error("fdb_fdm_star_create: device allocation or upload failed");
        fdb_fdm_star_destroy(h);
        return 1;
    }
    *out = h;
    return 0;
}

// alpha, beta and kappa (device, node-wise; NULL: 1) of the patch operators: a_v = alpha * mean kappa over the star
int fdb_fdm_star_update(fdb_fdm_star_t h, double alpha, double beta, const double *kappa)
{
    if (require_init()) return 1;
    if (!h) {
        set_error("fdb_fdm_star_update: NULL handle");
        return 1;
    }
    h->beta = beta;
    switch (h->degree) {
        case 1: return launch_mean<1>(h, alpha, kappa);
        case 2: return launch_mean<2>(h, alpha, kappa);
        case 3: return launch_mean<3>(h, alpha, kappa);
        case 4: return launch_mean<4>(h, alpha, kappa);
        default: return launch_mean<5>(h, alpha, kappa);
    }
}

// z = sum_v R_v^T A_v^-1 R_v r (device pointers; z is overwritten)
int fdb_fdm_star_apply(fdb_fdm_star_t h, const double *r, double *z)
{
    if (require_init()) return 1;
    if (!h || !r || !z || r == z) {
        set_error("fdb_fdm_star_apply: NULL handle or vector, or r == z");
        return 1;
    }
    FDB_CUDA(cudaMemsetAsync(z, 0, sizeof(double) * (size_t)h->node_count, ctx().stream));
    switch (h->degree) {
        case 1: return launch_apply<1>(h, r, z);
        case 2: return launch_apply<2>(h, r, z);
        case 3: return launch_apply<3>(h, r, z);
        case 4: return launch_apply<4>(h, r, z);
        default: return launch_apply<5>(h, r, z);
    }
}

}  // extern "C"
