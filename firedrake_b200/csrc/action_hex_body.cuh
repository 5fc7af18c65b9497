// Body of the slab-thread kernels of action_hex.cu (helmholtz_action_kernel, helmholtz_coef_kernel,
// nonlinear_residual_kernel, nonlinear_jacobian_kernel, advection_diffusion_kernel), included inside each
// __global__ function: the template parameters N, MASS, ATOMIC, MATRIX, SLIM, AFFINE, the parameter block P
// and, from the including kernel, `constexpr bool COEF`, `constexpr int NL`, `constexpr bool ADV`,
// `const double *kappa` and `const double *dcoef` are in scope.  A textual include rather than a __forceinline__ function taking
// P by reference: the reference changes the register allocation of the existing matrix-mode kernels,
// whose machine code this layout keeps exactly as it was before the coefficient form existed.
//
// NL (nonlinear diffusion, D(s) = dcoef[0] + dcoef[1] s + dcoef[2] s^2):
//   1  residual: x is u; the stiffness weight at a point is w D(u_q), u_q = U[qx][0] (no kappa buffer)
//   2  Jacobian: x is w, u is gathered into the kappa buffer (COEF layout) and interpolated to the
//      points there; the reference gradient g of w becomes D(u_q) g + D'(u_q) w_q ghat(u)_q, with
//      ghat(u)_q taken by collocated differentiation (Dt) of the buffer's quadrature values
//
// ADV (advection-diffusion, alpha*inner(grad u, grad v)*dx + inner(dot(b, grad u), v)*dx + beta*inner(u, v)*dx):
//   the COEF layout with three kappa buffers, one per component of b (AoS, gathered at 3 g + c with x's
//   indices g) and interpolated to the points in place like kappa; the stiffness weight stays w, and
//   w sign(det J) (b_q . h) -- h = sum_m r_m ghat_m = det J grad u -- goes to the value slot with the mass
    static_assert(!(SLIM && MATRIX), "matrix mode keeps the per-cell index buffer");
    static_assert(!(AFFINE && MATRIX), "the affine variant exists for 1-forms only");
    static_assert(!(AFFINE && COEF), "the coefficient form has no affine variant");
    static_assert(NL != 1 || (!COEF && !MATRIX && !AFFINE), "the residual is a 1-form without a kappa buffer");
    static_assert(NL != 2 || (COEF && !AFFINE), "the Jacobian keeps u in the kappa buffer");
    static_assert(!ADV || (COEF && NL == 0 && !SLIM && !AFFINE), "b takes the coefficient layout, three times");
    using WS = WarpSmem<N, SLIM, COEF, ADV ? 3 : 1>;
    constexpr int CW = WS::CW;
    constexpr int CWS = WS::CWS;
    constexpr int ND = N * N * N;
    constexpr int US = WS::US;
    constexpr int CS = WS::CS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *wbase = reinterpret_cast<double *>(smem_raw + (size_t)warp * WS::BYTES);
    double *s_tile = wbase;
    double *s_u = s_tile + WS::TILE;                 // [CWS][US]   (single buffer)
    double *s_coord = s_u + WS::UBUF;                // [CWS][CS]   (single buffer)
    double *s_stash = s_coord + WS::COORD;           // [CWS][GS]   (geometry coefficients, if STASH)
    constexpr bool STASH = WS::STASH > 0 && !MATRIX && !AFFINE;
    double *s_kap = s_stash + WS::STASH;             // [NKAP][CWS][US]   (kappa, if COEF; b's components if ADV)
    int *s_idx = reinterpret_cast<int *>(s_kap + WS::KAPPA);   // [2][CWS][US]  (empty if SLIM)
    int *s_mapraw = s_idx + WS::IDX;                 // [CWS][US], or [3][2][US] if SLIM
    int *s_vidx = s_mapraw + WS::MAPRAW;             // [2][CWS][8], or [3][2][8] if SLIM
    int *s_off0 = reinterpret_cast<int *>(smem_raw + (size_t)WPC<N, SLIM, COEF>::value * WS::BYTES);
    int *s_off1 = s_off0 + ND;

    for (int i = threadIdx.x; i < ND; i += blockDim.x) s_off0[i] = P.off0[i];
    if (threadIdx.x < 8) s_off1[threadIdx.x] = P.off1[threadIdx.x];
    __syncthreads();

    const int cw = lane / N, t = lane - cw * N;
    const bool lane_active = cw < CW;
    Tile<N> tile(s_tile, cw, t);

    const int ncells = P.ncols * P.nlay_items;      // < 2^31, checked by the launcher
    const int nitems = (ncells + CW - 1) / CW;
    const double eta = P.xq[lane_active ? t : 0];
    const double wy_alpha = P.wq[lane_active ? t : 0] * P.alpha;
    const double wy_beta = P.wq[lane_active ? t : 0] * P.beta;
    // NL == 2: this lane's row of Dt (d/d eta at qy = t), for the gradient of u along y
    [[maybe_unused]] double dyr[N];
    if constexpr (NL == 2) {
#pragma unroll
        for (int q = 0; q < N; q++) dyr[q] = P.Dt[(lane_active ? t : 0) * N + q];
    }

    // warp-uniform work iterator: chunks of consecutive items (one column's
    // worth) handed out by an atomic counter -> locality inside a chunk,
    // dynamic balance across SMs
    auto advance = [&](Unit u) -> Unit {
        if (u.item >= 0 && u.comp + 1 < P.cdim) {
            u.comp++;
            return u;
        }
        u.comp = 0;
        u.ib = SLIM ? (u.ib == 2 ? 0 : u.ib + 1) : (u.ib ^ 1);
        if (u.item >= 0 && u.cur + 1 < u.end) {
            u.cur++;
            u.item = u.cur;
            return u;
        }
        if (u.item == -2) return u;                  // queue already drained
        int base = 0;
        if (lane == 0) base = atomicAdd(P.counter, P.chunk);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= nitems) {
            u.item = -2;
            return u;
        }
        u.cur = base;
        u.end = min(base + P.chunk, nitems);
        u.item = base;
        return u;
    };

    // per-lane decode of a unit (cell -> column, layer); division by the
    // launch-constant layer count through a precomputed reciprocal
    auto decode = [&](Unit &u) {
        const int lin = u.item * CW + cw;
        u.valid = lane_active && u.item >= 0 && lin < ncells;
        unsigned ci = __umulhi((unsigned)lin, P.nlay_rcp);
        int kk = lin - (int)ci * P.nlay_items;
        if (kk >= P.nlay_items) { kk -= P.nlay_items; ci++; }
        if (!u.valid) { ci = 0; kk = 0; }
        u.layer = P.lay_first + P.lay_step * kk;
        u.col = P.collist ? __ldg(P.collist + ci) : (P.col0 + (int)ci);
        // cells of the warp that sit in the same column share one staged copy of
        // the map / vertex rows: the lowest such cell (leader) copies, the
        // others read its slot
        if (SLIM) {
            // at most two distinct columns per warp (launcher guarantees nlay_items >= CW)
            const int col0 = __shfl_sync(0xffffffffu, u.col, 0);
            u.src = (u.col != col0) ? 1 : 0;
            const unsigned peers = __match_any_sync(0xffffffffu, u.valid ? u.src : -1 - cw);
            u.lead = (__ffs(peers) - 1) / N == cw;
        } else {
            const unsigned peers = __match_any_sync(0xffffffffu, u.valid ? u.col : -1 - cw);
            u.src = (__ffs(peers) - 1) / N;
            u.lead = u.src == cw;
        }
    };
    auto row_of = [&](const Unit &u) -> int * {
        return SLIM ? s_mapraw + (u.ib * 2 + u.src) * US : s_mapraw + u.src * US;
    };
    auto vrow_of = [&](const Unit &u) -> int * {
        return SLIM ? s_vidx + (u.ib * 2 + u.src) * 8 : s_vidx + (u.ib * CWS + u.src) * 8;
    };

    // Three-stage gather pipeline, all through cp.async (no registers held, no
    // load the warp has to wait for):
    //   stage A (unit i+2): copy the bottom-cell map row / vertex row to smem
    //   stage B (unit i+1): indices = row + offset*layer; copy x values and
    //                       vertex coordinates to smem
    //   stage C (unit i)  : compute + scatter
    // Stage B is issued in N slices from inside the quadrature loop so that its
    // integer/LSU instructions fill issue slots the fp64 pipe leaves free.
    // Every lane touches only its own slots of s_u / s_idx / s_mapraw; s_vidx and
    // s_coord are shared by the N lanes of a cell and are read after the
    // wait + __syncwarp at the top of the loop.
    auto stageA = [&](const Unit &u) {
        if (u.valid && u.comp == 0 && u.lead) {
            const int *mrow = P.map0 + (long long)u.col * ND;
            int *sm = row_of(u);
            if ((ND % 4) == 0 && (US % 4) == 0) {
                // rows are 16-byte aligned: 128-bit copies
                for (int j = t; j < ND / 4; j += N) cp_async16(sm + 4 * j, mrow + 4 * j);
            } else {
#pragma unroll
                for (int j = 0; j < N * N; j++) cp_async4(sm + j * N + t, mrow + j * N + t);
            }
            int *sv = vrow_of(u);
            for (int v = t; v < 8; v += N) cp_async4(sv + v, P.map1 + (long long)u.col * 8 + v);
        }
    };
    auto stageB_coords = [&](const Unit &u) {
        if (u.valid && u.comp == 0) {
            const int *sv = vrow_of(u);
            double *scd = s_coord + cw * CS;
            for (int i = t; i < 24; i += N) {
                int v = i / 3, a = i - v * 3;
                int g = sv[v] + s_off1[v] * u.layer;
                cp_async8(scd + i, P.coords + (long long)g * 3 + a);
            }
        }
    };
    auto stageB_part = [&](const Unit &u, int ubuf, int part) {
        if (u.valid) {
            double *su = s_u + cw * US;
            int *si = s_idx + (u.ib * CWS + cw) * US;
            const int *sm = row_of(u);
            int g[N];
            if (SLIM || u.comp == 0) {
#pragma unroll
                for (int j = 0; j < N; j++) {
                    const int loc = (part * N + j) * N + t;
                    g[j] = sm[loc] + s_off0[loc] * u.layer;
                }
                if (!SLIM) {
#pragma unroll
                    for (int j = 0; j < N; j++) si[(part * N + j) * N + t] = g[j];
                }
            } else {
#pragma unroll
                for (int j = 0; j < N; j++) g[j] = si[(part * N + j) * N + t];
            }
            if (!MATRIX) {
#pragma unroll
                for (int j = 0; j < N; j++)
                    cp_async8(su + (part * N + j) * N + t, P.x + (long long)g[j] * P.cdim + u.comp);
            }
        }
    };
    // COEF: kappa's dof values, once per cell, with the gather indices of x (this lane's own slots,
    // written by its stageB_part calls, or recomputed from the staged row if SLIM).  Issued after
    // the quadrature loop of the unit before, which reads kappa's quadrature values from the same
    // buffer.
    auto stageB_kappa = [&](const Unit &u) {
        if constexpr (COEF) {
            if (!u.valid || u.comp != 0) return;
            double *sk = s_kap + cw * US;
            const int *si = s_idx + (u.ib * CWS + cw) * US;
            const int *sm = row_of(u);
#pragma unroll
            for (int j = 0; j < N * N; j++) {
                const int loc = j * N + t;
                const int g = SLIM ? sm[loc] + s_off0[loc] * u.layer : si[loc];
                if constexpr (ADV) {
#pragma unroll
                    for (int c = 0; c < 3; c++) cp_async8(sk + c * WS::UBUF + loc, kappa + 3ll * g + c);
                } else {
                    cp_async8(sk + loc, kappa + g);
                }
            }
        }
    };

    Unit cur{-1, 0, 0, 0, 0, false, 0, 0, 0, false};
    cur = advance(cur);
    decode(cur);
    Unit nxt = advance(cur);
    decode(nxt);
    stageA(cur);
    cp_async_commit();
    cp_async_wait<0>();
    __syncwarp();
    int ubuf = 0;
    stageB_coords(cur);
#pragma unroll
    for (int part = 0; part < N; part++) stageB_part(cur, ubuf, part);
    stageB_kappa(cur);
    stageA(nxt);
    cp_async_commit();
    double A1[3], A3[3], A6[3], c2[3], c4[3], c5[3], c7[3];
    double Gm[6], adet_c = 1.0;       // AFFINE: metric (xx, xy, xz, yy, yz, zz) and |det J| of the cell
#pragma unroll
    for (int i = 0; i < 6; i++) Gm[i] = 0.0;

    while (cur.item >= 0) {
        cp_async_wait<0>();      // values of `cur`, rows of `nxt` have landed
        __syncwarp();
        Unit nn = advance(nxt);
        decode(nn);

        const bool valid = cur.valid;
        const int cbuf = cur.ib;
        const double *sc = s_coord + cw * CS;
        if (cur.comp == 0) {
            // trilinear coefficients reduced at this lane's eta (see header comment)
#pragma unroll
            for (int a = 0; a < 3; a++) {
                double X000 = sc[0 * 3 + a], X001 = sc[1 * 3 + a], X010 = sc[2 * 3 + a],
                       X011 = sc[3 * 3 + a], X100 = sc[4 * 3 + a], X101 = sc[5 * 3 + a],
                       X110 = sc[6 * 3 + a], X111 = sc[7 * 3 + a];
                if (!valid) {   // keep idle lanes finite: unit cube
                    X000 = 0; X001 = (a == 2); X010 = (a == 1); X011 = (a >= 1);
                    X100 = (a == 0); X101 = (a != 1); X110 = (a != 2); X111 = 1;
                }
                double c1 = X100 - X000;
                c2[a] = X010 - X000;
                double c3 = X001 - X000;
                c4[a] = X110 - X100 - X010 + X000;
                c5[a] = X011 - X010 - X001 + X000;
                double c6 = X101 - X100 - X001 + X000;
                c7[a] = X111 - X110 - X101 - X011 + X100 + X010 + X001 - X000;
                A1[a] = fma(c4[a], eta, c1);
                A3[a] = fma(c5[a], eta, c3);
                A6[a] = fma(c7[a], eta, c6);
            }
            if (AFFINE) {
                // constant Jacobian: columns a = A1 (dx/dxi), b = c2 (dx/deta), c = A3 (dx/dzeta)
                double r0[3], r1[3], r2[3];
                r0[0] = c2[1] * A3[2] - c2[2] * A3[1];
                r0[1] = c2[2] * A3[0] - c2[0] * A3[2];
                r0[2] = c2[0] * A3[1] - c2[1] * A3[0];
                r1[0] = A3[1] * A1[2] - A3[2] * A1[1];
                r1[1] = A3[2] * A1[0] - A3[0] * A1[2];
                r1[2] = A3[0] * A1[1] - A3[1] * A1[0];
                r2[0] = A1[1] * c2[2] - A1[2] * c2[1];
                r2[1] = A1[2] * c2[0] - A1[0] * c2[2];
                r2[2] = A1[0] * c2[1] - A1[1] * c2[0];
                const double det = A1[0] * r0[0] + A1[1] * r0[1] + A1[2] * r0[2];
                adet_c = fabs(det);
                const double rd = fast_rcp(adet_c);
                Gm[0] = rd * (r0[0] * r0[0] + r0[1] * r0[1] + r0[2] * r0[2]);
                Gm[1] = rd * (r0[0] * r1[0] + r0[1] * r1[1] + r0[2] * r1[2]);
                Gm[2] = rd * (r0[0] * r2[0] + r0[1] * r2[1] + r0[2] * r2[2]);
                Gm[3] = rd * (r1[0] * r1[0] + r1[1] * r1[1] + r1[2] * r1[2]);
                Gm[4] = rd * (r1[0] * r2[0] + r1[1] * r2[1] + r1[2] * r2[2]);
                Gm[5] = rd * (r2[0] * r2[0] + r2[1] * r2[1] + r2[2] * r2[2]);
            }
        }
        if (STASH && cur.comp == 0) {
            // c2, c4, c5, c7 (cell) and A1 (lane) are needed once per zeta plane only: park them in
            // shared memory and free 30 registers for the quadrature loop
            double *sg = s_stash + cw * WS::GS;
            if (t == 0) {
                double2 *d = reinterpret_cast<double2 *>(sg);
                d[0] = make_double2(c2[0], c2[1]);
                d[1] = make_double2(c2[2], c4[0]);
                d[2] = make_double2(c4[1], c4[2]);
                d[3] = make_double2(c5[0], c5[1]);
                d[4] = make_double2(c5[2], c7[0]);
                d[5] = make_double2(c7[1], c7[2]);
            }
            double2 *d = reinterpret_cast<double2 *>(sg + 12 + 4 * t);
            d[0] = make_double2(A1[0], A1[1]);
            sg[12 + 4 * t + 2] = A1[2];
            __syncwarp();
        }
        if constexpr (COEF) {
            // kappa to the quadrature points (B (x) B (x) B), once per cell and in place: x and y on
            // this lane's own layout-Z slots, then z on its own layout-Y slots, where the quadrature
            // loop reads them
            if (cur.comp == 0) {
                double *sk = s_kap + cw * US;
                double kz[N][N], kt[N][N];
#pragma unroll
                for (int x = 0; x < N; x++)
#pragma unroll
                    for (int yy = 0; yy < N; yy++) kz[x][yy] = valid ? sk[(x * N + yy) * N + t] : 0.0;
                apply_first<N, false>(P.B, kz, kt);
                apply_second<N, false>(P.B, kt, kz);
#pragma unroll
                for (int x = 0; x < N; x++)
#pragma unroll
                    for (int yy = 0; yy < N; yy++) sk[(x * N + yy) * N + t] = kz[x][yy];
                __syncwarp();
#pragma unroll
                for (int x = 0; x < N; x++)
#pragma unroll
                    for (int z = 0; z < N; z++) kt[x][z] = sk[(x * N + t) * N + z];
                apply_second<N, false>(P.B, kt, kz);
#pragma unroll
                for (int x = 0; x < N; x++)
#pragma unroll
                    for (int z = 0; z < N; z++) sk[(x * N + t) * N + z] = kz[x][z];
            }
        }
        if constexpr (ADV) {
            // b's second and third components, the same way on their own buffers (the first is in the
            // kappa buffer proper, done above; that block stays as it is, with the machine code of the
            // existing coefficient kernels)
            if (cur.comp == 0) {
                to_points_in_place<N>(P.B, s_kap + WS::UBUF + cw * US, valid, t);
                to_points_in_place<N>(P.B, s_kap + 2 * WS::UBUF + cw * US, valid, t);
            }
        }
        const int comp = cur.comp;
        const int *si = s_idx + (cbuf * CWS + cw) * US;
        {
            // ---- gathered values, layout Z (lane t == a_z)
            const double *su = s_u + cw * US;
            double u[N][N];
#pragma unroll
            for (int x = 0; x < N; x++)
#pragma unroll
                for (int yy = 0; yy < N; yy++) {
                    if (MATRIX) u[x][yy] = ((x * N + yy) * N + t == comp) ? 1.0 : 0.0;
                    else u[x][yy] = valid ? su[(x * N + yy) * N + t] : 0.0;
                }
            double tmp[N][N], U[N][N];
            double Vp[N][N];
            // ---- forward: interpolate to the quadrature points
            apply_first<N, false>(P.B, u, tmp);          // a_x -> q_x
            apply_second<N, false>(P.B, tmp, u);         // a_y -> q_y     u = w[qx][qy] @ a_z
            __syncwarp();
            tile.store_Z(u);
            __syncwarp();
            tile.load_Y(tmp);                            // tmp = w[qx][az] @ q_y
            apply_second<N, false>(P.B, tmp, U);         // a_z -> q_z     U[qx][qz] @ q_y
            __syncwarp();
            tile.store_Y(U);
            __syncwarp();
            tile.load_Z(tmp);                            // U[qx][qy] @ q_z
            apply_second<N, false>(P.Dt, tmp, u);        // d/d eta, still layout Z
            __syncwarp();
            tile.store_Z(u);
            __syncwarp();
            // d/d eta now sits in the tile in layout-Y order; each lane reads its
            // own slot (qx, qz) inside the quadrature loop and overwrites it
            // with the eta-flux, which the transpose path picks up from there

            // ---- quadrature points (layout Y), fused with the x/z derivative
            //      and its transpose so only U, Gy and Vp stay live
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = 0; j < N; j++) Vp[i][j] = 0.0;
            // single-buffered staging: the values / coordinates of `cur` were
            // consumed (and a __syncwarp passed) before this point
            stageB_coords(nxt);
            // The zeta loop is ROLLED (the fully unrolled body did not fit the
            // 32 KB instruction cache: ~15-20 % no-instruction stalls).  Register
            // arrays cannot be indexed by a run-time qz, so U and Vp are kept
            // rotated: column 0 is always the current zeta plane, and both are
            // rotated by one column at the end of each trip (N trips = identity).
            // DtR[qz][j] = Dt[qz][(j + qz) % N] is the matching rotation of the
            // derivative row.
#pragma unroll 1
            for (int qz = 0; qz < N; qz++) {
                stageB_part(nxt, ubuf ^ 1, qz);
                const double zeta = P.xq[qz];
                double dz[N];
#pragma unroll
                for (int j = 0; j < N; j++) dz[j] = P.DtR[qz * N + j];
                double ca[3], pb[3], qb[3];
                if (STASH) {
                    const double *sg = s_stash + cw * WS::GS;
                    const double2 *d = reinterpret_cast<const double2 *>(sg);
                    const double2 g0 = d[0], g1 = d[1], g2 = d[2], g3 = d[3], g4 = d[4], g5 = d[5];
                    const double2 a01 = *reinterpret_cast<const double2 *>(sg + 12 + 4 * t);
                    const double a2 = sg[12 + 4 * t + 2];
                    pb[0] = fma(g3.x, zeta, g0.x);     // c5 zeta + c2
                    pb[1] = fma(g3.y, zeta, g0.y);
                    pb[2] = fma(g4.x, zeta, g1.x);
                    qb[0] = fma(g4.y, zeta, g1.y);     // c7 zeta + c4
                    qb[1] = fma(g5.x, zeta, g2.x);
                    qb[2] = fma(g5.y, zeta, g2.y);
                    ca[0] = fma(A6[0], zeta, a01.x);   // dx/dxi
                    ca[1] = fma(A6[1], zeta, a01.y);
                    ca[2] = fma(A6[2], zeta, a2);
                } else if (!AFFINE) {
#pragma unroll
                    for (int a = 0; a < 3; a++) {
                        ca[a] = fma(A6[a], zeta, A1[a]);       // dx/dxi
                        pb[a] = fma(c5[a], zeta, c2[a]);
                        qb[a] = fma(c7[a], zeta, c4[a]);
                    }
                }
                const double wyz_a = wy_alpha * P.wq[qz];
                const double wyz_b = wy_beta * P.wq[qz];
                double *trow = tile.row_Y(qz);
#pragma unroll
                for (int qx = 0; qx < N; qx++) {
                    const double xi = P.xq[qx];
                    double cb[3], cc[3];
                    if (!AFFINE) {
#pragma unroll
                        for (int a = 0; a < 3; a++) {
                            cb[a] = fma(qb[a], xi, pb[a]);     // dx/deta
                            cc[a] = fma(A6[a], xi, A3[a]);     // dx/dzeta
                        }
                    }
                    double gx = 0.0, gz = 0.0;
#pragma unroll
                    for (int q = 0; q < N; q++) {
                        gx = fma(P.Dt[qx * N + q], U[q][0], gx);
                        gz = fma(dz[q], U[qx][q], gz);
                    }
                    const double gy = trow[qx * N * N];
                    if (AFFINE) {
                        const double wq3 = wyz_a * P.wq[qx];
                        const double fx = wq3 * (Gm[0] * gx + Gm[1] * gy + Gm[2] * gz);
                        const double fy = wq3 * (Gm[1] * gx + Gm[3] * gy + Gm[4] * gz);
                        const double fz = wq3 * (Gm[2] * gx + Gm[4] * gy + Gm[5] * gz);
                        trow[qx * N * N] = fy;
#pragma unroll
                        for (int q = 0; q < N; q++) {
                            Vp[q][0] = fma(P.Dt[qx * N + q], fx, Vp[q][0]);
                            Vp[qx][q] = fma(dz[q], fz, Vp[qx][q]);
                        }
                        if (MASS) Vp[qx][0] = fma(wyz_b * P.wq[qx] * adet_c, U[qx][0], Vp[qx][0]);
                        continue;
                    }
                    // cofactor rows: r0 = b x c, r1 = c x a, r2 = a x b
                    double r0[3], r1[3], r2[3];
                    r0[0] = cb[1] * cc[2] - cb[2] * cc[1];
                    r0[1] = cb[2] * cc[0] - cb[0] * cc[2];
                    r0[2] = cb[0] * cc[1] - cb[1] * cc[0];
                    r1[0] = cc[1] * ca[2] - cc[2] * ca[1];
                    r1[1] = cc[2] * ca[0] - cc[0] * ca[2];
                    r1[2] = cc[0] * ca[1] - cc[1] * ca[0];
                    r2[0] = ca[1] * cb[2] - ca[2] * cb[1];
                    r2[1] = ca[2] * cb[0] - ca[0] * cb[2];
                    r2[2] = ca[0] * cb[1] - ca[1] * cb[0];
                    const double det = ca[0] * r0[0] + ca[1] * r0[1] + ca[2] * r0[2];
                    const double adet = fabs(det);
                    const double s = stiff_weight<COEF && !ADV, NL>(wyz_a * P.wq[qx], s_kap + cw * US,
                                                                    (qx * N + t) * N + qz, U[qx][0], dcoef) *
                                     fast_rcp(adet);
                    double h[3];
                    if constexpr (NL == 2) {
                        // u and its reference gradient at (qx, qy = t, qz) from the buffer's quadrature
                        // values; the z row is dz (rotated), the buffer is not
                        const double *sk = s_kap + cw * US;
                        const int row = (qx * N + t) * N;
                        const double uq = sk[row + qz];
                        double ux = 0.0, uy = 0.0, uz = 0.0;
#pragma unroll
                        for (int q = 0; q < N; q++) {
                            const int zq = (q + qz < N) ? q + qz : q + qz - N;
                            ux = fma(P.Dt[qx * N + q], sk[(q * N + t) * N + qz], ux);
                            uy = fma(dyr[q], sk[(qx * N + q) * N + qz], uy);
                            uz = fma(dz[q], sk[row + zq], uz);
                        }
                        const double Dq = fma(fma(dcoef[2], uq, dcoef[1]), uq, dcoef[0]);
                        const double dpw = fma(2.0 * dcoef[2], uq, dcoef[1]) * U[qx][0];   // D'(u_q) w_q
                        const double g0 = fma(dpw, ux, Dq * gx);
                        const double g1 = fma(dpw, uy, Dq * gy);
                        const double g2 = fma(dpw, uz, Dq * gz);
#pragma unroll
                        for (int a = 0; a < 3; a++) h[a] = r0[a] * g0 + r1[a] * g1 + r2[a] * g2;
                    } else {
#pragma unroll
                        for (int a = 0; a < 3; a++) h[a] = r0[a] * gx + r1[a] * gy + r2[a] * gz;
                    }
                    const double fx = s * (r0[0] * h[0] + r0[1] * h[1] + r0[2] * h[2]);
                    const double fy = s * (r1[0] * h[0] + r1[1] * h[1] + r1[2] * h[2]);
                    const double fz = s * (r2[0] * h[0] + r2[1] * h[1] + r2[2] * h[2]);
                    trow[qx * N * N] = fy;
#pragma unroll
                    for (int q = 0; q < N; q++) {
                        Vp[q][0] = fma(P.Dt[qx * N + q], fx, Vp[q][0]);
                        Vp[qx][q] = fma(dz[q], fz, Vp[qx][q]);
                    }
                    if constexpr (ADV) {
                        // w |det J| b . grad u = w sign(det J) (b . h), whatever beta is
                        const double *sb = s_kap + cw * US + (qx * N + t) * N + qz;
                        const double bh = sb[0] * h[0] + sb[WS::UBUF] * h[1] + sb[2 * WS::UBUF] * h[2];
                        const double w = P.wq[lane_active ? t : 0] * P.wq[qz] * P.wq[qx];
                        Vp[qx][0] = fma(copysign(w, det), bh, Vp[qx][0]);
                    }
                    if (MASS) Vp[qx][0] = fma(wyz_b * P.wq[qx] * adet, U[qx][0], Vp[qx][0]);
                }
                // rotate: column j <- column j+1
#pragma unroll
                for (int x = 0; x < N; x++) {
                    const double u0 = U[x][0], v0 = Vp[x][0];
#pragma unroll
                    for (int j = 0; j < N - 1; j++) {
                        U[x][j] = U[x][j + 1];
                        Vp[x][j] = Vp[x][j + 1];
                    }
                    U[x][N - 1] = u0;
                    Vp[x][N - 1] = v0;
                }
            }

            __syncwarp();            // all lanes are done reading the staged rows of `nxt`
            stageB_kappa(nxt);       // (and kappa's quadrature values of `cur`)
            stageA(nn);
            cp_async_commit();

            // ---- backward (the tile holds Fy[qx][qz] @ q_y)
            __syncwarp();
            tile.load_Z(tmp);                            // Fy[qx][qy] @ q_z
            apply_second<N, true>(P.Dt, tmp, u);         // Dt^T along eta
            __syncwarp();
            tile.store_Z(u);
            __syncwarp();
            tile.load_Y(tmp);
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = 0; j < N; j++) Vp[i][j] += tmp[i][j];
            apply_second<N, true>(P.B, Vp, tmp);         // q_z -> a_z     W[qx][az] @ q_y
            __syncwarp();
            tile.store_Y(tmp);
            __syncwarp();
            tile.load_Z(u);                              // W[qx][qy] @ a_z
            apply_first<N, true>(P.B, u, tmp);           // q_x -> a_x
            apply_second<N, true>(P.B, tmp, u);          // q_y -> a_y     R[ax][ay] @ a_z

            // ---- scatter-add, layout Z
            if (MATRIX && P.vals == nullptr) {
                // diagonal of the bilinear form: only the entry i == j of column j
                if (valid) {
#pragma unroll
                    for (int x = 0; x < N; x++)
#pragma unroll
                        for (int yy = 0; yy < N; yy++)
                            if ((x * N + yy) * N + t == comp) atomicAdd(P.y + si[comp], u[x][yy]);
                }
            } else if (MATRIX) {
                // MatSetValuesLocal(ADD_VALUES): column = trial dof `comp`, rows = this
                // lane's test dofs; negative (BC-masked) indices are dropped
                int gcol = valid ? si[comp] : -1;
                if (gcol >= 0 && P.col_lg) gcol = __ldg(P.col_lg + gcol);
                const unsigned short *rk = nullptr;
                if (P.rank_tab && valid) {
                    const int lay = cur.layer;
                    const int v = P.nlay_total < 3 ? lay : (lay == 0 ? 0 : (lay == P.nlay_total - 1 ? 2 : 1));
                    rk = P.rank_tab + (((long long)cur.col * P.nvar + v) * ND + comp) * ND;
                }
                if (gcol >= 0) {
#pragma unroll
                    for (int x = 0; x < N; x++)
#pragma unroll
                        for (int yy = 0; yy < N; yy++) {
                            int grow = si[(x * N + yy) * N + t];
                            if (P.row_lg) grow = __ldg(P.row_lg + grow);
                            if (grow < 0) continue;
                            long long lo = __ldg(P.rowptr + grow);
                            if (rk) {
                                lo += __ldg(rk + (x * N + yy) * N + t);
                            } else {
                                long long hi = __ldg(P.rowptr + grow + 1);
                                while (hi - lo > 1) {
                                    long long mid = (lo + hi) >> 1;
                                    if (__ldg(P.colidx + mid) <= gcol) lo = mid; else hi = mid;
                                }
                            }
                            if (ATOMIC) atomicAdd(P.vals + lo, u[x][yy]);
                            else P.vals[lo] += u[x][yy];
                        }
                }
            } else if (valid) {
                const int *smc = row_of(cur);
#pragma unroll
                for (int x = 0; x < N; x++)
#pragma unroll
                    for (int yy = 0; yy < N; yy++) {
                        const int loc = (x * N + yy) * N + t;
                        const int g = SLIM ? smc[loc] + s_off0[loc] * cur.layer : si[loc];
                        double *dst = P.y + (long long)g * P.cdim + comp;
                        if (ATOMIC) atomicAdd(dst, u[x][yy]);
                        else *dst += u[x][yy];
                    }
            }
        }
        cur = nxt;
        nxt = nn;
        ubuf ^= 1;
    }
    cp_async_wait<0>();
