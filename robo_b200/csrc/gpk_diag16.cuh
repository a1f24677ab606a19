// gpk_diag16.cuh — diagonal block of the blocked Cholesky (gpk_potrf_diag_dmma_kernel):
//   L_kk = chol(A_kk) and inv(L_kk) of one 128 x 128 diagonal block, one CTA of 256 threads.
// It writes L_kk (lower) back to K, the rows of inv(L_kk) up to their diagonal 16-block to P, sum log diag(L_kk) to
// logdet_part[kb], and flags a non-positive pivot in *status (1 + global pivot index), which is what
// scipy.linalg.cholesky reports as LinAlgError.  The zeros right of the 16 x 16 sub-blocks and Q = P^T are written off
// the critical chain by gpk_diag_prezero_kernel and gpk_diag_qfill_kernel.
//
// A column-by-column kernel pays one block-wide barrier per pivot (128 intervals of ~950 cycles; 3/4 of its issued
// instructions are not arithmetic).  Here the block is processed in 8 panels of 16 columns with two barriers per
// panel:
//   S  "factor + solve": warp 0 eliminates the published 16 x 16 diagonal sub-block in registers (lane & 15 = row)
//      in square-root-free form (L' D L'^T): the serial chain per pivot is mul -> fma -> reciprocal, the raw column goes
//      through a warp-private shared vector before its pivot's reciprocal is known, and the 16 rsqrt that give the factor
//      L = L' D^1/2 run in parallel after the last pivot.  Every column of L' is published through shared memory and
//      signalled with a named barrier (bar.arrive, one id per pivot); warps 1..4 wait on that id (bar.sync) and apply
//      it to one unit-lower forward substitution per thread -- the 128 - 16(p+1) rows of the panel below the
//      sub-block (L_ik = A_ik L_kk^-T) and the 16(p+1) columns of the inverse's row block (X_k. = L_kk^-1 Xtilde_k.),
//      always 128 vectors -- then scale by D^-1/2.  (Alternatives with more cycles per panel: all 8 warps
//      factorising redundantly with the substitutions in the same loop, DP-issue bound; one warp carrying the sqrt
//      chain AND 32 substitutions.)
//   U  "update + publish": rank-16 update of the trailing matrix and of the inverse's residual (kept in shared
//      memory) on the fp64 tensor pipe (see gpk_potrf_diag_dmma_kernel); then the next panel's sub-block and rows
//      are published.
// Every element receives the pivots in increasing order, as in the column-by-column algorithm, so the factor agrees
// with an unblocked Cholesky to rounding.  The panel loop is rolled: the kernel runs once per launch on one SM, i.e.
// out of a cold instruction cache, and a fully unrolled blocked kernel (38k instructions) was fetch-bound.
#pragma once

constexpr int D3PS = 17;      // row stride (doubles) of the panel staging array: odd -> thread-per-row and
                              // 16-rows-per-half-warp 64-bit loads are bank-conflict-free
struct __align__(16) DiagSmem {
    static constexpr int XS = 129;    // row stride of the inverse's residual: odd -> conflict-free B fragments out of it
    double xs[128 * XS];          // Xtilde / finished rows of inv(L_kk), row-major
    double pan[2][128 * D3PS];    // pan[i][k]: column 16 kb + k of the current panel, row i (raw, then solved)
    double din[2][16 * 17];       // the 16 x 16 diagonal sub-block as published
    double colp[16][16];          // colp[j][c] = L'_D[c][j]: column j as published by the factorising warp
    double rsp[16];               // 1 / L_D[j][j]
    double ub[2][16];             // raw column of the sub-block about to be eliminated (factorising warp only)
    double ldd[2][16 * 17];       // the factorised sub-block (lower) by panel parity, for the coalesced store
};
constexpr int DIAG_SMEM = (int)sizeof(DiagSmem);

__device__ __forceinline__ double d3_shfl(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }

// 1/sqrt(p): hardware seed (MUFU.RSQ64H, ~22 bits) + two Newton steps -> ~1 ulp; 9 instructions, no branches
// (the library rsqrt() carries special-case paths this chain does not need: p is a checked positive finite pivot).
__device__ __forceinline__ double d3_rsqrt(double p)
{
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(p));
    double t = p * y, e = fma(-t, y, 1.0);
    y = fma(0.5 * y, e, y);
    t = p * y;
    e = fma(-t, y, 1.0);
    return fma(0.5 * y, e, y);
}

// 1/p: hardware seed (MUFU.RCP64H) + two Newton steps; 5 instructions on the pivot chain
__device__ __forceinline__ double d3_rcp(double p)
{
    double y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(p));
    y = fma(y, fma(-p, y, 1.0), y);
    return fma(y, fma(-p, y, 1.0), y);
}

// named barriers between the factorising warp (arrive) and the four substitution warps (sync): 32 + 128 threads
__device__ __forceinline__ void d3_bar_arrive(int id) { asm volatile("bar.arrive %0, 160;" :: "r"(id) : "memory"); }
__device__ __forceinline__ void d3_bar_sync(int id) { asm volatile("bar.sync %0, 160;" :: "r"(id) : "memory"); }

// ---- coalesced 128-bit stores of what panel kp finished: the factorised sub-block, the solved panel rows below it
// (final L values) and the row block of the inverse up to its diagonal (what lies right of it is zeroed off the
// chain by gpk_diag_prezero_kernel).  Executed by threads t = 0..nth-1.  Measured on a B200: issued at the start of U
// by all threads they cost the issuing warps ~1.4k cycles per panel; issued by the three warps that idle during phase
// S of the NEXT panel the kernel went from 69.2k to 64.3k cycles per block (a run with the stores disabled takes the
// same time: they are hidden).
__device__ __forceinline__ void d3_store_panel(const DiagSmem& sm, const int kp, const int t, const int nth,
                                               double* __restrict__ Kt, const long ld, double* __restrict__ Pt, const long ldp)
{
    const double* pan = sm.pan[kp & 1];
    const double* ldd = sm.ldd[kp & 1];
    for (int it = t; it < 128; it += nth) {                       // sub-block: 16 rows x 8 pairs
        const int r16 = it >> 3, cp = (it & 7) * 2;
        *reinterpret_cast<double2*>(Kt + (long)(16 * kp + r16) * ld + 16 * kp + cp) =
            make_double2(ldd[r16 * 17 + cp], ldd[r16 * 17 + cp + 1]);
    }
    const int nitem = (128 - 16 * (kp + 1)) * 8;                  // panel rows: 8 pairs per row
    for (int it = t; it < nitem; it += nth) {
        const int row = 16 * (kp + 1) + (it >> 3), cp = (it & 7) * 2;
        *reinterpret_cast<double2*>(Kt + (long)row * ld + 16 * kp + cp) =
            make_double2(pan[row * D3PS + cp], pan[row * D3PS + cp + 1]);
    }
    const int npair = 8 * (kp + 1);                               // inverse rows 16 kp .. +15, columns 0 .. 16 (kp + 1)
    for (int it = t; it < 16 * npair; it += nth) {
        const int r16 = it / npair, c = (it - r16 * npair) * 2;
        const double* xr = sm.xs + (16 * kp + r16) * DiagSmem::XS;
        *reinterpret_cast<double2*>(Pt + (long)(16 * kp + r16) * ldp + c) = make_double2(xr[c], xr[c + 1]);
    }
}

// ---- S: warp 0 factorises the published 16 x 16 sub-block, warps 1..4 run the 128 forward substitutions of panel
// kbp
__device__ __forceinline__ void d3_phase_s(DiagSmem& sm, const int kbp, const int kb, const int tid, int* s_bad, double& lsum,
                                           long long* __restrict__ prof, const bool fine)
{
    const int lane = tid & 31, r = lane & 15;
    double* pan = sm.pan[kbp & 1];
    const double* din = sm.din[kbp & 1];
    const int u = tid - 32;                                  // vector of threads 32..159
    const int nrows = 128 - 16 * (kbp + 1);                  // panel rows below the sub-block
    const bool is_vec = u >= 0 && u < 128;
    const bool is_pan = is_vec && u < nrows;
    const int irow = 16 * (kbp + 1) + u;                     // panel row (is_pan)
    const int ccol = u - nrows;                              // column of the inverse's row block (is_x)
            if (fine) prof[34] = clock64();
    if (prof != nullptr && kbp == 3 && tid == 0) prof[46] = clock64();
    if (tid < 32) {
        // -- the factorising warp.  Square-root-free elimination (L' D L'^T with unit-lower L'): the serial chain
        // per pivot is  mul -> fma -> reciprocal  (the raw column is broadcast before its pivot's reciprocal is
        // known), and the 16 rsqrt that turn L' D^1/2 into the Cholesky factor run in parallel at the end.
        double d[16];
#pragma unroll
        for (int c = 0; c < 16; ++c) d[c] = (c <= r) ? din[r * 17 + c] : 0.0;
        double p = d3_shfl(d[0], 0);
        bool ok = (p > 0.0) && !isinf(p);
        int bad = ok ? 0 : kb * 128 + 16 * kbp + 1;  // first failing pivot (1-based), in a register: no branches
        double myp = p;                              // lane r keeps pivot r
        const double i0 = d3_rcp(p);
        double inv = ok ? i0 : 1.0;
        double x = d3_shfl(d[0], 1), y = d3_shfl(d[1], 1);   // row j+1: its entry in column j and its diagonal
        if (lane < 16) sm.ub[0][r] = d[0];
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 15; ++j) {
            // column j of the unit-lower factor, published for the substitutions.  The signal comes FIRST: the
            // barrier instruction fences the scheduler, and the two independent halves of this pivot -- the
            // reciprocal of the next pivot (the serial chain) and the update with column j -- must be free to
            // interleave on this one in-order warp (with the chain ahead of the signal they ran back to back:
            // 200 cycles per pivot instead of ~100).
            const double t = d[j] * inv;
            if (lane < 16) sm.colp[j][r] = t;
            if (j < 14) d3_bar_arrive(1 + j);
            const double t1 = x * inv;
            const double pn = fma(-t1, x, y);
            ok = (pn > 0.0) && !isinf(pn);
            bad = (bad == 0 && !ok) ? kb * 128 + 16 * kbp + j + 2 : bad;
            const double rn = d3_rcp(pn);            // unconditional: stays in the straight-line block
            const double inv_next = ok ? rn : 1.0;
            myp = (r == j + 1) ? pn : myp;
            if (j == 14) {                           // all pivots known: reciprocal square roots, then the last signal
                const double rsq = d3_rsqrt(myp);
                if (lane < 16) sm.rsp[r] = rsq;
                d3_bar_arrive(15);
            }
            // raw entries (c, j) come back as broadcast loads of the vector stored one pivot earlier (they do not
            // wait for the reciprocal; 2 x 15 shuffles per pivot cost a single warp ~4 issue cycles each)
            const double* ubj = sm.ub[j & 1];
#pragma unroll
            for (int c = j + 1; c < 16; ++c) d[c] = fma(-t, ubj[c], d[c]);
            if (lane < 16) sm.ub[(j + 1) & 1][r] = d[j + 1];
            __syncwarp();
            if (j < 14) {
                x = d3_shfl(d[j + 1], j + 2);
                y = d3_shfl(d[j + 2], j + 2);
            }
            inv = inv_next;
            if (prof != nullptr && kbp == 3 && tid == 0 && (j & 3) == 3) prof[42 + (j >> 2)] = clock64();
        }
        if (prof != nullptr && kbp == 3 && tid == 0) prof[45] = clock64();
        __syncwarp();
        if (tid < 16) {                               // the Cholesky factor of the sub-block, for the store in U
#pragma unroll
            for (int c = 0; c < 16; ++c) {
                const double sc = (c == r) ? myp : d[c];          // raw column entry (or the pivot) * 1/sqrt(pivot c)
                sm.ldd[kbp & 1][r * 17 + c] = (c <= r) ? sc * sm.rsp[c] : 0.0;
            }
            lsum += 0.5 * log(myp);
            if (tid == 0 && bad != 0 && *s_bad == 0) *s_bad = bad;
        }
    } else if (is_vec) {
        // -- one forward substitution per thread against the unit-lower factor, column by column as published
        double v[16];
        {
            const double* src = is_pan ? pan + irow * D3PS : sm.xs + (16 * kbp) * DiagSmem::XS + ccol;
            const int step = is_pan ? 1 : DiagSmem::XS;
#pragma unroll
            for (int k = 0; k < 16; ++k) v[k] = src[k * step];
        }
#pragma unroll
        for (int j = 0; j < 15; ++j) {
            d3_bar_sync(1 + j);
            const double wj = v[j];
            const double* col = sm.colp[j];
            if ((j + 1) & 1) v[j + 1] = fma(-col[j + 1], wj, v[j + 1]);
#pragma unroll
            for (int c = (j + 2) & ~1; c < 16; c += 2) {
                const double2 l2 = *reinterpret_cast<const double2*>(col + c);
                v[c] = fma(-l2.x, wj, v[c]);
                v[c + 1] = fma(-l2.y, wj, v[c + 1]);
            }
            if (fine && (j & 3) == 3) prof[35 + (j >> 2)] = clock64();
        }
        if (fine) prof[38] = clock64();
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] *= sm.rsp[k];          // D^-1/2
        if (is_pan) {                                 // finished panel row: operand of U
#pragma unroll
            for (int k = 0; k < 16; ++k) pan[irow * D3PS + k] = v[k];
        } else {                                      // finished column of the inverse's row block
#pragma unroll
            for (int k = 0; k < 16; ++k) sm.xs[(16 * kbp + k) * DiagSmem::XS + ccol] = v[k];
        }
    }
}

// ---------------------------------------------------------------------------------------
// Phase U on the fp64 tensor pipe.  With DFMA on 8 x 8 cyclic register tiles the rank-16 update needs one 64-bit
// shared load per 2.3 FMAs, and LDS.64 occupies the LSU for 2 cycles per warp whatever the broadcast degree: such a
// U phase is LSU-bound at ~2.4x the DP-pipe time.  Here the trailing matrix lives in m8n8k4 accumulator fragments: the block is cut into 16 x 16 "tiles" of 8 rows x
// 8 columns, tile t = rows 16 (t/2) + 2 (t%2) + {0,4,8,12,1,5,9,13} (the interleave makes the 34-word row stride of
// the panel array bank-conflict-free for fragment loads AND for the thread-per-row substitutions of phase S);
// warp w owns tile rows w and 15 - w (18 tiles, all tiles (I, J) with J/2 <= I/2, so that the A fragment of a tile row is
// loaded once per k-chunk and reused along the row).  Per panel and warp: <= 8 + 72 fragment loads for <= 72 DMMA
// (DFMA register tiles: 190 loads), and the inverse's residual is updated in shared memory through the same fragments.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ int d4_row(int t, int idx) { return 16 * (t >> 1) + 2 * (t & 1) + 4 * (idx & 3) + (idx >> 2); }

// write the elements of the tiles in tile columns 2 kp, 2 kp + 1 (the next panel) to din / pan
template <int NS>
__device__ __forceinline__ void d4_publish_row(const double (&c)[NS][2], const int I, const int kp, DiagSmem& sm, const int g,
                                               const int q)
{
    if ((I >> 1) < kp) return;
    const int row = d4_row(I, g);
    double* pan = sm.pan[kp & 1];
    double* din = sm.din[kp & 1];
#pragma unroll
    for (int J = 0; J < NS; ++J) {
        if ((J >> 1) != kp) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int coff = d4_row(J, 2 * q + e) - 16 * kp;
            if ((I >> 1) == kp) din[(row - 16 * kp) * 17 + coff] = c[J][e];
            else pan[row * D3PS + coff] = c[J][e];
        }
    }
}

// rank-16 update of one owned tile row: trailing-matrix tiles (registers) and the inverse's residual (shared memory)
template <int NS>
__device__ __forceinline__ void d4_update_row(double (&c)[NS][2], const int I, const int kbp, DiagSmem& sm, const int g,
                                              const int q)
{
    const int c0 = 2 * (kbp + 1);                    // first tile row / column behind the panel
    if (I < c0) return;
    const double* pan = sm.pan[kbp & 1];
    const int row = d4_row(I, g);
    double af[4];
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) af[ch] = -pan[row * D3PS + 4 * ch + q];
    const int jmax = 2 * (I >> 1) + 1;
    // tiles come in pairs (c0 is even, jmax odd): two independent accumulator chains per pair keep the DMMA pipe fed
#pragma unroll
    for (int J = 0; J < NS; J += 2) {
        if (J < c0 || J > jmax) continue;
        const double* p0 = pan + d4_row(J, g) * D3PS + q;
        const double* p1 = pan + d4_row(J + 1, g) * D3PS + q;
        double b0[4], b1[4];
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) { b0[ch] = p0[4 * ch]; b1[ch] = p1[4 * ch]; }
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
            dmma884(c[J][0], c[J][1], af[ch], b0[ch]);
            dmma884(c[J + 1][0], c[J + 1][1], af[ch], b1[ch]);
        }
    }
    // Xtilde[I-rows, 0 : 16 (kbp+1)) -= L_panel[I-rows, :] X[panel rows, :]
    double* xrow = sm.xs + row * DiagSmem::XS;
    const double* xb = sm.xs + (16 * kbp + q) * DiagSmem::XS;
#pragma unroll 1
    for (int Jc = 0; Jc < c0; Jc += 2) {                 // c0 is even: two tiles (independent chains) per iteration
        int col[2][2], colb[2];
        double x[2][2], bx[2][4];
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            col[t][0] = d4_row(Jc + t, 2 * q);
            col[t][1] = d4_row(Jc + t, 2 * q + 1);
            colb[t] = d4_row(Jc + t, g);
            x[t][0] = xrow[col[t][0]];
            x[t][1] = xrow[col[t][1]];
#pragma unroll
            for (int ch = 0; ch < 4; ++ch) bx[t][ch] = xb[4 * ch * DiagSmem::XS + colb[t]];
        }
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
            dmma884(x[0][0], x[0][1], af[ch], bx[0][ch]);
            dmma884(x[1][0], x[1][1], af[ch], bx[1][ch]);
        }
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            xrow[col[t][0]] = x[t][0];
            xrow[col[t][1]] = x[t][1];
        }
    }
}

__global__ void __launch_bounds__(256, 1)
gpk_potrf_diag_dmma_kernel(double* __restrict__ K, long ld, int kb,
                           double* __restrict__ P, double* __restrict__ Q, long ldp,
                           int* __restrict__ status, double* __restrict__ logdet_part,
                           long long* __restrict__ prof)
{
    extern __shared__ __align__(16) unsigned char d3_raw[];
    DiagSmem& sm = *reinterpret_cast<DiagSmem*>(d3_raw);
    constexpr int XS = DiagSmem::XS;
    __shared__ int s_bad;

    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int g = lane >> 2, q = lane & 3;
    cudaGridDependencySynchronize();      // programmatic dependent launch (see gpk_gemm_nt_kernel)
    if (*status != 0) return;
    if (tid == 0) s_bad = 0;
    const bool stamp = prof != nullptr && tid == 159;
    const bool nostore = prof != nullptr && prof[63] != 0;  // timing experiment: results are not written
    if (stamp) prof[0] = clock64();

    double* Kt = K + (long)kb * 128 * ld + (long)kb * 128;
    double* Pt = P + (long)kb * 128 * ldp + (long)kb * 128;
    // coalesced read of the lower triangle into shared memory, then every warp picks up its fragments
#pragma unroll 16
    for (int e = tid; e < 128 * 128; e += 256) {          // 16 independent loads in flight per thread
        const int i = e >> 7, c = e & 127;
        sm.xs[i * XS + c] = (c <= i) ? Kt[(long)i * ld + c] : 0.0;
    }
    __syncthreads();
    const int Ia = w, Ib = 15 - w;
    double ca[8][2], cb[16][2];
#pragma unroll
    for (int J = 0; J < 8; ++J)
#pragma unroll
        for (int e = 0; e < 2; ++e)
            ca[J][e] = (J <= 2 * (Ia >> 1) + 1) ? sm.xs[d4_row(Ia, g) * XS + d4_row(J, 2 * q + e)] : 0.0;
#pragma unroll
    for (int J = 0; J < 16; ++J)
#pragma unroll
        for (int e = 0; e < 2; ++e)
            cb[J][e] = (J <= 2 * (Ib >> 1) + 1) ? sm.xs[d4_row(Ib, g) * XS + d4_row(J, 2 * q + e)] : 0.0;
    __syncthreads();
    for (int e = tid; e < 128 * XS; e += 256) {            // Xtilde = I
        const int i = e / XS, c = e - i * XS;
        sm.xs[e] = (i == c) ? 1.0 : 0.0;
    }
    d4_publish_row(ca, Ia, 0, sm, g, q);
    d4_publish_row(cb, Ib, 0, sm, g, q);
    double lsum = 0.0;
    __syncthreads();
    if (stamp) prof[1] = clock64();

#pragma unroll 1
    for (int kbp = 0; kbp < 8; ++kbp) {
        const bool fine = stamp && kbp == 3;
        d3_phase_s(sm, kbp, kb, tid, &s_bad, lsum, prof, fine);
        if (tid >= 160 && kbp > 0 && !nostore) d3_store_panel(sm, kbp - 1, tid - 160, 96, Kt, ld, Pt, ldp);   // idle warps 5..7
        if (fine) prof[39] = clock64();
        __syncthreads();
        if (stamp) prof[2 + 2 * kbp] = clock64();
        // ---- U: rank-16 updates on the tensor pipe, publish the next panel
        if (kbp == 7) break;
        if (fine) prof[40] = clock64();
        d4_update_row(ca, Ia, kbp, sm, g, q);
        d4_update_row(cb, Ib, kbp, sm, g, q);
        d4_publish_row(ca, Ia, kbp + 1, sm, g, q);
        d4_publish_row(cb, Ib, kbp + 1, sm, g, q);
        if (fine) prof[41] = clock64();
        __syncthreads();
        if (stamp) prof[3 + 2 * kbp] = clock64();
    }

    if (!nostore) d3_store_panel(sm, 7, tid, 256, Kt, ld, Pt, ldp);
    if (tid < 32) {
        double s = (tid < 16) ? lsum : 0.0;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (tid == 0) {
            logdet_part[kb] = s;
            if (s_bad != 0) atomicCAS(status, 0, s_bad);
        }
    }
    if (stamp) prof[33] = clock64();
}

// Off-chain helpers of the blocked kernel: zero what lies right of the 16 x 16 sub-blocks in every diagonal tile of
// K (the covariance builder leaves the symmetric values there; later GEMMs read the tile as a lower-triangular
// operand), likewise in P (the kernel stores the inverse's rows only up to their diagonal 16-block); Q's diagonal tiles =
// transposed diagonal tiles of P.  One CTA per diagonal tile.
__global__ void __launch_bounds__(256) gpk_diag_prezero_kernel(double* __restrict__ K, long ld, double* __restrict__ P,
                                                               long ldp)
{
    double* Kt = K + (long)blockIdx.x * 128 * ld + (long)blockIdx.x * 128;
    double* Pt = P + (long)blockIdx.x * 128 * ldp + (long)blockIdx.x * 128;
    for (int e = threadIdx.x; e < 128 * 128; e += 256) {
        const int i = e >> 7, c = e & 127;
        if ((c >> 4) > (i >> 4)) {
            Kt[(long)i * ld + c] = 0.0;
            Pt[(long)i * ldp + c] = 0.0;
        }
    }
}

__global__ void __launch_bounds__(256) gpk_diag_qfill_kernel(const double* __restrict__ P, double* __restrict__ Q,
                                                             long ldp, const int* __restrict__ status)
{
    __shared__ double t[32][33];
    if (*status != 0) return;
    const double* Pt = P + (long)blockIdx.x * 128 * ldp + (long)blockIdx.x * 128;
    double* Qt = Q + (long)blockIdx.x * 128 * ldp + (long)blockIdx.x * 128;
    const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;          // 32 x 8
    for (int bi = 0; bi < 4; ++bi)
        for (int bj = 0; bj < 4; ++bj) {
            for (int q = 0; q < 4; ++q) t[ly + 8 * q][lx] = Pt[(long)(32 * bi + ly + 8 * q) * ldp + 32 * bj + lx];
            __syncthreads();
            for (int q = 0; q < 4; ++q) Qt[(long)(32 * bj + ly + 8 * q) * ldp + 32 * bi + lx] = t[lx][ly + 8 * q];
            __syncthreads();
        }
}
