// gpk_hyper_blocked.cuh — the GP hyper-parameter log-posterior of many theta at large N (gpk_hyper_lnpost_blocked,
// gpk_sample_hypers_blocked, gpk_optimize_hypers_blocked): one dense fp64 matrix per theta in HBM, factored by the fit's
// blocked Cholesky with every GEMM launch covering all B matrices of a chunk, so B factorisations cost the nb serial
// steps of one.  gpk_hy_eval (gpk_hyper.cuh) keeps its factor in one SM's shared memory and stops at GPK_HYPER_MAX_N;
// this path runs to GPK_HYPER_BLOCKED_MAX_N.
//
// Layout of a chunk: the B matrices back to back, matrix b = rows [b R, (b + 1) R) of one row-major array with
// ld = NP = 128 nb (nb = ceil(n / 128)) and R = NP + 128 rows, as the fit's Kbuf: K_b in the lower tiles of block rows
// 0 .. nb-1, padding rows and columns (index >= n) the identity; block row nb carries the residual r = y - mean as its
// first row (the other rows zero), so the factorisation leaves z = L^-1 r there, as gpk_fit_begin does.  One 2-D tensor
// map covers the stacked matrices, so a GEMM job addresses matrix b by offsetting its rows by b R.  P: one 128-row
// strip per matrix (rows [128 b, 128 (b + 1)), ld NP) that receives inv(L_kk) of the current step at columns k 128.
//
// Per chunk of B theta (every per-matrix step independent of B and of the other matrices):
//   prep:    one CTA per theta, gpk_hy_eval's parameter step: the |theta_j| > 20 rule, the prior gpk_hy_prior (the
//            same routine), amp = exp(0.0 + the amplitude slots in order), diag_add = fl(sqrt(fl(yerr^2 + tiny)))^2,
//            the factor (gpk_factor_build) and inv_metric_t = 1 / exp(theta[term_param[t]])
//   build:   one CTA per lower tile, K_ij = amp prod_g gpk_radial(family, sum_{t in g} (x_i - x_j)^2 inv_metric_t)
//            [* gpk_factor_value(z_i, z_j)], + diag_add on the diagonal: gpk_hy_eval's element expression
//   step k:  diag   the fit's gpk_potrf_diag_dmma_kernel once per matrix (its own status word and log-det slots)
//            panel  one gpk_gemm_ws_kernel launch, one job per block row i > k of every matrix (the residual block
//                   included): L_ik = A_ik inv(L_kk)^T, as the fit's panel solve
//            update one gpk_gemm_ws_kernel launch, one job per tile (i, j), k < j <= i (j < nb), of every matrix:
//                   A_ij -= L_ik L_jk^T, as the fit's trailing update
//   finish:  one CTA per matrix: z^T z as gpk_hy_eval's fixed-order tree over 256 threads, log det = 2 sum_k (the diag
//            kernel's block sums in k order), ll = -1/2 z^T z - 1/2 log det - n/2 log(2 pi), -inf when not finite, out of
//            range or not positive definite; the sampler's log-posterior gpk_hy_post and the optimiser's objective
//            gpk_ho_objective of (ll, lp)
// A matrix that fails keeps going through the GEMMs (NaN at worst): the finish kernel reads its status.  The jobs of a
// matrix depend on n only and a tile's arithmetic on its job only, so the bits of a theta's ll and lp depend on theta,
// the data and n, never on B, its chunk, its position or the other theta.
//
// Sampler (gpk_sample_hypers_blocked): gpk_sample_hypers's run with the log-posteriors of this file: the initial walkers
// scored once, then per half-step gpk_hb_propose_kernel writes the active half's proposals (gpk_hy_step_kernel's
// Philox counters, tags and rounding), one batched log-posterior, and gpk_hb_accept_kernel applies
// gpk_stretch_accept.  Optimiser (gpk_optimize_hypers_blocked): per round gpk_hb_stencil_kernel writes the trial point
// and its dim forward-difference neighbours (gpk_ho_round_kernel's rule), one batched objective, and
// gpk_hb_update_ho_kernel runs gpk_ho_update (gpk_hyperopt.cuh) in one warp and raises the chunk's skip word once the
// status is final: every later prep, diag and GEMM CTA of the host's chunk of rounds then returns at once.
#pragma once
#include "gpk_gemm.cuh"
#include "gpk_hyperopt.cuh"

#define HB_T 128                // rows per tile: the fit's block (BM)

// per-theta parameters of a chunk (global memory), written by gpk_hb_prep_kernel
struct HBPar {
    double amp, dg, lp;
    int bad;                    // 0: running; 1: |theta_j| > 20; 2: skipped (the chunk's skip word was set)
    KFactor kf;
    double im[GPK_MAX_TERMS];
};

__host__ __device__ inline int gpk_hb_nb(int n) { return (n + HB_T - 1) / HB_T; }

// doubles of one matrix for n training points
__host__ __device__ inline long gpk_hb_matrix_doubles(int n)
{
    const long nb = gpk_hb_nb(n);
    return (nb + 1) * HB_T * nb * HB_T;
}

// bytes one theta of a chunk needs: its matrix, its P strip, its HBPar, its block log-sums, its status word
__host__ __device__ inline long gpk_hb_theta_bytes(int n)
{
    return gpk_hb_matrix_doubles(n) * 8 + (long)HB_T * gpk_hb_nb(n) * HB_T * 8 + (long)((sizeof(HBPar) + 7) / 8) * 8 +
           (long)gpk_hb_nb(n) * 8 + 8;
}

// the parameter step of gpk_hy_eval for theta row `b` of T (D entries each); st[b]: the diag kernel's status word, 0
// while the matrix is worth factoring.  skip: the chunk's skip word (non-zero: mark the theta skipped).
__global__ void __launch_bounds__(32) gpk_hb_prep_kernel(const HyperModel m, const double* __restrict__ T,
                                                         const int* __restrict__ skip, HBPar* __restrict__ par,
                                                         int* __restrict__ st)
{
    __shared__ double th[GPK_HYPER_MAX_DIM];
    __shared__ double fpv[GPK_MAX_TASKS * (GPK_MAX_TASKS + 1) / 2];
    const int b = blockIdx.x, D = m.n_params + 1, tid = threadIdx.x;
    HBPar* p = par + b;
    if (*skip) {
        if (tid == 0) { p->bad = 2; st[b] = 1; }
        return;
    }
    for (int j = tid; j < D; j += 32) th[j] = T[(long)b * D + j];
    __syncwarp();
    bool out = false;
    for (int j = 0; j < D; ++j) out = out || th[j] < -20.0 || th[j] > 20.0;
    if (tid == 0) {
        p->lp = gpk_hy_prior(m, th, D);
        double log_amp = 0.0;
        for (int q = 0; q < m.n_params; ++q)
            if (m.amp[q]) log_amp = __dadd_rn(log_amp, th[q]);
        p->amp = exp(log_amp);
        const double yerr = sqrt(exp(th[D - 1]));
        const double s = sqrt(__dadd_rn(__dmul_rn(yerr, yerr), m.tiny));
        p->dg = __dmul_rn(s, s);
        KFactor& kf = p->kf;
        kf.kind = m.f_kind; kf.axis = m.f_axis; kf.n_tasks = m.f_n_tasks;
        if (m.f_kind != GPK_FACTOR_NONE) {
            for (int k = 0; k < m.n_fp; ++k) fpv[k] = th[m.fp[k]];
            gpk_factor_build(kf, fpv);
        }
        p->bad = out ? 1 : 0;
        st[b] = out ? 1 : 0;
    }
    for (int t = tid; t < m.n_terms; t += 32) p->im[t] = 1.0 / exp(th[m.term_param[t]]);
}

// one lower tile (blockIdx.y, blockIdx.x) of matrix blockIdx.z, block row nb = the residual
__global__ void __launch_bounds__(256) gpk_hb_build_kernel(const HyperModel m, const double* __restrict__ Xt, long ldx,
                                                           const double* __restrict__ y, int n,
                                                           const HBPar* __restrict__ par, double* __restrict__ A)
{
    const int tj = blockIdx.x, ti = blockIdx.y, b = blockIdx.z;
    const int nb = gpk_hb_nb(n);
    const long ld = (long)nb * HB_T;
    if (tj > ti || tj >= nb) return;
    const HBPar* p = par + b;
    if (p->bad) return;
    double* M = A + (long)b * gpk_hb_matrix_doubles(n);
    __shared__ double im[GPK_MAX_TERMS];
    __shared__ KFactor kf;
    for (int t = threadIdx.x; t < m.n_terms; t += 256) im[t] = p->im[t];
    if (threadIdx.x == 0) kf = p->kf;
    __syncthreads();
    const double amp = p->amp, dg = p->dg;
    for (int e = threadIdx.x; e < HB_T * HB_T; e += 256) {
        const int r = e / HB_T, c = e % HB_T;
        const int i = ti * HB_T + r, j = tj * HB_T + c;
        double v;
        if (ti == nb) {
            v = (r == 0 && j < n) ? y[j] - m.mean : 0.0;
        } else if (i >= n || j >= n) {
            v = i == j ? 1.0 : 0.0;
        } else if (j > i) {
            v = 0.0;
        } else {
            double pr = 1.0, r2 = 0.0;
            for (int t = 0; t < m.n_terms; ++t) {
                const double* xa = Xt + (long)m.axis[t] * ldx;
                const double d = xa[i] - xa[j];
                r2 = fma(d * d, im[t], r2);
                if (m.last[t]) { pr *= gpk_radial(m.family, r2); r2 = 0.0; }
            }
            v = amp * pr;
            if (m.f_kind != GPK_FACTOR_NONE) {
                const double* za = Xt + (long)m.f_axis * ldx;
                v *= gpk_factor_value(kf, za[i], za[j]);
            }
            if (j == i) v = v + dg;
        }
        M[(long)i * ld + j] = v;
    }
}

// ll, lp and the combinations of matrix blockIdx.x; ll / lp / post / fobj may be NULL
__global__ void __launch_bounds__(GPK_HY_THREADS) gpk_hb_finish_kernel(const HyperModel m, int n,
                                                                       const HBPar* __restrict__ par,
                                                                       const double* __restrict__ A,
                                                                       const double* __restrict__ logpart,
                                                                       const int* __restrict__ st,
                                                                       double* __restrict__ ll, double* __restrict__ lp,
                                                                       double* __restrict__ post,
                                                                       double* __restrict__ fobj)
{
    constexpr int NT = GPK_HY_THREADS;
    __shared__ double red[NT];
    const int b = blockIdx.x, tid = threadIdx.x;
    if (par[b].bad == 2) return;
    const bool bad = par[b].bad != 0 || st[b] != 0;
    const int nb = gpk_hb_nb(n);
    const long ld = (long)nb * HB_T;
    const double* z = A + (long)b * gpk_hb_matrix_doubles(n) + (long)nb * HB_T * ld;
    double s2 = 0.0;
    if (!bad)
        for (int i = tid; i < n; i += NT) s2 = fma(z[i], z[i], s2);
    red[tid] = s2;
    __syncthreads();
    for (int o = NT / 2; o > 0; o >>= 1) {
        if (tid < o) red[tid] += red[tid + o];
        __syncthreads();
    }
    if (tid != 0) return;
    double l = -INFINITY;
    if (!bad) {
        double s1 = 0.0;
        for (int k = 0; k < nb; ++k) s1 += logpart[(long)b * nb + k];
        const double ld2 = 2.0 * s1;
        l = -0.5 * red[0] - 0.5 * ld2 - 0.5 * (double)n * 1.8378770664093453;     // log(2 pi)
        if (!isfinite(l)) l = -INFINITY;
    }
    const double p = par[b].lp;
    if (ll) ll[b] = l;
    if (lp) lp[b] = p;
    if (post) post[b] = gpk_hy_post(m, l, p);
    if (fobj) fobj[b] = gpk_ho_objective(m, l, p);
}

// half-step (step, half): the active half's proposals, row blockIdx.x of Q for walker half * nw / 2 + blockIdx.x
__global__ void __launch_bounds__(32) gpk_hb_propose_kernel(int D, int nw, int step, int half, unsigned long long seed,
                                                            const double* __restrict__ P, double* __restrict__ Q)
{
    const int hb = nw / 2, k = half * hb + blockIdx.x;
    uint32_t w[4];
    gpk_philox4x32_10((uint32_t)k, (uint32_t)step, (uint32_t)half, GPK_HY_TAG_MOVE, (uint32_t)seed,
                      (uint32_t)(seed >> 32), w);
    const double z = gpk_stretch_z(w[0], w[1]);
    const int c = gpk_stretch_partner(w[2], half, hb);
    for (int j = threadIdx.x; j < D; j += 32)
        Q[(long)blockIdx.x * D + j] = gpk_stretch_coord(P[(long)c * D + j], P[(long)k * D + j], z);
}

// half-step (step, half): walker half * nw / 2 + blockIdx.x takes its proposal with log-posterior V[blockIdx.x] or not
__global__ void __launch_bounds__(32) gpk_hb_accept_kernel(int D, int nw, int step, int half, unsigned long long seed,
                                                           const double* __restrict__ Q, const double* __restrict__ V,
                                                           double* __restrict__ P, double* __restrict__ L,
                                                           long long* __restrict__ acc)
{
    const int hb = nw / 2, k = half * hb + blockIdx.x;
    uint32_t w[4], u[4];
    gpk_philox4x32_10((uint32_t)k, (uint32_t)step, (uint32_t)half, GPK_HY_TAG_MOVE, (uint32_t)seed,
                      (uint32_t)(seed >> 32), w);
    gpk_philox4x32_10((uint32_t)k, (uint32_t)step, (uint32_t)half, GPK_HY_TAG_ACC, (uint32_t)seed,
                      (uint32_t)(seed >> 32), u);
    const double z = gpk_stretch_z(w[0], w[1]);
    const double v = V[blockIdx.x];
    const bool take = gpk_stretch_accept(D, z, v, L[k], u[0], u[1]);
    __syncwarp();
    if (!take) return;
    for (int j = threadIdx.x; j < D; j += 32) P[(long)k * D + j] = Q[(long)blockIdx.x * D + j];
    if (threadIdx.x == 0) { L[k] = v; acc[k] += 1; }
}

// one round's stencil: row 0 of T = the trial point w.xt, row 1 + j = its forward-difference neighbour along j
__global__ void __launch_bounds__(32) gpk_hb_stencil_kernel(int D, const HOParams q, const double* __restrict__ work,
                                                            const HOState* __restrict__ st, double* __restrict__ T)
{
    if (st->status != GPK_LB_RUNNING) return;
    const HOWork w = gpk_ho_work(const_cast<double*>(work), D, q.maxcor);
    const int b = blockIdx.x;
    for (int j = threadIdx.x; j < D; j += 32) {
        const double v = w.xt[j];
        T[(long)b * D + j] = j == b - 1 ? __dadd_rn(v, gpk_ho_h(v, q.eps)) : v;
    }
}

// one round's update after the stencil's dim + 1 objective values are in w.fv (gpk_ho_update, one warp); a final status
// raises the skip word
__global__ void __launch_bounds__(32) gpk_hb_update_ho_kernel(int D, const HOParams q, double* __restrict__ work,
                                                              HOState* __restrict__ st, int* __restrict__ skip)
{
    if (st->status != GPK_LB_RUNNING) return;
    const HOWork w = gpk_ho_work(work, D, q.maxcor);
    gpk_ho_update(st, q, w, D);
    __syncwarp();
    if (threadIdx.x == 0 && st->status != GPK_LB_RUNNING) *skip = 1;
}
