// gpk_blr.cuh — Bayesian linear regression on the device (robo/models/bayesian_linear_regression.py with
// robo/priors/bayesian_linear_regression_prior.py): the features, the marginal log-likelihood of theta = (log alpha,
// log beta) for the stretch-move sampler, the weight posteriors and the marginalised predictive pass that scores
// candidates for every device maximizer.
//
// Features (basis code, gpk_blr_basis): LINEAR phi(x) = [x, 1] (F = D + 1), QUADRATIC [x*x, x, 1] (F = 2 D + 1), NONE
// phi(x) = x (F = D); F <= GPK_BLR_MAX_F.  gpk_blr_set_data keeps Phi (N x F), y, G = Phi^T Phi and b = Phi^T y on the
// device; every entry of G and b is one fixed-order tree reduction over the N rows (gpk_blr_gram_kernel).
//
// Log-posterior of one theta, one CTA (GPK_BLR_THREADS threads), gpk_blr_eval (bayesian_linear_regression.py:92-113):
//   alpha = exp(theta_0), beta = exp(theta_1)
//   A = fl(fl(beta G) + alpha I), Cholesky L in shared memory (right-looking, one column at a time) with beta b carried as
//   an extra row, so it ends as z = L^-1 (beta b); m = L^-T z (= beta A^-1 Phi^T y).  A pivot that is not > 0 (NaN
//   included) gives -inf where the reference's inv would raise LinAlgError (a documented divergence).
//   r = y - Phi m over all N rows, directly (not through the Gram form, which cancels); ||r|| = sqrt of its fixed-order
//   tree sum of squares; log det A = 2 sum log L_ii (thread 0, in order).  det A overflows to +inf (log det A >
//   log DBL_MAX: mll = -inf) or underflows to 0 (log det A < log 2^-1075: mll = +inf) where numpy's det would.
//   mll = F/2 log alpha + N/2 log beta - N/2 log 2 pi - beta/2 ||r|| - alpha/2 m^T m - 1/2 log det A, in that order
//   (the 2-norm itself, not its square: :108), plus the prior (:45-49): lognorm.logpdf(theta_0, 0.1, loc=-10) +
//   Horseshoe(0.1).lnprob(1 / theta_1).  NaN -> -inf (EnsembleSampler._lnprob_many).
//
// The run (gpk_blr_sample), as gpk_hyper.cuh's: one launch evaluates the walkers, then one launch per half-step with one
// CTA per walker of the active half proposes (gpk_stretch_z / _partner / _coord of (k, s, h, GPK_BLR_TAG_MOVE)),
// evaluates and accepts (gpk_stretch_accept with u of (k, s, h, GPK_BLR_TAG_ACC)).  The tags are disjoint from
// GPK_HY_TAG_*, GPK_RS_TAG_*, GPK_DE_TAG_* and the other samplers' tags.  Every rounding step of the move is explicit
// (gpk_rs.cuh), so tests/blr_model.py restates a run bit for bit given the log-posteriors gpk_blr_lnpost returns.
//
// Weight posteriors (gpk_blr_fit, :197-210): for every (alpha_i, beta_i) the same factorisation gives m_i and L_i; the
// fit keeps m_i, L_i^-1 (row-major, lower) and S_i = L_i^-T L_i^-1 (for the host's `models`) and 1 / beta_i.
//
// Predictive pass (gpk_blr_score_kernel, :213-254): one thread per candidate, its features in shared memory;
// mu_i = phi^T m_i, var_i = 1 / beta_i + ||L_i^-1 phi||^2; the sums over i in order divided by k (numpy's mean over
// axis 0); var clipped to eps; then gpk_acq_value, the negative-EI count and the block arg-max of gpk_finish_kernel.
#pragma once
#include "gpk_hyper.cuh"

#define GPK_BLR_TAG_MOVE 0x424C0002u
#define GPK_BLR_TAG_ACC 0x424C0003u
#define GPK_BLR_THREADS 256
#define GPK_BLR_SCORE_THREADS 128
#define GPK_BLR_LOG_DBL_MAX 709.782712893384          // log(DBL_MAX)
#define GPK_BLR_LOG_DET_ZERO -745.1332191019412       // log(2^-1075): a smaller det rounds to 0

struct BlrPrior {
    double ln_sigma, ln_loc, hs_scale;
};

// the features of one input row x (D entries) at phi (stride s between features)
__device__ __forceinline__ void gpk_blr_features(int basis, const double* x, int D, double* phi, int s)
{
    if (basis == GPK_BLR_LINEAR) {
        for (int j = 0; j < D; ++j) phi[j * s] = x[j];
        phi[D * s] = 1.0;
    } else if (basis == GPK_BLR_QUADRATIC) {
        for (int j = 0; j < D; ++j) { phi[j * s] = __dmul_rn(x[j], x[j]); phi[(D + j) * s] = x[j]; }
        phi[2 * D * s] = 1.0;
    } else {
        for (int j = 0; j < D; ++j) phi[j * s] = x[j];
    }
}

// Phi (n x F, row-major) of the n rows X (n x D): one thread per row
__global__ void gpk_blr_phi_kernel(const double* __restrict__ X, int n, int D, int F, int basis, double* __restrict__ Phi)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) gpk_blr_features(basis, X + (long)i * D, D, Phi + (long)i * F, 1);
}

// G = Phi^T Phi (F x F) and b = Phi^T y (F): one CTA per entry (blockIdx.x < F * F: G, else b), a strided fma sum per
// thread and a fixed-order tree over the CTA
__global__ void __launch_bounds__(256) gpk_blr_gram_kernel(const double* __restrict__ Phi, const double* __restrict__ y,
                                                           int n, int F, double* __restrict__ G, double* __restrict__ b)
{
    __shared__ double red[256];
    const int e = blockIdx.x;
    const bool gram = e < F * F;
    const int a = gram ? e / F : e - F * F, c = gram ? e - (e / F) * F : 0;
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256)
        s = fma(Phi[(long)i * F + a], gram ? Phi[(long)i * F + c] : y[i], s);
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        if (gram) G[e] = red[0];
        else b[a] = red[0];
    }
}

// doubles of dynamic shared memory gpk_blr_factor / gpk_blr_eval need for F features
__host__ __device__ inline long gpk_blr_smem_doubles(int F)
{
    return (long)F * F + 2 * (F + 1) + 2 * GPK_BLR_THREADS + 8;
}

// On the whole CTA: A = fl(fl(beta G) + alpha I) factorised in place (L in the lower triangle of sm, row-major F x F),
// m = beta A^-1 b at m_out (shared).  Returns whether every pivot was > 0 (the same value in every thread).
__device__ bool gpk_blr_factor(const double* __restrict__ G, const double* __restrict__ b, int F, double alpha,
                               double beta, double* A, double* col, double* m_out)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NT = GPK_BLR_THREADS, NW = GPK_BLR_THREADS / 32;
    double* r = m_out;                                 // beta b, then z = L^-1 (beta b), then m
    for (int e = tid; e < F * F; e += NT) {
        const int i = e / F, j = e - i * F;
        const double v = __dmul_rn(beta, G[e]);
        A[e] = (i == j) ? __dadd_rn(v, alpha) : v;
    }
    for (int i = tid; i < F; i += NT) r[i] = __dmul_rn(beta, b[i]);
    bool ok = true;
    for (int k = 0; k < F; ++k) {
        __syncthreads();
        const double p = A[k * F + k];
        if (!(p > 0.0)) { ok = false; break; }           // the same value in every thread: a uniform exit
        const double lkk = sqrt(p);
        for (int i = k + 1 + tid; i <= F; i += NT) col[i] = ((i < F) ? A[i * F + k] : r[k]) / lkk;
        __syncthreads();
        if (tid == 0) { A[k * F + k] = lkk; r[k] = col[F]; }
        for (int i = k + 1 + tid; i < F; i += NT) A[i * F + k] = col[i];
        for (int i = k + 1 + warp; i <= F; i += NW) {
            double* row = (i < F) ? A + i * F : r;
            const double li = col[i];
            const int jmax = (i < F) ? i : F - 1;
            for (int j = k + 1 + lane; j <= jmax; j += 32) row[j] = fma(-li, col[j], row[j]);
        }
    }
    __syncthreads();
    if (!ok) return false;
    // back substitution L^T m = z, one column of L^T per step
    for (int k = F - 1; k >= 0; --k) {
        if (tid == 0) r[k] = r[k] / A[k * F + k];
        __syncthreads();
        const double mk = r[k];
        for (int j = tid; j < k; j += NT) r[j] = fma(-A[k * F + j], mk, r[j]);
        __syncthreads();
    }
    return true;
}

// The log-posterior of theta (th[0], th[1]) on the whole CTA (every thread must call it); valid in every thread.
__device__ double gpk_blr_eval(const double* __restrict__ Phi, const double* __restrict__ y, const double* __restrict__ G,
                               const double* __restrict__ b, int n, int F, const BlrPrior pr, double t0, double t1,
                               double* sm)
{
    const int tid = threadIdx.x;
    constexpr int NT = GPK_BLR_THREADS;
    double* A = sm;
    double* m = A + (long)F * F;
    double* col = m + (F + 1);
    double* red = col + (F + 1);
    double* par = red + 2 * NT;                       // alpha, beta, result
    if (tid == 0) { par[0] = exp(t0); par[1] = exp(t1); }
    __syncthreads();
    const double alpha = par[0], beta = par[1];
    const bool ok = gpk_blr_factor(G, b, F, alpha, beta, A, col, m);
    double s = 0.0;
    if (ok)
        for (int i = tid; i < n; i += NT) {
            const double* ph = Phi + (long)i * F;
            double f = 0.0;
            for (int j = 0; j < F; ++j) f = fma(ph[j], m[j], f);
            const double ri = y[i] - f;
            s = fma(ri, ri, s);
        }
    red[tid] = s;
    __syncthreads();
    for (int o = NT / 2; o > 0; o >>= 1) {
        if (tid < o) red[tid] += red[tid + o];
        __syncthreads();
    }
    if (tid == 0) {
        double v = -INFINITY;
        if (ok) {
            double ld = 0.0, mtm = 0.0;
            for (int j = 0; j < F; ++j) { ld += log(A[j * F + j]); mtm = fma(m[j], m[j], mtm); }
            ld = 2.0 * ld;
            const double logdet = ld > GPK_BLR_LOG_DBL_MAX ? INFINITY : ld < GPK_BLR_LOG_DET_ZERO ? -INFINITY : ld;
            const double nrm = sqrt(red[0]);
            double mll = __dmul_rn(0.5 * (double)F, log(alpha));
            mll = __dadd_rn(mll, __dmul_rn(0.5 * (double)n, log(beta)));
            mll = __dsub_rn(mll, __dmul_rn(0.5 * (double)n, 1.8378770664093453));        // log(2 pi)
            mll = __dsub_rn(mll, __dmul_rn(__ddiv_rn(beta, 2.0), nrm));
            mll = __dsub_rn(mll, __dmul_rn(__ddiv_rn(alpha, 2.0), mtm));
            mll = __dsub_rn(mll, __dmul_rn(0.5, logdet));
            double lp = __dadd_rn(0.0, gpk_hy_lognorm(t0, pr.ln_sigma, pr.ln_loc));
            lp = __dadd_rn(lp, gpk_hy_horseshoe(__ddiv_rn(1.0, t1), pr.hs_scale));
            v = __dadd_rn(mll, lp);
        }
        par[2] = isnan(v) ? -INFINITY : v;
    }
    __syncthreads();
    return par[2];
}

// count thetas (count x 2), one CTA each
__global__ void __launch_bounds__(GPK_BLR_THREADS) gpk_blr_eval_kernel(const double* __restrict__ Phi,
                                                                       const double* __restrict__ y,
                                                                       const double* __restrict__ G,
                                                                       const double* __restrict__ b, int n, int F,
                                                                       const BlrPrior pr, const double* __restrict__ T,
                                                                       double* __restrict__ out)
{
    extern __shared__ double sm[];
    const int k = blockIdx.x;
    const double v = gpk_blr_eval(Phi, y, G, b, n, F, pr, T[2 * k], T[2 * k + 1], sm);
    if (threadIdx.x == 0) out[k] = v;
}

// half-step (step, half) of the run: one CTA per walker of the active half
__global__ void __launch_bounds__(GPK_BLR_THREADS) gpk_blr_step_kernel(const double* __restrict__ Phi,
                                                                       const double* __restrict__ y,
                                                                       const double* __restrict__ G,
                                                                       const double* __restrict__ b, int n, int F,
                                                                       const BlrPrior pr, int nw, int step, int half,
                                                                       unsigned long long seed, double* __restrict__ P,
                                                                       double* __restrict__ L, long long* __restrict__ acc)
{
    extern __shared__ double sm[];
    const int hb = nw / 2, k = half * hb + blockIdx.x;
    uint32_t w[4];
    gpk_philox4x32_10((uint32_t)k, (uint32_t)step, (uint32_t)half, GPK_BLR_TAG_MOVE, (uint32_t)seed,
                      (uint32_t)(seed >> 32), w);
    const double z = gpk_stretch_z(w[0], w[1]);
    const int c = gpk_stretch_partner(w[2], half, hb);
    const double q0 = gpk_stretch_coord(P[2 * c], P[2 * k], z);
    const double q1 = gpk_stretch_coord(P[2 * c + 1], P[2 * k + 1], z);
    const double v = gpk_blr_eval(Phi, y, G, b, n, F, pr, q0, q1, sm);
    if (threadIdx.x == 0) {
        uint32_t u[4];
        gpk_philox4x32_10((uint32_t)k, (uint32_t)step, (uint32_t)half, GPK_BLR_TAG_ACC, (uint32_t)seed,
                          (uint32_t)(seed >> 32), u);
        // every thread of the CTA read walker k before gpk_blr_eval's barriers: thread 0 may overwrite it now
        if (gpk_stretch_accept(2, z, v, L[k], u[0], u[1])) { L[k] = v; acc[k] += 1; P[2 * k] = q0; P[2 * k + 1] = q1; }
    }
}

// the weight posterior of hypers i = (alpha_i, beta_i), one CTA each: M (k x F) the means, Li (k x F x F) L_i^-1 row-major
// lower (upper triangle zero), S (k x F x F) = L_i^-T L_i^-1, ib (k) = 1 / beta_i, fail[i] = 1 where a pivot was not > 0
__global__ void __launch_bounds__(GPK_BLR_THREADS) gpk_blr_fit_kernel(const double* __restrict__ G,
                                                                      const double* __restrict__ b, int F,
                                                                      const double* __restrict__ H,
                                                                      double* __restrict__ M, double* __restrict__ Li,
                                                                      double* __restrict__ S, double* __restrict__ ib,
                                                                      int* __restrict__ fail)
{
    extern __shared__ double sm[];
    const int i = blockIdx.x, tid = threadIdx.x;
    double* A = sm;
    double* m = A + (long)F * F;
    double* col = m + (F + 1);
    double* V = col + (F + 1);                          // L^-1, F x F
    const double alpha = H[2 * i], beta = H[2 * i + 1];
    const bool ok = gpk_blr_factor(G, b, F, alpha, beta, A, col, m);
    if (tid == 0) { fail[i] = ok ? 0 : 1; ib[i] = 1.0 / beta; }
    if (!ok) return;
    // L^-1 one column per thread: forward substitution of L v = e_j
    for (int j = tid; j < F; j += GPK_BLR_THREADS)
        for (int r = 0; r < F; ++r) {
            if (r < j) { V[r * F + j] = 0.0; continue; }
            double s = (r == j) ? 1.0 : 0.0;
            for (int c = j; c < r; ++c) s = fma(-A[r * F + c], V[c * F + j], s);
            V[r * F + j] = s / A[r * F + r];
        }
    __syncthreads();
    double* Mi = M + (long)i * F;
    double* Lo = Li + (long)i * F * F;
    double* So = S + (long)i * F * F;
    for (int j = tid; j < F; j += GPK_BLR_THREADS) Mi[j] = m[j];
    for (int e = tid; e < F * F; e += GPK_BLR_THREADS) {
        Lo[e] = V[e];
        const int a = e / F, c = e - a * F;
        double s = 0.0;
        for (int r = max(a, c); r < F; ++r) s = fma(V[r * F + a], V[r * F + c], s);
        So[e] = s;
    }
}

struct BlrScoreArgs {
    const double* X; long m; int D, F, basis, k;
    const double* M; const double* Li; const double* ib;
    ScoreOut o;
};

// the marginalised predictive moments of every candidate, the acquisition and the block arg-max (gpk_finish_kernel's)
__global__ void __launch_bounds__(GPK_BLR_SCORE_THREADS) gpk_blr_score_kernel(const BlrScoreArgs a)
{
    extern __shared__ double phs[];                     // [F][GPK_BLR_SCORE_THREADS]
    constexpr int NT = GPK_BLR_SCORE_THREADS;
    const long c = (long)blockIdx.x * NT + threadIdx.x;
    double* ph = phs + threadIdx.x;
    double val = 0.0;
    long long idx = -1;
    if (c < a.m) {
        const int F = a.F;
        gpk_blr_features(a.basis, a.X + c * a.D, a.D, ph, NT);
        double smu = 0.0, svar = 0.0;
        for (int i = 0; i < a.k; ++i) {
            const double* mi = a.M + (long)i * F;
            const double* L = a.Li + (long)i * F * F;
            double mu = 0.0, q = 0.0;
            for (int j = 0; j < F; ++j) mu = fma(__ldg(mi + j), ph[j * NT], mu);
            for (int r = 0; r < F; ++r) {
                const double* Lr = L + (long)r * F;
                double t = 0.0;
                for (int j = 0; j <= r; ++j) t = fma(__ldg(Lr + j), ph[j * NT], t);
                q = fma(t, t, q);
            }
            smu += mu;
            svar += __ldg(a.ib + i) + q;
        }
        const double mu = smu / (double)a.k;
        double var = svar / (double)a.k;
        if (var < GPK_EPS) var = GPK_EPS;                  // np.clip(v, eps, inf); NaN stays NaN
        gpk_score_emit(a.o, c, mu, var, val, idx);
    }
    if (a.o.acq_kind == GPK_ACQ_NONE) return;
    gpk_block_best<NT / 32>(val, idx);
    if (threadIdx.x == 0) a.o.block_best[blockIdx.x] = {val, idx};
}
