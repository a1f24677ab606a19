// gpk_hyper.cuh — device-resident sampling of the GP-MCMC hyper-parameters for gpk_sample_hypers / gpk_hyper_lnpost:
// the emcee 2.x stretch move (a = 2) of robo_b200/util/ensemble_sampler.py over theta = (kernel parameters, log noise),
// with each walker's log-posterior computed on chip.  This replaces the host loop of GaussianProcessMCMC.train
// (gaussian_process_mcmc.py: EnsembleSampler driving _LikelihoodPool.loglik + the prior, one round trip per half-step).
//
// Log-posterior of one theta, one CTA (GPK_HY_THREADS threads), gpk_hy_eval:
//   - any theta_j < -20 or > 20: ll = -inf without a factorisation (gaussian_process_mcmc.py:187-188)
//   - kernel: log_amp = 0.0 + the amplitude-slot entries in slot order, amp = exp(log_amp); every term t takes
//     inv_metric_t = 1 / exp(theta[term_param[t]]) (an isotropic metric slot lists all the terms of its group);
//     K_ij = amp prod_g gpk_radial(family, sum_{t in g} (x_i - x_j)^2 inv_metric_t) on the handle's inputs, family /
//     axes / groups of the handle's KSpec; with a factor K_ij is multiplied by gpk_factor_value(z_i, z_j), z = the
//     factor's input column, the factor built by thread 0 (gpk_factor_build) into the reduction scratch from the
//     parameters theta[fp[k]] that feed it: log_a, log_b (slot kinds 2, 3) or the packed task entries (slot kind 4)
//   - diagonal: diag_add = fl(sqrt(fl(yerr^2 + tiny)))^2, yerr = sqrt(exp(theta[-1]))  (_LikelihoodPool.loglik)
//   - packed fp64 lower triangle in shared memory (n <= GPK_HYPER_MAX_N), right-looking Cholesky one column at a time
//     with the residual r = y - mean carried as an extra row, so r ends as z = L^-1 r; a pivot that is not > 0 (NaN
//     included) gives -inf
//   - ll = -1/2 z^T z - 1/2 (2 sum log L_ii) - n/2 log(2 pi), -inf when not finite.  The two sums are fixed-order
//     tree reductions over the CTA (no atomics): the same theta always gives the same bits.
//   - prior (thread 0), the reference classes' lnprob restated with their quirks: none; DefaultPrior = lognorm.logpdf
//     (theta_0, sigma, loc) + Tophat(theta[1:-1]) + Horseshoe(theta[-1]) (+inf at theta == 0); EnvPrior = lognorm(theta_0)
//     + Tophat(theta[1:n_ls+1]) + sum of NormalPrior.lnprob (the pdf, not its log) over theta[n_ls+1:n_ls+n_lr+1]
//     + Horseshoe(theta[-1]); MTBOPrior = lognorm(theta_0) + Tophat(theta[1:n_ls+1]) + Tophat(nrm_sigma, nrm_mean as
//     its bounds)(theta[n_ls+1:n_ls+n_lr+1]) + Horseshoe(theta[-1]); Python's slice bounds, the additions in the order
//     of the lnprob methods
//   - log-posterior = fl(lp + ll) where ll is finite (ll alone without a prior), -inf otherwise; NaN -> -inf
//     (loglikelihood_batch, EnsembleSampler._lnprob_many)
//
// The run (gpk_sample_hypers): nw walkers of dimension D = n_params + 1, P (nw x D) starts at p0.
//   init:             one launch, one CTA per walker: L[k] = log-posterior of P[k]
//   half-step (s, h): one launch, one CTA per walker k of S0 = walkers [h nw/2, (h + 1) nw/2); S1 = the other half
//     (first, second), then (second, first); S1 is read-only during the half-step, each CTA writes only walker k
//                     (r0, r1, r2) of (k, s, h, GPK_HY_TAG_MOVE): z = gpk_stretch_z(r0, r1), partner
//                     c = gpk_stretch_partner(r2), q_j = gpk_stretch_coord(c_j, s_j, z)  (gpk_rs.cuh)
//                     the log-posterior v of q, then gpk_stretch_accept(D, z, v, L[k], u) with u of (k, s, h,
//                     GPK_HY_TAG_ACC): fl(fl(fl((D - 1) log z) + v) - L[k]) > log u'; accepted moves are counted
// There is no box mask: the |theta| rule and the prior take its place.  Counter (c0, c1, c2, c3) = (walker, step, half,
// tag), key = the run's 64-bit seed; the tags are disjoint from GPK_RS_TAG_*, GPK_DE_TAG_* and gpk_candidates_kernel's
// c3 = 0.  Every rounding step of the move is explicit (__dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn, no fma
// contraction), so tests/hyper_model.py restates a run bit for bit given the log-posteriors gpk_hyper_lnpost returns
// (the same routine, the same block shape); log z and log u' use CUDA's log, which may differ from glibc's in the last
// bit, and the restatement refuses decisions within a few ulp of a tie.
#pragma once
#include "gpk_rs.cuh"

#define GPK_HY_TAG_MOVE 0x48590002u
#define GPK_HY_TAG_ACC 0x48590003u
#define GPK_HY_THREADS 256

struct HyperModel {
    int family, n_terms, n_params;            // D = n_params + 1 (the log noise last)
    int axis[GPK_MAX_TERMS];
    int last[GPK_MAX_TERMS];
    int term_param[GPK_MAX_TERMS];            // the metric slot (parameter index) of term t
    unsigned char amp[GPK_HYPER_MAX_DIM];     // 1: parameter p is an amplitude slot
    int f_kind, f_axis, f_n_tasks;            // the kernel's factor: KFactor's kind, axis, n_tasks
    int n_fp;                                 // the parameters that feed it, in gpk_factor_build's order
    unsigned char fp[GPK_MAX_TASKS * (GPK_MAX_TASKS + 1) / 2];
    double mean, tiny;
    int prior, n_ls, n_lr;
    double ln_sigma, ln_loc, th_lo, th_hi, hs_scale, nrm_sigma, nrm_mean;
};

// doubles of dynamic shared memory gpk_hy_eval needs for n training points
__host__ __device__ inline long gpk_hy_smem_doubles(int n)
{
    return (long)n * (n + 1) / 2 + n + (n + 1) + 2 * GPK_HY_THREADS + 4 + GPK_MAX_TERMS;
}

// scipy.stats.lognorm.logpdf(x, s, loc=loc): -inf for x <= loc, NaN stays NaN
__device__ __forceinline__ double gpk_hy_lognorm(double x, double s, double loc)
{
    const double y = __dsub_rn(x, loc);
    if (isnan(y)) return y;
    if (!(y > 0.0)) return -INFINITY;
    const double l = log(y);
    return __dsub_rn(__ddiv_rn(-__dmul_rn(l, l), __dmul_rn(2.0, __dmul_rn(s, s))),
                     log(__dmul_rn(__dmul_rn(s, y), 2.5066282746310002)));
}

// TophatPrior.lnprob over theta[a:b] (Python slice bounds on a vector of D entries)
__device__ __forceinline__ double gpk_hy_tophat(const double* th, int D, int a, int b, double lo, double hi)
{
    a = min(a, D);
    b = min(b, D);
    for (int j = a; j < b; ++j)
        if (th[j] < lo || th[j] > hi) return -INFINITY;
    return 0.0;
}

// HorseshoePrior.lnprob: +inf at 0, log(log(1 + 3 (scale / e^x)^2))
__device__ __forceinline__ double gpk_hy_horseshoe(double x, double scale)
{
    if (x == 0.0) return INFINITY;
    const double q = __ddiv_rn(scale, exp(x));
    return log(log(__dadd_rn(1.0, __dmul_rn(3.0, __dmul_rn(q, q)))));
}

// NormalPrior.lnprob = scipy.stats.norm.pdf(x, loc=mean, scale=sigma) (the pdf, not its log)
__device__ __forceinline__ double gpk_hy_normal_pdf(double x, double sigma, double mean)
{
    const double u = __ddiv_rn(__dsub_rn(x, mean), sigma);
    return __ddiv_rn(__ddiv_rn(exp(__ddiv_rn(-__dmul_rn(u, u), 2.0)), 2.5066282746310002), sigma);
}

__device__ double gpk_hy_prior(const HyperModel& m, const double* th, int D)
{
    double lp = 0.0;
    if (m.prior == GPK_PRIOR_DEFAULT) {
        lp = __dadd_rn(lp, gpk_hy_lognorm(th[0], m.ln_sigma, m.ln_loc));
        lp = __dadd_rn(lp, gpk_hy_tophat(th, D, 1, D - 1, m.th_lo, m.th_hi));
        lp = __dadd_rn(lp, gpk_hy_horseshoe(th[D - 1], m.hs_scale));
    } else if (m.prior == GPK_PRIOR_ENV) {
        lp = __dadd_rn(lp, gpk_hy_lognorm(th[0], m.ln_sigma, m.ln_loc));
        lp = __dadd_rn(lp, gpk_hy_tophat(th, D, 1, m.n_ls + 1, m.th_lo, m.th_hi));
        const int a = min(m.n_ls + 1, D), b = min(m.n_ls + m.n_lr + 1, D);
        for (int j = a; j < b; ++j) lp = __dadd_rn(lp, gpk_hy_normal_pdf(th[j], m.nrm_sigma, m.nrm_mean));
        lp = __dadd_rn(lp, gpk_hy_horseshoe(th[D - 1], m.hs_scale));
    } else if (m.prior == GPK_PRIOR_MTBO) {
        lp = __dadd_rn(lp, gpk_hy_lognorm(th[0], m.ln_sigma, m.ln_loc));
        lp = __dadd_rn(lp, gpk_hy_tophat(th, D, 1, m.n_ls + 1, m.th_lo, m.th_hi));
        lp = __dadd_rn(lp, gpk_hy_tophat(th, D, m.n_ls + 1, m.n_ls + 1 + m.n_lr, m.nrm_sigma, m.nrm_mean));
        lp = __dadd_rn(lp, gpk_hy_horseshoe(th[D - 1], m.hs_scale));
    }
    return lp;
}

// the sampler's log-posterior from the two parts
__device__ __forceinline__ double gpk_hy_post(const HyperModel& m, double ll, double lp)
{
    if (!isfinite(ll)) return -INFINITY;
    const double v = m.prior == GPK_PRIOR_NONE ? ll : __dadd_rn(lp, ll);
    return isnan(v) ? -INFINITY : v;
}

// Log-likelihood and log-prior of theta (shared memory, D entries), on the whole CTA; every thread must call it.
// Xt: the handle's inputs term-transposed (Xt[a * ldx + i]), y: its targets.  Results valid in every thread.
__device__ void gpk_hy_eval(const HyperModel& m, const double* __restrict__ Xt, long ldx, const double* __restrict__ y,
                            int n, const double* th, double* sm, double* ll_out, double* lp_out)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NT = GPK_HY_THREADS, NW = GPK_HY_THREADS / 32;
    const int D = m.n_params + 1;
    double* A = sm;                                  // row i at i (i + 1) / 2
    double* r = A + (long)n * (n + 1) / 2;           // y - mean, then z = L^-1 (y - mean)
    double* col = r + n;                             // column k of L (rows k + 1 .. n; row n = the residual row)
    double* red = col + n + 1;                       // 2 NT partial sums
    KFactor* kf = reinterpret_cast<KFactor*>(red);   // the factor during the K build (red is free until the sums)
    double* par = red + 2 * NT;                      // amp, diag_add, lp, ll
    double* im = par + 4;                            // inv_metric of every term

    bool out = false;
    for (int j = 0; j < D; ++j) out = out || th[j] < -20.0 || th[j] > 20.0;
    if (tid == 0) {
        par[2] = gpk_hy_prior(m, th, D);
        double log_amp = 0.0;
        for (int p = 0; p < m.n_params; ++p)
            if (m.amp[p]) log_amp = __dadd_rn(log_amp, th[p]);
        par[0] = exp(log_amp);
        const double yerr = sqrt(exp(th[D - 1]));
        const double s = sqrt(__dadd_rn(__dmul_rn(yerr, yerr), m.tiny));
        par[1] = __dmul_rn(s, s);
        if (m.f_kind != GPK_FACTOR_NONE) {
            double* fpv = red + sizeof(KFactor) / sizeof(double);   // the factor's parameters, gathered
            for (int k = 0; k < m.n_fp; ++k) fpv[k] = th[m.fp[k]];
            kf->kind = m.f_kind; kf->axis = m.f_axis; kf->n_tasks = m.f_n_tasks;
            gpk_factor_build(*kf, fpv);
        }
    }
    for (int t = tid; t < m.n_terms; t += NT) im[t] = 1.0 / exp(th[m.term_param[t]]);
    __syncthreads();
    bool ok = !out;
    if (ok) {
        const double amp = par[0], dg = par[1];
        for (int i = warp; i < n; i += NW) {
            double* row = A + (long)i * (i + 1) / 2;
            for (int j = lane; j <= i; j += 32) {
                double pr = 1.0, r2 = 0.0;
                for (int t = 0; t < m.n_terms; ++t) {
                    const double* xa = Xt + (long)m.axis[t] * ldx;
                    const double d = xa[i] - xa[j];
                    r2 = fma(d * d, im[t], r2);
                    if (m.last[t]) { pr *= gpk_radial(m.family, r2); r2 = 0.0; }
                }
                double v = amp * pr;
                if (m.f_kind != GPK_FACTOR_NONE) {
                    const double* za = Xt + (long)m.f_axis * ldx;
                    v *= gpk_factor_value(*kf, za[i], za[j]);
                }
                row[j] = (j == i) ? v + dg : v;
            }
            if (lane == 0) r[i] = y[i] - m.mean;
        }
        for (int k = 0; k < n; ++k) {
            __syncthreads();
            const long dk = (long)k * (k + 1) / 2 + k;
            const double p = A[dk];
            if (!(p > 0.0)) { ok = false; break; }           // the same value in every thread: a uniform exit
            const double lkk = sqrt(p);
            for (int i = k + 1 + tid; i <= n; i += NT)
                col[i] = ((i < n) ? A[(long)i * (i + 1) / 2 + k] : r[k]) / lkk;
            __syncthreads();
            if (tid == 0) { A[dk] = lkk; r[k] = col[n]; }
            for (int i = k + 1 + warp; i <= n; i += NW) {
                double* row = (i < n) ? A + (long)i * (i + 1) / 2 : r;
                const double li = col[i];
                const int jmax = (i < n) ? i : n - 1;
                for (int j = k + 1 + lane; j <= jmax; j += 32) row[j] = fma(-li, col[j], row[j]);
            }
        }
        __syncthreads();
    }
    double s1 = 0.0, s2 = 0.0;
    if (ok)
        for (int i = tid; i < n; i += NT) {
            s1 += log(A[(long)i * (i + 1) / 2 + i]);
            s2 = fma(r[i], r[i], s2);
        }
    red[tid] = s1;
    red[NT + tid] = s2;
    __syncthreads();
    for (int o = NT / 2; o > 0; o >>= 1) {
        if (tid < o) { red[tid] += red[tid + o]; red[NT + tid] += red[NT + tid + o]; }
        __syncthreads();
    }
    if (tid == 0) {
        double ll = -INFINITY;
        if (ok) {
            const double ld = 2.0 * red[0];
            ll = -0.5 * red[NT] - 0.5 * ld - 0.5 * (double)n * 1.8378770664093453;     // log(2 pi)
            if (!isfinite(ll)) ll = -INFINITY;
        }
        par[3] = ll;
    }
    __syncthreads();
    *ll_out = par[3];
    *lp_out = par[2];
}

// count thetas (count x D, row-major), one CTA each: ll / lp (may be NULL) the two parts, post (may be NULL) the
// sampler's log-posterior
__global__ void __launch_bounds__(GPK_HY_THREADS) gpk_hy_eval_kernel(const HyperModel m, const double* __restrict__ Xt,
                                                                     long ldx, const double* __restrict__ y, int n,
                                                                     const double* __restrict__ thetas,
                                                                     double* __restrict__ ll, double* __restrict__ lp,
                                                                     double* __restrict__ post)
{
    __shared__ double th[GPK_HYPER_MAX_DIM];
    extern __shared__ double sm[];
    const int b = blockIdx.x, D = m.n_params + 1;
    for (int j = threadIdx.x; j < D; j += blockDim.x) th[j] = thetas[(long)b * D + j];
    __syncthreads();
    double l, p;
    gpk_hy_eval(m, Xt, ldx, y, n, th, sm, &l, &p);
    if (threadIdx.x == 0) {
        if (ll) ll[b] = l;
        if (lp) lp[b] = p;
        if (post) post[b] = gpk_hy_post(m, l, p);
    }
}

// half-step (step, half) of the run: one CTA per walker of the active half
__global__ void __launch_bounds__(GPK_HY_THREADS) gpk_hy_step_kernel(const HyperModel m, const double* __restrict__ Xt,
                                                                     long ldx, const double* __restrict__ y, int n,
                                                                     int nw, int step, int half,
                                                                     unsigned long long seed, double* __restrict__ P,
                                                                     double* __restrict__ L, long long* __restrict__ acc)
{
    __shared__ double th[GPK_HYPER_MAX_DIM];
    __shared__ int take;
    extern __shared__ double sm[];
    const int hb = nw / 2, k = half * hb + blockIdx.x, D = m.n_params + 1;
    uint32_t w[4];
    gpk_philox4x32_10((uint32_t)k, (uint32_t)step, (uint32_t)half, GPK_HY_TAG_MOVE, (uint32_t)seed,
                      (uint32_t)(seed >> 32), w);
    const double z = gpk_stretch_z(w[0], w[1]);
    const int c = gpk_stretch_partner(w[2], half, hb);
    for (int j = threadIdx.x; j < D; j += blockDim.x) th[j] = gpk_stretch_coord(P[(long)c * D + j], P[(long)k * D + j], z);
    __syncthreads();
    double l, p;
    gpk_hy_eval(m, Xt, ldx, y, n, th, sm, &l, &p);
    if (threadIdx.x == 0) {
        const double v = gpk_hy_post(m, l, p);
        uint32_t u[4];
        gpk_philox4x32_10((uint32_t)k, (uint32_t)step, (uint32_t)half, GPK_HY_TAG_ACC, (uint32_t)seed,
                          (uint32_t)(seed >> 32), u);
        take = gpk_stretch_accept(D, z, v, L[k], u[0], u[1]) ? 1 : 0;
        if (take) { L[k] = v; acc[k] += 1; }
    }
    __syncthreads();
    if (take)
        for (int j = threadIdx.x; j < D; j += blockDim.x) P[(long)k * D + j] = th[j];
}
