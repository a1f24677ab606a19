// gpk_rs.cuh — device-resident representer sampling for gpk_sample_representers: the emcee 2.x stretch move
// (Goodman & Weare 2010, a = 2) as robo_b200/util/ensemble_sampler.py states it, run for n estimators at once.  Estimator
// i walks nb walkers of dimension dw on its own model; the log-density of a walker is the sampling acquisition of that
// model, -inf outside [lower, upper] (InformationGain._sampling_batch) and -inf where the acquisition is NaN
// (EnsembleSampler._lnprob_many).  This replaces the host loop of information_gain.py:68-81 and
// information_gain_per_unit_cost.py:152-172 (50 steps, up to 5 runs).
//
// Every product and sum that reaches a result is rounded explicitly (__dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn: no
// fma contraction), so tests/representer_model.py restates every kernel bit for bit.  The one exception is log(): the
// acceptance test compares fl(fl(fl((dw - 1) log z) + new) - old) with log u' using CUDA's log, which may differ from
// glibc's in the last bit; the restatement checks that no decision lies within a few ulp of a tie.
//
//   init, run r:      P[k][j] = fl(lower_j + fl(fl(upper_j - lower_j) u)),   u = u01(r0, r1) of (k, r, j, TAG_INIT)
//   half-step (s, h): S0 = walkers [h nb/2, (h + 1) nb/2), S1 = the other half (first, second), then (second, first)
//     walker k of S0:  (r0, r1, r2) of (k, s, 2 r + h, TAG_MOVE)
//                      z = fl(fl(t t) / a), t = fl(fl((a - 1) u01(r0, r1)) + 1)
//                      partner c = S1[(r2 * (nb/2)) >> 32]
//                      q_j = fl(c_j - fl(z fl(c_j - s_j)))
//     score:           every proposal on its own model; -inf outside [lower, upper] (any walker coordinate) or NaN
//     accept:          lnpdiff = fl(fl(fl((dw - 1) log z) + new) - old) > log u',  u' = u01(r0, r1) of (k, s, 2 r + h,
//                      TAG_ACC); a NaN lnpdiff (-inf - -inf) rejects.  Accepted moves are counted per walker and run.
// Counter (c0, c1, c2, c3) = (walker, step or run, 2 run + half or coordinate, tag), key = the estimator's 64-bit seed:
// an estimator's draws depend on its seed alone, not on n, its position in the list or stream timing.  The tags are
// disjoint from GPK_DE_TAG_*, GPK_HY_TAG_* and from gpk_candidates_kernel's c3 = 0.
//
// Estimators are addressed by their index i in the call; slot[i] >= 0 is the position of an estimator that runs in the
// current run in the compact scoring batch (n_active x nb/2 rows), slot[i] < 0 an estimator that is done.
#pragma once
#include "gpk_internal.cuh"

#define GPK_RS_TAG_INIT 0x52530001u
#define GPK_RS_TAG_MOVE 0x52530002u
#define GPK_RS_TAG_ACC 0x52530003u
#define GPK_RS_MAX_NB 64                  // the gpk_es_update limit on the representer points

// the stretch factor's parameter a of emcee (ensemble_sampler.py: a = 2.0)
#define GPK_RS_A 2.0

// The stretch move's arithmetic, shared by this sampler and the hyper-parameter sampler (gpk_hyper.cuh); every step is
// rounded explicitly.  z = fl(fl(t t) / a), t = fl(fl((a - 1) u01(w0, w1)) + 1)
__device__ __forceinline__ double gpk_stretch_z(uint32_t w0, uint32_t w1)
{
    const double tz = __dadd_rn(__dmul_rn(GPK_RS_A - 1.0, gpk_u01(w0, w1)), 1.0);
    return __ddiv_rn(__dmul_rn(tz, tz), GPK_RS_A);
}

// the partner of a walker of half h: walker (r2 * (hb)) >> 32 of the other half
__device__ __forceinline__ int gpk_stretch_partner(uint32_t w2, int half, int hb)
{
    return (1 - half) * hb + (int)__umulhi(w2, (uint32_t)hb);
}

// q_j = fl(c_j - fl(z fl(c_j - s_j)))
__device__ __forceinline__ double gpk_stretch_coord(double c, double s, double z)
{
    return __dsub_rn(c, __dmul_rn(z, __dsub_rn(c, s)));
}

// fl(fl(fl((dw - 1) log z) + new) - old) > log u01(r0, r1); a NaN difference (-inf - -inf) rejects
__device__ __forceinline__ bool gpk_stretch_accept(int dw, double z, double v, double old, uint32_t r0, uint32_t r1)
{
    const double lnpdiff = __dsub_rn(__dadd_rn(__dmul_rn((double)(dw - 1), log(z)), v), old);
    return lnpdiff > log(gpk_u01(r0, r1));
}

// init rows of run r: one thread per (estimator, walker, coordinate)
__global__ void gpk_rs_init_kernel(int n, int nb, int dw, int run, const unsigned long long* __restrict__ seeds,
                                   const int* __restrict__ slot, const double* __restrict__ lim, double* __restrict__ P,
                                   long long* __restrict__ acc)
{
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)n * nb * dw) return;
    const int i = (int)(t / ((long)nb * dw));
    if (slot[i] < 0) return;
    const int r = (int)(t - (long)i * nb * dw);
    const int k = r / dw, j = r - k * dw;
    const unsigned long long seed = seeds[i];
    uint32_t w[4];
    gpk_philox4x32_10((uint32_t)k, (uint32_t)run, (uint32_t)j, GPK_RS_TAG_INIT, (uint32_t)seed, (uint32_t)(seed >> 32), w);
    const double lo = lim[j], up = lim[dw + j];
    P[t] = __dadd_rn(lo, __dmul_rn(__dsub_rn(up, lo), gpk_u01(w[0], w[1])));
    if (j == 0) acc[(long)i * nb + k] = 0;
}

// The rows half h scores, one thread per (estimator, walker of S0).  step < 0: the walkers themselves (the initial
// log-probabilities); otherwise the stretch-move proposals of step `step`, kept in Q / Z for the accept kernel.  The
// scored row goes to X[slot][kk] (d columns): the walker coordinates, then env_value when d = dw + 1 (Fabolas).
__global__ void gpk_rs_propose_kernel(int n, int nb, int dw, int d, int run, int step, int half,
                                      const unsigned long long* __restrict__ seeds, const int* __restrict__ slot,
                                      double env_value, const double* __restrict__ P, double* __restrict__ Q,
                                      double* __restrict__ Z, double* __restrict__ X)
{
    const int hb = nb / 2;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)n * hb) return;
    const int i = (int)(t / hb), kk = (int)(t - (long)i * hb);
    const int si = slot[i];
    if (si < 0) return;
    const int k = half * hb + kk;
    const double* s = P + ((long)i * nb + k) * dw;
    double* q = Q + t * dw;
    double* x = X + ((long)si * hb + kk) * d;
    if (step < 0) {
        for (int j = 0; j < dw; ++j) { q[j] = s[j]; x[j] = s[j]; }
    } else {
        const unsigned long long seed = seeds[i];
        uint32_t w[4];
        gpk_philox4x32_10((uint32_t)k, (uint32_t)step, (uint32_t)(2 * run + half), GPK_RS_TAG_MOVE, (uint32_t)seed,
                          (uint32_t)(seed >> 32), w);
        const double z = gpk_stretch_z(w[0], w[1]);
        const int c = gpk_stretch_partner(w[2], half, hb);
        const double* cp = P + ((long)i * nb + c) * dw;
        for (int j = 0; j < dw; ++j) {
            const double v = gpk_stretch_coord(cp[j], s[j], z);
            q[j] = v;
            x[j] = v;
        }
        Z[t] = z;
    }
    if (d > dw) x[dw] = env_value;
}

// The scores A[slot][kk] of half h masked to log-densities; step < 0 sets the initial log-probabilities of S0, otherwise
// the stretch move's acceptance test.  EI values < 0 of in-box rows (the ones ei.py sees) are counted in *nneg.
__global__ void gpk_rs_accept_kernel(int n, int nb, int dw, int run, int step, int half, int kind,
                                     const unsigned long long* __restrict__ seeds, const int* __restrict__ slot,
                                     const double* __restrict__ lim, const double* __restrict__ A,
                                     const double* __restrict__ Q, const double* __restrict__ Z, double* __restrict__ P,
                                     double* __restrict__ L, long long* __restrict__ acc,
                                     unsigned long long* __restrict__ nneg)
{
    const int hb = nb / 2;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)n * hb) return;
    const int i = (int)(t / hb), kk = (int)(t - (long)i * hb);
    const int si = slot[i];
    if (si < 0) return;
    const int k = half * hb + kk;
    const long w = (long)i * nb + k;
    const double* q = Q + t * dw;
    bool inside = true;
    for (int j = 0; j < dw; ++j) inside = inside && q[j] >= lim[j] && q[j] <= lim[dw + j];
    const double a = A[(long)si * hb + kk];
    if (inside && kind == GPK_ACQ_EI && a < 0.0) atomicAdd(nneg, 1ULL);
    const double v = (inside && !isnan(a)) ? a : -INFINITY;
    if (step < 0) { L[w] = v; return; }
    const unsigned long long seed = seeds[i];
    uint32_t r[4];
    gpk_philox4x32_10((uint32_t)k, (uint32_t)step, (uint32_t)(2 * run + half), GPK_RS_TAG_ACC, (uint32_t)seed,
                      (uint32_t)(seed >> 32), r);
    if (gpk_stretch_accept(dw, Z[t], v, L[w], r[0], r[1])) {
        for (int j = 0; j < dw; ++j) P[w * dw + j] = q[j];
        L[w] = v;
        acc[w] += 1;
    }
}

// fin[i] = 1 when every final log-probability of estimator i is finite (information_gain.py:75), 0 otherwise; estimators
// that did not run keep their flag
__global__ void gpk_rs_finite_kernel(int n, int nb, const int* __restrict__ slot, const double* __restrict__ L,
                                     int* __restrict__ fin)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || slot[i] < 0) return;
    int ok = 1;
    for (int k = 0; k < nb; ++k) ok &= isfinite(L[(long)i * nb + k]) ? 1 : 0;
    fin[i] = ok;
}
