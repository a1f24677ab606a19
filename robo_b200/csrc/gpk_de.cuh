// gpk_de.cuh — device-resident differential evolution for gpk_maximize_de: scipy.optimize.differential_evolution with
// strategy 'best1bin', updating='deferred', init='latinhypercube' (scipy/optimize/_differentialevolution.py:
// init_population_lhs, _mutate_many / _best1, _ensure_constraint, __next__ deferred branch, converged, solve), the
// maximizer of robo/maximizers/differential_evolution.py:27-51.
//
// The population lives in unit-cube coordinates (pop x d, row-major).  Every product and sum that reaches a result is
// rounded explicitly (__dmul_rn / __dadd_rn / __dsub_rn: no fma contraction), so tests/de_model.py restates every
// kernel bit for bit.  Nothing here uses a result-affecting atomic.
//
// Random stream: Philox4x32-10 keyed by the 64-bit seed; counter (c0, c1, c2, c3) = (member, generation, word, tag).
// c3 is GPK_DE_TAG_INIT or GPK_DE_TAG_GEN, never 0, so the stream is disjoint from gpk_candidates_kernel's (c3 = 0).
//   init       (i, 0, j, TAG_INIT): r0 = LHS sort key of member i in column j, u01(r2, r3) = offset inside its stratum
//   generation (0, g, 0xFFFFFFFF, TAG_GEN): u01(r0, r1) = dither draw of F
//              (i, g, 0, TAG_GEN): r0 -> r0 index, r1 -> r1 index, r2 -> fill point of member i
//              (i, g, 1 + j, TAG_GEN): u01(r0, r1) = crossover draw, u01(r2, r3) = redraw of an out-of-cube coordinate
// Indices come from the multiply-shift (w * n) >> 32, never from a float floor.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include "gpk_internal.cuh"

#define GPK_DE_TAG_INIT 0x44450001u
#define GPK_DE_TAG_GEN 0x44450002u
#define GPK_DE_MAX_POP (1L << 24)         // member index in the low 24 bits of the LHS sort key
#define GPK_DE_RED 1024                   // threads of the reduction block (fixed: the summation order depends on it)

struct DEStatus {
    double best;                          // energy of slot 0 after promotion
    int converged;                        // std(E) <= atol + tol |mean(E)|
    int reserved;
};

// -acq as the reference's wrapper returns it (differential_evolution.py:29-33): an infinite energy becomes DBL_MAX
__device__ __forceinline__ double gpk_de_energy(double a) {
    const double e = -a;
    return isinf(e) ? 1.7976931348623157e308 : e;
}

// scipy _scale_parameters, then the reference's clip: clip(arg1 + (u - 0.5) * arg2, lower, upper)
// lim = [lower (d), upper (d), arg1 (d), arg2 (d)]
__device__ __forceinline__ double gpk_de_scale(const double* __restrict__ lim, int d, int j, double u) {
    const double v = __dadd_rn(lim[2 * d + j], __dmul_rn(__dsub_rn(u, 0.5), lim[3 * d + j]));
    return fmin(fmax(v, lim[j]), lim[d + j]);
}

// numpy.argmin ordering: NaN beats everything, then the smaller value, then the lower index
__device__ __forceinline__ bool gpk_de_before(double va, long ia, double vb, long ib) {
    if (ib < 0) return ia >= 0;
    if (ia < 0) return false;
    const bool na = isnan(va), nb = isnan(vb);
    if (na || nb) return na && nb ? ia < ib : na;
    if (va < vb) return true;
    if (va > vb) return false;
    return ia < ib;
}

// LHS sort keys: ((j << 56) | (philox word << 24) | i) for column j, member i.  One radix sort of all d * pop keys
// orders every column by its Philox words, ties by member index; the position inside the column is the stratum.
__global__ void gpk_de_lhs_keys_kernel(unsigned long long seed, long pop, int d, unsigned long long* __restrict__ keys)
{
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= pop * d) return;
    const int j = (int)(t / pop);
    const long i = t - (long)j * pop;
    uint32_t r[4];
    gpk_philox4x32_10((uint32_t)i, 0u, (uint32_t)j, GPK_DE_TAG_INIT, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    keys[t] = ((unsigned long long)j << 56) | ((unsigned long long)r[0] << 24) | (unsigned long long)i;
}

// member i of column j at sorted position `rank` of that column: fl(fl(seg * u) + fl(rank * seg)), seg = 1 / pop
// (init_population_lhs); writes the unit-cube population and the scaled parameters scoring reads
__global__ void gpk_de_lhs_place_kernel(unsigned long long seed, long pop, int d, const unsigned long long* __restrict__ sorted,
                                        const double* __restrict__ lim, double* __restrict__ P, double* __restrict__ X)
{
    const long s = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= pop * d) return;
    const int j = (int)(s / pop);
    const long rank = s - (long)j * pop;
    const long i = (long)(sorted[s] & 0xFFFFFFull);
    uint32_t r[4];
    gpk_philox4x32_10((uint32_t)i, 0u, (uint32_t)j, GPK_DE_TAG_INIT, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    const double seg = __ddiv_rn(1.0, (double)pop);
    const double x = __dadd_rn(__dmul_rn(seg, gpk_u01(r[2], r[3])), __dmul_rn((double)rank, seg));
    P[i * d + j] = x;
    X[i * d + j] = gpk_de_scale(lim, d, j, x);
}

// generation g >= 1, one thread per member: best1bin trial (bprime = p0 + F (p[r0] - p[r1]), binomial crossover with a
// forced fill point, out-of-cube coordinates redrawn), written in unit-cube (T) and scaled (X) form
__global__ void gpk_de_trial_kernel(unsigned long long seed, int g, long pop, int d, double mut_lo, double mut_hi,
                                    double cr, const double* __restrict__ lim, const double* __restrict__ P,
                                    double* __restrict__ T, double* __restrict__ X)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pop) return;
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    uint32_t r[4];
    gpk_philox4x32_10(0u, (uint32_t)g, 0xFFFFFFFFu, GPK_DE_TAG_GEN, k0, k1, r);
    const double F = __dadd_rn(mut_lo, __dmul_rn(__dsub_rn(mut_hi, mut_lo), gpk_u01(r[0], r[1])));
    gpk_philox4x32_10((uint32_t)i, (uint32_t)g, 0u, GPK_DE_TAG_GEN, k0, k1, r);
    long r0 = (long)__umulhi(r[0], (uint32_t)(pop - 1));           // uniform over the pop - 1 members != i
    r0 += (r0 >= i);
    long r1 = (long)__umulhi(r[1], (uint32_t)(pop - 2));           // uniform over the pop - 2 members != i, r0
    const long a = i < r0 ? i : r0, b = i < r0 ? r0 : i;
    r1 += (r1 >= a);
    r1 += (r1 >= b);
    const int fill = (int)__umulhi(r[2], (uint32_t)d);
    for (int j = 0; j < d; ++j) {
        gpk_philox4x32_10((uint32_t)i, (uint32_t)g, (uint32_t)(1 + j), GPK_DE_TAG_GEN, k0, k1, r);
        const double bp = __dadd_rn(P[j], __dmul_rn(F, __dsub_rn(P[r0 * d + j], P[r1 * d + j])));
        double t = (gpk_u01(r[0], r[1]) < cr || j == fill) ? bp : P[i * d + j];
        if (t > 1.0 || t < 0.0) t = gpk_u01(r[2], r[3]);
        T[i * d + j] = t;
        X[i * d + j] = gpk_de_scale(lim, d, j, t);
    }
}

// energies from the acquisition values of the scored batch: g = 0 sets them, g >= 1 accepts trial i when
// e_trial <= e_i (scipy _accept_trial) and copies its row into the population
__global__ void gpk_de_select_kernel(int g, long pop, int d, const double* __restrict__ acq, const double* __restrict__ T,
                                     double* __restrict__ P, double* __restrict__ E)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pop) return;
    const double e = gpk_de_energy(acq[i]);
    if (g == 0) {
        E[i] = e;
    } else if (e <= E[i]) {
        E[i] = e;
        for (int j = 0; j < d; ++j) P[i * d + j] = T[i * d + j];
    }
}

// one block of GPK_DE_RED threads: the first minimum of E (numpy.argmin) is swapped into slot 0 with its row
// (_promote_lowest_energy), then mean and std of E in this fixed order:
//   thread t sums E[t], E[t + 1024], ... from +0.0 in index order; the 1024 partials are added pairwise,
//   v[t] += v[t + s] for s = 512, 256, ..., 1; mean = v[0] / pop.  The squares fl(fl(E - mean)^2) go the same way,
//   std = sqrt(v[0] / pop).
// Writes the status record and the scaled winner (best_x, d doubles).
__global__ void __launch_bounds__(GPK_DE_RED) gpk_de_finish_kernel(long pop, int d, double tol, double atol,
                                                                   const double* __restrict__ lim, double* __restrict__ P,
                                                                   double* __restrict__ E, DEStatus* __restrict__ st,
                                                                   double* __restrict__ best_x)
{
    __shared__ double sv[GPK_DE_RED];
    __shared__ long si[GPK_DE_RED];
    const int t = threadIdx.x;
    double bv = 0.0;
    long bi = -1;
    for (long k = t; k < pop; k += GPK_DE_RED)
        if (gpk_de_before(E[k], k, bv, bi)) { bv = E[k]; bi = k; }
    sv[t] = bv; si[t] = bi;
    __syncthreads();
    for (int s = GPK_DE_RED / 2; s > 0; s >>= 1) {
        if (t < s && gpk_de_before(sv[t + s], si[t + s], sv[t], si[t])) { sv[t] = sv[t + s]; si[t] = si[t + s]; }
        __syncthreads();
    }
    const long b = si[0];
    __syncthreads();
    if (b > 0) {
        for (int j = t; j < d; j += GPK_DE_RED) {
            const double x = P[j];
            P[j] = P[b * d + j];
            P[b * d + j] = x;
        }
        if (t == 0) {
            const double e = E[0];
            E[0] = E[b];
            E[b] = e;
        }
    }
    __syncthreads();
    double acc = 0.0;
    for (long k = t; k < pop; k += GPK_DE_RED) acc = __dadd_rn(acc, E[k]);
    sv[t] = acc;
    __syncthreads();
    for (int s = GPK_DE_RED / 2; s > 0; s >>= 1) {
        if (t < s) sv[t] = __dadd_rn(sv[t], sv[t + s]);
        __syncthreads();
    }
    const double mean = __ddiv_rn(sv[0], (double)pop);
    __syncthreads();
    acc = 0.0;
    for (long k = t; k < pop; k += GPK_DE_RED) {
        const double q = __dsub_rn(E[k], mean);
        acc = __dadd_rn(acc, __dmul_rn(q, q));
    }
    sv[t] = acc;
    __syncthreads();
    for (int s = GPK_DE_RED / 2; s > 0; s >>= 1) {
        if (t < s) sv[t] = __dadd_rn(sv[t], sv[t + s]);
        __syncthreads();
    }
    if (t == 0) {
        const double sd = __dsqrt_rn(__ddiv_rn(sv[0], (double)pop));
        st->best = E[0];
        st->converged = sd <= __dadd_rn(atol, __dmul_rn(tol, fabs(mean))) ? 1 : 0;
        st->reserved = 0;
    }
    for (int j = t; j < d; j += GPK_DE_RED) best_x[j] = gpk_de_scale(lim, d, j, P[j]);
}
