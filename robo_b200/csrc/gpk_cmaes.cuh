// gpk_cmaes.cuh — device-resident CMA-ES for gpk_maximize_cmaes*: the (mu/mu_w, lambda)-CMA-ES of Hansen's tutorial
// ("The CMA Evolution Strategy: A Tutorial", 2016, Table 1 defaults, positive recombination weights only) under cma's
// BoundTransform (BoxConstraintsLinQuadTransformation) with IPOP restarts (cma.fmin, incpopsize = 2): the maximizer of
// robo/maximizers/cmaes.py:50-81, minimising the energy e = -acq.
//
// The distribution lives in genotype space; the objective scores the phenotype T(x); the result is the best phenotype.
// Every product, sum, quotient and square root on the state path is rounded explicitly (__dmul_rn / __dadd_rn /
// __dsub_rn / __ddiv_rn / __dsqrt_rn: no fma contraction), sums run in the order stated at each site, the two exp calls
// go through gpk_cmaes_exp (a fixed sequence of those operations), and nothing uses a result-affecting atomic.  With the
// normals read back through gpk_cmaes_draws, tests/cmaes_model.py restates a whole run bit for bit.
//
// Random stream: Philox4x32-10 keyed by the 64-bit seed; the normals z[2q], z[2q + 1] of member k in generation g of
// run r come from counter (c0, c1, c2, c3) = (q, k, g, GPK_CMA_TAG | r), r < 256, and the Box-Muller of
// gpk_mc_draws_kernel on its four words.  The tag 0x434D41xx is disjoint from the DE (0x4445...), MC (0x4D43...) and
// candidate (0) streams.  The generation counter g restarts at 0 with every run.
//
// Generation g of a run (lambda, mu, w and the other constants are the run's row of the host table, GPK_CMA_C_*):
//   sample   y_k[j] = sum_i B[j][i] fl(D_i z_k[i]) (i ascending from +0.0), x_k = m + sigma y_k, p_k = T(x_k)
//   score    e_k = -acq(p_k) + 0.0 (the + 0.0 turns -0.0 into +0.0)
//   rank     stable by (e, k): NaN last, ties by index (numpy.argsort(kind="stable"))
//   update   see gpk_cmaes_update_kernel; the Jacobi sweeps when the evaluations since the last decomposition exceed
//            lambda / ((c1 + cmu) d 10); then the stop tests
#pragma once
#include "gpk_internal.cuh"

#define GPK_CMA_TAG 0x434D4100u
#define GPK_CMA_THREADS 256               // threads of the update kernel
#define GPK_CMA_SWEEPS 30                 // Jacobi: at most this many sweeps ...
#define GPK_CMA_JACOBI_TOL 1e-16          // ... a pair rotates while |a_pq| > tol sqrt(|a_pp| |a_qq|)
#define GPK_CMA_TOLFUN_LIM 1e-11
#define GPK_CMA_TOLX_LIM 1e-11
#define GPK_CMA_CONDITIONCOV_LIM 1e14

// the persistent state of a run (and the best phenotype over all runs); C and B are d x d row-major
struct CMAState {
    double lo[GPK_CMA_MAX_D], up[GPK_CMA_MAX_D], al[GPK_CMA_MAX_D], au[GPK_CMA_MAX_D];
    double m[GPK_CMA_MAX_D], ps[GPK_CMA_MAX_D], pc[GPK_CMA_MAX_D], Dv[GPK_CMA_MAX_D], ev[GPK_CMA_MAX_D];
    double xbest[GPK_CMA_MAX_D];
    double C[GPK_CMA_MAX_D * GPK_CMA_MAX_D], B[GPK_CMA_MAX_D * GPK_CMA_MAX_D];
    double hist[GPK_CMA_HIST];            // best energy of generation g at hist[g % GPK_CMA_HIST]
    double sigma, pw, best;               // pw = (1 - c_sigma)^(2 g) by repeated multiplication
    long long nfev;                       // evaluations over all runs
    long long since;                      // evaluations of this run since the last eigendecomposition
    int g;                                // generations of this run
    int found;                            // best / xbest hold a finite energy
};

// the status record read back after every generation (24 bytes)
struct CMAStatus {
    double best;                          // lowest finite energy so far over all runs (NaN: none yet)
    long long nfev;                       // evaluations over all runs
    int stop;                             // gpk_cmaes_stop of this run after this generation
    int g;                                // generations of this run
};

// exp(x) as a fixed operation sequence: Cody-Waite reduction x = k ln2 + r (k = rint(x log2 e), ln2 split as fdlibm's
// ln2_hi + ln2_lo so that k ln2_hi is exact), exp(r) = 1 + (r + r^2 P(r)) with P the Taylor polynomial of degree 11
// by Horner from 1/13!, then 2^k exactly.  NaN stays NaN; x >= 709.78... gives +inf, x < -745.2 gives +0.0.
__device__ __forceinline__ double gpk_cmaes_exp(double x) {
    if (isnan(x)) return x;
    if (x >= 709.782712893384) return INFINITY;
    if (x < -745.2) return 0.0;
    const double k = rint(__dmul_rn(x, 1.4426950408889634));
    const double r = __dsub_rn(__dsub_rn(x, __dmul_rn(k, 6.93147180369123816490e-01)),
                               __dmul_rn(k, 1.90821492927058770002e-10));
    double p = 1.6059043836821613e-10;                                       // 1/13!, then 1/12! ... 1/2
    p = __dadd_rn(2.08767569878681e-09, __dmul_rn(p, r));
    p = __dadd_rn(2.505210838544172e-08, __dmul_rn(p, r));
    p = __dadd_rn(2.755731922398589e-07, __dmul_rn(p, r));
    p = __dadd_rn(2.7557319223985893e-06, __dmul_rn(p, r));
    p = __dadd_rn(2.48015873015873e-05, __dmul_rn(p, r));
    p = __dadd_rn(0.0001984126984126984, __dmul_rn(p, r));
    p = __dadd_rn(0.001388888888888889, __dmul_rn(p, r));
    p = __dadd_rn(0.008333333333333333, __dmul_rn(p, r));
    p = __dadd_rn(0.041666666666666664, __dmul_rn(p, r));
    p = __dadd_rn(0.16666666666666666, __dmul_rn(p, r));
    p = __dadd_rn(0.5, __dmul_rn(p, r));
    return ldexp(__dadd_rn(1.0, __dadd_rn(r, __dmul_rn(__dmul_rn(r, r), p))), (int)k);
}

// cma's BoxConstraintsLinQuadTransformation of one coordinate: shift periodically into [lb - al, ub + au] when far
// outside, mirror at ub + au and at lb - al, then quadratic on [lb - al, lb + al], identity, quadratic at the top
__device__ __forceinline__ double gpk_cmaes_T(double x, double lb, double ub, double al, double au) {
    const double half = __dmul_rn(__dsub_rn(ub, lb), 0.5);
    const double s = __dsub_rn(__dsub_rn(lb, __dmul_rn(2.0, al)), half);
    if (x < s || x > __dadd_rn(__dadd_rn(ub, __dmul_rn(2.0, au)), half)) {
        const double per = __dmul_rn(2.0, __dadd_rn(__dadd_rn(__dsub_rn(ub, lb), al), au));
        x = __dsub_rn(x, __dmul_rn(per, floor(__ddiv_rn(__dsub_rn(x, s), per))));
    }
    const double ua = __dadd_rn(ub, au), la = __dsub_rn(lb, al);
    if (x > ua) x = __dsub_rn(x, __dmul_rn(2.0, __dsub_rn(x, ua)));
    if (x < la) x = __dadd_rn(x, __dmul_rn(2.0, __dsub_rn(la, x)));
    if (x < __dadd_rn(lb, al)) {
        const double q = __dsub_rn(x, la);
        return __dadd_rn(lb, __ddiv_rn(__ddiv_rn(__dmul_rn(q, q), 4.0), al));
    }
    if (x < __dsub_rn(ub, au)) return x;
    const double q = __dsub_rn(x, ua);
    return __dsub_rn(ub, __ddiv_rn(__ddiv_rn(__dmul_rn(q, q), 4.0), au));
}

// the inverse of gpk_cmaes_T on [lb, ub] (the genotype of the start point)
__device__ __forceinline__ double gpk_cmaes_geno(double y, double lb, double ub, double al, double au) {
    if (y < __dadd_rn(lb, al)) return __dadd_rn(__dsub_rn(lb, al), __dmul_rn(2.0, __dsqrt_rn(__dmul_rn(al, __dsub_rn(y, lb)))));
    if (y < __dsub_rn(ub, au)) return y;
    return __dsub_rn(__dadd_rn(ub, au), __dmul_rn(2.0, __dsqrt_rn(__dmul_rn(au, __dsub_rn(ub, y)))));
}

// normals z[2q], z[2q + 1] of member k, generation g, run r (see the header)
__device__ __forceinline__ void gpk_cmaes_normals(unsigned long long seed, int r, int g, int k, int q, double* z0, double* z1) {
    uint32_t w[4];
    gpk_philox4x32_10((uint32_t)q, (uint32_t)k, (uint32_t)g, GPK_CMA_TAG | (uint32_t)r, (uint32_t)seed,
                      (uint32_t)(seed >> 32), w);
    const double u1 = (double)(((((unsigned long long)w[1] << 32) | w[0]) >> 11) + 1ull) * 1.1102230246251565e-16;
    const double u2 = gpk_u01(w[2], w[3]);
    const double rr = __dsqrt_rn(__dmul_rn(-2.0, log(u1)));
    double s, c;
    sincospi(__dmul_rn(2.0, u2), &s, &c);
    *z0 = __dmul_rn(rr, c);
    *z1 = __dmul_rn(rr, s);
}

// gpk_cmaes_draws: Z (g1 - g0) x lambda x d for generations g0 .. g1 - 1 of run r, one thread per (g, k, pair)
__global__ void gpk_cmaes_draws_kernel(unsigned long long seed, int r, int g0, int ng, int lam, int d, double* __restrict__ Z) {
    const int nq = (d + 1) / 2;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)ng * lam * nq) return;
    const int q = (int)(t % nq);
    const long gk = t / nq;
    const int k = (int)(gk % lam), gi = (int)(gk / lam);
    double z0, z1;
    gpk_cmaes_normals(seed, r, g0 + gi, k, q, &z0, &z1);
    double* row = Z + ((size_t)gi * lam + k) * d;
    row[2 * q] = z0;
    if (2 * q + 1 < d) row[2 * q + 1] = z1;
}

// the start of run r: lower / upper / x0 (d each, device), m = genotype of x0, C = B = I, D = 1, paths 0; run 0 also
// clears the best-so-far and the evaluation count.  One block of GPK_CMA_MAX_D threads.
__global__ void gpk_cmaes_init_kernel(int d, const double* __restrict__ lower, const double* __restrict__ upper,
                                      const double* __restrict__ x0, double sigma0, int first, CMAState* __restrict__ s) {
    const int j = threadIdx.x;
    if (j < d) {
        const double lb = lower[j], ub = upper[j];
        const double half = __dmul_rn(__dsub_rn(ub, lb), 0.5);
        const double al = fmin(half, __ddiv_rn(__dadd_rn(1.0, fabs(lb)), 20.0));
        const double au = fmin(half, __ddiv_rn(__dadd_rn(1.0, fabs(ub)), 20.0));
        s->lo[j] = lb; s->up[j] = ub; s->al[j] = al; s->au[j] = au;
        s->m[j] = gpk_cmaes_geno(x0[j], lb, ub, al, au);
        s->ps[j] = 0.0; s->pc[j] = 0.0; s->Dv[j] = 1.0; s->ev[j] = 1.0;
        for (int i = 0; i < d; ++i) {
            s->C[j * d + i] = i == j ? 1.0 : 0.0;
            s->B[j * d + i] = i == j ? 1.0 : 0.0;
        }
        if (first) s->xbest[j] = 0.0;
    }
    if (j == 0) {
        s->sigma = sigma0; s->pw = 1.0; s->since = 0; s->g = 0;
        if (first) { s->best = __longlong_as_double(0x7FF8000000000000ll); s->nfev = 0; s->found = 0; }
    }
}

// Sampling of one generation: one warp per member k, lane q owns the coordinate pair (2q, 2q + 1).  Writes the normals
// Z, the steps Y, the genotypes G and the phenotypes P (lambda x d each, row-major).
__global__ void __launch_bounds__(32) gpk_cmaes_sample_kernel(unsigned long long seed, int r, int d,
                                                              const CMAState* __restrict__ s, double* __restrict__ Z,
                                                              double* __restrict__ Y, double* __restrict__ G,
                                                              double* __restrict__ P) {
    __shared__ double dz[GPK_CMA_MAX_D];
    const int k = blockIdx.x, q = threadIdx.x;
    const size_t row = (size_t)k * d;
    if (2 * q < d) {
        double z0, z1;
        gpk_cmaes_normals(seed, r, s->g, k, q, &z0, &z1);
        Z[row + 2 * q] = z0;
        dz[2 * q] = __dmul_rn(s->Dv[2 * q], z0);
        if (2 * q + 1 < d) {
            Z[row + 2 * q + 1] = z1;
            dz[2 * q + 1] = __dmul_rn(s->Dv[2 * q + 1], z1);
        }
    }
    __syncwarp();
    const double sigma = s->sigma;
    for (int j = 2 * q; j < 2 * q + 2 && j < d; ++j) {
        double y = 0.0;
        for (int i = 0; i < d; ++i) y = __dadd_rn(y, __dmul_rn(s->B[j * d + i], dz[i]));
        const double x = __dadd_rn(s->m[j], __dmul_rn(sigma, y));
        Y[row + j] = y;
        G[row + j] = x;
        P[row + j] = gpk_cmaes_T(x, s->lo[j], s->up[j], s->al[j], s->au[j]);
    }
}

// (e_a, a) before (e_b, b) in numpy.argsort(kind="stable") order: NaN last, ties by index
__device__ __forceinline__ bool gpk_cmaes_before(double ea, int a, double eb, int b) {
    const bool na = isnan(ea), nb = isnan(eb);
    if (na || nb) return na && nb ? a < b : nb;
    if (ea < eb) return true;
    if (ea > eb) return false;
    return a < b;
}

// dynamic shared memory of the update kernel: C, A (Jacobi work), B (d x d each), the energies (lambda), the ranked
// indices (mu ints)
__host__ __device__ __forceinline__ size_t gpk_cmaes_smem(int d, int lam) {
    return (3 * (size_t)d * d + (size_t)lam) * 8 + (size_t)(lam / 2) * 4;
}

// One generation's update, one CTA of GPK_CMA_THREADS threads; cst = the run's constant row (GPK_CMA_C_*, weights at
// GPK_CMA_C_W), acq = the scored values of the lambda phenotypes.  In this order:
//   e_k = -acq_k + 0.0; ranking (counting sort on gpk_cmaes_before); best so far = rank 0 when finite and lower than the
//   best (an earlier generation, then the lower index, keep ties); the history entry of this generation = e_(0).
//   y_w[j] = sum_{i<mu} fl(w_i y_(i)[j]) from +0.0;  m[j] += fl(sigma y_w[j])
//   t_i = fl(sum_j fl(B[j][i] y_w[j]) / D_i);  u_j = sum_i fl(B[j][i] t_i);  ps = fl(omcs ps) + fl(cps u)
//   |ps| = sqrt(sum_j fl(ps_j ps_j));  pw = fl(fl(pw omcs) omcs);  h_sigma = fl(|ps| / sqrt(1 - pw)) < hth
//   pc = h_sigma ? fl(omcc pc) + fl(ccc y_w) : fl(omcc pc)
//   C_ij = fl(fl(a0 C_ij) + fl(c1 fl(fl(pc_i pc_j) + fl(dh C_ij)))) + fl(cmu S_ij), dh = h_sigma ? 0 : ccd,
//          S_ij = sum_{l<mu} fl(w_l fl(y_(l)i y_(l)j)) from +0.0
//   sigma = fl(sigma exp(fl(csds fl(fl(|ps| / chi) - 1))));  flat fitness e_(0) == e_(flat): sigma = fl(sigma exp(0.2 + csds))
//   evaluations += lambda; when the evaluations since the last decomposition exceed eig_gap: C is symmetrised from its
//   upper triangle and parallel cyclic Jacobi runs on a copy (round-robin pairing, d/2 rotations per step, Rutishauser's
//   rotation, the stop rule of GPK_CMA_SWEEPS / GPK_CMA_JACOBI_TOL; after a sweep without rotation it stops);
//   D_i = sqrt(a_ii), B = the accumulated rotations.
//   Stop tests, the first that holds: maxfevals, tolfun, tolx, conditioncov, numerical (gpk_cmaes_stop).
__global__ void __launch_bounds__(GPK_CMA_THREADS) gpk_cmaes_update_kernel(int d, const double* __restrict__ cst,
                                                                           long long budget, const double* __restrict__ acq,
                                                                           const double* __restrict__ Y,
                                                                           const double* __restrict__ P,
                                                                           CMAState* s,
                                                                           CMAStatus* __restrict__ st) {
    extern __shared__ double sm[];
    const int lam = (int)cst[GPK_CMA_C_LAMBDA], mu = (int)cst[GPK_CMA_C_MU];
    const double* w = cst + GPK_CMA_C_W;
    const int dd = d * d;
    double* sC = sm;
    double* sA = sC + dd;
    double* sB = sA + dd;
    double* se = sB + dd;
    int* so = (int*)(se + lam);
    __shared__ double yw[GPK_CMA_MAX_D], tv[GPK_CMA_MAX_D];
    __shared__ double jc[GPK_CMA_MAX_D / 2], js[GPK_CMA_MAX_D / 2];
    __shared__ int jp[GPK_CMA_MAX_D / 2], jq[GPK_CMA_MAX_D / 2];
    __shared__ int k_first, k_flat, hsig, bad, rot, eig_due, improve;
    __shared__ double norm_ps;
    const int tid = threadIdx.x;
    const int flat = (int)cst[GPK_CMA_C_FLAT];
    for (int k = tid; k < lam; k += GPK_CMA_THREADS) se[k] = __dadd_rn(-acq[k], 0.0);
    for (int i = tid; i < dd; i += GPK_CMA_THREADS) { sC[i] = s->C[i]; sB[i] = s->B[i]; }
    if (tid == 0) bad = 0;
    __syncthreads();
    for (int k = tid; k < lam; k += GPK_CMA_THREADS) {
        const double ek = se[k];
        int rk = 0;
        for (int j = 0; j < lam; ++j) rk += gpk_cmaes_before(se[j], j, ek, k);
        if (rk < mu) so[rk] = k;
        if (rk == 0) k_first = k;
        if (rk == flat) k_flat = k;
    }
    __syncthreads();
    const double sigma = s->sigma;
    const double e0 = se[k_first];
    if (tid == 0) improve = isfinite(e0) && (!s->found || e0 < s->best);
    __syncthreads();
    if (tid < d) {
        if (improve) s->xbest[tid] = P[(size_t)k_first * d + tid];
        double acc = 0.0;
        for (int i = 0; i < mu; ++i) acc = __dadd_rn(acc, __dmul_rn(w[i], Y[(size_t)so[i] * d + tid]));
        yw[tid] = acc;
        s->m[tid] = __dadd_rn(s->m[tid], __dmul_rn(sigma, acc));
    }
    __syncthreads();
    if (tid < d) {
        double acc = 0.0;
        for (int j = 0; j < d; ++j) acc = __dadd_rn(acc, __dmul_rn(sB[j * d + tid], yw[j]));
        tv[tid] = __ddiv_rn(acc, s->Dv[tid]);
    }
    __syncthreads();
    if (tid < d) {
        double acc = 0.0;
        for (int i = 0; i < d; ++i) acc = __dadd_rn(acc, __dmul_rn(sB[tid * d + i], tv[i]));
        s->ps[tid] = __dadd_rn(__dmul_rn(cst[GPK_CMA_C_OMCS], s->ps[tid]), __dmul_rn(cst[GPK_CMA_C_CPS], acc));
    }
    __syncthreads();
    if (tid == 0) {
        double acc = 0.0;
        for (int j = 0; j < d; ++j) acc = __dadd_rn(acc, __dmul_rn(s->ps[j], s->ps[j]));
        norm_ps = __dsqrt_rn(acc);
        const double omcs = cst[GPK_CMA_C_OMCS];
        s->pw = __dmul_rn(__dmul_rn(s->pw, omcs), omcs);
        hsig = __ddiv_rn(norm_ps, __dsqrt_rn(__dsub_rn(1.0, s->pw))) < cst[GPK_CMA_C_HTH];
        if (improve) { s->best = e0; s->found = 1; }
        s->hist[s->g % GPK_CMA_HIST] = e0;
    }
    __syncthreads();
    if (tid < d) {
        const double pc = __dmul_rn(cst[GPK_CMA_C_OMCC], s->pc[tid]);
        s->pc[tid] = hsig ? __dadd_rn(pc, __dmul_rn(cst[GPK_CMA_C_CCC], yw[tid])) : pc;
    }
    __syncthreads();
    {
        const double a0 = cst[GPK_CMA_C_A0], c1 = cst[GPK_CMA_C_C1], cmu = cst[GPK_CMA_C_CMU];
        const double dh = hsig ? 0.0 : cst[GPK_CMA_C_CCD];
        for (int idx = tid; idx < dd; idx += GPK_CMA_THREADS) {
            const int i = idx / d, j = idx - i * d;
            double S = 0.0;
            for (int l = 0; l < mu; ++l) {
                const double* yl = Y + (size_t)so[l] * d;
                S = __dadd_rn(S, __dmul_rn(w[l], __dmul_rn(yl[i], yl[j])));
            }
            const double c = sC[idx];
            const double r1 = __dmul_rn(c1, __dadd_rn(__dmul_rn(s->pc[i], s->pc[j]), __dmul_rn(dh, c)));
            const double v = __dadd_rn(__dadd_rn(__dmul_rn(a0, c), r1), __dmul_rn(cmu, S));
            sC[idx] = v;
            if (!isfinite(v)) bad = 1;
        }
    }
    if (tid == 0) {
        const double csds = cst[GPK_CMA_C_CSDS];
        double sg = __dmul_rn(sigma, gpk_cmaes_exp(__dmul_rn(csds, __dsub_rn(__ddiv_rn(norm_ps, cst[GPK_CMA_C_CHI]), 1.0))));
        if (se[k_first] == se[k_flat]) sg = __dmul_rn(sg, gpk_cmaes_exp(__dadd_rn(0.2, csds)));
        s->sigma = sg;
        s->g += 1;
        s->nfev += lam;
        s->since += lam;
        eig_due = (double)s->since > cst[GPK_CMA_C_EIG];
    }
    __syncthreads();
    // every decision that guards a barrier comes from shared memory, so all threads take the same branch
    const bool eigen = eig_due;
    if (eigen) {
        for (int idx = tid; idx < dd; idx += GPK_CMA_THREADS) {
            const int i = idx / d, j = idx - i * d;
            sA[idx] = i <= j ? sC[idx] : sC[j * d + i];
            sB[idx] = i == j ? 1.0 : 0.0;
        }
        __syncthreads();
        for (int idx = tid; idx < dd; idx += GPK_CMA_THREADS) sC[idx] = sA[idx];
        const int n2 = d + (d & 1), half = n2 / 2;
        for (int sweep = 0; sweep < GPK_CMA_SWEEPS; ++sweep) {
            if (tid == 0) rot = 0;
            __syncthreads();
            for (int rd = 0; rd < n2 - 1; ++rd) {
                // round rd pairs position i with position n2 - 1 - i; position 0 holds index 0, position j >= 1 holds
                // 1 + (j - 1 + rd) mod (n2 - 1)
                double app = 0.0, aqq = 0.0, apq = 0.0, t = 0.0;
                if (tid < half) {
                    const int a = tid == 0 ? 0 : 1 + (tid - 1 + rd) % (n2 - 1);
                    const int b = 1 + (n2 - 2 - tid + rd) % (n2 - 1);
                    const int p = a < b ? a : b, q = a < b ? b : a;
                    jp[tid] = -1;
                    if (q < d) {
                        app = sA[p * d + p]; aqq = sA[q * d + q]; apq = sA[p * d + q];
                        if (fabs(apq) > __dmul_rn(GPK_CMA_JACOBI_TOL, __dsqrt_rn(__dmul_rn(fabs(app), fabs(aqq))))) {
                            const double theta = __ddiv_rn(__dsub_rn(aqq, app), __dmul_rn(2.0, apq));
                            const double at = fabs(theta);
                            t = at > 1e150 ? __ddiv_rn(0.5, at)
                                           : __ddiv_rn(1.0, __dadd_rn(at, __dsqrt_rn(__dadd_rn(__dmul_rn(theta, theta), 1.0))));
                            if (theta < 0.0) t = -t;
                            const double c = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(__dmul_rn(t, t), 1.0)));
                            jc[tid] = c;
                            js[tid] = __dmul_rn(t, c);
                            jp[tid] = p;
                            jq[tid] = q;
                            rot = 1;
                        }
                    }
                }
                __syncthreads();
                // rows p, q of A: A <- J^T A
                for (int idx = tid; idx < half * d; idx += GPK_CMA_THREADS) {
                    const int pi = idx / d, k = idx - pi * d, p = jp[pi];
                    if (p < 0) continue;
                    const int q = jq[pi];
                    const double c = jc[pi], sn = js[pi];
                    const double x = sA[p * d + k], y = sA[q * d + k];
                    sA[p * d + k] = __dsub_rn(__dmul_rn(c, x), __dmul_rn(sn, y));
                    sA[q * d + k] = __dadd_rn(__dmul_rn(sn, x), __dmul_rn(c, y));
                }
                __syncthreads();
                // columns p, q of A and of B: A <- A J, B <- B J
                for (int idx = tid; idx < half * d; idx += GPK_CMA_THREADS) {
                    const int pi = idx / d, k = idx - pi * d, p = jp[pi];
                    if (p < 0) continue;
                    const int q = jq[pi];
                    const double c = jc[pi], sn = js[pi];
                    double x = sA[k * d + p], y = sA[k * d + q];
                    sA[k * d + p] = __dsub_rn(__dmul_rn(c, x), __dmul_rn(sn, y));
                    sA[k * d + q] = __dadd_rn(__dmul_rn(sn, x), __dmul_rn(c, y));
                    x = sB[k * d + p]; y = sB[k * d + q];
                    sB[k * d + p] = __dsub_rn(__dmul_rn(c, x), __dmul_rn(sn, y));
                    sB[k * d + q] = __dadd_rn(__dmul_rn(sn, x), __dmul_rn(c, y));
                }
                __syncthreads();
                // Rutishauser's diagonal update; the pair's off-diagonal entries are zero by construction
                if (tid < half && jp[tid] >= 0) {
                    const int p = jp[tid], q = jq[tid];
                    sA[p * d + p] = __dsub_rn(app, __dmul_rn(t, apq));
                    sA[q * d + q] = __dadd_rn(aqq, __dmul_rn(t, apq));
                    sA[p * d + q] = 0.0;
                    sA[q * d + p] = 0.0;
                }
                __syncthreads();
            }
            const int any = rot;
            __syncthreads();
            if (!any) break;
        }
        if (tid < d) {
            const double e = sA[tid * d + tid];
            s->ev[tid] = e;
            s->Dv[tid] = __dsqrt_rn(e);
            if (!(e > 0.0) || !isfinite(e)) bad = 1;
        }
        if (tid == 0) s->since = 0;
    }
    for (int i = tid; i < dd; i += GPK_CMA_THREADS) { s->C[i] = sC[i]; if (eigen) s->B[i] = sB[i]; }
    __syncthreads();
    if (tid == 0) {
        int stop = GPK_CMA_RUNNING;
        const int g = s->g;
        const int H = (int)cst[GPK_CMA_C_HIST];
        const double sg = s->sigma;
        if (s->nfev >= budget) {
            stop = GPK_CMA_MAXFEVALS;
        } else {
            bool tolfun = false;
            if (g >= H) {
                double mx = se[0], mn = se[0];
                for (int k = 1; k < lam; ++k) { mx = fmax(mx, se[k]); mn = fmin(mn, se[k]); }
                for (int i = g - H; i < g; ++i) {
                    const double h = s->hist[i % GPK_CMA_HIST];
                    mx = fmax(mx, h); mn = fmin(mn, h);
                }
                tolfun = __dsub_rn(mx, mn) < GPK_CMA_TOLFUN_LIM;
            }
            double mxs = 0.0;
            for (int j = 0; j < d; ++j) mxs = fmax(mxs, fmax(fabs(s->pc[j]), __dsqrt_rn(sC[j * d + j])));
            double emax = s->ev[0], emin = s->ev[0];
            for (int j = 1; j < d; ++j) { emax = fmax(emax, s->ev[j]); emin = fmin(emin, s->ev[j]); }
            bool numerical = bad || !(sg > 0.0) || !isfinite(sg);
            for (int j = 0; j < d; ++j) numerical = numerical || !isfinite(s->m[j]);
            if (tolfun) stop = GPK_CMA_TOLFUN;
            else if (__dmul_rn(sg, mxs) < GPK_CMA_TOLX_LIM) stop = GPK_CMA_TOLX;
            else if (__ddiv_rn(emax, emin) > GPK_CMA_CONDITIONCOV_LIM) stop = GPK_CMA_CONDITIONCOV;
            else if (numerical) stop = GPK_CMA_NUMERICAL;
        }
        st->best = s->best;
        st->nfev = s->nfev;
        st->stop = stop;
        st->g = g;
    }
}
