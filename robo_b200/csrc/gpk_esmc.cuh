// gpk_esmc.cuh — the sampling-based entropy search (robo/acquisition_functions/information_gain_mc.py) and its p_min
// estimator joint_pmin (robo/util/mc_part.py): p_min over Nb representer points by Monte-Carlo function draws.
//
// gpk_mc_draws_kernel: F (nb x nf, row-major) standard normals, drawn once per update and shared by every candidate
// (common random numbers).  Philox4x32-10 keyed by the 64-bit seed, counter (q, k, 0, GPK_MC_TAG) for the pair
// q = f / 2 of row k; Box-Muller on its four words:
//   u1 = ((w1 << 32 | w0) >> 11) + 1) 2^-53 in (0, 1],  u2 = ((w3 << 32 | w2) >> 11) 2^-53 in [0, 1),
//   r = sqrt(-2 log u1),  F[k][2q] = r cospi(2 u2),  F[k][2q + 1] = r sinpi(2 u2)  (the second dropped for odd nf).
// F[k][f] depends on (seed, k, f) only, not on nb or nf.
//
// gpk_mc_pmin_kernel: one CTA per candidate.  With iv = 1 / (v - sn2), nc_a = sigma_a iv, dm_a = nc_a sqrt(v + 1e-10):
//   M[a][p] = Mb_a + dm_a W_p                       (or the caller's m[a][p] when one is given)
//   A[a][b] = Vb[a][b] + -(nc_a sigma_b), a >= b   (the lower triangle is all the factorisation reads; A = Vb at sigma = 0)
//   A + noise I factorised by the left-looking Cholesky below, noise on the reference's ladder (mc_part.py:31-43):
//     0, then 1e-10 * 10 = 1e-9, and * 10 before every retry up to 10000.0 (1e-10 times 10 fourteen times); a failure
//     there is numpy.linalg.LinAlgError (the candidate is flagged not PD).
//   funcs[a][f] = sum_{k <= a} L[a][k] F[k][f], summed for k = 0, 1, ..., a from 0.0;
//   for every column (f, p): argmin_a fl(M[a][p] + funcs[a][f]), numpy's rule (the first index wins a tie; the values
//     are finite wherever the factorisation succeeded, so numpy's NaN rule never applies);
//   pmin_a = count_a / (nf np), clamped below at 1e-70;
//   value = sum_a pmin_a (log pmin_a + lmb_a) + H, summed for a = 0, 1, ... from 0.0; NaN or +inf -> -DBL_MAX.
// Cholesky of S = A + noise I, column j = 0, 1, ...: s = S[j][j] - L[j][0]^2 - L[j][1]^2 - ... (in that order),
// L[j][j] = sqrt(s) (not PD unless s > 0), then L[i][j] = (S[i][j] - L[i][0] L[j][0] - ...) / L[j][j] for i > j.
// Every product and sum above is rounded on its own (__dmul_rn / __dadd_rn: no fma contraction), so tests/mc_model.py
// restates the counts bit for bit.  The counts are integers in shared memory: their order does not matter.
#pragma once
#include "gpk_internal.cuh"

#define GPK_MC_MAX_NB 64                 // the entropy-search limit (GPK_EP_MAX_NB)
#define GPK_MC_THREADS 256
#define GPK_MC_FT 32                     // draws f per chunk
#define GPK_MC_PC 64                     // innovations p per chunk
#define GPK_MC_TF 2                      // register tile of a thread: TF draws x TP innovations
#define GPK_MC_TP 4
#define GPK_MC_TAG 0x4D430001u
#define GPK_MC_NOISE_LAST 10000.0
// shared memory of gpk_mc_pmin_kernel: L (64 x 64), the F chunk and the funcs chunk (64 x FT each), the M chunk (64 x PC)
#define GPK_MC_SMEM ((GPK_MC_MAX_NB * GPK_MC_MAX_NB + 2 * GPK_MC_MAX_NB * GPK_MC_FT + GPK_MC_MAX_NB * GPK_MC_PC) * 8)

// status words of a pass: [0] factorisations that needed jitter, [1] candidates whose every rung failed
#define GPK_MC_STAT_JITTER 0
#define GPK_MC_STAT_NOT_PD 1

__global__ void gpk_mc_draws_kernel(unsigned long long seed, int nb, int nf, double* __restrict__ F) {
    const int nq = (nf + 1) / 2;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)nb * nq) return;
    const int k = (int)(t / nq), q = (int)(t - (long)k * nq);
    uint32_t w[4];
    gpk_philox4x32_10((uint32_t)q, (uint32_t)k, 0u, GPK_MC_TAG, (uint32_t)seed, (uint32_t)(seed >> 32), w);
    const double u1 = (double)(((((unsigned long long)w[1] << 32) | w[0]) >> 11) + 1ull) * 1.1102230246251565e-16;
    const double u2 = gpk_u01(w[2], w[3]);
    const double r = __dsqrt_rn(__dmul_rn(-2.0, log(u1)));
    double s, c;
    sincospi(__dmul_rn(2.0, u2), &s, &c);
    F[(size_t)k * nf + 2 * q] = __dmul_rn(r, c);
    if (2 * q + 1 < nf) F[(size_t)k * nf + 2 * q + 1] = __dmul_rn(r, s);
}

// One CTA per candidate c (see the header).  m_full (nb x np) replaces Mb + dm W when given (joint_pmin on caller
// operands; then sig must be NULL).  sig == NULL: A = Vb and M[a][p] = m_full[a][p] (or Mb_a).  var / sig: rows and
// rows x nb (the scoring pass's variance and the clipped covariance to zb).  Out (each may be NULL): value[c],
// pmin[c][nb], rung[c] (0: no jitter; -1: not PD); stat (2 ints, atomically incremented).
__global__ void __launch_bounds__(GPK_MC_THREADS) gpk_mc_pmin_kernel(
    const double* __restrict__ m_full, const double* __restrict__ Mb, const double* __restrict__ W, int np_,
    const double* __restrict__ Vb, int nb, const double* __restrict__ F, int nf, const double* __restrict__ var,
    const double* __restrict__ sig, double sn2, const double* __restrict__ lmb, double H, double* __restrict__ value,
    double* __restrict__ pmin, int* __restrict__ rung, int* __restrict__ stat)
{
    extern __shared__ double mc_sm[];
    double* L = mc_sm;                                        // nb x nb (row stride GPK_MC_MAX_NB)
    double* Fs = L + GPK_MC_MAX_NB * GPK_MC_MAX_NB;           // F chunk, nb x FT
    double* Fu = Fs + GPK_MC_MAX_NB * GPK_MC_FT;              // funcs chunk, nb x FT
    double* Ms = Fu + GPK_MC_MAX_NB * GPK_MC_FT;              // M chunk, nb x PC
    __shared__ double s_nc[GPK_MC_MAX_NB], s_dm[GPK_MC_MAX_NB], s_sg[GPK_MC_MAX_NB];
    __shared__ int cnt[GPK_MC_MAX_NB];
    __shared__ int s_fail;
    const long c = blockIdx.x;
    const int t = threadIdx.x;
    const int LD = GPK_MC_MAX_NB;

    if (t < nb) {
        cnt[t] = 0;
        if (sig != nullptr) {
            const double v = var[c];
            const double iv = __ddiv_rn(1.0, __dsub_rn(v, sn2));
            const double sg = sig[c * nb + t];
            const double nc = __dmul_rn(sg, iv);
            s_sg[t] = sg;
            s_nc[t] = nc;
            s_dm[t] = __dmul_rn(nc, __dsqrt_rn(__dadd_rn(v, 1e-10)));
        } else {
            s_sg[t] = 0.0;
            s_nc[t] = 0.0;
            s_dm[t] = 0.0;
        }
    }
    __syncthreads();

    // ---- the factorisation on the jitter ladder ----
    double noise = 0.0;
    int r = 0;
    for (;; ++r) {
        for (int x = t; x < nb * nb; x += blockDim.x) {
            const int a = x / nb, b = x - a * nb;
            if (b > a) continue;
            double s = Vb[x];
            if (sig != nullptr) s = __dadd_rn(s, -__dmul_rn(s_nc[a], s_sg[b]));
            if (a == b && r > 0) s = __dadd_rn(s, noise);
            L[a * LD + b] = s;
        }
        if (t == 0) s_fail = 0;
        __syncthreads();
        for (int j = 0; j < nb; ++j) {
            if (t == 0) {
                double s = L[j * LD + j];
                for (int m = 0; m < j; ++m) s = __dsub_rn(s, __dmul_rn(L[j * LD + m], L[j * LD + m]));
                if (!(s > 0.0)) s_fail = 1;
                L[j * LD + j] = __dsqrt_rn(s);
            }
            __syncthreads();
            if (s_fail) break;
            const double ljj = L[j * LD + j];
            for (int i = j + 1 + t; i < nb; i += blockDim.x) {
                double s = L[i * LD + j];
                for (int m = 0; m < j; ++m) s = __dsub_rn(s, __dmul_rn(L[i * LD + m], L[j * LD + m]));
                L[i * LD + j] = __ddiv_rn(s, ljj);
            }
            __syncthreads();
        }
        const bool failed = s_fail != 0;
        __syncthreads();
        if (!failed) break;
        // mc_part.py:37-43: 0 -> 1e-10, stop at 10000, otherwise * 10 (so the first retry is at 1e-9)
        if (noise == 0.0) noise = 1e-10;
        if (noise == GPK_MC_NOISE_LAST || r >= 32) {
            if (t == 0) {
                if (stat) atomicAdd(stat + GPK_MC_STAT_NOT_PD, 1);
                if (rung) rung[c] = -1;
                if (value) value[c] = NAN;
            }
            if (pmin)
                for (int a = t; a < nb; a += blockDim.x) pmin[c * nb + a] = NAN;
            return;
        }
        noise = __dmul_rn(noise, 10.0);
    }
    if (t == 0) {
        if (rung) rung[c] = r;
        if (r > 0 && stat) atomicAdd(stat + GPK_MC_STAT_JITTER, 1);
    }

    // ---- draws, innovations and the arg-min of every column ----
    const int fg = t & 15, pg = t >> 4;                       // this thread's tile: draws fg*TF.., innovations pg*TP..
    for (int f0 = 0; f0 < nf; f0 += GPK_MC_FT) {
        const int fc = min(GPK_MC_FT, nf - f0);
        for (int x = t; x < nb * GPK_MC_FT; x += blockDim.x) {
            const int k = x / GPK_MC_FT, f = x - k * GPK_MC_FT;
            Fs[x] = f < fc ? F[(size_t)k * nf + f0 + f] : 0.0;
        }
        __syncthreads();
        for (int x = t; x < nb * GPK_MC_FT; x += blockDim.x) {
            const int a = x / GPK_MC_FT, f = x - a * GPK_MC_FT;
            double s = 0.0;
            for (int k = 0; k <= a; ++k) s = __dadd_rn(s, __dmul_rn(L[a * LD + k], Fs[k * GPK_MC_FT + f]));
            Fu[x] = s;
        }
        for (int p0 = 0; p0 < np_; p0 += GPK_MC_PC) {
            const int pc = min(GPK_MC_PC, np_ - p0);
            if (f0 == 0 || np_ > GPK_MC_PC) {                 // M is built once when it fits in one chunk
                for (int x = t; x < nb * GPK_MC_PC; x += blockDim.x) {
                    const int a = x / GPK_MC_PC, p = x - a * GPK_MC_PC;
                    double mv = 0.0;
                    if (p < pc)
                        mv = m_full ? m_full[(size_t)a * np_ + p0 + p]
                                    : __dadd_rn(Mb[a], __dmul_rn(s_dm[a], W[p0 + p]));
                    Ms[x] = mv;
                }
            }
            __syncthreads();
            if (fg * GPK_MC_TF < fc && pg * GPK_MC_TP < pc) {
                const double* fu = Fu + fg * GPK_MC_TF;
                const double* ms = Ms + pg * GPK_MC_TP;
                double best[GPK_MC_TF][GPK_MC_TP];
                int arg[GPK_MC_TF][GPK_MC_TP];
#pragma unroll
                for (int i = 0; i < GPK_MC_TF; ++i)
#pragma unroll
                    for (int j = 0; j < GPK_MC_TP; ++j) {
                        best[i][j] = __dadd_rn(ms[j], fu[i]);
                        arg[i][j] = 0;
                    }
                for (int a = 1; a < nb; ++a) {
                    double u[GPK_MC_TF], mm[GPK_MC_TP];
#pragma unroll
                    for (int i = 0; i < GPK_MC_TF; ++i) u[i] = fu[a * GPK_MC_FT + i];
#pragma unroll
                    for (int j = 0; j < GPK_MC_TP; ++j) mm[j] = ms[a * GPK_MC_PC + j];
#pragma unroll
                    for (int i = 0; i < GPK_MC_TF; ++i)
#pragma unroll
                        for (int j = 0; j < GPK_MC_TP; ++j) {
                            const double v = __dadd_rn(mm[j], u[i]);
                            if (v < best[i][j]) {
                                best[i][j] = v;
                                arg[i][j] = a;
                            }
                        }
                }
#pragma unroll
                for (int i = 0; i < GPK_MC_TF; ++i)
#pragma unroll
                    for (int j = 0; j < GPK_MC_TP; ++j)
                        if (fg * GPK_MC_TF + i < fc && pg * GPK_MC_TP + j < pc) atomicAdd(&cnt[arg[i][j]], 1);
            }
            __syncthreads();
        }
    }

    // ---- p_min, its clamp and the value ----
    const double total = (double)nf * (double)np_;
    if (t < nb) {
        double p = __ddiv_rn((double)cnt[t], total);
        if (p < 1e-70) p = 1e-70;
        s_sg[t] = p;
        if (pmin) pmin[c * nb + t] = p;
    }
    __syncthreads();
    if (t == 0 && value) {
        double acc = 0.0;
        for (int a = 0; a < nb; ++a) acc = __dadd_rn(acc, __dmul_rn(s_sg[a], __dadd_rn(log(s_sg[a]), lmb[a])));
        const double v = __dadd_rn(acc, H);
        value[c] = (isnan(v) || v == INFINITY) ? -1.7976931348623157e308 : v;
    }
}
