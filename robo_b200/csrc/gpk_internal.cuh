// gpk_internal.cuh — shared device helpers and structs (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/gpk.h"

#define GPK_TILE 128          // block size of every blocked algorithm (rows per tile)
#define GPK_EPS 2.220446049250313e-16

// The kernel's single-column factor: k *= gpk_factor_value(f, z, z'), z = column `axis` of each input row.  The kind
// decides everything else: the environment factor (gpk_set_env_factor) c0 + c1 z z' on the input-bounds-scaled
// coordinate, the task factor (gpk_set_task_factor) K[t * n_tasks + t'] on the raw coordinate (never scaled; gpk_fit
// refuses input bounds with it).  A kernel has at most one factor, so one descriptor carries either.
enum { GPK_FACTOR_NONE = 0, GPK_FACTOR_ENV = 1, GPK_FACTOR_TASK = 2 };
struct KFactor {
    int kind;                       // GPK_FACTOR_*; NONE: every other field is zero
    int axis;                       // the input column z is read from
    int n_tasks;                    // task: K is n_tasks x n_tasks, row-major
    double c0, c1;                  // environment: c0 = exp(log_a), c1 = exp(log_b)
    double K[GPK_MAX_TASKS * GPK_MAX_TASKS];
};

// Kernel specification passed by value to the covariance-building kernels.
// k(x,x') = amp * prod_g f( sum_{t in g} (x[axis_t]-x'[axis_t])^2 * inv_metric_t ) [* the factor]
struct KSpec {
    int family;
    int n_terms;
    double amp;
    int axis[GPK_MAX_TERMS];
    int last[GPK_MAX_TERMS];        // 1 if term t closes its product group
    double inv_metric[GPK_MAX_TERMS];
    double scale[GPK_MAX_TERMS];    // sqrt(c_f / metric_t): coordinates pre-scaled so that q = sum (s - s')^2 is the
                                    // radial argument directly (c_f = 5 Matern-5/2, 3 Matern-3/2, 1/2 ExpSquared)
    KFactor factor;                 // last, so the kernels that never read it see the same parameter layout
};

// The environment factor of Fabolas, restated from arXiv:1605.07079 (not checked against the george fork that defines
// BayesianLinearRegressionKernel): c0 + c1 z z', with c0 = exp(log_a), c1 = exp(log_b).  Its derivatives are
// d/dlog_a = c0, d/dlog_b = c1 z z', d/dz = c1 z' (gpk_env_dz).  Test restatement: tests/env_kernel_model.py (env_value).
__device__ __forceinline__ double gpk_env(double c0, double c1, double z, double z2) { return fma(c1 * z, z2, c0); }
__device__ __forceinline__ double gpk_env_dz(double c1, double z2) { return c1 * z2; }

// The task factor of MTBO, restated from Swersky, Snoek, Adams (NIPS 2013) and the reference's call sites (not checked
// against the george fork that defines TaskKernel): K_t = L L^T, L lower triangular, L_pq = exp(theta[p (p + 1) / 2 + q])
// packed row by row; K_t[a][b] = sum_{q <= min(a, b)} L_aq L_bq, multiplied and added in ascending q with no fused
// multiply-add.  Host and device share this definition; the test restatement is tests/task_kernel_model.py
// (task_value).  Kt: n x n row-major.
__host__ __device__ inline void gpk_task_matrix(int n, const double* theta, double* Kt) {
    for (int a = 0; a < n; ++a)
        for (int b = 0; b <= a; ++b) {
            double s = 0.0;
            for (int q = 0; q <= b; ++q) {
#ifdef __CUDA_ARCH__
                s = __dadd_rn(s, __dmul_rn(exp(theta[a * (a + 1) / 2 + q]), exp(theta[b * (b + 1) / 2 + q])));
#else
                s = s + exp(theta[a * (a + 1) / 2 + q]) * exp(theta[b * (b + 1) / 2 + q]);   // x86-64: no contraction
#endif
            }
            Kt[a * n + b] = s;
            Kt[b * n + a] = s;
        }
}

// the task a coordinate names: an integer in [0, n), otherwise -1 (NaN included)
__host__ __device__ __forceinline__ int gpk_task_index(double t, int n) {
    return (t >= 0.0 && t < (double)n && t == floor(t)) ? (int)t : -1;
}

// The factor's coordinate in one row of raw inputs: row[axis], scaled (x - lower) / (upper - lower) when bounds are
// given and the factor is the environment factor.  FK here and in gpk_factor_value: the kind when the caller's
// instance fixes it at compile time (the gradient kernels), so the other kind's code is compiled out; -1: f.kind.
template <int FK = -1>
__device__ __forceinline__ double gpk_factor_coord(const KFactor& f, const double* row, const double* lower,
                                                   const double* upper) {
    double v = row[f.axis];
    if ((FK < 0 ? f.kind : FK) == GPK_FACTOR_ENV && lower != nullptr)
        v = (v - lower[f.axis]) / (upper[f.axis] - lower[f.axis]);
    return v;
}

// The factor's value at coordinates z, z' (kind != NONE): gpk_env, or K_t[z][z'] (NaN when either is not a task)
template <int FK = -1>
__device__ __forceinline__ double gpk_factor_value(const KFactor& f, double z, double z2) {
    if ((FK < 0 ? f.kind : FK) == GPK_FACTOR_ENV) return gpk_env(f.c0, f.c1, z, z2);
    const int a = gpk_task_index(z, f.n_tasks), b = gpk_task_index(z2, f.n_tasks);
    return (a < 0 || b < 0) ? __longlong_as_double(0x7ff8000000000000LL) : f.K[a * f.n_tasks + b];
}

// The factor's values from its log-parameters p (kind, axis and n_tasks already set): environment (log_a, log_b),
// task the n_tasks (n_tasks + 1) / 2 packed entries of gpk_task_matrix.  Host or device exp, whichever side calls it.
__host__ __device__ inline void gpk_factor_build(KFactor& f, const double* p) {
    if (f.kind == GPK_FACTOR_ENV) { f.c0 = exp(p[0]); f.c1 = exp(p[1]); }
    else if (f.kind == GPK_FACTOR_TASK) gpk_task_matrix(f.n_tasks, p, f.K);
}

// f as a function of q = c_f * r2 (pre-scaled coordinates, gpk_cov_tma_kernel)
__device__ __forceinline__ double gpk_radial_q(int family, double q) {
    if (family == GPK_MATERN52) {
        double r = sqrt(q);
        return fma(q, 1.0 / 3.0, 1.0 + r) * exp(-r);           // 1 + r + 5 r2 / 3
    } else if (family == GPK_EXPSQUARED) {
        return exp(-q);
    } else {
        double r = sqrt(q);
        return (1.0 + r) * exp(-r);
    }
}

// f(r2) for the radial families (oracle/george_oracle.py: Matern52Kernel._f etc.).
__device__ __forceinline__ double gpk_radial(int family, double r2) {
    if (family == GPK_MATERN52) {
        double r = sqrt(5.0 * r2);
        return (1.0 + r + 5.0 * r2 / 3.0) * exp(-r);
    } else if (family == GPK_EXPSQUARED) {
        return exp(-0.5 * r2);
    } else {
        double r = sqrt(3.0 * r2);
        return (1.0 + r) * exp(-r);
    }
}

// d f / d r2 (george_oracle.py: _dfdr2)
__device__ __forceinline__ double gpk_radial_dr2(int family, double r2) {
    if (family == GPK_MATERN52) {
        double r = sqrt(5.0 * r2);
        return -(5.0 / 6.0) * (1.0 + r) * exp(-r);
    } else if (family == GPK_EXPSQUARED) {
        return -0.5 * exp(-0.5 * r2);
    } else {
        double r = sqrt(3.0 * r2);
        return -1.5 * exp(-r);
    }
}

// d log f / d r2 (ratio f'/f in closed form: no 0/0 when f underflows)
__device__ __forceinline__ double gpk_radial_dlog(int family, double r2) {
    if (family == GPK_MATERN52) {
        double r = sqrt(5.0 * r2);
        return -(5.0 / 6.0) * (1.0 + r) / (1.0 + r + 5.0 * r2 / 3.0);
    } else if (family == GPK_EXPSQUARED) {
        return -0.5;
    } else {
        double r = sqrt(3.0 * r2);
        return -1.5 / (1.0 + r);
    }
}

// ---- standard normal helpers (scipy.special.ndtr / log_ndtr / norm.pdf restated) -------
__device__ __forceinline__ double gpk_ndtr(double z) {
    return 0.5 * erfc(-z * 0.70710678118654752440);
}
__device__ __forceinline__ double gpk_norm_pdf(double z) {
    return exp(-0.5 * z * z) * 0.39894228040143267794;       // 1/sqrt(2 pi)
}
__device__ __forceinline__ double gpk_norm_logpdf(double z) {
    return -0.5 * z * z - 0.91893853320467274178;             // log sqrt(2 pi)
}
__device__ __forceinline__ double gpk_log_ndtr(double z) {
    double t = z * 0.70710678118654752440;
    if (z < -1.0) return log(erfcx(-t) * 0.5) - t * t;
    return log1p(-0.5 * erfc(t));
}

// Acquisition closed forms on (mu, var); var already clipped/un-normalised.
// kind: gpk_acq_kind.  Mirrors ei.py:70-78, log_ei.py:72-120, pi.py:61-63, lcb.py:65.
__device__ __forceinline__ double gpk_acq_value(int kind, double m, double v, double eta, double par) {
    double s = sqrt(v);
    if (kind == GPK_ACQ_EI) {
        double z = (eta - m - par) / s;
        if (z < -30.0) {
            // deep lower tail: z Phi(z) + phi(z) = phi(z) (1 - |z| R(|z|)), R = Mills ratio
            // = sqrt(pi/2) erfcx(|z|/sqrt 2).  Same value as the direct form (both lose ~z^2 ulp to
            // cancellation) but the sign is decided in the normal range, so EI never turns negative
            // when phi and Phi go subnormal (|z| > 37.6), where the reference's scipy result is >= 0.
            double az = -z;
            double bracket = 1.0 - az * 1.25331413731550025121 * erfcx(az * 0.70710678118654752440);
            return s * (gpk_norm_pdf(z) * bracket);
        }
        return s * (z * gpk_ndtr(z) + gpk_norm_pdf(z));
    } else if (kind == GPK_ACQ_PI) {
        return gpk_ndtr((eta - m - par) / s);
    } else if (kind == GPK_ACQ_LCB) {
        return -(m - par * s);
    } else if (kind == GPK_ACQ_LOG_EI) {
        double f_min = eta - par;
        double z = (f_min - m) / s;
        const double ninf = -INFINITY;
        if (fabs(f_min - m) == 0.0) {                       // log_ei.py:85-89
            return (s > 0.0) ? log(s) + gpk_norm_logpdf(z) : ninf;
        } else if (s == 0.0) {                              // log_ei.py:92-96
            return (m < f_min) ? log(f_min - m) : ninf;
        } else {
            double b = log(s) + gpk_norm_logpdf(z);         // log_ei.py:99
            if (f_min > m) {                                // log_ei.py:101-107
                double a = log(f_min - m) + gpk_log_ndtr(z);
                return fmax(a, b) + log(1.0 + exp(-fabs(b - a)));
            } else {                                        // log_ei.py:114-120
                double a = log(m - f_min) + gpk_log_ndtr(z);
                if (a >= b) return ninf;
                return b + log(1.0 - exp(a - b));
            }
        }
    }
    return 0.0;
}

// numpy.argmax ordering: NaN beats everything, then larger value, then lower index.
__device__ __forceinline__ bool gpk_better(double va, long long ia, double vb, long long ib) {
    if (ib < 0) return ia >= 0;
    if (ia < 0) return false;
    bool na = isnan(va), nb = isnan(vb);
    if (na || nb) {
        if (na && nb) return ia < ib;
        return na;
    }
    if (va > vb) return true;
    if (va < vb) return false;
    return ia < ib;
}

struct BestPair { double val; long long idx; };

// warp arg-max: every lane ends with the warp's best pair
__device__ __forceinline__ void gpk_warp_best(double& val, long long& idx) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        double ov = __shfl_xor_sync(0xffffffffu, val, off);
        long long oi = __shfl_xor_sync(0xffffffffu, idx, off);
        if (gpk_better(ov, oi, val, idx)) { val = ov; idx = oi; }
    }
}

// block arg-max over NW warps: thread 0 ends with the block's best pair.  Every thread of the block must call it.
template <int NW>
__device__ __forceinline__ void gpk_block_best(double& val, long long& idx) {
    gpk_warp_best(val, idx);
    __shared__ double sv[NW];
    __shared__ long long si[NW];
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = val; si[threadIdx.x >> 5] = idx; }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < NW; ++w)
            if (gpk_better(sv[w], si[w], val, idx)) { val = sv[w]; idx = si[w]; }
}

// What a scoring kernel writes, shared by the GP epilogue and every surrogate's scoring kernel
struct ScoreOut {
    long base;                  // global index of the launch's candidate 0 (arg-max)
    int acq_kind; double eta, par;
    double* out_mu; double* out_var; double* out_acq;    // launch-local device arrays, may be NULL
    BestPair* block_best;       // one per block
    unsigned long long* n_negative;
};

// Candidate c's outputs: mu and var and, with an acquisition, its value, the negative-EI count and the pair (val, idx)
// the arg-max starts from.  zero_std_ei: EI is 0 at zero variance instead of gpk_acq_value's (the random forest's rule).
__device__ __forceinline__ void gpk_score_emit(const ScoreOut& o, long c, double mu, double var, double& val,
                                               long long& idx, bool zero_std_ei = false) {
    if (o.out_mu) o.out_mu[c] = mu;
    if (o.out_var) o.out_var[c] = var;
    if (o.acq_kind != GPK_ACQ_NONE) {
        val = (zero_std_ei && o.acq_kind == GPK_ACQ_EI && var == 0.0) ? 0.0 : gpk_acq_value(o.acq_kind, mu, var, o.eta, o.par);
        if (o.out_acq) o.out_acq[c] = val;
        if (o.acq_kind == GPK_ACQ_EI && val < 0.0 && o.n_negative) atomicAdd(o.n_negative, 1ULL);
        idx = o.base + c;
    }
}
