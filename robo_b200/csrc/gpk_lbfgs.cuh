// gpk_lbfgs.cuh — device-resident multi-start bounded L-BFGS for gpk_maximize_lbfgs*: the maximizer of
// robo/maximizers/scipy_optimizer.py (scipy.optimize.minimize(method='L-BFGS-B') from n_restarts starts on the
// reference's single-point objective, scipy_optimizer.py:39-49) and of robo/util/posterior_optimization.py.
//
// Every start runs independently; the starts share only the scoring pass.  A round scores, for every start still
// active, its trial point and the D forward-difference neighbours of it (rows a (D + 1) + k of the batch, a = the
// start's position in the active list, k = 0 the trial point, k = 1 + j the neighbour in coordinate j), so an accepted
// trial already has its gradient.  The first round scores the starts, clipped into the box.
//
// Energy of a scored row: -acq (acquisitions, information gain), mu (GPK_LB_MU) or mu + sqrt(v) (GPK_LB_MU_STD); a
// value that is not finite becomes DBL_MAX (the reference's wrapper maps +-inf; a NaN value is mapped too, so that it
// cannot enter the curvature pairs).
//
// Gradient (scipy approx_derivative, method='2-point'): h_j = 2^-26 sign+(x_j) max(1, |x_j|) (sqrt(DBL_EPSILON) is 2^-26,
// sign+(0) = +1), negated when x_j + h_j leaves [lower_j, upper_j]; the neighbour is clip(x_j + h_j) and
// g_j = (e_j - e) / ((x_j + h_j) - x_j).
//
// Iteration (projected L-BFGS; not L-BFGS-B's Cauchy point, subspace minimisation and More-Thuente search):
//   free set: j is fixed when x_j = lower_j and g_j > 0, or x_j = upper_j and g_j < 0; q = g on the free set, 0 else
//   direction: the two-loop recursion over the last k <= maxcor pairs (oldest first in the second loop),
//              H0 = gamma = s'y / y'y of the newest pair; k = 0: d = -q.  d = -r on the free set, 0 on the fixed one.
//              If g'd < 0 does not hold the memory is cleared and d = -q.
//   step:      alpha0 = min(1, 1 / ||d||_2) while nit = 0, 1 afterwards; trial P(x + alpha d), P = clip to the box.
//              Accept when e(trial) <= e + 1e-4 g'(trial - x); otherwise alpha *= 0.5, at most 20 times, then the
//              start stops with GPK_LB_ABNORMAL (scipy's ABNORMAL_TERMINATION_IN_LNSRCH).
//   pair:      s = x+ - x, y = g+ - g, stored when s'y > DBL_EPSILON y'y (scipy's rule), with rho = 1 / s'y.
//   stopping:  after the first round and after every accepted step, in this order: ||P(x - g) - x||_inf <= pgtol
//              (GPK_LB_PGTOL), (e_old - e) / max(|e_old|, |e|, 1) <= ftol (GPK_LB_FTOL, not after the first round),
//              nit >= maxiter (GPK_LB_MAXITER), nfev >= maxfun (GPK_LB_MAXFUN; also checked before a backtrack).  A
//              start whose first energy is DBL_MAX stops at once (GPK_LB_INVALID).
//
// Rounding: every product, sum, difference, quotient and square root that reaches a result is rounded explicitly
// (__dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn / __dsqrt_rn: no fma contraction).  A dot product over the D <= 64
// coordinates is p_l = fl(fl(a_l b_l) + fl(a_{l+32} b_{l+32})) per lane l (missing coordinates are 0), then
// p += shfl_xor(p, o) for o = 16, 8, 4, 2, 1.  tests/lbfgs_model.py restates all of it bit for bit.
#pragma once
#include "gpk_internal.cuh"

// GPK_LB_MAX_D (gpk.h) = 64: two coordinates per lane of the step kernel's warp
#define GPK_LB_MAX_COR 32
#define GPK_LB_MAX_STARTS (1 << 20)
#define GPK_LB_MAX_BACKTRACK 20
#define GPK_LB_DBL_MAX 1.7976931348623157e308
#define GPK_LB_DBL_EPS 2.220446049250313e-16

// energy of a scored row
enum { GPK_LB_NEG = 0, GPK_LB_MU = 1, GPK_LB_MU_STD = 2 };
// per-start status while running; the final ones are gpk.h's gpk_lb_status
#define GPK_LB_RUNNING (-1)

struct LBStart {
    double f;                             // energy of the accepted iterate
    double alpha;                         // step of the current trial
    double gamma;                         // s'y / y'y of the newest stored pair
    long long nfev;                       // rows scored for this start
    int nit;                              // accepted steps
    int status;                           // GPK_LB_RUNNING or the final status
    int phase;                            // 0: the trial is the start itself; 1: line search
    int nback;                            // halvings of alpha in the current line search
    int k;                                // stored pairs (<= maxcor)
    int head;                             // ring slot the next pair goes to
};

struct LBStatus {
    int n_active;                         // starts still running after the round
    int rows;                             // rows of the next scoring pass: n_active (d + 1)
    unsigned int done;                    // blocks of the step kernel finished (reset by the last one)
    int reserved;
};

__device__ __forceinline__ double gpk_lb_energy(int obj, const double* __restrict__ v1, const double* __restrict__ v2,
                                                long r) {
    double e;
    if (obj == GPK_LB_MU) e = v1[r];
    else if (obj == GPK_LB_MU_STD) e = __dadd_rn(v1[r], __dsqrt_rn(v2[r]));
    else e = -v1[r];
    return isfinite(e) ? e : GPK_LB_DBL_MAX;
}

// forward-difference step of coordinate x in [lo, up] (before the (x + h) - x correction)
__device__ __forceinline__ double gpk_lb_h(double x, double lo, double up) {
    double h = __dmul_rn(x >= 0.0 ? 1.4901161193847656e-08 : -1.4901161193847656e-08, fmax(1.0, fabs(x)));
    const double xh = __dadd_rn(x, h);
    if (xh > up || xh < lo) h = -h;
    return h;
}

__device__ __forceinline__ double gpk_lb_clip(double v, double lo, double up) { return fmin(fmax(v, lo), up); }

// the fixed-order dot product of the header comment; every lane returns the same value
__device__ __forceinline__ double gpk_lb_dot(double a0, double b0, double a1, double b1) {
    double p = __dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) p = __dadd_rn(p, __shfl_xor_sync(0xffffffffu, p, o));
    return p;
}

__device__ __forceinline__ double gpk_lb_max(double p) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) p = fmax(p, __shfl_xor_sync(0xffffffffu, p, o));
    return p;
}

// one thread per row: the trial point of active start act[a] (XT, already in the box) and its d neighbours
// lim = [lower (d), upper (d)]
__global__ void gpk_lb_stencil_kernel(int d, long rows, const int* __restrict__ act, const double* __restrict__ lim,
                                      const double* __restrict__ XT, double* __restrict__ Xb)
{
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= rows) return;
    const long a = t / (d + 1);
    const int k = (int)(t - a * (d + 1));
    const double* x = XT + (size_t)act[a] * d;
    double* out = Xb + (size_t)t * d;
    for (int j = 0; j < d; ++j) {
        double v = x[j];
        if (j == k - 1) v = gpk_lb_clip(__dadd_rn(v, gpk_lb_h(v, lim[j], lim[d + j])), lim[j], lim[d + j]);
        out[j] = v;
    }
}

// One warp per active start (block b serves act_in[b]; its rows start at b (d + 1)).  Lane l owns coordinates l and
// l + 32.  The stored pairs of the start are staged in shared memory, oldest first: S (maxcor x d), Y (maxcor x d),
// rho (maxcor), alpha (maxcor).  The last block to finish compacts the running starts into act_out in start order and
// writes the status record.
__global__ void __launch_bounds__(32) gpk_lb_step_kernel(
    int d, int R, int maxcor, int maxiter, long long maxfun, double ftol, double pgtol, int obj,
    const double* __restrict__ v1, const double* __restrict__ v2, const double* __restrict__ lim,
    const int* __restrict__ act_in, int* __restrict__ act_out, int* __restrict__ flag, LBStart* __restrict__ sts,
    double* __restrict__ X, double* __restrict__ G, double* __restrict__ Dir, double* __restrict__ XT,
    double* __restrict__ S, double* __restrict__ Y, double* __restrict__ RHO, LBStatus* __restrict__ st)
{
    extern __shared__ double sm[];
    double* sS = sm;
    double* sY = sS + (size_t)maxcor * d;
    double* sR = sY + (size_t)maxcor * d;
    double* sA = sR + maxcor;
    __shared__ bool last;
    const int lane = threadIdx.x;
    const int s = act_in[blockIdx.x];
    const long row0 = (long)blockIdx.x * (d + 1);
    const int j0 = lane, j1 = lane + 32;
    const bool in0 = j0 < d, in1 = j1 < d;
    const double lo0 = in0 ? lim[j0] : 0.0, up0 = in0 ? lim[d + j0] : 0.0;
    const double lo1 = in1 ? lim[j1] : 0.0, up1 = in1 ? lim[d + j1] : 0.0;
    double* xs = X + (size_t)s * d;
    double* gs = G + (size_t)s * d;
    double* ds = Dir + (size_t)s * d;
    double* ts = XT + (size_t)s * d;
    LBStart p = sts[s];

    // the scored trial and its forward-difference gradient
    const double ft = gpk_lb_energy(obj, v1, v2, row0);
    const double xt0 = in0 ? ts[j0] : 0.0, xt1 = in1 ? ts[j1] : 0.0;
    double gt0 = 0.0, gt1 = 0.0;
    if (in0) {
        const double hh = __dsub_rn(__dadd_rn(xt0, gpk_lb_h(xt0, lo0, up0)), xt0);
        gt0 = __ddiv_rn(__dsub_rn(gpk_lb_energy(obj, v1, v2, row0 + 1 + j0), ft), hh);
    }
    if (in1) {
        const double hh = __dsub_rn(__dadd_rn(xt1, gpk_lb_h(xt1, lo1, up1)), xt1);
        gt1 = __ddiv_rn(__dsub_rn(gpk_lb_energy(obj, v1, v2, row0 + 1 + j1), ft), hh);
    }
    p.nfev += d + 1;

    double x0 = 0.0, x1 = 0.0, g0 = 0.0, g1 = 0.0, f_old = 0.0;
    bool moved = false, check_ftol = false;
    int stop = GPK_LB_RUNNING;
    if (p.phase == 0) {
        x0 = xt0; x1 = xt1; g0 = gt0; g1 = gt1;
        p.f = ft;
        p.phase = 1;
        if (ft == GPK_LB_DBL_MAX) stop = GPK_LB_INVALID;
        else moved = true;
    } else {
        x0 = in0 ? xs[j0] : 0.0; x1 = in1 ? xs[j1] : 0.0;
        g0 = in0 ? gs[j0] : 0.0; g1 = in1 ? gs[j1] : 0.0;
        const double s0 = __dsub_rn(xt0, x0), s1 = __dsub_rn(xt1, x1);
        const double gs_ = gpk_lb_dot(g0, s0, g1, s1);
        if (ft <= __dadd_rn(p.f, __dmul_rn(1e-4, gs_))) {
            const double y0 = __dsub_rn(gt0, g0), y1 = __dsub_rn(gt1, g1);
            const double sy = gpk_lb_dot(s0, y0, s1, y1);
            const double yy = gpk_lb_dot(y0, y0, y1, y1);
            if (sy > __dmul_rn(GPK_LB_DBL_EPS, yy)) {
                double* Sp = S + ((size_t)s * maxcor + p.head) * d;
                double* Yp = Y + ((size_t)s * maxcor + p.head) * d;
                if (in0) { Sp[j0] = s0; Yp[j0] = y0; }
                if (in1) { Sp[j1] = s1; Yp[j1] = y1; }
                if (lane == 0) RHO[(size_t)s * maxcor + p.head] = __ddiv_rn(1.0, sy);
                p.gamma = __ddiv_rn(sy, yy);
                p.head = (p.head + 1) % maxcor;
                p.k = min(p.k + 1, maxcor);
            }
            f_old = p.f;
            x0 = xt0; x1 = xt1; g0 = gt0; g1 = gt1;
            p.f = ft;
            p.nit += 1;
            moved = check_ftol = true;
        } else if (p.nback == GPK_LB_MAX_BACKTRACK) {
            stop = GPK_LB_ABNORMAL;
        } else if (p.nfev >= maxfun) {
            stop = GPK_LB_MAXFUN;
        } else {
            p.nback += 1;
            p.alpha = __dmul_rn(p.alpha, 0.5);
            if (in0) ts[j0] = gpk_lb_clip(__dadd_rn(x0, __dmul_rn(p.alpha, ds[j0])), lo0, up0);
            if (in1) ts[j1] = gpk_lb_clip(__dadd_rn(x1, __dmul_rn(p.alpha, ds[j1])), lo1, up1);
        }
    }

    if (moved) {
        if (in0) { xs[j0] = x0; gs[j0] = g0; }
        if (in1) { xs[j1] = x1; gs[j1] = g1; }
        const double pg = gpk_lb_max(fmax(in0 ? fabs(__dsub_rn(gpk_lb_clip(__dsub_rn(x0, g0), lo0, up0), x0)) : 0.0,
                                          in1 ? fabs(__dsub_rn(gpk_lb_clip(__dsub_rn(x1, g1), lo1, up1), x1)) : 0.0));
        if (pg <= pgtol) stop = GPK_LB_PGTOL;
        else if (check_ftol && __ddiv_rn(__dsub_rn(f_old, p.f), fmax(fmax(fabs(f_old), fabs(p.f)), 1.0)) <= ftol)
            stop = GPK_LB_FTOL;
        else if (p.nit >= maxiter) stop = GPK_LB_MAXITER;
        else if (p.nfev >= maxfun) stop = GPK_LB_MAXFUN;
        else {
            const bool fr0 = in0 && !((x0 == lo0 && g0 > 0.0) || (x0 == up0 && g0 < 0.0));
            const bool fr1 = in1 && !((x1 == lo1 && g1 > 0.0) || (x1 == up1 && g1 < 0.0));
            double d0 = fr0 ? -g0 : 0.0, d1 = fr1 ? -g1 : 0.0;
            if (p.k > 0) {
                const int k = p.k;
                for (int i = 0; i < k; ++i) {
                    const int slot = (p.head - k + i + maxcor) % maxcor;
                    const double* Sp = S + ((size_t)s * maxcor + slot) * d;
                    const double* Yp = Y + ((size_t)s * maxcor + slot) * d;
                    for (int j = lane; j < d; j += 32) { sS[i * d + j] = Sp[j]; sY[i * d + j] = Yp[j]; }
                    if (lane == 0) sR[i] = RHO[(size_t)s * maxcor + slot];
                }
                __syncwarp();
                double q0 = fr0 ? g0 : 0.0, q1 = fr1 ? g1 : 0.0;
                for (int i = k - 1; i >= 0; --i) {
                    const double a = __dmul_rn(sR[i], gpk_lb_dot(in0 ? sS[i * d + j0] : 0.0, q0,
                                                                 in1 ? sS[i * d + j1] : 0.0, q1));
                    if (lane == 0) sA[i] = a;
                    if (fr0) q0 = __dsub_rn(q0, __dmul_rn(a, sY[i * d + j0]));
                    if (fr1) q1 = __dsub_rn(q1, __dmul_rn(a, sY[i * d + j1]));
                }
                __syncwarp();
                double r0 = fr0 ? __dmul_rn(p.gamma, q0) : 0.0, r1 = fr1 ? __dmul_rn(p.gamma, q1) : 0.0;
                for (int i = 0; i < k; ++i) {
                    const double b = __dmul_rn(sR[i], gpk_lb_dot(in0 ? sY[i * d + j0] : 0.0, r0,
                                                                 in1 ? sY[i * d + j1] : 0.0, r1));
                    const double c = __dsub_rn(sA[i], b);
                    if (fr0) r0 = __dadd_rn(r0, __dmul_rn(sS[i * d + j0], c));
                    if (fr1) r1 = __dadd_rn(r1, __dmul_rn(sS[i * d + j1], c));
                }
                d0 = fr0 ? -r0 : 0.0;
                d1 = fr1 ? -r1 : 0.0;
                if (!(gpk_lb_dot(g0, d0, g1, d1) < 0.0)) {
                    p.k = 0;
                    p.head = 0;
                    d0 = fr0 ? -g0 : 0.0;
                    d1 = fr1 ? -g1 : 0.0;
                }
            }
            p.alpha = p.nit == 0 ? fmin(1.0, __ddiv_rn(1.0, __dsqrt_rn(gpk_lb_dot(d0, d0, d1, d1)))) : 1.0;
            p.nback = 0;
            if (in0) { ds[j0] = d0; ts[j0] = gpk_lb_clip(__dadd_rn(x0, __dmul_rn(p.alpha, d0)), lo0, up0); }
            if (in1) { ds[j1] = d1; ts[j1] = gpk_lb_clip(__dadd_rn(x1, __dmul_rn(p.alpha, d1)), lo1, up1); }
        }
    }
    if (stop != GPK_LB_RUNNING) {
        p.status = stop;
        if (lane == 0) flag[s] = 0;
    }
    if (lane == 0) sts[s] = p;

    // the last block compacts the running starts (start order) and writes the status record
    __threadfence();
    __syncwarp();
    if (lane == 0) last = atomicAdd(&st->done, 1u) == gridDim.x - 1;
    __syncwarp();
    if (!last) return;
    __threadfence();
    int base = 0;
    for (int c = 0; c < R; c += 32) {
        const int i = c + lane;
        const int fl = i < R ? __ldcg(flag + i) : 0;
        const unsigned bal = __ballot_sync(0xffffffffu, fl != 0);
        if (fl) act_out[base + __popc(bal & ((1u << lane) - 1u))] = i;
        base += __popc(bal);
    }
    if (lane == 0) {
        st->n_active = base;
        st->rows = base * (d + 1);
        st->done = 0;
    }
}
