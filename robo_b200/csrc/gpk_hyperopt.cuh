// gpk_hyperopt.cuh — device-resident hyper-parameter optimisation for gpk_optimize_hypers: GaussianProcess.optimize
// (gaussian_process.py:193-219), i.e. scipy.optimize.minimize(nll, p0, method='L-BFGS-B') without a gradient, so that
// scipy differentiates nll by forward differences.
//
// Objective of one theta (GaussianProcess.nll restated on gpk_hy_eval's two parts ll, lp, gpk_hyper.cuh):
//   no prior: f = -ll when ll is finite; with a prior: v = fl(ll + lp), f = -v when v is finite; 1e25 otherwise (|theta_j|
//   > 20, a pivot that is not > 0, a non-finite result, lp = +inf of the horseshoe at 0).
//
// Round: one launch of D + 1 CTAs (D = dim <= GPK_HYPER_MAX_DIM, one wave at one CTA per SM).  CTA 0 scores the trial
// point xt, CTA 1 + j its forward-difference neighbour xt + h_j e_j (scipy approx_derivative, 2-point, abs_step = eps):
//   h_j = eps, or sqrt(DBL_EPSILON) sign+(x_j) max(1, |x_j|) where fl(fl(x_j + eps) - x_j) == 0 (sign+(0) = +1);
//   g_j = fl(fl(f_j - f_0) / fl(fl(xt_j + h_j) - xt_j)).
// Every CTA counts D + 1 evaluations towards nfev, as scipy's ScalarFunction does.  The last CTA to finish takes the
// ticket and runs the optimiser's update in its first warp (lane l owns coordinates l, l + 32, l + 64), which writes the
// next trial point and the status record.  Once the status is final a round returns at once.
//
// Update: L-BFGS-B (Byrd, Lu, Nocedal & Zhu 1995; Zhu, Byrd, Lu & Nocedal 1997, v3.0 of Morales & Nocedal 2011) as scipy
// runs it for this call: every variable free and unbounded.  The generalized Cauchy point followed by the subspace
// minimisation then gives the quasi-Newton step p = -H g; with an empty memory p = -g.
//   direction: the two-loop recursion over the k <= maxcor stored pairs (s_i, y_i, dr_i), rho_i = 1 / dr_i, newest first
//              in the first loop, H0 = gamma = dr / y'y of the newest pair (L-BFGS-B's theta = y'y / dr);
//              z = fl(x + p), d = fl(z - x) (L-BFGS-B forms d = z - x)
//   step:      stp = min(1 / ||d||_2, 1e10) while nit = 0, 1 afterwards (lnsrlb); trial = z when stp == 1, else
//              fl(x + fl(stp d))
//   search:    More & Thuente (1994), "Line search algorithms with guaranteed sufficient decrease", ACM TOMS 20:286-307,
//              as MINPACK-2's dcsrch / dcstep: ftol = 1e-3, gtol = 0.9, xtol = 0.1, stpmin = 0, stpmax = 1e10, on
//              phi(stp) = f(x + stp d) and phi'(stp) = g(trial)'d
//   failures:  g'd >= 0 for a new direction, or a search asking for trial maxls + 1: the last iterate is restored; with
//              an empty memory the run stops with GPK_LB_ABNORMAL, otherwise the memory is cleared and a new direction
//              is taken (a restart does not reset the initial-step rule: nit > 0 keeps stp = 1)
//   accepted:  nit += 1, then, in scipy's order (its driver checks the budgets before L-BFGS-B sees the new iterate):
//              nit >= maxiter (GPK_LB_MAXITER), nfev > maxfun (GPK_LB_MAXFUN), ||g||_inf <= pgtol (GPK_LB_PGTOL),
//              fl(f_old - f) <= fl(tol max(|f_old|, |f|, 1)) (GPK_LB_FTOL, tol = fl(fl(ftol / eps_mach) eps_mach)).
//              The first point only has the pgtol test.
//   pair:      y = g+ - g, rr = y'y; stp == 1: dr = gd - gd0, ddum = -gd0, s = d; otherwise dr = fl(fl(gd - gd0) stp),
//              ddum = fl(-gd0 stp), s = fl(stp d) (gd, gd0: g'd at the accepted trial and at the start of the search);
//              the pair is skipped when dr <= eps_mach ddum.  The oldest pair is dropped beyond maxcor.
//   result:    the last accepted iterate (results.x), its f, nit, nfev and the status.
//
// Rounding: every product, sum, difference, quotient and square root is rounded explicitly (__dmul_rn / __dadd_rn /
// __dsub_rn / __ddiv_rn / __dsqrt_rn: no fma contraction).  A dot product over the D <= 96 coordinates is
// p_l = fl(fl(fl(a_l b_l) + fl(a_{l+32} b_{l+32})) + fl(a_{l+64} b_{l+64})) per lane l (missing coordinates are 0), then
// p += shfl_xor(p, o) for o = 16, 8, 4, 2, 1.  tests/hyperopt_model.py restates all of it bit for bit.
#pragma once
#include "gpk_hyper.cuh"
#include "gpk_lbfgs.cuh"

#define GPK_HO_BIG 1e25
#define GPK_HO_STPMAX 1e10

// what the round's update does with the scored trial
enum { GPK_HO_START = 0, GPK_HO_SEARCH = 1 };

struct HOState {
    double f, gd0, stp, gamma;                    // f of x; g'd at the search start; the trial's step; H0
    double finit, ginit, gtest, stx, fx, gx, sty, fy, gy, stmin, stmax, width, width1;   // dcsrch
    long long nfev;
    int nit, status, phase, ifun;                 // ifun: trials asked for in this search
    int brackt, stage, k, head;                   // dcsrch; stored pairs and the ring slot of the next one
    int rounds;                                   // rounds that scored a point
    unsigned int ticket;
};

struct HOParams {
    int maxcor, maxiter, maxls;
    long long maxfun;
    double tol, pgtol, eps;
};

// GaussianProcess.nll from the two parts of gpk_hy_eval
__device__ __forceinline__ double gpk_ho_objective(const HyperModel& m, double ll, double lp)
{
    if (!isfinite(ll)) return GPK_HO_BIG;
    if (m.prior == GPK_PRIOR_NONE) return -ll;
    const double v = __dadd_rn(ll, lp);
    return isfinite(v) ? -v : GPK_HO_BIG;
}

// the forward-difference step of coordinate x
__device__ __forceinline__ double gpk_ho_h(double x, double eps)
{
    if (__dsub_rn(__dadd_rn(x, eps), x) != 0.0) return eps;
    return __dmul_rn(x >= 0.0 ? 1.4901161193847656e-08 : -1.4901161193847656e-08, fmax(1.0, fabs(x)));
}

// the fixed-order dot product of the header comment over three coordinates per lane
__device__ __forceinline__ double gpk_ho_dot(const double* a, const double* b)
{
    double p = __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) p = __dadd_rn(p, __shfl_xor_sync(0xffffffffu, p, o));
    return p;
}

__device__ __forceinline__ double gpk_ho_sgn(double v) { return v > 0.0 ? 1.0 : v < 0.0 ? -1.0 : 0.0; }

// s * sqrt((t / s)^2 - (a / s)(b / s)), with the radicand clamped at 0 when `clamp`
__device__ __forceinline__ double gpk_ho_gamma(double s, double t, double a, double b, bool clamp)
{
    const double ts = __ddiv_rn(t, s);
    double r = __dsub_rn(__dmul_rn(ts, ts), __dmul_rn(__ddiv_rn(a, s), __ddiv_rn(b, s)));
    if (clamp) r = fmax(0.0, r);
    return __dmul_rn(s, __dsqrt_rn(r));
}

// theta = 3 (fa - fb) / (sa - sb) + da + db
__device__ __forceinline__ double gpk_ho_theta(double fa, double fb, double sa, double sb, double da, double db)
{
    return __dadd_rn(__dadd_rn(__ddiv_rn(__dmul_rn(3.0, __dsub_rn(fa, fb)), __dsub_rn(sa, sb)), da), db);
}

// dcstep (MINPACK-2): the safeguarded step of the More-Thuente search; updates the interval and returns the new step
__device__ double gpk_ho_dcstep(double& stx, double& fx, double& dx, double& sty, double& fy, double& dy, double stp,
                                double fp, double dp, int& brackt, double stpmin, double stpmax)
{
    const double sgnd = __dmul_rn(gpk_ho_sgn(dp), gpk_ho_sgn(dx));
    double stpf;
    if (fp > fx) {
        const double th = gpk_ho_theta(fx, fp, stp, stx, dx, dp);
        const double s = fmax(fmax(fabs(th), fabs(dx)), fabs(dp));
        double gm = gpk_ho_gamma(s, th, dx, dp, false);
        if (stp < stx) gm = -gm;
        const double p = __dadd_rn(__dsub_rn(gm, dx), th);
        const double q = __dadd_rn(__dadd_rn(__dsub_rn(gm, dx), gm), dp);
        const double r = __ddiv_rn(p, q);
        const double stpc = __dadd_rn(stx, __dmul_rn(r, __dsub_rn(stp, stx)));
        const double stpq = __dadd_rn(stx, __dmul_rn(__ddiv_rn(__ddiv_rn(dx, __dadd_rn(__ddiv_rn(__dsub_rn(fx, fp),
                                                                                          __dsub_rn(stp, stx)), dx)),
                                                               2.0),
                                                     __dsub_rn(stp, stx)));
        stpf = fabs(__dsub_rn(stpc, stx)) < fabs(__dsub_rn(stpq, stx))
                   ? stpc : __dadd_rn(stpc, __ddiv_rn(__dsub_rn(stpq, stpc), 2.0));
        brackt = 1;
    } else if (sgnd < 0.0) {
        const double th = gpk_ho_theta(fx, fp, stp, stx, dx, dp);
        const double s = fmax(fmax(fabs(th), fabs(dx)), fabs(dp));
        double gm = gpk_ho_gamma(s, th, dx, dp, false);
        if (stp > stx) gm = -gm;
        const double p = __dadd_rn(__dsub_rn(gm, dp), th);
        const double q = __dadd_rn(__dadd_rn(__dsub_rn(gm, dp), gm), dx);
        const double r = __ddiv_rn(p, q);
        const double stpc = __dadd_rn(stp, __dmul_rn(r, __dsub_rn(stx, stp)));
        const double stpq = __dadd_rn(stp, __dmul_rn(__ddiv_rn(dp, __dsub_rn(dp, dx)), __dsub_rn(stx, stp)));
        stpf = fabs(__dsub_rn(stpc, stp)) > fabs(__dsub_rn(stpq, stp)) ? stpc : stpq;
        brackt = 1;
    } else if (fabs(dp) < fabs(dx)) {
        const double th = gpk_ho_theta(fx, fp, stp, stx, dx, dp);
        const double s = fmax(fmax(fabs(th), fabs(dx)), fabs(dp));
        double gm = gpk_ho_gamma(s, th, dx, dp, true);
        if (stp > stx) gm = -gm;
        const double p = __dadd_rn(__dsub_rn(gm, dp), th);
        const double q = __dadd_rn(__dadd_rn(gm, __dsub_rn(dx, dp)), gm);
        const double r = __ddiv_rn(p, q);
        double stpc;
        if (r < 0.0 && gm != 0.0) stpc = __dadd_rn(stp, __dmul_rn(r, __dsub_rn(stx, stp)));
        else stpc = stp > stx ? stpmax : stpmin;
        const double stpq = __dadd_rn(stp, __dmul_rn(__ddiv_rn(dp, __dsub_rn(dp, dx)), __dsub_rn(stx, stp)));
        if (brackt) {
            stpf = fabs(__dsub_rn(stpc, stp)) < fabs(__dsub_rn(stpq, stp)) ? stpc : stpq;
            const double lim = __dadd_rn(stp, __dmul_rn(0.66, __dsub_rn(sty, stp)));
            stpf = stp > stx ? fmin(lim, stpf) : fmax(lim, stpf);
        } else {
            stpf = fabs(__dsub_rn(stpc, stp)) > fabs(__dsub_rn(stpq, stp)) ? stpc : stpq;
            stpf = fmax(stpmin, fmin(stpmax, stpf));
        }
    } else {
        if (brackt) {
            const double th = gpk_ho_theta(fp, fy, sty, stp, dy, dp);
            const double s = fmax(fmax(fabs(th), fabs(dy)), fabs(dp));
            double gm = gpk_ho_gamma(s, th, dy, dp, false);
            if (stp > sty) gm = -gm;
            const double p = __dadd_rn(__dsub_rn(gm, dp), th);
            const double q = __dadd_rn(__dadd_rn(__dsub_rn(gm, dp), gm), dy);
            const double r = __ddiv_rn(p, q);
            stpf = __dadd_rn(stp, __dmul_rn(r, __dsub_rn(sty, stp)));
        } else {
            stpf = stp > stx ? stpmax : stpmin;
        }
    }
    if (fp > fx) {
        sty = stp; fy = fp; dy = dp;
    } else {
        if (sgnd < 0.0) { sty = stx; fy = fx; dy = dx; }
        stx = stp; fx = fp; dx = dp;
    }
    return stpf;
}

// dcsrch's START: the search of direction d from f with slope g at the first step p.stp
__device__ __forceinline__ void gpk_ho_dcsrch_start(HOState& p, double f, double g)
{
    p.brackt = 0;
    p.stage = 1;
    p.finit = f;
    p.ginit = g;
    p.gtest = __dmul_rn(1e-3, g);
    p.width = GPK_HO_STPMAX;
    p.width1 = __ddiv_rn(GPK_HO_STPMAX, 0.5);
    p.stx = 0.0; p.fx = f; p.gx = g;
    p.sty = 0.0; p.fy = f; p.gy = g;
    p.stmin = 0.0;
    p.stmax = __dadd_rn(p.stp, __dmul_rn(4.0, p.stp));
}

// dcsrch after the value f and slope g at p.stp: true when the search has ended (convergence or a warning), else p.stp
// is the next trial step
__device__ bool gpk_ho_dcsrch(HOState& p, double f, double g)
{
    const double stp = p.stp;
    const double ftest = __dadd_rn(p.finit, __dmul_rn(stp, p.gtest));
    if (p.stage == 1 && f <= ftest && g >= 0.0) p.stage = 2;
    bool end = false;
    if (p.brackt && (stp <= p.stmin || stp >= p.stmax)) end = true;
    if (p.brackt && __dsub_rn(p.stmax, p.stmin) <= __dmul_rn(0.1, p.stmax)) end = true;
    if (stp == GPK_HO_STPMAX && f <= ftest && g <= p.gtest) end = true;
    if (stp == 0.0 && (f > ftest || g >= p.gtest)) end = true;
    if (f <= ftest && fabs(g) <= __dmul_rn(0.9, -p.ginit)) end = true;
    if (end) return true;
    double nstp;
    if (p.stage == 1 && f <= p.fx && f > ftest) {
        const double gt = p.gtest;
        double fm = __dsub_rn(f, __dmul_rn(stp, gt));
        double fxm = __dsub_rn(p.fx, __dmul_rn(p.stx, gt));
        double fym = __dsub_rn(p.fy, __dmul_rn(p.sty, gt));
        double gm = __dsub_rn(g, gt);
        double gxm = __dsub_rn(p.gx, gt);
        double gym = __dsub_rn(p.gy, gt);
        nstp = gpk_ho_dcstep(p.stx, fxm, gxm, p.sty, fym, gym, stp, fm, gm, p.brackt, p.stmin, p.stmax);
        p.fx = __dadd_rn(fxm, __dmul_rn(p.stx, gt));
        p.fy = __dadd_rn(fym, __dmul_rn(p.sty, gt));
        p.gx = __dadd_rn(gxm, gt);
        p.gy = __dadd_rn(gym, gt);
    } else {
        nstp = gpk_ho_dcstep(p.stx, p.fx, p.gx, p.sty, p.fy, p.gy, stp, f, g, p.brackt, p.stmin, p.stmax);
    }
    if (p.brackt) {
        if (fabs(__dsub_rn(p.sty, p.stx)) >= __dmul_rn(0.66, p.width1))
            nstp = __dadd_rn(p.stx, __dmul_rn(0.5, __dsub_rn(p.sty, p.stx)));
        p.width1 = p.width;
        p.width = fabs(__dsub_rn(p.sty, p.stx));
        p.stmin = fmin(p.stx, p.sty);
        p.stmax = fmax(p.stx, p.sty);
    } else {
        p.stmin = __dadd_rn(nstp, __dmul_rn(1.1, __dsub_rn(nstp, p.stx)));
        p.stmax = __dadd_rn(nstp, __dmul_rn(4.0, __dsub_rn(nstp, p.stx)));
    }
    nstp = fmin(fmax(nstp, 0.0), GPK_HO_STPMAX);
    if ((p.brackt && (nstp <= p.stmin || nstp >= p.stmax)) ||
        (p.brackt && __dsub_rn(p.stmax, p.stmin) <= __dmul_rn(0.1, p.stmax)))
        nstp = p.stx;
    p.stp = nstp;
    return false;
}

// Work buffer of a run, doubles: x, g, d, z, xt (D each), the stencil's values (D + 1), S, Y (maxcor x D each), dr
// (maxcor), then the two-loop's alphas (maxcor)
struct HOWork {
    double *x, *g, *d, *z, *xt, *fv, *S, *Y, *dr, *al;
};

__host__ __device__ inline long gpk_ho_work_doubles(int D, int maxcor)
{
    return 5L * D + (D + 1) + 2L * maxcor * D + 2L * maxcor;
}

__host__ __device__ inline HOWork gpk_ho_work(double* base, int D, int maxcor)
{
    HOWork w;
    w.x = base; w.g = w.x + D; w.d = w.g + D; w.z = w.d + D; w.xt = w.z + D; w.fv = w.xt + D;
    w.S = w.fv + D + 1; w.Y = w.S + (long)maxcor * D; w.dr = w.Y + (long)maxcor * D; w.al = w.dr + maxcor;
    return w;
}

// A new search from x (every lane: x, g in registers): the direction, the failure rule for g'd >= 0 and the first
// trial.  Returns GPK_LB_RUNNING or GPK_LB_ABNORMAL.
__device__ int gpk_ho_new_search(HOState& p, const HOParams& q, const HOWork& w, int D, const double* x,
                                 const double* g)
{
    const int lane = threadIdx.x & 31;
    for (;;) {
        double r[3], d[3], z[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) r[c] = g[c];
        if (p.k > 0) {                                          // the two-loop recursion, newest pair first
            for (int i = p.k - 1; i >= 0; --i) {
                const int slot = (p.head - p.k + i + q.maxcor) % q.maxcor;
                const double* Sp = w.S + (long)slot * D;
                const double* Yp = w.Y + (long)slot * D;
                double sv[3], yv[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const int j = lane + 32 * c;
                    sv[c] = j < D ? Sp[j] : 0.0;
                    yv[c] = j < D ? Yp[j] : 0.0;
                }
                const double a = __ddiv_rn(gpk_ho_dot(sv, r), w.dr[slot]);
                if (lane == 0) w.al[i] = a;
#pragma unroll
                for (int c = 0; c < 3; ++c) r[c] = __dsub_rn(r[c], __dmul_rn(a, yv[c]));
            }
            __syncwarp();
#pragma unroll
            for (int c = 0; c < 3; ++c) r[c] = __dmul_rn(p.gamma, r[c]);
            for (int i = 0; i < p.k; ++i) {
                const int slot = (p.head - p.k + i + q.maxcor) % q.maxcor;
                const double* Sp = w.S + (long)slot * D;
                const double* Yp = w.Y + (long)slot * D;
                double sv[3], yv[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const int j = lane + 32 * c;
                    sv[c] = j < D ? Sp[j] : 0.0;
                    yv[c] = j < D ? Yp[j] : 0.0;
                }
                const double b = __ddiv_rn(gpk_ho_dot(yv, r), w.dr[slot]);
                const double cc = __dsub_rn(w.al[i], b);
#pragma unroll
                for (int c = 0; c < 3; ++c) r[c] = __dadd_rn(r[c], __dmul_rn(sv[c], cc));
            }
            __syncwarp();
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            z[c] = __dsub_rn(x[c], r[c]);                         // z = x + p, p = -H g
            d[c] = __dsub_rn(z[c], x[c]);
        }
        const double gd = gpk_ho_dot(g, d);
        if (!(gd < 0.0)) {                                         // not a descent direction
            if (p.k == 0) return GPK_LB_ABNORMAL;
            p.k = 0;
            p.head = 0;
            continue;
        }
        const double dnorm = __dsqrt_rn(gpk_ho_dot(d, d));
        p.stp = p.nit == 0 ? fmin(__ddiv_rn(1.0, dnorm), GPK_HO_STPMAX) : 1.0;
        p.gd0 = gd;
        gpk_ho_dcsrch_start(p, p.f, gd);
        p.ifun = 1;
        p.phase = GPK_HO_SEARCH;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int j = lane + 32 * c;
            if (j < D) {
                w.d[j] = d[c];
                w.z[j] = z[c];
                w.xt[j] = p.stp == 1.0 ? z[c] : __dadd_rn(x[c], __dmul_rn(p.stp, d[c]));
            }
        }
        return GPK_LB_RUNNING;
    }
}

// the update of one round, on one warp, after the stencil's D + 1 values are in w.fv
__device__ void gpk_ho_update(HOState* __restrict__ st, const HOParams& q, const HOWork& w, int D)
{
    const int lane = threadIdx.x & 31;
    HOState p = *st;
    p.rounds += 1;
    p.nfev += D + 1;
    const double ft = __ldcg(w.fv);
    double xt[3], gt[3], x[3], g[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int j = lane + 32 * c;
        xt[c] = gt[c] = x[c] = g[c] = 0.0;
        if (j < D) {
            xt[c] = w.xt[j];
            const double hh = __dsub_rn(__dadd_rn(xt[c], gpk_ho_h(xt[c], q.eps)), xt[c]);
            gt[c] = __ddiv_rn(__dsub_rn(__ldcg(w.fv + 1 + j), ft), hh);
            x[c] = w.x[j];
            g[c] = w.g[j];
        }
    }
    int stop = GPK_LB_RUNNING;
    bool accept = false, search = false;
    if (p.phase == GPK_HO_SEARCH) {
        double dv[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int j = lane + 32 * c;
            dv[c] = j < D ? w.d[j] : 0.0;
        }
        const double gdt = gpk_ho_dot(gt, dv);
        const double stp = p.stp;
        if (gpk_ho_dcsrch(p, ft, gdt)) {
            // the search ended: the trial is the new iterate
            const double fold = p.f;
            p.f = ft;
            p.nit += 1;
            if (p.nit >= q.maxiter) stop = GPK_LB_MAXITER;
            else if (p.nfev > q.maxfun) stop = GPK_LB_MAXFUN;
            else {
                double pg = 0.0;
#pragma unroll
                for (int c = 0; c < 3; ++c) pg = fmax(pg, fabs(gt[c]));
                pg = gpk_lb_max(pg);
                if (pg <= q.pgtol) stop = GPK_LB_PGTOL;
                else if (__dsub_rn(fold, ft) <= __dmul_rn(q.tol, fmax(fmax(fabs(fold), fabs(ft)), 1.0)))
                    stop = GPK_LB_FTOL;
            }
            if (stop == GPK_LB_RUNNING) {
                double yv[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) yv[c] = __dsub_rn(gt[c], g[c]);
                const double rr = gpk_ho_dot(yv, yv);
                double dr, ddum;
                if (stp == 1.0) {
                    dr = __dsub_rn(gdt, p.gd0);
                    ddum = -p.gd0;
                } else {
                    dr = __dmul_rn(__dsub_rn(gdt, p.gd0), stp);
                    ddum = __dmul_rn(-p.gd0, stp);
                }
                if (!(dr <= __dmul_rn(GPK_LB_DBL_EPS, ddum))) {
                    double* Sp = w.S + (long)p.head * D;
                    double* Yp = w.Y + (long)p.head * D;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const int j = lane + 32 * c;
                        if (j < D) {
                            Sp[j] = stp == 1.0 ? dv[c] : __dmul_rn(stp, dv[c]);
                            Yp[j] = yv[c];
                        }
                    }
                    if (lane == 0) w.dr[p.head] = dr;
                    p.gamma = __ddiv_rn(dr, rr);
                    p.head = (p.head + 1) % q.maxcor;
                    p.k = min(p.k + 1, q.maxcor);
                    __syncwarp();
                }
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) { x[c] = xt[c]; g[c] = gt[c]; }
            accept = true;
            search = stop == GPK_LB_RUNNING;
        } else if (p.ifun >= q.maxls) {
            // trial maxls + 1 asked for: the last iterate stands (x, g, f unchanged)
            if (p.k == 0) stop = GPK_LB_ABNORMAL;
            else { p.k = 0; p.head = 0; search = true; }
        } else {
            p.ifun += 1;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int j = lane + 32 * c;
                if (j < D) w.xt[j] = p.stp == 1.0 ? w.z[j] : __dadd_rn(x[c], __dmul_rn(p.stp, dv[c]));
            }
        }
    } else {
        // the first point: scipy's start and L-BFGS-B's projected-gradient test
#pragma unroll
        for (int c = 0; c < 3; ++c) { x[c] = xt[c]; g[c] = gt[c]; }
        p.f = ft;
        accept = true;
        double pg = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) pg = fmax(pg, fabs(gt[c]));
        pg = gpk_lb_max(pg);
        if (pg <= q.pgtol) stop = GPK_LB_PGTOL;
        else search = true;
    }
    if (accept) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int j = lane + 32 * c;
            if (j < D) { w.x[j] = x[c]; w.g[j] = g[c]; }
        }
    }
    if (search) stop = gpk_ho_new_search(p, q, w, D, x, g);
    p.status = stop;
    p.ticket = 0;
    __syncwarp();
    if (lane == 0) *st = p;
}

// One round: CTA b scores row b of the stencil of w.xt; the last CTA updates.  Xt / y: the handle's inputs and targets.
__global__ void __launch_bounds__(GPK_HY_THREADS) gpk_ho_round_kernel(const HyperModel m, const double* __restrict__ Xt,
                                                                      long ldx, const double* __restrict__ y, int n,
                                                                      const HOParams q, double* __restrict__ work,
                                                                      HOState* __restrict__ st)
{
    __shared__ double th[GPK_HYPER_MAX_DIM];
    __shared__ int skip;
    __shared__ bool last;
    extern __shared__ double sm[];
    const int b = blockIdx.x, D = m.n_params + 1;
    if (threadIdx.x == 0) skip = st->status != GPK_LB_RUNNING;
    __syncthreads();
    if (skip) return;
    const HOWork w = gpk_ho_work(work, D, q.maxcor);
    for (int j = threadIdx.x; j < D; j += blockDim.x) {
        const double v = w.xt[j];
        th[j] = j == b - 1 ? __dadd_rn(v, gpk_ho_h(v, q.eps)) : v;
    }
    __syncthreads();
    double l, lp;
    gpk_hy_eval(m, Xt, ldx, y, n, th, sm, &l, &lp);
    if (threadIdx.x == 0) {
        w.fv[b] = gpk_ho_objective(m, l, lp);
        __threadfence();
        last = atomicAdd(&st->ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last || threadIdx.x >= 32) return;
    __threadfence();
    gpk_ho_update(st, q, w, D);
}
