"""Exact numpy restatement of gpk_optimize_hypers (robo_b200/csrc/gpk_hyperopt.cuh) — TEST INFRASTRUCTURE ONLY.

scipy.optimize.minimize(fun, p0, method='L-BFGS-B') with every variable unbounded, as the device runs it: the
forward-difference stencil of every scored point, the two-loop direction, the More-Thuente search (MINPACK-2 dcsrch /
dcstep), L-BFGS-B's restarts, skip rule and stopping tests in scipy's order.  numpy float64 scalars round every
operation once, like the kernel's __dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn / __dsqrt_rn, and the dot products
follow the kernel's lane order, so given the same objective values the trial points, f, nit, nfev and the status equal
the device's bit for bit.

The objective is pluggable:
  - ``run(values, p0)``: ``values(T)`` maps the rows T (the trial point and its dim neighbours, the stencil of one
    round) to their objective values; on the GPU it is ``_lib.hyper_lnpost`` combined by ``objective``;
  - ``run(fg, p0, jac=True)``: ``fg(x)`` returns (f, g) with an analytic gradient, one evaluation per point (scipy's
    ``jac=True``).
The ``defect`` argument injects a known-wrong variant, so that the tests can show the comparison with scipy detects it.
"""
import numpy as np

F = np.float64
BIG = F(1e25)
STPMAX = F(1e10)
EPS = F(2.220446049250313e-16)
SQRT_EPS = F(1.4901161193847656e-08)
CHUNK = 16                                     # GPK_HO_CHUNK
FTOL, PGTOL, MAXITER, MAXFUN, ABNORMAL = range(5)
DEFAULTS = dict(maxcor=10, maxiter=15000, maxfun=15000, ftol=2.220446049250313e-09, pgtol=1e-5, eps=1e-8, maxls=20)


def objective(ll, lp, has_prior):
    """GaussianProcess.nll from gpk_hy_eval's two parts (the kernel's gpk_ho_objective)."""
    ll, lp = np.asarray(ll, dtype=F), np.asarray(lp, dtype=F)
    with np.errstate(all="ignore"):
        v = ll + lp if has_prior else ll
        return np.where(np.isfinite(ll) & np.isfinite(v), -v, BIG)


def step(x, eps):
    """The forward-difference step of every coordinate of x (scipy approx_derivative with abs_step = eps)."""
    x = np.asarray(x, dtype=F)
    h = np.full(x.shape, F(eps))
    fall = ((x + h) - x) == 0
    h[fall] = np.where(x[fall] >= 0, SQRT_EPS, -SQRT_EPS) * np.maximum(F(1.0), np.abs(x[fall]))
    return h


def stencil(x, eps, defect=None):
    """The D + 1 rows one round scores: x, then x + h_j e_j."""
    x = np.asarray(x, dtype=F)
    h = step(x, eps)
    if defect == "relative_step":
        h = SQRT_EPS * np.where(x >= 0, F(1.0), F(-1.0)) * np.maximum(F(1.0), np.abs(x))
    T = np.repeat(x[None], len(x) + 1, axis=0)
    for j in range(len(x)):
        T[1 + j, j] = x[j] + h[j]
    return T, h


def dot(a, b):
    """The kernel's fixed-order dot product: three coordinates per lane, then the xor butterfly."""
    A = np.zeros(96, dtype=F)
    B = np.zeros(96, dtype=F)
    A[:len(a)] = a
    B[:len(b)] = b
    A, B = A.reshape(3, 32), B.reshape(3, 32)
    p = (A[0] * B[0] + A[1] * B[1]) + A[2] * B[2]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        p = p + p[lanes ^ o]
    return F(p[0])


def _sgn(v):
    return F(1.0) if v > 0 else F(-1.0) if v < 0 else F(0.0)


def _gamma(s, t, a, b, clamp):
    ts = t / s
    r = ts * ts - (a / s) * (b / s)
    if clamp:
        r = np.fmax(F(0.0), r)
    return s * np.sqrt(r)


def _theta(fa, fb, sa, sb, da, db):
    return ((F(3.0) * (fa - fb)) / (sa - sb) + da) + db


def dcstep(stx, fx, dx, sty, fy, dy, stp, fp, dp, brackt, stpmin, stpmax):
    """MINPACK-2 dcstep -> (stx, fx, dx, sty, fy, dy, new step, brackt)."""
    sgnd = _sgn(dp) * _sgn(dx)
    if fp > fx:
        th = _theta(fx, fp, stp, stx, dx, dp)
        s = np.fmax(np.fmax(abs(th), abs(dx)), abs(dp))
        gm = _gamma(s, th, dx, dp, False)
        if stp < stx:
            gm = -gm
        p = (gm - dx) + th
        q = ((gm - dx) + gm) + dp
        r = p / q
        stpc = stx + r * (stp - stx)
        stpq = stx + ((dx / ((fx - fp) / (stp - stx) + dx)) / F(2.0)) * (stp - stx)
        stpf = stpc if abs(stpc - stx) < abs(stpq - stx) else stpc + (stpq - stpc) / F(2.0)
        brackt = True
    elif sgnd < 0:
        th = _theta(fx, fp, stp, stx, dx, dp)
        s = np.fmax(np.fmax(abs(th), abs(dx)), abs(dp))
        gm = _gamma(s, th, dx, dp, False)
        if stp > stx:
            gm = -gm
        p = (gm - dp) + th
        q = ((gm - dp) + gm) + dx
        r = p / q
        stpc = stp + r * (stx - stp)
        stpq = stp + (dp / (dp - dx)) * (stx - stp)
        stpf = stpc if abs(stpc - stp) > abs(stpq - stp) else stpq
        brackt = True
    elif abs(dp) < abs(dx):
        th = _theta(fx, fp, stp, stx, dx, dp)
        s = np.fmax(np.fmax(abs(th), abs(dx)), abs(dp))
        gm = _gamma(s, th, dx, dp, True)
        if stp > stx:
            gm = -gm
        p = (gm - dp) + th
        q = (gm + (dx - dp)) + gm
        r = p / q
        if r < 0 and gm != 0:
            stpc = stp + r * (stx - stp)
        else:
            stpc = stpmax if stp > stx else stpmin
        stpq = stp + (dp / (dp - dx)) * (stx - stp)
        if brackt:
            stpf = stpc if abs(stpc - stp) < abs(stpq - stp) else stpq
            lim = stp + F(0.66) * (sty - stp)
            stpf = np.fmin(lim, stpf) if stp > stx else np.fmax(lim, stpf)
        else:
            stpf = stpc if abs(stpc - stp) > abs(stpq - stp) else stpq
            stpf = np.fmax(stpmin, np.fmin(stpmax, stpf))
    else:
        if brackt:
            th = _theta(fp, fy, sty, stp, dy, dp)
            s = np.fmax(np.fmax(abs(th), abs(dy)), abs(dp))
            gm = _gamma(s, th, dy, dp, False)
            if stp > sty:
                gm = -gm
            p = (gm - dp) + th
            q = ((gm - dp) + gm) + dy
            r = p / q
            stpf = stp + r * (sty - stp)
        else:
            stpf = stpmax if stp > stx else stpmin
    if fp > fx:
        sty, fy, dy = stp, fp, dp
    else:
        if sgnd < 0:
            sty, fy, dy = stx, fx, dx
        stx, fx, dx = stp, fp, dp
    return stx, fx, dx, sty, fy, dy, stpf, brackt


class Search(object):
    """MINPACK-2 dcsrch with ftol = 1e-3, gtol = 0.9, xtol = 0.1, stpmin = 0, stpmax = 1e10."""

    def __init__(self, f, g, stp):
        self.brackt, self.stage = False, 1
        self.finit, self.ginit, self.gtest = f, g, F(1e-3) * g
        self.width = STPMAX
        self.width1 = STPMAX / F(0.5)
        self.stx, self.fx, self.gx = F(0.0), f, g
        self.sty, self.fy, self.gy = F(0.0), f, g
        self.stmin, self.stmax = F(0.0), stp + F(4.0) * stp
        self.stp = stp

    def __call__(self, f, g):
        """True when the search has ended; else self.stp is the next trial step."""
        stp = self.stp
        ftest = self.finit + stp * self.gtest
        if self.stage == 1 and f <= ftest and g >= 0:
            self.stage = 2
        end = False
        if self.brackt and (stp <= self.stmin or stp >= self.stmax):
            end = True
        if self.brackt and self.stmax - self.stmin <= F(0.1) * self.stmax:
            end = True
        if stp == STPMAX and f <= ftest and g <= self.gtest:
            end = True
        if stp == 0 and (f > ftest or g >= self.gtest):
            end = True
        if f <= ftest and abs(g) <= F(0.9) * -self.ginit:
            end = True
        if end:
            return True
        if self.stage == 1 and f <= self.fx and f > ftest:
            gt = self.gtest
            fm, fxm, fym = f - stp * gt, self.fx - self.stx * gt, self.fy - self.sty * gt
            gm, gxm, gym = g - gt, self.gx - gt, self.gy - gt
            self.stx, fxm, gxm, self.sty, fym, gym, nstp, self.brackt = dcstep(
                self.stx, fxm, gxm, self.sty, fym, gym, stp, fm, gm, self.brackt, self.stmin, self.stmax)
            self.fx, self.fy = fxm + self.stx * gt, fym + self.sty * gt
            self.gx, self.gy = gxm + gt, gym + gt
        else:
            self.stx, self.fx, self.gx, self.sty, self.fy, self.gy, nstp, self.brackt = dcstep(
                self.stx, self.fx, self.gx, self.sty, self.fy, self.gy, stp, f, g, self.brackt, self.stmin, self.stmax)
        if self.brackt:
            if abs(self.sty - self.stx) >= F(0.66) * self.width1:
                nstp = self.stx + F(0.5) * (self.sty - self.stx)
            self.width1 = self.width
            self.width = abs(self.sty - self.stx)
            self.stmin, self.stmax = np.fmin(self.stx, self.sty), np.fmax(self.stx, self.sty)
        else:
            self.stmin = nstp + F(1.1) * (nstp - self.stx)
            self.stmax = nstp + F(4.0) * (nstp - self.stx)
        nstp = np.fmin(np.fmax(nstp, F(0.0)), STPMAX)
        if self.brackt and (nstp <= self.stmin or nstp >= self.stmax or self.stmax - self.stmin <= F(0.1) * self.stmax):
            nstp = self.stx
        self.stp = nstp
        return False


class _Armijo(object):
    """The injected 'armijo' defect: backtracking on sufficient decrease alone (gpk_lbfgs.cuh's search)."""

    def __init__(self, f, g, stp):
        self.f0, self.g0, self.stp = f, g, stp

    def __call__(self, f, g):
        if f <= self.f0 + F(1e-4) * self.stp * self.g0:
            return True
        self.stp = self.stp * F(0.5)
        return False


def direction(g, S, Y, DR, gamma):
    """-H g by the two-loop recursion (newest pair first in the first loop); the pairs oldest first."""
    r = np.array(g, dtype=F)
    k = len(S)
    if k:
        al = [F(0.0)] * k
        for i in range(k - 1, -1, -1):
            al[i] = dot(S[i], r) / DR[i]
            r = r - al[i] * Y[i]
        r = gamma * r
        for i in range(k):
            b = dot(Y[i], r) / DR[i]
            r = r + S[i] * (al[i] - b)
    return -r


def run(fun, p0, jac=False, defect=None, trace=None, **opt):
    """One gpk_optimize_hypers run -> dict(x, f, nit, nfev, status, rounds, restarts (memory refreshes)).  trace (a list) receives every scored
    point."""
    o = dict(DEFAULTS)
    o.update(opt)
    maxcor, maxiter, maxfun, maxls = int(o["maxcor"]), int(o["maxiter"]), int(o["maxfun"]), int(o["maxls"])
    pgtol, eps = F(o["pgtol"]), F(o["eps"])
    tol = (F(o["ftol"]) / EPS) * EPS
    D = len(p0)
    per = 1 if jac else D + 1

    def score(xt):
        if trace is not None:
            trace.append(np.array(xt, dtype=F))
        if jac:
            f, g = fun(np.array(xt, dtype=F))
            return F(f), np.asarray(g, dtype=F).copy()
        T, h = stencil(xt, eps, defect)
        v = np.asarray(fun(T.copy()), dtype=F)
        hh = (xt + h) - xt
        if defect == "relative_step":
            hh = T[1:].diagonal() - xt
        return v[0], (v[1:] - v[0]) / hh

    with np.errstate(all="ignore"):
        x = np.array(p0, dtype=F)
        S, Y, DR = [], [], []
        gamma = F(1.0)
        nit, nfev, rounds, restarts = 0, 0, 0, 0
        f, g = score(x)
        nfev += per
        rounds += 1
        if np.max(np.abs(g)) <= pgtol:
            return dict(x=x, f=f, nit=nit, nfev=nfev, status=PGTOL, rounds=rounds, restarts=restarts)
        while True:
            # a new search (gpk_ho_new_search)
            while True:
                p = direction(g, S, Y, DR, gamma)
                z = x + p
                d = z - x
                gd = dot(g, d)
                if not gd < 0:
                    if not S:
                        return dict(x=x, f=f, nit=nit, nfev=nfev, status=ABNORMAL, rounds=rounds, restarts=restarts)
                    S, Y, DR = [], [], []
                    restarts += 1
                    continue
                break
            dnorm = np.sqrt(dot(d, d))
            if defect == "initial_step":
                stp = F(1.0)
            else:
                stp = np.fmin(F(1.0) / dnorm, STPMAX) if nit == 0 else F(1.0)
            gd0 = gd
            ls = (_Armijo if defect == "armijo" else Search)(f, gd, stp)
            ifun = 1
            accepted = False
            while True:
                xt = z.copy() if ls.stp == 1 else x + ls.stp * d
                stp = ls.stp
                ft, gt = score(xt)
                nfev += per
                rounds += 1
                gdt = dot(gt, d)
                if ls(ft, gdt):
                    accepted = True
                    break
                if ifun >= maxls:
                    break
                ifun += 1
            if not accepted:
                if not S:
                    return dict(x=x, f=f, nit=nit, nfev=nfev, status=ABNORMAL, rounds=rounds, restarts=restarts)
                S, Y, DR = [], [], []
                restarts += 1
                continue
            fold = f
            nit += 1
            stop = None
            if nit >= maxiter:
                stop = MAXITER
            elif nfev > maxfun:
                stop = MAXFUN
            elif np.max(np.abs(gt)) <= pgtol:
                stop = PGTOL
            elif fold - ft <= tol * np.fmax(np.fmax(abs(fold), abs(ft)), F(1.0)):
                stop = FTOL
            if stop is None:
                y = gt - g
                rr = dot(y, y)
                if stp == 1:
                    dr, ddum, s = gdt - gd0, -gd0, d.copy()
                else:
                    dr, ddum, s = (gdt - gd0) * stp, -gd0 * stp, stp * d
                if defect == "skip_rule":                  # the curvature of the unscaled step
                    dr, ddum = gdt - gd0, -gd0
                skip = dr <= EPS * ddum
                if not skip:
                    S.append(s)
                    Y.append(y)
                    DR.append(dr)
                    if len(S) > maxcor:
                        S, Y, DR = S[1:], Y[1:], DR[1:]
                    gamma = dr / rr
            x, f, g = xt, ft, gt
            if stop is not None:
                return dict(x=x, f=f, nit=nit, nfev=nfev, status=stop, rounds=rounds, restarts=restarts)


def noop_rounds(rounds):
    """Rounds the host launches after the final one: the rest of the last chunk."""
    return -(-rounds // CHUNK) * CHUNK - rounds
