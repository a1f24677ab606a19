"""Exact numpy restatement of gpk_maximize_lbfgs* (robo_b200/csrc/gpk_lbfgs.cuh) — TEST INFRASTRUCTURE ONLY.

Multi-start projected L-BFGS with forward-difference gradients, run in the device's rounds: every round scores the
trial points of the running starts (in start order) and their d neighbours in one batch, then advances every start.
Each product, sum, quotient and square root below is one IEEE double operation rounded once, as the kernels' __dmul_rn /
__dadd_rn / __ddiv_rn / __dsqrt_rn are, and the dot products follow the kernels' fixed order (``dot``).  Given the same
scores the iterates, energies, nit, nfev and statuses are the device's bit for bit.  The objective is pluggable:
``energy_fn(X)`` maps a (rows, d) batch to raw energies (-acq, mu or mu + sqrt(v)); a value that is not finite becomes
DBL_MAX here, as on the device."""
import math

import numpy as np

DBL_MAX = np.finfo(np.float64).max
DBL_EPS = np.finfo(np.float64).eps
SQRT_EPS = 1.4901161193847656e-08            # sqrt(DBL_EPSILON) = 2^-26
MAX_BACKTRACK = 20
FTOL, PGTOL, MAXITER, MAXFUN, ABNORMAL, INVALID = range(6)
SUCCESS = (FTOL, PGTOL)
DEFAULTS = dict(maxcor=10, maxiter=15000, maxfun=15000, ftol=2.220446049250313e-09, pgtol=1e-5)


def finite_or_max(e):
    e = np.asarray(e, dtype=np.float64)
    return np.where(np.isfinite(e), e, DBL_MAX)


def step(x, lower, upper):
    """Forward-difference step of every coordinate of x (before the (x + h) - x correction)."""
    h = np.where(x >= 0, SQRT_EPS, -SQRT_EPS) * np.maximum(1.0, np.abs(x))
    xh = x + h
    return np.where((xh > upper) | (xh < lower), -h, h)


def stencil(x, lower, upper):
    """The trial point x and its d neighbours: (d + 1, d) rows, as gpk_lb_stencil_kernel writes them."""
    d = x.size
    rows = np.repeat(x[None, :], d + 1, axis=0)
    nb = np.clip(x + step(x, lower, upper), lower, upper)
    rows[1 + np.arange(d), np.arange(d)] = nb
    return rows


def gradient(x, e0, e_nb, lower, upper):
    """g_j = (e_j - e0) / ((x_j + h_j) - x_j)."""
    return (e_nb - e0) / ((x + step(x, lower, upper)) - x)


def dot(a, b):
    """The kernels' dot product: lane l adds the products of coordinates l and l + 32, then a butterfly over 32 lanes."""
    pa, pb = np.zeros(64), np.zeros(64)
    pa[:a.size], pb[:b.size] = a, b
    p = pa[:32] * pb[:32] + pa[32:] * pb[32:]
    w = 16
    while w >= 1:
        p = p[:w] + p[w:2 * w]
        w //= 2
    return float(p[0])


class _Start(object):
    def __init__(self, x, maxcor):
        d = x.size
        self.x, self.g, self.dir, self.xt = x.copy(), np.zeros(d), np.zeros(d), x.copy()
        self.f, self.alpha, self.gamma = 0.0, 0.0, 0.0
        self.nfev = self.nit = self.nback = self.k = self.head = 0
        self.phase, self.status = 0, None
        self.S, self.Y, self.rho = np.zeros((maxcor, d)), np.zeros((maxcor, d)), np.zeros(maxcor)


def _direction(p, lower, upper, maxcor):
    x, g = p.x, p.g
    free = ~(((x == lower) & (g > 0)) | ((x == upper) & (g < 0)))
    d = np.where(free, -g, 0.0)
    if p.k > 0:
        slots = [(p.head - p.k + i + maxcor) % maxcor for i in range(p.k)]
        q = np.where(free, g, 0.0)
        al = [0.0] * p.k
        for i in range(p.k - 1, -1, -1):
            s = slots[i]
            al[i] = p.rho[s] * dot(p.S[s], q)
            q = np.where(free, q - al[i] * p.Y[s], q)
        r = np.where(free, p.gamma * q, 0.0)
        for i in range(p.k):
            s = slots[i]
            b = p.rho[s] * dot(p.Y[s], r)
            c = al[i] - b
            r = np.where(free, r + p.S[s] * c, r)
        d = np.where(free, -r, 0.0)
        if not dot(g, d) < 0.0:
            p.k = p.head = 0
            d = np.where(free, -g, 0.0)
    return d


def _advance(p, ft, gt, lower, upper, o):
    """gpk_lb_step_kernel for one start."""
    d = p.x.size
    p.nfev += d + 1
    moved = check_ftol = False
    f_old = 0.0
    if p.phase == 0:
        p.x, p.g, p.f, p.phase = p.xt.copy(), gt, ft, 1
        if ft == DBL_MAX:
            p.status = INVALID
        else:
            moved = True
    else:
        s = p.xt - p.x
        if ft <= p.f + 1e-4 * dot(p.g, s):
            y = gt - p.g
            sy, yy = dot(s, y), dot(y, y)
            if sy > DBL_EPS * yy:
                p.S[p.head], p.Y[p.head], p.rho[p.head] = s, y, 1.0 / sy
                p.gamma = sy / yy
                p.head = (p.head + 1) % o["maxcor"]
                p.k = min(p.k + 1, o["maxcor"])
            f_old = p.f
            p.x, p.g, p.f = p.xt.copy(), gt, ft
            p.nit += 1
            moved = check_ftol = True
        elif p.nback == MAX_BACKTRACK:
            p.status = ABNORMAL
        elif p.nfev >= o["maxfun"]:
            p.status = MAXFUN
        else:
            p.nback += 1
            p.alpha = p.alpha * 0.5
            p.xt = np.clip(p.x + p.alpha * p.dir, lower, upper)
    if not moved:
        return
    pg = float(np.max(np.abs(np.clip(p.x - p.g, lower, upper) - p.x)))
    if pg <= o["pgtol"]:
        p.status = PGTOL
    elif check_ftol and (f_old - p.f) / max(max(abs(f_old), abs(p.f)), 1.0) <= o["ftol"]:
        p.status = FTOL
    elif p.nit >= o["maxiter"]:
        p.status = MAXITER
    elif p.nfev >= o["maxfun"]:
        p.status = MAXFUN
    else:
        dd = _direction(p, lower, upper, o["maxcor"])
        p.alpha = min(1.0, 1.0 / math.sqrt(dot(dd, dd))) if p.nit == 0 and dot(dd, dd) > 0 else 1.0
        p.nback = 0
        p.dir = dd
        p.xt = np.clip(p.x + p.alpha * dd, lower, upper)


def minimize(energy_fn, x0, lower, upper, trace=None, **options):
    """The whole run from the starts x0 (n_starts, d) -> dict(x (n_starts, d), energy, nit, nfev, status,
    rounds).  ``trace`` (a list) receives the batch size of every round."""
    o = dict(DEFAULTS, **options)
    lower, upper = np.asarray(lower, dtype=np.float64).ravel(), np.asarray(upper, dtype=np.float64).ravel()
    x0 = np.clip(np.atleast_2d(np.asarray(x0, dtype=np.float64)), lower, upper)
    d = lower.size
    starts = [_Start(x, o["maxcor"]) for x in x0]
    active = list(range(len(starts)))
    rounds = 0
    while active:
        X = np.concatenate([stencil(starts[i].xt, lower, upper) for i in active])
        if trace is not None:
            trace.append(len(X))
        with np.errstate(all="ignore"):
            E = finite_or_max(energy_fn(X)).reshape(len(active), d + 1)
            for a, i in enumerate(active):
                p = starts[i]
                gt = gradient(p.xt, E[a, 0], E[a, 1:], lower, upper)
                _advance(p, float(E[a, 0]), gt, lower, upper, o)
        active = [i for i in active if starts[i].status is None]
        rounds += 1
    return dict(x=np.array([p.x for p in starts]), energy=np.array([p.f for p in starts]),
                nit=np.array([p.nit for p in starts]), nfev=np.array([p.nfev for p in starts]),
                status=np.array([p.status for p in starts]), rounds=rounds)
