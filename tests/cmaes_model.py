"""Exact numpy restatement of gpk_maximize_cmaes (robo_b200/csrc/gpk_cmaes.cuh) — TEST INFRASTRUCTURE ONLY.

The (mu/mu_w, lambda)-CMA-ES with cma's BoundTransform and IPOP restarts, every rounding step as the kernels take it:
numpy's elementwise float64 operations round each product, sum, quotient and square root once, like the kernels'
__dmul_rn / __dadd_rn / __ddiv_rn / __dsqrt_rn, and every sum runs in the kernels' order.  Given the device's normals
(gpk_cmaes_draws) and the same acquisition values, a run is the device's bit for bit.  The acquisition is pluggable:
``acq_fn(P)`` maps a (lambda, d) batch of phenotypes to acquisition values (the energy is -acq).  ``normals(run, g,
lam, d)`` gives the (lam, d) standard normals of a generation; ``numpy_normals(seed)`` is a Box-Muller stand-in for
tests without a device."""
import numpy as np

from robo_b200._lib import (CMA_CONDITIONCOV, CMA_HIST, CMA_MAXFEVALS, CMA_NUMERICAL, CMA_RUNNING, CMA_TOLFUN,
                            CMA_TOLX, cmaes_lambda, cmaes_run_constants)

SWEEPS, JACOBI_TOL = 30, 1e-16
TOLFUN, TOLX, CONDITIONCOV = 1e-11, 1e-11, 1e14
_EXP_C = (1.6059043836821613e-10, 2.08767569878681e-09, 2.505210838544172e-08, 2.755731922398589e-07,
          2.7557319223985893e-06, 2.48015873015873e-05, 0.0001984126984126984, 0.001388888888888889,
          0.008333333333333333, 0.041666666666666664, 0.16666666666666666, 0.5)


def exp(x):
    """gpk_cmaes_exp: Cody-Waite reduction, degree-11 Horner tail, 2^k (elementwise)."""
    x = np.asarray(x, dtype=np.float64)
    k = np.rint(x * 1.4426950408889634)
    r = (x - k * 6.93147180369123816490e-01) - k * 1.90821492927058770002e-10
    p = np.full_like(r, _EXP_C[0])
    for c in _EXP_C[1:]:
        p = c + p * r
    with np.errstate(over="ignore", invalid="ignore"):
        out = np.ldexp(1.0 + (r + (r * r) * p), np.where(np.isfinite(k), k, 0).astype(np.int64))
    out = np.where(x >= 709.782712893384, np.inf, out)
    out = np.where(x < -745.2, 0.0, out)
    return np.where(np.isnan(x), x, out)[()]


def margins(lower, upper):
    """a_l, a_u of BoxConstraintsLinQuadTransformation."""
    half = (upper - lower) * 0.5
    return np.fmin(half, (1.0 + np.fabs(lower)) / 20.0), np.fmin(half, (1.0 + np.fabs(upper)) / 20.0)


def transform(x, lower, upper):
    """gpk_cmaes_T elementwise over the last axis: genotype -> phenotype in [lower, upper]."""
    x = np.array(x, dtype=np.float64, copy=True)
    lb, ub = np.broadcast_to(lower, x.shape), np.broadcast_to(upper, x.shape)
    al, au = (np.broadcast_to(a, x.shape) for a in margins(lower, upper))
    half = (ub - lb) * 0.5
    s = (lb - 2.0 * al) - half
    far = (x < s) | (x > (ub + 2.0 * au) + half)
    per = 2.0 * (((ub - lb) + al) + au)
    x = np.where(far, x - per * np.floor((x - s) / per), x)
    ua, la = ub + au, lb - al
    x = np.where(x > ua, x - 2.0 * (x - ua), x)
    x = np.where(x < la, x + 2.0 * (la - x), x)
    ql, qu = x - la, x - ua
    return np.where(x < lb + al, lb + ((ql * ql) / 4.0) / al,
                    np.where(x < ub - au, x, ub - ((qu * qu) / 4.0) / au))


def genotype(y, lower, upper):
    """gpk_cmaes_geno: the inverse of transform on [lower, upper]."""
    y = np.asarray(y, dtype=np.float64)
    al, au = margins(lower, upper)
    with np.errstate(invalid="ignore"):
        lo = (lower - al) + 2.0 * np.sqrt(al * (y - lower))
        hi = (upper + au) - 2.0 * np.sqrt(au * (upper - y))
    return np.where(y < lower + al, lo, np.where(y < upper - au, y, hi))


def rank(e):
    """numpy.argsort(kind="stable") of the energies (NaN last, ties by index, -0.0 == +0.0) as the kernel's counting
    sort computes it."""
    e = np.asarray(e, dtype=np.float64)
    nan = np.isnan(e)
    key = np.where(nan, 0.0, e)
    idx = np.arange(e.size)
    before = np.where(nan[:, None] | nan[None, :], nan[None, :] & nan[:, None] & (idx[:, None] < idx[None, :]) |
                      (~nan[:, None] & nan[None, :]),
                      (key[:, None] < key[None, :]) | ((key[:, None] == key[None, :]) & (idx[:, None] < idx[None, :])))
    r = before.sum(axis=0)                        # r[k] = #{j before k}
    order = np.empty_like(idx)
    order[r] = idx
    return order


def round_robin(d):
    """The Jacobi pairs of every round: list of (p, q) arrays (p < q < d; pairs with the dummy index dropped)."""
    n2 = d + (d & 1)
    rounds = []
    for rd in range(n2 - 1):
        i = np.arange(n2 // 2)
        a = np.where(i == 0, 0, 1 + (i - 1 + rd) % (n2 - 1))
        b = 1 + (n2 - 2 - i + rd) % (n2 - 1)
        p, q = np.minimum(a, b), np.maximum(a, b)
        keep = q < d
        rounds.append((p[keep], q[keep]))
    return rounds


def jacobi(C, trace=None):
    """The kernel's parallel cyclic Jacobi on the symmetrised C -> (eigenvalues, B, sweeps).  ``trace`` (a list) gets
    the (p, q) pairs rotated, round by round."""
    d = C.shape[0]
    A = np.triu(C) + np.triu(C, 1).T
    V = np.eye(d)
    rounds = round_robin(d)
    sweeps = 0
    for _ in range(SWEEPS):
        sweeps += 1
        any_rot = False
        for p, q in rounds:
            app, aqq, apq = A[p, p], A[q, q], A[p, q]
            act = np.fabs(apq) > JACOBI_TOL * np.sqrt(np.fabs(app) * np.fabs(aqq))
            p, q, app, aqq, apq = p[act], q[act], app[act], aqq[act], apq[act]
            if p.size == 0:
                continue
            any_rot = True
            if trace is not None:
                trace.append((p.copy(), q.copy()))
            theta = (aqq - app) / (2.0 * apq)
            at = np.fabs(theta)
            with np.errstate(over="ignore", divide="ignore"):
                t = np.where(at > 1e150, 0.5 / at, 1.0 / (at + np.sqrt(theta * theta + 1.0)))
            t = np.where(theta < 0.0, -t, t)
            c = 1.0 / np.sqrt(t * t + 1.0)
            s = t * c
            x, y = A[p, :].copy(), A[q, :].copy()
            A[p, :] = c[:, None] * x - s[:, None] * y
            A[q, :] = s[:, None] * x + c[:, None] * y
            x, y = A[:, p].copy(), A[:, q].copy()
            A[:, p] = c[None, :] * x - s[None, :] * y
            A[:, q] = s[None, :] * x + c[None, :] * y
            x, y = V[:, p].copy(), V[:, q].copy()
            V[:, p] = c[None, :] * x - s[None, :] * y
            V[:, q] = s[None, :] * x + c[None, :] * y
            A[p, p] = app - t * apq
            A[q, q] = aqq + t * apq
            A[p, q] = 0.0
            A[q, p] = 0.0
        if not any_rot:
            break
    return np.diag(A).copy(), V, sweeps


def _seqsum(terms, axis=0):
    """sum from +0.0 in index order along ``axis``."""
    terms = np.moveaxis(np.asarray(terms), axis, 0)
    acc = np.zeros(terms.shape[1:])
    for t in terms:
        acc = acc + t
    return acc


def numpy_normals(seed):
    """A Box-Muller stand-in for the device's Philox normals (same law, not the same numbers)."""
    def normals(run, g, lam, d):
        rs = np.random.RandomState([int(seed) & 0xFFFFFFFF, run, g])
        return rs.standard_normal((lam, d))
    return normals


def run(acq_fn, normals, x0, lower, upper, n_func_evals=1000, restarts=0, sigma0=0.6, trace=None):
    """The whole CMAES.maximize -> dict(x, energy, nfev_total, nit, nfev, stop (per run), m, sigma, ps, pc, C (last
    run), found).  ``trace`` (a list) gets a dict per generation (run, g, energies, sigma, eigen)."""
    lower, upper = np.asarray(lower, dtype=np.float64), np.asarray(upper, dtype=np.float64)
    d = lower.size
    m0 = genotype(np.asarray(x0, dtype=np.float64), lower, upper)
    runs = int(restarts) + 1
    nit, nfev, stop = np.zeros(runs, np.int64), np.zeros(runs, np.int64), np.zeros(runs, np.int64)
    best, xbest, found = np.nan, np.zeros(d), False
    total = 0
    for r in range(runs):
        c = cmaes_run_constants(d, cmaes_lambda(d, r))
        lam, mu, w = c["lam"], c["mu"], c["w"]
        m, sigma = m0.copy(), float(sigma0)
        ps, pc = np.zeros(d), np.zeros(d)
        C, B, Dv, ev = np.eye(d), np.eye(d), np.ones(d), np.ones(d)
        pw, since, g = 1.0, 0, 0
        hist = []
        before = total
        st = CMA_RUNNING
        while st == CMA_RUNNING:
            z = np.asarray(normals(r, g, lam, d), dtype=np.float64)
            dz = Dv[None, :] * z
            Y = _seqsum(B[None, :, :] * dz[:, None, :], axis=2)
            G = m[None, :] + sigma * Y
            P = transform(G, lower, upper)
            e = -np.asarray(acq_fn(P), dtype=np.float64) + 0.0
            order = rank(e)
            o = order[:mu]
            e0 = e[order[0]]
            if np.isfinite(e0) and (not found or e0 < best):
                best, xbest, found = float(e0), P[order[0]].copy(), True
            yw = _seqsum(w[:, None] * Y[o])
            m = m + sigma * yw
            t = _seqsum(B * yw[:, None], axis=0) / Dv
            u = _seqsum(B * t[None, :], axis=1)
            ps = c["omcs"] * ps + c["cps"] * u
            norm = np.sqrt(_seqsum(ps * ps))
            pw = (pw * c["omcs"]) * c["omcs"]
            hsig = norm / np.sqrt(1.0 - pw) < c["hth"]
            pc = c["omcc"] * pc + c["ccc"] * yw if hsig else c["omcc"] * pc
            dh = 0.0 if hsig else c["ccd"]
            S = _seqsum(w[:, None, None] * (Y[o][:, :, None] * Y[o][:, None, :]))
            with np.errstate(over="ignore", invalid="ignore"):
                C = (c["a0"] * C + c["c1"] * (pc[:, None] * pc[None, :] + dh * C)) + c["cmu"] * S
                bad = not np.all(np.isfinite(C))
                sigma = sigma * exp(c["csds"] * (norm / c["chi"] - 1.0))
                if e[order[0]] == e[order[c["flat"]]]:
                    sigma = sigma * exp(0.2 + c["csds"])
            hist.append(e0)
            g += 1
            total += lam
            since += lam
            eigen = since > c["eig_gap"]
            if eigen:
                C = np.triu(C) + np.triu(C, 1).T
                ev, B, _ = jacobi(C)
                with np.errstate(invalid="ignore"):
                    Dv = np.sqrt(ev)
                bad = bad or not np.all((ev > 0.0) & np.isfinite(ev))
                since = 0
            if trace is not None:
                trace.append(dict(run=r, g=g - 1, energies=e, sigma=sigma, eigen=eigen))
            if total >= n_func_evals:
                st = CMA_MAXFEVALS
            else:
                H = c["hist"]
                tolfun = False
                if g >= H:
                    vals = np.concatenate([e, np.asarray(hist[g - H:g])])
                    if not np.all(np.isnan(vals)):
                        with np.errstate(invalid="ignore"):
                            tolfun = np.nanmax(vals) - np.nanmin(vals) < TOLFUN
                with np.errstate(invalid="ignore"):
                    mxs = np.nanmax(np.concatenate([[0.0], np.fmax(np.fabs(pc), np.sqrt(np.diag(C)))]))
                    cond = np.nanmax(ev) / np.nanmin(ev) if not np.all(np.isnan(ev)) else np.nan
                numerical = bad or not (sigma > 0.0) or not np.isfinite(sigma) or not np.all(np.isfinite(m))
                if tolfun:
                    st = CMA_TOLFUN
                elif sigma * mxs < TOLX:
                    st = CMA_TOLX
                elif cond > CONDITIONCOV:
                    st = CMA_CONDITIONCOV
                elif numerical:
                    st = CMA_NUMERICAL
        nit[r], nfev[r], stop[r] = g, total - before, st
        if st == CMA_MAXFEVALS:
            break
    return dict(x=xbest, energy=best, nfev_total=total, nit=nit, nfev=nfev, stop=stop, m=m, sigma=float(sigma), ps=ps,
                pc=pc, C=C, found=found)


assert CMA_HIST >= 130
