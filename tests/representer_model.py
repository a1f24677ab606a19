"""Exact numpy restatement of gpk_sample_representers (robo_b200/csrc/gpk_rs.cuh) — TEST INFRASTRUCTURE ONLY.

The emcee 2.x stretch move of robo_b200/util/ensemble_sampler.py (a = 2) driven by the library's counter-based Philox
stream, for each estimator on its own: init, the two half-steps of every step, the box mask, NaN -> -inf, the acceptance
test, the accept counts and the restart loop.  numpy's elementwise float64 operations round every product and sum once,
like the kernels' __dmul_rn / __dadd_rn, so positions and log-probabilities equal the device's bit for bit given the
same scores.  The log-density is pluggable: ``lnp_fn(i, X)`` returns the raw sampling-acquisition values of estimator
i's model on the rows X (nb / 2 walker rows, exactly the half-batch the device scores, out-of-box rows included).

log z and log u' come from numpy; CUDA's log may differ from glibc's in the last bit.  Every acceptance decision whose
two sides lie within a few ulp of each other raises NearTie, so such a case fails with its own message rather than as a
trajectory mismatch."""
import numpy as np

from tests.de_model import _mulshift, _philox, _u01

TAG_INIT, TAG_MOVE, TAG_ACC = 0x52530001, 0x52530002, 0x52530003
A = 2.0
TIE_ULPS = 8


class NearTie(AssertionError):
    pass


def _mask(X, a, lower, upper):
    """(log-densities, in-box mask): -inf outside [lower, upper] or where the acquisition is NaN."""
    inside = np.all((X >= lower) & (X <= upper), axis=1)
    return np.where(inside & ~np.isnan(a), a, -np.inf), inside


def init_walkers(seed, run, nb, lower, upper):
    k = np.arange(nb, dtype=np.uint64)[:, None]
    j = np.arange(lower.size, dtype=np.uint64)[None, :]
    w0, w1, _, _ = _philox(seed, k, run, j, TAG_INIT)
    return lower + (upper - lower) * _u01(w0, w1)


def proposals(seed, run, step, half, P):
    """(q, z, partner index) of the walkers of half `half` at step `step`."""
    nb = P.shape[0]
    hb = nb // 2
    k = half * hb + np.arange(hb)
    w0, w1, w2, _ = _philox(seed, k.astype(np.uint64), step, 2 * run + half, TAG_MOVE)
    t = (A - 1.0) * _u01(w0, w1) + 1.0
    z = (t * t) / A
    c = (1 - half) * hb + _mulshift(w2, hb)
    S, Cc = P[k], P[c]
    return Cc - z[:, None] * (Cc - S), z, c


def accept_draws(seed, run, step, half, hb):
    k = half * hb + np.arange(hb)
    a0, a1, _, _ = _philox(seed, k.astype(np.uint64), step, 2 * run + half, TAG_ACC)
    return _u01(a0, a1)


def _check_ties(lhs, rhs, logz, dw):
    both = np.isfinite(lhs) & np.isfinite(rhs)
    tol = TIE_ULPS * (np.spacing(np.abs(lhs)) + np.spacing(np.abs(rhs)) + max(dw - 1, 0) * np.spacing(np.abs(logz)))
    near = both & (np.abs(lhs - rhs) <= tol)
    if np.any(near):
        raise NearTie("acceptance decision within %d ulp of a tie (lnpdiff %r, log u' %r): CUDA's log and numpy's may "
                      "decide it differently" % (TIE_ULPS, lhs[near][0], rhs[near][0]))


def sample_one(lnp_fn, i, seed, nb, lower, upper, steps=50, max_runs=5, trace=None):
    """One estimator -> dict(zb (nb, dw), lmb (nb,), runs, n_accepted (nb,), n_negative (in-box values < 0))."""
    lower, upper = np.asarray(lower, dtype=np.float64), np.asarray(upper, dtype=np.float64)
    dw, hb = lower.size, nb // 2
    n_negative = 0
    for run in range(max_runs):
        P = init_walkers(seed, run, nb, lower, upper)
        L = np.empty(nb)
        acc = np.zeros(nb, dtype=np.int64)
        for half in (0, 1):
            rows = P[half * hb:(half + 1) * hb].copy()
            a = np.asarray(lnp_fn(i, rows), dtype=np.float64)
            L[half * hb:(half + 1) * hb], inside = _mask(rows, a, lower, upper)
            n_negative += int(np.sum(inside & (a < 0)))
        for step in range(steps):
            for half in (0, 1):
                k = half * hb + np.arange(hb)
                q, z, c = proposals(seed, run, step, half, P)
                if trace is not None:
                    trace.append((run, step, half, k, c, z))
                a = np.asarray(lnp_fn(i, q.copy()), dtype=np.float64)
                v, inside = _mask(q, a, lower, upper)
                n_negative += int(np.sum(inside & (a < 0)))
                with np.errstate(invalid="ignore", divide="ignore"):
                    logz = np.log(z)
                    lhs = (dw - 1.0) * logz + v - L[k]
                    rhs = np.log(accept_draws(seed, run, step, half, hb))
                _check_ties(lhs, rhs, logz, dw)
                ok = lhs > rhs
                P[k[ok]] = q[ok]
                L[k[ok]] = v[ok]
                acc[k[ok]] += 1
        if np.all(np.isfinite(L)):
            break
    return dict(zb=P, lmb=L, runs=run + 1, n_accepted=acc, n_negative=n_negative)


def sample(lnp_fn, seeds, nb, lower, upper, steps=50, max_runs=5):
    """Every estimator i of seeds -> dict(zb (n, nb, dw), lmb (n, nb), runs (n,), n_accepted (n, nb), n_negative);
    n_negative counts in-box values < 0 (meaningful for EI only)."""
    rs = [sample_one(lnp_fn, i, s, nb, lower, upper, steps, max_runs) for i, s in enumerate(seeds)]
    return dict(zb=np.array([r["zb"] for r in rs]), lmb=np.array([r["lmb"] for r in rs]),
                runs=np.array([r["runs"] for r in rs], dtype=np.int32),
                n_accepted=np.array([r["n_accepted"] for r in rs]), n_negative=sum(r["n_negative"] for r in rs))
