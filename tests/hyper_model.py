"""Exact numpy restatement of gpk_sample_hypers (robo_b200/csrc/gpk_hyper.cuh) — TEST INFRASTRUCTURE ONLY.

One EnsembleSampler.run_mcmc of the emcee 2.x stretch move (a = 2) driven by the library's counter-based Philox stream:
the initial log-posteriors, then for every step the two half-steps with the proposals, partners and acceptance tests of
the kernels, and the per-walker accept counts.  numpy's elementwise float64 operations round every product and sum once,
like the kernels' __dmul_rn / __dadd_rn, so positions and log-posteriors equal the device's bit for bit given the same
log-posteriors.  The log-posterior is pluggable: ``lnpost_fn(T)`` maps the rows T (walkers or proposals) to their
log-posteriors; on the GPU it is ``_lib.hyper_lnpost`` combined by ``post`` (the kernel's order), on the CPU the oracle
likelihood plus the host prior classes (``oracle_lnpost``).

log z and log u' come from numpy; CUDA's log may differ from glibc's in the last bit.  An acceptance decision whose two
sides lie within a few ulp of each other raises representer_model.NearTie."""
import numpy as np

from tests.de_model import _mulshift, _philox, _u01
from tests.representer_model import NearTie, _check_ties  # noqa: F401  (NearTie is part of this module's surface)

TAG_MOVE, TAG_ACC = 0x48590002, 0x48590003
A = 2.0
TINY = 1.25e-12


def post(ll, lp, has_prior=True):
    """The sampler's log-posterior: fl(lp + ll) where ll is finite (ll alone without a prior), -inf otherwise, NaN ->
    -inf."""
    ll, lp = np.asarray(ll, dtype=np.float64), np.asarray(lp, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        v = np.where(np.isfinite(ll), lp + ll if has_prior else ll, -np.inf)
    return np.where(np.isnan(v), -np.inf, v)


def proposals(seed, step, half, P):
    """(q, z, partner index) of the walkers of half `half` at step `step`."""
    nw = P.shape[0]
    hb = nw // 2
    k = half * hb + np.arange(hb)
    w0, w1, w2, _ = _philox(seed, k.astype(np.uint64), step, half, TAG_MOVE)
    t = (A - 1.0) * _u01(w0, w1) + 1.0
    z = (t * t) / A
    c = (1 - half) * hb + _mulshift(w2, hb)
    S, Cc = P[k], P[c]
    return Cc - z[:, None] * (Cc - S), z, c


def accept_draws(seed, step, half, hb):
    k = half * hb + np.arange(hb)
    a0, a1, _, _ = _philox(seed, k.astype(np.uint64), step, half, TAG_ACC)
    return _u01(a0, a1)


def run(lnpost_fn, p0, steps, seed, trace=None):
    """One run -> dict(pos (nw, dim), lnpost (nw,), n_accepted (nw,))."""
    P = np.array(p0, dtype=np.float64, copy=True)
    nw, dim = P.shape
    hb = nw // 2
    L = np.asarray(lnpost_fn(P.copy()), dtype=np.float64).copy()
    L[np.isnan(L)] = -np.inf
    acc = np.zeros(nw, dtype=np.int64)
    for step in range(steps):
        for half in (0, 1):
            k = half * hb + np.arange(hb)
            q, z, c = proposals(seed, step, half, P)
            if trace is not None:
                trace.append((step, half, k, c, z, q.copy()))
            v = np.asarray(lnpost_fn(q.copy()), dtype=np.float64).copy()
            v[np.isnan(v)] = -np.inf
            with np.errstate(invalid="ignore", divide="ignore"):
                logz = np.log(z)
                lhs = (dim - 1.0) * logz + v - L[k]
                rhs = np.log(accept_draws(seed, step, half, hb))
            _check_ties(lhs, rhs, logz, dim)
            ok = lhs > rhs
            P[k[ok]] = q[ok]
            L[k[ok]] = v[ok]
            acc[k[ok]] += 1
    return dict(pos=P, lnpost=L, n_accepted=acc)


# ---- the CPU log-posterior: the oracle likelihood and the host prior classes --------------------------------------
def prior_object(kind, par, n_ls, n_lr, dim):
    """A robo_b200.priors object with the constants gpk_set_hyper_model received (None for no prior)."""
    from robo_b200 import priors as PR
    if kind == 0:
        return None
    if kind == 1:
        p = PR.DefaultPrior(dim, rng=np.random.RandomState(0))
    else:
        p = PR.EnvPrior(dim, n_ls, n_lr, rng=np.random.RandomState(0))
        p.bayes_lin_prior = PR.NormalPrior(par[5], par[6])
    p.ln_prior = PR.LognormalPrior(par[0], par[1])
    p.tophat = PR.TophatPrior(par[2], par[3])
    p.horseshoe = PR.HorseshoePrior(par[4])
    return p


def oracle_ll(X, y, mean, flat, theta, tiny=TINY):
    """_LikelihoodPool.loglik of one theta on the oracle (tests/fake_gpk.py): |theta| > 20, a failed factorisation or
    a non-finite value give -inf."""
    from tests.fake_gpk import FakeHandle
    theta = np.asarray(theta, dtype=np.float64)
    if np.any((-20 > theta) + (theta > 20)):
        return -np.inf
    log_amp, lm = 0.0, np.array(flat["log_metric"], dtype=np.float64)
    for p, (kind, terms) in enumerate(flat["slots"]):
        if kind == "amp":
            log_amp += theta[p]
        else:
            lm[terms] = theta[p]
    h = FakeHandle()
    h.set_data(X, y)
    h.set_kernel(flat["family"], log_amp, flat["axis"], flat["group"], lm)
    yerr = np.sqrt(np.exp(theta[-1]))
    try:
        with np.errstate(all="ignore"):
            _, ll = h.fit(float(np.sqrt(np.float64(yerr) ** 2 + tiny) ** 2), mean)
    except (np.linalg.LinAlgError, ValueError):
        return -np.inf
    return ll if np.isfinite(ll) else -np.inf


def oracle_cond(X, flat, theta, tiny=TINY):
    """2-norm condition number of the K that oracle_ll factorises for theta."""
    from tests.fake_gpk import FakeHandle
    theta = np.asarray(theta, dtype=np.float64)
    log_amp, lm = 0.0, np.array(flat["log_metric"], dtype=np.float64)
    for p, (kind, terms) in enumerate(flat["slots"]):
        if kind == "amp":
            log_amp += theta[p]
        else:
            lm[terms] = theta[p]
    h = FakeHandle()
    h.set_data(X, np.zeros(len(X)))
    h.set_kernel(flat["family"], log_amp, flat["axis"], flat["group"], lm)
    K = h.kernel.get_value(X)
    K[np.diag_indices_from(K)] += float(np.sqrt(np.sqrt(np.exp(theta[-1])) ** 2 + tiny) ** 2)
    return np.linalg.cond(K)


def oracle_lnpost(X, y, mean, flat, prior):
    """lnpost_fn for run(): the oracle likelihood plus prior.lnprob, combined as loglikelihood_batch does."""
    def fn(T):
        ll = np.array([oracle_ll(X, y, mean, flat, t) for t in T])
        if prior is None:
            return post(ll, np.zeros(len(T)), has_prior=False)
        with np.errstate(all="ignore"):
            lp = np.array([prior.lnprob(t) if np.isfinite(l) else 0.0 for t, l in zip(T, ll)], dtype=np.float64)
        return post(ll, lp)
    return fn
