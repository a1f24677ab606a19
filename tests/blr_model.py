"""Exact numpy restatement of gpk_blr_sample (robo_b200/csrc/gpk_blr.cuh) and the reference's Bayesian linear
regression arithmetic — TEST INFRASTRUCTURE ONLY.

``run`` is one EnsembleSampler.run_mcmc of the emcee 2.x stretch move (a = 2) over theta = (log alpha, log beta) driven
by the library's counter-based Philox stream with the BLR tags: the initial log-posteriors, then for every step the two
half-steps with the proposals, partners and acceptance tests of the kernels, and the per-walker accept counts.  numpy's
elementwise float64 operations round every product and sum once, like the kernels' __dmul_rn / __dadd_rn, so
positions and log-posteriors equal the device's bit for bit given the same log-posteriors.  ``lnpost_fn(T)`` maps
the rows T to their log-posteriors: ``_lib.blr_lnpost`` on the GPU, ``lnpost`` below on the CPU.  log z and log u' come
from numpy; CUDA's log may differ from glibc's in the last bit, so a decision within a few ulp of a tie raises NearTie.

``features`` / ``lnpost`` / ``fit`` / ``predict`` restate robo/models/bayesian_linear_regression.py in the reference's
order of operations (np.linalg.inv, np.linalg.det, the mean of the means and of the variances)."""
import numpy as np

from tests.de_model import _mulshift, _philox, _u01
from tests.representer_model import NearTie, _check_ties  # noqa: F401  (NearTie is part of this module's surface)

TAG_MOVE, TAG_ACC = 0x424C0002, 0x424C0003
A = 2.0
# BayesianLinearRegressionPrior: LognormalPrior(sigma=0.1, mean=-10), HorseshoePrior(scale=0.1)
PRIOR_PAR = (0.1, -10.0, 0.1)


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


def run(lnpost_fn, p0, steps, seed):
    """One run -> dict(pos (nw, 2), lnpost (nw,), n_accepted (nw,))."""
    P = np.array(p0, dtype=np.float64, copy=True)
    nw, dim = P.shape
    hb = nw // 2
    L = np.asarray(lnpost_fn(P.copy()), dtype=np.float64).copy()
    L[np.isnan(L)] = -np.inf
    acc = np.zeros(nw, dtype=np.int64)
    for step in range(steps):
        for half in (0, 1):
            k = half * hb + np.arange(hb)
            q, z, _ = proposals(seed, step, half, P)
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


# ---- the reference's arithmetic ----------------------------------------------------------------------------------
def features(X, basis):
    """Phi of the rows X for a gpk_blr_basis code (bayesian_linear_regression.py:11-17, basis_func=None)."""
    X = np.asarray(X, dtype=np.float64)
    if basis == 0:
        return np.append(X, np.ones([X.shape[0], 1]), axis=1)
    if basis == 1:
        x = np.append(X ** 2, X, axis=1)
        return np.append(x, np.ones([X.shape[0], 1]), axis=1)
    return X


def prior_object(par=PRIOR_PAR):
    """A BayesianLinearRegressionPrior (the host classes) with the given constants."""
    from robo_b200 import priors as PR
    p = PR.BayesianLinearRegressionPrior(rng=np.random.RandomState(0))
    p.ln_prior_alpha = PR.LognormalPrior(sigma=par[0], mean=par[1])
    p.horseshoe = PR.HorseshoePrior(scale=par[2])
    return p


def prior_lnprob(theta, par=PRIOR_PAR):
    """BayesianLinearRegressionPrior.lnprob with the given constants."""
    return prior_object(par).lnprob(theta)


def mll(Phi, y, theta, par=PRIOR_PAR, prior=None):
    """marginal_log_likelihood (:76-113) in the reference's order, the prior included; LinAlgError of inv -> -inf,
    NaN -> -inf (what the sampler sees)."""
    theta = np.asarray(theta, dtype=np.float64)
    with np.errstate(all="ignore"):
        alpha, beta = np.exp(theta[0]), np.exp(theta[1])
        D, N = Phi.shape[1], Phi.shape[0]
        A_ = beta * np.dot(Phi.T, Phi)
        A_ += np.eye(D) * alpha
        try:
            A_inv = np.linalg.inv(A_)
        except np.linalg.LinAlgError:
            return -np.inf
        m = beta * np.dot(A_inv, Phi.T)
        m = np.dot(m, y)
        v = D / 2 * np.log(alpha)
        v += N / 2 * np.log(beta)
        v -= N / 2 * np.log(2 * np.pi)
        v -= beta / 2. * np.linalg.norm(y - np.dot(Phi, m), 2)
        v -= alpha / 2. * np.dot(m.T, m)
        v -= 0.5 * np.log(np.linalg.det(A_))
        v += (prior_object(par) if prior is None else prior).lnprob(theta)
    return -np.inf if np.isnan(v) else float(v)


def lnpost(Phi, y, par=PRIOR_PAR):
    """lnpost_fn for run() on the CPU."""
    prior = prior_object(par)
    return lambda T: np.array([mll(Phi, y, t, par, prior) for t in np.atleast_2d(T)])


def fit(Phi, y, hypers):
    """models (:197-210): [(m, S)] of the (alpha, beta) rows of hypers."""
    out = []
    for alpha, beta in hypers:
        S_inv = beta * np.dot(Phi.T, Phi)
        S_inv += np.eye(Phi.shape[1]) * alpha
        S = np.linalg.inv(S_inv)
        m = beta * np.dot(np.dot(S, Phi.T), y)
        out.append((m, S))
    return out


def predict(Phi_test, hypers, models):
    """predict (:213-254): the mean of the means and of the variances, clipped to eps."""
    mu = np.zeros([len(hypers), Phi_test.shape[0]])
    var = np.zeros([len(hypers), Phi_test.shape[0]])
    for i, h in enumerate(hypers):
        mu[i] = np.dot(models[i][0].T, Phi_test.T)
        var[i] = 1. / h[1] + np.diag(np.dot(np.dot(Phi_test, models[i][1]), Phi_test.T))
    m = mu.mean(axis=0)
    v = var.mean(axis=0)
    v = np.clip(v, np.finfo(v.dtype).eps, np.inf)
    return m, v
