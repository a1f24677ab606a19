"""GP-MCMC hyper-parameters on the device (gpk_hyper_lnpost / gpk_sample_hypers, hyper_sampler="device").

- gpk_hyper_lnpost's log-likelihood against today's pool path (_LikelihoodPool.loglik) and the oracle, and its log-prior
  against the host prior classes;
- gpk_sample_hypers bit for bit against tests/hyper_model.py fed by gpk_hyper_lnpost, on the runs the models make;
- determinism, the end-to-end train, every argument error."""
import numpy as np
import pytest

from tests import hyper_model as M
from tests.test_de_es_cpu import LO, UP, branin

pytestmark = pytest.mark.gpu

TINY = 1.25e-12


def _fmin_kernel(D):
    from robo_b200 import kernels as K
    return 2 * K.Matern52Kernel(np.ones(D), ndim=D)


def _prod_kernel(D=3):
    """the config 4 structure: an amplitude times one 1-D Matern-5/2 factor per column"""
    from robo_b200 import kernels as K
    k = K.ConstantKernel(0.0, ndim=D)
    for d in range(D):
        k = K.Product(k, K.Matern52Kernel(np.ones(1), ndim=D, axes=d))
    return k


def _handle(X, y, kernel, prior=None):
    from robo_b200 import _lib
    from robo_b200.models.gaussian_process_mcmc import _hyper_prior
    f = kernel.flatten()
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    kind, par, n_ls, n_lr = _hyper_prior(prior)
    _lib.set_hyper_model(h, f["slots"], len(f["axis"]), float(np.mean(y)), TINY, kind, par, n_ls, n_lr)
    return h, f


def _lnpost_fn(h, has_prior):
    from robo_b200 import _lib
    return lambda T: M.post(*_lib.hyper_lnpost(h, T), has_prior=has_prior)


# ---- 1. the log-likelihood ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kname", ["fmin", "prod1d"])
@pytest.mark.parametrize("N", [3, 17, 128, 129, 232])
def test_loglik_matches_pool_and_oracle(N, kname):
    from robo_b200 import _lib
    from robo_b200.models.gaussian_process_mcmc import _LikelihoodPool
    assert _lib.HYPER_MAX_N == 232
    rng = np.random.RandomState(N)
    D = 2 if kname == "fmin" else 3
    kernel = _fmin_kernel(D) if kname == "fmin" else _prod_kernel(D)
    X = rng.rand(N, D)
    y = np.sin(6 * X).sum(axis=1) + 0.1 * rng.randn(N)
    dim = len(kernel) + 1
    T = np.c_[rng.uniform(-1, 1, 12), rng.uniform(-1, 1, (12, dim - 2)), rng.uniform(-6, -2, 12)]
    extra = np.array([np.r_[0.5, np.zeros(dim - 2), 21.0],             # |theta| > 20
                      np.r_[-20.5, np.zeros(dim - 2), -3.0],
                      np.r_[0.0, np.zeros(dim - 2), -20.0],            # the smallest noise the |theta| rule admits
                      np.r_[-20.0, np.zeros(dim - 2), -20.0]])         # amplitude at the same scale as that noise
    T = np.vstack([T, extra])
    h, f = _handle(X, y, kernel)
    ll, lp = _lib.hyper_lnpost(h, T)
    assert np.all(lp == 0.0)
    pool = _LikelihoodPool(kernel, X, y, float(np.mean(y)), len(T))
    try:
        ref = pool.loglik(T)
    finally:
        pool.close()
    orc = np.array([M.oracle_ll(X, y, float(np.mean(y)), f, t) for t in T])
    assert np.array_equal(np.isneginf(ll), np.isneginf(ref)) and np.array_equal(np.isneginf(ll), np.isneginf(orc))
    assert np.all(np.isneginf(ll[12:14])) and np.all(np.isfinite(ll[:12]))
    ok = np.isfinite(ref)
    # 1e-10 relative to max(|ll|, 1) for the thetas of a sampler's range; at the smallest admitted noise K is ill
    # conditioned and any two factorisations differ by about cond(K) eps, so the bound there is 64 cond(K) eps
    cond = np.array([M.oracle_cond(X, f, t) if o else 1.0 for t, o in zip(T, ok)])
    tol = np.maximum(1e-10, 64 * cond * np.finfo(np.float64).eps)
    for r in (ref, orc):
        err = np.where(ok, np.abs(ll - np.where(ok, r, 0.0)) / np.maximum(np.abs(np.where(ok, r, 0.0)), 1.0), 0.0)
        assert np.max(err[:12]) < 1e-10, (np.max(err[:12]), N, kname)
        assert np.all(err < tol), (err, tol, N, kname)
    # the same theta gives the same bits, alone or in a batch
    ll1, _ = _lib.hyper_lnpost(h, T[3:4])
    assert ll1.tobytes() == ll[3:4].tobytes()


@pytest.mark.parametrize("N", [40, 128])
def test_not_positive_definite_is_minus_inf(N):
    """Identical inputs: K = amp J exactly (the jitter is below half an ulp of amp = e^19.9), rank one, so every
    factorisation meets a pivot <= 0."""
    from robo_b200 import _lib
    from robo_b200.models.gaussian_process_mcmc import _LikelihoodPool
    X = np.full((N, 2), 0.3)
    y = np.random.RandomState(0).rand(N)
    kernel = _fmin_kernel(2)
    T = np.array([[19.9, 0.0, 0.0, -19.9], [19.9, 5.0, -5.0, -19.9]])
    h, _ = _handle(X, y, kernel)
    ll, _ = _lib.hyper_lnpost(h, T)
    pool = _LikelihoodPool(kernel, X, y, float(np.mean(y)), len(T))
    try:
        ref = pool.loglik(T)
    finally:
        pool.close()
    assert np.all(np.isneginf(ll)) and np.all(np.isneginf(ref))


# ---- 2. the priors -------------------------------------------------------------------------------------------------
def _prior_cases():
    from robo_b200 import priors as PR
    return [("default", PR.DefaultPrior(4, rng=np.random.RandomState(0)), 2),
            ("env", PR.EnvPrior(6, 3, 2, rng=np.random.RandomState(0)), 4),
            ("env_short", PR.EnvPrior(5, 3, 2, rng=np.random.RandomState(0)), 3)]   # the slices reach the noise


@pytest.mark.parametrize("case", [0, 1, 2])
def test_device_prior_matches_host_classes(case):
    from robo_b200 import _lib
    name, prior, D = _prior_cases()[case]
    rng = np.random.RandomState(case)
    X = rng.rand(10, D)
    y = rng.rand(10)
    kernel = _fmin_kernel(D)
    dim = len(kernel) + 1
    h, _ = _handle(X, y, kernel, prior)
    T = rng.uniform(-3, 3, (40, dim))
    T[:5, 0] = rng.uniform(0.1, 3, 5)                                   # inside the lognormal's support
    loc = prior.ln_prior.mean
    special = [np.r_[loc, np.zeros(dim - 2), -1.0],                     # theta_0 == loc: -inf
               np.r_[loc - 0.5, np.zeros(dim - 2), -1.0],               # theta_0 < loc
               np.r_[1.0, np.full(dim - 2, -10.5), -1.0],               # below the tophat
               np.r_[1.0, np.full(dim - 2, 2.5), -1.0],                 # above the tophat
               np.r_[1.0, np.full(dim - 2, -10.0), -1.0],               # on the tophat's bounds
               np.r_[1.0, np.full(dim - 2, 2.0), -1.0],
               np.r_[1.0, np.zeros(dim - 2), 0.0],                      # horseshoe at 0: +inf
               np.r_[loc - 1.0, np.zeros(dim - 2), 0.0]]                # -inf + inf
    T = np.vstack([T, special])
    _, lp = _lib.hyper_lnpost(h, T)
    with np.errstate(all="ignore"):
        ref = np.array([prior.lnprob(t) for t in T], dtype=np.float64)
    assert np.array_equal(np.isnan(lp), np.isnan(ref))
    inf = np.isinf(ref)
    assert np.array_equal(lp[inf], ref[inf]) and np.array_equal(np.isinf(lp), inf)
    fin = np.isfinite(ref)
    assert fin.sum() >= 5
    err = np.abs(lp[fin] - ref[fin]) / np.maximum(np.abs(ref[fin]), 1.0)
    assert np.max(err) < 1e-13, (name, np.max(err))
    assert np.isneginf(lp[-8]) and np.isneginf(lp[-7]) and lp[-2] == np.inf


# ---- 3. the sampler bit for bit --------------------------------------------------------------------------------------
@pytest.fixture
def spy(monkeypatch):
    from robo_b200 import _lib
    real, seen = _lib.sample_hypers, []

    def rec(h, p0, steps, seed):
        r = real(h, p0, steps, seed)
        seen.append(dict(h=h, p0=np.array(p0, dtype=np.float64), steps=steps, seed=seed, r=r))
        return r
    monkeypatch.setattr(_lib, "sample_hypers", rec)
    return seen


def _replay(seen, has_prior=True):
    for c in seen:
        ref = M.run(_lnpost_fn(c["h"], has_prior), c["p0"], c["steps"], c["seed"])
        assert c["r"]["pos"].tobytes() == ref["pos"].tobytes()
        assert c["r"]["lnpost"].tobytes() == ref["lnpost"].tobytes()
        assert np.array_equal(c["r"]["n_accepted"], ref["n_accepted"])
        assert np.any(ref["n_accepted"] > 0)


def _branin_data(n, seed=0):
    rng = np.random.RandomState(seed)
    X = LO + (UP - LO) * rng.rand(n, 2)
    return X, np.array([branin(x) for x in X])


def _branin_model(n_hypers=10, chain=200, burnin=100, prior=True):
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    kernel = _fmin_kernel(2)
    p = DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)) if prior else None
    return GaussianProcessMCMC(kernel, prior=p, n_hypers=n_hypers, chain_length=chain, burnin_steps=burnin,
                               normalize_input=True, lower=LO, upper=UP, rng=np.random.RandomState(2),
                               hyper_sampler="device")


def test_branin_default_prior_bit_for_bit(spy):
    m = _branin_model()
    m.train(*_branin_data(30))
    assert [c["steps"] for c in spy] == [100, 200]
    assert spy[1]["p0"].tobytes() == spy[0]["r"]["pos"].tobytes()
    _replay(spy)


def test_n200_dim8_bit_for_bit(spy):
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    rng = np.random.RandomState(8)
    X = rng.rand(200, 6)
    y = np.sin(5 * X).sum(axis=1) + 0.05 * rng.randn(200)
    kernel = _fmin_kernel(6)                                              # theta: amplitude, 6 length scales, noise
    m = GaussianProcessMCMC(kernel, prior=DefaultPrior(8, rng=np.random.RandomState(3)), n_hypers=18, chain_length=40,
                            burnin_steps=20, normalize_input=True, lower=np.zeros(6), upper=np.ones(6),
                            rng=np.random.RandomState(4), hyper_sampler="device")
    m.train(X, y)
    assert m.hypers.shape == (18, 8)
    _replay(spy)


def _fabolas_model(hyper_sampler="device"):
    from robo_b200 import kernels as K
    from robo_b200.models.fabolas_gp import FabolasGPMCMC
    from robo_b200.priors import EnvPrior
    kernel = K.Product(K.ConstantKernel(0.0, ndim=3),
                       K.Product(K.Matern52Kernel(np.ones(2), ndim=3, axes=[0, 1]),
                                 K.Matern52Kernel(np.ones(1), ndim=3, axes=[2])))
    return FabolasGPMCMC(kernel, basis_func=lambda s: (1 - s) ** 2,
                         prior=EnvPrior(len(kernel) + 1, 2, 1, rng=np.random.RandomState(6)), n_hypers=12,
                         chain_length=60, burnin_steps=40, lower=LO, upper=UP, rng=np.random.RandomState(5),
                         hyper_sampler=hyper_sampler)


def _fabolas_data(n=120):
    rng = np.random.RandomState(0)
    X = np.c_[LO + (UP - LO) * rng.rand(n, 2), rng.uniform(0.05, 1, n)]
    return X, np.log(np.array([branin(x) for x in X]) + 1) * (1 + 0.2 * X[:, 2])


def test_fabolas_env_prior_bit_for_bit(spy):
    m = _fabolas_model()
    m.train(*_fabolas_data())
    assert m.hypers.shape == (12, 5) and len(spy) == 2
    _replay(spy)


# ---- 4. determinism --------------------------------------------------------------------------------------------------
def test_same_seed_same_result_on_any_handle():
    from robo_b200 import _lib
    from robo_b200.priors import DefaultPrior
    X, y = _branin_data(30)
    prior = DefaultPrior(4, rng=np.random.RandomState(1))
    p0 = prior.sample_from_prior(10)
    h1, _ = _handle(X / 15.0, y, _fmin_kernel(2), prior)
    h2, _ = _handle(X / 15.0, y, _fmin_kernel(2), prior)
    a = _lib.sample_hypers(h1, p0, 50, 12345)
    b = _lib.sample_hypers(h1, p0, 50, 12345)
    c = _lib.sample_hypers(h2, p0, 50, 12345)
    d = _lib.sample_hypers(h2, p0, 50, 12346)
    for r in (b, c):
        assert r["pos"].tobytes() == a["pos"].tobytes() and r["lnpost"].tobytes() == a["lnpost"].tobytes()
        assert np.array_equal(r["n_accepted"], a["n_accepted"])
    assert d["pos"].tobytes() != a["pos"].tobytes()
    z = _lib.sample_hypers(h1, p0, 0, 1)                                   # no steps: the initial log-posteriors
    assert np.array_equal(z["pos"], p0) and np.all(z["n_accepted"] == 0)
    assert z["lnpost"].tobytes() == M.post(*_lib.hyper_lnpost(h1, p0)).tobytes()


# ---- 5. end to end ---------------------------------------------------------------------------------------------------
def test_train_end_to_end_and_predict_matches_oracle(monkeypatch, spy):
    from robo_b200.models import GaussianProcess
    from tests import fake_gpk
    m = _branin_model(chain=30, burnin=20)
    X, y = _branin_data(30)
    m.train(X, y)
    assert m.hypers.shape == (10, 4) and m.p0.shape == (10, 4) and m.burned
    assert m.n_lnprob_calls == 10 * 21 + 10 * 31
    assert len(m.models) == 10 and all(s.is_trained for s in m.models)
    assert m.hypers.tobytes() == spy[-1]["r"]["pos"].tobytes()
    Xs = LO + (UP - LO) * np.random.RandomState(9).rand(50, 2)
    mu, var = m.predict(Xs)
    hypers = m.hypers.copy()
    # a second train continues from p0: one run of chain_length steps, no burn-in
    p0 = m.p0.copy()
    n = len(spy)
    m.train(*_branin_data(31))
    assert len(spy) == n + 1 and spy[-1]["steps"] == 30 and spy[-1]["p0"].tobytes() == p0.tobytes()
    assert m.n_lnprob_calls == 10 * 31
    # the oracle mixture moments for the hypers of the first train
    fake_gpk.install(monkeypatch)
    mus, vs = [], []
    for s in hypers:
        k = _fmin_kernel(2)
        k.set_parameter_vector(s[:-1])
        g = GaussianProcess(k, noise=np.exp(s[-1]), normalize_input=True, lower=LO, upper=UP,
                            rng=np.random.RandomState(0))
        g.train(X, y, do_optimize=False)
        a, b = g.predict(Xs)
        mus.append(a)
        vs.append(b)
    mus, vs = np.array(mus), np.array(vs)
    ref_mu = mus.mean(axis=0)
    ref_var = np.clip(np.mean((mus - ref_mu) ** 2, axis=0) + vs.mean(axis=0), np.finfo(np.float64).eps, np.inf)
    assert np.max(np.abs(mu - ref_mu) / np.maximum(np.abs(ref_mu), np.std(y))) < 1e-10
    assert np.max(np.abs(var - ref_var) / np.maximum(ref_var, 1e-6 * np.max(ref_var))) < 1e-10


def test_fallback_above_the_limit(spy):
    from robo_b200 import _lib
    m = _branin_model(chain=3, burnin=2)
    m.train(*_branin_data(_lib.HYPER_MAX_N + 1))
    assert spy == [] and m.hypers.shape == (10, 4)


# ---- 6. argument errors --------------------------------------------------------------------------------------------
def test_bad_arguments():
    from robo_b200 import _lib
    X, y = _branin_data(20)
    kernel = _fmin_kernel(2)
    f = kernel.flatten()
    p0 = np.random.RandomState(0).rand(10, 4)
    h = _lib.Handle(0)
    with pytest.raises(ValueError, match="gpk_set_kernel"):             # no kernel
        _lib.set_hyper_model(h, f["slots"], 2, 0.0, TINY)
    h.set_data(X / 15, y)
    with pytest.raises(ValueError, match="gpk_set_kernel"):
        _lib.set_hyper_model(h, f["slots"], 2, 0.0, TINY)
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    with pytest.raises(ValueError, match="gpk_set_hyper_model"):        # no hyper model yet
        _lib.sample_hypers(h, p0, 5, 1)
    with pytest.raises(ValueError):                                     # the slot table misses a term
        _lib.set_hyper_model(h, [("amp", None), ("metric", [0]), ("amp", None)], 2, 0.0, TINY)
    with pytest.raises(ValueError):                                     # unknown prior kind
        _lib.set_hyper_model(h, f["slots"], 2, 0.0, TINY, 7, np.zeros(7))
    _lib.set_hyper_model(h, f["slots"], 2, 0.0, TINY)
    with pytest.raises(ValueError, match="even"):
        _lib.sample_hypers(h, p0[:9], 5, 1)
    with pytest.raises(ValueError, match="even"):                       # fewer walkers than 2 dim
        _lib.sample_hypers(h, p0[:6], 5, 1)
    with pytest.raises(ValueError, match="dim"):
        _lib.sample_hypers(h, np.random.rand(10, 3), 5, 1)
    with pytest.raises(ValueError, match="dim"):
        _lib.hyper_lnpost(h, np.random.rand(2, 5))
    with pytest.raises(ValueError, match="steps"):
        _lib.sample_hypers(h, p0, -1, 1)
    Xb = np.random.RandomState(1).rand(_lib.HYPER_MAX_N + 1, 2)
    h.set_data(Xb, Xb[:, 0])
    with pytest.raises(ValueError, match="GPK_HYPER_MAX_N"):
        _lib.sample_hypers(h, p0, 5, 1)
    with pytest.raises(ValueError, match="GPK_HYPER_MAX_N"):
        _lib.hyper_lnpost(h, p0)
    h2 = _lib.Handle(0)                                                 # no data
    with pytest.raises(ValueError, match="gpk_set_data"):
        _lib.hyper_lnpost(h2, p0)
    h.close()
    h2.close()
