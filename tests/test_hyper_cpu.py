"""Hyper-parameter sampling without a GPU: invariants of the exact restatement of gpk_sample_hypers
(tests/hyper_model.py), its agreement in law with EnsembleSampler, and the Python dispatch of hyper_sampler="device"
on the oracle-backed fake handles, with a fake of the three _lib entry points defined here."""
import importlib
import logging
import os
import re
from copy import deepcopy

import numpy as np
import pytest
import scipy.stats

from tests import hyper_model as M
from tests.test_de_es_cpu import LO, UP, _data, branin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the restatement ---------------------------------------------------------------------------------------------
def _gauss(T):
    return -0.5 * np.sum(((T - 0.3) / 0.2) ** 2, axis=1)


def test_header_constants_match_the_binding():
    from robo_b200 import _lib
    src = open(os.path.join(ROOT, "include", "gpk.h")).read()
    assert int(re.search(r"#define GPK_HYPER_MAX_N (\d+)", src).group(1)) == _lib.HYPER_MAX_N >= 200
    assert int(re.search(r"#define GPK_HYPER_MAX_DIM (\d+)", src).group(1)) == _lib.HYPER_MAX_DIM


def test_partners_from_the_other_half_and_z_in_range():
    trace = []
    p0 = np.random.RandomState(0).rand(12, 4)
    M.run(_gauss, p0, 30, 123, trace=trace)
    assert len(trace) == 60
    for step, half, k, c, z, q in trace:
        other = np.arange(6) + (6 if half == 0 else 0)
        assert np.all(np.isin(c, other)) and not np.any(np.isin(c, k))
        assert np.all(z >= 1 / M.A) and np.all(z <= M.A)


def test_abs_rule_nan_and_minus_inf_never_accepted():
    """|theta| > 20 is -inf before any factorisation; NaN and -inf proposals are never accepted."""
    X, y = _data(6)
    from robo_b200 import kernels as K
    flat = (2 * K.Matern52Kernel(np.ones(2), ndim=2)).flatten()
    assert M.oracle_ll(X, y, 0.0, flat, [0.0, 0.0, 21.0, -1.0]) == -np.inf
    assert M.oracle_ll(X, y, 0.0, flat, [-20.5, 0.0, 0.0, -1.0]) == -np.inf
    assert np.isfinite(M.oracle_ll(X, y, 0.0, flat, [0.0, 0.0, 0.0, -1.0]))

    def lnp(T):                                      # the largest values where |theta| > 20 or in a NaN corner
        v = np.sum(T, axis=1)
        v[np.any(np.abs(T) > 20, axis=1)] = -np.inf
        v[(T[:, 0] < -5) & (T[:, 1] < -5)] = np.nan
        return v
    for seed in range(5):
        p0 = np.random.RandomState(seed).uniform(-3, 3, size=(10, 3))
        r = M.run(lnp, p0, 60, seed)
        assert np.all(np.abs(r["pos"]) <= 20) and np.all(np.isfinite(r["lnpost"]))
        assert not np.any((r["pos"][:, 0] < -5) & (r["pos"][:, 1] < -5))
    assert np.array_equal(M.post([1.0, -np.inf, np.nan, 2.0], [np.inf, 0.0, 0.0, -np.inf]), [np.inf, -np.inf, -np.inf,
                                                                                          -np.inf])
    assert np.array_equal(M.post([1.0, np.inf], [5.0, 0.0], has_prior=False), [1.0, -np.inf])


def test_agreement_in_law_with_ensemble_sampler():
    """A 2-D Gaussian: every 2nd final walker of 80 runs of each sampler, two-sample KS per coordinate (different random
    streams: agreement in law only)."""
    from robo_b200.util.ensemble_sampler import EnsembleSampler
    host, dev = [], []
    rng = np.random.RandomState(0)
    for run in range(80):
        p0 = rng.uniform(size=(8, 2))
        s = EnsembleSampler(8, 2, lambda x: _gauss(x[None])[0], batch_lnpostfn=_gauss)
        host.append(s.run_mcmc(p0, 60, rstate0=rng)[0][::2])
        dev.append(M.run(_gauss, p0, 60, 1000 + run)["pos"][::2])
    host, dev = np.concatenate(host), np.concatenate(dev)
    for j in range(2):
        assert scipy.stats.ks_2samp(host[:, j], dev[:, j]).pvalue > 1e-3, j


def test_restated_priors_follow_the_host_classes():
    from robo_b200 import priors as PR
    rng = np.random.RandomState(4)
    d = PR.DefaultPrior(4)
    e = PR.EnvPrior(6, 3, 2)
    for _ in range(20):
        t = rng.uniform(-3, 3, size=4)
        assert M.prior_object(1, [1.0, 0.0, -10, 2, 0.1, 0, 0], 0, 0, 4).lnprob(t) == d.lnprob(t)
        t = rng.uniform(-3, 3, size=6)
        assert M.prior_object(2, [1.0, -2.0, -10, 2, 0.001, 1.0, 0.0], 3, 2, 6).lnprob(t) == e.lnprob(t)
    # EnvPrior adds the pdf of the environment parameters; with n_ls + n_lr + 1 = dim the slice reaches the noise
    t = np.array([0.5, 0.1, 0.2, 0.3, 0.4, -1.0])
    ref = (scipy.stats.lognorm.logpdf(0.5, 1.0, loc=-2) + np.sum(scipy.stats.norm.pdf([0.4, -1.0], 0, 1))
           + np.log(np.log(1 + 3.0 * (0.001 / np.exp(-1.0)) ** 2)))
    assert e.lnprob(t) == pytest.approx(ref, rel=1e-14)
    assert np.isfinite(PR.EnvPrior(3, 3, 2).lnprob(np.array([0.5, 0.1, -1.0])))
    assert PR.DefaultPrior(3).lnprob(np.array([0.5, 0.1, 0.0])) == np.inf
    assert PR.DefaultPrior(3).lnprob(np.array([0.0, 0.1, 0.5])) == -np.inf


# ---- the Python dispatch on the fake ---------------------------------------------------------------------------------
class Fake(object):
    """The three entry points on the fake handles: the restatement driven by the oracle likelihood and the host
    priors.  Records every call."""

    def __init__(self, run_chain=True):
        self.calls, self.models, self.run_chain = [], [], run_chain

    def set_hyper_model(self, h, slots, n_terms, mean, tiny, prior_kind=0, prior_par=None, n_ls=0, n_lr=0):
        assert len(h.spec[2]) == n_terms
        h.hyper = dict(slots=list(slots), mean=mean, tiny=tiny, prior=(prior_kind, prior_par, n_ls, n_lr))
        self.models.append(h.hyper)

    def _lnpost(self, h, dim):
        from robo_b200 import _lib
        if len(h.y) > _lib.HYPER_MAX_N:
            raise ValueError("gpk_sample_hypers: n exceeds GPK_HYPER_MAX_N")
        if dim != len(h.hyper["slots"]) + 1:
            raise ValueError("gpk_sample_hypers: dim does not match the slot table")
        family, _, axis, group, lm = h.spec
        flat = dict(family=family, axis=axis, group=group, log_metric=lm, slots=h.hyper["slots"])
        prior = M.prior_object(*h.hyper["prior"], dim=dim)
        return M.oracle_lnpost(h.X, h.y, h.hyper["mean"], flat, prior)

    def sample_hypers(self, h, p0, steps, seed):
        p0 = np.array(p0, dtype=np.float64)
        nw, dim = p0.shape
        if nw % 2 or nw < 2 * dim:
            raise ValueError("gpk_sample_hypers: bad number of walkers")
        self.calls.append(dict(handle=h, p0=p0.copy(), steps=steps, seed=seed))
        if not self.run_chain:
            return dict(pos=p0 + 0.01, lnpost=np.zeros(nw), n_accepted=np.zeros(nw, dtype=np.int64))
        return M.run(self._lnpost(h, dim), p0, steps, seed)


@pytest.fixture
def fake(monkeypatch):
    from robo_b200 import _lib
    from tests import fake_de_es
    fake_de_es.install(monkeypatch)
    f = Fake()
    for name in ("set_hyper_model", "sample_hypers"):
        monkeypatch.setattr(_lib, name, getattr(f, name))
    return f


def _model(sampler="device", prior="default", n_hypers=8, chain=4, burnin=3, **kw):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    p = DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)) if prior == "default" else prior
    return GaussianProcessMCMC(kernel, prior=p, n_hypers=n_hypers, chain_length=chain, burnin_steps=burnin,
                               normalize_input=True, lower=LO, upper=UP, rng=np.random.RandomState(2),
                               hyper_sampler=sampler, **kw)


def test_seed_per_run_burn_in_once_and_bookkeeping(fake):
    from robo_b200 import _lib
    m = _model()
    X, y = _data(10)
    rng = deepcopy(m.rng)
    m.train(X, y)
    assert [c["steps"] for c in fake.calls] == [3, 4]
    assert [c["seed"] for c in fake.calls] == [int(rng.randint(0, 2 ** 63, dtype=np.int64)) for _ in range(2)]
    # p0 of the burn-in comes from the prior (as on the host path), the chain starts where the burn-in ended
    assert np.array_equal(fake.calls[0]["p0"], DefaultPriorSample(8, 4))
    burned = M.run(fake._lnpost(fake.calls[0]["handle"], 4), fake.calls[0]["p0"], 3, fake.calls[0]["seed"])["pos"]
    assert fake.calls[1]["p0"].tobytes() == burned.tobytes()
    final = M.run(fake._lnpost(fake.calls[1]["handle"], 4), burned, 4, fake.calls[1]["seed"])["pos"]
    assert m.hypers.shape == (8, 4) and m.hypers.tobytes() == final.tobytes() and m.p0.tobytes() == final.tobytes()
    assert m.burned and m.n_lnprob_calls == 8 * (3 + 1) + 8 * (4 + 1)
    assert len(m.models) == 8 and all(s.is_trained for s in m.models)
    # the hyper model the device received: slots of the kernel, the mean of y, george's jitter, the default prior
    hm = fake.models[0]
    assert hm["slots"] == [("amp", None), ("metric", [0]), ("metric", [1])]
    assert hm["mean"] == float(np.mean(y)) and hm["tiny"] == 1.25e-12
    assert hm["prior"] == (_lib.PRIOR_DEFAULT, [1.0, 0.0, -10, 2, 0.1, 0.0, 0.0], 0, 0)
    # a later train: no burn-in, one run of chain_length from p0, a new seed
    X2, y2 = _data(12, seed=1)
    m.train(X2, y2)
    assert len(fake.calls) == 3 and fake.calls[2]["steps"] == 4
    assert fake.calls[2]["p0"].tobytes() == final.tobytes()
    assert fake.calls[2]["seed"] == int(rng.randint(0, 2 ** 63, dtype=np.int64))
    assert m.n_lnprob_calls == 8 * (4 + 1)


def DefaultPriorSample(n, dim):
    from robo_b200.priors import DefaultPrior
    return DefaultPrior(dim, rng=np.random.RandomState(1)).sample_from_prior(n)


def test_no_prior_starts_from_the_model_rng(fake):
    m = _model(prior=None)
    rng = deepcopy(m.rng)
    m.train(*_data(10))
    assert np.array_equal(fake.calls[0]["p0"], rng.rand(8, 4))
    assert fake.calls[0]["seed"] == int(rng.randint(0, 2 ** 63, dtype=np.int64))
    assert fake.models[0]["prior"][0] == 0


def test_fallback_above_the_limit_logs_once(fake, monkeypatch, caplog):
    from robo_b200 import _lib
    monkeypatch.setattr(_lib, "HYPER_MAX_N", 9)
    m = _model()
    with caplog.at_level(logging.INFO, logger="robo_b200.models.gaussian_process_mcmc"):
        m.train(*_data(10))
        m.train(*_data(11))
    assert fake.calls == []
    assert len([r for r in caplog.records if "GPK_HYPER_MAX_N" in r.getMessage()]) == 1
    assert m.hypers.shape == (8, 4) and m.burned
    monkeypatch.setattr(_lib, "HYPER_MAX_N", 232)
    m.train(*_data(10))                                    # back under the limit: the device continues from p0
    assert len(fake.calls) == 1 and fake.calls[0]["steps"] == 4


def test_unsupported_prior_or_kernel_raises_type_error(fake):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcessMCMC

    class MyPrior(object):
        def lnprob(self, theta):
            return 0.0

        def sample_from_prior(self, n):
            return np.zeros((n, 4))
    with pytest.raises(TypeError):
        _model(prior=MyPrior())
    _model(prior=MyPrior(), sampler="host")                 # the host sampler takes any prior
    with pytest.raises(TypeError):
        GaussianProcessMCMC(K.Matern52Kernel(np.ones(2), ndim=2) + K.Matern32Kernel(np.ones(2), ndim=2),
                            hyper_sampler="device")
    with pytest.raises(ValueError):
        _model(sampler="gpu")
    # a prior swapped in after construction is refused at the first train
    m = _model()
    m.prior = MyPrior()
    with pytest.raises(TypeError):
        m.train(*_data(10))
    assert fake.calls == []


def test_host_never_reaches_the_device_and_keeps_its_stream(fake):
    a, b = _model(sampler="host"), _model()
    b.hyper_sampler = "host"
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    c = GaussianProcessMCMC(a.kernel, prior=DefaultPrior(4, rng=np.random.RandomState(1)), n_hypers=8, chain_length=4, burnin_steps=3, normalize_input=True,
                            lower=LO, upper=UP, rng=np.random.RandomState(2))
    assert c.hyper_sampler == "host"
    X, y = _data(10)
    for m in (a, b, c):
        m.train(X, y)
    assert fake.calls == [] and fake.models == []
    assert a.hypers.tobytes() == c.hypers.tobytes()
    assert a.rng.get_state()[1].tobytes() == c.rng.get_state()[1].tobytes()


def test_fabolas_model_passes_the_sampler_and_env_prior(fake):
    from robo_b200 import _lib
    from robo_b200 import kernels as K
    from robo_b200.models.fabolas_gp import FabolasGPMCMC
    from robo_b200.priors import EnvPrior
    kernel = 1.0 * K.Matern52Kernel(np.ones(2), ndim=3, axes=[0, 1]) * K.Matern52Kernel(np.ones(1), ndim=3, axes=[2])
    m = FabolasGPMCMC(kernel, basis_func=lambda s: (1 - s) ** 2, prior=EnvPrior(len(kernel) + 1, 2, 1), n_hypers=10,
                      chain_length=2, burnin_steps=2, lower=LO, upper=UP, rng=np.random.RandomState(5),
                      hyper_sampler="device")
    assert m.hyper_sampler == "device"
    rng = np.random.RandomState(0)
    X = np.c_[LO + (UP - LO) * rng.rand(9, 2), rng.uniform(0.1, 1, 9)]
    y = np.array([branin(x) for x in X]) * X[:, 2]
    m.train(X, y)
    assert len(fake.calls) == 2 and m.hypers.shape == (10, 5)
    assert fake.models[0]["prior"] == (_lib.PRIOR_ENV, [1.0, -2, -10, 2, 0.001, 1, 0], 2, 1)
    # the MCMC phase sees the Fabolas-transformed inputs
    h = fake.calls[0]["handle"]
    assert np.array_equal(h.X, m.X) and np.allclose(h.X[:, 2], (1 - X[:, 2]) ** 2)


@pytest.mark.parametrize("facade", ["bayesian_optimization", "entropy_search"])
def test_facades_pass_the_sampler(facade, monkeypatch):
    mod = importlib.import_module("robo_b200.fmin." + facade)
    seen = []

    class Stop(Exception):
        pass

    def stub(*a, **k):
        seen.append(k)
        raise Stop()
    monkeypatch.setattr(mod, "GaussianProcessMCMC", stub)
    fn = getattr(mod, facade)
    with pytest.raises(Stop):
        fn(branin, LO, UP, num_iterations=4, rng=np.random.RandomState(0), hyper_sampler="device")
    with pytest.raises(Stop):
        fn(branin, LO, UP, num_iterations=4, rng=np.random.RandomState(0))
    assert [k["hyper_sampler"] for k in seen] == ["device", "host"]
