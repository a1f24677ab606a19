"""hyper_sampler / hyper_optimizer = "device_blocked" without a GPU: option validation and the Python dispatch on the
oracle-backed fake handles, with a fake of the three blocked _lib entry points defined here (the restatements
tests/hyper_model.py and tests/hyperopt_model.py driven by the oracle likelihood, with no limit on N)."""
import importlib
import logging
import os
import re
from copy import deepcopy

import numpy as np
import pytest

from tests import hyper_model as HM
from tests import hyperopt_model as OM
from tests.test_de_es_cpu import LO, UP, _data, branin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_constants_match_the_binding():
    from robo_b200 import _lib
    src = open(os.path.join(ROOT, "include", "gpk.h")).read()
    assert int(re.search(r"#define GPK_HYPER_BLOCKED_MAX_N (\d+)", src).group(1)) == _lib.HYPER_BLOCKED_MAX_N == 8192
    assert int(re.search(r"#define GPK_HYPER_BATCH_BYTES (\d+)L", src).group(1)) == _lib.HYPER_BATCH_BYTES
    binding = open(_lib.__file__).read()
    for name in ("gpk_hyper_lnpost_blocked", "gpk_sample_hypers_blocked", "gpk_optimize_hypers_blocked"):
        assert '"%s"' % name in binding and "int %s(" % name in src


class Fake(object):
    """The three blocked entry points on the fake handles.  Records every call; the non-blocked ones must not be
    reached."""

    def __init__(self):
        self.calls, self.models = [], []

    def set_hyper_model(self, h, slots, n_terms, mean, tiny, prior_kind=0, prior_par=None, n_ls=0, n_lr=0):
        assert len(h.spec[2]) == n_terms
        h.hyper = dict(slots=list(slots), mean=mean, tiny=tiny, prior=(prior_kind, prior_par, n_ls, n_lr))
        self.models.append(h.hyper)

    def _parts(self, h, dim):
        from robo_b200 import _lib
        if not 2 <= len(h.y) <= _lib.HYPER_BLOCKED_MAX_N:
            raise ValueError("gpk_*_blocked: need 2 <= n <= GPK_HYPER_BLOCKED_MAX_N")
        if dim != len(h.hyper["slots"]) + 1:
            raise ValueError("gpk_*_blocked: dim does not match the slot table")
        family, _, axis, group, lm = h.spec
        flat = dict(family=family, axis=axis, group=group, log_metric=lm, slots=h.hyper["slots"])
        prior = HM.prior_object(*h.hyper["prior"], dim=dim)

        def parts(T):
            ll = np.array([HM.oracle_ll(h.X, h.y, h.hyper["mean"], flat, t) for t in T])
            if prior is None:
                return ll, np.zeros(len(T))
            with np.errstate(all="ignore"):
                return ll, np.array([prior.lnprob(t) for t in T])
        return parts, prior is not None

    def hyper_lnpost_blocked(self, h, thetas):
        T = np.atleast_2d(np.asarray(thetas, dtype=np.float64))
        return self._parts(h, T.shape[1])[0](T)

    def sample_hypers_blocked(self, h, p0, steps, seed):
        p0 = np.array(p0, dtype=np.float64)
        nw, dim = p0.shape
        if nw % 2 or nw < 2 * dim:
            raise ValueError("gpk_sample_hypers_blocked: bad number of walkers")
        parts, has_prior = self._parts(h, dim)
        self.calls.append(dict(kind="sample", handle=h, p0=p0.copy(), steps=steps, seed=seed))
        return HM.run(lambda T: HM.post(*parts(T), has_prior=has_prior), p0, steps, seed)

    def optimize_hypers_blocked(self, h, p0, **kw):
        p0 = np.array(p0, dtype=np.float64)
        parts, has_prior = self._parts(h, len(p0))
        self.calls.append(dict(kind="optimize", handle=h, p0=p0.copy()))
        r = OM.run(lambda T: OM.objective(*parts(T), has_prior), p0, maxiter=30)
        return dict(theta=r["x"], f=r["f"], nit=r["nit"], nfev=r["nfev"], status=r["status"], rounds=r["rounds"],
                    noop_rounds=OM.noop_rounds(r["rounds"]))

    def refuse(self, *a, **k):
        raise AssertionError("the blocked path reached a non-blocked entry point")


@pytest.fixture
def fake(monkeypatch):
    from robo_b200 import _lib
    from tests import fake_de_es
    fake_de_es.install(monkeypatch)
    f = Fake()
    for name in ("set_hyper_model", "hyper_lnpost_blocked", "sample_hypers_blocked", "optimize_hypers_blocked"):
        monkeypatch.setattr(_lib, name, getattr(f, name))
    for name in ("hyper_lnpost", "sample_hypers", "optimize_hypers"):
        monkeypatch.setattr(_lib, name, f.refuse)
    return f


def _mcmc(prior="default", n_hypers=8, chain=4, burnin=3, sampler="device_blocked"):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    p = DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)) if prior == "default" else prior
    return GaussianProcessMCMC(kernel, prior=p, n_hypers=n_hypers, chain_length=chain, burnin_steps=burnin,
                               normalize_input=True, lower=LO, upper=UP, rng=np.random.RandomState(2),
                               hyper_sampler=sampler)


def _gp(prior="default", opt="device_blocked", **kw):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    from robo_b200.priors import DefaultPrior
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    p = DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(0)) if prior == "default" else prior
    return GaussianProcess(kernel, prior=p, normalize_input=True, lower=LO, upper=UP, rng=np.random.RandomState(0),
                           hyper_optimizer=opt, **kw)


# ---- the sampler -----------------------------------------------------------------------------------------------------
def test_sampler_seeds_burn_in_p0_and_calls(fake):
    from robo_b200.priors import DefaultPrior
    m = _mcmc()
    X, y = _data(10)
    rng = deepcopy(m.rng)
    m.train(X, y)
    assert [c["steps"] for c in fake.calls] == [3, 4]
    assert [c["seed"] for c in fake.calls] == [int(rng.randint(0, 2 ** 63, dtype=np.int64)) for _ in range(2)]
    assert np.array_equal(fake.calls[0]["p0"], DefaultPrior(4, rng=np.random.RandomState(1)).sample_from_prior(8))
    h = fake.calls[0]["handle"]
    burned = fake.sample_hypers_blocked(h, fake.calls[0]["p0"], 3, fake.calls[0]["seed"])["pos"]
    assert fake.calls[1]["p0"].tobytes() == burned.tobytes()
    assert m.burned and m.n_lnprob_calls == 8 * (3 + 1) + 8 * (4 + 1)
    assert len(m.models) == 8 and all(s.is_trained for s in m.models)
    assert fake.models[0]["tiny"] == 1.25e-12 and fake.models[0]["mean"] == float(np.mean(y))
    final = m.p0.copy()
    del fake.calls[2:]
    m.train(*_data(12, seed=1))                              # a later train: no burn-in, the chain from p0
    assert len(fake.calls) == 3 and fake.calls[2]["steps"] == 4
    assert fake.calls[2]["p0"].tobytes() == final.tobytes()
    assert fake.calls[2]["seed"] == int(rng.randint(0, 2 ** 63, dtype=np.int64))
    assert m.n_lnprob_calls == 8 * (4 + 1)


def test_sampler_has_no_fallback_above_232(fake, caplog):
    from robo_b200 import _lib
    m = _mcmc(chain=1, burnin=1)
    with caplog.at_level(logging.INFO, logger="robo_b200.models.gaussian_process_mcmc"):
        m.train(*_data(_lib.HYPER_MAX_N + 8))
    assert [c["kind"] for c in fake.calls] == ["sample", "sample"]
    assert len(fake.calls[0]["handle"].y) == _lib.HYPER_MAX_N + 8
    assert not [r for r in caplog.records if "GPK_HYPER_MAX_N" in r.getMessage()]


def test_sampler_type_and_value_errors(fake):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcessMCMC

    class MyPrior(object):
        def lnprob(self, theta):
            return 0.0
    with pytest.raises(TypeError, match="device_blocked"):
        _mcmc(prior=MyPrior())
    with pytest.raises(TypeError, match="device_blocked"):
        GaussianProcessMCMC(K.Matern52Kernel(np.ones(2), ndim=2) + K.Matern32Kernel(np.ones(2), ndim=2),
                            hyper_sampler="device_blocked")
    with pytest.raises(ValueError):
        _mcmc(sampler="blocked")
    m = _mcmc()
    m.prior = MyPrior()
    with pytest.raises(TypeError):
        m.train(*_data(10))
    assert fake.calls == []


def test_fabolas_and_mtbo_models_pass_the_value(fake):
    from robo_b200 import kernels as K
    from robo_b200.models.fabolas_gp import FabolasGP, FabolasGPMCMC
    from robo_b200.models.mtbo_gp import MTBOGP, MTBOGPMCMC
    from robo_b200.priors import EnvPrior
    kernel = 1.0 * K.Matern52Kernel(np.ones(2), ndim=3, axes=[0, 1]) * K.Matern52Kernel(np.ones(1), ndim=3, axes=[2])
    m = FabolasGPMCMC(kernel, basis_func=lambda s: (1 - s) ** 2, prior=EnvPrior(len(kernel) + 1, 2, 1), n_hypers=10,
                      chain_length=2, burnin_steps=2, lower=LO, upper=UP, rng=np.random.RandomState(5),
                      hyper_sampler="device_blocked")
    rng = np.random.RandomState(0)
    X = np.c_[LO + (UP - LO) * rng.rand(9, 2), rng.uniform(0.1, 1, 9)]
    m.train(X, np.array([branin(x) for x in X]) * X[:, 2])
    assert [c["kind"] for c in fake.calls] == ["sample", "sample"] and m.hypers.shape == (10, 5)
    assert FabolasGP(kernel, basis_function=lambda s: s, hyper_optimizer="device_blocked").hyper_optimizer == \
        "device_blocked"
    assert MTBOGP(kernel, hyper_optimizer="device_blocked").hyper_optimizer == "device_blocked"
    assert MTBOGPMCMC(kernel, hyper_sampler="device_blocked").hyper_sampler == "device_blocked"


# ---- the optimiser ---------------------------------------------------------------------------------------------------
def test_optimizer_hyper_result_and_p0(fake):
    from robo_b200 import _lib
    m = _gp()
    X, y = _data(10)
    p0 = np.append(m.kernel.get_parameter_vector(), np.log(m.noise))
    m.train(X, y)
    assert [c["kind"] for c in fake.calls] == ["optimize"] and np.array_equal(fake.calls[0]["p0"], p0)
    h = fake.calls[0]["handle"]
    ref = fake.optimize_hypers_blocked(h, p0)
    for key in ("theta", "f", "nit", "nfev", "status", "rounds"):
        assert np.array_equal(m.hyper_result[key], ref[key]), key
    assert np.array_equal(m.hypers, ref["theta"]) and m.noise == np.exp(m.hypers[-1])
    assert fake.models[0]["prior"] == (_lib.PRIOR_DEFAULT, [1.0, 0.0, -10, 2, 0.1, 0.0, 0.0], 0, 0)
    p1 = np.append(m.kernel.get_parameter_vector(), np.log(m.noise))
    m.train(*_data(11, seed=1))
    assert len(fake.calls) == 3 and np.array_equal(fake.calls[2]["p0"], p1)


def test_optimizer_has_no_fallback_above_232(fake, caplog):
    from robo_b200 import _lib
    m = _gp(prior=None)
    with caplog.at_level(logging.INFO, logger="robo_b200.models.gaussian_process"):
        m.train(*_data(_lib.HYPER_MAX_N + 8))
    assert [c["kind"] for c in fake.calls] == ["optimize"]
    assert not [r for r in caplog.records if "GPK_HYPER_MAX_N" in r.getMessage()]


def test_optimizer_type_and_value_errors(fake):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess

    class MyPrior(object):
        def lnprob(self, theta):
            return 0.0
    with pytest.raises(TypeError, match="hyper_optimizer='device_blocked'"):
        _gp(prior=MyPrior())
    with pytest.raises(TypeError, match="hyper_optimizer='device_blocked'"):
        GaussianProcess(K.Matern52Kernel(np.ones(2), ndim=2) + K.Matern32Kernel(np.ones(2), ndim=2),
                        hyper_optimizer="device_blocked")
    with pytest.raises(ValueError, match="use_gradients"):
        _gp(use_gradients=True)
    with pytest.raises(ValueError):
        _gp(opt="blocked")
    assert fake.calls == []


@pytest.mark.parametrize("facade", ["bayesian_optimization", "entropy_search"])
def test_facades_pass_device_blocked(facade, monkeypatch):
    mod = importlib.import_module("robo_b200.fmin." + facade)
    seen = []

    class Stop(Exception):
        pass

    def stub(*a, **k):
        seen.append(k)
        raise Stop()
    monkeypatch.setattr(mod, "GaussianProcessMCMC", stub)
    monkeypatch.setattr(mod, "GaussianProcess", stub)
    fn = getattr(mod, facade)
    with pytest.raises(Stop):
        fn(branin, LO, UP, num_iterations=4, rng=np.random.RandomState(0), hyper_sampler="device_blocked")
    with pytest.raises(Stop):
        fn(branin, LO, UP, num_iterations=4, rng=np.random.RandomState(0), hyper_optimizer="device_blocked",
           **{"model_type" if facade == "bayesian_optimization" else "model": "gp"})
    assert seen[0]["hyper_sampler"] == "device_blocked" and seen[1]["hyper_optimizer"] == "device_blocked"
