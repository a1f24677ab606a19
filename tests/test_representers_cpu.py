"""Representer sampling without a GPU: invariants of the exact restatement (tests/representer_model.py), its agreement
in law with EnsembleSampler, and the Python dispatch of representer_sampler="device" on the oracle-backed fake
(tests/fake_de_es.py), whose _lib.sample_representers is the restatement scored by the fake handles."""
import numpy as np
import pytest
import scipy.stats

from tests import fabolas_acq_model as F
from tests import representer_model as M
from tests.test_de_es_cpu import EXT_LO, EXT_UP, IS_ENV, LO, UP, _fabolas_pair, _gp, _mcmc


# ---- the restatement ---------------------------------------------------------------------------------------------
def _gauss(i, X):
    return -0.5 * np.sum(((X - 0.3) / 0.2) ** 2, axis=1)


def test_partners_from_the_other_half_and_z_in_range():
    lo, up = np.zeros(3), np.ones(3)
    trace = []
    M.sample_one(_gauss, 0, 123, 12, lo, up, steps=30, trace=trace)
    assert len(trace) == 60
    for run, step, half, k, c, z in trace:
        other = np.arange(6) + (6 if half == 0 else 0)
        assert np.all(np.isin(c, other)) and not np.any(np.isin(c, k))
        assert np.all(z >= 1 / M.A) and np.all(z <= M.A)


def test_out_of_box_never_accepted_and_nan_is_minus_inf():
    lo, up = np.array([0.0, 0.0]), np.array([1.0, 2.0])

    def lnp(i, X):                                   # the largest values outside the box, NaN in one corner
        v = np.sum(X, axis=1)
        v[(X[:, 0] < 0.1) & (X[:, 1] < 0.1)] = np.nan
        return v
    for seed in range(5):
        r = M.sample_one(lnp, 0, seed, 10, lo, up, steps=40)
        assert np.all(r["zb"] >= lo) and np.all(r["zb"] <= up)
        assert not np.any(np.isnan(r["lmb"]))
        inside = ~((r["zb"][:, 0] < 0.1) & (r["zb"][:, 1] < 0.1))
        assert np.array_equal(r["lmb"][inside], np.sum(r["zb"][inside], axis=1))


def test_run_counts():
    lo, up = np.zeros(2), np.ones(2)
    assert M.sample_one(lambda i, X: np.full(len(X), -np.inf), 0, 1, 8, lo, up, steps=3, max_runs=5)["runs"] == 5
    assert M.sample_one(lambda i, X: np.full(len(X), -np.inf), 0, 1, 8, lo, up, steps=3, max_runs=2)["runs"] == 2
    r = M.sample_one(_gauss, 0, 1, 8, lo, up, steps=3, max_runs=5)
    assert r["runs"] == 1 and np.all(np.isfinite(r["lmb"]))
    # estimators are independent: the restatement of several equals each alone
    both = M.sample(_gauss, [4, 9], 8, lo, up, steps=5)
    assert both["zb"][1].tobytes() == M.sample_one(_gauss, 1, 9, 8, lo, up, steps=5)["zb"].tobytes()


def test_agreement_in_law_with_ensemble_sampler():
    """A 2-D Gaussian truncated to the box: every 5th final walker of 80 runs of each sampler, two-sample KS per
    coordinate (different random streams: agreement in law only)."""
    from robo_b200.util.ensemble_sampler import EnsembleSampler
    lo, up = np.array([0.0, -1.0]), np.array([1.0, 1.0])

    def lnp(X):
        out = np.full(len(X), -np.inf)
        inside = np.all((X >= lo) & (X <= up), axis=1)
        out[inside] = _gauss(0, X[inside])
        return out
    host, dev = [], []
    rng = np.random.RandomState(0)
    for run in range(80):
        p0 = lo + (up - lo) * rng.uniform(size=(20, 2))
        s = EnsembleSampler(20, 2, lambda x: lnp(x[None])[0], batch_lnpostfn=lnp)
        host.append(s.run_mcmc(p0, 50, rstate0=rng)[0][::5])
        dev.append(M.sample_one(lambda i, X: _gauss(i, X), 0, 1000 + run, 20, lo, up, steps=50)["zb"][::5])
    host, dev = np.concatenate(host), np.concatenate(dev)
    for j in range(2):
        assert scipy.stats.ks_2samp(host[:, j], dev[:, j]).pvalue > 1e-3, j


# ---- the Python dispatch on the fake ---------------------------------------------------------------------------------
def _fake_sample(models, seeds, nb, steps, max_runs, kind, eta, par, lower, upper, fabolas=None):
    from tests import fake_de_es
    lower, upper = np.asarray(lower, float).ravel(), np.asarray(upper, float).ravel()
    n = len(models)
    eta = np.broadcast_to(np.asarray(eta, dtype=np.float64), (n,))
    if n < 1 or len(set(map(id, models))) != n or nb % 2 or nb < 2 * lower.size or nb > 64 or steps < 1 \
            or max_runs < 1 or kind not in (1, 2, 3, 4) or not np.all(lower < upper):
        raise ValueError("gpk_sample_representers: bad arguments")

    def lnp(i, X):
        if fabolas is not None:
            X = fake_de_es._transform(np.c_[X, np.full(len(X), fabolas["env_value"])], fabolas["cfg_lower"],
                                      fabolas["cfg_upper"], fabolas["basis"])
        return models[i].acq(X, kind, float(eta[i]), par)["values"]
    r = M.sample(lnp, [int(s) for s in seeds], nb, lower, upper, steps, max_runs)
    if kind != 1:
        r["n_negative"] = 0
    return r


@pytest.fixture
def calls(monkeypatch):
    from robo_b200 import _lib
    from tests import fake_de_es
    fake_de_es.install(monkeypatch)
    seen = []

    def spy(*a, **k):
        seen.append(dict(models=a[0], seeds=list(a[1]), nb=a[2], kind=a[5], eta=list(a[6]), par=a[7],
                         lower=a[8], upper=a[9], fabolas=k.get("fabolas")))
        return _fake_sample(*a, **k)
    monkeypatch.setattr(_lib, "sample_representers", spy)
    return seen


def _ig(model, sampler="device", sa=None):
    from robo_b200.acquisition_functions import LogEI, InformationGain
    return InformationGain(model, LO, UP, Nb=10, sampling_acquisition=sa or LogEI, rng=np.random.RandomState(3),
                           representer_sampler=sampler)


def _puc(obj, cost, sampler="device", sa=None, is_env=IS_ENV, lo=EXT_LO, up=EXT_UP):
    from robo_b200.acquisition_functions import LogEI, InformationGainPerUnitCost
    return InformationGainPerUnitCost(obj, cost, lo, up, is_env, sampling_acquisition=sa or LogEI, n_representer=10,
                                      rng=np.random.RandomState(3), representer_sampler=sampler)


def test_one_call_for_all_estimators(calls):
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import MarginalizationGPMCMC
    from copy import deepcopy
    mcmc = _mcmc()
    acq = MarginalizationGPMCMC(_ig(mcmc))
    acq.estimators[1].rng = np.random.RandomState(17)
    own = [deepcopy(e.rng).randint(0, 2 ** 63, dtype=np.int64) for e in acq.estimators]
    acq.update(mcmc)
    assert len(calls) == 1
    c = calls[0]
    n = len(mcmc.models)
    assert len(c["models"]) == n and c["nb"] == 10 and c["kind"] == _lib.ACQ_LOG_EI and c["fabolas"] is None
    assert c["seeds"] == own                               # each estimator draws its seed from its own rng
    assert c["seeds"][1] != c["seeds"][0]
    assert c["eta"] == [float(m.get_incumbent()[1]) for m in mcmc.models]
    assert [h for h in c["models"]] == [m.gp.handle for m in mcmc.models]
    for e in acq.estimators:
        assert e.zb.shape == (10, 2) and e.lmb.shape == (10, 1) and e.logP.shape == (10, 1)
    acq.update(mcmc)                                       # one seed draw per update: new seeds
    assert len(calls) == 2 and not set(calls[1]["seeds"]) & set(c["seeds"])
    assert acq.compute(LO + (UP - LO) * np.random.RandomState(0).rand(7, 2)).shape == (7,)


def test_single_estimator_matches_restatement(calls):
    gp = _gp()
    ig = _ig(gp)
    ig.update(gp)
    seed = calls[0]["seeds"][0]
    assert seed == np.random.RandomState(3).randint(0, 2 ** 63, dtype=np.int64)
    h = gp.gp.handle
    eta = float(gp.get_incumbent()[1])
    ref = M.sample_one(lambda i, X: h.acq(X, 2, eta, 0.0)["values"], 0, seed, 10, LO, UP)
    assert ig.zb.tobytes() == ref["zb"].tobytes() and ig.lmb.ravel().tobytes() == ref["lmb"].tobytes()


def test_fabolas_arguments_and_env_column(calls):
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import MarginalizationGPMCMC
    from tests.test_de_es_cpu import _Ensemble
    pairs = [_fabolas_pair(s) for s in (1, 2)]
    om, cm = _Ensemble([p[0] for p in pairs]), _Ensemble([p[1] for p in pairs])
    acq = MarginalizationGPMCMC(_puc(om, cm))
    acq.update(om, cm, overhead=0.1)
    assert len(calls) == 1
    c = calls[0]
    assert len(c["models"]) == 2 and np.array_equal(c["lower"], LO) and np.array_equal(c["upper"], UP)
    fab = c["fabolas"]
    assert fab["basis"] == _lib.BASIS_ONE_MINUS_S_SQ and fab["env_value"] == 1.0
    assert np.array_equal(fab["cfg_lower"], LO) and np.array_equal(fab["cfg_upper"], UP)
    assert c["eta"] == [float(p[0].get_incumbent()[1]) for p in pairs]
    for e in acq.estimators:
        assert e.zb.shape == (10, 3) and np.all(e.zb[:, 2] == 1.0) and e.lmb.shape == (10, 1)
        assert e.overhead == 0.1


def test_errors(calls, monkeypatch):
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import EI, InformationGain
    gp = _gp()
    with pytest.raises(ValueError):
        InformationGain(gp, LO, UP, representer_sampler="gpu")
    with pytest.raises(TypeError):                         # not a closed-form sampling acquisition
        _ig(gp, sa=F.ConstantSampling).update(gp)
    obj, cost = _fabolas_pair()
    with pytest.raises(TypeError):                         # a FabolasGP is not a raw-input GP
        _ig(obj).update(obj)
    with pytest.raises(TypeError):                         # the environment column is not the last one
        _puc(obj, cost, is_env=np.array([1, 0, 0])).update(obj, cost)
    with pytest.raises(TypeError):                         # a plain GP under the per-unit-cost class
        _puc(gp, cost).update(gp, cost)
    # EI with a negative value: ei.py's ValueError
    monkeypatch.setattr(_lib, "sample_representers", lambda *a, **k: dict(_fake_sample(*a, **k), n_negative=2))
    with pytest.raises(ValueError):
        _ig(gp, sa=EI).update(gp)
    # -inf after every run: the per-unit-cost class raises, InformationGain keeps the infinite lmb
    monkeypatch.setattr(_lib, "sample_representers",
                        lambda *a, **k: dict(_fake_sample(*a, **k), lmb=np.full((len(a[0]), a[2]), -np.inf)))
    with pytest.raises(ValueError, match="Could not sample valid representer points! LogEI is -infinity"):
        _puc(obj, cost).update(obj, cost)
    ig = _ig(gp)
    monkeypatch.setattr(ig, "_end_update", lambda h: None)
    ig.update(gp)
    assert np.all(np.isinf(ig.lmb)) and ig.lmb.shape == (10, 1)
    with pytest.raises(ValueError, match="lmb should not be infinite"):
        ig.compute(LO[None, :])


def test_host_default_unchanged(calls, monkeypatch):
    from robo_b200.util import ensemble_sampler
    runs = []
    real = ensemble_sampler.EnsembleSampler.run_mcmc

    def spy(self, *a, **k):
        runs.append(1)
        return real(self, *a, **k)
    monkeypatch.setattr(ensemble_sampler.EnsembleSampler, "run_mcmc", spy)
    from robo_b200.acquisition_functions import LogEI, InformationGain
    gp = _gp()
    a = InformationGain(gp, LO, UP, Nb=10, sampling_acquisition=LogEI, rng=np.random.RandomState(3))
    b = _ig(gp, sampler="host")
    assert a.representer_sampler == "host"
    a.update(gp)
    b.update(gp)
    assert calls == [] and len(runs) == 2
    assert a.zb.tobytes() == b.zb.tobytes() and a.lmb.tobytes() == b.lmb.tobytes()


def test_entropy_search_passes_the_sampler(calls):
    from robo_b200.fmin import entropy_search
    from tests.test_de_es_cpu import branin
    np.random.seed(1)
    r = entropy_search(branin, LO, UP, num_iterations=4, model="gp", n_init=3, rng=np.random.RandomState(1),
                       representer_sampler="device")
    assert len(r["X"]) == 4 and len(calls) >= 1
