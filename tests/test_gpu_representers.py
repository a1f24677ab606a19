"""Representer points on the device (gpk_sample_representers, representer_sampler="device").

The device's walkers, log-probabilities, run counts and accept counts equal tests/representer_model.py bit for bit when
the restatement is fed the library's own public scoring calls on the half-batches the device scored: handle.acq of the
walker rows, and for Fabolas handle.acq of FabolasGP.normalize([x, env]).  Setups: one Branin GP, the 10-model
entropy_search ensemble (EI and LogEI) and a small Fabolas pair ensemble."""
import numpy as np
import pytest

from tests import representer_model as M
from tests import test_gpu_fabolas_acq as FA

pytestmark = pytest.mark.gpu

LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])


def _branin(x):
    return (x[1] - 5.1 / (4 * np.pi ** 2) * x[0] ** 2 + 5 / np.pi * x[0] - 6) ** 2 \
        + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x[0]) + 10


def _data(n=20, seed=4):
    rng = np.random.RandomState(seed)
    X = LO + (UP - LO) * rng.rand(n, 2)
    return X, np.array([_branin(x) for x in X])


_CACHE = {}


def _gp():
    if "gp" not in _CACHE:
        from robo_b200 import kernels as K
        from robo_b200.models import GaussianProcess
        X, y = _data()
        gp = GaussianProcess(2 * K.Matern52Kernel(np.ones(2), ndim=2), normalize_input=True, lower=LO, upper=UP,
                             rng=np.random.RandomState(1))
        gp.train(X, y, do_optimize=True)
        _CACHE["gp"] = gp
    return _CACHE["gp"]


def _mcmc():
    if "mcmc" not in _CACHE:
        from robo_b200 import kernels as K
        from robo_b200.models import GaussianProcessMCMC
        from robo_b200.priors import DefaultPrior
        X, y = _data()
        kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
        model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)),
                                    n_hypers=10, chain_length=20, burnin_steps=20, normalize_input=True,
                                    normalize_output=False, lower=LO, upper=UP, rng=np.random.RandomState(2))
        model.train(X, y, do_optimize=True)
        assert len(model.models) == 10
        _CACHE["mcmc"] = model
    return _CACHE["mcmc"]


def _fabolas():
    if "fab" not in _CACHE:
        objm, costm, X = FA._mcmc_pair(10, 60)
        _CACHE["fab"] = (objm, costm, X)
    return _CACHE["fab"]


def _handles(models):
    for m in models:
        m.gp._restore()
        m.gp._push_cfg()
    return [m.gp.handle for m in models]


def _setup(which, kind):
    """-> (models, handles, etas, lower, upper, fabolas dict or None, lnp_fn for the restatement)."""
    from robo_b200 import _lib
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import basis_code
    k = _lib.ACQ_KIND[kind]
    if which == "one":
        models = [_gp()]
    elif which == "ten":
        models = list(_mcmc().models)
    else:
        models = list(_fabolas()[0].models)
    hs = _handles(models)
    etas = [0.0 if kind == "lcb" else float(m.get_incumbent()[1]) for m in models]
    par = 0.0
    if which != "fab":
        def lnp(i, X):
            return hs[i].acq(X, k, etas[i], par)["values"]
        return models, hs, etas, LO, UP, None, lnp
    env = float(FA.EXT_UP[-1])
    fab = dict(cfg_lower=models[0].lower, cfg_upper=models[0].upper, basis=basis_code(models[0].basis_function),
               env_value=env)

    def lnp(i, X):
        return hs[i].acq(models[i].normalize(np.c_[X, np.full(len(X), env)]), k, etas[i], par)["values"]
    return models, hs, etas, LO, UP, fab, lnp


def _run(hs, seeds, etas, kind, lower, upper, fab, nb=50, steps=50, max_runs=5):
    from robo_b200 import _lib
    return _lib.sample_representers(hs, seeds, nb, steps, max_runs, _lib.ACQ_KIND[kind], etas, 0.0, lower, upper,
                                    fabolas=fab)


def _assert_same(dev, ref):
    assert dev["runs"].tolist() == ref["runs"].tolist()
    assert dev["zb"].tobytes() == ref["zb"].tobytes()
    assert dev["lmb"].tobytes() == ref["lmb"].tobytes()
    assert dev["n_accepted"].tolist() == ref["n_accepted"].tolist()


CASES = [("one", "log_ei", 50, 50), ("one", "ei", 20, 10), ("one", "pi", 4, 3), ("one", "lcb", 6, 5),
         ("ten", "ei", 50, 50), ("ten", "log_ei", 50, 50), ("fab", "ei", 50, 20), ("fab", "log_ei", 50, 50)]


@pytest.mark.parametrize("which,kind,nb,steps", CASES)
def test_bit_for_bit(which, kind, nb, steps):
    models, hs, etas, lower, upper, fab, lnp = _setup(which, kind)
    seeds = [1000 + 7 * i for i in range(len(hs))]
    dev = _run(hs, seeds, etas, kind, lower, upper, fab, nb=nb, steps=steps)
    ref = M.sample(lnp, seeds, nb, lower, upper, steps=steps)
    assert dev["zb"].shape == (len(hs), nb, 2) and dev["lmb"].shape == (len(hs), nb)
    _assert_same(dev, ref)
    assert dev["n_negative"] == (ref["n_negative"] if kind == "ei" else 0)
    assert np.all(dev["zb"] >= lower) and np.all(dev["zb"] <= upper)
    assert np.all(dev["n_accepted"] <= steps)
    if steps >= 10:
        assert dev["n_accepted"].sum() > 0


def test_independent_of_list_order_and_repeat():
    models, hs, etas, lower, upper, fab, _ = _setup("ten", "log_ei")
    seeds = np.arange(10, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(3)
    a = _run(hs, seeds, etas, "log_ei", lower, upper, fab, steps=20)
    b = _run(hs, seeds, etas, "log_ei", lower, upper, fab, steps=20)
    for key in ("zb", "lmb", "runs", "n_accepted"):
        assert a[key].tobytes() == b[key].tobytes(), key
    perm = np.random.RandomState(0).permutation(10)
    c = _run([hs[i] for i in perm], seeds[perm], [etas[i] for i in perm], "log_ei", lower, upper, fab, steps=20)
    for key in ("zb", "lmb", "runs", "n_accepted"):
        assert c[key].tobytes() == a[key][perm].tobytes(), key
    # one estimator alone: its own result
    one = _run([hs[3]], seeds[3:4], etas[3:4], "log_ei", lower, upper, fab, steps=20)
    assert one["zb"][0].tobytes() == a["zb"][3].tobytes() and one["lmb"][0].tobytes() == a["lmb"][3].tobytes()


def test_restart_path():
    models, hs, etas, lower, upper, fab, lnp = _setup("ten", "log_ei")
    bad = [-1e300] * 3
    seeds = [5, 6, 7]
    dev = _run(hs[:3], seeds, bad, "log_ei", lower, upper, fab, steps=3)
    assert dev["runs"].tolist() == [5, 5, 5] and np.all(np.isinf(dev["lmb"]))
    from robo_b200 import _lib
    k = _lib.ACQ_KIND["log_ei"]
    ref = M.sample(lambda i, X: hs[i].acq(X, k, bad[i], 0.0)["values"], seeds, 50, lower, upper, steps=3)
    _assert_same(dev, ref)
    # mixed: estimators that are finite after the first run keep it while the others run again
    mixed = _run(hs[:3], seeds, [etas[0], bad[1], etas[2]], "log_ei", lower, upper, fab, steps=3)
    assert mixed["runs"].tolist() == [1, 5, 1]
    solo = _run([hs[2]], seeds[2:], [etas[2]], "log_ei", lower, upper, fab, steps=3)
    assert solo["zb"][0].tobytes() == mixed["zb"][2].tobytes()
    # Fabolas: the reference's ValueError
    from robo_b200.acquisition_functions import LogEI, InformationGainPerUnitCost
    objm, costm, _ = _fabolas()
    ig = InformationGainPerUnitCost(objm.models[0], costm.models[0], FA.EXT_LO, FA.EXT_UP, FA.IS_ENV,
                                    sampling_acquisition=LogEI, rng=np.random.RandomState(0),
                                    representer_sampler="device")
    ig.sampling_acquisition.par = 1e300
    with pytest.raises(ValueError, match="Could not sample valid representer points"):
        ig.update(objm.models[0], costm.models[0])


def test_acquisition_classes_take_the_device_path(monkeypatch):
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import EI, InformationGain, InformationGainPerUnitCost, MarginalizationGPMCMC
    calls = []
    real = _lib.sample_representers

    def spy(*a, **k):
        calls.append(len(a[0]))
        return real(*a, **k)
    monkeypatch.setattr(_lib, "sample_representers", spy)
    model = _mcmc()
    acq = MarginalizationGPMCMC(InformationGain(model, LO, UP, sampling_acquisition=EI, rng=np.random.RandomState(0),
                                                representer_sampler="device"))
    acq.update(model)
    assert calls == [10]
    for e in acq.estimators:
        assert e.zb.shape == (50, 2) and e.lmb.shape == (50, 1) and np.all(np.isfinite(e.lmb))
    C = LO + (UP - LO) * np.random.RandomState(1).rand(200, 2)
    v = acq.compute(C)
    assert v.shape == (200,) and np.all(np.isfinite(v))
    objm, costm, _ = _fabolas()
    pacq = MarginalizationGPMCMC(InformationGainPerUnitCost(objm, costm, FA.EXT_LO, FA.EXT_UP, FA.IS_ENV,
                                                           sampling_acquisition=EI, rng=np.random.RandomState(0),
                                                           representer_sampler="device"))
    pacq.update(objm, costm, overhead=0.05)
    assert calls == [10, 10]
    for e in pacq.estimators:
        assert e.zb.shape == (50, 3) and np.all(e.zb[:, 2] == 1.0) and np.all(np.isfinite(e.lmb))
    w = pacq.compute(np.c_[C, np.full(200, 0.5)])
    assert w.shape == (200,) and np.all(np.isfinite(w))


def test_agreement_in_law_with_host_sampler():
    """Final walkers of 60 host runs against 60 device runs on one Branin GP (LogEI), every 10th walker of each run
    pooled (the walkers of one run are correlated): two-sample KS per coordinate.  The two paths use different random
    streams, so they agree in law only."""
    import scipy.stats
    from robo_b200.acquisition_functions import LogEI, InformationGain
    gp = _gp()
    pooled = {}
    for sampler in ("host", "device"):
        ig = InformationGain(gp, LO, UP, Nb=50, sampling_acquisition=LogEI, rng=np.random.RandomState(11),
                             representer_sampler=sampler)
        pts = []
        for _ in range(60):
            ig.model = gp
            ig.sample_representer_points()
            pts.append(ig.zb[::10])
        pooled[sampler] = np.concatenate(pts)
    for j in range(2):
        p = scipy.stats.ks_2samp(pooled["host"][:, j], pooled["device"][:, j]).pvalue
        print("KS coordinate", j, "p =", p)
        assert p > 1e-3


def test_argument_validation():
    from robo_b200 import _lib
    models, hs, etas, lower, upper, _, _ = _setup("ten", "ei")
    ok = dict(seeds=[1, 2], nb=10, steps=2, max_runs=1, kind=_lib.ACQ_EI, eta=etas[:2], par=0.0, lower=lower,
              upper=upper)
    assert _lib.sample_representers(hs[:2], **ok)["zb"].shape == (2, 10, 2)
    for b in (dict(nb=11), dict(nb=2), dict(nb=66), dict(steps=0), dict(max_runs=0), dict(kind=0), dict(kind=5),
              dict(lower=upper, upper=lower), dict(lower=np.array([lower[0], upper[1]])),
              dict(lower=lower[:1], upper=upper[:1]),
              dict(lower=np.r_[lower, 0.0], upper=np.r_[upper, 1.0])):
        with pytest.raises(ValueError):
            _lib.sample_representers(hs[:2], **dict(ok, **b))
    with pytest.raises(ValueError):                          # a handle listed twice
        _lib.sample_representers([hs[0], hs[1], hs[0]], **dict(ok, seeds=[1, 2, 3], eta=etas[:3]))
    with pytest.raises(ValueError):
        _lib.sample_representers([], **ok)
    # a handle of another input dimension, an unfitted handle
    objm = _fabolas()[0]
    fh = _handles(objm.models[:1])
    with pytest.raises(ValueError):
        _lib.sample_representers([hs[0], fh[0]], **ok)
    fresh = _lib.Handle(0)
    with pytest.raises(ValueError):
        _lib.sample_representers([hs[0], fresh], **ok)
    fresh.close()
    # Fabolas arguments
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import basis_code
    fab = dict(cfg_lower=LO, cfg_upper=UP, basis=basis_code(objm.models[0].basis_function), env_value=1.0)
    fok = dict(ok, seeds=[1], eta=[0.0])
    assert _lib.sample_representers(fh, fabolas=fab, **fok)["zb"].shape == (1, 10, 2)
    for b in (dict(basis=2), dict(basis=-1), dict(cfg_lower=UP, cfg_upper=LO)):
        with pytest.raises(ValueError):
            _lib.sample_representers(fh, fabolas=dict(fab, **b), **fok)
    with pytest.raises(ValueError):                          # dw = d for a Fabolas call
        _lib.sample_representers(fh, fabolas=dict(fab, cfg_lower=np.r_[LO, 0.0], cfg_upper=np.r_[UP, 1.0]),
                                 **dict(fok, lower=np.r_[LO, 0.0], upper=np.r_[UP, 1.0]))
    with pytest.raises(ValueError):                          # dw = d - 1 without fabolas
        _lib.sample_representers(fh, **fok)
