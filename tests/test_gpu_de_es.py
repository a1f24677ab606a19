"""Differential evolution over the information-gain acquisitions on the GPU (gpk_es_multi, gpk_maximize_de_es,
gpk_maximize_de_es_cost, DifferentialEvolution over InformationGain / InformationGainPerUnitCost and the entropy_search
facade with maximizer="differential_evolution").

The device evolutions equal tests/de_model.py bit for bit when the restatement is fed the library's own public scoring
calls on the same batches: gpk_es_compute (one model), gpk_es_multi (a marginalised ensemble) and gpk_es_cost_multi
(Fabolas pairs).  gpk_es_multi equals the per-estimator loop of MarginalizationGPMCMC bit for bit: the same kernels,
every candidate independent of the others, and the same sum over models."""
import numpy as np
import pytest

from oracle import robo_oracle as O
from tests import de_model as M
from tests import test_gpu_fabolas_acq as FA
from tests.product_cases import product_kernel

pytestmark = pytest.mark.gpu

LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])


def _branin(x):
    return (x[1] - 5.1 / (4 * np.pi ** 2) * x[0] ** 2 + 5 / np.pi * x[0] - 6) ** 2 \
        + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x[0]) + 10


_CACHE = {}


def _single():
    """InformationGain on one device GP: the N = 512, D = 4 problem of smoke(), whose batches of >= 2048 rows take the
    int8 contraction -> (acq, lower, upper)."""
    if "one" not in _CACHE:
        from robo_b200.acquisition_functions import EI, InformationGain
        from robo_b200.models.gaussian_process import GaussianProcess
        X, y, _, theta, noise = O.synthetic_problem(512, 4, 16, seed_train=11)
        model = GaussianProcess(product_kernel("matern52", theta, 4), noise=noise, normalize_input=False)
        model.train(X, y, do_optimize=False)
        lower, upper = np.zeros(4), np.ones(4)
        ig = InformationGain(model, lower, upper, sampling_acquisition=EI, rng=np.random.RandomState(3))
        ig.update(model)
        _CACHE["one"] = (ig, lower, upper)
    return _CACHE["one"]


def _ensemble():
    """InformationGain marginalised over a 10-model gp_mcmc ensemble on Branin (facade kernel and prior)."""
    if "ten" not in _CACHE:
        from robo_b200 import kernels as K
        from robo_b200.acquisition_functions import EI, InformationGain, MarginalizationGPMCMC
        from robo_b200.models import GaussianProcessMCMC
        from robo_b200.priors import DefaultPrior
        rng = np.random.RandomState(4)
        X = LO + (UP - LO) * rng.rand(20, 2)
        y = np.array([_branin(x) for x in X])
        kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
        model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)),
                                    n_hypers=10, chain_length=20, burnin_steps=20, normalize_input=True,
                                    normalize_output=False, lower=LO, upper=UP, rng=np.random.RandomState(2))
        model.train(X, y, do_optimize=True)
        acq = MarginalizationGPMCMC(InformationGain(model, LO, UP, sampling_acquisition=EI, rng=np.random.RandomState(0)))
        acq.update(model)
        assert len(acq.estimators) == 10
        _CACHE["ten"] = (acq, LO, UP, X)
    return _CACHE["ten"]


def _fabolas(n_pairs):
    """InformationGainPerUnitCost on the fixtures of test_gpu_fabolas_acq.py: one pair, or 12 marginalised pairs."""
    key = "cost%d" % n_pairs
    if key not in _CACHE:
        from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost, MarginalizationGPMCMC
        if n_pairs == 1:
            obj, cost, X = FA._pair()
            acq = FA._ig(obj, cost, overhead=0.1)
        else:
            objm, costm, X = FA._mcmc_pair(n_pairs, 60)
            acq = MarginalizationGPMCMC(InformationGainPerUnitCost(objm, costm, FA.EXT_LO, FA.EXT_UP, FA.IS_ENV,
                                                                   sampling_acquisition=EI,
                                                                   rng=np.random.RandomState(0)))
            np.random.seed(0)
            acq.update(objm, costm, overhead=0.05)
            assert len(acq.estimators) == n_pairs
        _CACHE[key] = (acq, FA.EXT_LO, FA.EXT_UP, X)
    return _CACHE[key]


def _problem(which):
    """-> (acquisition, lower, upper, device run(seed, pop, maxiter), the public scoring call for de_model)."""
    from robo_b200 import _lib
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import device_spec
    kw = dict(mutation=(0.5, 1.0), recombination=0.7, tol=0.01, atol=0.0, want_population=True)
    if which in ("one", "ten"):
        acq, lower, upper = (_single() if which == "one" else _ensemble())[:3]
        estimators = [acq] if which == "one" else acq.estimators
        handles = [e._ready_handle() for e in estimators]
        score = (lambda X: handles[0].es_compute(X)) if which == "one" else (lambda X: _lib.es_multi(handles, X)["values"])
        return acq, lower, upper, lambda s, p, it: _lib.maximize_de_es(handles, s, p, it, lower=lower, upper=upper, **kw), score
    acq, lower, upper = _fabolas(1 if which == "cost1" else 12)[:3]
    ho, hc, lo, up, bo, bc, oh = device_spec([acq] if which == "cost1" else acq.estimators)

    def run(s, p, it):
        return _lib.maximize_de_es_cost(ho, hc, s, p, it, lower=lower, upper=upper, cfg_lower=lo, cfg_upper=up,
                                        basis_objective=bo, basis_cost=bc, overhead=oh, **kw)
    return acq, lower, upper, run, lambda X: _lib.es_cost_multi(ho, hc, X, lo, up, bo, bc, oh)["values"]


def _assert_same(dev, ref):
    assert dev["nit"] == ref["nit"] and dev["nfev"] == ref["nfev"]
    assert dev["population"].tobytes() == ref["population"].tobytes()
    assert dev["energies"].tobytes() == ref["energies"].tobytes()
    assert np.float64(dev["energy"]).tobytes() == np.float64(ref["energy"]).tobytes()
    assert dev["x"].tobytes() == ref["x"].tobytes()


def _candidates(lower, upper, m, seed=5):
    rng = np.random.RandomState(seed)
    C = lower + (upper - lower) * rng.rand(m, lower.size)
    C[0] = upper + 1.0                                       # outside the bounds
    C[1] = lower - 0.5
    return C


# ---- gpk_es_multi ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,m", [(1, 500), (1, 4096), (10, 500), (10, 4096)])
def test_es_multi_bit_identical_to_per_estimator_loop(n, m):
    import torch
    from robo_b200 import _lib
    acq, lower, upper, _ = _ensemble()
    estimators = acq.estimators[:n]
    handles = [e._ready_handle() for e in estimators]
    C = _candidates(lower, upper, m)
    per = np.array([h.es_compute(C) for h in handles])
    ref = _lib.moments_handle().reduce_models(per)
    r = _lib.es_multi(handles, C)
    assert r["values"].tobytes() == ref.tobytes()
    assert r["best_idx"] == int(np.argmax(ref)) and r["best_val"] == ref[r["best_idx"]]
    assert _lib.es_multi(handles, C, want_values=False)["best_idx"] == int(np.argmax(ref))
    # the per-estimator loop of MarginalizationGPMCMC.compute, forced by hand, and the fused path it now takes
    loop = _lib.moments_handle().reduce_models(np.array([e.compute(C) for e in estimators]))
    assert loop.tobytes() == ref.tobytes()
    if n == 10:
        assert acq._es_spec() is not None
        assert acq.compute(C).tobytes() == ref.tobytes() and acq.argmax(C) == int(np.argmax(ref))
    # invariant over the scoring pass's chunking and cluster size
    for key, val in (("chunk", 2048), ("ozcluster", 1), ("chunk", 0), ("ozcluster", 4)):
        for h in handles:
            h.set_option(key, val)
        assert _lib.es_multi(handles, C)["values"].tobytes() == ref.tobytes(), (key, val)
    dX = torch.tensor(C, dtype=torch.float64, device="cuda")
    dout = torch.empty(m, dtype=torch.float64, device="cuda")
    dbest = torch.empty(2, dtype=torch.float64, device="cuda")
    _lib.es_multi_dev(handles, dX.data_ptr(), m, dout.data_ptr(), dbest.data_ptr())
    handles[0].synchronize()
    assert dout.cpu().numpy().tobytes() == ref.tobytes()
    assert int(dbest.cpu().numpy().view(np.int64)[1]) == int(np.argmax(ref))


def test_es_multi_single_model_matches_es_compute():
    from robo_b200 import _lib
    ig, lower, upper = _single()
    h = ig._ready_handle()
    C = _candidates(lower, upper, 3000)
    ref = _lib.moments_handle().reduce_models(h.es_compute(C)[None, :])
    assert _lib.es_multi([h], C)["values"].tobytes() == ref.tobytes()


# ---- the evolutions against de_model -----------------------------------------------------------------------------
CASES = [(w, p) for w in ("one", "ten", "cost1", "cost12") for p in (30, 240)] + [("one", 2048), ("ten", 2048),
                                                                                  ("cost1", 2048)]


@pytest.mark.parametrize("which,pop", CASES)
def test_trajectory_bit_for_bit(which, pop):
    acq, lower, upper, run, score = _problem(which)
    for seed, maxiter in [(3, 0), (4, 1), (5, 2), (6, 20)]:
        dev = run(seed, pop, maxiter)
        ref = M.maximize_de(score, seed, pop, lower, upper, maxiter)
        _assert_same(dev, ref)
        assert dev["nit"] <= maxiter and (maxiter == 0) == (dev["nit"] == 0)
    # the unpolished winner's energy against compute() of the returned point alone
    e = -float(np.asarray(acq.compute(dev["x"][None, :])).ravel()[0])
    if pop < 2048:
        assert np.float64(e).tobytes() == np.float64(dev["energy"]).tobytes()        # both take the fp64 variance
    else:
        # the population's variance came from the int8 contraction, the one-row compute's from fp64: they agree to
        # 1e-10 relative, which moves the entropy change by far less than 1e-8 of its size
        np.testing.assert_allclose(e, dev["energy"], rtol=1e-8, atol=1e-12)


@pytest.mark.parametrize("which", ["one", "ten", "cost1", "cost12"])
def test_maximizer_with_and_without_polish(which):
    from robo_b200.maximizers import DifferentialEvolution
    acq, lower, upper = _problem(which)[:3]
    raw = DifferentialEvolution(acq, lower, upper, n_iters=5, rng=np.random.RandomState(1), polish=False)
    x0 = raw.maximize()
    assert raw.last["polished"] is False and np.all(x0 >= lower) and np.all(x0 <= upper)
    de = DifferentialEvolution(acq, lower, upper, n_iters=5, rng=np.random.RandomState(1))
    x = de.maximize()
    assert x.shape == lower.shape and np.all(x >= lower) and np.all(x <= upper)
    assert de.last["device_energy"] == raw.last["device_energy"]                # same seed, same device run
    value = float(np.asarray(acq.compute(x[None, :])).ravel()[0])
    assert value >= -de.last["device_energy"] - 1e-8 * abs(de.last["device_energy"])


F_OPT_BOUND = {"gp": 10.0, "gp_mcmc": 3.0}


def test_entropy_search_facade_differential_evolution():
    """Branin, seed 1, 12 evaluations with maximizer="differential_evolution": two runs identical, every point inside
    the box.  Measured on one H100 80GB HBM3 at a 400 W power limit: f_opt = 8.336 (gp) and 1.518 (gp_mcmc); the
    bounds leave room above both."""
    from robo_b200.fmin import entropy_search
    for model in ("gp", "gp_mcmc"):
        runs = []
        for _ in range(2):
            np.random.seed(1)
            runs.append(entropy_search(_branin, LO, UP, num_iterations=12, model=model, n_init=3,
                                       maximizer="differential_evolution", rng=np.random.RandomState(1)))
        a, b = runs
        X = np.array(a["X"])
        assert len(X) == 12 and np.all(X >= LO) and np.all(X <= UP)
        assert np.array_equal(X, np.array(b["X"])) and a["f_opt"] == b["f_opt"]
        print("entropy_search differential_evolution", model, "f_opt", a["f_opt"])
        assert a["f_opt"] < F_OPT_BOUND[model]



# ---- argument validation -----------------------------------------------------------------------------------------
def test_argument_validation():
    from robo_b200 import _lib
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import device_spec
    acq, lower, upper, X = _ensemble()
    handles = [e._ready_handle() for e in acq.estimators]
    ok = dict(seed=1, pop=20, maxiter=2, mutation=(0.5, 1.0), recombination=0.7, tol=0.01, atol=0.0, lower=lower,
              upper=upper)
    assert _lib.maximize_de_es(handles, **ok)["nit"] >= 1
    for b in (dict(pop=4), dict(pop=(1 << 24) + 1), dict(maxiter=-1), dict(lower=upper, upper=lower),
              dict(lower=np.array([lower[0], upper[1]]))):
        with pytest.raises(ValueError):
            _lib.maximize_de_es(handles, **dict(ok, **b))
    with pytest.raises(ValueError):                          # a handle listed twice
        _lib.maximize_de_es([handles[0], handles[1], handles[0]], **ok)
    with pytest.raises(ValueError):
        _lib.es_multi([handles[0], handles[0]], X)
    # an objective without gpk_es_update
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    fresh = GaussianProcess(2 * K.Matern52Kernel(np.ones(2), ndim=2), normalize_input=True, lower=LO, upper=UP,
                            rng=np.random.RandomState(0))
    fresh.train(X, np.array([_branin(x) for x in X]), do_optimize=False)
    with pytest.raises(ValueError):
        _lib.maximize_de_es([fresh.gp.handle], **ok)
    with pytest.raises(ValueError):
        _lib.es_multi([handles[0], fresh.gp.handle], X)
    # Fabolas pairs
    cacq, elo, eup, Xf = _fabolas(1)
    ho, hc, lo, up, bo, bc, oh = device_spec([cacq])
    cok = dict(seed=1, pop=20, maxiter=2, mutation=(0.5, 1.0), recombination=0.7, tol=0.01, atol=0.0, lower=elo,
               upper=eup, cfg_lower=lo, cfg_upper=up, basis_objective=bo, basis_cost=bc, overhead=oh)
    assert _lib.maximize_de_es_cost(ho, hc, **cok)["nit"] >= 1
    for b in (dict(pop=4), dict(maxiter=-1), dict(lower=eup, upper=elo), dict(basis_objective=2),
              dict(basis_cost=-1), dict(cfg_lower=lo[:1], cfg_upper=up[:1]), dict(cfg_lower=up, cfg_upper=lo)):
        with pytest.raises(ValueError):
            _lib.maximize_de_es_cost(ho, hc, **dict(cok, **b))
    with pytest.raises(ValueError):                          # the objective handle as its own cost handle
        _lib.maximize_de_es_cost(ho, ho, **cok)
    # refitted since gpk_es_update (last: it invalidates the cached fixtures' states)
    obj = cacq.model
    obj.train(Xf, np.cos(Xf[:, 0]), do_optimize=False)
    with pytest.raises(ValueError):
        _lib.maximize_de_es_cost([obj.gp.handle], hc, **cok)
    m0 = acq.estimators[0].model
    m0.train(m0.X, m0.y + 1.0, do_optimize=False)
    with pytest.raises(ValueError):
        _lib.maximize_de_es([m0.gp.handle] + handles[1:], **ok)
    with pytest.raises(ValueError):
        acq.compute(X)
    _CACHE.clear()
