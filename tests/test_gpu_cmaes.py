"""gpk_maximize_cmaes* on the GPU: whole runs equal the exact restatement (tests/cmaes_model.py) bit for bit when the
restatement is fed the device's normals (gpk_cmaes_draws) and the library's own one-shot scores of the same rows;
determinism; quality against the device L-BFGS and random sampling; the CMAES class; argument validation."""
import numpy as np
import pytest

from oracle import robo_oracle as O
from tests import cmaes_model as M
from tests import test_gpu_de as DE
from tests import test_gpu_de_es as DES
from tests import test_gpu_esmc as ESMC
from tests import test_gpu_lbfgs as LB
from tests.product_cases import product_kernel

pytestmark = pytest.mark.gpu

KINDS = {"ei": 1, "log_ei": 2, "pi": 3, "lcb": 4}


def _normals(h, seed):
    """The device's normals, fetched 64 generations at a time."""
    cache = {}

    def normals(run, g, lam, d):
        key = (run, g // 64)
        if key not in cache:
            cache[key] = _lib().cmaes_draws(h, seed, run, 64 * (g // 64), 64 * (g // 64) + 64, lam, d)
        return cache[key][g % 64]
    return normals


def _lib():
    from robo_b200 import _lib
    return _lib


def _x0(lower, upper, seed):
    return lower + (upper - lower) * np.random.RandomState(seed).rand(lower.size)


def _assert_same(dev, ref):
    assert dev["stop"].tolist() == ref["stop"].tolist()
    assert dev["nit"].tolist() == ref["nit"].tolist() and dev["nfev"].tolist() == ref["nfev"].tolist()
    assert dev["nfev_total"] == ref["nfev_total"]
    assert np.float64(dev["energy"]).tobytes() == np.float64(ref["energy"]).tobytes()
    assert dev["x"].tobytes() == ref["x"].tobytes()
    for k in ("m", "ps", "pc", "C"):
        assert dev[k].tobytes() == np.asarray(ref[k], dtype=np.float64).tobytes(), k
    assert np.float64(dev["sigma"]).tobytes() == np.float64(ref["sigma"]).tobytes()


def _check(h, score, run, lower, upper, seed, n_func_evals, restarts=0):
    x0 = _x0(lower, upper, seed)
    dev = run(seed, x0, n_func_evals, restarts)
    ref = M.run(score, _normals(h, seed), x0, lower, upper, n_func_evals, restarts)
    _assert_same(dev, ref)
    assert np.all(dev["x"] >= lower) and np.all(dev["x"] <= upper)
    return dev


def _acq(models, kind, d=2):
    handles, etas, lower, upper = (LB._gp(d) if models == "one" else DE._ensemble())[:4]
    k = KINDS[kind]
    par = 1.0 if kind == "lcb" else 0.0
    etas = [0.0] * len(handles) if kind == "lcb" else etas
    run = lambda s, x0, n, r: _lib().maximize_cmaes(handles, k, etas, par, s, x0, lower, upper, n, r)
    return handles[0], DE._acq_fn(handles, k, etas, par), run, lower, upper


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("models", ["one", "ten"])
def test_acquisitions_bit_for_bit(kind, models):
    h, score, run, lower, upper = _acq(models, kind)
    for seed, n in [(3, 60), (4, 600)]:
        dev = _check(h, score, run, lower, upper, seed, n)
        assert dev["nfev_total"] >= min(n, 6)


def test_information_gain_bit_for_bit():
    acq, lower, upper, _, score = DES._problem("one")
    handles = [acq._ready_handle()]
    run = lambda s, x0, n, r: _lib().maximize_cmaes_es(handles, s, x0, lower, upper, n, r)
    _check(handles[0], score, run, lower, upper, 5, 300)


def test_information_gain_mc_bit_for_bit():
    ig, lower, upper, _ = ESMC._single()
    handles = [ig._ready_handle()]
    run = lambda s, x0, n, r: _lib().maximize_cmaes_esmc(handles, s, x0, lower, upper, n, r)
    _check(handles[0], lambda X: handles[0].esmc_compute(X), run, lower, upper, 6, 120)


@pytest.mark.parametrize("which", ["cost1", "cost12"])
def test_information_gain_per_unit_cost_bit_for_bit(which):
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import device_spec
    acq, lower, upper, _, score = DES._problem(which)
    ho, hc, lo, up, bo, bc, oh = device_spec([acq] if which == "cost1" else acq.estimators)
    run = lambda s, x0, n, r: _lib().maximize_cmaes_es_cost(ho, hc, s, x0, lower, upper, lo, up, bo, bc, oh, n, r)
    _check(ho[0], score, run, lower, upper, 7, 200)


_BIG = {}


def _gp64():
    if "g" not in _BIG:
        from robo_b200.models.gaussian_process import GaussianProcess
        X, y, _, theta, noise = O.synthetic_problem(40, 64, 16, seed_train=9)
        model = GaussianProcess(product_kernel("matern52", theta, 64), noise=noise, normalize_input=False)
        model.train(X, y, do_optimize=False)
        model.gp._restore()
        model.gp._push_cfg()
        _BIG["g"] = ([model.gp.handle], [float(model.get_incumbent()[1])], np.zeros(64), np.ones(64), model)
    return _BIG["g"]


@pytest.mark.parametrize("d,n", [(2, 2000), (16, 1500), (64, 800)])
def test_dimensions_bit_for_bit(d, n):
    handles, etas, lower, upper = (_gp64() if d == 64 else LB._gp(d))[:4]
    run = lambda s, x0, nn, r: _lib().maximize_cmaes(handles, 4, [0.0], 1.0, s, x0, lower, upper, nn, r)
    dev = _check(handles[0], DE._acq_fn(handles, 4, [0.0], 1.0), run, lower, upper, 8 + d, n)
    assert dev["nit"][0] >= 3


def test_restarts_bit_for_bit():
    handles, etas, lower, upper = LB._gp(2)[:4]
    run = lambda s, x0, n, r: _lib().maximize_cmaes(handles, 4, [0.0], 1.0, s, x0, lower, upper, n, r)
    dev = _check(handles[0], DE._acq_fn(handles, 4, [0.0], 1.0), run, lower, upper, 21, 20000, restarts=2)
    assert dev["nit"][1] > 0                                             # IPOP ran a second run with 2 lambda
    assert dev["nfev"][1] == 2 * _lib().cmaes_lambda(2) * dev["nit"][1]


def test_deterministic_across_calls_and_int8_schedules():
    """Run 8 of the N = 512, D = 4 problem has lambda = 2048, whose passes take the int8 contraction."""
    handles, etas, lower, upper, _ = DE._single(True)
    h = handles[0]
    x0 = _x0(lower, upper, 1)

    def run(seed):
        return _lib().maximize_cmaes(handles, 1, etas, 0.0, seed, x0, lower, upper, 200000, 8)
    base = run(11)
    assert base["nit"][8] > 0 and h.timings()["launches_ozaki"] >= 1
    _assert_same(run(11), base)
    try:
        for cluster, persist in [(1, 0), (2, 1), (4, 0)]:
            h.set_option("ozcluster", cluster)
            h.set_option("ozpersist", persist)
            _assert_same(run(11), base)
    finally:
        h.set_option("ozcluster", 4)
        h.set_option("ozpersist", 3)
    assert run(12)["x"].tobytes() != base["x"].tobytes()


def test_quality_on_an_lcb_bowl_against_device_lbfgs():
    from robo_b200.acquisition_functions import LCB
    from robo_b200.maximizers import CMAES
    from robo_b200.models.gaussian_process import GaussianProcess
    from robo_b200 import kernels as K
    rng = np.random.RandomState(0)
    lower, upper = np.zeros(3), np.ones(3)
    X = rng.rand(30, 3)
    y = np.sum((X - 0.4) ** 2, axis=1)
    model = GaussianProcess(2 * K.Matern52Kernel(np.ones(3) * 0.5, ndim=3), normalize_input=True, lower=lower,
                            upper=upper, rng=np.random.RandomState(1))
    model.train(X, y, do_optimize=False)
    acq = LCB(model, par=0.0)                                         # the posterior mean: a smooth bowl around 0.4
    handles, etas, par = [model.gp.handle], [0.0], float(acq.par)
    lb = _lib().maximize_lbfgs(handles, 4, etas, par, lower + (upper - lower) * rng.rand(64, 3), lower, upper)
    best = float(np.min(lb["energy"]))
    cm = CMAES(acq, lower, upper, rng=np.random.RandomState(2))
    x = cm.maximize()
    e = -float(acq.compute(x[None, :]).ravel()[0])
    assert x.shape == (3,) and np.all(x >= lower) and np.all(x <= upper)
    assert e <= best + 1e-4 * max(1.0, abs(best)), (e, best, cm.last)


def test_quality_on_branin_ei_against_random_sampling():
    """EI on Branin is multi-modal.  At the class defaults (1000 evaluations, no restarts) the single run stops on
    tolfun in a local maximum whose energy is above the best of the 65,536 random candidates (on an H100:
    -2.1559 after 624 evaluations, against -2.4010); IPOP restarts (cma.fmin's ``restarts``) take CMA-ES out of it
    (-2.4099 after 5,256 evaluations over five runs).  With the same rng, the defaults' run is a prefix of the first IPOP
    run (same seed, start point and normals), so the IPOP result is never worse than the defaults'."""
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import CMAES
    handles, etas, lower, upper, model = DE._single(False)
    acq = EI(model)
    n = 65536
    inc = model.get_incumbent()[0]
    xr, _, _ = handles[0].maximize_random(2024, 0, n, n, lower, upper, inc, 0.1, 1, etas[0], 0.0)
    er = -float(acq.compute(xr[None, :]).ravel()[0])
    default = CMAES(acq, lower, upper, rng=np.random.RandomState(0))
    xd = default.maximize()
    assert xd.shape == (2,) and np.all(xd >= lower) and np.all(xd <= upper) and np.isfinite(default.last["best_energy"])
    cm = CMAES(acq, lower, upper, restarts=4, n_func_evals=20000, rng=np.random.RandomState(0))
    x = cm.maximize()
    assert x.shape == (2,) and np.all(x >= lower) and np.all(x <= upper)
    assert cm.last["best_energy"] <= er, (cm.last, er)
    assert cm.last["best_energy"] <= default.last["best_energy"]
    np.testing.assert_allclose(-acq.compute(x[None, :]).ravel()[0], cm.last["best_energy"], rtol=1e-12)


def test_conditioncov_bit_for_bit():
    """A GP whose posterior mean is steep in x0 and nearly flat in x1 (length scales 0.3 and 1e6, outputs scaled by
    1e8 so that tolfun stays out of reach): the device run stops on conditioncov, when the ratio of C's extreme
    eigenvalues passes 1e14, in the generation the restatement does."""
    from robo_b200 import kernels as K
    from robo_b200.models.gaussian_process import GaussianProcess
    lower, upper = np.zeros(2), np.ones(2)
    X = np.random.RandomState(0).rand(12, 2)
    scale = 1e8
    model = GaussianProcess((scale ** 2) * K.Matern52Kernel(np.array([0.3 ** 2, 1e6 ** 2]), ndim=2),
                            noise=1e-6 * scale ** 2, normalize_input=False, normalize_output=False)
    model.train(X, scale * (X[:, 0] - 0.5) ** 2, do_optimize=False)
    model.gp._restore()
    model.gp._push_cfg()
    handles = [model.gp.handle]
    run = lambda s, x0, n, r: _lib().maximize_cmaes(handles, 4, [0.0], 0.0, s, x0, lower, upper, n, r)
    dev = _check(handles[0], DE._acq_fn(handles, 4, [0.0], 0.0), run, lower, upper, 2, 10 ** 6)
    assert dev["stop"].tolist() == [_lib().CMA_CONDITIONCOV]
    ev = M.jacobi(dev["C"])[0]
    assert 1e14 < ev.max() / ev.min() < 1e16


def test_marginalised_and_entropy_search_maximizers_end_to_end():
    from robo_b200.maximizers import CMAES
    handles, etas, lower, upper, acq = DE._ensemble()
    cm = CMAES(acq, lower, upper, rng=np.random.RandomState(1))
    x = cm.maximize()
    np.testing.assert_allclose(-acq.compute(x[None, :]).ravel()[0], cm.last["best_energy"], rtol=1e-12)
    ig, lower, upper = DES._problem("one")[:3]
    cm = CMAES(ig, lower, upper, n_func_evals=200, rng=np.random.RandomState(1))
    x = cm.maximize()
    assert x.shape == lower.shape and np.all(x >= lower) and np.all(x <= upper)
    np.testing.assert_allclose(-ig.compute(x[None, :]).ravel()[0], cm.last["best_energy"], rtol=1e-12)


def test_two_dim_maximizer_shape():
    """test/test_maximizers/test_maximizers_two_dim.py's shape check on the device."""
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import CMAES
    handles, etas, lower, upper, model = DE._single(False)
    cm = CMAES(EI(model), lower, upper, n_func_evals=10, rng=np.random.RandomState(0))
    x = cm.maximize()
    assert x.shape == (2,) and np.all(x >= lower) and np.all(x <= upper)


def test_argument_validation():
    from robo_b200 import _lib
    handles, etas, lower, upper = LB._gp(2)[:4]
    h = handles[0]
    ok = dict(kind=1, eta=etas, par=0.0, seed=1, x0=_x0(lower, upper, 0), lower=lower, upper=upper, n_func_evals=30,
              restarts=0)
    assert _lib.maximize_cmaes(handles, **ok)["nfev_total"] >= 30
    bad = [dict(lower=upper, upper=lower), dict(lower=np.array([lower[0], upper[1]])), dict(x0=np.array([np.nan, 0.5])),
           dict(x0=upper + 1.0), dict(sigma0=0.0), dict(sigma0=-1.0), dict(n_func_evals=0), dict(restarts=-1),
           dict(restarts=9), dict(kind=0), dict(kind=5)]
    for b in bad:
        with pytest.raises(ValueError):
            _lib.maximize_cmaes(handles, **dict(ok, **b))
    with pytest.raises(ValueError):
        _lib.maximize_cmaes([h, h], **dict(ok, eta=[etas[0]] * 2))
    h1 = LB._gp(1)[0]
    # d > GPK_CMA_MAX_D cannot occur: a handle holds at most GPK_MAX_TERMS = 64 input dimensions
    with pytest.raises(ValueError):                                    # d < 2
        _lib.maximize_cmaes(h1, **dict(ok, eta=[0.0], x0=[0.5], lower=[0.0], upper=[1.0]))
    with pytest.raises(ValueError):
        _lib.cmaes_draws(h, 1, 0, 3, 3, 6, 2)
