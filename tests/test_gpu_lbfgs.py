"""gpk_maximize_lbfgs* on the GPU: the device run equals the exact restatement (tests/lbfgs_model.py) bit for bit, for
every start (x, energy, nit, nfev, status), when the restatement is fed the library's own public scoring calls on the
same batches: EI / LogEI / PI / LCB on one GP and on a marginalised GP-MCMC, InformationGain alone and marginalised,
InformationGainPerUnitCost on Fabolas models, and the posterior mean and mean + std, at D in {1, 2, 16} and
R in {1, 10, 64} starts.  Then the posterior optimisation on a device GP trained on the reference's quadratic,
DifferentialEvolution(polish="device"), SciPyOptimizer end to end and argument validation."""
import numpy as np
import pytest

from oracle import robo_oracle as O
from tests import lbfgs_model as M
from tests import test_gpu_de as DE
from tests import test_gpu_de_es as DES
from tests.product_cases import product_kernel

pytestmark = pytest.mark.gpu

KINDS = {"ei": 1, "log_ei": 2, "pi": 3, "lcb": 4}
_CACHE = {}


def _gp(d):
    """One fitted device GP of input dimension d on the synthetic problem -> (handles, etas, lower, upper, model)."""
    if d == 2:
        return DE._single(False)
    if d not in _CACHE:
        from robo_b200.models.gaussian_process import GaussianProcess
        X, y, _, theta, noise = O.synthetic_problem(200 if d == 16 else 40, d, 16, seed_train=3 + d)
        model = GaussianProcess(product_kernel("matern52", theta, d), noise=noise, normalize_input=False)
        model.train(X, y, do_optimize=False)
        model.gp._restore()
        model.gp._push_cfg()
        _CACHE[d] = ([model.gp.handle], [float(model.get_incumbent()[1])], np.zeros(d), np.ones(d), model)
    return _CACHE[d]


def _acq_problem(models, d, kind):
    from robo_b200 import _lib
    handles, etas, lower, upper = (_gp(d) if models == "one" else DE._ensemble())[:4]
    k = KINDS[kind]
    par = 1.0 if kind == "lcb" else 0.0
    etas = [0.0] * len(handles) if kind == "lcb" else etas
    score = DE._acq_fn(handles, k, etas, par)
    return lower, upper, lambda X: -score(X), \
        lambda x0: _lib.maximize_lbfgs(handles, k, etas, par, x0, lower, upper)


def _posterior_problem(models, d, kind):
    from robo_b200 import _lib
    handles, _, lower, upper = (_gp(d) if models == "one" else DE._ensemble())[:4]
    obj = _lib.OBJ_MEAN if kind == "mean" else _lib.OBJ_MEAN_STD

    def energy(X):
        r = _lib.acq_multi(handles, X, 1)
        return r["mean"] if kind == "mean" else r["mean"] + np.sqrt(r["var"])
    return lower, upper, energy, lambda x0: _lib.maximize_lbfgs(handles, obj, None, 0.0, x0, lower, upper)


def _es_problem(which):
    from robo_b200 import _lib
    acq, lower, upper, _, score = DES._problem(which)
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import device_spec
    if which in ("one", "ten"):
        handles = [e._ready_handle() for e in ([acq] if which == "one" else acq.estimators)]
        run = lambda x0: _lib.maximize_lbfgs_es(handles, x0, lower, upper)
    else:
        ho, hc, lo, up, bo, bc, oh = device_spec([acq] if which == "cost1" else acq.estimators)
        run = lambda x0: _lib.maximize_lbfgs_es_cost(ho, hc, x0, lower, upper, cfg_lower=lo, cfg_upper=up,
                                                     basis_objective=bo, basis_cost=bc, overhead=oh)
    return lower, upper, lambda X: -score(X), run


def _starts(lower, upper, R, seed):
    rng = np.random.RandomState(seed)
    x0 = lower + (upper - lower) * rng.rand(R, lower.size)
    if R > 2:
        x0[1] = upper + 0.5                                    # clipped onto the upper corner
        x0[2, 0] = lower[0]                                    # on a bound
    return x0


def _assert_same(dev, ref):
    assert dev["status"].tolist() == ref["status"].tolist()
    assert dev["nit"].tolist() == ref["nit"].tolist() and dev["nfev"].tolist() == ref["nfev"].tolist()
    assert dev["energy"].tobytes() == ref["energy"].tobytes()
    assert dev["x"].tobytes() == ref["x"].tobytes()


def _check(problem, R, seed=1):
    lower, upper, energy, run = problem
    x0 = _starts(lower, upper, R, seed)
    dev = run(x0)
    ref = M.minimize(energy, x0, lower, upper)
    _assert_same(dev, ref)
    assert np.all(dev["x"] >= lower) and np.all(dev["x"] <= upper)
    return dev


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("models", ["one", "ten"])
def test_acquisitions_bit_for_bit(kind, models):
    dev = _check(_acq_problem(models, 2, kind), 10)
    # EI and PI of the single Branin GP are flat to below pgtol at these starts: every start stops after the first round
    if models == "ten" or kind in ("log_ei", "lcb"):
        assert np.any(dev["nit"] > 0)


@pytest.mark.parametrize("d,R", [(1, 1), (1, 10), (1, 64), (2, 1), (2, 64), (16, 1), (16, 10), (16, 64)])
def test_shapes_bit_for_bit(d, R):
    _check(_acq_problem("one", d, "log_ei"), R, seed=d + R)


@pytest.mark.parametrize("which", ["one", "ten", "cost1", "cost12"])
def test_information_gain_bit_for_bit(which):
    _check(_es_problem(which), 10)


@pytest.mark.parametrize("kind", ["mean", "mean_std"])
@pytest.mark.parametrize("models,d", [("one", 2), ("one", 16), ("ten", 2)])
def test_posterior_bit_for_bit(kind, models, d):
    _check(_posterior_problem(models, d, kind), 10)


def test_deterministic_and_maxiter_zero():
    problem = _acq_problem("ten", 2, "log_ei")
    lower, upper, _, run = problem
    x0 = _starts(lower, upper, 10, 4)
    a, b = run(x0), run(x0)
    _assert_same(a, b)
    from robo_b200 import _lib
    handles, etas = DE._ensemble()[:2]
    r = _lib.maximize_lbfgs(handles, 2, etas, 0.0, x0, lower, upper, maxiter=0)
    np.testing.assert_array_equal(r["x"], np.clip(x0, lower, upper))
    assert np.all(r["nit"] == 0) and np.all(r["nfev"] == 3)


@pytest.mark.parametrize("which", ["mean", "mean_std"])
def test_posterior_optimization_on_the_quadratic(which):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    from robo_b200.util import posterior_mean_optimization, posterior_mean_plus_std_optimization
    g = np.linspace(0.0, 1.0, 5)
    X = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)       # symmetric about (0.5, 0.5): so is the posterior
    y = np.sum((0.5 - X) ** 2, axis=1)
    model = GaussianProcess(1.0 * K.ExpSquaredKernel(np.ones(2), ndim=2), noise=1e-6, lower=np.zeros(2),
                            upper=np.ones(2), rng=np.random.RandomState(0))
    model.train(X, y, do_optimize=False)
    fn = posterior_mean_optimization if which == "mean" else posterior_mean_plus_std_optimization
    np.random.seed(0)
    x = fn(model, np.array([0, 0]), np.array([1, 1]), with_gradients=False)
    np.testing.assert_almost_equal(x, [0.5, 0.5], decimal=5)


@pytest.mark.parametrize("which", ["acq", "es"])
def test_differential_evolution_device_polish_no_worse(which):
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DifferentialEvolution
    if which == "acq":
        acq, lower, upper = EI(DE._single(False)[4]), DE._single(False)[2], DE._single(False)[3]
    else:
        acq, lower, upper = DES._ensemble()[:3]
    plain = DifferentialEvolution(acq, lower, upper, rng=np.random.RandomState(2), polish=False)
    plain.maximize()
    dev = DifferentialEvolution(acq, lower, upper, rng=np.random.RandomState(2), polish="device")
    x = dev.maximize()
    assert dev.last["best_energy"] <= plain.last["best_energy"]
    assert np.all(x >= lower) and np.all(x <= upper)
    np.testing.assert_allclose(-np.ravel(acq.compute(x[None, :]))[0], dev.last["best_energy"], rtol=1e-10)


def test_scipy_optimizer_end_to_end():
    from robo_b200.acquisition_functions import LogEI
    from robo_b200.maximizers import SciPyOptimizer
    handles, etas, lower, upper, model = DE._single(False)
    acq = LogEI(model)
    opt = SciPyOptimizer(acq, lower, upper, rng=np.random.RandomState(0))
    x = opt.maximize()
    assert opt.last["device"] and x.shape == (2,) and np.all(x >= lower) and np.all(x <= upper)
    np.testing.assert_allclose(-acq.compute(x[None, :]).ravel()[0], opt.last["energy"].min(), rtol=1e-10)
    starts = opt.last["starts"]
    ref = M.minimize(lambda X: -acq.compute(X).ravel(), starts, lower, upper)
    assert opt.last["energy"].min() <= ref["energy"].min() * (1 - 1e-9) or \
        np.isclose(opt.last["energy"].min(), ref["energy"].min(), rtol=1e-9)


def test_argument_validation():
    from robo_b200 import _lib
    handles, etas, lower, upper, _ = DE._single(False)
    x0 = _starts(lower, upper, 4, 0)
    assert _lib.maximize_lbfgs(handles, 1, etas, 0.0, x0, lower, upper, maxiter=2)["nit"].max() <= 2
    bad = [dict(maxcor=0), dict(maxcor=33), dict(maxiter=-1), dict(maxfun=0), dict(ftol=-1.0), dict(pgtol=np.nan)]
    for b in bad:
        with pytest.raises(ValueError):
            _lib.maximize_lbfgs(handles, 1, etas, 0.0, x0, lower, upper, **b)
    with pytest.raises(ValueError):
        _lib.maximize_lbfgs(handles, 1, etas, 0.0, x0, upper, lower)
    with pytest.raises(ValueError):
        _lib.maximize_lbfgs(handles, 0, etas, 0.0, x0, lower, upper)
    with pytest.raises(ValueError):
        _lib.maximize_lbfgs(handles, 7, etas, 0.0, x0, lower, upper)
    nan = x0.copy()
    nan[1, 0] = np.nan
    with pytest.raises(ValueError):
        _lib.maximize_lbfgs(handles, 1, etas, 0.0, nan, lower, upper)
    with pytest.raises(ValueError):
        _lib.maximize_lbfgs(handles, 1, etas, 0.0, x0[:, :1], lower, upper)
