"""Multi-start L-BFGS without a GPU: invariants of the exact restatement of gpk_maximize_lbfgs (tests/lbfgs_model.py),
its quality against scipy's L-BFGS-B from the same starts, the reference's own known answers, and the dispatch of
SciPyOptimizer, DifferentialEvolution(polish="device") and the posterior optimisation on the oracle-backed fake handle
(tests/fake_lbfgs.py)."""
import numpy as np
import pytest
import scipy.optimize

from tests import lbfgs_model as M


@pytest.fixture
def fake(monkeypatch):
    from tests import fake_lbfgs
    fake_lbfgs.install(monkeypatch)
    return fake_lbfgs


def quadratic(X, c=(0.3, -0.2, 0.7)):
    c = np.asarray(c)[:X.shape[-1]]
    return np.sum((X - c) ** 2 * (1.0 + np.arange(X.shape[-1])), axis=-1)


def branin(X):
    x1, x2 = X[..., 0], X[..., 1]
    return (x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x1) + 10


def rosenbrock(X):
    return 100.0 * (X[..., 1] - X[..., 0] ** 2) ** 2 + (1 - X[..., 0]) ** 2


def _starts(lower, upper, n, seed):
    rng = np.random.RandomState(seed)
    return lower + (upper - lower) * rng.rand(n, lower.size)


# ------------------------------------------------------------------ model invariants
def test_dot_order_is_the_warp_butterfly():
    rng = np.random.RandomState(0)
    for d in (1, 2, 16, 33, 64):
        a, b = rng.randn(d), rng.randn(d)
        p = np.zeros(64)
        p[:d] = a * b
        lanes = p[:32] + p[32:]
        for o in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[np.arange(32) ^ o]
        assert np.float64(M.dot(a, b)).tobytes() == lanes[0].tobytes()


def test_stencil_steps_inwards_at_the_upper_bound():
    lower, upper = np.array([-1.0, 0.0, -3.0]), np.array([1.0, 1.0, 0.0])
    x = np.array([1.0, 0.0, -3.0])
    rows = M.stencil(x, lower, upper)
    assert rows.shape == (4, 3) and np.array_equal(rows[0], x)
    assert rows[1, 0] < 1.0 and rows[2, 1] > 0.0 and rows[3, 2] > -3.0           # every neighbour inside the box
    h = M.step(x, lower, upper)
    assert h[0] == -2.0 ** -26 and h[1] == 2.0 ** -26 and h[2] == 3 * 2.0 ** -26   # sign+(0) = +1; -3: turned inwards


def test_iterate_never_leaves_the_box():
    lower, upper = np.array([0.0, 0.0, 0.0]), np.array([0.2, 1.0, 0.5])          # the minimum (0.3, -0.2, 0.7) is outside
    seen = []

    def f(X):
        seen.append(X.copy())
        return quadratic(X)
    r = M.minimize(f, _starts(lower - 1, upper + 1, 12, 1), lower, upper)
    X = np.concatenate(seen)
    assert np.all(X >= lower) and np.all(X <= upper)
    np.testing.assert_allclose(r["x"], np.tile([0.2, 0.0, 0.5], (12, 1)), atol=1e-7)
    assert np.all(np.isin(r["status"], M.SUCCESS))


def test_start_on_a_bound_with_an_outward_gradient_stays_on_it():
    lower, upper = np.zeros(2), np.ones(2)
    seen = []

    def f(X):
        seen.append(X[0::3].copy())
        return (X[:, 0] - 2.0) ** 2 + (X[:, 1] - 0.4) ** 2                   # x0 = 1 is the constrained minimum
    r = M.minimize(f, np.array([[1.0, 0.9]]), lower, upper)
    assert all(np.all(s[:, 0] == 1.0) for s in seen)
    np.testing.assert_allclose(r["x"][0], [1.0, 0.4], atol=1e-6)


def test_non_finite_values_become_dbl_max():
    np.testing.assert_array_equal(M.finite_or_max([1.0, np.inf, -np.inf, np.nan]), [1.0, M.DBL_MAX, M.DBL_MAX, M.DBL_MAX])
    r = M.minimize(lambda X: np.full(len(X), np.nan), np.array([[0.5], [2.0]]), np.zeros(1), np.ones(1))
    assert np.all(r["status"] == M.INVALID) and np.all(r["energy"] == M.DBL_MAX) and np.all(r["nfev"] == 2)
    np.testing.assert_array_equal(r["x"], [[0.5], [1.0]])


def test_maxiter_zero_returns_the_clipped_starts():
    lower, upper = np.array([-1.0, 0.0]), np.array([1.0, 2.0])
    x0 = np.array([[-3.0, 1.0], [0.5, 5.0], [0.1, 0.2]])
    r = M.minimize(quadratic, x0, lower, upper, maxiter=0)
    np.testing.assert_array_equal(r["x"], np.clip(x0, lower, upper))
    assert np.all(r["nit"] == 0) and np.all(r["nfev"] == 3)


def test_every_status_can_be_reached():
    lower, upper = np.zeros(2), np.ones(2)
    st = lambda **kw: set(M.minimize(kw.pop("f", quadratic), kw.pop("x0", np.array([[0.9, 0.9]])), lower, upper,
                                     **kw)["status"])
    assert st(maxiter=1) == {M.MAXITER}
    assert st(maxfun=7) == {M.MAXFUN}
    assert st(f=lambda X: np.full(len(X), np.inf)) == {M.INVALID}
    assert st(x0=np.array([[0.3, 0.0]])) == {M.PGTOL}                           # already the constrained minimum
    assert st(f=lambda X: 5.0 + 1e-6 * np.sum((X - 0.5) ** 2, axis=1), pgtol=0.0) == {M.FTOL}
    # a gradient that promises descent the function never delivers: the line search gives up after 20 halvings
    liar = lambda X: np.where(np.arange(len(X)) % 3 == 0, 1.0 + 1e-3 * np.arange(len(X)), 0.0)
    r = M.minimize(liar, np.array([[0.5, 0.5]]), lower, upper)
    assert r["status"][0] == M.ABNORMAL and r["nfev"][0] == 3 * 22


def test_memory_and_pairs_bounded():
    lower, upper = -2 * np.ones(16), 2 * np.ones(16)
    w = 1.0 + np.arange(16)
    r = M.minimize(lambda X: np.sum(w * (X - 0.1) ** 2, axis=1) + np.sum(X ** 4, axis=1), _starts(lower, upper, 4, 3),
                   lower, upper, maxcor=3)
    assert np.all(np.isin(r["status"], M.SUCCESS)) and np.all(r["nit"] > 3)


# ------------------------------------------------------------------ quality against scipy
@pytest.mark.parametrize("name,fn,lower,upper", [
    ("quadratic", quadratic, np.array([-1.0, -1.0, 0.0]), np.array([1.0, 1.0, 0.5])),
    ("branin", branin, np.array([-5.0, 0.0]), np.array([10.0, 15.0])),
    ("rosenbrock", rosenbrock, np.array([-2.0, -1.0]), np.array([2.0, 3.0])),
])
def test_same_minimum_as_scipy_lbfgsb(name, fn, lower, upper):
    x0 = _starts(lower, upper, 10, 7)
    r = M.minimize(fn, x0, lower, upper)
    ref = [scipy.optimize.minimize(lambda x: float(fn(x)), x, method="L-BFGS-B", bounds=list(zip(lower, upper)))
           for x in x0]
    assert abs(r["energy"].min() - min(s.fun for s in ref)) <= 1e-6
    assert np.all(r["x"] >= lower) and np.all(r["x"] <= upper)
    np.testing.assert_array_equal(r["energy"], fn(r["x"]))


# ------------------------------------------------------------------ the reference's own known answers
class _Quadratic(object):
    """test/dummy_model.py:DemoQuadraticModel and the DemoAcquisitionFunction of test_maximizers_two_dim.py."""

    def __new__(cls):
        from robo_b200.acquisition_functions.base_acquisition import BaseAcquisitionFunction
        from robo_b200.models.base_model import BaseModel

        class DemoQuadraticModel(BaseModel):
            @BaseModel._check_shapes_predict
            def predict(self, X_test):
                return np.sum((0.5 - X_test) ** 2, axis=1), np.ones(X_test.shape[0]) * 0.001

            @BaseModel._check_shapes_train
            def train(self, X, y):
                self.X, self.y = X, y

        class DemoAcquisitionFunction(BaseAcquisitionFunction):
            def __init__(self):
                model = DemoQuadraticModel()
                X = np.random.rand(10, 2)
                model.train(X, (X ** 2)[:, 0])
                super(DemoAcquisitionFunction, self).__init__(model)

            def compute(self, x, **kwargs):
                return np.array([np.sum((0.5 - x) ** 2, axis=1)])
        return DemoQuadraticModel, DemoAcquisitionFunction


def test_reference_test_scipy_on_the_host_loop():
    from robo_b200.maximizers import SciPyOptimizer
    _, Acq = _Quadratic()
    lower, upper = np.array([0, 0]), np.array([1, 1])
    opt = SciPyOptimizer(Acq(), lower, upper, rng=np.random.RandomState(0))
    x = opt.maximize()
    assert x.shape == (2,) and np.all(x >= lower) and np.all(x <= upper)
    assert opt.last["device"] is False and len(opt.last["starts"]) == 10


@pytest.mark.parametrize("which", ["mean", "mean_std"])
def test_reference_posterior_optimization_on_the_host_loop(which):
    from robo_b200.util import posterior_mean_optimization, posterior_mean_plus_std_optimization
    Model, _ = _Quadratic()
    X = np.random.RandomState(0).randn(5, 2)
    model = Model()
    model.train(X, np.sum((0.5 - X) ** 2, axis=1))
    fn = posterior_mean_optimization if which == "mean" else posterior_mean_plus_std_optimization
    x = fn(model, np.array([0, 0]), np.array([1, 1]), with_gradients=False)
    np.testing.assert_almost_equal(x, [0.5, 0.5], decimal=5)


def test_model_on_the_reference_quadratic():
    r = M.minimize(lambda X: np.sum((0.5 - X) ** 2, axis=1) + np.sqrt(0.001), _starts(np.zeros(2), np.ones(2), 10, 4),
                   np.zeros(2), np.ones(2))
    np.testing.assert_almost_equal(r["x"][np.argmin(r["energy"])], [0.5, 0.5], decimal=5)


# ------------------------------------------------------------------ dispatch on the fake library
def _gp(seed=0, n=12):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    rng = np.random.RandomState(seed)
    X = rng.rand(n, 2)
    y = np.sinc(X * 6 - 3).sum(axis=1)
    model = GaussianProcess(2.0 * K.Matern52Kernel(np.ones(2) * 0.3, ndim=2), noise=1e-3, lower=np.zeros(2),
                            upper=np.ones(2), rng=np.random.RandomState(1))
    model.train(X, y, do_optimize=False)
    return model


@pytest.mark.parametrize("acq_name", ["EI", "LogEI", "PI", "LCB"])
def test_scipy_optimizer_reaches_the_acquisition_entry_point(fake, acq_name):
    from robo_b200 import _lib, acquisition_functions as A
    from robo_b200.maximizers import SciPyOptimizer
    model = _gp()
    acq = getattr(A, acq_name)(model)
    opt = SciPyOptimizer(acq, np.zeros(2), np.ones(2), n_restarts=6, rng=np.random.RandomState(3))
    x = opt.maximize()
    assert [c["kind"] for c in fake.calls] == [_lib.ACQ_KIND[acq.kind]] and fake.calls[0]["x0"].shape == (6, 2)
    assert opt.last["device"] and x.shape == (2,) and np.all((x >= 0) & (x <= 1))
    best = int(np.argmin(opt.last["energy"]))
    assert opt.last["best"] == best
    np.testing.assert_array_equal(x, np.clip(opt.last["x"][best], 0, 1))
    np.testing.assert_allclose(-acq.compute(x[None, :]).ravel()[0], opt.last["energy"][best], rtol=1e-12)


def test_scipy_optimizer_starts_follow_the_reference_recipe_from_rng(fake):
    from robo_b200.acquisition_functions import EI
    from robo_b200.initial_design import init_random_uniform
    from robo_b200.maximizers import SciPyOptimizer
    model = _gp()
    lower, upper = np.zeros(2), np.ones(2)
    np.random.seed(0)
    a = SciPyOptimizer(EI(model), lower, upper, n_restarts=10, rng=np.random.RandomState(11))
    a.maximize()
    np.random.seed(1)                                           # the global stream plays no part
    b = SciPyOptimizer(EI(model), lower, upper, n_restarts=10, rng=np.random.RandomState(11))
    b.maximize()
    np.testing.assert_array_equal(a.last["starts"], b.last["starts"])
    rng = np.random.RandomState(11)
    uni = init_random_uniform(lower, upper, 5, rng=rng)
    inc = model.get_incumbent()[0]
    norm = np.array([rng.normal(loc=inc, scale=np.ones(2) * 0.5) for _ in range(5)])
    np.testing.assert_array_equal(a.last["starts"], np.append(uni, norm, axis=0))
    c = SciPyOptimizer(EI(model), lower, upper, n_restarts=10, rng=np.random.RandomState(12))
    c.maximize()
    assert not np.array_equal(a.last["starts"], c.last["starts"])


def test_scipy_optimizer_first_minimum_wins_ties(fake, monkeypatch):
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import SciPyOptimizer

    def tied(handles, kind, eta, par, x0, lower, upper, **options):
        n = len(x0)
        return dict(x=np.linspace(0.1, 0.9, n)[:, None] * np.ones((1, 2)), energy=np.array([3.0, 1.0, 2.0, 1.0][:n]),
                    nit=np.ones(n, int), nfev=np.ones(n, int), status=np.zeros(n, int), n_negative=0)
    monkeypatch.setattr(_lib, "maximize_lbfgs", tied)
    opt = SciPyOptimizer(EI(_gp()), np.zeros(2), np.ones(2), n_restarts=4, rng=np.random.RandomState(0))
    x = opt.maximize()
    assert opt.last["best"] == 1
    np.testing.assert_array_equal(x, np.linspace(0.1, 0.9, 4)[1] * np.ones(2))


def test_scipy_optimizer_host_fallback_for_fabolas_models(fake, golden_dir):
    import os
    from robo_b200 import kernels as K
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import SciPyOptimizer
    from robo_b200.models import FabolasGP
    d = np.load(os.path.join(golden_dir, "fabolas_ref.npz"))
    k = 1.3 * K.Matern52Kernel(np.ones(1) * 0.4, ndim=3, axes=0)
    k *= K.Matern52Kernel(np.ones(1) * 0.6, ndim=3, axes=1)
    k *= K.Matern52Kernel(np.ones(1) * 0.9, ndim=3, axes=2)
    fab = FabolasGP(k, basis_function=lambda s: (1 - s) ** 2, noise=1e-3, lower=d["lower"], upper=d["upper"],
                    rng=np.random.RandomState(0))
    fab.train(d["X"], d["y"], do_optimize=False)
    lower, upper = np.append(d["lower"], 0.0), np.append(d["upper"], 1.0)
    opt = SciPyOptimizer(EI(fab), lower, upper, n_restarts=2, rng=np.random.RandomState(0))
    x = opt.maximize()
    assert not fake.calls and opt.last["device"] is False
    assert x.shape == (3,) and np.all(x >= lower) and np.all(x <= upper)


def test_marginalised_acquisition_uses_every_model(fake):
    from robo_b200 import kernels as K
    from robo_b200.acquisition_functions import LogEI, MarginalizationGPMCMC
    from robo_b200.maximizers import SciPyOptimizer
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    rng = np.random.RandomState(0)
    X = rng.rand(10, 2)
    y = np.sinc(X * 10 - 5).sum(axis=1)
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)), n_hypers=8,
                                chain_length=5, burnin_steps=5, normalize_input=True, lower=np.zeros(2),
                                upper=np.ones(2), rng=np.random.RandomState(2))
    model.train(X, y, do_optimize=True)
    acq = MarginalizationGPMCMC(LogEI(model))
    opt = SciPyOptimizer(acq, np.zeros(2), np.ones(2), n_restarts=4, rng=np.random.RandomState(1))
    x = opt.maximize()
    assert fake.calls[0]["n_models"] == 8
    np.testing.assert_allclose(-acq.compute(x[None, :]).ravel()[0], opt.last["energy"][opt.last["best"]], rtol=1e-12)


@pytest.mark.parametrize("polish", [False, "device"])
def test_differential_evolution_device_polish(fake, polish):
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DifferentialEvolution
    acq = EI(_gp())
    de = DifferentialEvolution(acq, np.zeros(2), np.ones(2), n_iters=3, rng=np.random.RandomState(5), polish=polish)
    x = de.maximize()
    if polish:
        assert len(fake.calls) == 1 and fake.calls[0]["kind"] == _lib.ACQ_EI
        np.testing.assert_array_equal(fake.calls[0]["x0"][0], np.clip(fake.calls[0]["x0"][0], 0, 1))
        assert de.last["best_energy"] <= de.last["device_energy"]
        assert de.last["nfev"] > 2 * 15 * 4
    else:
        assert not fake.calls and not de.last["polished"]
    np.testing.assert_allclose(-acq.compute(x[None, :]).ravel()[0], de.last["best_energy"], rtol=1e-12)


def test_differential_evolution_device_polish_acceptance(fake, monkeypatch):
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DifferentialEvolution
    acq = EI(_gp())
    outcome = {}

    def polish(handles, kind, eta, par, x0, lower, upper, **options):
        return dict(x=np.array([outcome["x"]]), energy=np.array([outcome["e"]]), nit=np.array([2]), nfev=np.array([9]),
                    status=np.array([outcome["status"]]), n_negative=0)
    monkeypatch.setattr(_lib, "maximize_lbfgs", polish)
    for x, e_delta, status, accepted in [([0.25, 0.75], -1.0, _lib.LB_PGTOL, True),
                                          ([0.25, 0.75], -1.0, _lib.LB_ABNORMAL, False),
                                          ([0.25, 0.75], 0.0, _lib.LB_FTOL, False)]:
        de = DifferentialEvolution(acq, np.zeros(2), np.ones(2), n_iters=2, rng=np.random.RandomState(5),
                                   polish="device")
        de.polish = False
        de.maximize()
        outcome.update(x=x, e=de.last["device_energy"] + e_delta, status=status)
        de = DifferentialEvolution(acq, np.zeros(2), np.ones(2), n_iters=2, rng=np.random.RandomState(5),
                                   polish="device")
        got = de.maximize()
        assert de.last["polished"] is accepted
        if accepted:
            np.testing.assert_array_equal(got, x)


@pytest.mark.parametrize("which", ["mean", "mean_std"])
def test_posterior_optimization_reaches_the_device(fake, which):
    from robo_b200 import _lib
    from robo_b200.util import posterior_mean_optimization, posterior_mean_plus_std_optimization
    model = _gp(n=15)
    fn = posterior_mean_optimization if which == "mean" else posterior_mean_plus_std_optimization
    np.random.seed(3)
    x = fn(model, np.zeros(2), np.ones(2), n_restarts=5)
    assert [c["kind"] for c in fake.calls] == [_lib.OBJ_MEAN if which == "mean" else _lib.OBJ_MEAN_STD]
    assert fake.calls[0]["x0"].shape == (5, 2) and np.all((x >= 0) & (x <= 1))
    mu, var = model.predict(x[None, :])
    f = mu[0] if which == "mean" else mu[0] + np.sqrt(var[0])
    grid = np.stack(np.meshgrid(np.linspace(0, 1, 41), np.linspace(0, 1, 41)), -1).reshape(-1, 2)
    mg, vg = model.predict(grid)
    assert f <= np.min(mg if which == "mean" else mg + np.sqrt(vg)) + 1e-9
