"""The exact restatement of the device DIRECT (tests/direct_model.py) against scipy.optimize.direct, and the Direct and
GridSearch classes on the oracle-backed fake handle (tests/fake_direct.py).

scipy.optimize.direct wraps a C translation of Gablonsky's DIRECT 2.0.4, the code the `DIRECT` package wraps.  With
locally_biased=False, eps=1e-4, vol_tol=0, len_tol=0 and f_min=-inf it runs the algorithm DIRECT.solve runs at the
package's defaults, so the model must evaluate the same points, iteration by iteration, bit for bit."""
import math

import numpy as np
import pytest
from scipy.optimize import direct

from robo_b200 import _lib
from tests import direct_model as M


def _scipy(fn, lower, upper, maxf, maxT):
    pts, marks = [], []

    def f(x):
        pts.append(np.array(x, dtype=np.float64))
        return fn(np.asarray(x)[None, :])[0]

    r = direct(f, list(zip(lower, upper)), eps=1e-4, maxfun=maxf, maxiter=maxT, locally_biased=False, vol_tol=0.0,
               len_tol=0.0, f_min=-np.inf, callback=lambda xk: marks.append(len(pts)))
    return r, np.array(pts), marks


def _check_equal(fn, lower, upper, maxf, maxT, pin_x=True):
    r, pts, marks = _scipy(fn, lower, upper, maxf, maxT)
    m = M.run(fn, lower, upper, maxf, maxT)
    assert pts.shape == m["points"].shape
    assert np.array_equal(pts.view(np.int64), m["points"].view(np.int64))
    # the callback follows every iteration but the last: the same boundaries
    d = len(lower)
    ends = np.cumsum([1 + 2 * d] + list(m["rows"]))[1:]
    assert list(ends[:len(marks)]) == marks
    assert (r.nfev, r.nit) == (m["nfev"], m["nit"])
    assert r.fun == m["fun"]
    if pin_x:
        assert np.array_equal(np.asarray(r.x).view(np.int64), m["x"].view(np.int64))
    return r, m


def _bumps(X):
    X = np.atleast_2d(X)
    d = X.shape[1]
    a, b = np.linspace(0.2, 0.7, d), np.linspace(-0.3, 0.4, d)
    return (-np.exp(-3 * np.sum((X - a) ** 2, axis=1)) - 0.5 * np.exp(-8 * np.sum((X - b) ** 2, axis=1))
            + 0.01 * np.sum(np.sin(3 * X + np.arange(d)), axis=1))


@pytest.mark.parametrize("d", [1, 2, 3, 16, 64])
def test_smooth_surfaces_equal_scipy(d):
    r, m = _check_equal(_bumps, [-1.0] * d, [1.5] * d, 400, 200)
    assert r.status == 1 and m["stop"] == M.MAXF and m["nfev"] >= 400


@pytest.mark.parametrize("lower,upper", [([-5.0, 0.0], [10.0, 15.0]), (list(np.linspace(-3, 0.1, 6)),
                                                                       list(np.linspace(0.3, 7, 6)))])
def test_asymmetric_boxes_equal_scipy(lower, upper):
    _check_equal(_bumps, lower, upper, 400, 200)


def test_first_point_uses_gablonskys_box_map():
    _, m = _check_equal(_bumps, [-5.0, 0.0], [10.0, 15.0], 50, 5)
    assert m["points"][0, 0] == 2.5000000000000004      # (0.5 + l / (u - l)) (u - l), not l + 0.5 (u - l)


def test_iteration_limit_equal_scipy():
    r, m = _check_equal(_bumps, [-1.0, -1.0], [1.5, 1.5], 4000, 20)
    assert r.status == 2 and m["stop"] == M.MAXT and m["nit"] == 20


@pytest.mark.parametrize("maxf", [5, 7, 9, 10])
def test_budget_is_taken_after_each_iteration(maxf):
    r, m = _check_equal(_bumps, [-1.0], [1.5], maxf, 200)
    assert m["nfev"] >= maxf and m["stop"] == M.MAXF


def _plateau(X):
    X = np.atleast_2d(X)
    return np.where(np.sum((X - 0.7) ** 2, axis=1) < 0.05, -np.exp(-np.sum((X - 0.72) ** 2, axis=1)), 0.0)


@pytest.mark.parametrize("d", [2, 3])
def test_plateau_with_a_bump_equal_scipy(d):
    _check_equal(_plateau, [0.0] * d, [1.0] * d, 400, 200)


@pytest.mark.parametrize("d", [1, 3])
def test_constant_function_equal_scipy(d):
    _check_equal(lambda X: np.ones(len(np.atleast_2d(X))), [0.0] * d, [1.0] * d, 400, 50)


def test_too_many_ties_stop_before_sampling():
    # |x - c| has mirror ties at every level; the iteration that would choose more than MAXDIV rectangles samples
    # nothing and ends the run (scipy: status -6)
    fn = lambda X: np.abs(np.atleast_2d(X)[:, 0] - 0.1234567891234)
    r, m = _check_equal(fn, [0.0], [1.0], 20000, 20000, pin_x=False)
    assert r.status == -6 and m["stop"] == M.MAXDIV_HIT and m["rows"][-1] == 0


def test_level_and_size_tables():
    levels, thirds = M.tables(3)
    assert M.level_of([1, 1, 1]) == 3 and M.level_of([1, 1, 2]) == 4 and M.level_of([2, 1, 2]) == 5
    assert levels[4] == 0.5 * math.sqrt(3 - 1 + 1 / 9.0) / 3.0
    assert thirds[2] == 1.0 / 9.0


def test_nonfinite_energies_follow_the_stated_rule():
    # NaN is stored as +inf: the run equals the run on the surface with +inf in its place
    def nan_fn(X):
        e = _bumps(X)
        return np.where(np.atleast_2d(X)[:, 0] > 0.9, np.nan, e)

    def inf_fn(X):
        e = _bumps(X)
        return np.where(np.atleast_2d(X)[:, 0] > 0.9, np.inf, e)
    a, b = M.run(nan_fn, [-1.0, -1.0], [1.5, 1.5], 300, 100), M.run(inf_fn, [-1.0, -1.0], [1.5, 1.5], 300, 100)
    assert np.array_equal(a["points"], b["points"]) and a["fun"] == b["fun"] and np.isfinite(a["fun"])
    # -inf as the incumbent ends the run on the package's fglobal test after that iteration
    c = M.run(lambda X: np.where(np.atleast_2d(X)[:, 0] < -0.5, -np.inf, _bumps(X)), [-1.0, -1.0], [1.5, 1.5], 300,
              100)
    assert c["stop"] == M.FGLOBAL_HIT and c["fun"] == -np.inf


# ---------------------------------------------------------------------------------------------------------------
# the classes on the fake handle
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture
def fake(monkeypatch):
    from tests import fake_direct
    return fake_direct.install(monkeypatch)


def _gp(d, n=8, seed=0):
    from robo_b200 import kernels as K
    from robo_b200.models.gaussian_process import GaussianProcess
    rng = np.random.RandomState(seed)
    lower, upper = np.zeros(d), np.ones(d)
    X = rng.rand(n, d)
    y = np.sin(3 * X).sum(axis=1)
    model = GaussianProcess(2 * K.Matern52Kernel(np.ones(d) * 0.3, ndim=d), normalize_input=True, lower=lower,
                            upper=upper, rng=np.random.RandomState(1))
    model.train(X, y, do_optimize=False)
    return model, lower, upper


@pytest.mark.parametrize("kind", ["ei", "log_ei", "pi", "lcb"])
@pytest.mark.parametrize("d", [1, 2])
def test_direct_shape_bounds_and_energy(fake, kind, d):
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    from robo_b200.maximizers import Direct
    model, lower, upper = _gp(d)
    acq = {"ei": EI, "log_ei": LogEI, "pi": PI, "lcb": LCB}[kind](model)
    dr = Direct(acq, lower, upper, n_func_evals=100, n_iters=50, verbose=False)
    x = dr.maximize()
    assert x.shape == (d,) and np.all(x >= lower) and np.all(x <= upper)
    assert dr.last["nfev"] >= 100 or dr.last["stop"] != _lib.DIRECT_MAXF
    np.testing.assert_allclose(-acq.compute(x[None, :]).ravel()[0], dr.last["best_energy"], rtol=1e-9, atol=1e-12)
    assert np.array_equal(dr.maximize(), x)                     # deterministic


def test_direct_refuses_host_acquisitions(fake):
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import Direct
    from robo_b200.models.base_model import BaseModel

    class HostModel(BaseModel):
        def train(self, X, y, **kwargs):
            self.X, self.y = X, y

        def predict(self, X_test, **kwargs):
            return np.zeros(len(X_test)), np.ones(len(X_test))
    hm = HostModel()
    hm.train(np.zeros((2, 2)), np.zeros(2))
    with pytest.raises(TypeError, match="Direct"):
        Direct(EI(hm), np.zeros(2), np.ones(2)).maximize()


@pytest.mark.parametrize("lower,upper,maxf,maxT", [
    (np.zeros(65), np.ones(65), 400, 200),                     # d above GPK_DIRECT_MAX_D
    (np.array([0.0, 1.0]), np.array([1.0, 1.0]), 400, 200),    # lower == upper
    (np.zeros(2), np.ones(2), 0, 200),
    (np.zeros(2), np.ones(2), 400, 0),
    (np.zeros(64), np.ones(64), 40000, 200),                   # (2 d + 1) maxf above GPK_DIRECT_MAX_RECTS
])
def test_direct_argument_validation(fake, lower, upper, maxf, maxT):
    from robo_b200.acquisition_functions import LCB
    from robo_b200.maximizers import Direct
    model, _, _ = _gp(2)
    with pytest.raises(ValueError):
        Direct(LCB(model), lower, upper, n_func_evals=maxf, n_iters=maxT).maximize()


def test_grid_search_one_dim_only(fake):
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import GridSearch
    model, lower, upper = _gp(2)
    with pytest.raises(RuntimeError):
        GridSearch(EI(model), lower, upper)


@pytest.mark.parametrize("kind", ["ei", "log_ei", "pi", "lcb"])
def test_grid_search_device_path_equals_the_reference_loop(fake, kind):
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    from robo_b200.maximizers import GridSearch
    model, lower, upper = _gp(1)
    acq = {"ei": EI, "log_ei": LogEI, "pi": PI, "lcb": LCB}[kind](model)
    gs = GridSearch(acq, lower, upper, resolution=257)
    x = gs.maximize()
    grid = np.linspace(lower[0], upper[0], 257).reshape(257, 1, 1)
    ys = np.array([acq(g) for g in grid]).ravel()
    assert x.shape == (1,)
    np.testing.assert_array_equal(x, grid[ys.argmax()][0])


def test_grid_search_host_acquisition_keeps_the_loop():
    from robo_b200.maximizers import GridSearch
    calls = []

    def acq(x):
        calls.append(x.shape)
        return -float((x.ravel()[0] - 0.3) ** 2)
    x = GridSearch(acq, np.zeros(1), np.ones(1), resolution=11).maximize()
    assert len(calls) == 11 and calls[0] == (1, 1)
    np.testing.assert_array_equal(x, np.linspace(0.0, 1.0, 11)[3:4])
