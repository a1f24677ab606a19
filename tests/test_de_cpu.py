"""Differential evolution without a GPU: invariants of the exact restatement of gpk_maximize_de (tests/de_model.py),
its faithfulness to scipy.optimize.differential_evolution in distribution, and the DifferentialEvolution maximizer
plus the facade on the oracle-backed fake handle (tests/fake_de.py)."""
import numpy as np
import pytest
import scipy.optimize

from tests import de_model as M


@pytest.fixture
def fake(monkeypatch):
    from tests import fake_de
    return fake_de.install(monkeypatch)


def branin(x):
    x1, x2 = x[0], x[1]
    return (x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x1) + 10


def rosenbrock(X):
    return np.sum(100.0 * (X[..., 1:] - X[..., :-1] ** 2) ** 2 + (1 - X[..., :-1]) ** 2, axis=-1)


def ackley(X):
    d = X.shape[-1]
    return (-20 * np.exp(-0.2 * np.sqrt(np.sum(X ** 2, axis=-1) / d)) - np.exp(np.sum(np.cos(2 * np.pi * X), axis=-1) / d)
            + 20 + np.e)


@pytest.mark.parametrize("pop,d,seed", [(5, 1, 0), (37, 5, 1), (240, 16, 2), (1000, 3, 3)])
def test_lhs_one_member_per_stratum(pop, d, seed):
    P = M.init_population(seed, pop, d)
    assert P.shape == (pop, d) and np.all(P >= 0) and np.all(P < 1)
    strata = np.floor(P * pop).astype(int)
    assert np.array_equal(np.sort(strata, axis=0), np.repeat(np.arange(pop)[:, None], d, axis=1))


@pytest.mark.parametrize("pop,d", [(5, 1), (6, 2), (50, 4), (300, 16)])
def test_trial_invariants(pop, d):
    rng = np.random.RandomState(pop)
    for seed, g in [(0, 1), (12345, 7), (2 ** 40 + 3, 19)]:
        P = rng.rand(pop, d)
        T, t = M.trial(seed, g, P, (0.5, 1.0), 0.7, details=True)
        i = np.arange(pop)
        assert np.all(t["r0"] != i) and np.all(t["r1"] != i) and np.all(t["r0"] != t["r1"])
        assert np.all((t["r0"] >= 0) & (t["r0"] < pop) & (t["r1"] >= 0) & (t["r1"] < pop))
        assert 0.5 <= t["F"] < 1.0
        f = t["fill"]
        assert np.all((f >= 0) & (f < d)) and np.all(t["cross"][i, f])
        assert np.array_equal(t["crossed"][i, f], t["bprime"][i, f])          # the fill point comes from bprime
        kept = ~t["cross"]
        assert np.array_equal(t["crossed"][kept], P[kept])
        assert np.all((T >= 0) & (T <= 1))
        inside = (t["crossed"] >= 0) & (t["crossed"] <= 1)
        assert np.array_equal(T[inside], t["crossed"][inside])


def test_r0_r1_cover_every_other_member():
    """pop = 5: over many members and generations every ordered pair (r0, r1) of the other four members appears."""
    seen = set()
    P = np.random.RandomState(0).rand(5, 1)
    for g in range(1, 200):
        _, t = M.trial(99, g, P, (0.5, 1.0), 0.7, details=True)
        seen.update((i, a, b) for i, a, b in zip(range(5), t["r0"], t["r1"]))
    assert len(seen) == 5 * 4 * 3


def test_energy_replaces_infinities():
    e = M.energy(np.array([np.inf, -np.inf, 1.5, np.nan, -0.25]))
    assert e[0] == M.DBL_MAX and e[1] == M.DBL_MAX and e[2] == -1.5 and np.isnan(e[3]) and e[4] == 0.25


def test_run_slot0_is_argmin_and_best_never_increases():
    lower, upper = np.array([-5.0, 0.0]), np.array([10.0, 15.0])

    def acq(X):                                   # -branin with an infinite band: those energies become DBL_MAX
        v = -np.array([branin(x) for x in X])
        v[X[:, 0] > 9.0] = -np.inf
        return v
    trace = []
    r = M.maximize_de(acq, 7, 40, lower, upper, 30, tol=0.0, trace=trace)
    E = r["energies"]
    assert E[0] == E.min() and int(np.argmin(E)) == 0
    assert np.all(np.diff(trace) <= 0) and len(trace) == r["nit"] + 1 and r["nit"] == 30
    assert r["nfev"] == 40 * 31
    assert np.all(E <= M.DBL_MAX) and r["energy"] < 0.5
    assert np.all(r["x"] >= lower) and np.all(r["x"] <= upper)
    # NaN is promoted first (numpy.argmin)
    P, E2 = np.zeros((4, 1)), np.array([1.0, -2.0, np.nan, np.nan])
    M.promote(P, E2)
    assert np.isnan(E2[0]) and E2[2] == 1.0


def test_convergence_stops_early_and_maxiter_zero():
    flat = M.maximize_de(lambda X: np.ones(len(X)), 3, 20, np.zeros(2), np.ones(2), 50)
    assert flat["nit"] == 1 and flat["nfev"] == 40                   # std 0 after the first generation
    zero = M.maximize_de(lambda X: -X.sum(axis=1), 3, 20, np.zeros(2), np.ones(2), 0)
    assert zero["nit"] == 0 and zero["nfev"] == 20
    np.testing.assert_array_equal(zero["population"][np.argsort(zero["population"][:, 0])],
                                  M.init_population(3, 20, 2)[np.argsort(M.init_population(3, 20, 2)[:, 0])])


def test_stats_order():
    E = np.random.RandomState(4).randn(5000) * 1e3
    mean, std = M.stats(E)
    assert abs(mean - E.mean()) <= 1e-12 * np.abs(E).max() and abs(std - E.std()) <= 1e-12 * E.std()


@pytest.mark.parametrize("name,fn,d,lo,hi,maxiter", [("rosenbrock", rosenbrock, 2, -5.0, 5.0, 40),
                                                     ("ackley", ackley, 5, -5.0, 5.0, 60)])
def test_faithful_to_scipy_in_distribution(name, fn, d, lo, hi, maxiter):
    """Median best energy over 20 seeds after maxiter generations: the restatement against scipy's deferred best1bin
    at the same population (15 d) and maxiter, no early stop, no polish.  The medians agree within a factor of 4
    (the spread between seeds is much wider than that)."""
    lower, upper = np.full(d, lo), np.full(d, hi)
    pop = 15 * d
    ours, theirs = [], []
    for s in range(20):
        ours.append(M.maximize_de(lambda X: -fn(X), 1000 + s, pop, lower, upper, maxiter, tol=0.0)["energy"])
        res = scipy.optimize.differential_evolution(lambda X: fn(X.T), list(zip(lower, upper)), maxiter=maxiter,
                                                    popsize=15, tol=0.0, polish=False, updating="deferred",
                                                    vectorized=True, rng=np.random.default_rng(s))
        theirs.append(res.fun)
    a, b = np.median(ours), np.median(theirs)
    assert 0.25 * b <= a <= 4.0 * b, (name, a, b)


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


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("kind", ["ei", "log_ei", "pi", "lcb"])
def test_maximizer_shape_and_bounds(fake, d, kind):
    """test/test_maximizers/test_maximizers_{one,two}_dim.py: shape (D,), inside the bounds."""
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    from robo_b200.maximizers import DifferentialEvolution
    model, lower, upper = _gp(d)
    acq = {"ei": EI, "log_ei": LogEI, "pi": PI, "lcb": LCB}[kind](model)
    de = DifferentialEvolution(acq, lower, upper, n_iters=5, rng=np.random.RandomState(3))
    x = de.maximize()
    assert x.shape == (d,) and np.all(x >= lower) and np.all(x <= upper)
    assert de.last["nit"] <= 5 and de.last["nfev"] >= 15 * d * (de.last["nit"] + 1)
    # the polish never makes it worse, and the seed advances per call
    assert de.last["best_energy"] <= de.last["device_energy"]
    seed0 = de.last["seed"]
    de.maximize()
    assert de.last["seed"] != seed0
    # the device winner maximises over the evaluated population
    de2 = DifferentialEvolution(acq, lower, upper, n_iters=5, rng=np.random.RandomState(3), polish=False)
    x2 = de2.maximize()
    assert de2.last["polished"] is False and de2.last["best_energy"] == de2.last["device_energy"]
    np.testing.assert_allclose(-acq.compute(x2[None, :]).ravel()[0], de2.last["device_energy"], rtol=1e-12)


class _Result(dict):
    __getattr__ = dict.__getitem__


@pytest.mark.parametrize("fun_delta,success,outside,accepted", [(-1.0, True, False, True), (-1.0, False, False, False),
                                                                (-1.0, True, True, False), (+1.0, True, False, False),
                                                                (0.0, True, False, False)])
def test_polish_acceptance_rule(fake, monkeypatch, fun_delta, success, outside, accepted):
    """scipy's rule: the polished point replaces the device winner only with a lower energy, success, inside bounds."""
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DifferentialEvolution
    from robo_b200.maximizers import differential_evolution as mod
    model, lower, upper = _gp(2)
    de = DifferentialEvolution(EI(model), lower, upper, n_iters=3, rng=np.random.RandomState(5))
    seen = {}

    def minimize(f, x0, method=None, bounds=None):
        seen.update(x0=x0.copy(), method=method, f0=f(x0))
        x = np.array([1.5, 0.5]) if outside else np.array([0.25, 0.75])
        return _Result(x=x, fun=seen["f0"] + fun_delta, success=success, nfev=7)
    monkeypatch.setattr(mod.scipy.optimize, "minimize", minimize)
    x = de.maximize()
    assert seen["method"] == "L-BFGS-B"
    assert de.last["polished"] is accepted
    if accepted:
        np.testing.assert_array_equal(x, [0.25, 0.75])
    else:
        np.testing.assert_array_equal(x, np.clip(seen["x0"], lower, upper))
    assert seen["f0"] == de.last["device_energy"] or np.isclose(seen["f0"], de.last["device_energy"], rtol=1e-12)


def test_refuses_fabolas_and_host_models(fake, golden_dir):
    import os
    from robo_b200 import kernels as K
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DifferentialEvolution
    from robo_b200.models import FabolasGP
    from robo_b200.models.base_model import BaseModel
    d = np.load(os.path.join(golden_dir, "fabolas_ref.npz"))
    k = 1.3 * K.Matern52Kernel(np.ones(1) * 0.4, ndim=3, axes=0)
    k *= K.Matern52Kernel(np.ones(1) * 0.6, ndim=3, axes=1)
    k *= K.Matern52Kernel(np.ones(1) * 0.9, ndim=3, axes=2)
    fab = FabolasGP(k, basis_function=lambda s: (1 - s) ** 2, noise=1e-3, lower=d["lower"], upper=d["upper"],
                    rng=np.random.RandomState(0))
    fab.train(d["X"], d["y"], do_optimize=False)
    with pytest.raises(TypeError):
        DifferentialEvolution(EI(fab), d["lower"], d["upper"], rng=np.random.RandomState(0)).maximize()

    class HostModel(BaseModel):
        def train(self, X, y, **kwargs):
            self.X, self.y = X, y

        def predict(self, X_test, **kwargs):
            return np.zeros(len(X_test)), np.ones(len(X_test))
    hm = HostModel()
    hm.train(np.zeros((2, 2)), np.zeros(2))
    with pytest.raises(TypeError):
        DifferentialEvolution(EI(hm), np.zeros(2), np.ones(2), rng=np.random.RandomState(0)).maximize()


@pytest.mark.parametrize("model_type,acq", [("gp", "ei"), ("gp_mcmc", "log_ei")])
def test_facade_differential_evolution(fake, model_type, acq):
    from robo_b200.fmin import bayesian_optimization
    lower, upper = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
    res = bayesian_optimization(branin, lower, upper, num_iterations=6, maximizer="differential_evolution",
                                acquisition_func=acq, model_type=model_type, n_init=3, chain_length=6, burnin_steps=4,
                                rng=np.random.RandomState(0))
    assert len(res["y"]) == 6 and res["f_opt"] == min(res["y"]) and np.all(np.diff(res["incumbent_values"]) <= 0)
    assert np.all(np.array(res["X"]) >= lower) and np.all(np.array(res["X"]) <= upper)
    with pytest.raises(ValueError):
        bayesian_optimization(branin, lower, upper, num_iterations=4, maximizer="scipy")


def test_marginalised_acquisition_uses_every_model(fake):
    from robo_b200 import kernels as K
    from robo_b200.acquisition_functions import EI, MarginalizationGPMCMC
    from robo_b200.maximizers import DifferentialEvolution
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
    acq = MarginalizationGPMCMC(EI(model))
    de = DifferentialEvolution(acq, np.zeros(2), np.ones(2), n_iters=4, rng=np.random.RandomState(1), polish=False)
    x = de.maximize()
    np.testing.assert_allclose(-acq.compute(x[None, :]).ravel()[0], de.last["device_energy"], rtol=1e-12)
