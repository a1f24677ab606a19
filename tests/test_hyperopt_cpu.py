"""Hyper-parameter optimisation without a GPU: the exact restatement of gpk_optimize_hypers (tests/hyperopt_model.py)
against scipy's own L-BFGS-B, with analytic gradients and with scipy's forward differences, on the edges its logic
has; injected defects that the comparison must catch; and the Python dispatch of hyper_optimizer="device" on the
oracle-backed fake handles, with fakes of the two _lib entry points defined here."""
import importlib
import logging
import os
import re

import numpy as np
import pytest
from scipy.optimize import minimize, rosen, rosen_der

from tests import hyper_model as HM
from tests import hyperopt_model as M
from tests.test_de_es_cpu import LO, UP, _data, branin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _status(res):
    """scipy's message as a gpk_lb_status."""
    msg = res.message if isinstance(res.message, str) else res.message.decode()
    for key, st in (("PROJECTED", M.PGTOL), ("REDUCTION", M.FTOL), ("ABNORMAL", M.ABNORMAL),
                    ("ITERATIONS", M.MAXITER), ("EVALUATIONS", M.MAXFUN)):
        if key in msg.upper():
            return st
    raise AssertionError(msg)


def _agree(res, got, xtol):
    """Same status, nit and nfev, and x within xtol.  The direction differs from L-BFGS-B's in rounding only (the
    two-loop recursion against the compact representation), so the trajectories agree to a few ulp of the iterates
    times the conditioning of the problem; xtol states that bound per case."""
    assert (got["status"], got["nit"], got["nfev"]) == (_status(res), res.nit, res.nfev)
    assert np.max(np.abs(got["x"] - res.x)) <= xtol, np.max(np.abs(got["x"] - res.x))


def _quad(D, seed):
    rng = np.random.RandomState(seed)
    A = rng.randn(D, D)
    H = A @ A.T + D * np.eye(D)
    c = rng.randn(D)
    return lambda x: (0.5 * x @ H @ x - c @ x, H @ x - c)


def _rosen(x):
    return rosen(x), rosen_der(x)


def test_header_constants_match_the_binding():
    from robo_b200 import _lib
    src = open(os.path.join(ROOT, "include", "gpk.h")).read()
    assert int(re.search(r"#define GPK_HO_CHUNK (\d+)", src).group(1)) == _lib.HO_CHUNK == M.CHUNK
    assert "gpk_optimize_hypers" in _lib._SIGNATURES


# ---- against scipy, analytic gradients ------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 2, 5, 12])
def test_quadratics_match_scipy(D):
    for seed in range(3):
        fg = _quad(D, seed)
        p0 = np.random.RandomState(10 + seed).uniform(-3, 3, D)
        _agree(minimize(fg, p0, jac=True, method="L-BFGS-B"), M.run(fg, p0, jac=True), 1e-12)


@pytest.mark.parametrize("D", [2, 3, 5, 8])
def test_rosenbrock_matches_scipy(D):
    """Rosenbrock's valley amplifies rounding differences in the direction: 1e-10 on x at the optimum."""
    for seed in range(3):
        p0 = np.random.RandomState(seed).uniform(-2, 2, D)
        _agree(minimize(_rosen, p0, jac=True, method="L-BFGS-B"), M.run(_rosen, p0, jac=True), 1e-10)


def _golden_nll(name="gp_optimize"):
    """The reference's nll of a golden's training set on the oracle likelihood (tests/fake_gpk.py) plus the host
    DefaultPrior: GaussianProcess.nll as the oracle computes it."""
    from robo_b200 import kernels as K
    from robo_b200.priors import DefaultPrior
    from robo_b200.util import normalization
    d = np.load(os.path.join(GOLDEN, name + ".npz"))
    Xn, _, _ = normalization.zero_one_normalization(d["X"], d["lower"], d["upper"])
    flat = (float(d["cov_amp"]) * K.Matern52Kernel(np.ones(2), ndim=2)).flatten()
    prior = DefaultPrior(4, rng=np.random.RandomState(0))
    mean = float(np.mean(d["y"]))

    def nll(t):
        ll = HM.oracle_ll(Xn, d["y"], mean, flat, t)
        with np.errstate(all="ignore"):
            v = ll + prior.lnprob(t)
        return float(M.objective(ll, v - ll, True)) if np.isfinite(ll) else 1e25
    return d, nll


def test_golden_nll_with_a_gradient_matches_scipy():
    """The oracle nll of the gp_optimize case with a central-difference gradient as the analytic one: the optimiser's
    decisions, not the gradient, are under test.  The run stops on ftol in a flat valley (cond(K) ~ 1e12 at the
    optimum), where rounding differences in the direction move x along the valley by up to 1e-2 at the same f: status,
    nit and nfev must agree exactly, f to 1e-5 relative, x to 1e-2."""
    d, nll = _golden_nll()

    def fg(t):
        g = np.array([(nll(t + 1e-6 * e) - nll(t - 1e-6 * e)) / 2e-6 for e in np.eye(len(t))])
        return nll(t), g
    p0 = d["p0"]
    res = minimize(fg, p0, jac=True, method="L-BFGS-B")
    got = M.run(fg, p0, jac=True)
    _agree(res, got, 1e-2)
    assert abs(got["f"] - res.fun) <= 1e-5 * abs(res.fun) and got["f"] < nll(p0)


# ---- against scipy, forward differences -----------------------------------------------------------------------------
def _recording(fun):
    pts = []

    def f(x):
        pts.append(np.array(x, dtype=np.float64))
        return fun(x)
    return f, pts


@pytest.mark.parametrize("p0", [[-1.2, 1.0, 0.5], [0.0, 3e9, -2.5e-8], [1e9, -1e9, 7.0, 0.0]])
def test_stencil_is_scipys_evaluation_points(p0):
    """The first round's D + 1 rows are the points scipy calls f with, bit for bit, including the relative fallback
    where x + 1e-8 == x (|x| >= 2^27)."""
    p0 = np.array(p0)
    f, pts = _recording(lambda x: float(np.sum(x ** 2)))
    minimize(f, p0, method="L-BFGS-B", options=dict(maxiter=1))
    T, _ = M.stencil(p0, 1e-8)
    assert np.array_equal(np.array(pts[:len(p0) + 1]), T)
    if np.any(np.abs(p0) >= 2 ** 27):
        assert not np.array_equal(T[1:].diagonal() - p0, np.full(len(p0), 1e-8))


def _values(fun):
    return lambda T: np.array([fun(t) for t in T])


@pytest.mark.parametrize("D", [2, 3])
def test_forward_differences_follow_scipys_trajectory(D):
    """With f alone, every point the restatement scores is a point scipy scored, in the same order.  Forward
    differences carry an error of about 1e-8 / h relative in every gradient, which the valley amplifies along the
    run: the points agree to 1e-3, nit, nfev and the status exactly.  (At D = 6 the two runs part in the length of
    one late line search, a decision within the forward-difference error.)"""
    for seed in range(2):
        p0 = np.random.RandomState(seed).uniform(-2, 2, D)
        f, pts = _recording(rosen)
        res = minimize(f, p0, method="L-BFGS-B")
        trace = []
        got = M.run(_values(rosen), p0, trace=trace)
        _agree(res, got, 1e-3)
        scored = np.array(pts[::D + 1])
        assert len(trace) == len(scored)
        assert np.max(np.abs(np.array(trace) - scored)) <= 1e-3


def test_golden_nll_with_forward_differences():
    """The reference's own call on the oracle nll: the restatement reaches scipy's level."""
    d, nll = _golden_nll()
    res = minimize(nll, d["p0"], method="L-BFGS-B")
    got = M.run(_values(nll), d["p0"])
    assert got["f"] <= res.fun + 1e-6 * abs(res.fun) and got["f"] < 1e-3 * float(d["nll_p0"])


# ---- edges ----------------------------------------------------------------------------------------------------------
def test_degenerate_start_at_1e25():
    """gp_optimize_default: nll(p0) = 1e25 (theta_0 = 0 sits on the lognormal prior's edge) while the neighbour in
    theta_0 is finite, so the first gradient is about -1e33 and the first search starts from a 1e25 point."""
    d, nll = _golden_nll("gp_optimize_default")
    assert nll(d["p0"]) == 1e25
    res = minimize(nll, d["p0"], method="L-BFGS-B")
    got = M.run(_values(nll), d["p0"])
    _agree(res, got, 1e-30)
    assert got["nit"] >= 1 and got["f"] < 1e25


def test_trial_beyond_the_abs_limit():
    """A descent towards theta_0 > 20 whose first trials leave the box of the |theta| rule (1e25 there)."""
    def f(t):
        if np.any(np.abs(t) > 20):
            return 1e25
        return -3.0 * t[0] + 0.5 * (t[1] - 1.0) ** 2
    p0 = np.array([19.5, 0.0])
    trace = []
    res = minimize(f, p0, method="L-BFGS-B")
    got = M.run(_values(f), p0, trace=trace)
    _agree(res, got, 1e-9)
    assert any(np.any(np.abs(t) > 20) for t in trace)


@pytest.mark.parametrize("maxiter,maxfun", [(1, 15000), (3, 15000), (15000, 1), (15000, 20), (5, 12)])
def test_budgets(maxiter, maxfun):
    for fun, p0 in ((rosen, np.array([-1.2, 1.0, 0.3])), (lambda x: float(np.sum((x - 1) ** 4)), np.zeros(4))):
        res = minimize(fun, p0, method="L-BFGS-B", options=dict(maxiter=maxiter, maxfun=maxfun))
        got = M.run(_values(fun), p0, maxiter=maxiter, maxfun=maxfun)
        _agree(res, got, 1e-9)


def test_memory_refresh():
    """maxls = 1 and 2 make searches fail after pairs are stored: the memory is cleared and the iteration restarts
    (with stp = 1, since nit > 0), until a failure with an empty memory ends the run ABNORMAL."""
    seen = 0
    for maxls in (1, 2):
        for D, seed in ((2, 0), (2, 1), (4, 0), (4, 2)):
            p0 = np.random.RandomState(seed).uniform(-2, 2, D)
            res = minimize(_rosen, p0, jac=True, method="L-BFGS-B", options=dict(maxls=maxls))
            got = M.run(_rosen, p0, jac=True, maxls=maxls)
            _agree(res, got, 1e-10)
            seen += got["restarts"]
    assert seen >= 4


def test_small_memory():
    for maxcor in (1, 3):
        p0 = np.random.RandomState(4).uniform(-2, 2, 6)
        res = minimize(_rosen, p0, jac=True, method="L-BFGS-B", options=dict(maxcor=maxcor))
        _agree(res, M.run(_rosen, p0, jac=True, maxcor=maxcor), 1e-9)


# ---- injected defects -----------------------------------------------------------------------------------------------
def _mismatches(defect, jac):
    bad = 0
    cases = [(_rosen if jac else rosen, np.random.RandomState(s).uniform(-2, 2, D)) for D in (2, 4) for s in range(3)]
    for fun, p0 in cases:
        if jac:
            res, got = minimize(fun, p0, jac=True, method="L-BFGS-B"), M.run(fun, p0, jac=True, defect=defect)
        else:
            res, got = minimize(fun, p0, method="L-BFGS-B"), M.run(_values(fun), p0, defect=defect)
        try:
            _agree(res, got, 1e-6)
        except AssertionError:
            bad += 1
    return bad


@pytest.mark.parametrize("defect", ["initial_step", "skip_rule", "armijo"])
def test_injected_defects_are_caught(defect):
    assert _mismatches(None, True) == 0
    assert _mismatches(defect, True) >= 1


def test_relative_step_defect_is_caught():
    """A relative finite-difference step (scipy's default without eps) scores other points than scipy's call."""
    p0 = np.array([-1.2, 1.0, 0.5])
    f, pts = _recording(rosen)
    minimize(f, p0, method="L-BFGS-B", options=dict(maxiter=1))
    assert np.array_equal(np.array(pts[:4]), M.stencil(p0, 1e-8)[0])
    assert not np.array_equal(np.array(pts[:4]), M.stencil(p0, 1e-8, defect="relative_step")[0])


# ---- the Python dispatch on the fake --------------------------------------------------------------------------------
class Fake(object):
    """set_hyper_model and optimize_hypers on the fake handles: the restatement driven by the oracle likelihood and
    the host priors.  Records every call."""

    def __init__(self):
        self.calls, self.models = [], []

    def set_hyper_model(self, h, slots, n_terms, mean, tiny, prior_kind=0, prior_par=None, n_ls=0, n_lr=0):
        assert len(h.spec[2]) == n_terms
        h.hyper = dict(slots=list(slots), mean=mean, tiny=tiny, prior=(prior_kind, prior_par, n_ls, n_lr))
        self.models.append(h.hyper)

    def optimize_hypers(self, h, p0, **kw):
        from robo_b200 import _lib
        p0 = np.array(p0, dtype=np.float64)
        dim = len(p0)
        assert len(h.y) <= _lib.HYPER_MAX_N and dim == len(h.hyper["slots"]) + 1
        self.calls.append(dict(handle=h, p0=p0.copy()))
        family, _, axis, group, lm = h.spec
        flat = dict(family=family, axis=axis, group=group, log_metric=lm, slots=h.hyper["slots"])
        prior = HM.prior_object(*h.hyper["prior"], dim=dim)

        def values(T):
            ll = np.array([HM.oracle_ll(h.X, h.y, h.hyper["mean"], flat, t) for t in T])
            if prior is None:
                return M.objective(ll, np.zeros(len(T)), False)
            with np.errstate(all="ignore"):
                lp = np.array([prior.lnprob(t) for t in T])
            return M.objective(ll, lp, True)
        r = M.run(values, p0, maxiter=30)
        return dict(theta=r["x"], f=r["f"], nit=r["nit"], nfev=r["nfev"], status=r["status"], rounds=r["rounds"],
                    noop_rounds=M.noop_rounds(r["rounds"]))


@pytest.fixture
def fake(monkeypatch):
    from robo_b200 import _lib
    from tests import fake_de_es
    fake_de_es.install(monkeypatch)
    f = Fake()
    for name in ("set_hyper_model", "optimize_hypers"):
        monkeypatch.setattr(_lib, name, getattr(f, name))
    return f


def _gp(opt="device", prior="default", **kw):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    from robo_b200.priors import DefaultPrior
    kernel = 3.0 * K.Matern52Kernel(np.ones(2), ndim=2)
    p = DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)) if prior == "default" else prior
    return GaussianProcess(kernel, prior=p, normalize_input=True, lower=LO, upper=UP, rng=np.random.RandomState(2),
                           hyper_optimizer=opt, **kw)


def test_default_is_host_and_unchanged(fake, monkeypatch):
    from robo_b200.models import gaussian_process as GPM
    a = _gp(opt="host")
    assert a.hyper_optimizer == "host"
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    assert GaussianProcess(K.Matern52Kernel(np.ones(2), ndim=2)).hyper_optimizer == "host"
    seen = []
    real = GPM.optimize.minimize

    def spy(*args, **kw):
        seen.append(kw.get("method"))
        return real(*args, **kw)
    monkeypatch.setattr(GPM.optimize, "minimize", spy)
    X, y = _data(10)
    a.train(X, y)
    assert seen == ["L-BFGS-B"] and fake.calls == [] and fake.models == []


def test_device_calls_the_entry_point_once_per_optimize(fake):
    from robo_b200 import _lib
    m = _gp()
    X, y = _data(10)
    p0 = np.append(m.kernel.get_parameter_vector(), np.log(m.noise))
    m.train(X, y)
    assert len(fake.calls) == 1 and np.array_equal(fake.calls[0]["p0"], p0)
    hm = fake.models[0]
    assert hm["slots"] == [("amp", None), ("metric", [0]), ("metric", [1])]
    assert hm["mean"] == float(np.mean(y)) and hm["tiny"] == 1.25e-12
    assert hm["prior"] == (_lib.PRIOR_DEFAULT, [1.0, 0.0, -10, 2, 0.1, 0.0, 0.0], 0, 0)
    assert np.array_equal(m.hypers, m.hyper_result["theta"]) and m.noise == np.exp(m.hypers[-1])
    assert m.is_trained
    # a later train starts from the previous optimum
    X2, y2 = _data(11, seed=1)
    p1 = np.append(m.kernel.get_parameter_vector(), np.log(m.noise))
    m.train(X2, y2)
    assert len(fake.calls) == 2 and np.array_equal(fake.calls[1]["p0"], p1)
    m.train(X2, y2, do_optimize=False)
    assert len(fake.calls) == 2
    # the extra handle does not travel with the model
    assert m._hyper_handle is not None and m.__getstate__()["_hyper_handle"] is None


def test_no_prior(fake):
    m = _gp(prior=None)
    m.train(*_data(10))
    assert fake.models[0]["prior"][0] == 0 and len(fake.calls) == 1


def test_fallback_above_the_limit_logs_once(fake, monkeypatch, caplog):
    from robo_b200 import _lib
    monkeypatch.setattr(_lib, "HYPER_MAX_N", 9)
    m = _gp()
    with caplog.at_level(logging.INFO, logger="robo_b200.models.gaussian_process"):
        m.train(*_data(10))
        m.train(*_data(11))
    assert fake.calls == []
    assert len([r for r in caplog.records if "GPK_HYPER_MAX_N" in r.getMessage()]) == 1
    monkeypatch.setattr(_lib, "HYPER_MAX_N", 232)
    m.train(*_data(10))
    assert len(fake.calls) == 1


def test_type_and_value_errors(fake):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess

    class MyPrior(object):
        def lnprob(self, theta):
            return 0.0
    with pytest.raises(TypeError, match="hyper_optimizer"):
        _gp(prior=MyPrior())
    _gp(prior=MyPrior(), opt="host")
    with pytest.raises(TypeError, match="hyper_optimizer"):
        GaussianProcess(K.Matern52Kernel(np.ones(2), ndim=2) + K.Matern32Kernel(np.ones(2), ndim=2),
                        hyper_optimizer="device")
    with pytest.raises(ValueError, match="use_gradients"):
        _gp(use_gradients=True)
    _gp(opt="host", use_gradients=True)
    with pytest.raises(ValueError):
        _gp(opt="gpu")
    m = _gp()
    m.prior = MyPrior()
    with pytest.raises(TypeError):
        m.train(*_data(10))
    assert fake.calls == []


@pytest.mark.parametrize("facade", ["bayesian_optimization", "entropy_search"])
def test_facades_pass_the_optimizer(facade, monkeypatch):
    mod = importlib.import_module("robo_b200.fmin." + facade)
    seen = []

    class Stop(Exception):
        pass

    def stub(*a, **k):
        seen.append(k)
        raise Stop()
    monkeypatch.setattr(mod, "GaussianProcess", stub)
    fn = getattr(mod, facade)
    kw = dict(model_type="gp") if facade == "bayesian_optimization" else dict(model="gp")
    with pytest.raises(Stop):
        fn(branin, LO, UP, num_iterations=4, rng=np.random.RandomState(0), hyper_optimizer="device", **kw)
    with pytest.raises(Stop):
        fn(branin, LO, UP, num_iterations=4, rng=np.random.RandomState(0), **kw)
    assert [k["hyper_optimizer"] for k in seen] == ["device", "host"]


def test_fabolas_model_passes_the_optimizer_and_env_prior(fake):
    from robo_b200 import _lib
    from robo_b200 import kernels as K
    from robo_b200.models.fabolas_gp import FabolasGP
    from robo_b200.priors import EnvPrior
    kernel = 1.0 * K.Matern52Kernel(np.ones(2), ndim=3, axes=[0, 1]) * K.Matern52Kernel(np.ones(1), ndim=3, axes=[2])
    m = FabolasGP(kernel, basis_function=lambda s: (1 - s) ** 2, prior=EnvPrior(len(kernel) + 1, 2, 1), lower=LO,
                  upper=UP, rng=np.random.RandomState(5), hyper_optimizer="device")
    rng = np.random.RandomState(0)
    X = np.c_[LO + (UP - LO) * rng.rand(9, 2), rng.uniform(0.1, 1, 9)]
    y = np.array([branin(x) for x in X]) * X[:, 2]
    m.train(X, y)
    assert len(fake.calls) == 1 and m.hypers.shape == (5,)
    assert fake.models[0]["prior"] == (_lib.PRIOR_ENV, [1.0, -2, -10, 2, 0.001, 1, 0], 2, 1)
    h = fake.calls[0]["handle"]
    assert np.allclose(h.X[:, 2], (1 - X[:, 2]) ** 2)


def test_mtbo_model_passes_the_optimizer_and_task_prior(monkeypatch):
    """MTBOGP on the task-kernel fake (tests/task_kernel_model.py); the entry point records its call and returns p0."""
    from robo_b200 import _lib
    from robo_b200.models.mtbo_gp import MTBOGP
    from robo_b200.priors import MTBOPrior
    from tests import task_kernel_model as T
    from tests.test_mtbo_cpu import _kernel
    T.install(monkeypatch)
    calls, models = [], []
    monkeypatch.setattr(_lib, "set_hyper_model", lambda h, *a, **k: models.append(a))

    def opt(h, p0, **kw):
        calls.append(np.array(p0))
        return dict(theta=np.array(p0), f=0.0, nit=0, nfev=len(p0) + 1, status=M.PGTOL, rounds=1, noop_rounds=15)
    monkeypatch.setattr(_lib, "optimize_hypers", opt)
    rng = np.random.RandomState(5)
    X = np.hstack([rng.rand(10, 2), rng.randint(0, 2, (10, 1))])
    y = X[:, 0] + X[:, 2]
    k, task = _kernel(2, 2)
    m = MTBOGP(k, prior=MTBOPrior(len(k) + 1, 2, len(task), rng=rng), lower=np.zeros(2), upper=np.ones(2), rng=rng,
               hyper_optimizer="device")
    m.train(X, y)
    assert len(calls) == 1 and len(calls[0]) == len(k) + 1
    assert models[0][4] == _lib.PRIOR_MTBO and (models[0][6], models[0][7]) == (2, len(task))
    assert np.array_equal(m.hypers, calls[0])
