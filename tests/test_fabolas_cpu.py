"""The Fabolas environment kernel and the ``fabolas`` facade without a GPU: the numpy restatement of the factor against
a direct evaluation and finite differences, the BayesianLinearRegressionKernel parameter protocol and its flatten()
slots, and the facade's bookkeeping on the oracle-backed handle (tests/env_kernel_model.py)."""
import copy
import importlib
import json
import os

import numpy as np
import pytest

from tests import env_kernel_model as E


def test_env_value_matches_formula():
    rng = np.random.RandomState(0)
    z1, z2 = rng.rand(7), rng.rand(5)
    la, lb = 0.3, -1.2
    direct = np.array([[np.exp(la) + np.exp(lb) * a * b for b in z2] for a in z1])
    assert np.allclose(E.env_value(z1, z2, la, lb), direct, rtol=0, atol=1e-15)


def test_env_gradients_match_central_differences():
    rng = np.random.RandomState(1)
    z1, z2 = rng.rand(6), rng.rand(4)
    la, lb, h = 0.1, 0.1, 1e-5
    ga, gb, gz = E.env_gradient(z1, z2, la, lb)
    fa = (E.env_value(z1, z2, la + h, lb) - E.env_value(z1, z2, la - h, lb)) / (2 * h)
    fb = (E.env_value(z1, z2, la, lb + h) - E.env_value(z1, z2, la, lb - h)) / (2 * h)
    fz = np.empty_like(gz)
    for i in range(len(z1)):
        zp, zm = z1.copy(), z1.copy()
        zp[i] += h
        zm[i] -= h
        fz[i] = (E.env_value(zp, z2, la, lb)[i] - E.env_value(zm, z2, la, lb)[i]) / (2 * h)
    for g, f in ((ga, fa), (gb, fb), (gz, fz)):           # relative to the largest entry: the differences cancel
        assert np.max(np.abs(g - f)) <= 1e-7 * np.max(np.abs(g))


def _kernel(D=2):
    from robo_b200 import kernels
    k = 1
    for d in range(D):
        k *= kernels.Matern52Kernel(np.ones([1]) * 0.01, ndim=D + 1, axes=d)
    return k * kernels.BayesianLinearRegressionKernel(log_a=0.1, log_b=0.2, ndim=D + 1, axes=D)


def test_kernel_parameters_flatten_and_copy():
    from robo_b200 import kernels
    env = kernels.BayesianLinearRegressionKernel(log_a=0.1, log_b=0.2, ndim=3, axes=2)
    assert len(env) == 2 and list(env.get_parameter_vector()) == [0.1, 0.2]
    assert env.get_parameter_names() == ("log_a", "log_b")
    k = _kernel()
    assert len(k) == 5                                  # log 1, two log length scales, log_a, log_b
    f = k.flatten()
    assert f["env"] == (2, 0.1, 0.2)
    assert [s[0] for s in f["slots"]] == ["amp", "metric", "metric", "lin_a", "lin_b"]
    assert f["axis"] == [0, 1]
    v = k.get_parameter_vector()
    assert np.allclose(v[-2:], [0.1, 0.2])
    k2 = copy.deepcopy(k)
    k2.set_parameter_vector(v + 1.0)
    assert np.allclose(k.get_parameter_vector(), v)
    assert k2.flatten()["env"] == (2, 1.1, 1.2)
    # the facade's n_hypers rule replaces n_hypers only below 2 * len(kernel) = 10: the default 12 is kept
    assert not 12 < 2 * len(k)
    assert "BayesianLinearRegressionKernel" in kernels.__all__


def test_kernel_refusals():
    from robo_b200 import kernels
    with pytest.raises(ValueError):
        kernels.BayesianLinearRegressionKernel(0.1, 0.1, ndim=3, axes=[1, 2])
    twice = _kernel() * kernels.BayesianLinearRegressionKernel(0.0, 0.0, ndim=3, axes=0)
    with pytest.raises(NotImplementedError):
        twice.flatten()


def test_kernel_value_through_the_handle(monkeypatch):
    E.install(monkeypatch)
    rng = np.random.RandomState(2)
    X1, X2 = rng.rand(6, 3), rng.rand(4, 3)
    k = _kernel()
    # george turns the scalar 1 into ConstantKernel(log(1 / ndim))
    ref = E.fabolas_kernel(2, np.log(1.0 / 3), np.log([0.01, 0.01]), 0.1, 0.2).get_value(X1, X2)
    assert np.allclose(k.get_value(X1, X2), ref, rtol=1e-14, atol=0)


def test_compat_exposes_kernel():
    import sys
    from robo_b200 import compat, kernels
    compat.install()
    assert sys.modules["george.kernels"].BayesianLinearRegressionKernel is kernels.BayesianLinearRegressionKernel


def test_projected_incumbent_estimation(monkeypatch):
    """The definition: project every row to s = proj_value, take the lowest predicted mean of a FabolasGP on the
    oracle-backed handle."""
    E.install(monkeypatch)
    from robo_b200.models.fabolas_gp import FabolasGP
    from robo_b200.util.incumbent_estimation import projected_incumbent_estimation
    rng = np.random.RandomState(4)
    Xtr = rng.rand(20, 3)
    ytr = (Xtr[:, 0] - 0.3) ** 2 + 0.2 * Xtr[:, 2]
    model = FabolasGP(_kernel(), basis_function=lambda s: (1 - s) ** 2, lower=np.zeros(2), upper=np.ones(2))
    model.train(Xtr, ytr, do_optimize=False)
    X = rng.rand(7, 2)
    for proj in (1, 0.25):
        inc, val = projected_incumbent_estimation(model, X, proj_value=proj)
        Xp = np.hstack([X, np.full((7, 1), float(proj))])
        mu = model.predict(Xp)[0]
        best = int(np.argmin(mu))
        assert np.array_equal(inc, Xp[best]) and val == mu[best]


def _objective(x, s):
    # loss grows toward small subsets, cost grows with log s
    return float(np.sum((x - 0.4) ** 2) + 10.0 / s + 0.05), float(np.log(s) + 1.0)


class _HostAcquisition(object):
    """Stand-in for MarginalizationGPMCMC(InformationGainPerUnitCost): the facade's bookkeeping does not depend on
    what the acquisition computes, only that update() and compute() are called."""

    def __init__(self, ig):
        self.ig = ig
        self.updates = 0

    def update(self, model, cost_model):
        self.model = model
        self.updates += 1

    def __call__(self, X, **kw):
        X = np.atleast_2d(X)
        return -np.sum((X - 0.5) ** 2, axis=1)


def _run(monkeypatch, tmp_path=None, **kw):
    E.install(monkeypatch)
    F = importlib.import_module("robo_b200.fmin.fabolas")
    made = []

    class IG(object):
        def __init__(self, *a, **k):
            pass
    monkeypatch.setattr(F, "InformationGainPerUnitCost", IG)
    monkeypatch.setattr(F, "MarginalizationGPMCMC", lambda ig: made.append(_HostAcquisition(ig)) or made[-1])
    lower, upper = np.zeros(2), np.ones(2)
    args = dict(s_min=100, s_max=50000, subsets=[10, 20], n_init=1, num_iterations=3, burnin=5, chain_length=5,
                n_hypers=4, rng=np.random.RandomState(3))
    np.random.seed(3)
    args.update(kw)
    if tmp_path is not None:
        args["output_path"] = str(tmp_path)
    return F.fabolas(_objective, lower, upper, **args), made


def test_fabolas_facade_bookkeeping(monkeypatch, tmp_path):
    F = importlib.import_module("robo_b200.fmin.fabolas")
    res, made = _run(monkeypatch, tmp_path)
    assert set(res) == {"x_opt", "incumbents", "runtime", "overhead", "time_func_eval", "X", "y", "c"}
    assert len(res["X"]) == 3 and len(res["y"]) == 3 and len(res["c"]) == 3
    assert len(res["incumbents"]) == 3 and len(res["runtime"]) == 3 and len(res["overhead"]) == 3
    assert all(len(inc) == 2 for inc in res["incumbents"])
    x = np.array(res["x_opt"])
    assert x.shape == (2,) and np.all(x >= 0) and np.all(x <= 1)
    X = np.array(res["X"])
    s = np.array([F.retransform(v, 100, 50000) for v in X[:, -1]])
    assert np.all(s >= 100) and np.all(s <= 50000)
    # the first two evaluations are the subsets s_max / 10 and s_max / 20
    assert list(s[:2]) == [5000, 2500]
    for xi, yi, ci, si in zip(X, res["y"], res["c"], s):
        fy, fc = _objective(xi[:-1], si)
        assert yi == pytest.approx(fy, rel=1e-12)           # exp(log y)
        assert ci == pytest.approx(np.log(fc), rel=1e-12)    # c stays on the log scale, as in the reference
    assert made[0].updates == 1
    names = sorted(os.listdir(str(tmp_path)))
    assert names == ["fabolas_iter_0.json", "fabolas_iter_2.json"]
    d = json.load(open(os.path.join(str(tmp_path), "fabolas_iter_2.json")))
    assert d["iteration"] == 2 and len(d["incumbent"]) == 2


def test_fabolas_initial_design_assertion(monkeypatch):
    with pytest.raises(AssertionError):
        _run(monkeypatch, n_init=2, num_iterations=3)


def test_fabolas_last_seen_is_argmin_y(monkeypatch):
    res, _ = _run(monkeypatch, inc_estimation="last_seen")
    X, y = np.array(res["X"]), np.log(np.array(res["y"]))
    best = int(np.argmin(y[:2]))
    assert np.allclose(res["incumbents"][2], X[best][:-1])
