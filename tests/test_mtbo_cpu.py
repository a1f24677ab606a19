"""The MTBO task kernel and the ``mtbo`` facade without a GPU: the numpy restatement of the factor against a direct
evaluation and central differences for 1 to 8 tasks, the TaskKernel parameter protocol, flatten() and compat shim,
MTBOPrior, MTBOGP / MTBOGPMCMC input maps and the get_incumbent quirk, and the facade's bookkeeping on the
oracle-backed handle (tests/task_kernel_model.py)."""
import copy
import importlib
import json
import os

import numpy as np
import pytest

from tests import task_kernel_model as T


@pytest.mark.parametrize("n_tasks", range(1, 9))
def test_task_value_matches_definition(n_tasks):
    rng = np.random.RandomState(n_tasks)
    theta = rng.uniform(-1, 0.5, T.n_kt(n_tasks))
    L = T.cholesky_factor(theta, n_tasks)
    assert np.allclose(T.task_matrix(theta, n_tasks), L @ L.T, rtol=1e-15, atol=0)
    t1 = rng.randint(0, n_tasks, 9).astype(float)
    t2 = rng.randint(0, n_tasks, 5).astype(float)
    K = T.task_value(t1, t2, theta, n_tasks)
    assert np.array_equal(K, T.task_matrix(theta, n_tasks)[t1.astype(int)][:, t2.astype(int)])
    # not a task: NaN
    bad = np.array([-1.0, n_tasks, 0.5, np.nan])
    assert np.all(np.isnan(T.task_value(bad, t2, theta, n_tasks)))


@pytest.mark.parametrize("n_tasks", range(1, 9))
def test_task_gradient_matches_central_differences(n_tasks):
    rng = np.random.RandomState(10 + n_tasks)
    theta = rng.uniform(-1, 0.5, T.n_kt(n_tasks))
    t = np.arange(n_tasks, dtype=float)
    g = T.task_gradient(t, t, theta, n_tasks)
    h = 1e-6
    for k in range(T.n_kt(n_tasks)):
        tp, tm = theta.copy(), theta.copy()
        tp[k] += h
        tm[k] -= h
        fd = (T.task_value(t, t, tp, n_tasks) - T.task_value(t, t, tm, n_tasks)) / (2 * h)
        assert np.max(np.abs(g[:, :, k] - fd)) <= 1e-8 * max(1.0, np.max(np.abs(g[:, :, k])))


def _kernel(D=2, n_tasks=2):
    from robo_b200 import kernels
    k = 1
    for d in range(D):
        k *= kernels.Matern52Kernel(np.ones([1]) * 0.01, ndim=D + 1, axes=d)
    task = kernels.TaskKernel(D + 1, D, n_tasks)
    return k * task, task


def test_kernel_parameters_flatten_and_copy():
    k, task = _kernel(2, 3)
    assert len(task) == 6 and np.array_equal(task.get_parameter_vector(), np.zeros(6))
    assert len(task.get_parameter_names()) == 6
    assert len(k) == 9                                   # log 1, two log length scales, six task entries
    f = k.flatten()
    assert f["task"] == (2, 3, (0.0,) * 6) and f["env"] is None
    assert [s[0] for s in f["slots"]] == ["amp", "metric", "metric"] + ["task"] * 6
    assert [s[1] for s in f["slots"][3:]] == list(range(6))
    v = k.get_parameter_vector()
    k2 = copy.deepcopy(k)
    k2.vector = v + 0.5                                  # george 0.2's setter, used by mtbo_gp.py
    assert np.array_equal(k.get_parameter_vector(), v)
    assert np.allclose(k2.get_parameter_vector(), v + 0.5)
    assert k2.flatten()["task"] == (2, 3, (0.5,) * 6)
    assert not 20 < 2 * len(_kernel(2, 2)[0])            # the facade keeps n_hypers = 20 for D = 2, two tasks


def test_kernel_refusals():
    from robo_b200 import kernels
    with pytest.raises(ValueError):
        kernels.TaskKernel(3, 2, 9)
    with pytest.raises(ValueError):
        kernels.TaskKernel(3, 2, 0)
    with pytest.raises(ValueError):
        kernels.TaskKernel(3, 3, 2)
    k, _ = _kernel()
    with pytest.raises(NotImplementedError):
        (k * kernels.TaskKernel(3, 2, 2)).flatten()
    with pytest.raises(NotImplementedError):
        (k * kernels.BayesianLinearRegressionKernel(0.1, 0.1, ndim=3, axes=2)).flatten()


def test_kernel_value_through_the_handle(monkeypatch):
    T.install(monkeypatch)
    rng = np.random.RandomState(2)
    X1 = np.hstack([rng.rand(6, 2), rng.randint(0, 3, (6, 1))])
    X2 = np.hstack([rng.rand(4, 2), rng.randint(0, 3, (4, 1))])
    k, task = _kernel(2, 3)
    task.set_parameter_vector(rng.uniform(-1, 0, 6))
    ref = T.mtbo_kernel(2, np.log(1.0 / 3), np.log([0.01, 0.01]), task.theta, 3).get_value(X1, X2)
    assert np.allclose(k.get_value(X1, X2), ref, rtol=1e-14, atol=0)


def test_compat_exposes_kernel():
    import sys
    from robo_b200 import compat, kernels
    compat.install()
    gk = sys.modules["george.kernels"]
    assert gk.TaskKernel is kernels.TaskKernel
    k = gk.TaskKernel(3, 2, 2)
    assert len(k) == 3 and k.axes.tolist() == [2]


def test_mtbo_prior_matches_definition():
    import scipy.stats as sps
    from robo_b200.priors import MTBOPrior
    p = MTBOPrior(1 + 2 + 3 + 1, n_ls=2, n_kt=3, rng=np.random.RandomState(0))
    th = np.array([0.7, -3.0, 1.0, -0.5, -0.2, -0.9, -4.0])
    lp = sps.lognorm.logpdf(0.7, 1.0, loc=0.0) + np.log(np.log(1 + 3 * (0.1 / np.exp(-4.0)) ** 2))
    assert p.lnprob(th) == pytest.approx(lp, rel=1e-14)
    for j, v in ((3, 0.1), (4, -1.1), (1, 3.0)):
        bad = th.copy()
        bad[j] = v
        assert p.lnprob(bad) == -np.inf
    s = p.sample_from_prior(5)
    assert s.shape == (5, 7)
    assert np.all((s[:, 3:6] >= -1) & (s[:, 3:6] <= 0)) and np.all((s[:, 1:3] >= -10) & (s[:, 1:3] <= 2))
    # the task slice comes from numpy's (1, n, n_kt) broadcast: column k is the k-th tophat draw of n samples
    rng = np.random.RandomState(0)
    rng.lognormal(mean=0.0, sigma=1.0, size=5)
    for _ in range(2):
        rng.rand(5)
    for k in range(3):
        assert np.array_equal(s[:, 3 + k], -1 + rng.rand(5) * 1.0)


def test_mtbogp_maps_and_incumbent_quirk(monkeypatch):
    T.install(monkeypatch)
    from robo_b200.models.mtbo_gp import MTBOGP, normalize
    rng = np.random.RandomState(4)
    lower, upper = np.array([-1.0, 0.0]), np.array([1.0, 2.0])
    X = np.hstack([rng.uniform(lower, upper, (12, 2)), rng.randint(0, 2, (12, 1))])
    y = np.sin(X[:, 0]) + X[:, 1] * 0.3 + 0.5 * X[:, 2]
    Xn = normalize(np.hstack([X[:, :2], [[0.5], [1.5], [2.5]] * 4]), lower, upper)
    assert list(Xn[:3, -1]) == [0.0, 2.0, 2.0]            # np.rint: half to even
    assert np.allclose(Xn[:, :2], (X[:, :2] - lower) / (upper - lower))
    k, _ = _kernel(2, 2)
    model = MTBOGP(k, lower=lower, upper=upper)
    model.train(X, y, do_optimize=False)
    mu, var = model.predict(X)
    assert mu.shape == (12,) and np.all(var > 0)
    inc, val = model.get_incumbent()
    # the quirk: the projected rows are normalised twice before predict
    Xp = np.hstack([X[:, :2], np.ones((12, 1))])
    m2 = model.predict(normalize(Xp, lower, upper))[0]
    assert np.array_equal(inc, Xp[int(np.argmin(m2))]) and val == m2[int(np.argmin(m2))]


def test_mtbogpmcmc_keeps_samples_without_optimisation(monkeypatch):
    T.install(monkeypatch)
    from robo_b200.models.mtbo_gp import MTBOGP, MTBOGPMCMC
    from robo_b200.priors import MTBOPrior
    rng = np.random.RandomState(5)
    X = np.hstack([rng.rand(10, 2), rng.randint(0, 2, (10, 1))])
    y = X[:, 0] + X[:, 2]
    k, task = _kernel(2, 2)
    m = MTBOGPMCMC(k, prior=MTBOPrior(len(k) + 1, 2, len(task), rng=rng), n_hypers=14, chain_length=3, burnin_steps=3,
                   lower=np.zeros(2), upper=np.ones(2), rng=rng)
    assert (m.n_hypers, m.noise) == (14, -8)
    assert MTBOGPMCMC.__init__.__defaults__[:4] == (None, 20, 2000, 2000)
    m.train(X, y, do_optimize=False)
    assert len(m.models) == 1 and isinstance(m.models[0], MTBOGP)
    m.train(X, y, do_optimize=True)
    hypers = np.array(m.hypers)
    assert len(m.models) == 14
    m.train(X, y, do_optimize=False)
    assert np.array_equal(np.array(m.hypers), hypers) and len(m.models) == 14


def _objective(x, task):
    return float(np.sum((x - 0.4) ** 2) + 0.5 * (1 - task) + 0.05), float(1.0 + 3.0 * task)


class _HostAcquisition(object):
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
    T.install(monkeypatch)
    F = importlib.import_module("robo_b200.fmin.mtbo")
    made, igs = [], []

    class IG(object):
        def __init__(self, *a, **k):
            igs.append((a, k))
    monkeypatch.setattr(F, "InformationGainPerUnitCost", IG)
    monkeypatch.setattr(F, "MarginalizationGPMCMC", lambda ig: made.append(_HostAcquisition(ig)) or made[-1])
    args = dict(n_init=2, num_iterations=4, burnin=3, chain_length=3, n_hypers=4, rng=np.random.RandomState(3))
    np.random.seed(3)
    args.update(kw)
    if tmp_path is not None:
        args["output_path"] = str(tmp_path)
    return F.mtbo(_objective, np.zeros(2), np.ones(2), **args), made, igs


def test_mtbo_facade_bookkeeping(monkeypatch, tmp_path):
    res, made, igs = _run(monkeypatch, tmp_path)
    assert set(res) == {"x_opt", "incumbents", "runtime", "overhead", "time_func_eval", "X", "y", "c"}
    X, y, c = res["X"], res["y"], res["c"]
    assert isinstance(X, np.ndarray) and isinstance(y, np.ndarray) and isinstance(c, np.ndarray)
    assert X.shape == (4, 3) and y.shape == (4,) and c.shape == (4,)
    assert list(X[:2, -1]) == [0.0, 0.0]                  # the initial design runs on task 0
    assert np.all(np.isin(X[:, -1], [0.0, 1.0]))          # np.rint of the maximizer's task
    for xi, yi, ci in zip(X, y, c):
        fy, fc = _objective(xi[:-1], xi[-1])
        assert yi == pytest.approx(np.log(fy), rel=1e-12)   # y stays on the log scale
        assert ci == pytest.approx(np.log(fc), rel=1e-12)
    assert len(res["incumbents"]) == 4 and all(len(v) == 2 for v in res["incumbents"])
    best = int(np.argmin(y[:2]))
    assert np.allclose(res["incumbents"][2], X[best][:-1])
    assert made[0].updates == 2
    (a, k), = igs
    assert np.array_equal(a[2], [0, 0, 0]) and np.array_equal(a[3], [1, 1, 1])   # the box extended by [0, n_tasks - 1]
    assert list(k["is_env_variable"]) == [0, 0, 1]
    names = sorted(os.listdir(str(tmp_path)))
    assert names == ["mtbo_iter_%d.json" % i for i in range(4)]
    d = json.load(open(os.path.join(str(tmp_path), "mtbo_iter_3.json")))
    assert d["iteration"] == 3 and len(d["incumbent"]) == 2
    assert np.array(res["x_opt"]).shape == (2,)


def test_mtbo_n_hypers_rule_and_final_projection(monkeypatch):
    F = importlib.import_module("robo_b200.fmin.mtbo")
    k, task = F._mtbo_kernel(2, 3)
    assert len(k) == 9 and len(task) == 6
    seen = {}
    real = F.projected_incumbent_estimation

    def spy(model, X, proj_value=1):
        seen["proj"] = proj_value
        seen["n_hypers"] = model.n_hypers
        return real(model, X, proj_value)
    monkeypatch.setattr(F, "projected_incumbent_estimation", spy)
    _run(monkeypatch, n_tasks=3, n_hypers=4)
    assert seen["proj"] == 2                              # the final incumbent on task n_tasks - 1
    assert seen["n_hypers"] == 28                         # 3 * len(kernel) = 27, made even


# ---- tests/golden/mtbo_ref.npz (tools/make_mtbo_golden.py): the reference's own MTBO wrapper code on the oracle --------
def _golden_kernel(G, amp, ls, theta):
    from robo_b200 import kernels
    k = amp * kernels.Matern52Kernel(np.ones(1) * ls[0], ndim=3, axes=0)
    k *= kernels.Matern52Kernel(np.ones(1) * ls[1], ndim=3, axes=1)
    task = kernels.TaskKernel(3, 2, int(G["n_tasks"]))
    task.set_parameter_vector(theta)
    return k * task


def _golden():
    from tests.conftest import GOLDEN
    return np.load(GOLDEN + "/mtbo_ref.npz")


def test_mtbo_prior_against_reference_golden():
    from robo_b200.priors import MTBOPrior
    G = _golden()
    th = G["prior_theta"]
    p = MTBOPrior(th.shape[1], n_ls=2, n_kt=th.shape[1] - 4, rng=np.random.RandomState(int(G["prior_seed"])))
    for t, ref in zip(th, G["prior_lnprob"]):
        assert p.lnprob(t) == ref or abs(p.lnprob(t) - ref) <= 1e-15 * abs(ref)
    assert np.array_equal(p.sample_from_prior(len(G["prior_samples"])), G["prior_samples"])


def test_mtbogp_against_reference_golden(monkeypatch):
    """Predictions and the get_incumbent winner of the reference's MTBOGP, on the oracle-backed handle: the input map,
    the unscaled rint task column and the double normalisation of get_incumbent agree with the reference's code."""
    T.install(monkeypatch)
    from robo_b200.models.mtbo_gp import MTBOGP
    G = _golden()
    k = _golden_kernel(G, float(G["obj_amp"]), G["obj_ls"], G["obj_theta"])
    gp = MTBOGP(k, noise=float(G["noise"]), lower=G["lower"], upper=G["upper"], rng=np.random.RandomState(0))
    gp.train(G["X"], G["y"], do_optimize=False)
    mu, var = gp.predict(G["Xt"])
    np.testing.assert_allclose(mu, G["gp_mu"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(var, G["gp_var"], rtol=1e-9, atol=1e-14)
    inc, val = gp.get_incumbent()
    assert np.array_equal(inc, G["inc"]) and val == pytest.approx(float(G["inc_val"]), rel=1e-10)


def test_mtbogpmcmc_against_reference_golden(monkeypatch):
    """The reference's MTBOGPMCMC.train(do_optimize=False): one sub-model on the kernel's own parameters with noise -8,
    and, with earlier samples set, one sub-model per sample through ``kernel.vector = sample[:-1]``."""
    T.install(monkeypatch)
    from robo_b200.models.mtbo_gp import MTBOGPMCMC
    G = _golden()
    k = _golden_kernel(G, float(G["obj_amp"]), G["obj_ls"], G["obj_theta"])
    m = MTBOGPMCMC(k, lower=G["lower"], upper=G["upper"], rng=np.random.RandomState(0))
    m.train(G["X"], G["y"], do_optimize=False)
    mu, var = m.predict(G["Xt"])
    np.testing.assert_allclose(mu, G["mc_mu"], rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(var, G["mc_var"], rtol=1e-8, atol=1e-13)
    m2 = MTBOGPMCMC(_golden_kernel(G, float(G["obj_amp"]), G["obj_ls"], G["obj_theta"]), lower=G["lower"],
                    upper=G["upper"], rng=np.random.RandomState(0))
    m2.hypers = G["hypers"]
    m2.train(G["X"], G["y"], do_optimize=False)
    assert len(m2.models) == len(G["hypers"])
    mu, var = m2.predict(G["Xt"])
    np.testing.assert_allclose(mu, G["mc2_mu"], rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(var, G["mc2_var"], rtol=1e-8, atol=1e-13)
