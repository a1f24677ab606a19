"""The MTBO task factor on the device (gpk_set_task_factor) against the numpy restatement of
tests/task_kernel_model.py: K and the fit across 128-row block edges, moments on the fp64 scoring path, full covariance,
mean-only prediction, the incremental refit, both gradients against central differences, the device hyper sampler's
log-posterior with MTBOPrior, and the ABI's refusals.

Tolerances as in tests/test_gpu_fabolas.py: every value with the factor passes through the fp64 path, which agrees with
a scipy restatement to rounding amplified by the conditioning of K (1e-9 relative for log-likelihoods, 1e-8 for moments
on these well-conditioned problems)."""
import numpy as np
import pytest
import scipy.linalg as spla

from tests import task_kernel_model as T

pytestmark = pytest.mark.gpu

LM = (-1.0, -0.5)


def _theta(n_tasks, seed=0):
    return np.random.RandomState(100 + seed).uniform(-1.0, 0.3, T.n_kt(n_tasks))


def _problem(n, n_tasks, seed=0, lonely=False):
    rng = np.random.RandomState(seed)
    X = np.hstack([rng.rand(n, 2), rng.randint(0, max(1, n_tasks - 1 if lonely else n_tasks), (n, 1))])
    if lonely and n_tasks > 1:
        X[n // 2, -1] = n_tasks - 1                       # the last task in one row only
    y = np.sin(3 * X[:, 0]) + 0.3 * X[:, -1] + 0.1 * rng.randn(n)
    return X, y


def _handle(X, y, n_tasks, theta, log_amp=0.2, out=None):
    from robo_b200 import _lib
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(_lib.MATERN52, log_amp, [0, 1], [0, 1], list(LM))
    h.set_task_factor(2, n_tasks, theta)
    if out is not None:
        h.set_output_transform(True, *out)
    return h


def _ref_kernel(n_tasks, theta, log_amp=0.2):
    return T.mtbo_kernel(2, log_amp, LM, theta, n_tasks)


def _ref_fit(X, y, n_tasks, theta, diag, mean=0.0, log_amp=0.2):
    K = _ref_kernel(n_tasks, theta, log_amp).get_value(X) + diag * np.eye(len(X))
    L = spla.cholesky(K, lower=True)
    z = spla.solve_triangular(L, y - mean, lower=True)
    logdet = 2 * np.sum(np.log(np.diag(L)))
    return L, -0.5 * z @ z - 0.5 * logdet - 0.5 * len(y) * np.log(2 * np.pi), logdet


def _ref_moments(X, y, Xs, n_tasks, theta, diag, out=None):
    k = _ref_kernel(n_tasks, theta)
    L, _, _ = _ref_fit(X, y, n_tasks, theta, diag)
    Ks = k.get_value(Xs, X)
    alpha = spla.cho_solve((L, True), y)
    V = spla.solve_triangular(L, Ks.T, lower=True)
    mu = Ks @ alpha
    var = np.diag(k.get_value(Xs)) - np.einsum("ij,ij->j", V, V)
    cov = k.get_value(Xs) - V.T @ V
    if out is not None:
        mu, var, cov = mu * out[1] + out[0], var * out[1] ** 2, cov * out[1] ** 2
    return mu, var, cov


@pytest.mark.parametrize("n", [1, 127, 128, 129, 300, 1024])
@pytest.mark.parametrize("n_tasks", [1, 2, 3, 8])
def test_kernel_matrix_and_fit(n, n_tasks):
    X, y = _problem(n, n_tasks, seed=n, lonely=True)
    th = _theta(n_tasks, n)
    h = _handle(X, y, n_tasks, th)
    Xb, _ = _problem(37, n_tasks, seed=n + 1)
    ref = _ref_kernel(n_tasks, th).get_value(X[:300], Xb)
    assert np.allclose(h.kernel_matrix(X[:300], Xb), ref, rtol=1e-12, atol=1e-300)
    diag = 1e-2
    logdet, ll = h.fit(diag, 0.0)
    _, ll_ref, logdet_ref = _ref_fit(X, y, n_tasks, th, diag)
    assert logdet == pytest.approx(logdet_ref, rel=1e-9, abs=1e-9)
    assert ll == pytest.approx(ll_ref, rel=1e-9, abs=1e-9)
    h.close()


@pytest.mark.parametrize("m", [500, 4096])
@pytest.mark.parametrize("transform", [False, True])
@pytest.mark.parametrize("opts", [{}, {"chunk": 1024}])
def test_predict_moments(m, transform, opts):
    from robo_b200 import _lib
    X, y = _problem(300, 3, seed=m)
    th = _theta(3, 1)
    out = (0.7, 1.9) if transform else None
    h = _lib.Handle(0)
    for key, v in opts.items():
        h.set_option(key, v)
    h.set_data(X, y)
    h.set_kernel(_lib.MATERN52, 0.2, [0, 1], [0, 1], list(LM))
    h.set_task_factor(2, 3, th)
    if out is not None:
        h.set_output_transform(True, *out)
    diag = 1e-2
    h.fit(diag, 0.0)
    Xs, _ = _problem(m, 3, seed=m + 7)
    mu, var = h.predict(Xs)
    mu_ref, var_ref, _ = _ref_moments(X, y, Xs, 3, th, diag, out=out)
    scale = 1.9 if transform else 1.0
    assert np.max(np.abs(mu - mu_ref)) < 1e-8 * scale * max(1.0, np.max(np.abs(mu_ref)))
    var_ref = np.clip(var_ref, np.finfo(float).eps, np.inf)
    assert np.max(np.abs(var - var_ref) / np.maximum(var_ref, 1e-6 * scale ** 2)) < 1e-8
    assert h.timings()["launches_ozaki"] == 0
    mm = h.predict_mean(Xs)
    assert np.max(np.abs(mm - mu)) < 1e-10 * scale * max(1.0, np.max(np.abs(mu)))
    mu_c, cov = h.predict_cov(Xs[:200])
    _, _, cov_ref = _ref_moments(X, y, Xs[:200], 3, th, diag, out=out)
    assert np.allclose(mu_c, mu[:200], rtol=1e-10, atol=1e-10 * scale)
    assert np.allclose(cov, np.clip(cov_ref, np.finfo(float).eps, np.inf), rtol=1e-7, atol=1e-9 * scale ** 2)
    h.close()


def test_nan_factor_for_a_candidate_that_is_not_a_task():
    X, y = _problem(100, 2, seed=3)
    h = _handle(X, y, 2, _theta(2))
    h.fit(1e-2, 0.0)
    Xs = np.array([[0.5, 0.5, 0.0], [0.5, 0.5, 1.0], [0.5, 0.5, 0.5], [0.5, 0.5, 2.0], [0.5, 0.5, -1.0]])
    mu, var = h.predict(Xs)
    assert np.all(np.isfinite(mu[:2])) and np.all(np.isnan(mu[2:])) and np.all(np.isnan(var[2:]))
    h.close()


def test_fit_append_matches_refit():
    X, y = _problem(300, 3, seed=5)
    th = _theta(3, 5)
    h = _handle(X[:260], y[:260], 3, th)
    h.fit(1e-2, 0.1)
    h.predict(X[:10])
    res = h.fit_append(X, y, 1e-2, 0.1)
    assert res is not None
    _, ll_ref, logdet_ref = _ref_fit(X, y, 3, th, 1e-2, mean=0.1)
    assert res[0] == pytest.approx(logdet_ref, rel=1e-9)
    assert res[1] == pytest.approx(ll_ref, rel=1e-9)
    g = _handle(X, y, 3, th)
    g.fit(1e-2, 0.1)
    Xs, _ = _problem(100, 3, seed=6)
    assert np.allclose(h.predict(Xs)[0], g.predict(Xs)[0], rtol=1e-9, atol=1e-10)
    h.close()
    g.close()


@pytest.mark.parametrize("n_tasks", [1, 2, 3])
def test_nll_grad_against_central_differences(n_tasks):
    X, y = _problem(200, n_tasks, seed=7)
    nkt = T.n_kt(n_tasks)
    theta = np.r_[0.2, LM, _theta(n_tasks, 7)]
    diag = 1e-2

    def ll(t):
        from robo_b200 import _lib
        h = _lib.Handle(0)
        h.set_data(X, y)
        h.set_kernel(_lib.MATERN52, t[0], [0, 1], [0, 1], list(t[1:3]))
        h.set_task_factor(2, n_tasks, t[3:])
        v = h.fit(diag, 0.0)[1]
        h.close()
        return v
    h = _handle(X, y, n_tasks, theta[3:], log_amp=theta[0])
    h.fit(diag, 0.0)
    g = h.nll_grad(diag, 2, n_kt=nkt)
    assert g.shape == (4 + nkt,)
    eps = 1e-5
    for p in range(3 + nkt):
        tp, tm = theta.copy(), theta.copy()
        tp[p] += eps
        tm[p] -= eps
        fd = -(ll(tp) - ll(tm)) / (2 * eps)
        assert g[p] == pytest.approx(fd, rel=1e-5, abs=1e-6)
    h.close()


def test_predict_grad_against_central_differences():
    X, y = _problem(200, 3, seed=8)
    h = _handle(X, y, 3, _theta(3, 8), out=(0.3, 1.5))
    h.fit(1e-2, 0.0)
    Xs, _ = _problem(20, 3, seed=9)
    r = h.predict_grad(Xs)
    dmu, dvar = r["dmu"], r["dvar"]
    eps = 1e-6
    for a in range(2):
        Xp, Xm = Xs.copy(), Xs.copy()
        Xp[:, a] += eps
        Xm[:, a] -= eps
        (mp, vp), (mm, vm) = h.predict(Xp), h.predict(Xm)
        assert np.allclose(dmu[:, a], (mp - mm) / (2 * eps), rtol=1e-5, atol=1e-6)
        assert np.allclose(dvar[:, a], (vp - vm) / (2 * eps), rtol=1e-5, atol=1e-6)
    assert np.all(dmu[:, 2] == 0) and np.all(dvar[:, 2] == 0)     # the task index is piecewise constant
    h.close()


def test_hyper_lnpost_and_sampler_with_mtbo_prior():
    from robo_b200 import _lib
    from robo_b200.device_gp import TINY
    from robo_b200.fmin.mtbo import _mtbo_kernel
    from robo_b200.models.gaussian_process_mcmc import _hyper_prior
    from robo_b200.priors import MTBOPrior
    rng = np.random.RandomState(12)
    X, y = _problem(60, 3, seed=12)
    kernel, task = _mtbo_kernel(2, 3)
    prior = MTBOPrior(len(kernel) + 1, n_ls=2, n_kt=len(task), rng=np.random.RandomState(0))
    f = kernel.flatten()
    kind, par, n_ls, n_lr = _hyper_prior(prior)
    assert kind == _lib.PRIOR_MTBO and n_lr == 6
    mean = float(np.mean(y))
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    h.set_task_factor(*f["task"])
    _lib.set_hyper_model(h, f["slots"], len(f["axis"]), mean, TINY, kind, par, n_ls, n_lr)
    dim = len(kernel) + 1
    Th = np.column_stack([rng.uniform(0.1, 2, 30), rng.uniform(-3, 1, (30, 2)), rng.uniform(-1.05, 0.05, (30, 6)),
                          rng.uniform(-8, -2, 30)])
    ll, lp = _lib.hyper_lnpost(h, Th)
    for t, l, p in zip(Th, ll, lp):
        k = T.mtbo_kernel(2, t[0], t[1:3], t[3:9], 3)
        yerr = np.sqrt(np.exp(t[-1]))
        K = k.get_value(X) + np.sqrt(yerr ** 2 + TINY) ** 2 * np.eye(len(y))
        Lc = spla.cholesky(K, lower=True)
        z = spla.solve_triangular(Lc, y - mean, lower=True)
        ref = -0.5 * z @ z - np.sum(np.log(np.diag(Lc))) - 0.5 * len(y) * np.log(2 * np.pi)
        assert l == pytest.approx(ref, rel=1e-9, abs=1e-9)
        assert p == pytest.approx(prior.lnprob(t), rel=1e-12, abs=1e-12)
    p0 = np.tile(np.r_[1.0, -1.0, -1.0, -0.5 * np.ones(6), -5.0], (2 * dim, 1)) + 0.05 * rng.randn(2 * dim, dim)
    r = _lib.sample_hypers(h, p0, 20, 123)
    assert r["pos"].shape == (2 * dim, dim) and np.all(np.isfinite(r["pos"])) and np.all(np.isfinite(r["lnpost"]))
    h.close()


def test_bad_arguments():
    from robo_b200 import _lib
    X, y = _problem(50, 2)
    h = _handle(X, y, 2, _theta(2))
    with pytest.raises(Exception):
        h.set_task_factor(2, 2, [0.0, np.nan, 0.0])
    with pytest.raises(Exception):
        h.set_task_factor(2, 9, np.zeros(45))
    with pytest.raises(Exception):
        h.set_env_factor(2, 0.0, 0.0)                        # a task factor is set
    h.set_task_factor(7, 2, np.zeros(3))
    with pytest.raises(Exception):
        h.fit(1e-2, 0.0)
    with pytest.raises(Exception):
        h.kernel_matrix(X[:4], X[:4])
    h.set_task_factor(2, 1, np.zeros(1))                    # task 1 is not a task of a one-task factor
    with pytest.raises(Exception):
        h.fit(1e-2, 0.0)
    h.set_task_factor(2, 2, np.zeros(3))
    h.set_input_bounds(np.zeros(3), np.ones(3) * 2)
    with pytest.raises(Exception):
        h.fit(1e-2, 0.0)
    h.set_input_bounds(None, None)
    Xh = X.copy()
    Xh[3, 2] = 0.5
    h.set_data(Xh, y)
    with pytest.raises(Exception):
        h.fit(1e-2, 0.0)
    h.set_data(X, y)
    h.fit(1e-2, 0.0)
    h.set_task_factor(-1)
    h.set_env_factor(2, 0.0, 0.0)
    with pytest.raises(Exception):
        h.set_task_factor(2, 2, np.zeros(3))                # an environment factor is set
    h.set_kernel(_lib.MATERN52, 0.2, [0, 1], [0, 1], list(LM))
    h.set_task_factor(2, 2, np.zeros(3))
    h.set_kernel(_lib.MATERN52, 0.2, [0, 1], [0, 1], list(LM))   # removes the factor
    k0 = h.kernel_matrix(X[:5], X[:5])
    assert np.all(np.diag(k0) == np.exp(0.2))
    h.close()


@pytest.mark.parametrize("n_tasks", [1, 2, 3, 8])
def test_task_table_bit_identical_to_restatement(n_tasks):
    """gpk_task_matrix (host side, the table every device site reads) and tests/task_kernel_model.task_matrix are the
    two places the definition is written: read back through gpk_kernel_matrix at zero distance with amp = 1 (the
    radial factor is exactly 1 there), the table equals the restatement bit for bit."""
    from robo_b200 import _lib
    th = np.random.RandomState(40 + n_tasks).uniform(-3.0, 2.0, T.n_kt(n_tasks))
    X = np.column_stack([np.full(n_tasks, 0.3), np.full(n_tasks, 0.7), np.arange(n_tasks, dtype=float)])
    h = _lib.Handle(0)
    h.set_data(X, np.zeros(n_tasks))
    h.set_kernel(_lib.MATERN52, 0.0, [0, 1], [0, 1], list(LM))
    h.set_task_factor(2, n_tasks, th)
    K = h.kernel_matrix(X, X)
    assert np.array_equal(K.view(np.int64), T.task_matrix(th, n_tasks).view(np.int64))
    h.close()


def test_mtbogp_on_the_device_against_reference_golden():
    """tests/golden/mtbo_ref.npz (tools/make_mtbo_golden.py): the reference's MTBOGP and MTBOGPMCMC(do_optimize=False)
    on the oracle; the device path agrees to the fp64 path's rounding."""
    from robo_b200 import kernels
    from robo_b200.models.mtbo_gp import MTBOGP, MTBOGPMCMC
    from tests.conftest import GOLDEN
    G = np.load(GOLDEN + "/mtbo_ref.npz")

    def kernel():
        k = float(G["obj_amp"]) * kernels.Matern52Kernel(np.ones(1) * G["obj_ls"][0], ndim=3, axes=0)
        k *= kernels.Matern52Kernel(np.ones(1) * G["obj_ls"][1], ndim=3, axes=1)
        task = kernels.TaskKernel(3, 2, int(G["n_tasks"]))
        task.set_parameter_vector(G["obj_theta"])
        return k * task
    gp = MTBOGP(kernel(), noise=float(G["noise"]), lower=G["lower"], upper=G["upper"], rng=np.random.RandomState(0))
    gp.train(G["X"], G["y"], do_optimize=False)
    mu, var = gp.predict(G["Xt"])
    np.testing.assert_allclose(mu, G["gp_mu"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(var, G["gp_var"], rtol=1e-7, atol=1e-12)
    inc, _ = gp.get_incumbent()
    assert np.array_equal(inc, G["inc"])
    m = MTBOGPMCMC(kernel(), lower=G["lower"], upper=G["upper"], rng=np.random.RandomState(0))
    m.hypers = G["hypers"]
    m.train(G["X"], G["y"], do_optimize=False)
    mu, var = m.predict(G["Xt"])
    np.testing.assert_allclose(mu, G["mc2_mu"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(var, G["mc2_var"], rtol=1e-7, atol=1e-12)


def test_refused_append_keeps_the_fitted_training_set():
    """gpk_fit_append refuses rows whose task value is not a task before it uploads anything; the handle keeps the
    fitted set, and a refit of it is accepted."""
    X, y = _problem(300, 3, seed=15)
    th = _theta(3, 15)
    h = _handle(X[:260], y[:260], 3, th)
    ll0 = h.fit(1e-2, 0.0)[1]
    h.predict(X[:10])
    Xb = X.copy()
    Xb[280, 2] = 0.5
    with pytest.raises(Exception):
        h.fit_append(Xb, y, 1e-2, 0.0)
    assert h.fit(1e-2, 0.0)[1] == pytest.approx(ll0, rel=1e-13)
    h.close()


def test_kernel_matrix_reads_raw_inputs_under_input_bounds():
    """gpk_kernel_matrix evaluates the kernel on the raw inputs it is given (it never applies the handle's input
    bounds), so input bounds do not touch the task column there; gpk_fit refuses them with the factor."""
    X, y = _problem(40, 3, seed=16)
    th = _theta(3, 16)
    h = _handle(X, y, 3, th)
    h.set_input_bounds(np.array([-1.0, 0.0, 0.0]), np.array([2.0, 3.0, 5.0]))
    ref = _ref_kernel(3, th).get_value(X[:10], X[10:30])
    assert np.allclose(h.kernel_matrix(X[:10], X[10:30]), ref, rtol=1e-12, atol=1e-300)
    with pytest.raises(Exception):
        h.fit(1e-2, 0.0)
    h.close()
