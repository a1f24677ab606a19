"""GPU parity tests (pytest -m gpu): the CUDA path, called through the C ABI (ctypes ->
libgpk.so), against the CPU oracle on the same seeded inputs, against the committed golden
vectors (produced by the reference's own classes), and through size-independent properties at
the benchmark's full size.

Tolerances (BASELINE.json north_star): 1e-10 relative on the posterior mean / variance,
1e-8 on EI; denominators are stated in tests/product_cases.py.
"""
import copy
import os

import numpy as np
import pytest
import scipy.linalg as spla

from oracle import george_oracle as G
from oracle import robo_oracle as O
from tests.golden_cases import GP_CASES, kernel_spec, load_case, oracle_kernel
from tests.product_cases import (assert_acq_close, assert_mean_close, assert_var_close, product_kernel,
                                 product_model)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _handle_for(family, theta, X, y, noise, mean=None):
    from robo_b200 import _lib
    D = X.shape[1]
    h = _lib.Handle(0)
    h.set_data(X, y)
    f = product_kernel(family, theta, D).flatten()
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    yerr = np.sqrt(noise)
    diag_add = float(np.sqrt(np.float64(yerr) ** 2 + G.TINY) ** 2)
    mean = float(np.mean(y)) if mean is None else mean
    logdet, ll = h.fit(diag_add, mean)
    return h, logdet, ll, diag_add, mean


# --------------------------------------------------------------------------- kernel values
@pytest.mark.parametrize("family,D", [("matern52", 5), ("rbf", 3), ("prod1d_matern52", 3), ("matern52_noamp", 2)])
def test_kernel_matrix_matches_oracle(family, D):
    rng = np.random.RandomState(0)
    X1, X2 = rng.rand(77, D), rng.rand(201, D)
    theta = rng.randn(D + 1) * 0.7 if family != "matern52_noamp" else rng.randn(D) * 0.7
    ref = oracle_kernel(family, theta, D).get_value(X1, X2)
    got = product_kernel(family, theta, D).get_value(X1, X2)
    np.testing.assert_allclose(got, ref, rtol=1e-13, atol=1e-300)
    sym = product_kernel(family, theta, D).get_value(X1)
    np.testing.assert_array_equal(sym, sym.T)
    np.testing.assert_allclose(sym, oracle_kernel(family, theta, D).get_value(X1), rtol=1e-13)


def test_matern32_and_isotropic_kernels():
    """the remaining george kernel shapes RoBO can build: Matern-3/2, and an isotropic metric (one
    parameter for all axes): values, log-likelihood, posterior and the gradient mapping (the isotropic
    parameter collects the per-axis terms)."""
    from robo_b200 import kernels as K
    from robo_b200.models.gaussian_process import GaussianProcess
    rng = np.random.RandomState(8)
    X, Xs = rng.rand(90, 3), rng.rand(40, 3)
    y = np.cos(4 * X).sum(axis=1)
    for make_p, make_o in (
            (lambda: K.Product(K.ConstantKernel(0.4, ndim=3), K.Matern32Kernel(np.array([0.5, 0.2, 1.1]), ndim=3)),
             lambda: G.Product(G.ConstantKernel(0.4, ndim=3), G.Matern32Kernel(np.array([0.5, 0.2, 1.1]), ndim=3))),
            (lambda: 1.5 * K.ExpSquaredKernel(0.3, ndim=3), lambda: 1.5 * G.ExpSquaredKernel(0.3, ndim=3)),
            (lambda: K.Matern52Kernel(0.7, ndim=3), lambda: G.Matern52Kernel(0.7, ndim=3))):
        kp, ko = make_p(), make_o()
        np.testing.assert_allclose(kp.get_parameter_vector(), ko.get_parameter_vector())
        np.testing.assert_allclose(kp.get_value(Xs, X), ko.get_value(Xs, X), rtol=1e-13, atol=1e-300)
        model = GaussianProcess(kp, noise=1e-3, normalize_input=False)
        model.train(X, y, do_optimize=False)
        st = O.gp_fit(ko, X, y, noise=1e-3, normalize_input=False)
        mu, var = model.predict(Xs)
        mu_ref, var_ref = O.gp_predict(st, Xs)
        assert_mean_close(mu, mu_ref, y)
        assert_var_close(var, var_ref, float(ko.get_value(X[:1])[0, 0]))
        theta = np.append(kp.get_parameter_vector(), np.log(1e-3))
        g = model.grad_nll(theta)
        g_ref = O.gp_grad_nll_correct(st, theta)
        assert g.shape == g_ref.shape
        np.testing.assert_allclose(g, g_ref, rtol=1e-8, atol=1e-8 * np.abs(g_ref).max())


# --------------------------------------------------------------------------- factorisation
@pytest.mark.parametrize("N,D", [(10, 2), (127, 3), (128, 3), (129, 4), (300, 8), (700, 16)])
def test_cholesky_forward_solve_logdet(N, D):
    X, y, _, theta, noise = O.synthetic_problem(N, D, 1, seed_train=N)
    h, logdet, ll, diag_add, mean = _handle_for("matern52", theta, X, y, noise)
    K = O.make_kernel("matern52", D, theta).get_value(X)
    K[np.diag_indices_from(K)] += diag_add
    L_ref = spla.cholesky(K, lower=True)
    L = h.get_factor(N)
    np.testing.assert_allclose(L, L_ref, rtol=0, atol=2e-12 * np.abs(L_ref).max())
    z_ref = spla.solve_triangular(L_ref, y - mean, lower=True)
    np.testing.assert_allclose(h.get_z(N), z_ref, rtol=0, atol=1e-10 * np.abs(z_ref).max())
    logdet_ref = 2 * np.sum(np.log(np.diag(L_ref)))
    assert abs(logdet - logdet_ref) <= 1e-11 * max(1.0, abs(logdet_ref))
    st = O.gp_fit(O.make_kernel("matern52", D, theta), X, y, noise=noise, normalize_input=False)
    ll_ref, _ = O.gp_loglik_terms(st)
    assert abs(ll - ll_ref) <= 1e-10 * abs(ll_ref)
    # triangular inverse
    Linv = h.get_linv(N)
    I = Linv @ L_ref
    assert np.abs(I - np.eye(N)).max() < 1e-9
    assert np.abs(np.triu(Linv, 1)).max() == 0.0


@pytest.mark.parametrize("N", [384, 1500, 4096])
def test_depth2_trailing_update_is_bit_identical(N):
    """the depth-2 trailing update (two panels per K = 256 contraction) applies the panels to every tile in the same
    order as one K = 128 update per step: identical bits in the factor, z and log-det, whether it is forced on (1) or
    chosen from N (2, the default)"""
    from robo_b200 import _lib
    D = 6
    X, y, _, theta, noise = O.synthetic_problem(N, D, 1, seed_train=5)
    got = []
    for depth2 in (1, 0, 2):
        h = _lib.Handle(0)
        h.set_option("depth2", depth2)                      # K = 256 trailing updates vs one K = 128 update per step
        h.set_data(X, y)
        f = product_kernel("matern52", theta, D).flatten()
        h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
        for _ in range(3):                                  # repeated fits: no dependence on what the streams did before
            logdet, ll = h.fit(1e-3 + G.TINY, float(np.mean(y)))
        n_chk = min(N, 1024)
        got.append((logdet, ll, h.get_z(N), h.get_factor(N)[-n_chk:], h.get_linv(N)[-n_chk:]))
        h.close()
    for other in got[1:]:
        assert got[0][0] == other[0] and got[0][1] == other[1]
        for a, b in zip(got[0][2:], other[2:]):
            np.testing.assert_array_equal(a, b)


def test_not_positive_definite_is_linalgerror():
    from robo_b200 import _lib
    X = np.zeros((6, 2))
    y = np.arange(6.0)
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(0, 0.0, [0, 1], [0, 0], [0.0, 0.0])
    with pytest.raises(np.linalg.LinAlgError):
        h.fit(0.0, 0.0)
    # and the handle is reusable afterwards
    h.fit(1e-3, 0.0)


# --------------------------------------------------------------------------- golden vectors
@pytest.mark.parametrize("name", GP_CASES)
def test_golden_case(name):
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    d, _ = load_case(name)
    family, theta = kernel_spec(name)
    model = product_model(d, family, theta)
    model.train(d["X"], d["y"], do_optimize=False)
    np.testing.assert_allclose(model.hypers, d["hypers"], rtol=1e-15)
    kss = float(np.exp(theta[0])) if family != "matern52_noamp" else 1.0
    if bool(d["normalize_output"]):
        kss *= float(np.std(d["y"])) ** 2
    mu, var = model.predict(d["Xs"])
    assert mu.shape == d["mu"].shape and var.shape == d["var"].shape
    assert_mean_close(mu, d["mu"], d["y"])
    assert_var_close(var, d["var"], kss)
    m = int(d["full_cov_m"])
    mu_c, cov = model.predict(d["Xs"][:m], full_cov=True)
    assert cov.shape == (m, m)
    assert_mean_close(mu_c, d["mu"][:m], d["y"])
    assert np.max(np.abs(cov - d["cov"])) <= 1e-10 * kss
    inc_x, inc_y = model.get_incumbent()
    np.testing.assert_allclose(inc_x, d["inc_x"], rtol=1e-15)
    assert inc_y == d["inc_y"]
    pv = model.predict_variance(d["Xs"][:1], d["Xs"][1:9])
    assert pv.shape == d["predict_variance"].shape
    assert np.max(np.abs(pv - d["predict_variance"])) <= 1e-10 * kss
    ll = model.gp.log_likelihood(model.y)
    assert abs(ll - float(d["ll"])) <= 1e-10 * abs(float(d["ll"]))
    assert abs(model.gp.log_determinant - float(d["logdet"])) <= 1e-10 * max(1.0, abs(float(d["logdet"])))
    # acquisition functions through the RoBO API
    assert_acq_close(EI(model).compute(d["Xs"]), d["acq_ei"])
    assert_acq_close(PI(model).compute(d["Xs"]), d["acq_pi"])
    assert_acq_close(LCB(model).compute(d["Xs"]), d["acq_lcb"], rtol=1e-9)
    assert_acq_close(LogEI(model).compute(d["Xs"]), d["acq_log_ei"], rtol=1e-8, atol=1e-8)
    assert_acq_close(EI(model, par=0.1).compute(d["Xs"]), d["acq_ei_par"])
    assert_acq_close(LCB(model, par=2.5).compute(d["Xs"]), d["acq_lcb_par"], rtol=1e-9)
    assert_acq_close(EI(model).compute(d["Xs"], eta=float(np.median(d["y"]))), d["acq_ei_eta"])
    # arg-max = numpy.argmax of the reference's values (random_sampling.py:50)
    for acq, key in ((EI(model), "acq_ei"), (LCB(model), "acq_lcb"), (LogEI(model), "acq_log_ei")):
        got = acq.argmax(d["Xs"])
        ref_vals = d[key]
        assert ref_vals[got] >= ref_vals.max() - 1e-8 * max(1.0, abs(ref_vals.max()))


@pytest.mark.parametrize("name", ["gp_unit", "gp_branin_ny0", "gp_branin_ny1", "gp_prod1d", "gp_rbf_d8"])
def test_golden_nll(name):
    """GaussianProcess.nll incl. the reference's priors and its 1e25 guards."""
    d, _ = load_case(name)
    family, theta = kernel_spec(name)
    prior = None
    if name == "gp_unit":
        prior = _Tophat(-2, 2)
    elif name.startswith("gp_branin"):
        prior = _DefaultPriorLike()
    model = product_model(d, family, theta, prior=prior)
    model.train(d["X"], d["y"], do_optimize=False)
    for t, ref in zip(d["nll_thetas"], d["nll_vals"]):
        got = model.nll(t)
        if ref == 1e25:
            assert got == 1e25
        else:
            assert abs(got - ref) <= 1e-10 * abs(ref), (t, got, ref)


class _Tophat(object):
    """robo/priors/base_prior.py TophatPrior.lnprob restated for the test (host, O(H))."""

    def __init__(self, lo, hi):
        self.lo, self.hi = lo, hi

    def lnprob(self, theta):
        return -np.inf if np.any(theta < self.lo) or np.any(theta > self.hi) else 0


class _DefaultPriorLike(object):
    """robo/priors/default_priors.py:28-37 restated: lognormal(amp) + tophat(ls) + horseshoe(noise)."""

    def lnprob(self, theta):
        import scipy.stats as sps
        lp = sps.lognorm.logpdf(theta[0], 1.0, loc=0.0)
        lp += _Tophat(-10, 2).lnprob(theta[1:-1])
        t = theta[-1]
        lp += np.inf if t == 0 else np.log(np.log(1 + 3.0 * (0.1 / np.exp(t)) ** 2))
        return lp


def test_acq_moments_golden(golden_dir):
    """closed forms on supplied moments (non-GPU models), every log_ei.py branch."""
    from robo_b200 import _lib
    d = np.load(os.path.join(golden_dir, "acq_moments.npz"))
    m, v, eta = d["m"], d["v"], float(d["eta"])
    h = _lib.moments_handle()
    for par in (0.0, 0.3):
        got, _ = h.acq_moments(m, v, _lib.ACQ_LOG_EI, eta, par)
        # log_ei.py:114-120 decides "a >= b -> -inf" between two numbers that agree to ~1/z^2;
        # for |z| >~ 1e3 that margin is below the rounding noise of a and b themselves (the
        # reference's own comment: "can only happen due to numerical inaccuracies"), so there the
        # -inf / finite pattern is noise in the reference too: compare only well-conditioned points.
        with np.errstate(all="ignore"):
            zz = (eta - par - m) / np.sqrt(v)
        ok = ~((m > eta - par) & (np.abs(zz) > 1e3))
        assert ok.sum() > 200
        assert_acq_close(got[ok], d["log_ei_par%g" % par][ok], rtol=1e-8, atol=1e-8)
        bad = got[~ok]
        assert np.all((bad == -np.inf) | (bad < -1e5))
        got, _ = h.acq_moments(m, v, _lib.ACQ_LCB, 0.0, 1.0 + par)
        assert_acq_close(got, d["lcb_par%g" % (1 + par)], rtol=1e-12)
        pos = v > 0
        got, nneg = h.acq_moments(m[pos], v[pos], _lib.ACQ_EI, eta, par)
        assert nneg == 0
        assert_acq_close(got, d["ei_pos_par%g" % par], rtol=1e-8, atol=1e-15)
        got, _ = h.acq_moments(m[pos], v[pos], _lib.ACQ_PI, eta, par)
        assert_acq_close(got, d["pi_par%g" % par][pos], rtol=1e-8, atol=1e-15)


def test_acquisition_on_generic_model_like_reference_tests():
    """test/test_acquisition_functions/test_{ei,log_ei,pi,lcb}.py with test/dummy_model.py's
    constant model: shapes, the LCB known answer (test_lcb.py:25), EI's whole-batch zero."""
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    from robo_b200.models.base_model import BaseModel

    class DemoModel(BaseModel):
        def train(self, X, y):
            self.X, self.y, self.m, self.v = X, y, np.mean(y), np.var(y)

        def predict(self, X_test):
            return np.ones(X_test.shape[0]) * self.m, np.ones(X_test.shape[0]) * self.v

    rng = np.random.RandomState(1)
    X = rng.rand(10, 2)
    y = np.sinc(X * 10 - 5).sum(axis=1)
    model = DemoModel()
    model.train(X, y)
    X_test = rng.rand(5, 2)
    for cls in (EI, LogEI, PI, LCB):
        a = cls(model).compute(X_test)
        assert a.shape == (5,)
    np.testing.assert_almost_equal(LCB(model).compute(X_test), np.ones(5) * (-np.mean(y) + np.std(y)), decimal=3)
    ref = O.acq_ei(np.ones(5) * model.m, np.ones(5) * model.v, np.min(y))
    assert_acq_close(EI(model).compute(X_test), ref)
    model.v = 0.0
    assert EI(model).compute(X_test).shape == (1, 1)


# --------------------------------------------------------------------------- model behaviour
def test_train_retries_with_more_noise_when_not_pd(monkeypatch):
    """gaussian_process.py:118-122: LinAlgError -> noise *= 10 -> retry; a second failure propagates."""
    from robo_b200 import kernels as K
    from robo_b200.device_gp import DeviceGP
    from robo_b200.models.gaussian_process import GaussianProcess
    X = np.repeat(np.random.RandomState(0).rand(3, 2), 20, axis=0)       # 20 exact duplicates each
    y = np.sin(X.sum(axis=1))
    k = K.Product(K.ConstantKernel(np.log(1e6), ndim=2), K.ExpSquaredKernel(np.ones(2) * 50.0, ndim=2))
    model = GaussianProcess(k, noise=1e-13, normalize_input=False)
    with pytest.raises(np.linalg.LinAlgError):          # singular even with 10x the noise, like LAPACK
        model.train(X, y, do_optimize=False)
    assert model.noise == 1e-12
    # first factorisation fails (real GPU status), the retry with 10x noise succeeds
    model = GaussianProcess(K.Matern52Kernel(np.ones(2), ndim=2), noise=1e-3, normalize_input=False)
    real = DeviceGP.compute
    calls = []

    def flaky(self, x=None, yerr=0.0, **kw):
        calls.append(yerr)
        if len(calls) == 1:
            return real(self, x, yerr=float("nan"))      # NaN diagonal -> GPK_NOT_PD from the device
        return real(self, x, yerr=yerr)
    monkeypatch.setattr(DeviceGP, "compute", flaky)
    model.train(np.random.RandomState(1).rand(20, 2), np.random.RandomState(2).rand(20), do_optimize=False)
    assert model.is_trained and model.noise == pytest.approx(1e-2) and len(calls) == 2


def test_deepcopy_and_update_keep_working():
    """marginalization.py:36,67 deep-copies models; base_model.py:30-45 update() retrains."""
    d, _ = load_case("gp_branin_ny1")
    family, theta = kernel_spec("gp_branin_ny1")
    model = product_model(d, family, theta)
    model.train(d["X"], d["y"], do_optimize=False)
    mu, var = model.predict(d["Xs"])
    clone = copy.deepcopy(model)
    mu2, var2 = clone.predict(d["Xs"])
    np.testing.assert_array_equal(mu, mu2)
    np.testing.assert_array_equal(var, var2)
    # update() appends in normalised space exactly like the reference does
    clone.update(model.X[:3], model.y[:3])
    assert clone.X.shape[0] == d["X"].shape[0] + 3 and clone.is_trained


def test_optimize_reaches_reference_optimum(golden_dir):
    """train(do_optimize=True): L-BFGS-B on the GPU nll lands where the reference's did."""
    from robo_b200 import kernels as K
    from robo_b200.models.gaussian_process import GaussianProcess
    d = np.load(os.path.join(golden_dir, "gp_optimize.npz"))
    kernel = float(d["cov_amp"]) * K.Matern52Kernel(np.ones(2), ndim=2)
    prior = _DefaultPriorLike()
    model = GaussianProcess(kernel, prior=prior, normalize_input=True, lower=d["lower"], upper=d["upper"],
                            rng=np.random.RandomState(0))
    model.train(d["X"], d["y"], do_optimize=False)
    assert abs(model.nll(d["p0"]) - float(d["nll_p0"])) <= 1e-9 * abs(float(d["nll_p0"]))
    assert abs(model.nll(d["theta_opt"]) - float(d["nll_opt"])) <= 1e-8 * abs(float(d["nll_opt"]))
    model = GaussianProcess(float(d["cov_amp"]) * K.Matern52Kernel(np.ones(2), ndim=2), prior=prior,
                            normalize_input=True, lower=d["lower"], upper=d["upper"], rng=np.random.RandomState(0))
    model.train(d["X"], d["y"], do_optimize=True)
    # the optimum sits at sigma^2 ~ 1e-8 (cond(K) ~ 1e12): nll is noisy at 1e-4 relative there and
    # L-BFGS-B differentiates it numerically, so trajectories differ; the reached level must match
    got = model.nll(model.hypers)
    assert got <= float(d["nll_opt"]) * 1.02 and got < 1e-3 * float(d["nll_p0"])


def test_random_sampling_maximizer():
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import RandomSampling
    d, _ = load_case("gp_branin_ny0")
    family, theta = kernel_spec("gp_branin_ny0")
    model = product_model(d, family, theta)
    model.train(d["X"], d["y"], do_optimize=False)
    acq = EI(model)
    np.random.seed(3)
    rs = RandomSampling(acq, d["lower"], d["upper"], n_samples=500, rng=np.random.RandomState(0))
    x = rs.maximize()
    assert x.shape == (2,) and np.all(x >= d["lower"]) and np.all(x <= d["upper"])
    X = rs.candidates()
    assert X.shape == (500, 2)
    assert acq.argmax(X) == int(np.argmax(acq.compute(X)))


@pytest.mark.parametrize("family,N,D", [("matern52", 200, 3), ("rbf", 333, 5), ("prod1d_matern52", 150, 3)])
def test_nll_gradient_matches_oracle_and_finite_differences(family, N, D):
    """grad_nll (config 5 kernel): against the oracle's analytic gradient (K^-1 and dK/dtheta
    materialised on the CPU) and against central differences of the device nll."""
    rng = np.random.RandomState(N)
    X = rng.rand(N, D)
    y = np.sin(3 * X).sum(axis=1) + 0.05 * rng.randn(N)
    theta_k = np.concatenate(([0.3], rng.uniform(-1.5, 0.5, D)))
    theta = np.append(theta_k, np.log(3e-3))
    from robo_b200.models.gaussian_process import GaussianProcess
    model = GaussianProcess(product_kernel(family, theta_k, D), noise=3e-3, normalize_input=False)
    model.train(X, y, do_optimize=False)
    g = model.grad_nll(theta)
    st = O.gp_fit(oracle_kernel(family, theta_k, D), X, y, noise=3e-3, normalize_input=False)
    g_ref = O.gp_grad_nll_correct(st, theta)
    assert g.shape == g_ref.shape == (D + 2,)
    np.testing.assert_allclose(g, g_ref, rtol=1e-8, atol=1e-8 * np.abs(g_ref).max())
    h = 1e-5
    for p in (0, 1, D + 1):
        tp, tm = theta.copy(), theta.copy()
        tp[p] += h
        tm[p] -= h
        fd = (model.nll(tp) - model.nll(tm)) / (2 * h)
        assert abs(g[p] - fd) <= 1e-5 * max(1.0, abs(fd))


def test_gp_mcmc_and_marginalised_acquisition():
    """test/test_models/test_gaussian_process_mcmc.py:12-45 + test_marginalization.py:59-93:
    n_hypers=6 walkers, burn-in + chain, predict shapes; mixture moments and the marginalised EI
    against the oracle formulas evaluated on the same per-model moments; batched log-likelihood
    (concurrent streams) == one-at-a-time log-likelihood."""
    from robo_b200 import kernels as K
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI, MarginalizationGPMCMC
    from robo_b200.models import GaussianProcessMCMC
    rng = np.random.RandomState(4)
    X = rng.rand(10, 2)
    y = np.sinc(X * 10 - 5).sum(axis=1)
    kernel = K.Matern52Kernel(np.ones(2), ndim=2)
    prior = _Tophat(-2, 2)
    prior.sample_from_prior = lambda n: rng.uniform(-2, 2, size=(n, 3))
    model = GaussianProcessMCMC(kernel, prior=prior, n_hypers=6, chain_length=20, burnin_steps=10,
                                normalize_input=False, normalize_output=False, rng=np.random.RandomState(1))
    model.train(X, y, do_optimize=True)
    assert len(model.models) == 6 and np.asarray(model.hypers).shape == (6, 3) and model.burned
    assert model.n_lnprob_calls == 6 + 10 * 6 + 6 + 20 * 6
    X_test = rng.rand(10, 2)
    m, v = model.predict(X_test)
    assert m.shape == (10,) and v.shape == (10,)
    mus = np.array([sub.predict(X_test)[0] for sub in model.models])
    vs = np.array([sub.predict(X_test)[1] for sub in model.models])
    m_ref, v_ref = O.mcmc_mixture_moments(mus, vs)
    np.testing.assert_allclose(m, m_ref, rtol=1e-13)
    np.testing.assert_allclose(v, v_ref, rtol=1e-12)
    inc, inc_val = model.get_incumbent()
    b = np.argmin(y)
    np.testing.assert_almost_equal(inc, X[b], decimal=5)
    assert inc_val == y[b]
    # batched == sequential log-likelihood, and both == oracle
    thetas = np.array([[0.2, 0.2, -3.0], [-1.0, 0.5, -6.0], [25.0, 0.0, 0.0], [1.5, -1.5, -1.0]])
    from robo_b200.models.gaussian_process_mcmc import _LikelihoodPool
    model._pool = _LikelihoodPool(kernel, model.X, model.y, model.mean, 4)
    lb = model.loglikelihood_batch(thetas)
    ls = np.array([model.loglikelihood(t) for t in thetas])
    np.testing.assert_array_equal(lb, ls)
    st = O.gp_fit(G.Matern52Kernel(np.ones(2), ndim=2), X, y, noise=1e-3, normalize_input=False)
    for t, l in zip(thetas, lb):
        ref = -O.gp_nll(st, t, prior)
        if ref == -1e25:
            assert l == -np.inf
        else:
            assert abs(l - ref) <= 1e-10 * abs(ref)
    # marginalised acquisitions: shapes + value
    for cls in (LCB, EI, LogEI, PI):
        acq = MarginalizationGPMCMC(cls(model))
        acq.update(model)
        a = acq.compute(X_test)
        assert a.shape == (10,)
        per_model = np.array([cls(sub).compute(X_test) for sub in model.models])
        np.testing.assert_allclose(a, O.marginalised_acquisition(per_model), rtol=1e-13)


def _branin(x):
    x1, x2 = x[0], x[1]
    return (x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x1) + 10


def test_fmin_branin_config0():
    """BASELINE.json configs[0]: fmin.bayesian_optimization on Branin (D=2), GP + EI + random
    maximizer, N <= 50 (test/test_fmin/test_fmin_interface.py:18-87 checks bounds and bookkeeping;
    here additionally that BO actually makes progress towards the known minimum 0.397887)."""
    from robo_b200.fmin import bayesian_optimization
    lower, upper = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
    np.random.seed(0)
    res = bayesian_optimization(_branin, lower, upper, num_iterations=30, maximizer="random",
                                acquisition_func="ei", model_type="gp", n_init=3, rng=np.random.RandomState(0))
    assert len(res["X"]) == 30 and len(res["y"]) == 30 and len(res["incumbents"]) == 30
    assert np.all(np.array(res["X"]) >= lower) and np.all(np.array(res["X"]) <= upper)
    assert res["f_opt"] == min(res["y"]) and np.all(np.diff(res["incumbent_values"]) <= 0)
    assert res["f_opt"] < 2.0          # random search with 30 points averages ~5; BO gets close to 0.398
    # the default facade path: gp_mcmc + log_ei marginalised over the hyper-parameter samples
    res = bayesian_optimization(_branin, lower, upper, num_iterations=6, n_init=3, chain_length=10, burnin_steps=10,
                                rng=np.random.RandomState(1))
    assert len(res["y"]) == 6 and np.all(np.array(res["X"]) >= lower) and np.all(np.array(res["X"]) <= upper)


@pytest.mark.parametrize("N,D,M", [(1, 1, 1), (2, 1, 3), (5, 64, 7), (128, 2, 129), (257, 3, 1000)])
def test_edge_shapes(N, D, M):
    """Smallest / ragged sizes: single training point, single candidate, D = 1 and D = GPK_MAX_TERMS,
    N and M straddling the 128-row tile boundary."""
    rng = np.random.RandomState(N * 1000 + D)
    X, Xs = rng.rand(N, D), rng.rand(M, D)
    y = np.sin(X.sum(axis=1)) + 0.5
    theta = np.concatenate(([0.2], rng.uniform(-1.0, 1.0, D)))
    st = O.gp_fit(oracle_kernel("matern52", theta, D), X, y, noise=1e-3, normalize_input=False)
    mu_ref, var_ref = O.gp_predict(st, Xs)
    from robo_b200.acquisition_functions import EI, LCB
    from robo_b200.models.gaussian_process import GaussianProcess
    model = GaussianProcess(product_kernel("matern52", theta, D), noise=1e-3, normalize_input=False)
    model.train(X, y, do_optimize=False)
    mu, var = model.predict(Xs)
    assert mu.shape == (M,) and var.shape == (M,)
    assert_mean_close(mu, mu_ref, np.append(y, [0.0, 1.0]))
    assert_var_close(var, var_ref, float(np.exp(theta[0])))
    assert_acq_close(EI(model).compute(Xs), O.acquisition(st, Xs, "ei"))
    assert_acq_close(LCB(model).compute(Xs), O.acquisition(st, Xs, "lcb"), rtol=1e-9)
    mu_c, cov = model.predict(Xs[:min(M, 130)], full_cov=True)
    _, cov_ref = O.gp_predict(st, Xs[:min(M, 130)], full_cov=True)
    assert np.max(np.abs(cov - cov_ref)) <= 1e-10 * float(np.exp(theta[0]))
    ll_ref, _ = O.gp_loglik_terms(st)
    assert abs(model.gp.log_likelihood(y) - ll_ref) <= 1e-10 * max(1.0, abs(ll_ref))


@pytest.mark.parametrize("N,D,M", [(100, 3, 2048), (129, 2, 2049), (256, 16, 2177), (640, 5, 4099), (384, 8, 2500)])
def test_int8_scoring_edge_shapes(N, D, M):
    """Ragged sizes on the default large-batch path (int8 tensor-pipe contraction): one, two (CTA pair), three (odd: one-pass
    kernel) and five row blocks, candidate counts that are not multiples of the 128 / 64-candidate tiles."""
    from robo_b200 import _lib
    rng = np.random.RandomState(N * 7 + D)
    X, Xs = rng.rand(N, D), rng.rand(M, D)
    y = np.sin(X.sum(axis=1)) + 0.5
    theta = np.concatenate(([0.2], rng.uniform(-0.5, 0.5, D)))
    h, logdet, ll, diag_add, mean = _handle_for("matern52", theta, X, y, 1e-3)
    h.set_option("ozaki", 1)
    eta = float(np.min(y))
    r = h.acq(Xs, _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)
    t = h.timings()
    h.close()
    assert t["launches_ozaki"] >= 1, t
    st = O.gp_fit(oracle_kernel("matern52", theta, D), X, y, noise=1e-3, normalize_input=False)
    mu_ref, var_ref = O.gp_predict_var_only_fast(st, Xs)
    assert_mean_close(r["mu"], mu_ref, np.append(y, [0.0, 1.0]))
    assert_var_close(r["var"], var_ref, float(np.exp(theta[0])))
    ei_ref = O.acq_ei(mu_ref, var_ref, eta)
    assert_acq_close(r["values"], ei_ref, rtol=1e-8, atol=1e-13)
    assert r["best_idx"] == int(np.argmax(ei_ref))


def test_bad_arguments_raise_value_errors():
    from robo_b200 import _lib
    h = _lib.Handle(0)
    with pytest.raises(ValueError):
        h.set_data(np.zeros((3, 65)), np.zeros(3))                 # d > GPK_MAX_TERMS
    with pytest.raises(ValueError):
        h.fit(1e-3, 0.0)                                           # no data / kernel yet
    h.set_data(np.random.rand(4, 2), np.random.rand(4))
    with pytest.raises(ValueError):
        h.set_kernel(7, 0.0, [0, 1], [0, 0], [0.0, 0.0])            # unknown family
    with pytest.raises(ValueError):
        h.set_kernel(0, 0.0, [0, 1], [1, 1], [0.0, 0.0])            # groups must start at 0
    h.set_kernel(0, 0.0, [0, 5], [0, 0], [0.0, 0.0])
    with pytest.raises(ValueError):
        h.fit(1e-3, 0.0)                                           # kernel axis >= d
    h.set_kernel(0, 0.0, [0, 1], [0, 0], [0.0, 0.0])
    with pytest.raises(RuntimeError):
        h.predict(np.random.rand(3, 2))                            # not fitted
    h.fit(1e-3, 0.0)
    with pytest.raises(ValueError):
        h.set_option("chunk", 100)
    for key in ("nonsense", "diag", "smalltile", "fusechain", "lookahead", "cov", "persist", "ozfused", "ozpdl", "covctas",
                "chainsplit", "graph", "pdl", "loader"):
        with pytest.raises(ValueError):
            h.set_option(key, 1)


def test_device_candidate_generation_and_fused_maximize():
    """gpk_generate_candidates against the oracle's Philox4x32-10 restatement (uniform part bit-exact,
    Gaussian part to rounding), independence of the split into ranges, and the fused maximizer
    returning exactly the arg-max of the acquisition over those candidates."""
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DeviceRandomSampling
    d, _ = load_case("gp_branin_ny0")
    family, theta = kernel_spec("gp_branin_ny0")
    model = product_model(d, family, theta)
    model.train(d["X"], d["y"], do_optimize=False)
    h = model.gp.handle
    lower, upper = d["lower"], d["upper"]
    inc = model.get_incumbent()[0]
    seed, M = 0x1234567890ABCDEF, 5000
    nu = int(M * .7)
    got = h.generate_candidates(seed, 0, M, nu, lower, upper, inc, 0.1)
    ref = O.generate_candidates(seed, 0, M, nu, lower, upper, inc, 0.1)
    np.testing.assert_array_equal(got[:nu], ref[:nu])                       # integer + one fma-free affine map
    np.testing.assert_allclose(got[nu:], ref[nu:], rtol=0, atol=1e-13)
    assert np.all(got >= lower) and np.all(got <= upper)
    # statistics of the proposal (random_sampling.py:38-47)
    u = (got[:nu] - lower) / (upper - lower)
    assert abs(u.mean() - 0.5) < 0.02 and abs(u.var() - 1 / 12.0) < 0.01
    # any split of the index range reproduces the same candidates
    part = np.vstack([h.generate_candidates(seed, 0, 1234, nu, lower, upper, inc, 0.1),
                      h.generate_candidates(seed, 1234, M - 1234, nu, lower, upper, inc, 0.1)])
    np.testing.assert_array_equal(part, got)
    # fused maximise == argmax of EI over exactly these candidates
    acq = EI(model)
    vals = acq.compute(got)
    x, val, idx = h.maximize_random(seed, 0, M, nu, lower, upper, inc, 0.1, _lib.ACQ_EI, float(model.get_incumbent()[1]), 0.0)
    assert idx == int(np.argmax(vals)) and val == vals[idx]
    np.testing.assert_array_equal(x, got[idx])
    # sharded ranges (what each rank of a multi-GPU run does) merge to the same winner
    from robo_b200.distributed import merge_best, shard_bounds
    pairs = []
    for r in range(3):
        lo, hi = shard_bounds(M, r, 3)
        _, v, i = h.maximize_random(seed, lo, hi - lo, nu, lower, upper, inc, 0.1, _lib.ACQ_EI,
                                    float(model.get_incumbent()[1]), 0.0)
        pairs.append((v, i))
    assert merge_best([p[0] for p in pairs], [p[1] for p in pairs])[1] == idx
    # the maximizer class
    mx = DeviceRandomSampling(acq, lower, upper, n_samples=2000, rng=np.random.RandomState(3))
    x1 = mx.maximize()
    assert x1.shape == (2,) and np.all(x1 >= lower) and np.all(x1 <= upper)
    cand = h.generate_candidates(mx.last["seed"], 0, 2000, 1400, lower, upper, inc, 0.1)
    assert mx.last["best_idx"] == int(np.argmax(acq.compute(cand)))


@pytest.mark.parametrize("name", ["gp_branin_ny1", "gp_prod1d", "gp_rbf_d8"])
def test_predictive_and_acquisition_gradients(name):
    """d mu/dx, d var/dx and the EI / PI / LCB input gradients against central differences of the
    oracle (the reference-faithful CPU predict + closed forms), incl. input scaling and output
    un-normalisation chain rules."""
    from robo_b200.acquisition_functions import EI, LCB, PI
    d, kernel_fn = load_case(name)
    family, theta = kernel_spec(name)
    model = product_model(d, family, theta)
    model.train(d["X"], d["y"], do_optimize=False)
    st = O.gp_fit(kernel_fn(), d["X"], d["y"], noise=float(d["noise"]), normalize_input=bool(d["normalize_input"]),
                  normalize_output=bool(d["normalize_output"]), lower=d["lower_"], upper=d["upper_"])
    Xq = d["Xs"][:7]
    D = Xq.shape[1]
    span = 1.0 if d["lower_"] is None else (d["upper_"] - d["lower_"])
    h = 1e-6 * span
    dmu, dvar = model.predictive_gradients(Xq)
    assert dmu.shape == dvar.shape == Xq.shape
    eta = float(O.gp_get_incumbent(st)[1])

    def fd(fun):
        g = np.zeros((len(Xq), D))
        for a in range(D):
            e = np.zeros(D)
            e[a] = (h[a] if np.ndim(h) else h)
            g[:, a] = (fun(Xq + e) - fun(Xq - e)) / (2 * e[a])
        return g
    g_mu = fd(lambda X: O.gp_predict(st, X)[0])
    g_var = fd(lambda X: O.gp_predict(st, X)[1])
    np.testing.assert_allclose(dmu, g_mu, rtol=2e-5, atol=2e-6 * np.abs(g_mu).max())
    np.testing.assert_allclose(dvar, g_var, rtol=2e-5, atol=2e-6 * np.abs(g_var).max())
    for cls, kind in ((EI, "ei"), (PI, "pi"), (LCB, "lcb")):
        f, df = cls(model).compute(Xq, derivative=True)
        assert f.shape == (len(Xq),) and df.shape == Xq.shape
        assert_acq_close(f, O.acquisition(st, Xq, kind), rtol=1e-8, atol=1e-13)
        g = fd(lambda X: O.acquisition(st, X, kind, eta=None if kind == "lcb" else eta))
        np.testing.assert_allclose(df, g, rtol=5e-5, atol=5e-6 * max(np.abs(g).max(), 1e-12))


# --------------------------------------------------------------------------- larger sizes
@pytest.mark.parametrize("N,D,M,family", [(1000, 8, 3000, "matern52"), (1536, 16, 1000, "rbf")])
def test_mid_size_against_oracle(N, D, M, family, monkeypatch):
    """multi-block factorisation + several candidate chunks, against the oracle."""
    monkeypatch.setenv("GPK_CHUNK", "1024")
    X, y, Xs, theta, noise = O.synthetic_problem(N, D, M, seed_train=7, seed_cand=8)
    st = O.gp_fit(O.make_kernel(family, D, theta), X, y, noise=noise, normalize_input=False)
    mu_ref, var_ref = O.gp_predict_var_only(st, Xs)
    h, logdet, ll, _, mean = _handle_for(family, theta, X, y, noise)
    ll_ref, logdet_ref = O.gp_loglik_terms(st)
    assert abs(ll - ll_ref) <= 1e-10 * abs(ll_ref) and abs(logdet - logdet_ref) <= 1e-10 * abs(logdet_ref)
    from robo_b200 import _lib
    eta = float(np.min(y))
    r = h.acq(Xs, _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)
    assert_mean_close(r["mu"], mu_ref, y)
    assert_var_close(r["var"], var_ref, float(np.exp(theta[0])))
    ei_ref = O.acq_ei(mu_ref, var_ref, eta)
    assert_acq_close(r["values"], ei_ref, rtol=1e-8, atol=1e-13)
    assert r["n_negative"] == 0
    assert r["best_idx"] == int(np.argmax(r["values"]))
    assert ei_ref[r["best_idx"]] >= ei_ref.max() * (1 - 1e-8)


def test_george_shim_call_pattern():
    """robo_b200.compat.GeorgeGP with george's own call order (targets only at log_likelihood / predict
    time), as the reference's gaussian_process.py:106-159,280 drives it, against the oracle's george.GP."""
    from robo_b200 import compat
    from robo_b200 import kernels as K
    rng = np.random.RandomState(5)
    X, Xs = rng.rand(40, 3), rng.rand(25, 3)
    y = np.sin(X.sum(axis=1))
    theta = np.array([0.3, -0.5, 0.2, -1.0])
    ref = G.GP(oracle_kernel("matern52", theta, 3), mean=float(y.mean()))
    gp = compat.GeorgeGP(product_kernel("matern52", theta, 3), mean=float(y.mean()))
    for yerr in (0.03, 0.1):
        ref.compute(X, yerr=yerr)
        gp.compute(X, yerr=yerr)
        assert abs(gp.log_likelihood(y, quiet=True) - ref.log_likelihood(y, quiet=True)) <= 1e-10 * abs(ref.log_likelihood(y))
    mu_ref, cov_ref = ref.predict(y, Xs)
    mu, cov = gp.predict(y, Xs)
    assert_mean_close(mu, mu_ref, y)
    # george's predict returns the RAW covariance (negative entries included); the reference clips it itself
    assert np.max(np.abs(cov - cov_ref)) <= 1e-10 * np.exp(theta[0])
    y2 = y + 1.0                                             # new targets -> transparent refit
    ref.compute(X, yerr=0.1)
    assert abs(gp.log_likelihood(y2) - ref.log_likelihood(y2)) <= 1e-10 * abs(ref.log_likelihood(y2))
    with pytest.raises(np.linalg.LinAlgError):
        gp.compute(np.zeros((5, 3)), yerr=float("nan"))


def test_piecewise_host_feeding_is_invisible():
    """gpk_acq feeds host batches larger than 4 chunks in pieces (H2D of piece i+1 overlapped with the
    scoring of piece i): values, moments, arg-max and negative count must equal the one-shot path."""
    from robo_b200 import _lib
    X, y, Xs, theta, noise = O.synthetic_problem(300, 4, 1500, seed_train=3, seed_cand=4)
    h, _, _, _, _ = _handle_for("matern52", theta, X, y, noise)
    eta = float(np.min(y))
    r1 = h.acq(Xs, _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)
    h.set_option("chunk", 128)                                  # piece = 512 candidates -> 3 pieces
    r2 = h.acq(Xs, _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)
    for k in ("values", "mu", "var"):
        np.testing.assert_array_equal(r1[k], r2[k])
    assert r1["best_idx"] == r2["best_idx"] == int(np.argmax(r1["values"])) and r1["best_val"] == r2["best_val"]
    r3 = h.acq(Xs, _lib.ACQ_LCB, 0.0, 1.0, want_values=False)
    h.set_option("chunk", 16384)
    r4 = h.acq(Xs, _lib.ACQ_LCB, 0.0, 1.0, want_values=True)
    assert r3["best_idx"] == r4["best_idx"] == int(np.argmax(r4["values"]))


def test_pageable_batches_are_staged_through_pinned_buffers():
    """host candidate batches above 1 MB that are not page-locked go through the handle's two pinned staging buffers
    (gpk_acq), one-shot and piecewise; page-locked callers' buffers are used in place: identical results either way."""
    import torch
    from robo_b200 import _lib
    X, y, _, theta, noise = O.synthetic_problem(300, 4, 1, seed_train=3)
    Xs = np.random.RandomState(9).rand(40000, 4)               # 1.28 MB
    h, _, _, _, _ = _handle_for("matern52", theta, X, y, noise)
    eta = float(np.min(y))
    r1 = h.acq(Xs, _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)          # staged, one piece
    h.set_option("chunk", 1024)                                                          # staged, 10 pieces of 4096
    r2 = h.acq(Xs, _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)
    pinned = torch.from_numpy(Xs).pin_memory()
    r3 = h.acq(pinned.numpy(), _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)   # used in place
    for r in (r2, r3):
        for k in ("values", "mu", "var"):
            np.testing.assert_array_equal(r1[k], r[k])
        assert r["best_idx"] == r1["best_idx"] == int(np.argmax(r1["values"]))
    st = O.gp_fit(oracle_kernel("matern52", theta, 4), X, y, noise=noise, normalize_input=False)
    assert_acq_close(r1["values"][:2000], O.acquisition(st, Xs[:2000], "ei"))
    h.close()


def test_full_size_properties():
    """BASELINE.json config 2 size (N=4096, D=16): properties that need no CPU oracle run.
      * chunking invariance (bit-identical results for different candidate chunk sizes)
      * at the training inputs y - mu(X) = diag_add * alpha (alpha = L^-T z), and var(X) < noise
      * arg-max returned by the fused kernel == numpy.argmax of the returned values
      * L^-1 consistency: ||L^-1 k*||^2 = k*^T K^-1 k* checked through var >= eps and var <= k**
    """
    from robo_b200 import _lib
    N, D, M = 4096, 16, 4096
    X, y, Xs, theta, noise = O.synthetic_problem(N, D, M)
    os.environ.pop("GPK_CHUNK", None)
    h, logdet, ll, diag_add, mean = _handle_for("matern52", theta, X, y, noise)
    eta = float(np.min(y))
    r1 = h.acq(Xs, _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)
    h.set_option("chunk", 512)
    r2 = h.acq(Xs, _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)
    for k in ("values", "mu", "var"):
        np.testing.assert_array_equal(r1[k], r2[k])
    assert r1["best_idx"] == r2["best_idx"] == int(np.argmax(r1["values"]))
    amp = float(np.exp(theta[0]))
    assert np.all(r1["var"] >= np.finfo(float).eps) and np.all(r1["var"] <= amp * (1 + 1e-12))
    assert np.all(r1["values"] >= 0)
    # at the training inputs: mu(X) - mean = (K - diag_add I) alpha = r - diag_add alpha, i.e.
    # y - mu(X) = diag_add * alpha with alpha = L^-T z rebuilt from the device factors
    mu_t, var_t = h.predict(X[:1024])
    assert np.all(var_t < noise) and np.all(var_t > 0)
    alpha = h.get_linv(N).T @ h.get_z(N)
    resid = y[:1024] - mu_t - diag_add * alpha[:1024]
    assert np.max(np.abs(resid)) < 1e-9 * np.abs(y).max()
    # log-likelihood identity: ll = -1/2 z^T z - 1/2 logdet - n/2 log 2pi with z from the device
    z = h.get_z(N)
    assert abs(ll - (-0.5 * z @ z - 0.5 * logdet - 0.5 * N * np.log(2 * np.pi))) <= 1e-12 * abs(ll)
    # spot check 64 candidates against the oracle (one N=4096 CPU factorisation, a few seconds)
    st = O.gp_fit(O.make_kernel("matern52", D, theta), X, y, noise=noise, normalize_input=False)
    mu_ref, var_ref = O.gp_predict_var_only(st, Xs[:64])
    assert_mean_close(r1["mu"][:64], mu_ref, y)
    assert_var_close(r1["var"][:64], var_ref, amp)
    assert_acq_close(r1["values"][:64], O.acq_ei(mu_ref, var_ref, eta), rtol=1e-8, atol=1e-13)
    ll_ref, logdet_ref = O.gp_loglik_terms(st)
    assert abs(ll - ll_ref) <= 1e-10 * abs(ll_ref) and abs(logdet - logdet_ref) <= 1e-10 * abs(logdet_ref)


# --------------------------------------------------------------------------- incremental refit (SURVEY 8f-4)
def test_fit_append_matches_full_refit_and_oracle():
    """gpk_fit_append: rows appended inside the last 128-row block.  Against a full refit on the device (factor,
    inverse, z, log-likelihood) and against the CPU oracle (posterior moments + EI at the north_star tolerances);
    not-applicable cases leave the model untouched."""
    from robo_b200 import _lib
    D = 5
    X, y, Xs, theta, noise = O.synthetic_problem(700, D, 300, seed_train=21)
    f = product_kernel("matern52", theta, D).flatten()
    da = float(np.sqrt(np.float64(np.sqrt(noise)) ** 2 + G.TINY) ** 2)

    def full(n, d_add=da):
        hh = _lib.Handle(0)
        hh.set_data(X[:n], y[:n])
        hh.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
        return hh, hh.fit(d_add, float(np.mean(y[:n])))

    h, _ = full(650)                                           # NP = 768: rows 640..767 form the last block
    assert h.fit_append(X[:655], y[:655], da, float(np.mean(y[:655]))) is None      # L^-1 not built yet
    mu0, var0 = h.predict(Xs)
    assert h.fit_append(X[:655], y[:655], da * 1.5, float(np.mean(y[:655]))) is None    # other diagonal term
    assert h.fit_append(X[:650], y[:650], da, float(np.mean(y[:650]))) is None          # nothing appended
    np.testing.assert_array_equal(h.predict(Xs)[0], mu0)       # untouched by the refusals
    kss = float(np.exp(theta[0]))
    for n in (651, 655, 700):                                  # repeated appends; the mean moves every time
        mean = float(np.mean(y[:n]))
        res = h.fit_append(X[:n], y[:n], da, mean)
        assert res is not None
        hf, (ld_f, ll_f) = full(n)
        assert abs(res[0] - ld_f) <= 1e-12 * abs(ld_f) and abs(res[1] - ll_f) <= 1e-11 * abs(ll_f)
        L, Lf = h.get_factor(n), hf.get_factor(n)
        np.testing.assert_allclose(L, Lf, rtol=0, atol=1e-11 * np.abs(Lf).max())
        assert np.abs(np.triu(L, 1)).max() == 0.0
        Li, Lif = h.get_linv(n), hf.get_linv(n)
        np.testing.assert_allclose(Li, Lif, rtol=0, atol=1e-10 * np.abs(Lif).max())
        assert np.abs(np.triu(Li, 1)).max() == 0.0
        np.testing.assert_allclose(h.get_z(n), hf.get_z(n), rtol=0, atol=1e-10 * np.abs(hf.get_z(n)).max())
        st = O.gp_fit(oracle_kernel("matern52", theta, D), X[:n], y[:n], noise=noise, normalize_input=False)
        mu_ref, var_ref = O.gp_predict(st, Xs)
        r = h.acq(Xs, _lib.ACQ_EI, float(np.min(y[:n])), 0.0, want_values=True, want_moments=True)
        assert_mean_close(r["mu"], mu_ref, y[:n])
        assert_var_close(r["var"], var_ref, kss)
        assert_acq_close(r["values"], O.acquisition(st, Xs, "ei"))
        hf.close()
    # appended rows that open a new 128-row block: refused, model still the n = 700 one
    Xb = np.vstack([X, np.random.RandomState(5).rand(100, D)])
    yb = np.concatenate([y, np.zeros(100)])
    assert h.fit_append(Xb, yb, da, 0.0) is None
    assert h.predict(Xs)[0].shape == (300,)
    # a single block (N <= 128) has nothing to reuse
    h1, _ = full(100)
    h1.predict(Xs)
    assert h1.fit_append(X[:101], y[:101], da, float(np.mean(y[:101]))) is None
    h1.close()
    h.close()


def test_incremental_refit_through_the_model_classes():
    """train(do_optimize=False) with appended rows (what the solver does between hyper-parameter refits,
    solver/bayesian_optimization.py:161-167) takes the shortcut on the device (DeviceGP.n_appends) and agrees with a
    freshly trained model, output standardisation (a new mean / scale of y at every call) included."""
    from robo_b200 import kernels as K
    from robo_b200.models.gaussian_process import GaussianProcess
    rng = np.random.RandomState(4)
    X, y, Xs = rng.rand(330, 4), rng.rand(330), rng.rand(50, 4)

    def make():
        return GaussianProcess(1.3 * K.Matern52Kernel(np.full(4, 0.8), ndim=4), noise=1e-3, lower=np.zeros(4),
                               upper=np.ones(4), normalize_output=True)
    model = make()
    model.train(X[:300], y[:300], do_optimize=False)
    model.predict(Xs)
    model.train(X[:301], y[:301], do_optimize=False)
    model.predict(Xs)
    model.train(X[:330], y[:330], do_optimize=False)
    assert model.gp.n_appends == 2
    ref = make()
    ref.train(X[:330], y[:330], do_optimize=False)
    assert ref.gp.n_appends == 0
    mu, var = model.predict(Xs)
    mu_r, var_r = ref.predict(Xs)
    assert_mean_close(mu, mu_r, y[:330])
    assert_var_close(var, var_r, 1.3)
    assert abs(model.gp.log_likelihood(model.y) - ref.gp.log_likelihood(ref.y)) <= 1e-11 * abs(ref.gp.log_likelihood(ref.y))


# --------------------------------------------------------------------------- int8 tensor-pipe contraction (option "ozaki")
def test_int8_tile_walks_match_fp64_contraction_and_oracle():
    """Option "ozaki": V = L^-1 K*^T as 28 exact int8 slice products (wgmma s8) instead of fp64 DMMA.  Same
    posterior moments / EI within the north_star tolerances against the oracle AND against the fp64 kernel; the handle
    must fall back to fp64 when the factor is too ill-conditioned for 8 slices (max |L^-1| >= 64)."""
    from robo_b200 import _lib
    N, D, M = 1500, 8, 6000
    X, y, Xs, theta, noise = O.synthetic_problem(N, D, M, seed_train=3)
    eta = float(np.min(y))
    res = {}
    variants = (0, 1, 5)                                    # 1: persistent tile walk; 5: one CTA per tile
    for oz in variants:
        h, logdet, ll, diag_add, mean = _handle_for("matern52", theta, X, y, noise)
        h.set_option("ozaki", 1 if oz else 0)
        h.set_option("ozpersist", 0 if oz == 5 else 1)
        res[oz] = h.acq(Xs, _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)
        if oz:                                              # chunking must stay invisible on the int8 path too
            h.set_option("chunk", 1024)
            r2 = h.acq(Xs, _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)
            for k in ("values", "mu", "var"):
                np.testing.assert_array_equal(res[oz][k], r2[k])
            assert res[oz]["best_idx"] == r2["best_idx"]
        t = h.timings()
        if oz:
            assert t["launches_ozaki"] >= 1 and t["ozaki_max_row_exponent"] <= 7, t
        else:
            assert t["launches_ozaki"] == 0
        h.close()
    st = O.gp_fit(oracle_kernel("matern52", theta, D), X, y, noise=noise, normalize_input=False)
    mu_ref, var_ref = O.gp_predict_var_only_fast(st, Xs)
    amp = float(np.exp(theta[0]))
    for oz in variants:
        assert_mean_close(res[oz]["mu"], mu_ref, y)
        assert_var_close(res[oz]["var"], var_ref, amp)
        assert_acq_close(res[oz]["values"], O.acq_ei(mu_ref, var_ref, eta), rtol=1e-8, atol=1e-13)
    assert all(res[oz]["best_idx"] == int(np.argmax(O.acq_ei(mu_ref, var_ref, eta))) for oz in variants)
    # same integers, same epilogue order: the persistent tile walk changes nothing
    np.testing.assert_array_equal(res[1]["var"], res[5]["var"])
    # odd number of 128-row blocks (N = 1100 -> 9)
    Xo, yo, Xso, theta_o, noise_o = O.synthetic_problem(1100, D, 2500, seed_train=5)
    h, logdet, ll, diag_add, mean = _handle_for("matern52", theta_o, Xo, yo, noise_o)
    h.set_option("ozaki", 1)
    r = h.acq(Xso, _lib.ACQ_EI, float(np.min(yo)), 0.0, want_values=True, want_moments=True)
    assert h.timings()["launches_ozaki"] >= 1
    h.close()
    st = O.gp_fit(oracle_kernel("matern52", theta_o, D), Xo, yo, noise=noise_o, normalize_input=False)
    mu_ref, var_ref = O.gp_predict_var_only_fast(st, Xso)
    assert_mean_close(r["mu"], mu_ref, yo)
    assert_var_close(r["var"], var_ref, float(np.exp(theta_o[0])))
    # ill-conditioned factor (tiny noise, long length scales): row exponents of L^-1 exceed the 8-slice budget -> fp64
    theta_bad = theta + np.r_[0.0, np.full(D, np.log(4.0))]
    h, logdet, ll, diag_add, mean = _handle_for("matern52", theta_bad, X, y, 1e-8)
    h.set_option("ozaki", 1)
    r = h.acq(Xs[:4096], _lib.ACQ_EI, eta, 0.0, want_values=True, want_moments=True)
    t = h.timings()
    assert t["ozaki_max_row_exponent"] > 7 and t["launches_ozaki"] == 0, t
    st = O.gp_fit(oracle_kernel("matern52", theta_bad, D), X, y, noise=1e-8, normalize_input=False)
    mu_ref, var_ref = O.gp_predict_var_only_fast(st, Xs[:4096])
    assert_mean_close(r["mu"], mu_ref, y, tol=1e-8)          # cond ~1e11: the fp64 path itself is at its limit here
    h.close()
