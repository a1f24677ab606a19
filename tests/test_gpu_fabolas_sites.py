"""The environment factor at the sites built on the entropy-search kernel value and in the device hyper sampler:
gpk_es_update / gpk_es_moments / gpk_es_compute against numpy (U, the cross-covariance sigma, the variance) and the dH
restatement tests/es_model.py fed the device's own moments; gpk_es_cost_multi bit-identical to the per-estimator loop
over FabolasGPMCMC models with the factor; every device maximizer over InformationGainPerUnitCost with such models;
gpk_hyper_lnpost with EnvPrior against the numpy log-likelihood and the host prior; gpk_sample_hypers on them.

Tolerances: U, sigma and the variance come from the fp64 path and agree with scipy to rounding amplified by the
conditioning of K (1e-8 relative to the largest entry on these problems); dH against es_model on the device's own
moments differs only in summation order and CUDA's exp / log (1e-9 of |H| + max |lmb| + 1); log-likelihoods 1e-9."""
import numpy as np
import pytest
import scipy.linalg as spla

from tests import env_kernel_model as E
from tests import es_model as M

pytestmark = pytest.mark.gpu

EPS = np.finfo(float).eps
LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
EXT_LO, EXT_UP = np.append(LO, 0.0), np.append(UP, 1.0)
IS_ENV = np.array([0, 0, 1])
THETA = dict(log_amp=0.2, lm=(-1.0, -0.5), la=0.1, lb=-0.3)


def _handle(X, y, lo=None, up=None):
    from robo_b200 import _lib
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(_lib.MATERN52, THETA["log_amp"], [0, 1], [0, 1], list(THETA["lm"]))
    h.set_env_factor(2, THETA["la"], THETA["lb"])
    if lo is not None:
        h.set_input_bounds(lo, up)
    return h


def test_es_update_and_compute_with_the_factor():
    rng = np.random.RandomState(11)
    n, nb, Np, diag, sn2 = 150, 20, 30, 1e-2, 1e-3
    X = rng.rand(n, 3)
    X[:, 2] = (1 - X[:, 2]) ** 2
    y = np.sin(3 * X[:, 0]) + X[:, 2] + 0.05 * rng.randn(n)
    lo, up = np.array([-1.0, 0.0, 0.0]), np.array([2.0, 3.0, 1.0])
    h = _handle(X, y, lo, up)
    h.fit(diag, 0.0)
    zb = lo + (up - lo) * rng.rand(nb, 3)
    lmb = np.log(0.05 + rng.rand(nb))
    W = rng.randn(Np)
    r = h.es_update(zb, lmb, sn2, W, lo, up)
    k = E.fabolas_kernel(2, THETA["log_amp"], THETA["lm"], THETA["la"], THETA["lb"])
    zs = (zb - lo) / (up - lo)
    K = k.get_value(X) + diag * np.eye(n)
    L = spla.cholesky(K, lower=True)
    U_ref = spla.cho_solve((L, True), k.get_value(X, zs))
    U = h.es_get_u()
    assert np.max(np.abs(U - U_ref)) <= 1e-8 * np.max(np.abs(U_ref))
    Xs = lo + (up - lo) * rng.rand(300, 3)
    Xs[:3] = lo + (up - lo) * X[:3]                              # training inputs: sigma cancels and clips
    Xs[3:5] = zb[:2]                                             # the representer points themselves
    Xs[5] = up + 0.5                                             # outside the box
    xn = (Xs - lo) / (up - lo)
    Ks = k.get_value(xn, X)
    var_ref = np.diag(k.get_value(xn)) - np.einsum("ij,ij->i", Ks, spla.cho_solve((L, True), Ks.T).T)
    sig_ref = np.clip(k.get_value(xn, zs) - Ks @ U_ref, EPS, np.inf)
    var, sig = h.es_moments(Xs)
    assert np.max(np.abs(var - np.clip(var_ref, EPS, np.inf))) <= 1e-8 * np.max(np.abs(var_ref))
    assert np.max(np.abs(sig - sig_ref)) <= 1e-8 * np.max(np.abs(sig_ref))
    state = dict(logP=r["logP"], lmb=lmb, dlogPdMu=r["dlogPdMu"], dlogPdSigma=r["dlogPdSigma"],
                 dlogPdMudMu=r["dlogPdMudMu"], W=W, sn2=sn2)
    state["H"] = -float(np.sum(np.exp(r["logP"]) * (r["logP"] + lmb)))
    dh = h.es_compute(Xs)
    S = abs(state["H"]) + np.max(np.abs(lmb)) + 1.0
    n_checked = 0
    for i in range(len(Xs)):
        ref = M.compute_value(M.dh_folded(state, var[i], sig[i]), Xs[i], lo, up)
        if not np.isfinite(ref) or not np.isfinite(dh[i]) or ref == EPS:
            assert dh[i] == ref or (np.isnan(dh[i]) and np.isnan(ref)), (i, dh[i], ref)
            continue
        assert abs(dh[i] - ref) <= 1e-9 * S, (i, dh[i], ref)
        n_checked += 1
    assert n_checked > 250
    h.close()


def _env_kernel(amp=1.3, ls=(0.4, 0.6), la=0.1, lb=0.1):
    from robo_b200 import kernels as K
    k = amp * K.Matern52Kernel(np.ones(1) * ls[0], ndim=3, axes=0)
    k *= K.Matern52Kernel(np.ones(1) * ls[1], ndim=3, axes=1)
    return k * K.BayesianLinearRegressionKernel(la, lb, ndim=3, axes=2)


def _mcmc_pair(n_hypers, n, seed=0, hyper_sampler="host"):
    from robo_b200.models import FabolasGPMCMC
    from robo_b200.priors import EnvPrior
    rng = np.random.RandomState(seed)
    X = np.concatenate((LO + (UP - LO) * rng.rand(n, 2), rng.uniform(0.05, 1.0, (n, 1))), axis=1)
    y = np.sin(X[:, 0]) + 0.1 * X[:, 1] + X[:, 2]
    c = -1.5 + 3.0 * X[:, 2] + 0.05 * X[:, 0]
    out = []
    for i, (t, basis) in enumerate(((y, lambda s: (1 - s) ** 2), (c, lambda s: s))):
        k = _env_kernel()
        m = FabolasGPMCMC(k, basis_func=basis, prior=EnvPrior(len(k) + 1, 2, 2, rng=np.random.RandomState(1 + i)),
                          n_hypers=n_hypers, chain_length=4, burnin_steps=3, lower=LO, upper=UP,
                          rng=np.random.RandomState(2 + i), hyper_sampler=hyper_sampler)
        m.train(X, t, do_optimize=True)
        out.append(m)
    return out[0], out[1], X


def _acq(objm, costm):
    from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost, MarginalizationGPMCMC
    acq = MarginalizationGPMCMC(InformationGainPerUnitCost(objm, costm, EXT_LO, EXT_UP, IS_ENV, sampling_acquisition=EI,
                                                           rng=np.random.RandomState(0)))
    np.random.seed(0)
    acq.update(objm, costm, overhead=0.05)
    return acq


def test_es_cost_multi_equals_per_estimator_loop_with_the_factor():
    objm, costm, X = _mcmc_pair(12, 60)
    assert objm.models[0].gp.kernel.flatten()["env"] is not None
    acq = _acq(objm, costm)
    assert acq._es_cost_spec() is not None
    rng = np.random.RandomState(4)
    C = EXT_LO + (EXT_UP - EXT_LO) * rng.rand(2200, 3)
    vals = acq.compute(C)
    per = np.array([e.compute(C) for e in acq.estimators])
    assert np.array_equal(vals, per.mean(axis=0))
    assert np.isfinite(vals).sum() > 2000
    assert acq.argmax(C) == int(np.argmax(vals))


@pytest.mark.parametrize("name", ["DeviceRandomSampling", "DifferentialEvolution", "SciPyOptimizer", "CMAES", "Direct"])
def test_every_device_maximizer_completes(name):
    from robo_b200 import maximizers
    objm, costm, _ = _mcmc_pair(12, 40)
    acq = _acq(objm, costm)
    kw = dict(rng=np.random.RandomState(5))
    if name in ("CMAES", "Direct"):
        kw["verbose"] = False
    x = getattr(maximizers, name)(acq, EXT_LO, EXT_UP, **kw).maximize()
    x = np.asarray(x).ravel()
    assert x.shape == (3,) and np.all(np.isfinite(x)) and np.all(x >= EXT_LO) and np.all(x <= EXT_UP)


def test_hyper_lnpost_with_env_prior_matches_numpy():
    from robo_b200 import _lib
    from robo_b200.device_gp import TINY
    from robo_b200.models.gaussian_process_mcmc import _hyper_prior
    from robo_b200.priors import EnvPrior
    rng = np.random.RandomState(12)
    n = 60
    X = rng.rand(n, 3)
    X[:, 2] = (1 - X[:, 2]) ** 2
    y = np.sin(3 * X[:, 0]) + X[:, 2] + 0.05 * rng.randn(n)
    kernel = _env_kernel()
    prior = EnvPrior(len(kernel) + 1, n_ls=2, n_lr=2, rng=np.random.RandomState(0))
    f = kernel.flatten()
    kind, par, n_ls, n_lr = _hyper_prior(prior)
    mean = float(np.mean(y))
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    h.set_env_factor(*f["env"])
    _lib.set_hyper_model(h, f["slots"], len(f["axis"]), mean, TINY, kind, par, n_ls, n_lr)
    dim = len(kernel) + 1
    T = np.column_stack([rng.uniform(0.1, 2, 30), rng.uniform(-3, 1, (30, 2)), rng.uniform(-2, 2, (30, 2)),
                         rng.uniform(-8, -2, 30)])
    ll, lp = _lib.hyper_lnpost(h, T)
    for t, l, p in zip(T, ll, lp):
        k = E.fabolas_kernel(2, t[0], t[1:3], t[3], t[4])
        yerr = np.sqrt(np.exp(t[-1]))
        K = k.get_value(X) + np.sqrt(yerr ** 2 + TINY) ** 2 * np.eye(n)
        Lc = spla.cholesky(K, lower=True)
        z = spla.solve_triangular(Lc, y - mean, lower=True)
        ref = -0.5 * z @ z - np.sum(np.log(np.diag(Lc))) - 0.5 * n * np.log(2 * np.pi)
        assert l == pytest.approx(ref, rel=1e-9, abs=1e-9)
        assert p == pytest.approx(prior.lnprob(t), rel=1e-12, abs=1e-12)
    # the chain runs on the factor's parameters: finite log-posteriors and moves in log_a / log_b
    p0 = np.tile(np.r_[1.0, -1.0, -1.0, 0.1, 0.1, -5.0], (2 * dim, 1)) + 0.05 * rng.randn(2 * dim, dim)
    r = _lib.sample_hypers(h, p0, 20, 123)
    assert r["pos"].shape == (2 * dim, dim) and np.all(np.isfinite(r["lnpost"]))
    assert np.any(r["pos"][:, 3:5] != p0[:, 3:5])
    h.close()


def test_fabolas_gp_mcmc_device_sampler_with_the_factor():
    objm, costm, X = _mcmc_pair(12, 40, hyper_sampler="device")
    assert len(objm.models) == 12
    mu, var = objm.predict(X[:10])
    assert np.all(np.isfinite(mu)) and np.all(var > 0)
