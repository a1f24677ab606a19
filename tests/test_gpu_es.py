"""gpk_ep_joint_min (robo_b200.util.epmgp.joint_min) on the GPU against the numpy restatement tests/es_model.py and
the reference's outputs (tests/golden/es_ep.npz); the reference test's known answers; a fitted model left untouched;
argument validation and the reference's error on a NaN variance.

Tolerance against es_model.  Both evaluate every step in the same order with the same rounding; they differ only in
the libm functions of log_relative_gauss (CUDA's erfc is within 4 ulp, exp and log within 1 ulp, of the correctly
rounded value).  That perturbs each EP message by a few ulp per step.  EP is a contraction near its fixed point, so
the perturbations do not grow across sweeps, and the closed form turns them into at most cond(IRSR) times as much;
1e-9 of each array's max |entry| leaves three orders of magnitude over the 1e-12 this reasoning gives for
cond(IRSR) <= 1e3.  The sweep counts must be equal.
"""
import numpy as np
import pytest

from tests import es_model as M
from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu

KEYS = ("logP", "dlogPdMu", "dlogPdSigma", "dlogPdMudMu")


def _handle():
    from robo_b200 import _lib
    return _lib.moments_handle()


def _close(a, b, rel):
    scale = np.max(np.abs(b)) if b.size else 0.0
    assert np.all(np.abs(a - b) <= rel * scale), (np.max(np.abs(a - b)), scale)


def _random_posterior(nb, seed):
    rng = np.random.RandomState(seed)
    X = rng.rand(12, 3)
    Z = rng.rand(nb, 3)
    ls = 0.3 + rng.rand(3)

    def k(A, B):
        r2 = (((A[:, None, :] - B[None, :, :]) / ls) ** 2).sum(-1)
        r = np.sqrt(5.0 * r2)
        return 1.5 * (1.0 + r + 5.0 * r2 / 3.0) * np.exp(-r)

    K = k(X, X) + 1e-2 * np.eye(12)
    Ks = k(Z, X)
    mu = Ks @ np.linalg.solve(K, rng.randn(12))
    V = np.clip(k(Z, Z) - Ks @ np.linalg.solve(K, Ks.T), np.finfo(float).eps, np.inf)
    return mu, V


def _check_against_model(mu, V):
    dev = _handle().ep_joint_min(mu, V)
    ref = M.joint_min(mu, V)
    assert np.array_equal(dev["sweeps"], ref["sweeps"])
    for key in KEYS:
        _close(dev[key], ref[key], 1e-9)
    return dev


@pytest.mark.parametrize("nb,seed", [(nb, s) for nb in (2, 17, 50, 64) for s in range(5)])
def test_random_posteriors_match_model(nb, seed):
    _check_against_model(*_random_posterior(nb, 100 * nb + seed))


G = np.load(GOLDEN + "/es_ep.npz")


@pytest.mark.parametrize("name", [str(n) for n in G["names"]])
def test_golden(name):
    dev = _check_against_model(G[name + "_mu"], G[name + "_V"])
    # the reference's own outputs, at the restatement's tolerance to them (tests/test_es_cpu.py)
    _close(dev["logP"], G[name + "_logP"], 1e-12)
    keep = G[name + "_dlogPdMu"].shape[0]
    for key in KEYS[1:]:
        _close(dev[key][:keep], G[name + "_" + key], 1e-10)


def test_known_answers():
    from robo_b200.util import epmgp
    nb = 50
    p = np.exp(epmgp.joint_min(np.ones(nb), np.eye(nb)))
    assert p.shape == (nb,)
    assert np.all(p < 1 / nb + 0.03) and np.all(p > 1 / nb - 0.01)
    m = np.ones(nb) * 1000
    m[0] = 1
    p = np.exp(epmgp.joint_min(m, np.eye(nb)))
    assert p[0] == 1.0
    out = epmgp.joint_min(m, np.eye(nb), with_derivatives=True)
    assert [a.shape for a in out] == [(nb,), (nb, nb), (nb, nb * (nb + 1) // 2), (nb, nb, nb)]


def test_nan_variance_raises_reference_exception():
    from robo_b200.util import epmgp
    V = np.eye(4)
    V[2, 3] = V[3, 2] = np.nan
    with pytest.raises(Exception, match="an error occurs while running expectation propagation in entropy search. "
                                        "Resulting variance contains NaN"):
        epmgp.joint_min(np.zeros(4), V, with_derivatives=True)


@pytest.mark.parametrize("nb", [0, 1, 65])
def test_bad_nb(nb):
    with pytest.raises(ValueError):
        _handle().ep_joint_min(np.zeros(nb), np.eye(nb))


def test_bad_shape():
    with pytest.raises(ValueError):
        _handle().ep_joint_min(np.zeros(4), np.eye(5))


def test_fitted_model_untouched():
    from tests.golden_cases import kernel_spec, load_case
    from tests.product_cases import product_model
    d, _ = load_case("gp_branin_ny0")
    family, theta = kernel_spec("gp_branin_ny0")
    model = product_model(d, family, theta)
    model.train(d["X"], d["y"], do_optimize=False)
    Xs = d["lower"] + (d["upper"] - d["lower"]) * np.random.RandomState(3).rand(300, 2)
    before = model.predict(Xs)
    h = model.gp.handle
    h.ep_joint_min(*_random_posterior(50, 7))
    after = model.predict(Xs)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])


# ---- gpk_es_update / gpk_es_compute, InformationGain and the entropy_search facade --------------------------------
def _branin(x):
    return (x[1] - 5.1 / (4 * np.pi ** 2) * x[0] ** 2 + 5 / np.pi * x[0] - 6) ** 2 \
        + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x[0]) + 10


LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])


def _gp(n=30, seed=0):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    rng = np.random.RandomState(seed)
    X = LO + (UP - LO) * rng.rand(n, 2)
    y = np.array([_branin(x) for x in X])
    gp = GaussianProcess(2 * K.Matern52Kernel(np.ones(2), ndim=2), normalize_input=True, normalize_output=False,
                         lower=LO, upper=UP, rng=np.random.RandomState(1))
    gp.train(X, y, do_optimize=True)
    return gp, X


def _ig(gp, seed=3):
    from robo_b200.acquisition_functions import EI, InformationGain
    ig = InformationGain(gp, LO, UP, sampling_acquisition=EI, rng=np.random.RandomState(seed))
    ig.update(gp)
    return ig


def _candidates(X, m, seed=4):
    rng = np.random.RandomState(seed)
    C = LO + (UP - LO) * rng.rand(m, 2)
    C[:5] = X[:5]                                      # training inputs: v close to the noise, v_ may be negative
    C[5] = UP + 1.0                                    # outside the bounds
    C[6] = LO - 0.5
    return C


def test_compute_matches_model_on_device_moments():
    """Tolerance: sigma through the device's own predict_cov differs from the U-path by the rounding of a difference
    k(zb, x) - K(x, X) U whose terms are of size amp, i.e. by about N eps amp in absolute terms, and dH sees sigma
    through 1 / v_.  Away from v = sn2 (|v - sn2| >= 1e-3 v) and away from the training inputs (where that difference
    cancels to almost nothing, so its absolute rounding is its whole size, and entries flip across the eps clip),
    dH is a mean of sums of terms exp(l) (l + lmb) plus H, so the bound is taken against the size of those terms,
    S = |H| + max |lmb| + 1, not against |dH|, which cancels: 1e-7 S.  At the training inputs the two paths were seen
    0.5 % apart."""
    gp, X = _gp()
    ig = _ig(gp)
    C = _candidates(X, 300)
    dev = ig.compute(C)
    st = dict(logP=ig.logP.ravel(), lmb=ig.lmb.ravel(), dlogPdMu=ig.dlogPdMu, dlogPdSigma=ig.dlogPdSigma,
              dlogPdMudMu=ig.dlogPdMudMu, W=ig.W.ravel(), sn2=ig.sn2)
    _, v = gp.predict(C)
    lp, lm = ig.logP.ravel(), ig.lmb.ravel()
    S = abs(np.sum(np.exp(lp) * (lp + lm))) + np.max(np.abs(lm)) + 1.0
    n_checked = 0
    for i, x in enumerate(C):
        if np.any(x < LO) or np.any(x > UP):
            assert dev[i] == np.spacing(1)
            continue
        sigma = gp.predict_variance(ig.zb, x[None]).ravel()
        ref = M.compute_value(M.dh_folded(st, v[i], sigma), x, LO, UP)
        near_train = np.min(np.max(np.abs(X - x) / (UP - LO), axis=1)) < 1e-2
        if abs(v[i] - ig.sn2) >= 1e-3 * v[i] and np.isfinite(ref) and not near_train:
            assert abs(dev[i] - ref) <= 1e-7 * S, (i, dev[i], ref, S)
            n_checked += 1
    assert n_checked > 250
    assert np.all(np.isfinite(dev[:5]) | (dev[:5] == -np.inf))


def test_compute_deterministic_across_chunk_and_dev():
    import torch
    gp, X = _gp()
    ig = _ig(gp)
    C = _candidates(X, 4096)
    base = ig.compute(C)
    h = gp.gp.handle
    for key, val in (("chunk", 2048), ("ozcluster", 1), ("ozcluster", 4), ("chunk", 0)):
        h.set_option(key, val)
        assert np.array_equal(ig.compute(C), base), (key, val)
    dX = torch.tensor(C, dtype=torch.float64, device="cuda")
    dout = torch.empty(len(C), dtype=torch.float64, device="cuda")
    h.es_compute_dev(dX.data_ptr(), len(C), dout.data_ptr())
    h.synchronize()
    assert np.array_equal(dout.cpu().numpy(), base)


def test_marginalised_value_is_mean_of_models():
    from robo_b200 import kernels as K
    from robo_b200.acquisition_functions import EI, InformationGain, MarginalizationGPMCMC
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    rng = np.random.RandomState(4)
    X = LO + (UP - LO) * rng.rand(20, 2)
    y = np.array([_branin(x) for x in X])
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)), n_hypers=10,
                                chain_length=20, burnin_steps=20, normalize_input=True, normalize_output=False,
                                lower=LO, upper=UP, rng=np.random.RandomState(2))
    model.train(X, y, do_optimize=True)
    acq = MarginalizationGPMCMC(InformationGain(model, LO, UP, sampling_acquisition=EI, rng=np.random.RandomState(0)))
    acq.update(model)
    C = _candidates(X, 200)
    vals = acq.compute(C)
    per = []
    for e, m in zip(acq.estimators, model.models):
        st = dict(logP=e.logP.ravel(), lmb=e.lmb.ravel(), dlogPdMu=e.dlogPdMu, dlogPdSigma=e.dlogPdSigma,
                  dlogPdMudMu=e.dlogPdMudMu, W=e.W.ravel(), sn2=e.sn2)
        _, v = m.predict(C)
        per.append([M.compute_value(M.dh_folded(st, v[i], m.predict_variance(e.zb, x[None]).ravel()), x, LO, UP)
                    for i, x in enumerate(C)])
    ref = np.mean(np.array(per), axis=0)
    ok = np.isfinite(ref) & (np.abs(ref) < 1e300)
    assert ok.sum() > 150
    assert np.all(np.abs(vals[ok] - ref[ok]) <= 1e-6 * np.maximum(np.abs(ref[ok]), 1e-3))


def test_es_argument_validation():
    gp, X = _gp()
    h = gp.gp.handle
    zb = LO + (UP - LO) * np.random.RandomState(0).rand(10, 2)
    W = np.linspace(-2, 2, 10)
    with pytest.raises(ValueError):
        h.es_compute(X[:4])                                         # before update
    for nb in (1, 65):
        z = LO + (UP - LO) * np.random.RandomState(0).rand(nb, 2)
        with pytest.raises(ValueError):
            h.es_update(z, np.zeros(nb), 1e-3, W, LO, UP)
    with pytest.raises(ValueError):
        h.es_update(zb, np.zeros(10), 1e-3, np.zeros(0), LO, UP)    # Np < 1
    lmb = np.zeros(10)
    lmb[3] = -np.inf
    with pytest.raises(ValueError, match="lmb should not be infinite"):
        h.es_update(zb, lmb, 1e-3, W, LO, UP)
    from robo_b200 import _lib
    fresh = _lib.Handle()
    with pytest.raises((ValueError, RuntimeError)):
        fresh.es_update(zb, np.zeros(10), 1e-3, W, LO, UP)
    from robo_b200.acquisition_functions import InformationGain
    ig = InformationGain(gp, LO, UP, rng=np.random.RandomState(0))
    with pytest.raises(ValueError):
        ig.compute(X[:3])
    with pytest.raises(NotImplementedError):
        ig.compute(X[:3], derivative=True)


def test_information_gain_refuses_host_models():
    from robo_b200.acquisition_functions import InformationGain

    class Host(object):
        def get_noise(self):
            return 1e-3
    ig = InformationGain(Host(), LO, UP, rng=np.random.RandomState(0))
    with pytest.raises(TypeError):
        ig.update(Host())


@pytest.mark.parametrize("model", ["gp", "gp_mcmc"])
def test_facade_branin(model):
    """Seed 1 for the facade's rng and numpy's global stream (RandomSampling's candidates), 12 evaluations.  Measured
    on an H100: f_opt = 1.58 (gp) and 0.99 (gp_mcmc); the Branin minimum is 0.398."""
    from robo_b200.fmin import entropy_search
    runs = []
    for _ in range(2):
        np.random.seed(1)
        runs.append(entropy_search(_branin, LO, UP, num_iterations=12, model=model, n_init=3,
                                   rng=np.random.RandomState(1)))
    a, b = runs
    X = np.array(a["X"])
    assert np.all(X >= LO) and np.all(X <= UP)
    assert np.array_equal(X, np.array(b["X"])) and a["f_opt"] == b["f_opt"]
    print("entropy_search", model, "f_opt", a["f_opt"])
    assert a["f_opt"] < 3.0
    with pytest.raises(ValueError):
        entropy_search(_branin, LO, UP, maximizer="scipy")
