"""The sampling-based entropy search on the GPU (gpk_esmc.cuh): gpk_mc_pmin, gpk_esmc_update / gpk_esmc_compute,
gpk_esmc_multi, gpk_maximize_de_esmc and InformationGainMC under the maximizers.

The counts of every p_min are pinned bit for bit to tests/mc_model.py fed the device's own draws F (and, per candidate,
the device's v and sigma from gpk_es_moments and the update's Mb and Vb); the values then differ only by the Nb logs
(numpy's against CUDA's), which the bound below allows."""
import numpy as np
import pytest
from scipy.stats import norm

from oracle import robo_oracle as O
from tests import de_model as DE
from tests import mc_model as M
from tests.product_cases import product_kernel

pytestmark = pytest.mark.gpu

LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])


def _branin(x):
    return (x[1] - 5.1 / (4 * np.pi ** 2) * x[0] ** 2 + 5 / np.pi * x[0] - 6) ** 2 \
        + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x[0]) + 10


def _spd(nb, seed):
    rng = np.random.RandomState(seed)
    A = rng.randn(nb, nb)
    return A @ A.T / nb + 0.05 * np.eye(nb)


def _handle():
    from robo_b200 import _lib
    return _lib.moments_handle()


# ---- gpk_mc_pmin on caller operands ------------------------------------------------------------------------------
@pytest.mark.parametrize("nb,np_,nf", [(2, 1, 500), (50, 1, 500), (50, 50, 500), (64, 7, 333), (64, 400, 64),
                                       (1, 3, 10)])
def test_mc_pmin_bit_identical_to_restatement(nb, np_, nf):
    h = _handle()
    rng = np.random.RandomState(nb + np_)
    m = rng.randn(nb, np_) * 0.3
    V = _spd(nb, nb)
    seed = 1234567 + nb
    pmin, nj = h.mc_pmin(m, V, nf, seed)
    F = h.mc_draws(seed, nb, nf)
    ref = M.joint_pmin(m, V, F)
    assert pmin.tobytes() == ref["pmin"].tobytes()
    assert nj == (1 if ref["rung"] > 0 else 0)
    assert np.all(pmin >= 1e-70)


def test_mc_pmin_exact_ties_clamp_and_jitter():
    """Means so large that every draw rounds away tie exactly: the first index takes every column, the others clamp
    to 1e-70.  A singular V climbs the jitter ladder."""
    h = _handle()
    m = np.array([5e17, 1e17, 1e17, 3e17])
    pmin, nj = h.mc_pmin(m, np.eye(4), 300, 9)
    assert pmin.tolist() == [1e-70, 1.0, 1e-70, 1e-70] and nj == 0
    V = np.ones((3, 3))
    pmin, nj = h.mc_pmin(np.zeros(3), V, 400, 10)
    ref = M.joint_pmin(np.zeros(3), V, h.mc_draws(10, 3, 400))
    assert pmin.tobytes() == ref["pmin"].tobytes() and nj == 1 and ref["rung"] > 0


def test_mc_pmin_known_answer_and_not_pd():
    from robo_b200.util.mc_part import joint_pmin
    np.random.seed(0)
    p = joint_pmin(np.zeros(2), np.eye(2), 10000)          # test/test_util/test_mc_part.py
    np.testing.assert_allclose(p, [0.5, 0.5], atol=0.1)
    with pytest.raises(np.linalg.LinAlgError):
        joint_pmin(np.zeros(3), -1e5 * np.eye(3), 100)          # not PD even at noise 10000


@pytest.mark.parametrize("m2,v11,v22,v12", [(0.3, 1.0, 2.0, 0.4), (-1.0, 0.5, 0.5, -0.2), (0.0, 1.0, 1.0, 0.9)])
def test_mc_pmin_two_points_closed_form(m2, v11, v22, v12):
    h = _handle()
    nf = 200000
    p, _ = h.mc_pmin(np.array([0.0, m2]), np.array([[v11, v12], [v12, v22]]), nf, 77)
    q = norm.cdf((m2 - 0.0) / np.sqrt(v11 + v22 - 2 * v12))       # P(f1 < f2)
    assert abs(p[0] - q) <= 5 * np.sqrt(q * (1 - q) / nf) + 1e-12
    assert p[0] + p[1] == pytest.approx(1.0, abs=1e-12)


def test_draws_law_and_box_muller():
    h = _handle()
    F = h.mc_draws(2024, 64, 4001)
    n = F.size
    assert abs(F.mean()) <= 5 / np.sqrt(n)
    assert abs(F.var() - 1.0) <= 5 * np.sqrt(2.0 / n)
    ref = M.draws(2024, 64, 4001)
    # numpy's log and cos / sin against CUDA's log and sincospi: a few ulp of the radius (|F| <= 9 here)
    np.testing.assert_allclose(F, ref, rtol=0, atol=64 * np.finfo(float).eps * 9)
    # a prefix: F[k][f] depends on (seed, k, f) only
    assert h.mc_draws(2024, 3, 10).tobytes() == F[:3, :10].tobytes()


# ---- InformationGainMC on one GP -------------------------------------------------------------------------------
_CACHE = {}


def _single(Nb=50, Np=50, Nf=500):
    key = ("one", Nb, Np, Nf)
    if key not in _CACHE:
        from robo_b200.acquisition_functions import EI, InformationGainMC
        from robo_b200.models.gaussian_process import GaussianProcess
        X, y, _, theta, noise = O.synthetic_problem(256, 3, 16, seed_train=11)
        model = GaussianProcess(product_kernel("matern52", theta, 3), noise=noise, normalize_input=False)
        model.train(X, y, do_optimize=False)
        lower, upper = np.zeros(3), np.ones(3)
        ig = InformationGainMC(model, lower, upper, Nb=Nb, Np=Np, Nf=Nf, sampling_acquisition=EI,
                               rng=np.random.RandomState(3), representer_sampler="device")
        ig.update(model)
        _CACHE[key] = (ig, lower, upper, X)
    return _CACHE[key]


def _restate(ig, C):
    h = ig._ready_handle()
    var, sig = h.es_moments(C)
    Mb, Vb = h.esmc_get_state()
    F = h.esmc_get_draws()
    H = M.H_of(ig.logP, ig.lmb)
    return [M.candidate(Mb, Vb, ig.W, F, var[i], sig[i], ig.sn2, ig.lmb, H) for i in range(C.shape[0])]


def test_update_restated():
    ig = _single()[0]
    h = ig._ready_handle()
    Mb, Vb = h.esmc_get_state()
    ref = M.joint_pmin(Mb, Vb, h.esmc_get_draws())
    assert ig.pmin.tobytes() == ref["pmin"].tobytes()
    assert np.allclose(ig.logP.ravel(), np.log(ref["pmin"]), rtol=0, atol=1e-15)
    assert ig.zb.shape == (50, 3) and np.all(np.isfinite(ig.lmb))


@pytest.mark.parametrize("Nb,Np", [(50, 50), (16, 400), (64, 3)])
def test_compute_against_restatement(Nb, Np):
    ig, lower, upper, _ = _single(Nb=Nb, Np=Np, Nf=200)
    C = np.random.RandomState(5).rand(24, 3)
    dev = ig.compute(C)
    for i, r in enumerate(_restate(ig, C)):
        # identical counts give identical pmin; the values then differ by the Nb logs alone
        bound = 4 * Nb * np.finfo(float).eps * (1.0 + np.sum(np.abs(r["pmin"] * (np.log(r["pmin"]) + ig.lmb.ravel()))))
        assert abs(dev[i] - r["value"]) <= bound, (i, dev[i], r["value"])


def test_values_independent_of_position_chunking_and_split():
    ig, lower, upper, _ = _single()
    h = ig._ready_handle()
    C = np.random.RandomState(9).rand(16385, 3)               # ES_CH + 1: two passes
    ref = ig.compute(C)
    perm = np.random.RandomState(1).permutation(C.shape[0])
    assert ig.compute(C[perm]).tobytes() == ref[perm].tobytes()
    parts = np.concatenate([ig.compute(C[:7]), ig.compute(C[7:8000]), ig.compute(C[8000:])])
    assert parts.tobytes() == ref.tobytes()
    assert h.esmc_compute(C[:1]).tobytes() == ref[:1].tobytes()
    assert np.all(np.isfinite(ref))
    import torch
    dX = torch.tensor(C[:300], dtype=torch.float64, device="cuda")
    dout = torch.empty(300, dtype=torch.float64, device="cuda")
    h.esmc_compute_dev(dX.data_ptr(), 300, dout.data_ptr())
    h.synchronize()
    assert dout.cpu().numpy().tobytes() == ref[:300].tobytes()


def test_representer_and_training_points_take_the_jitter_path():
    """At a representer point the fantasised Vb_new loses a rank: its factorisation climbs the jitter ladder wherever
    rounding leaves a pivot <= 0.  The device counts those factorisations, scores them, and matches the restatement."""
    ig, lower, upper, X = _single()
    h = ig._ready_handle()
    C = np.concatenate([ig.zb, X[:4]])
    dev = ig.compute(C)
    rs = _restate(ig, C)
    jittered = sum(r["rung"] > 0 for r in rs)
    assert h.esmc_last_jitter() == jittered >= 1
    for d, r in zip(dev, rs):
        assert np.isfinite(d)
        assert abs(d - r["value"]) <= 1e-11 * (1.0 + abs(r["value"]))


def test_updates_exclude_each_other():
    from robo_b200.acquisition_functions import EI, InformationGain, InformationGainMC
    from robo_b200.models.gaussian_process import GaussianProcess
    X, y, _, theta, noise = O.synthetic_problem(64, 2, 4, seed_train=5)
    model = GaussianProcess(product_kernel("matern52", theta, 2), noise=noise, normalize_input=False)
    model.train(X, y, do_optimize=False)
    lo, up = np.zeros(2), np.ones(2)
    h = model.gp.handle
    C = np.random.RandomState(0).rand(5, 2)
    mc = InformationGainMC(model, lo, up, Nb=10, Nf=50, Np=5, sampling_acquisition=EI, rng=np.random.RandomState(0),
                           representer_sampler="device")
    mc.update(model)
    mc.compute(C)
    with pytest.raises(ValueError):
        h.es_compute(C)
    ep = InformationGain(model, lo, up, Nb=10, Np=5, sampling_acquisition=EI, rng=np.random.RandomState(0),
                         representer_sampler="device")
    ep.update(model)
    ep.compute(C)
    with pytest.raises(ValueError):
        h.esmc_compute(C)
    with pytest.raises(ValueError):
        mc.compute(C)
    mc.update(model)
    assert np.all(np.isfinite(mc.compute(C)))
    with pytest.raises(NotImplementedError):
        mc.compute(C, derivative=True)


# ---- marginalised over a GP-MCMC ensemble -------------------------------------------------------------------------
def _ensemble(sampler="device"):
    key = ("ten", sampler)
    if key not in _CACHE:
        from robo_b200 import kernels as K
        from robo_b200.acquisition_functions import EI, InformationGainMC, MarginalizationGPMCMC
        from robo_b200.models import GaussianProcessMCMC
        from robo_b200.priors import DefaultPrior
        rng = np.random.RandomState(4)
        X = LO + (UP - LO) * rng.rand(20, 2)
        y = np.array([_branin(x) for x in X])
        kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
        model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)),
                                    n_hypers=10, chain_length=20, burnin_steps=20, normalize_input=True,
                                    normalize_output=False, lower=LO, upper=UP, rng=np.random.RandomState(2))
        model.train(X, y, do_optimize=True)
        acq = MarginalizationGPMCMC(InformationGainMC(model, LO, UP, sampling_acquisition=EI,
                                                      rng=np.random.RandomState(0), representer_sampler=sampler))
        acq.update(model)
        assert len(acq.estimators) == 10
        _CACHE[key] = (acq, X)
    return _CACHE[key]


def test_esmc_multi_bit_identical_to_per_estimator_loop():
    from robo_b200 import _lib
    acq, X = _ensemble()
    handles = [e._ready_handle() for e in acq.estimators]
    assert len(set(e.seed for e in acq.estimators)) == 10              # one seed, one F per estimator
    C = LO + (UP - LO) * np.random.RandomState(5).rand(700, 2)
    per = np.array([e.compute(C) for e in acq.estimators])
    ref = _lib.moments_handle().reduce_models(per)
    r = _lib.esmc_multi(handles, C)
    assert r["values"].tobytes() == ref.tobytes()
    assert r["best_idx"] == int(np.argmax(ref))
    assert acq.compute(C).tobytes() == ref.tobytes() and acq.argmax(C) == int(np.argmax(ref))
    one = _lib.moments_handle().reduce_models(per[:1])
    assert _lib.esmc_multi(handles[:1], C)["values"].tobytes() == one.tobytes()


@pytest.mark.parametrize("which", ["one", "ten"])
def test_de_trajectory_bit_for_bit(which):
    from robo_b200 import _lib
    if which == "one":
        ig, lower, upper, _ = _single()
        handles, score = [ig._ready_handle()], (lambda Xb: ig._ready_handle().esmc_compute(Xb))
    else:
        acq, _ = _ensemble()
        lower, upper = LO, UP
        handles = [e._ready_handle() for e in acq.estimators]
        score = lambda Xb: _lib.esmc_multi(handles, Xb)["values"]
    for seed, maxiter in [(3, 0), (4, 2), (6, 8)]:
        dev = _lib.maximize_de_esmc(handles, seed, 30, maxiter, (0.5, 1.0), 0.7, 0.01, 0.0, lower, upper,
                                    want_population=True)
        ref = DE.maximize_de(score, seed, 30, lower, upper, maxiter)
        assert dev["nit"] == ref["nit"] and dev["nfev"] == ref["nfev"]
        assert dev["population"].tobytes() == ref["population"].tobytes()
        assert dev["energies"].tobytes() == ref["energies"].tobytes()
        assert dev["x"].tobytes() == ref["x"].tobytes()


@pytest.mark.parametrize("sampler", ["host", "device"])
def test_maximizers_end_to_end(sampler):
    from robo_b200.maximizers import DifferentialEvolution, RandomSampling, SciPyOptimizer
    acq, X = _ensemble(sampler)
    assert all(e.zb.shape == (50, 2) for e in acq.estimators)
    de = DifferentialEvolution(acq, LO, UP, n_iters=5, rng=np.random.RandomState(1), polish=False)
    x = de.maximize()
    assert np.all(x >= LO) and np.all(x <= UP)
    value = float(acq.compute(x[None, :])[0])
    assert value == pytest.approx(-de.last["device_energy"], rel=1e-12, abs=1e-12)
    np.random.seed(3)
    rs = RandomSampling(acq, LO, UP, n_samples=500, rng=np.random.RandomState(2))
    xr = rs.maximize()
    assert np.all(xr >= LO) and np.all(xr <= UP)
    with pytest.raises(ValueError):
        DifferentialEvolution(acq, LO, UP, n_iters=2, rng=np.random.RandomState(1), polish="device").maximize()
    so = SciPyOptimizer(acq.estimators[0], LO, UP, n_restarts=2, rng=np.random.RandomState(0))
    so.maximize()
    assert so.last["device"] is False


def test_bayesian_optimization_on_branin():
    """InformationGainMC with DifferentialEvolution as the acquisition of a BayesianOptimization loop."""
    from robo_b200 import kernels as K
    from robo_b200.acquisition_functions import EI, InformationGainMC
    from robo_b200.initial_design import init_latin_hypercube_sampling
    from robo_b200.maximizers import DifferentialEvolution
    from robo_b200.models import GaussianProcess
    from robo_b200.priors import DefaultPrior
    from robo_b200.solver import BayesianOptimization
    rng = np.random.RandomState(1)
    np.random.seed(1)
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    gp = GaussianProcess(kernel, prior=DefaultPrior(len(kernel) + 1), rng=rng, normalize_output=False,
                         normalize_input=True, lower=LO, upper=UP)
    acq = InformationGainMC(gp, LO, UP, sampling_acquisition=EI, rng=rng, representer_sampler="device")
    de = DifferentialEvolution(acq, LO, UP, rng=rng, polish=False)
    bo = BayesianOptimization(_branin, LO, UP, acq, gp, de, initial_design=init_latin_hypercube_sampling,
                              initial_points=3, rng=rng)
    x_best, f_min = bo.run(10)
    X = np.array(bo.X)
    assert len(X) == 10 and np.all(X >= LO) and np.all(X <= UP)
    print("InformationGainMC BO on Branin: f_min", f_min)
    assert f_min < 20.0
