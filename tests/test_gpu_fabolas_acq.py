"""Information gain per unit cost on the device (gpk_predict_mean, gpk_es_cost_multi, gpk_maximize_random_es_cost and
InformationGainPerUnitCost / MarginalizationGPMCMC / DeviceRandomSampling over FabolasGP models).

Tolerances.  The mean-only prediction runs the int8 path's covariance builder and the same fixed-order sum of its tile
shares, so it must equal gpk_predict's mean bit for bit wherever gpk_predict takes the int8 path; elsewhere gpk_predict
sums the mean in another order (fp64 GEMM epilogue) and the two agree to rounding: 1e-10 of the mean's scale.  The fused
value of one pair is the entropy change of gpk_es_compute on the transformed batch divided by exp(mu) + overhead: with a
cost model whose mean is exactly 0 the division is by 1 and the values must be bit-identical; with a real cost model
the only difference to a numpy restatement is CUDA's exp against numpy's (each within 1 ulp) followed by one addition
and one division, so 1e-15 relative.  The marginalised value adds a sequential sum over the pairs in the order of
numpy's mean over axis 0: bit-identical to the device's per-estimator loop, and within 1e-14 of the numpy restatement
where the values are finite, measured against the mean of the terms' magnitudes (the sum may cancel).
"""
import numpy as np
import pytest

from tests import fabolas_acq_model as F

pytestmark = pytest.mark.gpu

LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
EXT_LO, EXT_UP = np.append(LO, 0.0), np.append(UP, 1.0)
IS_ENV = np.array([0, 0, 1])


def _objective_basis(s):
    return (1 - s) ** 2                                      # robo/fmin/fabolas.py:96-98


def _cost_basis(s):
    return s                                                 # robo/fmin/fabolas.py:100-102


def _kernel(amp=1.3, ls=(0.4, 0.6, 0.9)):
    from robo_b200 import kernels as K
    k = amp * K.Matern52Kernel(np.ones(1) * ls[0], ndim=3, axes=0)
    k *= K.Matern52Kernel(np.ones(1) * ls[1], ndim=3, axes=1)
    k *= K.Matern52Kernel(np.ones(1) * ls[2], ndim=3, axes=2)
    return k


def _oracle_kernel(amp, ls):
    from oracle import george_oracle as G
    k = amp * G.kernels.Matern52Kernel(np.ones(1) * ls[0], ndim=3, axes=0)
    k *= G.kernels.Matern52Kernel(np.ones(1) * ls[1], ndim=3, axes=1)
    k *= G.kernels.Matern52Kernel(np.ones(1) * ls[2], ndim=3, axes=2)
    return k


def _data(n, seed):
    rng = np.random.RandomState(seed)
    X = np.concatenate((LO + (UP - LO) * rng.rand(n, 2), rng.uniform(0.05, 1.0, (n, 1))), axis=1)
    y = np.sin(X[:, 0]) + 0.1 * X[:, 1] + X[:, 2]
    c = -1.5 + 3.0 * X[:, 2] + 0.05 * X[:, 0]                # log cost: below 0 (cost < 1) for small s
    return X, y, c


def _pair(n=60, seed=0, zero_cost=False, noise=1e-2):
    from robo_b200.models import FabolasGP
    X, y, c = _data(n, seed)
    obj = FabolasGP(_kernel(), basis_function=_objective_basis, noise=noise, lower=LO, upper=UP,
                    rng=np.random.RandomState(1))
    obj.train(X, y, do_optimize=False)
    cost = FabolasGP(_kernel(0.8, (0.5, 0.5, 0.7)), basis_function=_cost_basis, noise=noise, lower=LO, upper=UP,
                     rng=np.random.RandomState(2))
    cost.train(X, np.zeros_like(c) if zero_cost else c, do_optimize=False)
    return obj, cost, X


def _ig(obj, cost, seed=3, overhead=None):
    from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost
    ig = InformationGainPerUnitCost(obj, cost, EXT_LO, EXT_UP, IS_ENV, sampling_acquisition=EI, n_representer=50,
                                    rng=np.random.RandomState(seed))
    np.random.seed(seed)
    ig.update(obj, cost, overhead)
    return ig


def _candidates(X, m, seed=4):
    rng = np.random.RandomState(seed)
    C = EXT_LO + (EXT_UP - EXT_LO) * rng.rand(m, 3)
    C[:5] = X[:5]                                            # training inputs
    C[5] = EXT_UP + 0.5                                      # outside the raw box
    C[6] = EXT_LO - 0.25
    C[7, 2] = 1.5                                            # outside in the environment column only
    C[8, 2] = 0.0                                            # cheapest corner, cost below 1
    return C


def _inside(C):
    return np.all((C >= EXT_LO) & (C <= EXT_UP), axis=1)


# ---- gpk_predict_mean ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [2048, 4100])
def test_predict_mean_bit_identical_to_int8_predict(m):
    _, cost, X = _pair()
    h = cost.gp.handle
    C = cost.normalize(_candidates(X, m))
    n_oz = h.timings()["launches_ozaki"]
    for key, val in (("ozcluster", 4), ("ozcluster", 1), ("chunk", 2048), ("chunk", 0), ("ozpersist", 0),
                     ("ozpersist", 1), ("ozpersist", 3)):
        h.set_option(key, val)
        mu, _ = h.predict(C)
        assert h.timings()["launches_ozaki"] > n_oz          # gpk_predict took the int8 path
        n_oz = h.timings()["launches_ozaki"]
        assert np.array_equal(h.predict_mean(C), mu), (key, val)


@pytest.mark.parametrize("m,ozaki", [(1, 1), (300, 1), (2047, 1), (3000, 0)])
def test_predict_mean_close_to_fp64_predict(m, ozaki):
    _, cost, X = _pair()
    h = cost.gp.handle
    C = cost.normalize(_candidates(X, max(m, 10))[:m])
    h.set_option("ozaki", ozaki)
    mu, _ = h.predict(C)
    # the oracle's mean: mean + K(C, X) K^-1 (y - mean), with the oracle's george restatement of the kernel
    k = _oracle_kernel(0.8, (0.5, 0.5, 0.7))
    K = k.get_value(cost.X) + (cost.noise + 1.25e-12) * np.eye(len(cost.X))
    ref = cost.mean + k.get_value(C, cost.X) @ np.linalg.solve(K, cost.y - cost.mean)
    scale = max(1.0, np.max(np.abs(ref)))
    got = h.predict_mean(C)
    assert np.max(np.abs(got - ref)) <= 1e-10 * scale
    assert np.max(np.abs(got - mu)) <= 1e-10 * scale


# ---- one pair --------------------------------------------------------------------------------------------------
def test_single_pair_dh_bit_identical_with_zero_cost():
    obj, cost, X = _pair(zero_cost=True)
    assert np.all(cost.gp.handle.predict_mean(cost.normalize(X)) == 0.0)
    ig = _ig(obj, cost)
    C = _candidates(X, 3000)
    vals = ig.compute(C)
    dh = obj.gp.handle.es_compute(obj.normalize(C))
    inside = _inside(C)
    assert np.array_equal(vals[inside], dh[inside])
    assert np.all(vals[~inside] == np.spacing(1))
    assert (~inside).sum() == 3


@pytest.mark.parametrize("overhead", [None, 0.3])
def test_single_pair_matches_numpy_ratio(overhead):
    obj, cost, X = _pair()
    ig = _ig(obj, cost, overhead=overhead)
    C = _candidates(X, 2500)
    vals = ig.compute(C)
    dh = obj.gp.handle.es_compute(obj.normalize(C))
    dh[~_inside(C)] = np.spacing(1)                          # the raw bounds test
    mu = cost.gp.handle.predict_mean(cost.normalize(C))
    ref = F.per_unit_cost(dh, mu, 0.0 if overhead is None else overhead)
    assert np.any(np.exp(mu) < 1.0)
    ok = np.isfinite(ref)
    assert np.all(np.abs(vals[ok] - ref[ok]) <= 1e-15 * np.abs(ref[ok]))
    assert np.array_equal(np.isfinite(vals), ok)
    assert ig.argmax(C) == int(np.argmax(vals))


# ---- the reference's own values ------------------------------------------------------------------------------
def test_golden_reference_values():
    """tests/golden/fabolas_ig.npz (tools/make_fabolas_ig_golden.py): the reference's InformationGainPerUnitCost over
    the reference's FabolasGP models.  Its representer points and their log-probabilities are injected, so the device
    path runs EP, U and the entropy change on the same zb.  Bound: the one test_gpu_es.py's
    test_compute_matches_model_on_device_moments uses and justifies for the entropy change, 1e-7 S with
    S = |H| + max |lmb| + 1, away from v = sn2 and from the training inputs, divided by the candidate's cost; plus 1e-12
    relative for the cost itself (the mean through the device and through the oracle differ by rounding)."""
    from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost
    from robo_b200.models import FabolasGP
    from tests.conftest import GOLDEN
    G = np.load(GOLDEN + "/fabolas_ig.npz")
    lo, up = G["lower"], G["upper"]
    elo, eup = G["extend_lower"], G["extend_upper"]
    noise = float(G["noise"])
    obj = FabolasGP(_kernel(float(G["obj_amp"]), tuple(G["obj_ls"])), basis_function=_objective_basis, noise=noise,
                    lower=lo, upper=up, rng=np.random.RandomState(0))
    obj.train(G["X"], G["y"], do_optimize=False)
    cost = FabolasGP(_kernel(float(G["cost_amp"]), tuple(G["cost_ls"])), basis_function=_cost_basis, noise=noise,
                     lower=lo, upper=up, rng=np.random.RandomState(1))
    cost.train(G["X"], G["c"], do_optimize=False)
    zb, lmb = G["zb"], G["lmb"]
    ig = InformationGainPerUnitCost(obj, cost, elo, eup, G["is_env"], sampling_acquisition=EI, n_representer=len(zb),
                                    rng=np.random.RandomState(0))

    def injected():
        ig.zb, ig.lmb = zb.copy(), lmb.copy()
    ig.sample_representer_points = injected
    ig.update(obj, cost, overhead=float(G["overhead"]))
    assert ig.Np == int(G["Np"])
    Xt, ref, log_cost = G["Xt"], G["values"], G["log_cost"]
    vals = ig.compute(Xt)
    mu = cost.gp.handle.predict_mean(cost.normalize(Xt))
    np.testing.assert_allclose(mu, log_cost, rtol=1e-10, atol=1e-12)
    c = np.exp(log_cost) + float(G["overhead"])
    lp, lm = ig.logP.ravel(), ig.lmb.ravel()
    S = abs(np.sum(np.exp(lp) * (lp + lm))) + np.max(np.abs(lm)) + 1.0
    _, v = obj.predict(Xt)
    inside = np.all((Xt >= elo) & (Xt <= eup), axis=1)
    assert (~inside).sum() == 10
    assert np.all(np.abs(vals[~inside] - ref[~inside]) <= 1e-12 * np.abs(ref[~inside]))
    n_checked = 0
    for i in np.where(inside)[0]:
        near_train = np.min(np.max(np.abs(G["X"] - Xt[i]) / (eup - elo), axis=1)) < 1e-2
        if abs(v[i] - noise) >= 1e-3 * v[i] and not near_train:
            assert abs(vals[i] - ref[i]) <= 1e-7 * S / c[i] + 1e-12 * abs(ref[i]), (i, vals[i], ref[i], S, c[i])
            n_checked += 1
    assert n_checked >= 120
    assert np.any(np.exp(log_cost[inside]) < 1.0)


# ---- determinism -----------------------------------------------------------------------------------------------
def test_deterministic_across_chunk_streams_and_dev():
    import torch
    from robo_b200 import _lib
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import device_spec
    obj, cost, X = _pair()
    ig = _ig(obj, cost, overhead=0.1)
    C = _candidates(X, 5000)
    base = ig.compute(C)
    for h in (obj.gp.handle, cost.gp.handle):
        for key, val in (("chunk", 2048), ("ozcluster", 1), ("chunk", 0), ("ozcluster", 4)):
            h.set_option(key, val)
            assert np.array_equal(ig.compute(C), base), (key, val)
    ho, hc, lo, up, bo, bc, oh = device_spec([ig])
    dX = torch.tensor(C, dtype=torch.float64, device="cuda")
    dout = torch.empty(len(C), dtype=torch.float64, device="cuda")
    dbest = torch.empty(2, dtype=torch.float64, device="cuda")
    _lib.es_cost_multi_dev(ho, hc, dX.data_ptr(), len(C), lo, up, bo, bc, oh, dout.data_ptr(), dbest.data_ptr())
    ho[0].synchronize()
    assert np.array_equal(dout.cpu().numpy(), base)
    assert int(dbest.cpu().numpy().view(np.int64)[1]) == int(np.argmax(base))
    for _ in range(3):
        assert np.array_equal(ig.compute(C), base)


# ---- marginalised over FabolasGPMCMC pairs ---------------------------------------------------------------------
class _Prior(object):
    def __init__(self, r):
        self.r = r

    def lnprob(self, t):
        return 0.0 if np.all(np.abs(t) < 6) else -np.inf

    def sample_from_prior(self, n):
        return self.r.uniform(-2, 1, size=(n, 5))


def _mcmc_pair(n_hypers, n, seed=0):
    from robo_b200.models import FabolasGPMCMC
    X, y, c = _data(n, seed)
    objm = FabolasGPMCMC(_kernel(), basis_func=_objective_basis, prior=_Prior(np.random.RandomState(1)),
                         n_hypers=n_hypers, chain_length=4, burnin_steps=3, lower=LO, upper=UP,
                         rng=np.random.RandomState(2))
    objm.train(X, y, do_optimize=True)
    costm = FabolasGPMCMC(_kernel(0.8, (0.5, 0.5, 0.7)), basis_func=_cost_basis, prior=_Prior(np.random.RandomState(3)),
                          n_hypers=n_hypers, chain_length=4, burnin_steps=3, lower=LO, upper=UP,
                          rng=np.random.RandomState(4))
    costm.train(X, c, do_optimize=True)
    return objm, costm, X


def test_marginalised_equals_per_estimator_loop():
    from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost, MarginalizationGPMCMC
    objm, costm, X = _mcmc_pair(12, 60)
    assert len(objm.models) == 12 and len(costm.models) == 12
    acq = MarginalizationGPMCMC(InformationGainPerUnitCost(objm, costm, EXT_LO, EXT_UP, IS_ENV, sampling_acquisition=EI,
                                                           rng=np.random.RandomState(0)))
    np.random.seed(0)
    acq.update(objm, costm, overhead=0.05)
    assert acq._es_cost_spec() is not None
    C = _candidates(X, 2200)
    vals = acq.compute(C)
    per = np.array([e.compute(C) for e in acq.estimators])
    assert all(e.model is m and e.cost_model is c for e, m, c in zip(acq.estimators, objm.models, costm.models))
    assert np.array_equal(vals, per.mean(axis=0))
    # the reference's loop in numpy: estimator i = objective sub-model i over cost sub-model i
    ref = []
    for e in acq.estimators:
        dh = e.model.gp.handle.es_compute(e.model.normalize(C))
        dh[~_inside(C)] = np.spacing(1)
        ref.append(F.per_unit_cost(dh, e.cost_model.gp.handle.predict_mean(e.cost_model.normalize(C)), 0.05))
    ref = np.array(ref)
    size = np.mean(np.abs(ref), axis=0)                      # the sum may cancel: bound against its terms
    ref = np.mean(ref, axis=0)
    ok = np.isfinite(ref)
    assert ok.sum() > 2000
    assert np.all(np.abs(vals[ok] - ref[ok]) <= 1e-14 * size[ok])
    assert acq.argmax(C) == int(np.argmax(vals))


def test_device_random_sampling_winner():
    from robo_b200.maximizers.device_random_sampling import DeviceRandomSampling
    obj, cost, X = _pair()
    ig = _ig(obj, cost, overhead=0.2)
    mx = DeviceRandomSampling(ig, EXT_LO, EXT_UP, n_samples=3000, rng=np.random.RandomState(5))
    x = mx.maximize()
    n_uniform = int(3000 * .7)
    n_total = n_uniform + int(3000 * .3)
    inc = obj.get_incumbent()[0]
    cands = obj.gp.handle.generate_candidates(mx.last["seed"], 0, n_total, n_uniform, EXT_LO, EXT_UP, inc, 0.1)
    vals = ig.compute(cands)
    idx = int(np.argmax(vals))
    assert mx.last["best_idx"] == idx
    assert np.array_equal(x, cands[idx]) and mx.last["best_val"] == vals[idx]


def test_c4_shape_update_and_maximize():
    """BASELINE config 4: N = 2048, two configuration columns and the environment, 20 + 20 sub-models."""
    from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost, MarginalizationGPMCMC
    from robo_b200.maximizers.device_random_sampling import DeviceRandomSampling
    objm, costm, X = _mcmc_pair(20, 2048)
    acq = MarginalizationGPMCMC(InformationGainPerUnitCost(objm, costm, EXT_LO, EXT_UP, IS_ENV, sampling_acquisition=EI,
                                                           rng=np.random.RandomState(0)))
    np.random.seed(1)
    acq.update(objm, costm)
    x = DeviceRandomSampling(acq, EXT_LO, EXT_UP, n_samples=500, rng=np.random.RandomState(2)).maximize()
    assert x.shape == (3,) and np.all(np.isfinite(x))
    assert np.all(x >= EXT_LO) and np.all(x <= EXT_UP)


# ---- argument validation ---------------------------------------------------------------------------------------
def test_argument_validation():
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import InformationGain
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import device_spec
    obj, cost, X = _pair()
    ho, hc = [obj.gp.handle], [cost.gp.handle]
    C = _candidates(X, 20)
    with pytest.raises(ValueError):                          # objective without gpk_es_update
        _lib.es_cost_multi(ho, hc, C, LO, UP, 1, 0, 0.0)
    ig = _ig(obj, cost)
    ho, hc, lo, up, bo, bc, oh = device_spec([ig])
    assert (bo, bc) == (_lib.BASIS_ONE_MINUS_S_SQ, _lib.BASIS_S)
    _lib.es_cost_multi(ho, hc, C, lo, up, bo, bc, oh)
    for bad in (dict(b=(2, 0)), dict(b=(0, -1))):
        with pytest.raises(ValueError):
            _lib.es_cost_multi(ho, hc, C, lo, up, bad["b"][0], bad["b"][1], oh)
    with pytest.raises(ValueError):                          # m = 0
        _lib.es_cost_multi(ho, hc, np.zeros((0, 3)), lo, up, bo, bc, oh)
    with pytest.raises(ValueError):                          # the objective handle as its own cost handle
        _lib.es_cost_multi(ho, ho, C, lo, up, bo, bc, oh)
    with pytest.raises(ValueError):                          # counts differ
        _lib.es_cost_multi(ho, hc + hc, C, lo, up, bo, bc, oh)
    with pytest.raises(ValueError):                          # configuration bounds of the wrong length
        _lib.es_cost_multi(ho, hc, C, lo[:1], up[:1], bo, bc, oh)
    with pytest.raises(ValueError):
        _lib.maximize_random_es_cost(ho, hc, 1, 100, 70, EXT_LO, EXT_UP, C[0], 0.1, lo, up[:1], bo, bc, oh)
    with pytest.raises(ValueError):                          # lower >= upper
        _lib.es_cost_multi(ho, hc, C, up, lo, bo, bc, oh)
    with pytest.raises(ValueError):                          # the model changed since gpk_es_update
        obj.train(X, np.cos(X[:, 0]), do_optimize=False)
        _lib.es_cost_multi([obj.gp.handle], hc, C, lo, up, bo, bc, oh)
    with pytest.raises(TypeError):                           # InformationGain keeps refusing FabolasGP
        InformationGain(obj, EXT_LO, EXT_UP, rng=np.random.RandomState(0)).update(obj)
    cost.basis_function = lambda s: 1 - s                    # no device kernel for this basis
    with pytest.raises(TypeError):
        device_spec([ig])


def test_meanonly_option_routes_through_scoring_pass():
    _, cost, X = _pair()
    h = cost.gp.handle
    C = cost.normalize(_candidates(X, 700))
    mu, _ = h.predict(C)
    fast = h.predict_mean(C)
    h.set_option("meanonly", 0)
    assert np.array_equal(h.predict_mean(C), mu)               # the mean of the full scoring pass itself
    h.set_option("meanonly", 1)
    assert np.array_equal(h.predict_mean(C), fast)
    with pytest.raises(ValueError):
        h.set_option("meanonly", 2)
