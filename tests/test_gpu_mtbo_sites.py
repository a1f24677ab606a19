"""The task factor at the sites built on the entropy-search kernel value: gpk_es_update / gpk_es_moments /
gpk_es_compute against numpy (U, sigma, the variance) and the dH restatement tests/es_model.py fed the device's own
moments, with task coordinates that are tasks and ones that are not; information gain per unit cost over MTBOGP models
against the reference's own values (tests/golden/mtbo_ig.npz); gpk_es_cost_multi with the BASIS_TASK input map over
MTBOGPMCMC models, bit-identical to the per-estimator loop; every maximizer over MTBO's marginalised
InformationGainPerUnitCost; the device representer sampler with the rint map; and ``mtbo()`` end to end with host and
with device samplers.

Tolerances as in tests/test_gpu_fabolas_sites.py and tests/test_gpu_fabolas_acq.py: U, sigma and the variance 1e-8
relative to the largest entry; dH against es_model on the device's own moments 1e-9 of |H| + max |lmb| + 1; against the
reference's values 1e-7 of that scale divided by the candidate's cost, away from v = sn2 and the training inputs."""
import numpy as np
import pytest
import scipy.linalg as spla

from tests import es_model as M
from tests import task_kernel_model as T

pytestmark = pytest.mark.gpu

EPS = np.finfo(float).eps

LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
N_TASKS = 3
EXT_LO, EXT_UP = np.append(LO, 0.0), np.append(UP, N_TASKS - 1.0)
IS_ENV = np.array([0, 0, 1])


def test_es_update_and_compute_with_the_task_factor():
    from robo_b200 import _lib
    rng = np.random.RandomState(11)
    n, nb, Np, diag, sn2, nT = 150, 20, 30, 1e-2, 1e-3, 3
    th = rng.uniform(-1.0, 0.3, T.n_kt(nT))
    X = np.column_stack([rng.rand(n, 2), rng.randint(0, nT, n)])
    y = np.sin(3 * X[:, 0]) + 0.4 * X[:, 2] + 0.05 * rng.randn(n)
    lo, up = np.array([0.0, 0.0, 0.0]), np.array([1.0, 1.0, nT - 1.0])
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(_lib.MATERN52, 0.2, [0, 1], [0, 1], [-1.0, -0.5])
    h.set_task_factor(2, nT, th)
    h.fit(diag, 0.0)
    zb = np.column_stack([rng.rand(nb, 2), rng.randint(0, nT, nb)])
    lmb = np.log(0.05 + rng.rand(nb))
    W = rng.randn(Np)
    r = h.es_update(zb, lmb, sn2, W, lo, up)
    k = T.mtbo_kernel(2, 0.2, (-1.0, -0.5), th, nT)
    K = k.get_value(X) + diag * np.eye(n)
    L = spla.cholesky(K, lower=True)
    U_ref = spla.cho_solve((L, True), k.get_value(X, zb))
    U = h.es_get_u()
    assert np.max(np.abs(U - U_ref)) <= 1e-8 * np.max(np.abs(U_ref))
    Xs = np.column_stack([rng.rand(300, 2), rng.randint(0, nT, 300).astype(float)])
    Xs[:3] = X[:3]                                               # training inputs: sigma cancels and clips
    Xs[3:5] = zb[:2]                                             # the representer points themselves
    Xs[5] = up + 0.5                                             # outside the box, and not a task
    Xs[6:10, 2] = [0.5, 1.5, -1.0, np.nan]                       # not tasks: NaN moments, -DBL_MAX entropy change
    task = T.task_index(Xs[:, 2], nT) >= 0
    xv = Xs[task]
    Ks = k.get_value(xv, X)
    var_ref = np.diag(k.get_value(xv)) - np.einsum("ij,ij->i", Ks, spla.cho_solve((L, True), Ks.T).T)
    sig_ref = np.clip(k.get_value(xv, zb) - Ks @ U_ref, EPS, np.inf)
    var, sig = h.es_moments(Xs)
    assert np.max(np.abs(var[task] - np.clip(var_ref, EPS, np.inf))) <= 1e-8 * np.max(np.abs(var_ref))
    assert np.max(np.abs(sig[task] - sig_ref)) <= 1e-8 * np.max(np.abs(sig_ref))
    assert np.all(np.isnan(var[~task])) and np.all(np.isnan(sig[~task]))
    state = dict(logP=r["logP"], lmb=lmb, dlogPdMu=r["dlogPdMu"], dlogPdSigma=r["dlogPdSigma"],
                 dlogPdMudMu=r["dlogPdMudMu"], W=W, sn2=sn2)
    state["H"] = -float(np.sum(np.exp(r["logP"]) * (r["logP"] + lmb)))
    dh = h.es_compute(Xs)
    S = abs(state["H"]) + np.max(np.abs(lmb)) + 1.0
    inside = np.all((Xs >= lo) & (Xs <= up), axis=1)
    assert dh[5] == EPS
    assert np.all(dh[~task & inside] == -np.finfo(float).max)
    n_checked = 0
    for i in np.where(task)[0]:
        ref = M.compute_value(M.dh_folded(state, var[i], sig[i]), Xs[i], lo, up)
        if not np.isfinite(ref) or not np.isfinite(dh[i]) or ref == EPS:
            assert dh[i] == ref or (np.isnan(dh[i]) and np.isnan(ref)), (i, dh[i], ref)
            continue
        assert abs(dh[i] - ref) <= 1e-9 * S, (i, dh[i], ref)
        n_checked += 1
    assert n_checked > 250
    h.close()


def test_golden_reference_values():
    """tests/golden/mtbo_ig.npz (tools/make_mtbo_golden.py): the reference's InformationGainPerUnitCost over the
    reference's MTBOGP models (with the restated task kernel).  Its representer points and their log-probabilities are
    injected, so the device runs EP, U and the entropy change on the same zb; the candidates include rint ties at 0.5
    and 1.5 and points outside the extended box."""
    from robo_b200 import kernels
    from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost
    from robo_b200.models import MTBOGP
    from tests.conftest import GOLDEN
    G = np.load(GOLDEN + "/mtbo_ig.npz")
    lo, up, elo, eup = G["lower"], G["upper"], G["extend_lower"], G["extend_upper"]
    noise = float(G["noise"])

    def kernel(amp, ls, theta):
        k = float(amp) * kernels.Matern52Kernel(np.ones(1) * ls[0], ndim=3, axes=0)
        k *= kernels.Matern52Kernel(np.ones(1) * ls[1], ndim=3, axes=1)
        task = kernels.TaskKernel(3, 2, int(G["n_tasks"]))
        task.set_parameter_vector(theta)
        return k * task
    obj = MTBOGP(kernel(G["obj_amp"], G["obj_ls"], G["obj_theta"]), noise=noise, lower=lo, upper=up,
                 rng=np.random.RandomState(0))
    obj.train(G["X"], G["y"], do_optimize=False)
    cost = MTBOGP(kernel(G["cost_amp"], G["cost_ls"], G["cost_theta"]), noise=noise, lower=lo, upper=up,
                  rng=np.random.RandomState(1))
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
    ties = np.isin(Xt[:, 2], [0.5, 1.5])
    assert ties.sum() == 4
    n_checked = n_ties = 0
    for i in np.where(inside)[0]:
        near_train = np.min(np.max(np.abs(G["X"] - Xt[i]) / (eup - elo), axis=1)) < 1e-2
        if abs(v[i] - noise) >= 1e-3 * v[i] and not near_train:
            assert abs(vals[i] - ref[i]) <= 1e-7 * S / c[i] + 1e-12 * abs(ref[i]), (i, vals[i], ref[i], S, c[i])
            n_checked += 1
            n_ties += int(ties[i])
    assert n_checked >= 100 and n_ties == 4


def _mcmc_pair(n_hypers, n, seed=0, hyper_sampler="host"):
    from robo_b200.fmin.mtbo import _mtbo_kernel
    from robo_b200.models import MTBOGPMCMC
    from robo_b200.priors import MTBOPrior
    rng = np.random.RandomState(seed)
    X = np.concatenate((LO + (UP - LO) * rng.rand(n, 2), rng.randint(0, N_TASKS, (n, 1))), axis=1)
    y = np.sin(X[:, 0]) + 0.1 * X[:, 1] + 0.5 * X[:, 2]
    c = -1.5 + 1.0 * X[:, 2] + 0.05 * X[:, 0]
    out = []
    for i, t in enumerate((y, c)):
        k, task = _mtbo_kernel(2, N_TASKS)
        m = MTBOGPMCMC(k, prior=MTBOPrior(len(k) + 1, 2, len(task), rng=np.random.RandomState(1 + i)),
                       n_hypers=n_hypers, chain_length=4, burnin_steps=3, lower=LO, upper=UP,
                       rng=np.random.RandomState(2 + i), hyper_sampler=hyper_sampler)
        m.train(X, t, do_optimize=True)
        out.append(m)
    return out[0], out[1], X


def _acq(objm, costm, representer_sampler="host"):
    from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost, MarginalizationGPMCMC
    acq = MarginalizationGPMCMC(InformationGainPerUnitCost(objm, costm, EXT_LO, EXT_UP, IS_ENV, sampling_acquisition=EI,
                                                           rng=np.random.RandomState(0),
                                                           representer_sampler=representer_sampler))
    np.random.seed(0)
    acq.update(objm, costm, overhead=0.05)
    return acq


def test_es_cost_multi_with_the_task_map_equals_per_estimator_loop():
    from robo_b200 import _lib
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import device_spec
    objm, costm, X = _mcmc_pair(20, 60)
    assert objm.models[0].gp.kernel.flatten()["task"] is not None
    acq = _acq(objm, costm)
    assert device_spec(acq.estimators)[4:6] == (_lib.BASIS_TASK, _lib.BASIS_TASK)
    rng = np.random.RandomState(4)
    C = EXT_LO + (EXT_UP - EXT_LO) * rng.rand(2200, 3)
    C[:8, 2] = [0.5, 1.5, 0.49, 1.51, 2.0, 0.0, 1.0, 1.5]  # rint ties round half to even
    vals = acq.compute(C)
    per = np.array([e.compute(C) for e in acq.estimators])
    assert np.array_equal(vals, per.mean(axis=0))
    assert np.all(np.isfinite(vals))
    assert acq.argmax(C) == int(np.argmax(vals))
    # the device map equals the host one: rows with the same rint task score the same
    D = C[:8].copy()
    D[:, 2] = np.rint(D[:, 2])
    assert np.array_equal(acq.compute(C[:8]), acq.compute(D))
    # the candidate sizes of the benchmark: a full 65,536-row pass
    big = EXT_LO + (EXT_UP - EXT_LO) * rng.rand(65536, 3)
    assert np.all(np.isfinite(acq.compute(big)))


@pytest.mark.parametrize("name", ["RandomSampling", "DeviceRandomSampling", "DifferentialEvolution", "SciPyOptimizer",
                                  "CMAES", "Direct"])
def test_every_maximizer_completes(name):
    from robo_b200 import maximizers
    objm, costm, _ = _mcmc_pair(20, 40)
    acq = _acq(objm, costm)
    kw = dict(rng=np.random.RandomState(5))
    if name in ("CMAES", "Direct"):
        kw["verbose"] = False
    x = getattr(maximizers, name)(acq, EXT_LO, EXT_UP, **kw).maximize()
    x = np.asarray(x).ravel()
    assert x.shape == (3,) and np.all(np.isfinite(x)) and np.all(x >= EXT_LO) and np.all(x <= EXT_UP)


def test_device_representer_sampler_with_the_task_map():
    objm, costm, _ = _mcmc_pair(20, 40, hyper_sampler="device")
    acq = _acq(objm, costm, representer_sampler="device")
    for e in acq.estimators:
        assert e.zb.shape == (50, 3) and np.all(np.isfinite(e.zb)) and np.all(np.isfinite(e.lmb))
        assert np.all(e.zb[:, 2] == 1.0)                  # the reference's projection: the number of task columns
        assert np.all(e.zb[:, :2] >= LO) and np.all(e.zb[:, :2] <= UP)
    C = EXT_LO + (EXT_UP - EXT_LO) * np.random.RandomState(6).rand(500, 3)
    assert np.all(np.isfinite(acq.compute(C)))


def _objective(x, task):
    return float(np.sum((x - 0.3) ** 2) + 0.2 * (1 - task) + 0.01), float(1.0 + 2.0 * task)


@pytest.mark.parametrize("samplers", ["host", "device"])
def test_mtbo_end_to_end(samplers):
    from robo_b200.fmin import mtbo
    lower, upper = np.zeros(2), np.ones(2)
    kw = dict(n_tasks=2, n_init=3, num_iterations=6, burnin=20, chain_length=20,
              hyper_sampler=samplers, representer_sampler=samplers)
    np.random.seed(7)
    r1 = mtbo(_objective, lower, upper, rng=np.random.RandomState(1), **kw)
    x = np.array(r1["x_opt"])
    assert x.shape == (2,) and np.all(x >= lower) and np.all(x <= upper)
    assert r1["X"].shape == (6, 3) and np.all(np.isin(r1["X"][:, 2], [0.0, 1.0]))
    np.random.seed(7)
    r2 = mtbo(_objective, lower, upper, rng=np.random.RandomState(1), **kw)
    assert np.array_equal(r1["X"], r2["X"])
