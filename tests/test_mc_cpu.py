"""The sampling-based entropy search without a GPU: the kernels' numpy restatement (tests/mc_model.py) against the
reference's own joint_pmin on the same draws (tests/golden/mc_pmin.npz, tools/make_mc_golden.py), the jitter ladder,
and the host logic of InformationGainMC / joint_pmin over the oracle-backed fake: which device path each maximizer and
MarginalizationGPMCMC take, the representer sampler's steps and runs, and the argument errors."""
import os

import numpy as np
import pytest

from tests import fabolas_acq_model as FM
from tests import mc_model as M

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mc_pmin.npz")
LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])


# ---- the restatement against the reference ----------------------------------------------------------------------
def _golden():
    g = np.load(GOLDEN)
    return [(str(n), g[n + "/m"], g[n + "/V"], g[n + "/F"], g[n + "/pmin"]) for n in g["names"]]


@pytest.mark.parametrize("case", range(9))
def test_restatement_reproduces_reference_pmin(case):
    name, m, V, F, pmin = _golden()[case]
    r = M.joint_pmin(m, V, F.T)                             # the reference draws F as Nf x Nb
    total = F.shape[0] * m.shape[1]
    ref_counts = np.rint(np.where(pmin > 1e-70, pmin, 0.0) * total).astype(np.int64)
    assert ref_counts.sum() == total
    # numpy's LAPACK factor and BLAS product round differently from the kernel's stated order: counts may move only
    # between the two candidates of a column the model flags as a near tie
    assert np.abs(r["counts"] - ref_counts).sum() <= 2 * r["near"], (name, r["near"])
    if r["near"] == 0:
        assert np.array_equal(r["pmin"], pmin), name
    if name == "ties_clamp":
        assert r["pmin"].tolist() == [1e-70, 1.0, 1e-70, 1e-70] and pmin.tolist() == r["pmin"].tolist()
    if name in ("singular", "rank_one"):
        assert r["rung"] > 0
    else:
        assert r["rung"] == 0


def test_jitter_ladder():
    lad = M.ladder()
    assert lad[0] == 0.0 and lad[1] == 1e-9 and lad[-1] == 10000.0 and len(lad) == 15
    x = 1e-10
    for r in range(1, 15):
        x = x * 10.0
        assert lad[r] == x                                  # float for float the reference's noise *= 10
    L, rung = M.factorise(np.ones((3, 3)))
    assert rung == 1
    L, rung = M.factorise(-5000.0 * np.eye(2))              # PD only at the last rung, 10000
    assert rung == 14
    with pytest.raises(np.linalg.LinAlgError):
        M.factorise(-1e5 * np.eye(2))


def test_restated_draws_are_standard_normal():
    F = M.draws(11, 16, 5001)
    assert F.shape == (16, 5001)
    assert abs(F.mean()) < 5 / np.sqrt(F.size) and abs(F.var() - 1.0) < 5 * np.sqrt(2.0 / F.size)
    assert np.array_equal(M.draws(11, 3, 7), F[:3, :7])


# ---- the host logic over the fake ------------------------------------------------------------------------------
def _esmc_update(self, zb, lmb, sn2, W, nf, seed):
    lmb = np.ravel(lmb)
    if not np.all(np.isfinite(lmb)):
        raise ValueError("lmb should not be infinite.")
    Mb, Vb = self.predict_cov(zb)
    r = M.joint_pmin(Mb, Vb, M.draws(seed, len(Mb), nf))
    self.mc_state = (self.L, seed)
    return dict(logP=np.log(r["pmin"]), pmin=r["pmin"], n_jitter=int(r["rung"] > 0))


def _esmc_compute(self, Xs):
    state = getattr(self, "mc_state", None)
    if state is None or state[0] is not self.L:
        raise ValueError("gpk_esmc_compute: call gpk_esmc_update first")
    return self.predict(np.asarray(Xs, dtype=np.float64))[1]        # a stand-in value: the predictive variance


def _mc_pmin(self, m, V, nf, seed):
    r = M.joint_pmin(m, V, M.draws(seed, np.shape(m)[0], nf))
    return r["pmin"], int(r["rung"] > 0)


@pytest.fixture
def fake(monkeypatch):
    from robo_b200 import _lib
    from tests import fake_de_es
    cls = fake_de_es.install(monkeypatch)
    for name, fn in (("esmc_update", _esmc_update), ("esmc_compute", _esmc_compute), ("mc_pmin", _mc_pmin)):
        monkeypatch.setattr(cls, name, fn, raising=False)
    calls = []

    def esmc_multi(objective, Xs, want_values=True):
        calls.append("esmc_multi")
        fake_de_es._distinct(objective)
        vals = np.mean([h.esmc_compute(Xs) for h in objective], axis=0)
        return dict(values=vals if want_values else None, best_val=float(np.max(vals)), best_idx=int(np.argmax(vals)))

    def maximize_de_esmc(objective, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper,
                         want_population=False):
        calls.append("maximize_de_esmc")
        fn = objective[0].esmc_compute if len(objective) == 1 else (lambda X: esmc_multi(objective, X)["values"])
        return fake_de_es._evolve(fn, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper,
                                  want_population)

    def es_multi(objective, Xs, want_values=True):
        calls.append("es_multi")
        return fake_de_es.es_multi(objective, Xs, want_values)

    def sample_representers(models, seeds, nb, steps, max_runs, kind, eta, par, lower, upper, fabolas=None):
        calls.append(("sample_representers", len(models), steps, max_runs))
        rng = np.random.RandomState(int(seeds[0]) % 1000)
        n, dw = len(models), np.size(lower)
        zb = np.asarray(lower) + (np.asarray(upper) - np.asarray(lower)) * rng.rand(n, nb, dw)
        return dict(zb=zb, lmb=np.zeros((n, nb)), runs=np.ones(n, np.int32), n_accepted=np.zeros((n, nb)), n_negative=0)

    for name, fn in (("esmc_multi", esmc_multi), ("maximize_de_esmc", maximize_de_esmc), ("es_multi", es_multi),
                     ("sample_representers", sample_representers)):
        monkeypatch.setattr(_lib, name, fn)
    return calls


def _gp(seed=0):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    rng = np.random.RandomState(seed)
    X = LO + (UP - LO) * rng.rand(10, 2)
    y = np.sin(X[:, 0]) + X[:, 1] * 0.1
    gp = GaussianProcess(2 * K.Matern52Kernel(np.ones(2), ndim=2), normalize_input=True, lower=LO, upper=UP,
                         rng=np.random.RandomState(1))
    gp.train(X, y, do_optimize=False)
    return gp


def _mcmc():
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    rng = np.random.RandomState(0)
    X = LO + (UP - LO) * rng.rand(10, 2)
    y = np.sin(X[:, 0]) + X[:, 1] * 0.1
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)), n_hypers=8,
                                chain_length=5, burnin_steps=5, normalize_input=True, lower=LO, upper=UP,
                                rng=np.random.RandomState(2))
    model.train(X, y, do_optimize=True)
    return model


def _mc(model, sampler="device", **kw):
    from robo_b200.acquisition_functions import EI, InformationGainMC
    return InformationGainMC(model, LO, UP, Nb=8, Np=5, Nf=40, sampling_acquisition=EI,
                             rng=np.random.RandomState(3), representer_sampler=sampler, **kw)


def test_device_spec_recognises_mc_before_information_gain(fake):
    from robo_b200.acquisition_functions import InformationGain, MarginalizationGPMCMC
    from robo_b200.maximizers.device_spec import device_spec, is_sampling_based
    gp = _gp()
    mc = _mc(gp)
    mc.update(gp)
    which, spec = device_spec(mc, "test")
    assert which == "esmc" and len(spec) == 1
    ig = InformationGain(gp, LO, UP, Nb=8, sampling_acquisition=FM.ConstantSampling, rng=np.random.RandomState(3))
    ig.update(gp)
    assert device_spec(ig, "test")[0] == "es" and not is_sampling_based(ig) and is_sampling_based(mc)
    model = _mcmc()
    acq = MarginalizationGPMCMC(_mc(model))
    acq.update(model)
    assert device_spec(acq, "test")[0] == "esmc" and is_sampling_based(acq)


def test_marginalization_routes_mc_through_esmc_multi(fake):
    from robo_b200.acquisition_functions import MarginalizationGPMCMC
    model = _mcmc()
    acq = MarginalizationGPMCMC(_mc(model))
    acq.update(model)
    # every estimator's representer points in ONE sampler call, with the reference's 200 steps and one run
    assert [c for c in fake if c[0] == "sample_representers"] == [("sample_representers", 8, 200, 1)]
    assert len(set(e.seed for e in acq.estimators)) == 8
    C = LO + (UP - LO) * np.random.RandomState(1).rand(20, 2)
    v = acq.compute(C)
    assert fake[-1] == "esmc_multi" and "es_multi" not in fake
    loop = np.mean([e.compute(C) for e in acq.estimators], axis=0)
    np.testing.assert_allclose(v, loop, rtol=1e-15)
    assert acq.argmax(C) == int(np.argmax(loop)) and fake[-1] == "esmc_multi"


def test_sampler_steps_and_runs_per_estimator(fake):
    from robo_b200.acquisition_functions import EI, InformationGain
    from robo_b200.acquisition_functions.information_gain import sample_representers_device
    gp = _gp()
    ig = InformationGain(gp, LO, UP, Nb=8, sampling_acquisition=EI, rng=np.random.RandomState(3),
                         representer_sampler="device")
    mc = _mc(gp)
    for e in (ig, mc):
        e._begin_update(gp)
    sample_representers_device([ig, mc])
    assert sorted(c[2:] for c in fake if c[0] == "sample_representers") == [(50, 5), (200, 1)]
    assert (InformationGain.REPRESENTER_STEPS, InformationGain.REPRESENTER_RUNS) == (50, 5)


def test_host_sampler_runs_200_steps(fake, monkeypatch):
    from robo_b200.util import ensemble_sampler
    seen = []
    run = ensemble_sampler.EnsembleSampler.run_mcmc

    def spy(self, p0, N, **kw):
        seen.append((np.shape(p0), N))
        return run(self, p0, N, **kw)
    monkeypatch.setattr(ensemble_sampler.EnsembleSampler, "run_mcmc", spy)
    gp = _gp()
    mc = _mc(gp, sampler="host")
    mc.update(gp)
    assert seen == [((8, 2), 200)]
    assert mc.zb.shape == (8, 2) and mc.lmb.shape == (8, 1) and mc.pmin.shape == (8,)
    assert np.all(mc.zb >= LO) and np.all(mc.zb <= UP)


def test_maximizers_take_their_paths(fake, monkeypatch):
    from robo_b200.acquisition_functions import MarginalizationGPMCMC
    from robo_b200.maximizers import DifferentialEvolution, RandomSampling, SciPyOptimizer
    from robo_b200.maximizers import device_spec as DS
    model = _mcmc()
    acq = MarginalizationGPMCMC(_mc(model))
    acq.update(model)
    de = DifferentialEvolution(acq, LO, UP, n_iters=3, rng=np.random.RandomState(1), polish=False)
    x = de.maximize()
    assert "maximize_de_esmc" in fake and np.all(x >= LO) and np.all(x <= UP)
    de_host = DifferentialEvolution(acq, LO, UP, n_iters=3, rng=np.random.RandomState(1), polish=True)
    de_host.maximize()
    with pytest.raises(ValueError, match="polish='device'"):
        DifferentialEvolution(acq, LO, UP, n_iters=3, rng=np.random.RandomState(1), polish="device").maximize()
    np.random.seed(0)
    RandomSampling(acq, LO, UP, n_samples=50, rng=np.random.RandomState(0)).maximize()
    assert fake[-1] == "esmc_multi"
    with pytest.raises(TypeError):                           # the device L-BFGS has no sampling-based path
        DS.maximize_lbfgs("esmc", [], np.zeros((1, 2)), LO, UP)
    # SciPyOptimizer: the reference's host loop, never the device L-BFGS
    monkeypatch.setattr(DS, "maximize_lbfgs", lambda *a, **k: pytest.fail("device L-BFGS over InformationGainMC"))
    import robo_b200.maximizers.scipy_optimizer as SO
    monkeypatch.setattr(SO, "maximize_lbfgs", lambda *a, **k: pytest.fail("device L-BFGS over InformationGainMC"))
    so = SciPyOptimizer(acq, LO, UP, n_restarts=2, rng=np.random.RandomState(0))
    x = so.maximize()
    assert so.last["device"] is False and np.all(x >= LO) and np.all(x <= UP)


def test_joint_pmin_reproducible_under_np_random_seed(fake):
    from robo_b200.util.mc_part import joint_pmin
    np.random.seed(5)
    a = joint_pmin(np.zeros(3), np.eye(3), 200)
    np.random.seed(5)
    b = joint_pmin(np.zeros((3, 1)), np.eye(3), 200)
    assert np.array_equal(a, b) and a.shape == (3,) and a.sum() == pytest.approx(1.0)
    c = joint_pmin(np.zeros(3), np.eye(3), 200, rng=np.random.RandomState(1))
    d = joint_pmin(np.zeros(3), np.eye(3), 200, rng=np.random.RandomState(1))
    assert np.array_equal(c, d)
    with pytest.raises(np.linalg.LinAlgError):
        joint_pmin(np.zeros(2), -1e5 * np.eye(2), 10)


def test_argument_errors(fake):
    gp = _gp()
    with pytest.raises(ValueError):
        _mc(gp, sampler="nowhere")
    mc = _mc(gp)
    C = np.zeros((2, 2))
    with pytest.raises(ValueError):                          # before update()
        mc.compute(C)
    mc.update(gp)
    with pytest.raises(NotImplementedError):
        mc.compute(C, derivative=True)
    assert mc.compute(C).shape == (2,)
    mc.lmb = mc.lmb.copy()
    mc.lmb[0] = -np.inf
    with pytest.raises(ValueError, match="lmb should not be infinite"):
        mc.compute(C)
    with pytest.raises(ValueError, match="lmb should not be infinite"):
        mc._end_update(gp.gp.handle)
