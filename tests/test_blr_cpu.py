"""BayesianLinearRegression's host layer against the reference's own results (tests/golden/blr.npz, written by
tools/make_blr_golden.py), on the numpy stand-in of the device entry points (tests/fake_blr.py): the quirks, the
bookkeeping, the reference's unit tests, the basis and prior recognition, device_spec's dispatch and the invariants of
the sampler restatement tests/blr_model.py."""
import os

import numpy as np
import pytest

from robo_b200 import _lib, priors
from robo_b200.models import BayesianLinearRegression
from robo_b200.models import bayesian_linear_regression as BLR
from tests import blr_model as BM
from tests import fake_blr

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "blr.npz"))
CODES = {"lin": 0, "quad": 1, "none": 2}


@pytest.fixture
def fake(monkeypatch):
    return fake_blr.install(monkeypatch)


def test_header_constants_match_the_binding():
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gpk.h")).read()
    assert "#define GPK_BLR_MAX_F %d " % _lib.BLR_MAX_F in src
    for name, v in (("LINEAR", _lib.BLR_LINEAR), ("QUADRATIC", _lib.BLR_QUADRATIC), ("NONE", _lib.BLR_NONE)):
        assert "GPK_BLR_%s = %d" % (name, v) in src
    cuh = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "robo_b200", "csrc",
                            "gpk_blr.cuh")).read()
    assert "GPK_BLR_TAG_MOVE 0x%08Xu" % BM.TAG_MOVE in cuh and "GPK_BLR_TAG_ACC 0x%08Xu" % BM.TAG_ACC in cuh


@pytest.mark.parametrize("name", sorted(CODES))
def test_mll_quirks_against_the_reference(name):
    """The 2-norm (not squared), log det overflowing to +inf (mll -inf), the lognormal prior's -inf below loc = -10 and
    the horseshoe of 1 / theta_1 (theta_1 = 0 -> 1 / 0 = inf -> -inf): the restatement equals the reference."""
    Phi = BM.features(G[name + "_X"], CODES[name])
    got = BM.lnpost(Phi, G[name + "_y"])(G[name + "_grid"])
    ref = G[name + "_mll"].copy()
    ref[np.isnan(ref)] = -np.inf
    assert np.array_equal(np.isfinite(got), np.isfinite(ref))
    fin = np.isfinite(ref)
    np.testing.assert_allclose(got[fin], ref[fin], rtol=1e-12)
    grid = G[name + "_grid"]
    assert np.all(got[grid[:, 0] <= -10] == -np.inf)            # lognormal prior with loc = -10
    if Phi.shape[1] * 150.0 > 709.79:                           # alpha^F alone overflows det A
        assert np.all(got[grid[:, 0] == 150.0] == -np.inf)
    assert np.all(got[grid[:, 1] == 0.0] == -np.inf)            # horseshoe of 1 / 0
    assert np.any(np.isfinite(got[grid[:, 1] < 0]))             # the horseshoe of a negative 1 / theta_1 is finite


def test_prior_restatement_and_sample_from_prior_quirk():
    from robo_b200.priors import BayesianLinearRegressionPrior, HorseshoePrior, LognormalPrior
    p = BayesianLinearRegressionPrior(rng=np.random.RandomState(5))
    th = np.array([-9.2, 3.0])
    assert p.lnprob(th) == LognormalPrior(0.1, -10).lnprob(-9.2) + HorseshoePrior(0.1).lnprob(1 / 3.0)
    p0 = p.sample_from_prior(20)
    r = np.random.RandomState(5)
    a = r.lognormal(mean=-10, sigma=0.1, size=20)
    lam = np.abs(r.standard_cauchy(size=20))
    sig = np.log(np.abs(r.randn() * lam * 0.1))
    assert np.array_equal(p0[:, 0], a) and np.all((a > 3e-5) & (a < 7e-5))
    assert np.array_equal(p0[:, 1], np.log(1 / np.exp(sig)))


def test_train_bookkeeping_and_models(fake):
    X, y = G["unit_X"], G["unit_y"]
    m = BayesianLinearRegression(alpha=1, beta=1000, rng=np.random.RandomState(0))
    m.train(X, y, do_optimize=False)
    assert m.hypers == [[1, 1000]]
    assert np.array_equal(m.X_transformed, BLR.linear_basis_func(X))
    np.testing.assert_allclose(m.models[0][0], G["unit_m"], rtol=1e-13)
    np.testing.assert_allclose(m.models[0][1], G["unit_S"], rtol=1e-13)
    mu, var = m.predict(G["unit_Xt"])
    np.testing.assert_allclose(mu, G["unit_mu"], rtol=1e-13)
    np.testing.assert_allclose(var, G["unit_var"], rtol=1e-13)
    assert m.marginal_log_likelihood(np.array([0.0, np.log(1000)])) == pytest.approx(float(G["unit_mll"]), rel=1e-13)
    assert m.negative_mll(np.array([0.0, np.log(1000)])) == pytest.approx(-float(G["unit_mll"]), rel=1e-13)
    assert m.get_json_data()["X"] == X.tolist()


@pytest.mark.parametrize("name", sorted(CODES))
def test_predict_over_several_hypers(fake, name):
    m = BayesianLinearRegression(basis_func={"lin": BLR.linear_basis_func, "quad": BLR.quadratic_basis_func,
                                             "none": None}[name], rng=np.random.RandomState(1))
    m.train(G[name + "_X"], G[name + "_y"], do_optimize=False)
    m.hypers = G[name + "_hypers"]
    m._fitted = False
    mu, var = m.predict(G[name + "_Xt"])
    np.testing.assert_allclose(mu, G[name + "_mu"], rtol=1e-12)
    np.testing.assert_allclose(var, G[name + "_var"], rtol=1e-12)


def test_mcmc_path_seeds_burn_in_and_hypers(fake):
    m = BayesianLinearRegression(rng=np.random.RandomState(3), n_hypers=6, chain_length=4, burnin_steps=3)
    X, y = G["mcmc_X"], G["mcmc_y"]
    m.train(X, y)
    h = m._handle
    assert m.burned and [c[2] for c in h.sample_calls] == [3, 4]
    assert np.array_equal(m.hypers, np.exp(m.p0))
    m.train(np.vstack([X, [[0.5]]]), np.append(y, 0.0))
    assert [c[2] for c in h.sample_calls] == [3, 4, 4]
    assert len(m.models) == 6 and m.models[0][1].shape == (2, 2)
    # the seeds come from the model's rng, one per run; the first run starts from the prior
    r = np.random.RandomState(3)
    pr = priors.BayesianLinearRegressionPrior(rng=np.random.RandomState(3))
    p0 = pr.sample_from_prior(6)
    r.set_state(pr.rng.get_state())
    seeds = [int(r.randint(0, 2 ** 63, dtype=np.int64)) for _ in range(2)]
    assert [c[0] for c in h.sample_calls[:2]] == seeds
    assert np.array_equal(h.sample_calls[0][1], p0)


def test_fmin_path_matches_the_reference(fake):
    m = BayesianLinearRegression(do_mcmc=False, rng=np.random.RandomState(3))
    m.train(G["lin_X"], G["lin_y"], do_optimize=True)
    np.testing.assert_allclose(np.array(m.hypers), G["fmin_hypers"], rtol=1e-10)


def test_reference_unit_tests(fake):
    # test/test_models/test_bayesian_linear_regression.py on the golden file's draws of its np.random.rand data (its
    # variance tolerance, decimal=3, does not hold for every draw of 10 points)
    X, y, X_test = G["unit_X"], G["unit_y"], G["unit_Xt"]
    model = BayesianLinearRegression(alpha=1, beta=1000)
    model.train(X, y, do_optimize=False)
    m, v = model.predict(X_test)
    assert m.shape == (10,) and v.shape == (10,)
    np.testing.assert_almost_equal(m, X_test[:, 0] * 2, decimal=2)
    np.testing.assert_almost_equal(v, np.ones([v.shape[0]]) / 1000., decimal=3)
    theta = np.array([np.log(1), np.log(1000)])
    assert np.isfinite(model.marginal_log_likelihood(theta))
    assert model.negative_mll(theta) == -model.marginal_log_likelihood(theta)
    inc, inc_val = model.get_incumbent()
    b = np.argmin(y)
    assert np.all(inc == X[b]) and inc_val == y[b]


def test_basis_recognition_and_refusals(fake):
    assert BLR.basis_code(BLR.linear_basis_func) == _lib.BLR_LINEAR
    assert BLR.basis_code(BLR.quadratic_basis_func) == _lib.BLR_QUADRATIC
    assert BLR.basis_code(None) == _lib.BLR_NONE
    assert BLR.basis_code(lambda x: x) == _lib.BLR_NONE
    assert BLR.basis_code(lambda x: np.hstack([x, np.ones((len(x), 1))])) == _lib.BLR_LINEAR
    for f in (lambda x: 2 * x, lambda x: np.hstack([x, x ** 2, np.ones((len(x), 1))]), lambda x: np.sin(x)):
        with pytest.raises(TypeError, match="three bases"):
            BayesianLinearRegression(basis_func=f).train(G["unit_X"], G["unit_y"], do_optimize=False)
    with pytest.raises(ValueError, match="GPK_BLR_MAX_F = 64"):
        BayesianLinearRegression().train(np.random.rand(5, 64), np.zeros(5), do_optimize=False)
    with pytest.raises(ValueError, match="GPK_BLR_MAX_F = 64"):
        BayesianLinearRegression(basis_func=BLR.quadratic_basis_func).train(np.random.rand(5, 32), np.zeros(5),
                                                                              do_optimize=False)
    BayesianLinearRegression(basis_func=BLR.quadratic_basis_func).train(np.random.rand(5, 31), np.zeros(5),
                                                                          do_optimize=False)
    with pytest.raises(TypeError, match="BayesianLinearRegressionPrior"):
        BayesianLinearRegression(prior=priors.DefaultPrior(2))


def test_device_spec_dispatch(fake):
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    from robo_b200.maximizers.device_spec import device_spec
    m = BayesianLinearRegression(alpha=1, beta=1000, rng=np.random.RandomState(0))
    m.train(G["unit_X"], G["unit_y"], do_optimize=False)
    for cls, kind in ((EI, "ei"), (LogEI, "log_ei"), (PI, "pi"), (LCB, "lcb")):
        which, (k, etas, par, hs) = device_spec(cls(m), "test")
        assert which == "acq" and k == kind and hs == [m._handle]
        assert etas == [0.0 if kind == "lcb" else float(np.min(G["unit_y"]))]


def test_sampler_restatement_invariants():
    P = np.column_stack([np.linspace(-9.5, -8.5, 10), np.linspace(1, 3, 10)])
    for step in range(5):
        for half in (0, 1):
            q, z, c = BM.proposals(77, step, half, P)
            assert np.all((z >= 0.5) & (z <= 2.0))
            assert np.all((c >= (1 - half) * 5) & (c < (2 - half) * 5))
    f = lambda T: -((np.atleast_2d(T) + 9) ** 2).sum(axis=1)       # noqa: E731
    a = BM.run(f, P, 30, 5)
    b = BM.run(f, P, 30, 5)
    assert np.array_equal(a["pos"], b["pos"]) and a["n_accepted"].sum() > 0
    nan = BM.run(lambda T: np.full(len(np.atleast_2d(T)), np.nan), P, 3, 5)
    assert np.array_equal(nan["pos"], P) and np.all(nan["n_accepted"] == 0)
