"""BayesianLinearRegression on the device (robo_b200/csrc/gpk_blr.cuh) against the reference's own results
(tests/golden/blr.npz, written by tools/make_blr_golden.py), an extended-precision restatement and the exact sampler
restatement tests/blr_model.py."""
import os

import mpmath
import numpy as np
import pytest

from robo_b200 import _lib
from robo_b200.models.bayesian_linear_regression import (BayesianLinearRegression, linear_basis_func,
                                                         quadratic_basis_func)
from tests import blr_model as BM
from tests import blr_reference

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "blr.npz"))
BASES = {"lin": _lib.BLR_LINEAR, "quad": _lib.BLR_QUADRATIC, "none": _lib.BLR_NONE}
FUNCS = {"lin": linear_basis_func, "quad": quadratic_basis_func, "none": None}


def _handle(X, y, basis):
    h = _lib.Handle(0)
    _lib.blr_set_data(h, X, y, basis, BM.PRIOR_PAR)
    return h


@pytest.mark.parametrize("name", sorted(BASES))
def test_lnpost_matches_the_reference_mll(name):
    h = _handle(G[name + "_X"], G[name + "_y"], BASES[name])
    got = _lib.blr_lnpost(h, G[name + "_grid"])
    ref = G[name + "_mll"].copy()
    ref[np.isnan(ref)] = -np.inf
    fin = np.isfinite(ref)
    assert np.array_equal(got[~fin], ref[~fin])
    assert np.any(~fin) and np.any(fin)
    ok = fin & (G[name + "_cond"] <= 1e8)
    assert ok.sum() >= 10
    np.testing.assert_allclose(got[ok], ref[ok], rtol=1e-9, atol=0)
    assert np.all(np.isfinite(got[fin]))


def _mll_mp(Phi, y, theta, dps=50):
    """The reference's mll (without the prior) in 50-digit arithmetic."""
    mpmath.mp.dps = dps
    a, b = mpmath.exp(mpmath.mpf(theta[0])), mpmath.exp(mpmath.mpf(theta[1]))
    P = mpmath.matrix(Phi.tolist())
    Y = mpmath.matrix(y.tolist())
    F, N = Phi.shape[1], Phi.shape[0]
    A = b * (P.T * P) + a * mpmath.eye(F)
    m = b * (mpmath.inverse(A) * (P.T * Y))
    r = Y - P * m
    nrm = mpmath.sqrt(sum(v ** 2 for v in r))
    mtm = sum(v ** 2 for v in m)
    v = F / mpmath.mpf(2) * mpmath.log(a) + N / mpmath.mpf(2) * mpmath.log(b) - N / mpmath.mpf(2) * mpmath.log(2 * mpmath.pi)
    v -= b / 2 * nrm + a / 2 * mtm + mpmath.log(mpmath.det(A)) / 2
    return v, mpmath.mpf(1) * mpmath.norm(A, 2) * mpmath.norm(mpmath.inverse(A), 2)


def test_ill_conditioned_against_extended_precision():
    """Nearly collinear quadratic features: error <= 1e-13 cond(A) |mll| against a 50-digit restatement."""
    rng = np.random.RandomState(7)
    X = 1.0 + 1e-3 * rng.rand(30, 2)
    y = X.sum(axis=1) + 1e-4 * rng.randn(30)
    theta = np.array([-9.0, 14.0])
    h = _handle(X, y, _lib.BLR_QUADRATIC)
    got = _lib.blr_lnpost(h, theta[None])[0] - BM.prior_lnprob(theta)
    ref, cond = _mll_mp(BM.features(X, 1), y, theta)
    assert float(cond) > 1e8
    assert abs(got - float(ref)) <= 1e-13 * float(cond) * abs(float(ref))


@pytest.mark.parametrize("name", sorted(BASES))
def test_fit_models_and_predict_match_the_reference(name):
    h = _handle(G[name + "_X"], G[name + "_y"], BASES[name])
    _lib.blr_fit(h, G[name + "_hypers"])
    models = _lib.blr_models(h)
    for i, (m, S) in enumerate(models):
        np.testing.assert_allclose(m, G[name + "_m"][i], rtol=1e-8, atol=1e-12 * np.abs(G[name + "_m"][i]).max())
        np.testing.assert_allclose(S, G[name + "_S"][i], rtol=1e-8, atol=1e-12 * np.abs(G[name + "_S"][i]).max())
    mu, var = h.predict(G[name + "_Xt"])
    np.testing.assert_allclose(mu, G[name + "_mu"], rtol=1e-9, atol=1e-12 * np.abs(G[name + "_mu"]).max())
    np.testing.assert_allclose(var, G[name + "_var"], rtol=1e-8)


def test_reference_unit_test_data():
    m = BayesianLinearRegression(alpha=1, beta=1000, rng=np.random.RandomState(0))
    m.train(G["unit_X"], G["unit_y"], do_optimize=False)
    mu, var = m.predict(G["unit_Xt"])
    np.testing.assert_allclose(mu, G["unit_mu"], rtol=1e-9)
    np.testing.assert_allclose(var, G["unit_var"], rtol=1e-8)
    np.testing.assert_almost_equal(mu, G["unit_Xt"][:, 0] * 2, decimal=2)
    np.testing.assert_almost_equal(var, np.ones(10) / 1000., decimal=3)
    np.testing.assert_allclose(m.models[0][0], G["unit_m"], rtol=1e-9)
    np.testing.assert_allclose(m.marginal_log_likelihood(np.array([0.0, np.log(1000)])), G["unit_mll"], rtol=1e-9)


@pytest.mark.parametrize("name,steps,D,N,nw", [
    ("lin", 40, None, None, 12), ("quad", 25, None, None, 12), ("none", 25, None, None, 12),
    ("lin", 6, 33, 257, 4), ("none", 4, 64, 4097, 202), ("quad", 5, 31, 4097, 4), ("lin", 3, 63, 129, 202),
    ("none", 0, 34, 257, 12)], ids=["lin-40", "quad-25", "none-25", "F34-N257-nw4", "F64-N4097-nw202", "F63-N4097-nw4",
                                  "F64-N129-nw202", "F34-N257-steps0"])
def test_sample_bit_for_bit_and_deterministic(name, steps, D, N, nw):
    """The golden sets (F <= 7, N <= 50), and F = 34 and 64, N = 257 and 4097, nwalkers 4 (the least) and 202, steps 0
    (the initial log-posteriors only)."""
    if D is None:
        X, y = G[name + "_X"], G[name + "_y"]
    else:
        X, y, _ = blr_reference.case(BASES[name], D, N)
    h = _handle(X, y, BASES[name])
    p0 = np.column_stack([-9.0 + 0.2 * np.random.RandomState(1).randn(nw), 2.0 + np.random.RandomState(2).rand(nw)])
    seed = 0x1234ABCD5678
    r = _lib.blr_sample(h, seed, p0, steps)
    ref = BM.run(lambda T: _lib.blr_lnpost(h, T), p0, steps, seed)
    assert np.array_equal(r["pos"].view(np.int64), ref["pos"].view(np.int64))
    assert np.array_equal(r["lnpost"].view(np.int64), ref["lnpost"].view(np.int64))
    assert np.array_equal(r["n_accepted"], ref["n_accepted"])
    assert (r["n_accepted"].sum() > 0) == (steps > 0)
    r2 = _lib.blr_sample(_handle(X, y, BASES[name]), seed, p0, steps)
    assert np.array_equal(r2["pos"].view(np.int64), r["pos"].view(np.int64))
    if steps == 0:
        assert np.array_equal(r["pos"], p0)


def test_chain_agrees_in_law_with_the_reference():
    """Over the three seeds at the default chain, the device's mean final log alpha and log beta lie within 4 standard
    errors of the reference's.  Both sides pool 3 x 20 final walkers; treating them as independent, the standard error
    of the difference of the two means is sqrt(sd_ref^2 / 60 + sd_dev^2 / 60)."""
    walkers = []
    for s in G["mcmc_seeds"]:
        m = BayesianLinearRegression(rng=np.random.RandomState(int(s)))
        m.train(G["mcmc_X"], G["mcmc_y"], do_optimize=True)
        walkers.append(m.p0)
        assert np.array_equal(m.hypers, np.exp(m.p0))
    W = np.array(walkers).reshape(-1, 2)
    ref = G["mcmc_walkers"].reshape(-1, 2)
    se = np.sqrt(ref.var(axis=0, ddof=1) / len(ref) + W.var(axis=0, ddof=1) / len(W))
    assert np.all(np.abs(W.mean(axis=0) - ref.mean(axis=0)) <= 4 * se), (W.mean(axis=0), ref.mean(axis=0), se)


def _trained(basis=quadratic_basis_func, d=2, n=40, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.rand(n, d)
    y = ((X - 0.3) ** 2).sum(axis=1) + 0.01 * rng.randn(n)
    m = BayesianLinearRegression(basis_func=basis, rng=np.random.RandomState(seed), chain_length=100, burnin_steps=100)
    m.train(X, y, do_optimize=True)
    return m


@pytest.mark.parametrize("kind", ["ei", "log_ei", "pi", "lcb"])
def test_scoring_equals_moments_over_predict(kind):
    m = _trained()
    X = np.random.RandomState(3).rand(65536, 2) * 1.4 - 0.2
    eta = 0.0 if kind == "lcb" else float(m.get_incumbent()[1])
    h = m._ready_handle()
    r = _lib.acq_multi([h], X, 0, kind=_lib.ACQ_KIND[kind], eta=[eta], par=0.01, want_argmax=True)
    mu, var = m.predict(X)
    ref, _ = _lib.moments_handle().acq_moments(mu, var, _lib.ACQ_KIND[kind], eta, 0.01)
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(r["values"]), fin)
    np.testing.assert_allclose(r["values"][fin], ref[fin], rtol=1e-12, atol=0)
    assert r["best_idx"] == int(np.argmax(ref))
    one = h.acq(X, _lib.ACQ_KIND[kind], eta, 0.01)
    assert np.array_equal(one["values"], r["values"]) and one["best_idx"] == r["best_idx"]


def test_device_maximizers_return_their_energy():
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import device_spec as DS
    m = _trained()
    acq = EI(m)
    lo, up = np.zeros(2), np.ones(2)
    spec = DS.device_spec(acq, "test")
    assert spec[0] == "acq"
    runs = [DS.maximize_de(*spec, 5, 30, 20, (0.5, 1.0), 0.7, 0.01, 0.0, lo, up),
            DS.maximize_cmaes(*spec, 9, np.full(2, 0.5), lo, up, 400, 0),
            DS.maximize_direct(*spec, lo, up, 400, 200)]
    r = DS.maximize_lbfgs(*spec, np.random.RandomState(2).rand(4, 2), lo, up)
    best = int(np.argmin(r["energy"]))
    runs.append(dict(x=r["x"][best], energy=r["energy"][best]))
    for r in runs:
        x = np.asarray(r["x"]).ravel()
        assert np.all(x >= lo) and np.all(x <= up)
        host = acq.compute(x[None])
        assert -r["energy"] == pytest.approx(float(np.ravel(host)[0]), rel=1e-12, abs=1e-300)


def test_maximizer_classes_over_ei():
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import (CMAES, DeviceRandomSampling, DifferentialEvolution, Direct, GridSearch,
                                      SciPyOptimizer)
    # GridSearch is one-dimensional and CMAES refuses one dimension (the reference's RuntimeErrors)
    for d, classes in ((1, (GridSearch, DifferentialEvolution, DeviceRandomSampling)),
                       (2, (DifferentialEvolution, SciPyOptimizer, CMAES, Direct, DeviceRandomSampling))):
        m = _trained(basis=quadratic_basis_func, d=d)
        acq = EI(m)
        lo, up = np.zeros(d), np.ones(d)
        for cls in classes:
            kw = dict(verbose=False) if cls in (CMAES, Direct) else {}
            x = np.asarray(cls(acq, lo, up, rng=np.random.RandomState(1), **kw).maximize()).ravel()
            assert x.shape == (d,) and np.all((lo <= x) & (x <= up)), cls.__name__
            assert np.isfinite(acq.compute(x[None])).all()


def test_bayesian_optimization_end_to_end():
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DifferentialEvolution
    from robo_b200.solver.bayesian_optimization import BayesianOptimization
    lo, up = np.zeros(2), np.ones(2)
    rng = np.random.RandomState(4)
    m = BayesianLinearRegression(basis_func=quadratic_basis_func, rng=rng, chain_length=200, burnin_steps=200)
    acq = EI(m)
    bo = BayesianOptimization(lambda x: float(((x - 0.3) ** 2).sum()), lo, up, acq, m,
                              DifferentialEvolution(acq, lo, up, rng=rng), rng=rng)
    x, fval = bo.run(num_iterations=5)
    assert len(bo.X) == 5 and np.all((np.asarray(bo.X) >= 0) & (np.asarray(bo.X) <= 1))
    assert np.isfinite(fval)


def test_argument_errors_and_gp_only_refusals():
    X, y = G["lin_X"], G["lin_y"]
    h = _lib.Handle(0)
    with pytest.raises(ValueError, match="gpk_blr_set_data has not been called"):
        _lib.blr_lnpost(h, np.zeros((1, 2)))
    with pytest.raises(ValueError, match="unknown basis"):
        _lib.blr_set_data(h, X, y, 7, BM.PRIOR_PAR)
    with pytest.raises(ValueError, match="GPK_BLR_MAX_F"):
        _lib.blr_set_data(h, np.random.rand(5, 32), np.zeros(5), _lib.BLR_QUADRATIC, BM.PRIOR_PAR)
    _lib.blr_set_data(h, X, y, _lib.BLR_LINEAR, BM.PRIOR_PAR)
    with pytest.raises(ValueError, match="even number of walkers"):
        _lib.blr_sample(h, 1, np.zeros((5, 2)), 3)
    with pytest.raises(ValueError, match="steps >= 0"):
        _lib.blr_sample(h, 1, np.zeros((6, 2)), -1)
    with pytest.raises(RuntimeError, match="not fitted"):
        h.predict(X[:3])
    with pytest.raises(np.linalg.LinAlgError):
        _lib.blr_fit(h, np.array([[0.0, 0.0]]))
    _lib.blr_fit(h, np.array([[1.0, 10.0]]))
    refuse = "Bayesian linear regression"
    with pytest.raises(ValueError, match=refuse):
        h.set_data(X, y)
    with pytest.raises(ValueError, match=refuse):
        h.set_kernel(0, 0.0, [0], [0], [0.0])
    with pytest.raises(ValueError, match=refuse):
        h.fit(1e-6, 0.0)
    with pytest.raises(ValueError, match=refuse):
        h.predict_grad(X[:3])
    with pytest.raises(ValueError, match=refuse):
        h.predict_cov(X[:3])
    with pytest.raises(ValueError, match=refuse):
        _lib.hyper_lnpost(h, np.zeros((1, 3)))
    with pytest.raises(ValueError, match=refuse):
        _lib.es_multi([h], X[:3])
    with pytest.raises(ValueError, match=refuse):
        _lib.esmc_multi([h], X[:3])
    gp = _lib.Handle(0)
    gp.set_data(X, y)
    with pytest.raises(ValueError, match="Gaussian-process model"):
        _lib.blr_set_data(gp, X, y, _lib.BLR_LINEAR, BM.PRIOR_PAR)
    # the model's own refusals
    with pytest.raises(TypeError, match="three bases"):
        BayesianLinearRegression(basis_func=lambda x: 2 * x).train(X, y, do_optimize=False)
    with pytest.raises(ValueError, match="GPK_BLR_MAX_F"):
        BayesianLinearRegression().train(np.random.rand(5, 64), np.zeros(5), do_optimize=False)
