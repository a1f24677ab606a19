"""DNGO on the device: the Adam training against tests/dngo_model.py bit for bit (the net, the features Theta and the
Adam state), the Bayesian linear regression of a DNGO handle against a BLR handle on the same Theta bit for bit, the
scoring pass against an extended-precision per-sample evaluation with a bound from the term magnitudes, the
acquisitions and the arg-max, every maximizer, copies, the model-kind refusals in both directions, one train at the
default settings and a short Bayesian-optimisation loop."""
import copy
import pickle

import numpy as np
import pytest

from robo_b200 import _lib
from robo_b200.models import DNGO
from tests import blr_model as LM
from tests import dngo_model as DM
from tests import fake_blr

pytestmark = pytest.mark.gpu


def _data(N, D, seed):
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    return X, np.sinc(X * 10 - 5).sum(axis=1) + 0.05 * rng.randn(N)


def _branin(N, seed):
    rng = np.random.RandomState(seed)
    X = rng.rand(N, 2) * [15, 15] - [5, 0]
    x1, x2 = X[:, 0], X[:, 1]
    y = (x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x1) + 10
    return X, y


def _trained_handle(X, y, seed, counter, batch, epochs, nx=True, ny=True, lr=0.01):
    h = _lib.Handle(0)
    _lib.dngo_set_data(h, X, y, nx, ny, LM.PRIOR_PAR)
    _lib.dngo_train(h, seed, counter, lr, batch, epochs)
    return h


@pytest.mark.parametrize("D,N,batch,epochs,nx,ny", [
    (1, 7, 10, 3, True, True),        # N < batch: B = N, one batch per epoch
    (2, 23, 10, 4, True, True),       # N not a multiple of B: 3 rows dropped per epoch
    (8, 16, 16, 2, True, False),      # N = B
    (64, 30, 10, 2, False, True),
    (2, 40, 16, 1, False, False),
    (2, 20, 5, 7, True, True),
    (8, 45, 10, 12, True, True)])
def test_training_equals_the_model_bit_for_bit(D, N, batch, epochs, nx, ny):
    X, y = _data(N, D, D * 100 + N)
    seed, counter = 7654321 + D, 2
    h = _trained_handle(X, y, seed, counter, batch, epochs, nx, ny)
    Xs, ys = DM.normalise(X, y, nx, ny)[:2]
    th, st, Theta = DM.train(Xs, ys, seed, counter, 0.01, batch, epochs)
    assert np.array_equal(_lib.dngo_net(h), th)
    ds = _lib.dngo_state(h)
    assert ds["t"] == st["t"] == epochs * (N // min(batch, N))
    assert np.array_equal(ds["m"], st["m"]) and np.array_equal(ds["v"], st["v"])
    assert np.array_equal(_lib.dngo_features(h, X), Theta)
    # the Theta the training kernel wrote: the regression's log-posterior runs over it, so a BLR handle on the model's
    # Theta gives the same bits only if the device's Theta is the model's
    blr = _lib.Handle(0)
    _lib.blr_set_data(blr, Theta, ys, _lib.BLR_NONE, LM.PRIOR_PAR)
    T = np.array([[0.0, 0.0], [-2.0, 3.0], [1.0, 5.0]])
    assert np.array_equal(_lib.blr_lnpost(h, T), _lib.blr_lnpost(blr, T))
    assert _lib.dngo_dims(h) == (N, D, DM.n_params(D), 0)


def test_epochs_seed_and_counter_change_the_net():
    X, y = _data(20, 2, 1)
    a = _lib.dngo_net(_trained_handle(X, y, 5, 0, 10, 2))
    assert np.array_equal(a, _lib.dngo_net(_trained_handle(X, y, 5, 0, 10, 2)))
    for args in ((6, 0, 10, 2), (5, 1, 10, 2), (5, 0, 10, 3), (5, 0, 7, 2)):
        assert not np.array_equal(a, _lib.dngo_net(_trained_handle(X, y, *args)))


def test_blr_stage_equals_a_blr_handle_bit_for_bit():
    X, y = _data(33, 3, 2)
    h = _trained_handle(X, y, 17, 0, 10, 5)
    Theta = _lib.dngo_features(h, X)
    ys = DM.normalise(X, y)[1]
    blr = _lib.Handle(0)
    _lib.blr_set_data(blr, Theta, ys, _lib.BLR_NONE, LM.PRIOR_PAR)
    rng = np.random.RandomState(3)
    T = np.c_[rng.uniform(-8, 3, 40), rng.uniform(-2, 8, 40)]
    assert np.array_equal(_lib.blr_lnpost(h, T), _lib.blr_lnpost(blr, T))
    p0 = np.c_[rng.uniform(-3, 1, 20), rng.uniform(0, 5, 20)]
    a, b = _lib.blr_sample(h, 99, p0, 30), _lib.blr_sample(blr, 99, p0, 30)
    for k in ("pos", "lnpost", "n_accepted"):
        assert np.array_equal(a[k], b[k]), k
    hypers = np.exp(a["pos"])
    _lib.dngo_fit(h, hypers)
    _lib.blr_fit(blr, hypers)
    for (m1, S1), (m2, S2) in zip(_lib.blr_models(h), _lib.blr_models(blr)):
        assert np.array_equal(m1, m2) and np.array_equal(S1, S2)
    assert _lib.dngo_dims(h)[3] == 20 and _lib.blr_models(h)[0][1].shape == (50, 50)


def _acq_interval(m, v, bm, bv, kind, eta, par):
    """The acquisition's range over the moment box [m -+ bm] x [v -+ bv] (monotone in each moment); LogEI as the log of
    EI's range."""
    vals = []
    for dm in (-1, 1):
        for dv in (-1, 1):
            with np.errstate(all="ignore"):
                f = np.asarray(fake_blr.moments(m + dm * bm, np.maximum(v + dv * bv, 1e-300),
                                                _lib.ACQ_EI if kind == _lib.ACQ_LOG_EI else kind, eta, par)[0],
                               dtype=np.float64)
                vals.append(np.log(f) if kind == _lib.ACQ_LOG_EI else f)
    vals = np.array(vals)
    return vals.min(axis=0), vals.max(axis=0)


_FITTED = {}


def _fitted(k):
    """A trained DNGO handle (D = 3, N = 40) fitted with k hyper-samples spread over two decades each."""
    if k not in _FITTED:
        X, y = _data(40, 3, 7)
        h = _trained_handle(X, y, 23, 0, 10, 30)
        rng = np.random.RandomState(k)
        hypers = np.c_[np.exp(rng.uniform(-3, 1, k)), np.exp(rng.uniform(1, 6, k))]
        _lib.dngo_fit(h, hypers)
        _FITTED[k] = (h, X, y, hypers)
    return _FITTED[k]


@pytest.mark.parametrize("k", [1, 2, 20])
@pytest.mark.parametrize("M", [1, 255, 256, 257, 1000])
def test_scoring_against_extended_precision(k, M):
    h, X, y, hypers = _fitted(k)
    rng = np.random.RandomState(M + k)
    Xt = rng.uniform(-0.2, 1.2, (M, 3))
    mu, var = h.predict(Xt)
    stats = DM.normalise(X, y)[2:]
    m_ld, v_ld, bm, bv = DM.predict_ld(_lib.dngo_net(h), _lib.blr_models(h), hypers, Xt, *stats)
    err_m, err_v = np.abs(mu - m_ld), np.abs(var - v_ld)
    print("k=%d M=%d: max error / bound: mean %.3g, variance %.3g" % (k, M, np.max(err_m / bm), np.max(err_v / bv)))
    assert np.all(err_m <= bm) and np.all(err_v <= bv)
    assert np.all(var > 0)
    m64, v64, bm64, bv64 = (a.astype(np.float64) for a in (m_ld, v_ld, bm, bv))
    eta = float(np.min(y))
    for kind in (_lib.ACQ_EI, _lib.ACQ_LOG_EI, _lib.ACQ_PI, _lib.ACQ_LCB):
        e = eta if kind != _lib.ACQ_LCB else 0.0
        r = h.acq(Xt, kind, e, 0.0)
        lo, hi = _acq_interval(m64, v64, bm64, bv64, kind, e, 0.0)
        tol = 1e-12 * np.maximum(np.abs(lo), np.abs(hi)) + 1e-300
        ok = (r["values"] >= lo - tol) & (r["values"] <= hi + tol)
        assert np.all(ok | ~np.isfinite(lo)), kind
        b = r["best_idx"]
        assert r["values"][b] == np.max(r["values"]) and b == int(np.argmax(r["values"]))
        assert hi[b] + tol[b] >= np.max(lo)                      # the arg-max equals the true one within the bound


def test_many_candidates_beyond_one_chunk():
    h, X, y, hypers = _fitted(20)
    Xt = np.random.RandomState(1).rand(70001, 3)
    r = h.acq(Xt, _lib.ACQ_EI, float(y.min()), 0.0, want_moments=True)
    for lo in (0, 65535, 70000):
        mu, var = h.predict(Xt[lo:lo + 1])
        assert mu[0] == r["mu"][lo] and var[0] == r["var"][lo]
    assert r["best_idx"] == int(np.argmax(r["values"])) and r["n_negative"] == 0


def test_model_train_copy_and_pickle():
    X, y = _data(12, 2, 5)
    m = DNGO(rng=np.random.RandomState(3), num_epochs=50, chain_length=100, burnin_steps=100)
    m.train(X, y)
    assert m.net.shape == (DM.n_params(2),) and m.counter == 1 and m.Theta.shape == (12, 50)
    assert len(m.models) == 20 and m.p0.shape == (20, 2) and m.burned
    Xt = np.random.RandomState(6).rand(300, 2)
    mu, v = m.predict(Xt)
    assert np.all(np.isfinite(mu)) and np.all(v > 0)
    for c in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        mu2, v2 = c.predict(Xt)
        assert np.array_equal(mu, mu2) and np.array_equal(v, v2)
    # set_net rebuilds Theta and the regression's products bit for bit
    h = _lib.Handle(0)
    _lib.dngo_set_data(h, X, y, True, True, LM.PRIOR_PAR)
    _lib.dngo_set_net(h, m.net)
    assert np.array_equal(_lib.dngo_features(h, X), m.Theta)
    T = np.log(np.asarray(m.hypers))
    assert np.array_equal(_lib.blr_lnpost(h, T), _lib.blr_lnpost(m._handle, T))
    with pytest.raises(RuntimeError, match="no training has run"):
        _lib.dngo_state(h)


def _trained(d=2, n=15):
    X, y = _data(n, d, 11 + d)
    m = DNGO(rng=np.random.RandomState(2), num_epochs=40, chain_length=50, burnin_steps=50)
    m.train(X, y)
    return m


def test_maximizer_classes():
    from robo_b200.acquisition_functions import EI, LCB, PI
    from robo_b200.maximizers import CMAES, DeviceRandomSampling, DifferentialEvolution, Direct, GridSearch, \
        SciPyOptimizer
    for d, classes in ((1, (GridSearch, DifferentialEvolution, DeviceRandomSampling)),
                       (2, (DifferentialEvolution, SciPyOptimizer, CMAES, Direct, DeviceRandomSampling))):
        m = _trained(d=d)
        for acq_cls in (EI, PI, LCB):
            acq = acq_cls(m)
            lo, up = np.zeros(d), np.ones(d)
            for cls in classes:
                kw = dict(verbose=False) if cls in (CMAES, Direct) else {}
                x = np.asarray(cls(acq, lo, up, rng=np.random.RandomState(1), **kw).maximize()).ravel()
                assert x.shape == (d,) and np.all((lo <= x) & (x <= up)), cls.__name__
                assert np.isfinite(acq.compute(x[None])).all()


def test_default_settings_on_branin():
    # 500 epochs, 2000 burn-in + 2000 chain steps on 30 Branin points: the predictive mean follows the targets and the
    # variance is positive and finite
    X, y = _branin(30, 0)
    m = DNGO(rng=np.random.RandomState(4))
    m.train(X, y)
    mu, v = m.predict(X)
    corr = float(np.corrcoef(mu, y)[0, 1])
    rel = float(np.sqrt(np.mean((mu - y) ** 2)) / np.std(y))
    print("Branin N=30 at the defaults: corr(mu, y) %.4f, RMSE / std(y) %.4f" % (corr, rel))
    assert corr > 0.9 and rel < 0.5
    Xt = np.random.RandomState(1).rand(500, 2) * [15, 15] - [5, 0]
    mu_t, v_t = m.predict(Xt)
    assert np.all(np.isfinite(mu_t)) and np.all(np.isfinite(v_t)) and np.all(v_t > 0) and np.all(v > 0)
    inc, inc_val = m.get_incumbent()
    assert np.array_equal(inc, X[np.argmin(y)])


def test_bayesian_optimization_end_to_end():
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DifferentialEvolution
    from robo_b200.solver.bayesian_optimization import BayesianOptimization

    def branin(x):
        a, b, c, r, s, t = 1, 5.1 / (4 * np.pi ** 2), 5 / np.pi, 6, 10, 1 / (8 * np.pi)
        return float(a * (x[1] - b * x[0] ** 2 + c * x[0] - r) ** 2 + s * (1 - t) * np.cos(x[0]) + s)
    lo, up = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
    rng = np.random.RandomState(4)
    m = DNGO(rng=rng, num_epochs=100, chain_length=200, burnin_steps=200)
    acq = EI(m)
    bo = BayesianOptimization(branin, lo, up, acq, m, DifferentialEvolution(acq, lo, up, rng=rng), rng=rng)
    x, fval = bo.run(num_iterations=6)
    assert len(bo.X) == 6 and np.all((np.asarray(bo.X) >= lo) & (np.asarray(bo.X) <= up))
    assert np.isfinite(fval) and m.counter >= 1


def test_refusals_and_limits():
    X, y = _data(30, 2, 8)
    par = LM.PRIOR_PAR
    h = _lib.Handle(0)
    with pytest.raises(ValueError, match="gpk_dngo_set_data has not been called"):
        _lib.dngo_train(h, 1, 0, 0.01, 10, 1)
    with pytest.raises(ValueError, match="n >= 2"):
        _lib.dngo_set_data(h, X[:1], y[:1], True, False, par)
    with pytest.raises(ValueError, match="constant"):
        _lib.dngo_set_data(h, np.c_[X, np.ones(30)], y, True, True, par)
    with pytest.raises(ValueError, match="constant"):
        _lib.dngo_set_data(h, X, np.ones(30), True, True, par)
    with pytest.raises(ValueError, match="GPK_DNGO_MAX_N = 4096"):
        _lib.dngo_set_data(h, np.random.rand(_lib.DNGO_MAX_N + 1, 1), np.random.rand(_lib.DNGO_MAX_N + 1), True, True,
                           par)
    with pytest.raises(ValueError, match="GPK_DNGO_MAX_D = 64"):
        _lib.dngo_set_data(h, np.random.rand(3, 65), np.random.rand(3), True, True, par)
    with pytest.raises(ValueError, match="finite"):
        _lib.dngo_set_data(h, np.array([[np.nan], [1.0]]), np.zeros(2), False, False, par)
    _lib.dngo_set_data(h, X, y, True, True, par)
    for call in (lambda: h.predict(X[:3]), lambda: _lib.blr_lnpost(h, np.zeros((1, 2))),
                 lambda: _lib.dngo_fit(h, [[1.0, 1.0]]), lambda: _lib.dngo_net(h), lambda: _lib.dngo_features(h, X)):
        with pytest.raises(RuntimeError, match="not trained|not fitted"):
            call()
    with pytest.raises(ValueError, match="GPK_DNGO_MAX_BATCH"):
        _lib.dngo_train(h, 1, 0, 0.01, 17, 1)
    with pytest.raises(ValueError, match="lr"):
        _lib.dngo_train(h, 1, 0, float("nan"), 10, 1)
    with pytest.raises(ValueError, match="epochs"):
        _lib.dngo_train(h, 1, 0, 0.01, 10, 0)
    _lib.dngo_train(h, 1, 0, 0.01, 10, 1)
    with pytest.raises(RuntimeError, match="not fitted"):
        h.predict(X[:3])
    _lib.dngo_fit(h, [[1.0, 1000.0]])
    # every other kind's entry points refuse the DNGO handle, naming its kind
    for call in (lambda: h.set_data(X, y), lambda: h.set_kernel(0, 0.0, [0], [0], [0.0]), lambda: h.fit(1e-6, 0.0),
                 lambda: h.predict_grad(X[:3]), lambda: h.predict_cov(X[:3]),
                 lambda: _lib.hyper_lnpost(h, np.zeros((1, 3))), lambda: _lib.es_multi([h], X[:3]),
                 lambda: _lib.blr_set_data(h, X, y, _lib.BLR_LINEAR, par), lambda: _lib.blr_fit(h, [[1.0, 1.0]]),
                 lambda: _lib.rf_set_data(h, X, y), lambda: _lib.rf_fit(h, 1, 0, 3, 0, True, True),
                 lambda: _lib.bnn_set_data(h, X, y), lambda: _lib.bnn_dims(h)):
        with pytest.raises(ValueError, match="DNGO model"):
            call()
    # the DNGO entry points refuse the other kinds
    gp = _lib.Handle(0)
    gp.set_data(X, y)
    blr = _lib.Handle(0)
    _lib.blr_set_data(blr, X, y, _lib.BLR_LINEAR, par)
    rf = _lib.Handle(0)
    _lib.rf_set_data(rf, X, y)
    bnn = _lib.Handle(0)
    _lib.bnn_set_data(bnn, X, y)
    for other, kind in ((gp, "Gaussian-process model"), (blr, "Bayesian linear regression"), (rf, "random forest"),
                        (bnn, "Bayesian neural network")):
        with pytest.raises(ValueError, match=kind):
            _lib.dngo_set_data(other, X, y, True, True, par)
        if other is not gp:
            for call in (lambda: _lib.dngo_train(other, 1, 0, 0.01, 10, 1), lambda: _lib.dngo_fit(other, [[1.0, 1.0]]),
                         lambda: _lib.dngo_dims(other), lambda: _lib.dngo_set_net(other, np.zeros(DM.n_params(2))),
                         lambda: _lib.dngo_features(other, X)):
                with pytest.raises(ValueError, match=kind):
                    call()
    with pytest.raises(ValueError, match="gpk_dngo_set_data has not been called"):
        _lib.dngo_dims(gp)
