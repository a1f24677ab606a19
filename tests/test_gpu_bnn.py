"""WrapperBohamiann on the device: the SGHMC chain against tests/bnn_model.py bit for bit on the device's normals, the
scoring pass against an extended-precision evaluation with a bound from the term magnitudes, the acquisitions and the
arg-max on those moments, ragged tiles and chunks, every maximizer, copies, the model-kind refusals and one fit at the
wrapper's full settings."""
import copy
import pickle

import numpy as np
import pytest

from robo_b200 import _lib
from robo_b200.models import WrapperBohamiann
from tests import bnn_model as BM
from tests import fake_blr

pytestmark = pytest.mark.gpu


def _data(N, D, seed):
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    return X, np.sinc(X * 10 - 5).sum(axis=1) + 0.05 * rng.randn(N)


def _device_chain(X, y, seed, counter, burn_in, num_steps, keep_every, batch=20, lr=1e-2):
    h = _lib.Handle(0)
    _lib.bnn_set_data(h, X, y)
    _lib.bnn_train(h, seed, counter, lr, 0.05, 1e-10, burn_in, num_steps, keep_every, batch)
    return h, _lib.bnn_samples(h), _lib.bnn_state(h)


@pytest.mark.parametrize("D,N,burn_in,num_steps,keep_every,batch", [
    (1, 7, 0, 9, 2, 20), (2, 20, 4, 12, 3, 20), (2, 21, 6, 14, 1, 20), (8, 45, 3, 10, 2, 20),
    (64, 21, 5, 9, 1, 20), (2, 45, 2, 8, 1, 32), (8, 7, 0, 6, 1, 3)])
def test_chain_equals_the_model_bit_for_bit(D, N, burn_in, num_steps, keep_every, batch):
    X, y = _data(N, D, D * 100 + N)
    seed, counter = 1234567 + D, 3
    h, S, st = _device_chain(X, y, seed, counter, burn_in, num_steps, keep_every, batch)
    Z = _lib.bnn_draws(h, seed, counter, -1, num_steps + 1)
    Xs, ys = BM.normalise(X, y)[:2]
    S_ref, st_ref = BM.chain(Xs, ys, seed, counter, lambda s: Z[s + 1], burn_in=burn_in, num_steps=num_steps,
                             keep_every=keep_every, batch=batch)
    assert S.shape == S_ref.shape == (BM.n_kept(burn_in, num_steps, keep_every), BM.n_params(D))
    assert np.array_equal(S, S_ref)
    for k in ("theta", "p", "tau", "g", "vhat"):
        assert np.array_equal(st[k], st_ref[k]), k
    # the adaptation stops after step burn_in: tau, g and vhat are the model's at the cut-over
    assert np.all(st["tau"] > 1.0) == (burn_in > 0)


def test_draws_are_standard_normals_and_the_initialisation_stream():
    X, y = _data(10, 2, 0)
    h = _lib.Handle(0)
    _lib.bnn_set_data(h, X, y)
    Z = _lib.bnn_draws(h, 5, 0, 0, 200)
    assert abs(Z.mean()) < 0.01 and abs(Z.std() - 1) < 0.01
    assert np.array_equal(_lib.bnn_draws(h, 5, 0, 10, 3), Z[10:13])
    assert not np.array_equal(_lib.bnn_draws(h, 5, 0, -1, 1)[0], Z[0])
    assert not np.array_equal(_lib.bnn_draws(h, 5, 1, 0, 1)[0], Z[0])


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


@pytest.mark.parametrize("D,S", [(1, 1), (2, 99), (8, 2), (64, 99)])
@pytest.mark.parametrize("M", [1, 255, 256, 257, 1000])
def test_scoring_against_extended_precision(D, S, M):
    X, y = _data(30, D, D + S)
    h = _lib.Handle(0)
    _lib.bnn_set_data(h, X, y)
    rng = np.random.RandomState(M + D)
    P = BM.n_params(D)
    samples = np.array([BM.init_theta(D, rng.randn(P)) + 0.1 * rng.randn(P) for _ in range(S)])
    samples[:, BM.layout(D)["lv"]] = rng.uniform(-6, 0, S)
    _lib.bnn_set_samples(h, samples)
    Xt = rng.uniform(-0.2, 1.2, (M, D))
    mu, var = h.predict(Xt)
    stats = BM.normalise(X, y)[2:]
    m_ld, v_ld, bm, bv = BM.predict_ld(samples, Xt, *stats)
    err_m = np.abs(mu - m_ld)
    err_v = np.abs(var - v_ld)
    assert np.all(err_m <= bm) and np.all(err_v <= bv), (np.max(err_m / bm), np.max(err_v / bv))
    m64, v64, bm64, bv64 = (a.astype(np.float64) for a in (m_ld, v_ld, bm, bv))
    eta = float(np.min(y))
    for kind in (_lib.ACQ_EI, _lib.ACQ_LOG_EI, _lib.ACQ_PI, _lib.ACQ_LCB):
        r = h.acq(Xt, kind, eta if kind != _lib.ACQ_LCB else 0.0, 0.0)
        lo, hi = _acq_interval(m64, v64, bm64, bv64, kind, eta if kind != _lib.ACQ_LCB else 0.0, 0.0)
        tol = 1e-12 * np.maximum(np.abs(lo), np.abs(hi)) + 1e-300
        ok = (r["values"] >= lo - tol) & (r["values"] <= hi + tol)
        assert np.all(ok | ~np.isfinite(lo)), kind
        b = r["best_idx"]
        assert r["values"][b] == np.max(r["values"]) and b == int(np.argmax(r["values"]))
        assert hi[b] + tol[b] >= np.max(lo)                      # the arg-max equals the true one within the bound


def test_many_candidates_beyond_one_chunk():
    X, y = _data(25, 3, 4)
    h, S, _ = _device_chain(X, y, 9, 0, 50, 350, 30)
    Xt = np.random.RandomState(1).rand(70001, 3)
    r = h.acq(Xt, _lib.ACQ_EI, float(y.min()), 0.0, want_moments=True)
    for lo in (0, 65535, 70000):
        mu, var = h.predict(Xt[lo:lo + 1])
        assert abs(mu[0] - r["mu"][lo]) <= 1e-13 * abs(mu[0]) + 1e-15 and abs(var[0] - r["var"][lo]) <= 1e-13 * var[0]
    assert r["best_idx"] == int(np.argmax(r["values"])) and r["n_negative"] == 0


def test_model_train_copy_and_pickle():
    X, y = _data(12, 2, 5)
    m = WrapperBohamiann(rng=np.random.RandomState(3))
    m.train(X, y)
    assert m.samples.shape == (99, BM.n_params(2)) and m.counter == 1
    Xt = np.random.RandomState(6).rand(300, 2)
    mu, v = m.predict(Xt)
    assert np.all(np.isfinite(mu)) and np.all(v > 0)
    for c in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        mu2, v2 = c.predict(Xt)
        assert np.array_equal(mu, mu2) and np.array_equal(v, v2)


def _trained(d=2, n=15):
    X, y = _data(n, d, 11 + d)
    m = WrapperBohamiann(rng=np.random.RandomState(2))
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


def test_fit_at_the_wrapper_settings_on_sinc():
    # the reference test's problem (test_wrapper_bohamiann.py: 10 rows in [0, 1]^2, sum of sinc(10 x - 5)); held-out RMSE
    # of the predictive mean on 500 rows.  Ten rows pin this surface loosely: the torch host restatement of pybnn's loop
    # (bnn_model.torch_train, float64, CPU) at the same settings gives 0.456, 0.656 and 2.99 for seeds 1, 2 and 3, against
    # 0.437 for the constant prediction y.mean().  The threshold 3.5 is the worst of those plus a margin of 0.5: it
    # catches a chain that diverges or a predictive pass that is off in scale, not a fit that is merely unlucky.  The
    # device run below (seed drawn from RandomState(4)) gave 0.570 on an H100, a margin of 2.93.
    rng = np.random.RandomState(0)
    X = rng.rand(10, 2)
    y = np.sinc(X * 10 - 5).sum(axis=1)
    Xt = np.random.RandomState(1).rand(500, 2)
    yt = np.sinc(Xt * 10 - 5).sum(axis=1)
    m = WrapperBohamiann(rng=np.random.RandomState(4))
    m.train(X, y)
    mu, v = m.predict(Xt)
    rmse = float(np.sqrt(np.mean((mu - yt) ** 2)))
    print("held-out RMSE %.4f" % rmse)
    assert rmse < 3.5
    inc, inc_val = m.get_incumbent()
    assert np.array_equal(inc, X[np.argmin(y)])


def test_refusals_and_limits():
    X, y = _data(30, 2, 8)
    h = _lib.Handle(0)
    with pytest.raises(ValueError, match="gpk_bnn_set_data has not been called"):
        _lib.bnn_train(h, 1, 0, 1e-2, 0.05, 1e-10, 0, 10, 1, 20)
    with pytest.raises(ValueError, match="n >= 2"):
        _lib.bnn_set_data(h, X[:1], y[:1])
    with pytest.raises(ValueError, match="constant"):
        _lib.bnn_set_data(h, np.c_[X, np.ones(30)], y)
    with pytest.raises(ValueError, match="constant"):
        _lib.bnn_set_data(h, X, np.ones(30))
    with pytest.raises(ValueError, match="GPK_BNN_MAX_N = 4096"):
        _lib.bnn_set_data(h, np.random.rand(_lib.BNN_MAX_N + 1, 1), np.random.rand(_lib.BNN_MAX_N + 1))
    with pytest.raises(ValueError, match="GPK_BNN_MAX_D = 64"):
        _lib.bnn_set_data(h, np.random.rand(3, 65), np.random.rand(3))
    _lib.bnn_set_data(h, X, y)
    with pytest.raises(RuntimeError, match="not trained"):
        h.predict(X[:3])
    with pytest.raises(ValueError, match="GPK_BNN_MAX_BATCH"):
        _lib.bnn_train(h, 1, 0, 1e-2, 0.05, 1e-10, 0, 10, 1, 33)
    with pytest.raises(ValueError, match="keeps no network"):
        _lib.bnn_train(h, 1, 0, 1e-2, 0.05, 1e-10, 10, 11, 1, 20)
    _lib.bnn_train(h, 1, 0, 1e-2, 0.05, 1e-10, 0, 10, 1, 20)
    for call in (lambda: h.set_data(X, y), lambda: h.set_kernel(0, 0.0, [0], [0], [0.0]), lambda: h.fit(1e-6, 0.0),
                 lambda: h.predict_grad(X[:3]), lambda: h.predict_cov(X[:3]),
                 lambda: _lib.hyper_lnpost(h, np.zeros((1, 3))), lambda: _lib.es_multi([h], X[:3]),
                 lambda: _lib.blr_set_data(h, X, y, _lib.BLR_LINEAR, (0.1, -10.0, 0.1)),
                 lambda: _lib.blr_lnpost(h, np.zeros((1, 2))), lambda: _lib.rf_set_data(h, X, y),
                 lambda: _lib.rf_fit(h, 1, 0, 3, 0, True, True)):
        with pytest.raises(ValueError, match="Bayesian neural network"):
            call()
    gp = _lib.Handle(0)
    gp.set_data(X, y)
    with pytest.raises(ValueError, match="Gaussian-process model"):
        _lib.bnn_set_data(gp, X, y)
    blr = _lib.Handle(0)
    _lib.blr_set_data(blr, X, y, _lib.BLR_LINEAR, (0.1, -10.0, 0.1))
    with pytest.raises(ValueError, match="Bayesian linear regression"):
        _lib.bnn_set_data(blr, X, y)
    rf = _lib.Handle(0)
    _lib.rf_set_data(rf, X, y)
    with pytest.raises(ValueError, match="random forest"):
        _lib.bnn_set_data(rf, X, y)
    with pytest.raises(ValueError, match="random forest"):
        _lib.bnn_dims(rf)
