"""DNGO's host layer and the training restatement tests/dngo_model.py, without a GPU: the loss gradient against
torch.autograd on the same fp64 network, Adam against torch.optim.Adam, the initialisation, the epoch schedule, the
normalisation flags, and the model's signature, refusals, rng and counter use, copies and device dispatch on the numpy
stand-in of the device entry points (tests/fake_dngo.py)."""
import copy
import os
import pickle

import numpy as np
import pytest

from robo_b200 import _lib
from robo_b200.models import DNGO
from tests import dngo_model as DM
from tests import fake_dngo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
torch = pytest.importorskip("torch")

SMALL = dict(num_epochs=3, chain_length=4, burnin_steps=3, n_hypers=4)


@pytest.fixture
def fake(monkeypatch):
    return fake_dngo.install(monkeypatch)


def _branin(N, seed):
    rng = np.random.RandomState(seed)
    X = rng.rand(N, 2) * [15, 15] - [5, 0]
    x1, x2 = X[:, 0], X[:, 1]
    y = (x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x1) + 10
    return X, y


def _theta(D, seed):
    """A net away from its initialisation."""
    rng = np.random.RandomState(seed)
    return DM.init_theta(D, seed, 0) + 0.3 * rng.randn(DM.n_params(D))


def test_header_constants_match_the_binding():
    src = open(os.path.join(ROOT, "include", "gpk.h")).read()
    for name, v in (("N", _lib.DNGO_MAX_N), ("D", _lib.DNGO_MAX_D), ("BATCH", _lib.DNGO_MAX_BATCH)):
        assert "#define GPK_DNGO_MAX_%s %d " % (name, v) in src
    cuh = open(os.path.join(ROOT, "robo_b200", "csrc", "gpk_dngo.cuh")).read()
    assert "GPK_DNGO_TAG_INIT 0x%08Xu" % DM.TAG_INIT in cuh and "GPK_DNGO_TAG_ORDER 0x%08Xu" % DM.TAG_ORDER in cuh
    assert "#define GPK_DNGO_H %d " % DM.H in cuh and DM.H == _lib.DNGO_H


def test_parameter_count_and_layout_follow_the_network():
    for D in (1, 2, 8, 64):
        net = DM.torch_net(D)
        assert sum(p.numel() for p in net.parameters()) == DM.n_params(D) == _lib.dngo_params(D) == 50 * D + 5201
        th = _theta(D, D)
        assert np.array_equal(DM.torch_flat(DM.torch_net(D, th)), th)
        L = DM.layout(D)
        assert L["b4"] == DM.n_params(D) - 1 and L["W4"].stop - L["W4"].start == 50


def test_initialisation_is_torch_linear_default_bounds():
    D = 3
    th = DM.init_theta(D, 11, 2)
    L = DM.layout(D)
    for k, fan in (("W1", D), ("b1", D), ("W2", 50), ("b2", 50), ("W3", 50), ("b3", 50), ("W4", 50)):
        v = th[L[k]]
        b = 1.0 / np.sqrt(fan)
        assert np.all(np.abs(v) <= b) and np.max(np.abs(v)) > 0.8 * b, k
    assert abs(th[L["b4"]]) <= 1 / np.sqrt(50)
    assert abs(th.mean()) < 0.01
    assert not np.array_equal(th, DM.init_theta(D, 11, 3)) and not np.array_equal(th, DM.init_theta(D, 12, 2))


@pytest.mark.parametrize("D,B", [(1, 1), (2, 10), (8, 16), (64, 5)])
def test_gradient_equals_torch_autograd(D, B):
    rng = np.random.RandomState(D + B)
    th = _theta(D, D * 7 + B)
    xb, yb = rng.randn(B, D), rng.randn(B)
    g = DM.grad(th, xb, yb)
    gt = DM.torch_grad(th, xb, yb)
    err = np.max(np.abs(g - gt)) / np.max(np.abs(gt))
    L = DM.layout(D)
    worst = 0.0
    for k in ("W1", "b1", "W2", "b2", "W3", "b3", "W4", "b4"):      # blockwise, so no small block hides behind a big one
        scale = max(np.max(np.abs(gt[L[k]])), 1e-300)
        worst = max(worst, np.max(np.abs(g[L[k]] - gt[L[k]])) / scale)
    print("D=%d B=%d: |G - autograd| / max |autograd| = %.2e overall, %.2e in the worst block" % (D, B, err, worst))
    # the fixed tanh (gpk_bnn_tanh) is within 2e-14 relative of torch's, and three layers carry its error back
    assert err <= 1e-14 and worst <= 1e-13


def test_adam_steps_equal_torch_optim_adam():
    D, N, B, lr = 2, 30, 10, 0.01
    rng = np.random.RandomState(5)
    X, y = rng.randn(N, D), rng.randn(N)
    th = DM.init_theta(D, 9, 1)
    st = DM.adam_state(len(th))
    net = DM.torch_net(D, th)
    opt = torch.optim.Adam(net.parameters(), lr=lr, foreach=False)
    for e in range(2):
        for rows in DM.batches(9, 1, e, N, B):
            G = DM.grad(th, X[rows], y[rows])
            th = DM.adam(th, st, G, lr)
            off = 0                                          # torch's update on the same gradient
            for p in net.parameters():
                p.grad = torch.as_tensor(G[off:off + p.numel()].reshape(p.shape).copy())
                off += p.numel()
            opt.step()
    tt = DM.torch_flat(net)
    assert st["t"] == 6
    err = np.max(np.abs(th - tt)) / np.max(np.abs(tt))
    print("6 Adam steps: max |theta - torch| / max |theta| = %.2e" % err)
    assert err <= 1e-15
    ms = [opt.state[p]["exp_avg"].ravel() for p in net.parameters()]
    vs = [opt.state[p]["exp_avg_sq"].ravel() for p in net.parameters()]
    m_t, v_t = torch.cat(ms).numpy(), torch.cat(vs).numpy()
    assert np.max(np.abs(st["m"] - m_t)) <= 1e-14 * np.max(np.abs(m_t))
    assert np.max(np.abs(st["v"] - v_t)) <= 1e-14 * np.max(np.abs(v_t))


@pytest.mark.parametrize("N,B", [(3, 10), (10, 10), (23, 10), (40, 16)])
def test_epoch_schedule_drops_the_remainder(N, B):
    Bt = min(B, N)
    for e in range(3):
        order = DM.epoch_order(3, 2, e, N)
        assert sorted(order.tolist()) == list(range(N))
        bs = DM.batches(3, 2, e, N, Bt)
        assert len(bs) == N // Bt and all(len(b) == Bt for b in bs)
        assert np.concatenate(bs).tolist() == order[:(N // Bt) * Bt].tolist()
    if N > 2:
        assert not np.array_equal(DM.epoch_order(3, 2, 0, N), DM.epoch_order(3, 2, 1, N))


def test_training_restatement_follows_the_torch_loop():
    # the bit-for-bit restatement and pybnn's loop in torch differ in their draws only: both fit the training set
    X, y = _branin(30, 0)
    th, st, Theta = DM.train(*DM.normalise(X, y)[:2], 5, 0, epochs=60)
    tt, Theta_t, stats = DM.torch_train(X, y, 5, epochs=60)
    Xs, ys = DM.normalise(X, y)[:2]
    for w in (th, tt):
        f = DM.forward(w, Xs)[3]
        assert np.mean((f - ys) ** 2) < 0.2
    assert st["t"] == 60 * 3 and Theta.shape == Theta_t.shape == (30, 50)


def test_normalisation_flags_and_refusals():
    X, y = _branin(10, 1)
    Xs, ys, xm, xs, ym, ysd = DM.normalise(X, y)
    np.testing.assert_allclose(Xs.mean(axis=0), 0, atol=1e-15)
    np.testing.assert_allclose([ym, ysd], [y.mean(), y.std()], rtol=1e-14)
    Xs, ys, xm, xs, ym, ysd = DM.normalise(X, y, False, False)
    assert np.array_equal(Xs, X) and np.array_equal(ys, y) and (ym, ysd) == (0.0, 1.0)
    assert np.array_equal(DM.normalise(X, y, True, False)[1], y)
    assert np.array_equal(DM.normalise(X, y, False, True)[0], X)
    DM.normalise(X[:1], y[:1], False, False)
    for bad in ((X[:1], y[:1]), (np.c_[X, np.ones(10)], y), (X, np.full(10, 2.0))):
        with pytest.raises(ValueError):
            DM.normalise(*bad)
    DM.normalise(np.c_[X, np.ones(10)], y, False, True)


def test_signature_and_argument_errors():
    import inspect
    params = list(inspect.signature(DNGO.__init__).parameters.items())[1:]
    assert [(k, p.default) for k, p in params] == [
        ("batch_size", 10), ("num_epochs", 500), ("learning_rate", 0.01), ("adapt_epoch", 5000), ("n_units_1", 50),
        ("n_units_2", 50), ("n_units_3", 50), ("alpha", 1.0), ("beta", 1000), ("prior", None), ("do_mcmc", True),
        ("n_hypers", 20), ("chain_length", 2000), ("burnin_steps", 2000), ("normalize_input", True),
        ("normalize_output", True), ("rng", None), ("device", 0)]
    for k in ("n_units_1", "n_units_2", "n_units_3"):
        with pytest.raises(ValueError, match="50"):
            DNGO(**{k: 100})
    from robo_b200 import priors
    with pytest.raises(TypeError):
        DNGO(prior=priors.TophatPrior(-1, 1))
    with pytest.raises(ValueError, match="train"):
        DNGO().predict(np.zeros((1, 2)))


def test_train_predict_and_attributes(fake):
    X, y = _branin(20, 2)
    m = DNGO(rng=np.random.RandomState(0), **SMALL)
    m.train(X, y)
    assert m.X is X or np.array_equal(m.X, X)
    assert m.Theta.shape == (20, 50) and m.burned and m.p0.shape == (4, 2) and len(m.models) == 4
    assert np.array_equal(m.hypers, np.exp(m.p0))
    h = m._handle
    assert [c[1] for c in h.sample_calls] == [3, 4]              # burn-in on the first train, then the chain
    assert h.train_calls == [(m.seed, 0, 0.01, 10, 3)]
    mu, v = m.predict(np.random.RandomState(1).rand(7, 2))
    assert mu.shape == (7,) and np.all(v > 0)
    inc, inc_val = m.get_incumbent()
    assert np.array_equal(inc, X[np.argmin(y)]) and inc_val == y.min()
    m.train(X, y)
    assert [c[1] for c in h.sample_calls] == [3, 4, 4] and [c[1] for c in h.train_calls] == [0, 1]
    m2 = DNGO(rng=np.random.RandomState(0), do_mcmc=False, **SMALL)
    m2.train(X, y)
    assert np.shape(m2.hypers) == (1, 2) and not m2._handle.sample_calls
    m3 = DNGO(rng=np.random.RandomState(0), alpha=2.0, beta=30.0, **SMALL)
    m3.train(X, y, do_optimize=False)
    assert m3.hypers == [[2.0, 30.0]] and not m3.burned


def test_adapt_epoch_has_no_effect(fake):
    X, y = _branin(12, 3)
    a = DNGO(rng=np.random.RandomState(4), adapt_epoch=1, **SMALL)
    b = DNGO(rng=np.random.RandomState(4), **SMALL)
    a.train(X, y)
    b.train(X, y)
    assert np.array_equal(a.net, b.net) and np.array_equal(a.hypers, b.hypers)


def test_rng_seeds_the_streams_and_each_train_advances_the_counter(fake):
    a = DNGO(rng=np.random.RandomState(7), **SMALL)
    b = DNGO(rng=np.random.RandomState(7), **SMALL)
    assert a.seed == b.seed == np.random.RandomState(7).randint(2 ** 31 - 1)
    X, y = _branin(12, 3)
    a.train(X, y)
    net0 = a.net.copy()
    a.train(X, y)
    assert a.counter == 2 and [c[1] for c in a._handle.train_calls] == [0, 1]
    assert not np.array_equal(net0, a.net)


def test_flags_reach_the_device(fake):
    X, y = _branin(12, 5)
    m = DNGO(rng=np.random.RandomState(1), normalize_input=False, normalize_output=False, **SMALL)
    m.train(X, y)
    Xs, ys, xm, xs, ym, ysd = m._handle.data
    assert np.array_equal(Xs, X) and np.array_equal(ys, y)


def test_pickle_and_deepcopy_predict_bit_identically(fake):
    X, y = _branin(15, 4)
    m = DNGO(rng=np.random.RandomState(1), **SMALL)
    m.train(X, y)
    Xt = np.random.RandomState(5).rand(40, 2)
    mu, v = m.predict(Xt)
    for c in (pickle.loads(pickle.dumps(m)), copy.deepcopy(m)):
        assert c._handle is None
        mu2, v2 = c.predict(Xt)
        assert np.array_equal(mu, mu2) and np.array_equal(v, v2)
        assert c.seed == m.seed and c.counter == m.counter


def test_device_spec_and_random_sampling_dispatch(fake):
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    from robo_b200.maximizers import DeviceRandomSampling
    from robo_b200.maximizers.device_spec import DEVICE_SURROGATES, device_spec
    assert DNGO in DEVICE_SURROGATES
    X, y = _branin(20, 13)
    m = DNGO(rng=np.random.RandomState(0), **SMALL)
    m.train(X, y)
    for cls, kind in ((EI, "ei"), (LogEI, "log_ei"), (PI, "pi"), (LCB, "lcb")):
        which, (k, etas, par, hs) = device_spec(cls(m), "test")
        assert which == "acq" and k == kind and hs == [m._handle]
        assert etas == [0.0 if kind == "lcb" else float(np.min(y))]
    x = DeviceRandomSampling(EI(m), np.zeros(2), np.ones(2), n_samples=40, rng=np.random.RandomState(1)).maximize()
    assert x.shape == (2,) and np.all((0 <= x) & (x <= 1))
    with pytest.raises(ValueError, match="DNGO runs on one GPU"):
        DeviceRandomSampling(EI(m), np.zeros(2), np.ones(2), world=2, rank=0).maximize()


def test_facade_and_pybnn_stubs_stay_as_they_were():
    from robo_b200 import compat
    assert "pybnn" in open(compat.__file__).read()
