"""WrapperBohamiann's host layer and the network restatement tests/bnn_model.py, without a GPU: the loss gradient against
torch.autograd on the reference's network structure, the SGHMC update against its torch restatement, the batch schedule,
the keep rule, the fixed tanh / exp, the reference's contracts, pickling and the device dispatch on the numpy stand-in
of the device entry points (tests/fake_bnn.py)."""
import copy
import os
import pickle

import numpy as np
import pytest

from robo_b200 import _lib
from robo_b200.models import WrapperBohamiann
from robo_b200.models.wrapper_bohamiann import get_default_network
from tests import bnn_model as BM
from tests import fake_bnn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
torch = pytest.importorskip("torch")


@pytest.fixture
def fake(monkeypatch):
    return fake_bnn.install(monkeypatch)


def _sinc(N, D, seed):
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    return X, np.sinc(X * 10 - 5).sum(axis=1)


def _theta(D, seed):
    """A network away from its initialisation: initial weights plus noise, and a non-default lv."""
    rng = np.random.RandomState(seed)
    th = BM.init_theta(D, rng.randn(BM.n_params(D))) + 0.3 * rng.randn(BM.n_params(D))
    th[BM.layout(D)["lv"]] = -1.7
    return th


def test_header_constants_match_the_binding():
    src = open(os.path.join(ROOT, "include", "gpk.h")).read()
    for name, v in (("N", _lib.BNN_MAX_N), ("D", _lib.BNN_MAX_D), ("BATCH", _lib.BNN_MAX_BATCH)):
        assert "#define GPK_BNN_MAX_%s %d " % (name, v) in src
    cuh = open(os.path.join(ROOT, "robo_b200", "csrc", "gpk_bnn.cuh")).read()
    assert "GPK_BNN_TAG_NOISE 0x%08Xu" % BM.TAG_NOISE in cuh and "GPK_BNN_TAG_ORDER 0x%08Xu" % BM.TAG_ORDER in cuh
    assert "GPK_BNN_LOG_LV0 %r " % BM.LOG_LV0 in cuh and "GPK_BNN_LOG_1EM6 %r " % BM.LOG_1EM6 in cuh
    assert BM.LOG_LV0 == np.log(1e-2) and BM.LOG_1EM6 == np.log(1e-6)


def test_parameter_count_and_layout_follow_the_reference_network():
    for D in (1, 2, 8, 64):
        net = get_default_network(D)
        assert sum(p.numel() for p in net.parameters()) == BM.n_params(D) == _lib.bnn_params(D) == 50 * D + 2652
        assert net[5].bias.item() == np.log(1e-2)
        assert net[0].bias.abs().max().item() == 0.0


@pytest.mark.parametrize("D,N,Bt", [(1, 7, 7), (2, 30, 20), (2, 30, 10), (8, 200, 20), (64, 45, 5)])
def test_gradient_equals_torch_autograd(D, N, Bt):
    rng = np.random.RandomState(D + N)
    th = _theta(D, D * 7 + Bt)
    xb, yb = rng.randn(Bt, D), rng.randn(Bt)
    g = BM.grad(th, xb, yb, N)
    gt = BM.torch_grad(th, xb, yb, N)
    err = np.max(np.abs(g - gt)) / np.max(np.abs(gt))
    print("D=%d N=%d B_t=%d: max |G - autograd| / max |autograd| = %.2e" % (D, N, Bt, err))
    assert err <= 1e-12
    L = BM.layout(D)
    for k in ("W1", "b1", "W2", "b2", "W3"):               # blockwise, so no small block hides behind a big one
        assert np.max(np.abs(g[L[k]] - gt[L[k]])) <= 1e-12 * max(np.max(np.abs(gt[L[k]])), 1e-300)
    assert abs(g[L["lv"]] - gt[L["lv"]]) <= 1e-12 * abs(gt[L["lv"]])


def test_sghmc_steps_equal_the_torch_update():
    D, N = 2, 30
    rng = np.random.RandomState(5)
    X, y = rng.randn(N, D), rng.randn(N)
    P = BM.n_params(D)
    th = BM.init_theta(D, rng.randn(P))
    st = dict(p=np.zeros(P), tau=np.ones(P), g=np.ones(P), vhat=np.ones(P))
    pt = torch.as_tensor(th.copy())
    stt = {k: torch.as_tensor(v.copy()) for k, v in st.items()}
    cache = {}
    for s in range(6):
        rows = BM.batch_rows(9, 1, s, N, 20, cache)
        G = BM.grad(th, X[rows], y[rows], N)
        xi = rng.randn(P)
        adapt = s + 1 <= 3                                  # the adaptation cut-over inside the window
        th = BM.step(th, st, G, xi, adapt)
        BM.torch_step(pt, torch.as_tensor(G), stt, torch.as_tensor(xi), adapt)
        for k in ("p", "tau", "g", "vhat"):
            ref = stt[k].numpy()
            np.testing.assert_allclose(st[k], ref, rtol=1e-13, atol=1e-13 * np.max(np.abs(ref)))
        np.testing.assert_allclose(th, pt.numpy(), rtol=1e-13, atol=1e-15)
    assert np.all(st["tau"] > 1.0)


@pytest.mark.parametrize("N", [1, 7, 19, 20, 21, 45])
def test_batch_schedule(N):
    B = 20
    nb = (N + B - 1) // B
    cache = {}
    for e in range(3):
        order = BM.epoch_order(3, 2, e, N)
        assert sorted(order.tolist()) == list(range(N))
        seen = []
        for b in range(nb):
            rows = BM.batch_rows(3, 2, e * nb + b, N, B, cache)
            assert len(rows) == (B if b < nb - 1 else N - B * (nb - 1))     # the last batch of an epoch is partial
            seen += rows.tolist()
        assert seen == order.tolist()                        # the epoch ends after its partial batch
    if N > 2:
        assert not np.array_equal(BM.epoch_order(3, 2, 0, N), BM.epoch_order(3, 2, 1, N))
        assert not np.array_equal(BM.epoch_order(3, 2, 0, N), BM.epoch_order(3, 3, 0, N))


def test_keep_rule_keeps_99_networks_at_the_wrapper_settings():
    burn_in, num_steps = 100 * 30, 100 * 30 + 10000
    kept = [s for s in range(num_steps) if BM.kept(s, burn_in, BM.KEEP_EVERY)]
    assert len(kept) == 99 == BM.n_kept(burn_in, num_steps, BM.KEEP_EVERY)
    assert kept[0] == burn_in + 100 and kept[-1] == burn_in + 9900
    assert BM.n_kept(0, 1, 1) == 0 and BM.n_kept(0, 2, 1) == 1 and BM.n_kept(5, 20, 7) == 2


def test_fixed_tanh_and_exp_against_numpy():
    x = np.concatenate([np.linspace(-40, 40, 200001), np.geomspace(1e-300, 1e-2, 2000), -np.geomspace(1e-12, 5, 2000),
                        [0.0, -0.0, 0.00390625, np.nextafter(0.00390625, 0)]])
    t = BM.tanh(x)
    ref = np.tanh(x.astype(np.longdouble))
    abs_err = np.max(np.abs(t - ref))
    nz = ref != 0
    rel_err = np.max(np.abs((t[nz] - ref[nz]) / ref[nz]))
    print("fixed tanh: max abs error %.2e, max rel error %.2e" % (abs_err, rel_err))
    assert abs_err <= 4e-16 and rel_err <= 2e-14
    assert np.all(np.abs(t) <= 1.0) and np.array_equal(np.sign(t), np.sign(x)) and np.isnan(BM.tanh(np.nan))
    xe = np.linspace(-30, 5, 100001)
    e = BM.exp(xe)
    rel = np.max(np.abs(e - np.exp(xe.astype(np.longdouble))) / np.exp(xe.astype(np.longdouble)))
    print("fixed exp: max rel error %.2e" % rel)
    assert rel <= 4e-16


def test_normalisation_and_its_refusals():
    X, y = _sinc(10, 2, 0)
    Xs, ys, xm, xs, ym, ysd = BM.normalise(X, y)
    np.testing.assert_allclose(Xs.mean(axis=0), 0, atol=1e-15)
    np.testing.assert_allclose(Xs.std(axis=0), 1, rtol=1e-14)
    np.testing.assert_allclose([ym, ysd], [y.mean(), y.std()], rtol=1e-14)
    for bad in ((X[:1], y[:1]), (np.c_[X, np.ones(10)], y), (X, np.full(10, 2.0))):
        with pytest.raises(ValueError):
            BM.normalise(*bad)


def test_reference_contracts(fake):
    X, y = _sinc(10, 2, 1)
    m = WrapperBohamiann(rng=np.random.RandomState(0))
    m.train(X, y)
    Xt = np.random.RandomState(2).rand(10, 2)
    mu, v = m.predict(Xt)
    assert mu.shape == (10,) and v.shape == (10,) and np.all(v > 0)
    inc, inc_val = m.get_incumbent()
    b = np.argmin(y)
    np.testing.assert_almost_equal(inc, X[b], decimal=5)
    assert inc_val == y[b]
    h = m._handle
    assert m.samples.shape == (99, BM.n_params(2))
    assert h.train_calls[-1][3:] == (1000, 11000)         # burn_in = 100 N, num_steps = 100 N + 10,000


def test_rng_and_counter(fake):
    a = WrapperBohamiann(rng=np.random.RandomState(7))
    b = WrapperBohamiann(rng=np.random.RandomState(7))
    assert a.seed == b.seed == np.random.RandomState(7).randint(2 ** 31 - 1)
    X, y = _sinc(12, 1, 3)
    a.train(X, y)
    a.train(X, y)
    assert [c[1] for c in a._handle.train_calls] == [0, 1]
    assert a._handle.train_calls[0][0] == a.seed


def test_argument_errors():
    with pytest.raises(TypeError):
        WrapperBohamiann(get_net=lambda d: None)
    with pytest.raises(ValueError):
        WrapperBohamiann(use_double_precision=False)
    with pytest.raises(ValueError):
        WrapperBohamiann().predict(np.zeros((1, 2)))


def test_pickle_and_deepcopy_predict_bit_identically(fake):
    X, y = _sinc(15, 3, 4)
    m = WrapperBohamiann(rng=np.random.RandomState(1))
    m.train(X, y)
    Xt = np.random.RandomState(5).rand(40, 3)
    mu, v = m.predict(Xt)
    for c in (pickle.loads(pickle.dumps(m)), copy.deepcopy(m)):
        assert c._handle is None
        mu2, v2 = c.predict(Xt)
        assert np.array_equal(mu, mu2) and np.array_equal(v, v2)
        assert c.seed == m.seed and c.counter == m.counter


def test_device_spec_and_random_sampling_dispatch(fake):
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    from robo_b200.maximizers import DeviceRandomSampling
    from robo_b200.maximizers.device_spec import device_spec
    X, y = _sinc(20, 2, 13)
    m = WrapperBohamiann(rng=np.random.RandomState(0))
    m.train(X, y)
    for cls, kind in ((EI, "ei"), (LogEI, "log_ei"), (PI, "pi"), (LCB, "lcb")):
        which, (k, etas, par, hs) = device_spec(cls(m), "test")
        assert which == "acq" and k == kind and hs == [m._handle]
        assert etas == [0.0 if kind == "lcb" else float(np.min(y))]
    x = DeviceRandomSampling(EI(m), np.zeros(2), np.ones(2), n_samples=40, rng=np.random.RandomState(1)).maximize()
    assert x.shape == (2,) and np.all((0 <= x) & (x <= 1))
    with pytest.raises(ValueError, match="one GPU"):
        DeviceRandomSampling(EI(m), np.zeros(2), np.ones(2), world=2, rank=0).maximize()


def test_facade_still_refuses_bohamiann():
    from robo_b200 import compat
    assert "pybnn" in open(compat.__file__).read()
