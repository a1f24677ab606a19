"""Numpy stand-in for the Bayesian-neural-network entry points of robo_b200._lib — TEST INFRASTRUCTURE ONLY.

The normalisation and the predictive moments are tests/bnn_model.py's; the chain is replaced by networks drawn from a
numpy stream keyed by (seed, counter) around bnn_model's initialisation, with the number of networks the chain keeps.
That is enough for the wrapper's plumbing (shapes, rng use, pickling, dispatch), which is what the CPU suite drives with
it; the chain itself is pinned on the device against bnn_model.chain.  Argument checks mirror the C side's GPK_BAD_ARG
cases as ValueError.  Acquisition closed forms are gpk_acq_moments' (through fake_blr.moments)."""
import numpy as np

from robo_b200 import _lib
from tests import bnn_model as BM
from tests import fake_blr


class FakeBnnHandle(object):
    def __init__(self, device=0):
        self.device = device
        self.stats = None
        self.samples = None
        self.train_calls = []

    def close(self):
        pass

    def predict(self, Xs):
        if self.samples is None:
            raise RuntimeError("model is not trained (gpk_bnn_train)")
        return BM.predict_samples(self.samples, np.asarray(Xs, dtype=np.float64), *self.stats)

    def acq(self, Xs, kind, eta=0.0, par=0.0, want_values=True, want_moments=False):
        m, v = self.predict(Xs)
        vals, nn = fake_blr.moments(m, v, kind, eta, par)
        vals = np.asarray(vals, dtype=np.float64)
        return dict(values=vals, mu=m, var=v, best_val=float(vals.max()), best_idx=int(np.argmax(vals)), n_negative=nn)

    def generate_candidates(self, seed, first, count, n_uniform, lower, upper, incumbent, scale):
        """A stand-in generator: uniform rows from a numpy stream keyed by seed (not the device's Philox rows)."""
        lo, up = np.asarray(lower, dtype=np.float64), np.asarray(upper, dtype=np.float64)
        r = np.random.RandomState(int(seed) % (2 ** 32)).rand(first + count, lo.size)
        return (lo + (up - lo) * r)[first:]

    def maximize_random(self, seed, first, count, n_uniform, lower, upper, incumbent, scale, kind, eta=0.0, par=0.0):
        X = self.generate_candidates(seed, first, count, n_uniform, lower, upper, incumbent, scale)
        r = self.acq(X, kind, eta, par)
        return X[r["best_idx"]], r["best_val"], first + r["best_idx"]


def bnn_set_data(handle, X, y):
    X, y = np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64).ravel()
    if X.shape[0] > _lib.BNN_MAX_N:
        raise ValueError("gpk_bnn_set_data: n exceeds GPK_BNN_MAX_N = %d" % _lib.BNN_MAX_N)
    if X.shape[1] > _lib.BNN_MAX_D:
        raise ValueError("gpk_bnn_set_data: d exceeds GPK_BNN_MAX_D = %d" % _lib.BNN_MAX_D)
    if not (np.isfinite(X).all() and np.isfinite(y).all()):
        raise ValueError("gpk_bnn_set_data: X and y must be finite")
    Xs, ys, xm, xs, ym, ysd = BM.normalise(X, y)
    handle.D, handle.stats, handle.samples = X.shape[1], (xm, xs, ym, ysd), None


def bnn_train(handle, seed, counter, lr, mdecay, eps, burn_in, num_steps, keep_every, batch):
    if handle.stats is None:
        raise ValueError("gpk_bnn_train: gpk_bnn_set_data has not been called")
    if not 1 <= batch <= _lib.BNN_MAX_BATCH or keep_every < 1 or burn_in < 0 or num_steps < 1:
        raise ValueError("gpk_bnn_train: bad arguments")
    S = BM.n_kept(burn_in, num_steps, keep_every)
    if S < 1:
        raise ValueError("gpk_bnn_train: the chain keeps no network")
    handle.train_calls.append((int(seed), int(counter), float(lr), int(burn_in), int(num_steps)))
    rs = np.random.RandomState([int(seed) % (2 ** 32), int(counter)])
    P = BM.n_params(handle.D)
    base = BM.init_theta(handle.D, rs.randn(P))
    handle.samples = base + 0.05 * rs.randn(S, P)


def bnn_samples(handle):
    return handle.samples.copy()


def bnn_set_samples(handle, samples):
    handle.samples = np.array(samples, dtype=np.float64)


def install(monkeypatch):
    """Route robo_b200's BNN entry points and handles through the numpy stand-ins for the duration of a test."""
    pool = {}

    def moments_handle(device=0):
        return pool.setdefault(device, fake_blr._MomentsHandle())
    monkeypatch.setattr(_lib, "Handle", FakeBnnHandle)
    monkeypatch.setattr(_lib, "moments_handle", moments_handle)
    for name in ("bnn_set_data", "bnn_train", "bnn_samples", "bnn_set_samples"):
        monkeypatch.setattr(_lib, name, globals()[name])
    return FakeBnnHandle
