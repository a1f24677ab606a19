"""Numpy stand-in for the DNGO entry points of robo_b200._lib — TEST INFRASTRUCTURE ONLY.

The normalisation, the training and the features are tests/dngo_model.py's (the restatement the device equals bit for
bit); the regression over the features is tests/blr_model.py's host arithmetic (its log-posterior, the sampler run
keyed like gpk_blr_sample, the reference's (m, S) loop); predict evaluates the mixture's mean and full variance per
hyper-sample in float64.  That is enough for DNGO's host layer (signature, refusals, rng and counter use, copies,
dispatch), which is what the CPU suite drives with it.  Argument checks mirror the C side's GPK_BAD_ARG cases as
ValueError.  Acquisition closed forms are gpk_acq_moments' (through fake_blr.moments)."""
import numpy as np

from robo_b200 import _lib
from tests import blr_model as LM
from tests import dngo_model as DM
from tests import fake_blr


class FakeDngoHandle(object):
    def __init__(self, device=0):
        self.device = device
        self.data = None
        self.net = None
        self.fit = None
        self.train_calls = []
        self.sample_calls = []

    def close(self):
        pass

    def predict(self, X):
        if self.fit is None:
            raise RuntimeError("model is not fitted (gpk_dngo_fit)")
        Xs, ys, xm, xs, ym, ysd = self.data
        phi = DM.features(self.net, (np.asarray(X, dtype=np.float64) - xm) / xs)
        hypers, models = self.fit
        mu = np.array([phi @ m for m, _ in models])
        var = np.array([1.0 / b + np.einsum("rj,jl,rl->r", phi, S, phi) for (_, b), (_, S) in zip(hypers, models)])
        m = mu.mean(axis=0)
        v = np.maximum(((mu - m) ** 2).mean(axis=0) + var.mean(axis=0), np.finfo(np.float64).eps)
        return m * ysd + ym, v * ysd * ysd

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

    def theta(self):
        return DM.features(self.net, self.data[0])


def dngo_set_data(handle, X, y, normalize_input, normalize_output, prior_par):
    X, y = np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64).ravel()
    if X.shape[0] > _lib.DNGO_MAX_N:
        raise ValueError("gpk_dngo_set_data: n exceeds GPK_DNGO_MAX_N = %d" % _lib.DNGO_MAX_N)
    if X.shape[1] > _lib.DNGO_MAX_D:
        raise ValueError("gpk_dngo_set_data: d exceeds GPK_DNGO_MAX_D = %d" % _lib.DNGO_MAX_D)
    if not (np.isfinite(X).all() and np.isfinite(y).all()):
        raise ValueError("gpk_dngo_set_data: X and y must be finite")
    handle.data = DM.normalise(X, y, normalize_input, normalize_output)
    handle.prior_par = tuple(prior_par)
    handle.net, handle.fit = None, None


def dngo_train(handle, seed, counter, lr, batch, epochs):
    if handle.data is None:
        raise ValueError("gpk_dngo_train: gpk_dngo_set_data has not been called")
    B = min(batch, handle.data[0].shape[0])
    if not (np.isfinite(lr) and lr > 0) or batch < 1 or epochs < 1 or B > _lib.DNGO_MAX_BATCH:
        raise ValueError("gpk_dngo_train: bad arguments")
    handle.train_calls.append((int(seed), int(counter), float(lr), int(batch), int(epochs)))
    handle.net = DM.train(handle.data[0], handle.data[1], seed, counter, lr, batch, epochs)[0]
    handle.fit = None


def dngo_net(handle):
    return handle.net.copy()


def dngo_set_net(handle, net):
    handle.net, handle.fit = np.array(net, dtype=np.float64), None


def dngo_features(handle, X):
    Xs, ys, xm, xs, ym, ysd = handle.data
    return DM.features(handle.net, (np.asarray(X, dtype=np.float64) - xm) / xs)


def blr_lnpost(handle, thetas):
    return LM.lnpost(handle.theta(), handle.data[1], handle.prior_par)(np.atleast_2d(thetas))


def blr_sample(handle, seed, p0, steps):
    handle.sample_calls.append((int(seed), int(steps)))
    return LM.run(LM.lnpost(handle.theta(), handle.data[1], handle.prior_par), np.atleast_2d(p0), int(steps), seed)


def dngo_fit(handle, hypers):
    H = np.atleast_2d(np.asarray(hypers, dtype=np.float64))
    handle.fit = (H, LM.fit(handle.theta(), handle.data[1], H))


def blr_models(handle):
    return [(m.copy(), S.copy()) for m, S in handle.fit[1]]


def install(monkeypatch):
    """Route robo_b200's DNGO entry points and handles through the numpy stand-ins for the duration of a test."""
    pool = {}

    def moments_handle(device=0):
        return pool.setdefault(device, fake_blr._MomentsHandle())
    monkeypatch.setattr(_lib, "Handle", FakeDngoHandle)
    monkeypatch.setattr(_lib, "moments_handle", moments_handle)
    for name in ("dngo_set_data", "dngo_train", "dngo_net", "dngo_set_net", "dngo_features", "dngo_fit",
                 "blr_lnpost", "blr_sample", "blr_models"):
        monkeypatch.setattr(_lib, name, globals()[name])
    return FakeDngoHandle
