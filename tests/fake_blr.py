"""Numpy stand-in for the BayesianLinearRegression entry points of robo_b200._lib — TEST INFRASTRUCTURE ONLY.

The arithmetic is tests/blr_model.py's, in the reference's order of operations; the sampler is blr_model.run, the
exact restatement of gpk_blr_sample, over that numpy log-posterior.  Argument checks mirror the C side's GPK_BAD_ARG
cases as ValueError.  Lets the CPU suite drive BayesianLinearRegression and device_spec without a GPU."""
import numpy as np

from robo_b200 import _lib
from tests import blr_model as BM


class FakeBlrHandle(object):
    def __init__(self, device=0):
        self.device = device
        self.Phi = self.y = None
        self.hypers = self.models = None
        self.sample_calls = []

    def close(self):
        pass

    def predict(self, Xs):
        if self.models is None:
            raise RuntimeError("model is not fitted (gpk_blr_fit)")
        return BM.predict(BM.features(Xs, self.basis), self.hypers, self.models)

    def acq(self, Xs, kind, eta=0.0, par=0.0, want_values=True, want_moments=False):
        m, v = self.predict(Xs)
        vals, nn = moments(m, v, kind, eta, par)
        return dict(values=vals, mu=m, var=v, best_val=float(vals.max()), best_idx=int(np.argmax(vals)), n_negative=nn)


def moments(m, v, kind, eta, par):
    """The closed forms of gpk_acq_moments for EI / PI / LCB (ei.py, pi.py, lcb.py)."""
    from scipy.stats import norm
    s = np.sqrt(v)
    if kind == _lib.ACQ_LCB:
        return -(m - par * s), 0
    z = (eta - m - par) / s
    if kind == _lib.ACQ_PI:
        return norm.cdf(z), 0
    f = s * (z * norm.cdf(z) + norm.pdf(z))
    return f, int(np.sum(f < 0))


def blr_set_data(handle, X, y, basis, prior_par):
    X, y = np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64)
    if basis not in (0, 1, 2):
        raise ValueError("gpk_blr_set_data: unknown basis %d" % basis)
    if _lib.blr_features(X.shape[1], basis) > _lib.BLR_MAX_F:
        raise ValueError("gpk_blr_set_data: features exceed GPK_BLR_MAX_F")
    handle.basis, handle.Phi, handle.y, handle.par = basis, BM.features(X, basis), y, tuple(prior_par)
    handle.hypers = handle.models = None


def blr_lnpost(handle, thetas):
    if handle.Phi is None:
        raise ValueError("gpk_blr_lnpost: gpk_blr_set_data has not been called")
    return BM.lnpost(handle.Phi, handle.y, handle.par)(np.atleast_2d(thetas))


def blr_sample(handle, seed, p0, steps):
    p0 = np.atleast_2d(np.asarray(p0, dtype=np.float64))
    if p0.shape[0] % 2 or p0.shape[0] < 4 or steps < 0:
        raise ValueError("gpk_blr_sample: bad arguments")
    handle.sample_calls.append((int(seed), p0.copy(), int(steps)))
    return BM.run(BM.lnpost(handle.Phi, handle.y, handle.par), p0, steps, seed)


def blr_fit(handle, hypers):
    H = np.atleast_2d(np.asarray(hypers, dtype=np.float64))
    handle.hypers, handle.models = H, BM.fit(handle.Phi, handle.y, H)


def blr_models(handle):
    return [(m.copy(), S.copy()) for m, S in handle.models]


def install(monkeypatch):
    """Route robo_b200's BLR entry points and handles through the numpy stand-ins for the duration of a test."""
    pool = {}

    def moments_handle(device=0):
        return pool.setdefault(device, _MomentsHandle())
    monkeypatch.setattr(_lib, "Handle", FakeBlrHandle)
    monkeypatch.setattr(_lib, "moments_handle", moments_handle)
    for name in ("blr_set_data", "blr_lnpost", "blr_sample", "blr_fit", "blr_models"):
        monkeypatch.setattr(_lib, name, globals()[name])
    return FakeBlrHandle


class _MomentsHandle(object):
    def acq_moments(self, mu, var, kind, eta=0.0, par=0.0):
        return moments(np.asarray(mu), np.asarray(var), kind, eta, par)
