"""Numpy stand-in for the random-forest entry points of robo_b200._lib — TEST INFRASTRUCTURE ONLY.

The forest is tests/rf_model.py's, the exact restatement of gpk_rf_set_data / gpk_rf_fit and the predictive pass;
the acquisition closed forms are gpk_acq_moments' (through fake_blr.moments) with the forest's zero-std EI rule.
Argument checks mirror the C side's GPK_BAD_ARG cases as ValueError.  Lets the CPU suite drive RandomForest,
device_spec and DeviceRandomSampling without a GPU."""
import numpy as np

from robo_b200 import _lib
from tests import fake_blr
from tests import rf_model as RM


class FakeRfHandle(object):
    def __init__(self, device=0):
        self.device = device
        self.X = self.y = None
        self.forest = None
        self.fit_calls = []

    def close(self):
        pass

    def predict(self, Xs):
        if self.forest is None:
            raise RuntimeError("model is not fitted (gpk_rf_fit)")
        return RM.predict(self.forest, np.asarray(Xs, dtype=np.float64), self.total)

    def acq(self, Xs, kind, eta=0.0, par=0.0, want_values=True, want_moments=False):
        m, v = self.predict(Xs)
        vals, nn = values(m, v, kind, eta, par)
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


def values(m, v, kind, eta, par):
    """The forest's acquisition values: gpk_acq_moments' closed forms, EI 0 where var is 0."""
    with np.errstate(divide="ignore", invalid="ignore"):
        vals, nn = fake_blr.moments(m, v, kind, eta, par)
    vals = np.asarray(vals, dtype=np.float64)
    if kind == _lib.ACQ_EI:
        vals = np.where(v == 0, 0.0, vals)
        nn = int(np.sum(vals < 0))
    return vals, nn


def rf_set_data(handle, X, y):
    X, y = np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64).ravel()
    if X.shape[0] > _lib.RF_MAX_N:
        raise ValueError("gpk_rf_set_data: n exceeds GPK_RF_MAX_N = %d" % _lib.RF_MAX_N)
    if X.shape[1] > _lib.RF_MAX_D:
        raise ValueError("gpk_rf_set_data: d exceeds GPK_RF_MAX_D = %d" % _lib.RF_MAX_D)
    if not (np.isfinite(X).all() and np.isfinite(y).all()):
        raise ValueError("gpk_rf_set_data: X and y must be finite")
    handle.X, handle.y, handle.forest = X, y, None


def rf_fit(handle, seed, counter, num_trees, n_per_tree, bootstrap, total_variance):
    if handle.X is None:
        raise ValueError("gpk_rf_fit: gpk_rf_set_data has not been called")
    if not 1 <= num_trees <= _lib.RF_MAX_T or n_per_tree < 0:
        raise ValueError("gpk_rf_fit: bad arguments")
    handle.fit_calls.append((int(seed), int(counter), int(num_trees), int(n_per_tree), bool(bootstrap)))
    handle.forest = RM.fit(handle.X, handle.y, seed, counter, num_trees, n_per_tree, bootstrap)
    handle.total = bool(total_variance)


def rf_trees(handle):
    return RM.pack(handle.forest, 2 * len(handle.y))


def rf_set_trees(handle, trees, total_variance):
    handle.forest, handle.total = RM.unpack(trees), bool(total_variance)


def install(monkeypatch):
    """Route robo_b200's RF entry points and handles through the numpy stand-ins for the duration of a test."""
    pool = {}

    def moments_handle(device=0):
        return pool.setdefault(device, fake_blr._MomentsHandle())
    monkeypatch.setattr(_lib, "Handle", FakeRfHandle)
    monkeypatch.setattr(_lib, "moments_handle", moments_handle)
    for name in ("rf_set_data", "rf_fit", "rf_trees", "rf_set_trees"):
        monkeypatch.setattr(_lib, name, globals()[name])
    return FakeRfHandle
