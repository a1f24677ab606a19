"""Numpy restatement of InformationGainPerUnitCost.compute's last step (robo/acquisition_functions/
information_gain_per_unit_cost.py:91-104) and host fakes for its CPU tests.  Test infrastructure only."""
import numpy as np

DBL_MAX = np.finfo(np.float64).max
EPS = np.spacing(1)


def per_unit_cost(dh, log_cost, overhead):
    """dh / (exp(log_cost) + overhead), in the reference's order: cost = np.exp(log_cost); dh / (cost + overhead)."""
    with np.errstate(over="ignore"):
        cost = np.exp(np.asarray(log_cost, dtype=np.float64))
        return np.asarray(dh, dtype=np.float64) / (cost + overhead)


class ConstantSampling(object):
    """Sampling acquisition stand-in: a constant value at every point, recording the points it was asked about."""

    def __init__(self, model, value=0.5, **kwargs):
        self.model = model
        self.value = value
        self.seen = []
        self.updates = 0

    def update(self, model):
        self.model = model
        self.updates += 1

    def __call__(self, X):
        X = np.asarray(X)
        self.seen.append(X.copy())
        return np.full(X.shape[0], self.value)


class HostModel(object):
    """A model that cannot go to the device."""

    def __init__(self, noise=1e-3):
        self.noise = noise

    def get_noise(self):
        return self.noise


class Ensemble(object):
    """The `models` list of a GP-MCMC model."""

    def __init__(self, n):
        self.models = [HostModel() for _ in range(n)]
