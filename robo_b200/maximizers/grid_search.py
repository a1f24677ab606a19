"""GridSearch — robo/maximizers/grid_search.py:6-48: the arg-max of the acquisition over an evenly spaced 1-D grid.

The reference scores the grid one point per call.  A device acquisition (EI / LogEI / PI / LCB, InformationGain,
InformationGainMC or InformationGainPerUnitCost, alone or marginalised) scores all ``resolution`` points in one call of
the one-shot multi-model scoring (gpk_acq_multi, gpk_es_multi, gpk_esmc_multi, gpk_es_cost_multi), which also takes
numpy's first-index arg-max on the device; any other acquisition keeps the reference's per-point loop.
"""
import numpy as np

from robo_b200.maximizers.base_maximizer import BaseMaximizer
from robo_b200.maximizers.device_spec import device_spec, score_batch


class GridSearch(BaseMaximizer):

    def __init__(self, objective_function, lower, upper, resolution=1000, rng=None):
        self.resolution = resolution
        if lower.shape[0] > 1:
            raise RuntimeError("Grid search works just for \
                one dimensional functions")
        super(GridSearch, self).__init__(objective_function, lower, upper, rng)

    def maximize(self):
        """The grid point with the highest acquisition value (numpy's first arg-max), shape (1,)."""
        x = np.linspace(self.lower[0], self.upper[0], self.resolution).reshape((self.resolution, 1, 1))
        try:
            which, spec = device_spec(self.objective_func, "GridSearch")
        except TypeError:
            which = None
        if which is None:
            ys = np.zeros([self.resolution])
            for i in range(self.resolution):
                ys[i] = self.objective_func(x[i])
            return x[ys.argmax()][0]
        r = score_batch(which, spec, x.reshape(self.resolution, 1))
        return x[int(r["best_idx"])][0]
