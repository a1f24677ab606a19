"""CMAES — robo/maximizers/cmaes.py:15-81 with the evolution strategy on the GPU and without the `cma` package.

The reference hands cma.fmin an objective that scores one point per call (cmaes.py:66-68): with the default
n_func_evals = 1000 that is 1000 single-row acquisition calls per BO iteration.  Here the whole strategy runs on the
device (gpk_maximize_cmaes*): every generation is one batched scoring pass over every sub-model, and the ranking, the
update of the mean, step size, paths and covariance, its eigendecomposition and the stop tests run in one CTA beside
the scores; only a 24-byte status record per generation crosses PCIe.

The algorithm is the (mu/mu_w, lambda)-CMA-ES of Hansen's tutorial under cma's BoundTransform with IPOP restarts, as
cma.fmin runs it for the reference (x0 from init_random_uniform, sigma0 = 0.6, maxfevals = n_func_evals, restarts).
It agrees with cma in law, not bit for bit; include/gpk.h lists what is not restated (active CMA, NaN resampling and
some stop rules).  The random stream is Philox keyed by a seed drawn from ``rng`` at construction and advanced per
call, as in DifferentialEvolution.

The acquisition may be EI / LogEI / PI / LCB, InformationGain, InformationGainMC or InformationGainPerUnitCost, each
alone or under MarginalizationGPMCMC; an acquisition that does not run on device models raises TypeError (there is no
host `cma` path).
"""
import logging

import numpy as np

from robo_b200.initial_design.init_random_uniform import init_random_uniform
from robo_b200.maximizers.base_maximizer import BaseMaximizer
from robo_b200.maximizers.device_spec import device_spec, maximize_cmaes

logger = logging.getLogger(__name__)


class CMAES(BaseMaximizer):

    def __init__(self, objective_function, lower, upper, verbose=True, restarts=0, n_func_evals=1000, rng=None):
        if lower.shape[0] == 1:
            raise RuntimeError("CMAES does not works in a one dimensional function space")
        super(CMAES, self).__init__(objective_function, lower, upper, rng)
        self.restarts = restarts
        self.verbose = verbose
        self.n_func_evals = n_func_evals
        self.calls = 0
        self.last = None
        self.seed = int(self.rng.randint(0, 2 ** 31 - 1))

    def maximize(self):
        """The point with the highest acquisition value found, shape (D,).  When no finite energy was seen, the
        reference's fallback (cmaes.py:76-79): the random start point, as init_random_uniform returns it, shape (1, D)."""
        which, spec = device_spec(self.objective_func, "CMAES")
        lower, upper = np.asarray(self.lower, dtype=np.float64), np.asarray(self.upper, dtype=np.float64)
        start_point = init_random_uniform(lower, upper, 1, self.rng)
        seed = (self.seed + 0x9E3779B97F4A7C15 * self.calls) & 0xFFFFFFFFFFFFFFFF
        self.calls += 1
        r = maximize_cmaes(which, spec, seed, start_point[0], lower, upper, int(self.n_func_evals), int(self.restarts))
        self.last = dict(seed=seed, nfev=r["nfev_total"], nit=r["nit"], stop=r["stop"], best_energy=r["energy"])
        if self.verbose:
            logger.info("CMAES: best energy %g after %d evaluations (stops per run: %s)", r["energy"], r["nfev_total"],
                        list(r["stop"]))
        if not np.isfinite(r["energy"]):
            logger.error("CMA-ES did not find anything. Return random configuration instead.")
            return start_point
        return np.clip(r["x"], lower, upper)
