"""DifferentialEvolution — robo/maximizers/differential_evolution.py:8-51 with the evolution on the GPU.

The reference hands scipy.optimize.differential_evolution an objective that scores one point per call: at D = 16 and
scipy's defaults (popsize 15, maxiter 20) that is 5,040 single-row acquisition calls per BO iteration before the
polish.  Here the population, the trials, the energies, selection and the convergence test live on the device
(gpk_maximize_de): each generation is one batched scoring pass over every sub-model, and only the winner and a
16-byte status record per generation cross PCIe.

Same algorithm as scipy's 'best1bin' with Latin-hypercube initialisation and the reference's clip / DBL_MAX wrapper,
with two deviations (include/gpk.h): updating='deferred' (scipy's default 'immediate' is serial by construction) and
the counter-based Philox stream keyed by the seed.  The reference never passes its ``rng`` to scipy, so its stream
cannot be reproduced by anyone; here the seed is drawn from ``rng`` at construction and advanced per call, as in
DeviceRandomSampling.

The acquisition may be EI / LogEI / PI / LCB (gpk_maximize_de), InformationGain (gpk_maximize_de_es: the entropy
change, marginalised by gpk_es_multi over a GP-MCMC ensemble), InformationGainMC (gpk_maximize_de_esmc: the
sampling-based entropy change on the update's common draws) or InformationGainPerUnitCost, Fabolas's acquisition
(gpk_maximize_de_es_cost over the extended box), each alone or under MarginalizationGPMCMC.

With ``polish=True`` (scipy's default, which the reference uses) L-BFGS-B refines the device winner on the host
through the reference's single-point objective, and scipy's acceptance rule applies: lower energy, success, inside
the bounds.  With ``polish="device"`` the same refinement runs as one start of the device's multi-start L-BFGS
(gpk_maximize_lbfgs*, the engine of SciPyOptimizer) over the same scoring path as the evolution, under the same
acceptance rule.  InformationGainMC refuses ``polish="device"`` with ValueError: its surface is piecewise constant
in x, so forward differences have nothing to follow; ``polish=True`` runs the reference's host polish over it.
"""
import sys

import numpy as np
import scipy.optimize

from robo_b200.maximizers.base_maximizer import BaseMaximizer
from robo_b200.maximizers.device_spec import device_spec, lbfgs_success, maximize_de, maximize_lbfgs


class DifferentialEvolution(BaseMaximizer):

    def __init__(self, objective_function, lower, upper, n_iters=20, rng=None, popsize=15, mutation=(0.5, 1),
                 recombination=0.7, tol=0.01, atol=0, polish=True):
        self.n_iters = n_iters
        self.popsize = popsize
        self.mutation = tuple(mutation) if np.ndim(mutation) else (mutation, mutation)
        self.recombination = recombination
        self.tol, self.atol = tol, atol
        self.polish = polish
        self.calls = 0
        self.last = None
        super(DifferentialEvolution, self).__init__(objective_function, lower, upper, rng)
        self.seed = int(self.rng.randint(0, 2 ** 31 - 1))

    def _device_spec(self):
        """device_spec.device_spec of the acquisition: what scores the population on the device."""
        return device_spec(self.objective_func, "DifferentialEvolution")

    def _objective(self, x):
        """The reference's single-point objective (differential_evolution.py:27-34)."""
        a = -np.asarray(self.objective_func(np.array([np.clip(x, self.lower, self.upper)])), dtype=np.float64)
        if np.any(np.isinf(a)):
            return sys.float_info.max
        return float(a.ravel()[0])

    def maximize(self):
        which, spec = self._device_spec()
        if which == "esmc" and self.polish == "device":
            raise ValueError("DifferentialEvolution: polish='device' does not apply to InformationGainMC, whose "
                             "surface is piecewise constant in x; use polish=True or polish=False")
        lower, upper = np.asarray(self.lower, dtype=np.float64), np.asarray(self.upper, dtype=np.float64)
        seed = (self.seed + 0x9E3779B97F4A7C15 * self.calls) & 0xFFFFFFFFFFFFFFFF
        self.calls += 1
        pop = max(5, int(self.popsize) * lower.size)                 # scipy: max(5, popsize * D)
        r = maximize_de(which, spec, seed, pop, int(self.n_iters), self.mutation, self.recombination, self.tol,
                        self.atol, lower, upper)
        x, fun, nfev, polished = r["x"], r["energy"], r["nfev"], False
        if self.polish == "device":
            res = maximize_lbfgs(which, spec, x[None, :], lower, upper)
            nfev += int(res["nfev"][0])
            xp, ep = res["x"][0], float(res["energy"][0])
            if ep < fun and lbfgs_success(res["status"][0]) and np.all(xp <= upper) and np.all(lower <= xp):
                x, fun, polished = xp, ep, True
        elif self.polish:
            res = scipy.optimize.minimize(self._objective, np.copy(x), method="L-BFGS-B",
                                          bounds=scipy.optimize.Bounds(lower, upper))
            nfev += int(res.get("nfev", 0))
            if res.fun < fun and res.success and np.all(res.x <= upper) and np.all(lower <= res.x):
                x, fun, polished = res.x, float(res.fun), True
        self.last = dict(seed=seed, nit=r["nit"], nfev=nfev, best_energy=fun, device_energy=r["energy"],
                         polished=polished)
        return np.clip(x, lower, upper)
