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
change, marginalised by gpk_es_multi over a GP-MCMC ensemble) or InformationGainPerUnitCost, Fabolas's acquisition
(gpk_maximize_de_es_cost over the extended box), each alone or under MarginalizationGPMCMC.

With ``polish=True`` (scipy's default, which the reference uses) L-BFGS-B refines the device winner on the host
through the reference's single-point objective, and scipy's acceptance rule applies: lower energy, success, inside
the bounds.  The polish stays per point by design.
"""
import sys

import numpy as np
import scipy.optimize

from robo_b200 import _lib
from robo_b200.maximizers.base_maximizer import BaseMaximizer
from robo_b200.models.gaussian_process import GaussianProcess

KINDS = ("ei", "log_ei", "pi", "lcb")


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
        """What scores the population on the device, by acquisition:
            ("es_cost", device_spec's tuple)   InformationGainPerUnitCost, alone or marginalised (gpk_es_cost_multi)
            ("es", handles)                    InformationGain, alone or marginalised (gpk_es_compute / gpk_es_multi)
            ("acq", (kind, etas, par, handles)) EI / LogEI / PI / LCB (gpk_acq_multi)
        TypeError when the acquisition does not run on device models."""
        from robo_b200.acquisition_functions.information_gain import InformationGain
        from robo_b200.acquisition_functions.information_gain_per_unit_cost import (InformationGainPerUnitCost,
                                                                                    device_spec)
        acq = self.objective_func
        estimators = acq.estimators if hasattr(acq, "_fused_spec") else [acq]
        # InformationGainPerUnitCost is an InformationGain: it is recognised first
        if estimators and all(isinstance(e, InformationGainPerUnitCost) for e in estimators):
            return "es_cost", device_spec(estimators)
        if estimators and all(isinstance(e, InformationGain) for e in estimators):
            if not all(_raw_inputs(e.model) for e in estimators):
                raise TypeError("DifferentialEvolution needs InformationGain on robo_b200 GaussianProcess models")
            return "es", [e._ready_handle() for e in estimators]
        return "acq", self._acq_spec()

    def _acq_spec(self):
        """(kind, eta per model, par, handles) of the acquisition, or TypeError when it does not run on device GPs
        whose inputs go to the handle untransformed."""
        acq = self.objective_func
        if hasattr(acq, "_fused_spec"):                          # MarginalizationGPMCMC
            fused = acq._fused_spec()
            if fused is None or not all(_raw_inputs(m) for m in acq.model.models):
                raise TypeError("DifferentialEvolution needs a marginalised EI / LogEI / PI / LCB over device "
                                "GaussianProcess sub-models")
            kind, etas, par, handles = fused
            return kind, etas, par, handles
        model = getattr(acq, "model", None)
        kind = getattr(acq, "kind", None)
        if kind not in KINDS or getattr(acq, "cost_model", None) is not None or not _raw_inputs(model) \
                or not hasattr(getattr(model, "gp", None), "handle"):
            raise TypeError("DifferentialEvolution needs EI / LogEI / PI / LCB on a robo_b200 GaussianProcess model")
        eta = 0.0 if kind == "lcb" else float(model.get_incumbent()[1])
        model.gp._restore()
        model.gp._push_cfg()
        return kind, [eta], float(acq.par), [model.gp.handle]

    def _objective(self, x):
        """The reference's single-point objective (differential_evolution.py:27-34)."""
        a = -np.asarray(self.objective_func(np.array([np.clip(x, self.lower, self.upper)])), dtype=np.float64)
        if np.any(np.isinf(a)):
            return sys.float_info.max
        return float(a.ravel()[0])

    def maximize(self):
        which, spec = self._device_spec()
        lower, upper = np.asarray(self.lower, dtype=np.float64), np.asarray(self.upper, dtype=np.float64)
        seed = (self.seed + 0x9E3779B97F4A7C15 * self.calls) & 0xFFFFFFFFFFFFFFFF
        self.calls += 1
        pop = max(5, int(self.popsize) * lower.size)                 # scipy: max(5, popsize * D)
        args = (seed, pop, int(self.n_iters), self.mutation, self.recombination, self.tol, self.atol, lower, upper)
        if which == "es_cost":
            ho, hc, lo, up, bo, bc, oh = spec
            r = _lib.maximize_de_es_cost(ho, hc, *args, cfg_lower=lo, cfg_upper=up, basis_objective=bo, basis_cost=bc,
                                         overhead=oh)
        elif which == "es":
            r = _lib.maximize_de_es(spec, *args)
        else:
            kind, etas, par, handles = spec
            r = _lib.maximize_de(handles, *args, kind=_lib.ACQ_KIND[kind], eta=etas, par=par)
            if kind == "ei" and r["n_negative"] > 0:
                raise ValueError("Expected Improvement is smaller than 0!")      # ei.py:86-88
        x, fun, nfev, polished = r["x"], r["energy"], r["nfev"], False
        if self.polish:
            res = scipy.optimize.minimize(self._objective, np.copy(x), method="L-BFGS-B",
                                          bounds=scipy.optimize.Bounds(lower, upper))
            nfev += int(res.get("nfev", 0))
            if res.fun < fun and res.success and np.all(res.x <= upper) and np.all(lower <= res.x):
                x, fun, polished = res.x, float(res.fun), True
        self.last = dict(seed=seed, nit=r["nit"], nfev=nfev, best_energy=fun, device_energy=r["energy"],
                         polished=polished)
        return np.clip(x, lower, upper)


def _raw_inputs(model):
    """The model hands its raw inputs to the handle (no host-side transform such as FabolasGP's)."""
    return model is not None and getattr(type(model), "device_inputs", None) is GaussianProcess.device_inputs
