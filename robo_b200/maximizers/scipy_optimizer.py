"""SciPyOptimizer — robo/maximizers/scipy_optimizer.py with the restarts on the GPU.

The reference runs scipy's L-BFGS-B from n_restarts starts, one after the other, on a single-point objective with
finite-difference gradients: at D = 16 every iteration of every start costs 17 single-row acquisition calls.  Here all
starts run in lockstep on the device (gpk_maximize_lbfgs*): each round scores the trial point of every running start
and its D neighbours in one batched pass through the scoring path DifferentialEvolution drives, and only a 16-byte
status record per round crosses PCIe.

The algorithm is projected L-BFGS with scipy's defaults (maxcor 10, ftol, pgtol, maxiter, maxfun) and scipy's
forward differences, not L-BFGS-B's Cauchy point and subspace minimisation (include/gpk.h states the deviation).

Starts follow the reference's recipe, drawn from ``self.rng`` instead of numpy's global stream: int(0.5 n) uniform in
the box, then int(0.5 n) normal around the incumbent with scale 0.5.  An acquisition that does not run on device
models takes the reference's host loop unchanged, so the class is a drop-in for the reference's.  So does
InformationGainMC, alone or marginalised: its Monte-Carlo surface is piecewise constant in x, so forward-difference
L-BFGS has nothing to follow on the device either (as in the reference), and each start scores one row per call.
"""
import sys
from functools import partial

import numpy as np
from scipy import optimize

from robo_b200.initial_design import init_random_uniform
from robo_b200.maximizers.base_maximizer import BaseMaximizer
from robo_b200.maximizers.device_spec import device_spec, is_sampling_based, maximize_lbfgs


class SciPyOptimizer(BaseMaximizer):

    def __init__(self, objective_function, lower, upper, n_restarts=10, verbosity=False, rng=None):
        self.n_restarts = n_restarts
        self.verbosity = verbosity
        self.last = None
        super(SciPyOptimizer, self).__init__(objective_function, lower, upper, rng)

    def _acquisition_fkt_wrapper(self, x, acq_f):
        """The reference's single-point objective (scipy_optimizer.py:39-49)."""
        if np.any(np.isnan(x)):
            return sys.float_info.max
        a = -acq_f(np.array([np.clip(x, self.lower, self.upper)]))[0]
        if np.any(np.isinf(a)):
            return sys.float_info.max
        return a

    def _starts(self):
        n = int(self.n_restarts * 0.5)
        lower = np.asarray(self.lower, dtype=np.float64)
        starts = init_random_uniform(lower, np.asarray(self.upper, dtype=np.float64), n, rng=self.rng)
        inc = self.objective_func.model.get_incumbent()[0]
        rand_incs = np.array([self.rng.normal(loc=inc, scale=np.ones([lower.shape[0]]) * 0.5) for _ in range(n)])
        return np.append(starts.reshape(n, lower.shape[0]), rand_incs.reshape(n, lower.shape[0]), axis=0)

    def maximize(self):
        """The point with the highest acquisition value found from the starts, clipped into the box."""
        lower, upper = np.asarray(self.lower, dtype=np.float64), np.asarray(self.upper, dtype=np.float64)
        starts = self._starts()
        if len(starts) == 0:
            raise ValueError("SciPyOptimizer needs n_restarts >= 2 (int(0.5 n_restarts) starts of each kind)")
        if is_sampling_based(self.objective_func):
            return self._maximize_host(starts)
        try:
            which, spec = device_spec(self.objective_func, "SciPyOptimizer")
        except TypeError:
            which = None
        if which is None:
            return self._maximize_host(starts)
        r = maximize_lbfgs(which, spec, starts, lower, upper)
        best = int(np.argmin(r["energy"]))
        self.last = dict(starts=starts, x=r["x"], energy=r["energy"], nit=r["nit"], nfev=r["nfev"], status=r["status"],
                         best=best, device=True)
        return np.clip(r["x"][best], lower, upper)

    def _maximize_host(self, starts):
        """scipy_optimizer.py:51-82: L-BFGS-B from every start on the single-point objective."""
        f = partial(self._acquisition_fkt_wrapper, acq_f=self.objective_func)
        cand, cand_vals = [], []
        for start in starts:
            res = optimize.minimize(f, start, method="L-BFGS-B", bounds=list(zip(self.lower, self.upper)),
                                    options={"disp": self.verbosity})
            cand.append(res["x"])
            cand_vals.append(res["fun"])
        best = int(np.argmin(cand_vals))
        self.last = dict(starts=starts, x=np.array(cand), energy=np.array(cand_vals, dtype=np.float64), best=best,
                         device=False)
        return np.clip(cand[best], self.lower, self.upper)
