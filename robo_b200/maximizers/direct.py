"""Direct — robo/maximizers/direct.py:17-85 with DIRECT on the GPU and without the `DIRECT` package.

The reference hands DIRECT.solve an objective that scores one point per call (direct.py:50-54): at the defaults
(n_func_evals = 400, n_iters = 200) that is about 400 single-row acquisition calls per BO iteration.  Here the whole
search runs on the device (gpk_maximize_direct*): once an iteration has chosen its potentially optimal rectangles,
every point it samples is known, so the iteration is one batched scoring pass over every sub-model, and the choice,
the trisection and the level lists run in one CTA beside the scores; only a 24-byte status record per iteration
crosses PCIe.

The algorithm is Jones' original DIRECT as Gablonsky's DIRECT 2.0.4 runs it with the package's defaults, restated
operation for operation (include/gpk.h lists what is not restated: the stdout report, the log file, the hidden-
constraint flag).  DIRECT is deterministic, so a run is a function of the acquisition and the box alone; ``rng`` is
accepted for the BaseMaximizer signature.

The acquisition may be EI / LogEI / PI / LCB, InformationGain, InformationGainMC or InformationGainPerUnitCost, each
alone or under MarginalizationGPMCMC; an acquisition that does not run on device models raises TypeError (there is no
host DIRECT).
"""
import logging

import numpy as np

from robo_b200 import _lib
from robo_b200.maximizers.base_maximizer import BaseMaximizer
from robo_b200.maximizers.device_spec import device_spec, maximize_direct

logger = logging.getLogger(__name__)


class Direct(BaseMaximizer):

    def __init__(self, objective_function, lower, upper, n_func_evals=400, n_iters=200, verbose=True, rng=None):
        self.n_func_evals = n_func_evals
        self.n_iters = n_iters
        self.verbose = verbose
        self.last = None
        super(Direct, self).__init__(objective_function, lower, upper, rng)

    def maximize(self):
        """The point with the highest acquisition value found, shape (D,)."""
        which, spec = device_spec(self.objective_func, "Direct")
        lower, upper = np.asarray(self.lower, dtype=np.float64), np.asarray(self.upper, dtype=np.float64)
        r = maximize_direct(which, spec, lower, upper, int(self.n_func_evals), int(self.n_iters))
        self.last = dict(nfev=r["nfev"], nit=r["nit"], stop=r["stop"], best_energy=r["energy"], rows=r["rows"])
        if self.verbose:
            logger.info("Direct: best energy %g after %d evaluations in %d iterations (stop: %s)", r["energy"],
                        r["nfev"], r["nit"], _lib.DIRECT_STOP_NAMES[r["stop"]])
        return r["x"]
