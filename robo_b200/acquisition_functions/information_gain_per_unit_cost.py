"""InformationGainPerUnitCost — the Fabolas acquisition of robo/acquisition_functions/information_gain_per_unit_cost.py
(Swersky et al., NIPS 2013, with the optimisation overhead added to the cost) with its numerical work on the GPU.

The entropy change dh of the objective model divided by the predicted cost, exp(log_cost) + overhead, where log_cost is
the cost model's predictive MEAN (:91).  Both models are FabolasGP models or both MTBOGP models, which map their inputs
on the host (configuration columns scaled to [0, 1], the last column through a basis function, or np.rint for MTBO's task
index); here the whole value is one device call (gpk_es_cost_multi): the raw batch is transformed on the device bit for
bit as the models' normalize does, the
objective's entropy change runs on the transformed batch with its bounds test on the raw one (DBL_EPSILON outside the
raw extended [lower, upper], as the reference's dh_fun tests), the cost model runs a mean-only prediction.

Reference behaviour kept: overhead None -> 0; representer points sampled in the configuration dimensions only, scored
at the upper bound of the environment dimensions, and then given the NUMBER of environment dimensions as their
environment coordinate (:151-153); up to 5 restarts of 50 steps and the reference's ValueError when the log-probabilities
stay infinite; derivative=True raises TypeError (the reference raises a string).  One deviation: the sampler runs with
rstate0=self.rng (as InformationGain does), so a run is reproducible under numpy.random.seed; the restarts are drawn from
numpy's global stream like the reference's.
"""
import logging

import numpy as np

from robo_b200 import _lib
from robo_b200.acquisition_functions.information_gain import InformationGain, sample_representers_device
from robo_b200.util.ensemble_sampler import EnsembleSampler

logger = logging.getLogger(__name__)

# basis recognition: the model's callable on this probe vector, compared bit for bit against the two Fabolas forms
_PROBE = np.array([0.0, 1.0, 0.5, 0.25, 1.0 / 3.0, 0.1, 0.7, 0.9, 2.0 ** -20, 1.0 - 2.0 ** -30, 0.123456789, 3.0, -0.5])


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def basis_code(basis_func):
    """gpk_basis code of a Fabolas basis function: s -> BASIS_S, (1 - s) ** 2 -> BASIS_ONE_MINUS_S_SQ (the two lambdas
    of robo/fmin/fabolas.py:96-102).  Any other function raises TypeError: the device has no kernel for it."""
    try:
        v = np.ascontiguousarray(basis_func(_PROBE.copy()), dtype=np.float64)
    except Exception as e:
        raise TypeError("Fabolas basis function could not be evaluated on a vector: %s" % e)
    if _same_bits(v, _PROBE):
        return _lib.BASIS_S
    t = 1.0 - _PROBE
    if _same_bits(v, t * t):
        return _lib.BASIS_ONE_MINUS_S_SQ
    raise TypeError("InformationGainPerUnitCost runs on the device only for the basis functions s and (1 - s) ** 2")


def model_basis(model):
    """gpk_basis code of the last column's map of a FabolasGP (its basis function) or an MTBOGP (BASIS_TASK)."""
    from robo_b200.models.mtbo_gp import MTBOGP
    if isinstance(model, MTBOGP):
        return _lib.BASIS_TASK
    return basis_code(model.basis_function)


def _fabolas_device(model, role):
    from robo_b200.models.fabolas_gp import FabolasGP
    from robo_b200.models.mtbo_gp import MTBOGP
    if not isinstance(model, (FabolasGP, MTBOGP)) or not hasattr(getattr(model, "gp", None), "handle"):
        raise TypeError("InformationGainPerUnitCost runs on robo_b200 FabolasGP or MTBOGP models (%s model)" % role)
    model.gp._restore()
    model.gp._push_cfg()
    return model.gp.handle


def device_spec(pairs):
    """(objective handles, cost handles, lower, upper, basis codes, overhead) of the fused call for a list of updated
    InformationGainPerUnitCost estimators.  Raises TypeError when a model cannot go to the device and ValueError when
    an estimator was not updated."""
    ho, hc = [], []
    lo = up = None
    codes = set()
    overheads = set()
    for e in pairs:
        if e.zb is None:
            raise ValueError("InformationGainPerUnitCost.compute needs update() first")
        if not np.all(np.isfinite(e.lmb)):
            raise ValueError("lmb should not be infinite.")
        ho.append(_fabolas_device(e.model, "objective"))
        hc.append(_fabolas_device(e.cost_model, "cost"))
        for m in (e.model, e.cost_model):
            mlo, mup = np.asarray(m.lower, dtype=np.float64).ravel(), np.asarray(m.upper, dtype=np.float64).ravel()
            if lo is None:
                lo, up = mlo, mup
            elif not (_same_bits(mlo, lo) and _same_bits(mup, up)):
                raise TypeError("InformationGainPerUnitCost on the device needs one set of configuration bounds for the "
                                "objective and the cost models")
        codes.add((model_basis(e.model), model_basis(e.cost_model)))
        overheads.add(float(e.overhead))
    if len(codes) != 1 or len(overheads) != 1:
        raise TypeError("InformationGainPerUnitCost on the device needs one basis per model family and one overhead")
    bo, bc = codes.pop()
    return ho, hc, lo, up, bo, bc, overheads.pop()


class InformationGainPerUnitCost(InformationGain):

    def __init__(self, model, cost_model, lower, upper, is_env_variable, sampling_acquisition=None, n_representer=50,
                 rng=None, representer_sampler="host"):
        self.cost_model = cost_model
        self.n_dims = lower.shape[0]
        self.is_env = is_env_variable
        self.overhead = 0
        super(InformationGainPerUnitCost, self).__init__(model, lower, upper, sampling_acquisition=sampling_acquisition,
                                                         Nb=n_representer, rng=rng,
                                                         representer_sampler=representer_sampler)

    def update(self, model, cost_model, overhead=None):
        self._set_cost(cost_model, overhead)
        super(InformationGainPerUnitCost, self).update(model)

    def _set_cost(self, cost_model, overhead=None):
        self.cost_model = cost_model
        if overhead is None:
            self.overhead = 0
        else:
            self.overhead = overhead

    # the device sampler's view: walkers in the configuration columns, scored at the environment's upper bound through
    # the objective's Fabolas transform (sampling_acquisition_wrapper); one environment column, the last one
    def _representer_spec(self):
        is_env = np.asarray(self.is_env).ravel()
        if int(np.sum(is_env == 1)) != 1 or is_env[-1] != 1 or is_env.size != self.lower.shape[0]:
            raise TypeError("representer_sampler='device' needs exactly one environment column, the last one")
        handle = self._device_handle(self.model)
        lower, upper = self._config_bounds()
        fabolas = dict(cfg_lower=np.asarray(self.model.lower, dtype=np.float64).ravel(),
                       cfg_upper=np.asarray(self.model.upper, dtype=np.float64).ravel(),
                       basis=model_basis(self.model), env_value=float(self.upper[is_env == 1][0]))
        return handle, np.asarray(lower, dtype=np.float64), np.asarray(upper, dtype=np.float64), fabolas

    def _set_representers(self, zb, lmb):
        if np.any(np.isinf(lmb)):
            raise ValueError("Could not sample valid representer points! LogEI is -infinity")
        self.zb, self.lmb = zb, lmb[:, None]
        self._append_env_column()

    def _append_env_column(self):
        # information_gain_per_unit_cost.py:151-153: the environment coordinate is the number of environment dimensions
        proj = np.ones([self.zb.shape[0], self.upper[self.is_env == 1].shape[0]])
        proj *= self.upper[self.is_env == 1].shape[0]
        self.zb = np.concatenate((self.zb, proj), axis=1)

    # InformationGain.update's device hooks: FabolasGP / MTBOGP handle; zb transformed on the host as the model maps its
    # inputs
    def _device_handle(self, model):
        return _fabolas_device(model, "objective")

    def _device_zb(self):
        return self.model.normalize(self.zb)

    def compute(self, X, derivative=False):
        """dh / (exp(log_cost) + overhead) of every row of X -> (N,)."""
        if len(X.shape) == 1:
            X = X[np.newaxis, :]
        if derivative:
            # the reference's `raise "Not implemented"`, under Python 3
            raise TypeError("exceptions must derive from BaseException")
        ho, hc, lo, up, bo, bc, oh = device_spec([self])
        return _lib.es_cost_multi(ho, hc, np.asarray(X, dtype=np.float64), lo, up, bo, bc, oh)["values"]

    def argmax(self, X_test):
        ho, hc, lo, up, bo, bc, oh = device_spec([self])
        r = _lib.es_cost_multi(ho, hc, np.asarray(X_test, dtype=np.float64), lo, up, bo, bc, oh, want_values=False)
        return int(r["best_idx"])

    def _config_bounds(self):
        return self.lower[np.where(self.is_env == 0)], self.upper[np.where(self.is_env == 0)]

    def sampling_acquisition_wrapper(self, x):
        lower, upper = self._config_bounds()
        if np.any(x < lower) or np.any(x > upper):
            return -np.inf
        proj_x = np.concatenate((x, self.upper[self.is_env == 1]))
        return self.sampling_acquisition(np.array([proj_x]))[0]

    def _sampling_batch(self, X):
        """The wrapper's one-point semantics over a whole half-ensemble, scored in one call."""
        lower, upper = self._config_bounds()
        out = np.full(X.shape[0], -np.inf)
        inside = np.all((X >= lower) & (X <= upper), axis=1)
        if np.any(inside):
            env = np.broadcast_to(self.upper[self.is_env == 1], (int(inside.sum()), int(np.sum(self.is_env == 1))))
            proj = np.concatenate((X[inside], env), axis=1)
            out[inside] = np.asarray(self.sampling_acquisition(proj), dtype=np.float64).ravel()
        return out

    def sample_representer_points(self):
        if self.representer_sampler == "device":
            sample_representers_device([self])
            return
        D = np.where(self.is_env == 0)[0].shape[0]
        lower, upper = self._config_bounds()
        self.sampling_acquisition.update(self.model)
        for i in range(5):
            restarts = np.random.uniform(low=lower, high=upper, size=(self.Nb, D))
            sampler = EnsembleSampler(self.Nb, D, self.sampling_acquisition_wrapper, batch_lnpostfn=self._sampling_batch)
            self.zb, self.lmb, _ = sampler.run_mcmc(restarts, 50, rstate0=self.rng)
            if not np.any(np.isinf(self.lmb)):
                break
            logger.info("infinite log-probability among the representer points, resampling")
        if np.any(np.isinf(self.lmb)):
            raise ValueError("Could not sample valid representer points! LogEI is -infinity")
        if len(self.zb.shape) == 1:
            self.zb = self.zb[:, None]
        if len(self.lmb.shape) == 1:
            self.lmb = self.lmb[:, None]
        self._append_env_column()
