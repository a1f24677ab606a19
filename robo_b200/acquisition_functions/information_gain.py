"""InformationGain — the entropy-search acquisition of robo/acquisition_functions/information_gain.py:19-272 (Hennig
and Schuler, JMLR 2012) with its numerical work on the GPU.

update(): the representer points zb are drawn by the ensemble sampler from the sampling acquisition (each
half-ensemble scored in ONE call of the fused acquisition), or with representer_sampler="device" by the stretch move on
the device (gpk_sample_representers: the same algorithm, a Philox stream, equal in law only); p_min over zb by EP, the derivatives of log p_min and
U = K^-1 K(X, zb) are computed and kept on the device (gpk_es_update).  compute(): the entropy change of every
candidate in one batched call (gpk_es_compute): the reference loops over candidates with one predict and one
(Nb + 1)-point predict(full_cov=True) each.  innovations() stays a host method, as in the reference.

Serves robo_b200 GaussianProcess models whose inputs go to the device untransformed; marginalised over a GP-MCMC
ensemble by MarginalizationGPMCMC (one estimator, with its own representer points, per sub-model).
"""
import logging

import numpy as np
import scipy.stats

from robo_b200.acquisition_functions.base_acquisition import BaseAcquisitionFunction
from robo_b200.acquisition_functions.log_ei import LogEI
from robo_b200.util.ensemble_sampler import EnsembleSampler

logger = logging.getLogger(__name__)


def _device_model(model):
    from robo_b200.maximizers.device_spec import raw_inputs as _raw_inputs
    if not _raw_inputs(model) or not hasattr(getattr(model, "gp", None), "handle"):
        raise TypeError("InformationGain runs on robo_b200 GaussianProcess models whose inputs go to the device "
                        "untransformed")
    model.gp._restore()
    model.gp._push_cfg()
    return model.gp.handle


_DEVICE_KINDS = ("ei", "log_ei", "pi", "lcb")


def sample_representers_device(estimators):
    """The representer points of every estimator (InformationGain or InformationGainPerUnitCost) drawn on the device by
    the stretch move (gpk_sample_representers), one call for all estimators that share the sampler's arguments.  Each
    estimator draws its seed from its own rng (one draw per update); eta is its sampling acquisition's incumbent value
    (0 for LCB); the stretch move runs the estimator's REPRESENTER_STEPS steps for at most REPRESENTER_RUNS runs (50 and 5
    for InformationGain, 200 and 1 for InformationGainMC), which join the grouping key.  Raises TypeError when an
    estimator cannot sample on the device, and the reference's ValueErrors: ei.py's on a negative EI value, and
    InformationGainPerUnitCost's when -inf remains after 5 runs."""
    from robo_b200 import _lib
    calls = {}
    for e in estimators:
        sa = e.sampling_acquisition
        kind = getattr(sa, "kind", None)
        if kind not in _DEVICE_KINDS or not hasattr(sa, "par"):
            raise TypeError("representer_sampler='device' needs EI, LogEI, PI or LCB as the sampling acquisition")
        sa.update(e.model)
        handle, lower, upper, fabolas = e._representer_spec()
        eta = 0.0 if kind == "lcb" else float(e.model.get_incumbent()[1])
        seed = int(e.rng.randint(0, 2 ** 63, dtype=np.int64))
        steps, runs = int(e.REPRESENTER_STEPS), int(e.REPRESENTER_RUNS)
        key = (kind, float(sa.par), int(e.Nb), steps, runs, lower.tobytes(), upper.tobytes(),
               None if fabolas is None else tuple((k, np.asarray(v).tobytes()) for k, v in sorted(fabolas.items())))
        calls.setdefault(key, (kind, float(sa.par), int(e.Nb), steps, runs, lower, upper, fabolas, []))[-1].append(
            (e, handle, seed, eta))
    for kind, par, nb, steps, runs, lower, upper, fabolas, members in calls.values():
        r = _lib.sample_representers([m[1] for m in members], [m[2] for m in members], nb, steps, runs,
                                     _lib.ACQ_KIND[kind],
                                     [m[3] for m in members], par, lower, upper, fabolas=fabolas)
        if kind == "ei" and r["n_negative"] > 0:
            raise ValueError("Expected Improvement is smaller than 0!")      # ei.py:86-88
        for i, (e, _, _, _) in enumerate(members):
            e._set_representers(r["zb"][i], r["lmb"][i])


class InformationGain(BaseAcquisitionFunction):

    # the stretch move of the representer points (information_gain.py:68-81): at most 5 runs of 50 steps
    REPRESENTER_STEPS, REPRESENTER_RUNS = 50, 5

    def __init__(self, model, lower, upper, Nb=50, Np=400, sampling_acquisition=None,
                 sampling_acquisition_kw={"par": 0.0}, rng=None, representer_sampler="host", **kwargs):
        if representer_sampler not in ("host", "device"):
            raise ValueError("representer_sampler must be 'host' or 'device', not %r" % (representer_sampler,))
        self.representer_sampler = representer_sampler
        self.Nb = Nb
        super(InformationGain, self).__init__(model)
        self.lower = lower
        self.upper = upper
        self.D = self.lower.shape[0]
        self.sn2 = None
        if sampling_acquisition is None:
            sampling_acquisition = LogEI
        self.sampling_acquisition = sampling_acquisition(model, **sampling_acquisition_kw)
        self.Np = Np
        if rng is None:
            self.rng = np.random.RandomState(np.random.randint(0, 10000))
        else:
            self.rng = rng
        self.zb = self.lmb = None

    def sampling_acquisition_wrapper(self, x):
        if np.any(x < self.lower) or np.any(x > self.upper):
            return -np.inf
        return self.sampling_acquisition(np.array([x]))[0]

    def _sampling_batch(self, X):
        """The wrapper's one-point semantics over a whole half-ensemble, scored in one call."""
        out = np.full(X.shape[0], -np.inf)
        inside = np.all((X >= self.lower) & (X <= self.upper), axis=1)
        if np.any(inside):
            out[inside] = np.asarray(self.sampling_acquisition(X[inside]), dtype=np.float64).ravel()
        return out

    def sample_representer_points(self):
        if self.representer_sampler == "device":
            sample_representers_device([self])
            return
        self.sampling_acquisition.update(self.model)
        for i in range(5):
            restarts = self.lower + (self.upper - self.lower) * self.rng.uniform(size=(self.Nb, self.D))
            sampler = EnsembleSampler(self.Nb, self.D, self.sampling_acquisition_wrapper,
                                      batch_lnpostfn=self._sampling_batch)
            self.zb, self.lmb, _ = sampler.run_mcmc(restarts, 50, rstate0=self.rng)
            if not np.any(np.isinf(self.lmb)):
                break
            logger.info("infinite log-probability among the representer points, resampling")
        if len(self.zb.shape) == 1:
            self.zb = self.zb[:, None]
        if len(self.lmb.shape) == 1:
            self.lmb = self.lmb[:, None]

    # the model's device handle, and zb as that handle takes its inputs (InformationGainPerUnitCost: FabolasGP models)
    def _device_handle(self, model):
        return _device_model(model)

    def _device_zb(self):
        return self.zb

    # the device sampler's view of this estimator: its handle, the walker box and the Fabolas arguments (None here)
    def _representer_spec(self):
        return self._device_handle(self.model), np.asarray(self.lower, dtype=np.float64), \
            np.asarray(self.upper, dtype=np.float64), None

    def _set_representers(self, zb, lmb):
        self.zb, self.lmb = zb, lmb[:, None]

    def update(self, model):
        handle = self._begin_update(model)
        self.sample_representer_points()
        self._end_update(handle)

    # update() around the representer points, so that MarginalizationGPMCMC can draw those of all estimators in one call
    def _begin_update(self, model):
        self.model = model
        handle = self._device_handle(model)
        self.sn2 = self.model.get_noise()
        return handle

    def _end_update(self, handle):
        self.W = scipy.stats.norm.ppf(np.linspace(1. / (self.Np + 1), 1 - 1. / (self.Np + 1), self.Np))[np.newaxis, :]
        r = handle.es_update(self._device_zb(), self.lmb, self.sn2, self.W, self.lower, self.upper)
        self.logP = np.reshape(r["logP"], (self.Nb, 1))
        self.dlogPdMu, self.dlogPdSigma, self.dlogPdMudMu = r["dlogPdMu"], r["dlogPdSigma"], r["dlogPdMudMu"]

    def compute(self, X_test, derivative=False, **kwargs):
        """Entropy change of every row of X_test -> (N,).  derivative=True is not implemented (the reference's finite
        differences are marked "Not tested!")."""
        if derivative:
            raise NotImplementedError("InformationGain has no derivative on the GPU path")
        return self._ready_handle().es_compute(np.asarray(X_test, dtype=np.float64))

    def _ready_handle(self):
        """The device handle compute() scores on, after compute()'s checks (ValueError before update() or with an
        infinite lmb)."""
        if self.zb is None:
            raise ValueError("InformationGain.compute needs update() first")
        if not np.all(np.isfinite(self.lmb)):
            raise ValueError("lmb should not be infinite.")
        return _device_model(self.model)

    def argmax(self, X_test):
        return int(np.argmax(self.compute(X_test)))

    def dh_fun(self, x, derivative=False):
        if derivative:
            raise NotImplementedError("InformationGain has no derivative on the GPU path")
        if not np.all(np.isfinite(self.lmb)):
            raise ValueError("lmb should not be infinite.")
        if len(x.shape) == 1:
            x = x[np.newaxis]
        if np.any(x < self.lower) or np.any(x > self.upper):
            return np.array([[np.spacing(1)]]), np.array([[np.zeros((x.shape[1], 1))]])
        return self.compute(x[:1])

    def innovations(self, x, rep):
        _, v = self.model.predict(x)
        v = v.reshape(-1, 1)
        v_ = v - self.sn2
        sigma_x_rep = self.model.predict_variance(rep, x)
        norm_cov = np.dot(sigma_x_rep, np.linalg.inv(v_))
        dm_rep = np.dot(norm_cov, np.linalg.cholesky(v + 1e-10))
        dv_rep = -norm_cov.dot(sigma_x_rep.T)
        return dm_rep, dv_rep
