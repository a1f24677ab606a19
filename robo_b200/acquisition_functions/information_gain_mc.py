"""InformationGainMC — the sampling-based ("asymptotically exact") entropy search of
robo/acquisition_functions/information_gain_mc.py (Hennig and Schuler, JMLR 2012) with its numerical work on the GPU.

update(): the representer points zb are drawn as the reference draws them (200 stretch-move steps, one run, walkers
started uniformly in the box), on the host through the sampling acquisition or with representer_sampler="device" by
gpk_sample_representers; then gpk_esmc_update computes Mb, Vb = predict(zb, full_cov=True), draws F (Nb x Nf) from a
seed that ``self.rng`` gives once per update, and p_min at (Mb, Vb) by joint_pmin.  compute(): the entropy change of
every candidate in one batched call (gpk_esmc_compute): one Nb x Nb factorisation, Nf correlated draws and an arg-min
over Nf Np columns per candidate, all on the device.

The reference cannot run as written (DESIGN.md §1 lists the repairs); this port implements what it plainly means:
    value(x) = sum_i new_i (log new_i + lmb_i) + H,   H = -sum_i exp(logP_i) (logP_i + lmb_i),
with new = joint_pmin(Mb + dm W, Vb + dv, Nf) under the innovations of InformationGain; larger means more information.
Deviation: one F per update serves the update and every candidate (common random numbers), so compute(x) is a
deterministic function of x between updates; each value still has the reference's marginal law.  Each estimator of a
MarginalizationGPMCMC has its own seed and its own F.
"""
import numpy as np
import scipy.stats

from robo_b200.acquisition_functions.information_gain import InformationGain
from robo_b200.util.ensemble_sampler import EnsembleSampler
from robo_b200.util.mc_part import draw_seed


class InformationGainMC(InformationGain):

    # the reference's sampler (information_gain_mc.py:84-91): one run of 200 steps
    REPRESENTER_STEPS, REPRESENTER_RUNS = 200, 1

    def __init__(self, model, lower, upper, Nb=50, Nf=500, sampling_acquisition=None,
                 sampling_acquisition_kw={"par": 0.0}, Np=50, rng=None, representer_sampler="host", **kwargs):
        super(InformationGainMC, self).__init__(model, lower, upper, Nb=Nb, Np=Np,
                                                sampling_acquisition=sampling_acquisition,
                                                sampling_acquisition_kw=sampling_acquisition_kw, rng=rng,
                                                representer_sampler=representer_sampler)
        self.Nf = Nf
        self.seed = None
        # MarginalizationGPMCMC numbers its deep-copied estimators, whose rngs start equal: the stream index keeps
        # their draws apart
        self.stream = 0

    def sample_representer_points(self):
        if self.representer_sampler == "device":
            from robo_b200.acquisition_functions.information_gain import sample_representers_device
            sample_representers_device([self])
            return
        self.sampling_acquisition.update(self.model)
        start = self.lower + (self.upper - self.lower) * self.rng.uniform(size=(self.Nb, self.D))
        sampler = EnsembleSampler(self.Nb, self.D, self.sampling_acquisition_wrapper,
                                  batch_lnpostfn=self._sampling_batch)
        self.zb, self.lmb, _ = sampler.run_mcmc(start, self.REPRESENTER_STEPS, rstate0=self.rng)
        if len(self.zb.shape) == 1:
            self.zb = self.zb[:, None]
        if len(self.lmb.shape) == 1:
            self.lmb = self.lmb[:, None]

    def _end_update(self, handle):
        if not np.all(np.isfinite(self.lmb)):
            raise ValueError("lmb should not be infinite.")
        self.W = scipy.stats.norm.ppf(np.linspace(1. / (self.Np + 1), 1 - 1. / (self.Np + 1), self.Np))[np.newaxis, :]
        self.seed = (draw_seed(self.rng) + 0x9E3779B97F4A7C15 * int(self.stream)) & 0xFFFFFFFFFFFFFFFF
        r = handle.esmc_update(self._device_zb(), self.lmb, self.sn2, self.W, self.Nf, self.seed)
        self.pmin = r["pmin"]
        self.logP = np.reshape(r["logP"], (self.Nb, 1))

    def compute(self, X_test, derivative=False, **kwargs):
        """Sampling-based entropy change of every row of X_test -> (N,).  derivative=True is not implemented, as in the
        reference."""
        if derivative:
            raise NotImplementedError("InformationGainMC has no derivative")
        return self._ready_handle().esmc_compute(np.asarray(X_test, dtype=np.float64))

    def dh_fun(self, x, derivative=False):
        raise NotImplementedError("InformationGainMC has no dh_fun; use compute()")
