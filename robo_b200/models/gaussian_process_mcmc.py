"""GaussianProcessMCMC — RoBO's GP with MCMC-marginalised hyper-parameters
(robo/models/gaussian_process_mcmc.py) on the GPU path.

Same constructor, attributes (`models`, `hypers`, `p0`, `burned`, ...) and methods as the
reference.  The cost of `train` is `n_hypers x (burnin + chain)` evaluations of
`loglikelihood` (K build + Cholesky each, :168-202), which the reference runs one after the other
on the CPU.  Here every half-ensemble of walkers is evaluated together: one gpk handle (own CUDA
stream) per proposal, `gpk_fit_begin` on all of them, then `gpk_fit_end` — the latency-bound
factorisation chains overlap on the GPU (SURVEY.md section 8f rank 1).

``hyper_sampler="device"`` runs each ``run_mcmc`` of ``train`` (burn-in, then chain) as one device call instead
(gpk_sample_hypers, robo_b200/csrc/gpk_hyper.cuh): one launch evaluates the initial walkers, one launch per half-step
proposes, evaluates the log-posteriors on chip (kernel, Cholesky and prior in one CTA per walker) and accepts; the
final positions come back in one copy.  It draws from a counter-based Philox stream seeded from ``self.rng`` once per
run, not from numpy's stream: the two samplers agree in law, not bit for bit, which is why ``"host"`` stays the default.
It needs N <= GPK_HYPER_MAX_N (232); larger N samples on the host.

``hyper_sampler="device_blocked"`` is the same run (gpk_sample_hypers_blocked, robo_b200/csrc/gpk_hyper_blocked.cuh)
with each half-ensemble's log-posteriors computed by one batched blocked Cholesky over the walkers' kernel matrices in
device memory, at every N up to GPK_HYPER_BLOCKED_MAX_N (8192) and without a fallback.
"""
import logging
from copy import deepcopy

import numpy as np

from robo_b200 import _lib, priors
from robo_b200.device_gp import DeviceGP, TINY
from robo_b200.kernels import load_kernel
from robo_b200.models.base_model import BaseModel
from robo_b200.models.gaussian_process import GaussianProcess
from robo_b200.util import normalization
from robo_b200.util.ensemble_sampler import EnsembleSampler

logger = logging.getLogger(__name__)


class _LikelihoodPool(object):
    """B handles sharing one training set; evaluates log-likelihoods of B thetas concurrently."""

    def __init__(self, kernel, X, y, mean, size, device=0):
        self.kernel = deepcopy(kernel)
        self.mean = float(mean)
        self.handles = []
        for _ in range(size):
            h = _lib.Handle(device)
            h.set_data(X, y)
            self.handles.append(h)

    def loglik(self, thetas):
        """thetas: (B', H) with B' <= pool size -> log-likelihoods (no prior), -inf where not PD."""
        out = np.full(len(thetas), -np.inf)
        started = []
        try:
            for i, theta in enumerate(thetas):
                if np.any((-20 > theta) + (theta > 20)):           # gaussian_process_mcmc.py:187-188
                    continue
                h = self.handles[i]
                try:                                                # :194-197: any failure of one theta is -inf for it
                    self.kernel.set_parameter_vector(theta[:-1])
                    load_kernel(h, self.kernel.flatten())
                    yerr = np.sqrt(np.exp(theta[-1]))
                    diag_add = float(np.sqrt(np.float64(yerr) ** 2 + TINY) ** 2)
                    h.fit_begin(diag_add, self.mean)
                except (ValueError, RuntimeError, np.linalg.LinAlgError):
                    continue
                started.append(i)
        finally:
            # every handle that started a factorisation is drained, whatever happened to the others
            for i in started:
                try:
                    _, ll = self.handles[i].fit_end()
                    out[i] = ll if np.isfinite(ll) else -np.inf
                except (np.linalg.LinAlgError, ValueError, RuntimeError):
                    out[i] = -np.inf
        return out

    def close(self):
        for h in self.handles:
            h.close()
        self.handles = []


def _hyper_prior(prior, option="hyper_sampler", value="device"):
    """(gpk_prior_kind, the 7 constants, n_ls, n_lr) of a prior the device restates: None, DefaultPrior, EnvPrior or
    MTBOPrior (the reference's classes or robo_b200.priors'); TypeError, naming `option` and its `value`, for any
    other."""
    if prior is None:
        return _lib.PRIOR_NONE, None, 0, 0
    cls = type(prior)
    mod = cls.__module__ or ""
    ours = mod == priors.__name__ or mod.startswith("robo.priors")
    if ours and cls.__name__ in ("DefaultPrior", "EnvPrior"):
        par = [prior.ln_prior.sigma, prior.ln_prior.mean, prior.tophat.min, prior.tophat.max, prior.horseshoe.scale,
               0.0, 0.0]
        if cls.__name__ == "DefaultPrior":
            return _lib.PRIOR_DEFAULT, par, 0, 0
        par[5:] = [prior.bayes_lin_prior.sigma, prior.bayes_lin_prior.mean]
        return _lib.PRIOR_ENV, par, int(prior.n_ls), int(prior.n_lr)
    if ours and cls.__name__ == "MTBOPrior":
        par = [prior.ln_prior.sigma, prior.ln_prior.mean, prior.tophat.min, prior.tophat.max, prior.horseshoe.scale,
               prior.tophat_task.min, prior.tophat_task.max]
        return _lib.PRIOR_MTBO, par, int(prior.n_ls), int(prior.n_kt)
    raise TypeError("%s=%r restates None, DefaultPrior, EnvPrior and MTBOPrior only, not %s.%s"
                    % (option, value, mod, cls.__name__))


def _hyper_kernel(kernel, option="hyper_sampler", value="device"):
    """kernel.flatten(), or TypeError, naming `option` and its `value`, when the device cannot represent the kernel."""
    try:
        return kernel.flatten()
    except Exception as e:
        raise TypeError("%s=%r cannot represent this kernel: %s" % (option, value, e))


# the values of hyper_sampler and hyper_optimizer
HYPER_PATHS = ("host", "device", "device_blocked")


class GaussianProcessMCMC(BaseModel):

    def __init__(self, kernel, prior=None, n_hypers=20, chain_length=2000, burnin_steps=2000,
                 normalize_output=False, normalize_input=True,
                 rng=None, lower=None, upper=None, noise=-8, device=0, hyper_sampler="host"):
        """Arguments as in gaussian_process_mcmc.py:17-70, plus ``device`` and ``hyper_sampler``: "host" (default)
        runs EnsembleSampler with numpy's stream, as before; "device" runs each run_mcmc on the device
        (gpk_sample_hypers) with its own Philox stream, so the two agree in law, not bit for bit.  A train whose N
        exceeds GPK_HYPER_MAX_N falls back to the host sampler.  "device_blocked" runs the same chain through
        gpk_sample_hypers_blocked at every N up to GPK_HYPER_BLOCKED_MAX_N, with no fallback.  Both device values raise
        TypeError for a prior other than None / DefaultPrior / EnvPrior / MTBOPrior or a kernel the device cannot
        represent."""
        if hyper_sampler not in HYPER_PATHS:
            raise ValueError("hyper_sampler must be 'host', 'device' or 'device_blocked', not %r" % (hyper_sampler,))
        if hyper_sampler != "host":
            _hyper_prior(prior, value=hyper_sampler)
            _hyper_kernel(kernel, value=hyper_sampler)
        self.hyper_sampler = hyper_sampler
        self._hyper_handle = None
        self._hyper_fallback_logged = False
        if rng is None:
            self.rng = np.random.RandomState(np.random.randint(0, 10000))
        else:
            self.rng = rng
        self.kernel = kernel
        self.prior = prior
        self.noise = noise
        self.n_hypers = n_hypers
        self.chain_length = chain_length
        self.burned = False
        self.burnin_steps = burnin_steps
        self.models = []
        self.normalize_output = normalize_output
        self.normalize_input = normalize_input
        self.X = None
        self.y = None
        self.is_trained = False
        self.lower = lower
        self.upper = upper
        self.device = device
        self._pool = None

    def __getstate__(self):
        st = self.__dict__.copy()
        st["_pool"] = None
        st["_hyper_handle"] = None
        return st

    @BaseModel._check_shapes_train
    def train(self, X, y, do_optimize=True, **kwargs):
        """gaussian_process_mcmc.py:76-166."""
        self.X = self._likelihood_inputs(X)
        if self.normalize_output:
            self.y, self.y_mean, self.y_std = normalization.zero_mean_unit_var_normalization(y)
            if self.y_std == 0:
                raise ValueError("Cannot normalize output. All targets have the same value")
        else:
            self.y = y
        self.mean = np.mean(self.y, axis=0)
        self.gp = DeviceGP(self.kernel, mean=self.mean, device=self.device)
        self.gp.set_data(self.X, self.y)

        on_device = do_optimize and self.hyper_sampler != "host"
        if on_device and self.hyper_sampler == "device" and len(self.X) > _lib.HYPER_MAX_N:
            # the device keeps one factor per SM in shared memory: larger N samples on the host for this train
            if not self._hyper_fallback_logged:
                logger.info("N = %d exceeds GPK_HYPER_MAX_N = %d: the hyper-parameters are sampled on the host",
                            len(self.X), _lib.HYPER_MAX_N)
                self._hyper_fallback_logged = True
            on_device = False
        if on_device:
            self._sample_hypers_device()
        elif do_optimize:
            if self._pool is not None:
                self._pool.close()
            self._pool = _LikelihoodPool(self.kernel, self.X, self.y, self.mean, self.n_hypers // 2, self.device)
            sampler = EnsembleSampler(self.n_hypers, len(self.kernel) + 1, self.loglikelihood,
                                      batch_lnpostfn=self.loglikelihood_batch)
            if not self.burned:
                if self.prior is None:
                    self.p0 = self.rng.rand(self.n_hypers, len(self.kernel) + 1)
                else:
                    self.p0 = self.prior.sample_from_prior(self.n_hypers)
                self.p0, _, _ = sampler.run_mcmc(self.p0, self.burnin_steps, rstate0=self.rng)
                self.burned = True
            pos, _, _ = sampler.run_mcmc(self.p0, self.chain_length, rstate0=self.rng)
            self.p0 = pos
            self.hypers = sampler.chain[:, -1]
            self.n_lnprob_calls = sampler.n_lnprob_calls
            self._pool.close()
            self._pool = None
        else:
            self.hypers = self._hypers_without_optimisation()

        self.models = []
        for sample in self.hypers:
            kernel = deepcopy(self.kernel)
            kernel.set_parameter_vector(sample[:-1])
            noise = np.exp(sample[-1])
            self.models.append(self._new_sub_model(kernel, noise))
        # all n_hypers factorisations are enqueued (one handle / stream per sub-model) before the first is collected:
        # the latency-bound Cholesky chains overlap on the GPU (gaussian_process_mcmc.py:163 trains them one by one)
        for model in self.models:
            model.train_begin(X, y)
        for model in self.models:
            model.train_end()
        self.is_trained = True

    def _sample_hypers_device(self):
        """train's MCMC phase on the device: the same p0 / burn-in / chain bookkeeping as the host path, each run_mcmc
        one gpk_sample_hypers (or, for "device_blocked", gpk_sample_hypers_blocked) call seeded from self.rng."""
        prior_kind, prior_par, n_ls, n_lr = _hyper_prior(self.prior, value=self.hyper_sampler)
        f = _hyper_kernel(self.kernel, value=self.hyper_sampler)
        sample = _lib.sample_hypers_blocked if self.hyper_sampler == "device_blocked" else _lib.sample_hypers
        dim = len(self.kernel) + 1
        if self._hyper_handle is None:
            self._hyper_handle = _lib.Handle(self.device)
        h = self._hyper_handle
        h.set_data(self.X, self.y)
        load_kernel(h, f)
        _lib.set_hyper_model(h, f["slots"], len(f["axis"]), float(self.mean), TINY, prior_kind, prior_par, n_ls, n_lr)

        def run(p0, steps):
            seed = int(self.rng.randint(0, 2 ** 63, dtype=np.int64))
            return sample(h, p0, steps, seed)["pos"]
        calls = 0
        if not self.burned:
            if self.prior is None:
                self.p0 = self.rng.rand(self.n_hypers, dim)
            else:
                self.p0 = self.prior.sample_from_prior(self.n_hypers)
            self.p0 = run(self.p0, self.burnin_steps)
            calls += self.n_hypers * (self.burnin_steps + 1)
            self.burned = True
        self.p0 = run(self.p0, self.chain_length)
        calls += self.n_hypers * (self.chain_length + 1)
        self.hypers = self.p0.copy()
        self.n_lnprob_calls = calls

    # hooks for FabolasGPMCMC (robo/models/fabolas_gp.py), which differs only in how inputs are prepared
    def _likelihood_inputs(self, X):
        """Inputs the MCMC phase factorises (gaussian_process_mcmc.py:95-99)."""
        if self.normalize_input:
            Xn, self.lower, self.upper = normalization.zero_one_normalization(X, self.lower, self.upper)
            return Xn
        return X

    def _hypers_without_optimisation(self):
        """gaussian_process_mcmc.py:144-147: the kernel's current parameters + the configured log-noise."""
        hypers = self.gp.kernel[:].tolist()
        hypers.append(self.noise)
        return [hypers]

    def _new_sub_model(self, kernel, noise):
        """One GP per hyper-parameter sample (gaussian_process_mcmc.py:156-162)."""
        return GaussianProcess(kernel, normalize_output=self.normalize_output, normalize_input=self.normalize_input,
                               noise=noise, lower=self.lower, upper=self.upper, rng=self.rng, device=self.device)

    def loglikelihood(self, theta):
        """Log-likelihood + prior of one theta (gaussian_process_mcmc.py:168-202)."""
        theta = np.asarray(theta, dtype=np.float64)
        if np.any((-20 > theta) + (theta > 20)):
            return -np.inf
        sigma_2 = np.exp(theta[-1])
        self.gp.kernel.set_parameter_vector(theta[:-1])
        try:
            self.gp.compute(self.X, yerr=np.sqrt(sigma_2))
        except Exception:
            return -np.inf
        ll = self.gp.log_likelihood(self.y, quiet=True)
        if self.prior is not None:
            return self.prior.lnprob(theta) + ll
        return ll

    def loglikelihood_batch(self, thetas):
        """The same for a batch of thetas (one half-ensemble), factorisations overlapped on the GPU."""
        thetas = np.asarray(thetas, dtype=np.float64)
        if self._pool is None or len(thetas) > len(self._pool.handles):
            return np.array([self.loglikelihood(t) for t in thetas])
        ll = self._pool.loglik(thetas)
        if self.prior is not None:
            for i, t in enumerate(thetas):
                if np.isfinite(ll[i]):
                    ll[i] = self.prior.lnprob(t) + ll[i]
        return ll

    @BaseModel._check_shapes_predict
    def predict(self, X_test, **kwargs):
        """Mixture moments over the hyper-parameter samples (gaussian_process_mcmc.py:205-249):
        m = mean_i mu_i ; v = var_i(mu_i) + mean_i var_i, clipped.  Per-model moments come from the
        fused GPU predict, the reduction over models runs on the GPU too (gpk_reduce_models)."""
        if not self.is_trained:
            raise Exception('Model has to be trained first!')
        handles = self.sub_model_handles()
        if handles is not None:
            # one H2D of X_test, every sub-model scores it on its own stream, the mixture moments are reduced on the
            # device: 2 M doubles come back instead of 2 n_hypers M (gpk_acq_multi mode 1)
            r = _lib.acq_multi(handles, self.models[0].device_inputs(np.asarray(X_test, dtype=np.float64)), 1)
            return r["mean"], r["var"]
        mu = np.zeros([len(self.models), X_test.shape[0]])
        var = np.zeros([len(self.models), X_test.shape[0]])
        for i, model in enumerate(self.models):
            mu[i], var[i] = model.predict(X_test)
        return _lib.moments_handle(self.device).reduce_models(mu, var)

    def sub_model_handles(self):
        """The fitted gpk handles of the hyper-parameter samples (device state restored / configuration pushed), or
        None when a sub-model is not a device GP (then callers loop over the models like the reference does)."""
        handles = []
        for model in self.models:
            gp = getattr(model, "gp", None)
            if not isinstance(gp, DeviceGP) or not getattr(model, "is_trained", False):
                return None
            gp._restore()
            if not gp.computed:
                return None
            gp._push_cfg()
            handles.append(gp.handle)
        return handles if handles else None

    def get_incumbent(self):
        """gaussian_process_mcmc.py:251-269."""
        inc, inc_value = super(GaussianProcessMCMC, self).get_incumbent()
        if self.normalize_input:
            inc = normalization.zero_one_unnormalization(inc, self.lower, self.upper)
        if self.normalize_output:
            inc_value = normalization.zero_mean_unit_var_unnormalization(inc_value, self.y_mean, self.y_std)
        return inc, inc_value
