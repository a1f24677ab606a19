"""GaussianProcess — RoBO's GP model (robo/models/gaussian_process.py) on the GPU path.

Same constructor, attributes and methods as the reference class, so
robo.solver.BayesianOptimization, the maximizers and the acquisition functions use it
unchanged.  What differs is where the arithmetic runs:

  reference (CPU)                                   here (GPU, libgpk.so)
  ------------------------------------------------  ------------------------------------------
  george kernel.get_value: K build, 1 thread        gpk_cov_tma_kernel (fused scaling + Matern/RBF)
  scipy.linalg.cholesky + cho_solve (LAPACK)        blocked right-looking Cholesky, DMMA tiles,
                                                    forward solve fused as an extra block row
  gp.predict: full M x M covariance, then np.diag   fused K* -> L^-1 K*^T -> (mu, var), no M x M
  scipy.stats.norm in ei.py/log_ei.py/pi.py         acquisition closed form in the same epilogue

Hyper-parameter optimisation (gaussian_process.py:193-219) runs where ``hyper_optimizer`` says:
  - "host" (default): scipy L-BFGS-B on the host, as the reference; every nll() evaluation is one gpk_fit, and scipy
    builds each gradient by forward differences, so one optimisation is hundreds of serial fits;
  - "device": the same minimize(nll, p0, method='L-BFGS-B') as one gpk_optimize_hypers call
    (robo_b200/csrc/gpk_hyperopt.cuh): each round scores the trial point and its forward-difference neighbours in one
    launch (the likelihood of one theta per CTA, as gpk_sample_hypers computes it) and runs L-BFGS-B's update on the
    device.  The likelihood is the same function as nll() computed by another routine, so the two arms agree to
    rounding at every point and may part where L-BFGS-B's decisions are that close; it needs N <= GPK_HYPER_MAX_N
    (larger N optimises on the host) and a kernel and prior the device restates;
  - "device_blocked": the same run as one gpk_optimize_hypers_blocked call (robo_b200/csrc/gpk_hyper_blocked.cuh),
    each round's stencil scored by one batched blocked Cholesky over the kernel matrices in device memory, at every N
    up to GPK_HYPER_BLOCKED_MAX_N (8192) and without a fallback.
"""
import logging

import numpy as np
from scipy import optimize

from robo_b200.device_gp import DeviceGP
from robo_b200.models.base_model import BaseModel
from robo_b200.util import normalization

logger = logging.getLogger(__name__)


class GaussianProcess(BaseModel):

    def __init__(self, kernel, prior=None, noise=1e-3, use_gradients=False,
                 normalize_output=False, normalize_input=True,
                 lower=None, upper=None, rng=None, device=0, hyper_optimizer="host"):
        """Arguments as in gaussian_process.py:16-67, plus ``device`` (CUDA ordinal) and ``hyper_optimizer``: "host"
        (default) runs scipy's L-BFGS-B over nll() on the host; "device" runs it as one gpk_optimize_hypers call (see
        the module docstring), "device_blocked" as one gpk_optimize_hypers_blocked call.  Both device values raise
        TypeError for a prior other than None / DefaultPrior / EnvPrior / MTBOPrior or a kernel the device cannot
        represent, and ValueError with use_gradients=True (the BFGS branch has no device path)."""
        from robo_b200.models.gaussian_process_mcmc import HYPER_PATHS, _hyper_kernel, _hyper_prior
        if hyper_optimizer not in HYPER_PATHS:
            raise ValueError("hyper_optimizer must be 'host', 'device' or 'device_blocked', not %r"
                             % (hyper_optimizer,))
        if hyper_optimizer != "host":
            if use_gradients:
                raise ValueError("hyper_optimizer=%r restates L-BFGS-B with finite differences; "
                                 "use_gradients=True (BFGS with grad_nll) runs on the host only" % (hyper_optimizer,))
            _hyper_prior(prior, "hyper_optimizer", hyper_optimizer)
            _hyper_kernel(kernel, "hyper_optimizer", hyper_optimizer)
        self.hyper_optimizer = hyper_optimizer
        self._hyper_handle = None
        self._hyper_fallback_logged = False
        self.hyper_result = None
        if rng is None:
            self.rng = np.random.RandomState(np.random.randint(0, 10000))
        else:
            self.rng = rng
        self.kernel = kernel
        self.gp = None
        self.prior = prior
        self.noise = noise
        self.use_gradients = use_gradients
        self.normalize_output = normalize_output
        self.normalize_input = normalize_input
        self.X = None
        self.y = None
        self.hypers = []
        self.is_trained = False
        self.lower = lower
        self.upper = upper
        self.device = device

    def __getstate__(self):
        st = self.__dict__.copy()
        st["_hyper_handle"] = None
        return st

    # ------------------------------------------------------------------ train
    @BaseModel._check_shapes_train
    def train(self, X, y, do_optimize=True):
        """gaussian_process.py:70-124."""
        self._train_prepare(X, y, do_optimize)
        try:
            self.gp.compute(self.X, yerr=np.sqrt(self.noise))
        except np.linalg.LinAlgError:
            self.noise *= 10
            self.gp.compute(self.X, yerr=np.sqrt(self.noise))
        self.is_trained = True

    # train(do_optimize=False) in two halves, for callers that fit many models at once (GaussianProcessMCMC builds
    # n_hypers sub-models, gaussian_process_mcmc.py:149-164): begin enqueues the factorisation, end collects it
    def train_begin(self, X, y):
        BaseModel._check_shapes_train(lambda s, a, b: None)(self, X, y)
        self._train_prepare(X, y, False)
        self.gp.compute_begin(self.X, yerr=np.sqrt(self.noise))

    def train_end(self):
        try:
            self.gp.compute_end()
        except np.linalg.LinAlgError:                      # :120-122: once more with ten times the noise
            self.noise *= 10
            self.gp.compute(self.X, yerr=np.sqrt(self.noise))
        self.is_trained = True

    def _train_prepare(self, X, y, do_optimize):
        if self.normalize_input:
            self.X, self.lower, self.upper = normalization.zero_one_normalization(X, self.lower, self.upper)
        else:
            self.X = X
        if self.normalize_output:
            self.y, self.y_mean, self.y_std = normalization.zero_mean_unit_var_normalization(y)
            if self.y_std == 0:
                raise ValueError("Cannot normalize output. All targets have the same value")
        else:
            self.y = y

        # the empirical mean of the (standardised) targets is the constant GP mean (:104)
        self.mean = np.mean(self.y, axis=0)

        if self.gp is None or not isinstance(self.gp, DeviceGP):
            self.gp = DeviceGP(self.kernel, mean=self.mean, device=self.device)
        self.gp.kernel = self.kernel
        self.gp.mean = float(self.mean)
        self.gp.set_data(self.X, self.y)
        # test inputs are scaled and moments un-scaled inside the scoring kernels
        if self.normalize_input:
            self.gp.set_input_bounds(self.lower, self.upper)
        else:
            self.gp.set_input_bounds(None, None)
        if self.normalize_output:
            self.gp.set_output_transform(True, self.y_mean, self.y_std)
        else:
            self.gp.set_output_transform(False)

        if do_optimize:
            self.hypers = self.optimize()
            self.gp.kernel.set_parameter_vector(self.hypers[:-1])
            self.noise = np.exp(self.hypers[-1])  # sigma^2
        else:
            self.hypers = self.gp.kernel.get_parameter_vector()
            self.hypers = np.append(self.hypers, np.log(self.noise))

        logger.debug("GP Hyperparameters: " + str(self.hypers))

    def get_noise(self):
        return self.noise

    # ------------------------------------------------------------------ likelihood
    def nll(self, theta):
        """Negative marginal log-likelihood (+ prior), gaussian_process.py:129-166."""
        theta = np.asarray(theta, dtype=np.float64)
        if np.any((-20 > theta) + (theta > 20)):
            return 1e25
        self.gp.kernel.set_parameter_vector(theta[:-1])
        noise = np.exp(theta[-1])  # sigma^2
        try:
            self.gp.compute(self.X, yerr=np.sqrt(noise))
        except np.linalg.LinAlgError:
            return 1e25
        ll = self.gp.log_likelihood(self.y, quiet=True)
        if self.prior is not None:
            ll += self.prior.lnprob(theta)
        return -ll if np.isfinite(ll) else 1e25

    def grad_nll(self, theta):
        """Gradient of nll w.r.t. theta (gaussian_process.py:168-191).  The reference's version is
        dead code (its only caller unpacks an OptimizeResult into three names, :208-210) and uses
        the identity instead of sigma^2 I for the noise slice (:179-182); this is the
        mathematically correct gradient  -1/2 tr((alpha alpha^T - K^-1) dK/dtheta) - prior.gradient,
        computed on the device without materialising dK/dtheta (validated against finite
        differences of nll in the tests)."""
        theta = np.asarray(theta, dtype=np.float64)
        self.gp.kernel.set_parameter_vector(theta[:-1])
        noise = np.exp(theta[-1])
        self.gp.compute(self.X, yerr=np.sqrt(noise))
        g = self.gp.grad_neg_log_likelihood(noise)
        if self.prior is not None:
            g = g - self.prior.gradient(theta)
        return g

    def optimize(self):
        """L-BFGS-B on nll from the current hyper-parameters (gaussian_process.py:193-219)."""
        p0 = self.gp.kernel.get_parameter_vector()
        p0 = np.append(p0, np.log(self.noise))
        if self.use_gradients:
            res = optimize.minimize(self.nll, p0, method="BFGS", jac=self.grad_nll)
            theta = res.x
        elif self._optimize_on_device():
            return self._optimize_device(p0)
        else:
            try:
                results = optimize.minimize(self.nll, p0, method='L-BFGS-B')
                theta = results.x
                self.hyper_result = dict(f=results.fun, nit=results.nit, nfev=results.nfev)
            except ValueError:
                logging.error("Could not find a valid hyperparameter configuration! Use initial configuration")
                theta = p0
        return theta

    def _optimize_on_device(self):
        from robo_b200 import _lib
        if self.hyper_optimizer == "host":
            return False
        if self.hyper_optimizer == "device" and len(self.X) > _lib.HYPER_MAX_N:
            # the device keeps one factor per SM in shared memory: larger N optimises on the host
            if not self._hyper_fallback_logged:
                logger.info("N = %d exceeds GPK_HYPER_MAX_N = %d: the hyper-parameters are optimised on the host",
                            len(self.X), _lib.HYPER_MAX_N)
                self._hyper_fallback_logged = True
            return False
        return True

    def _optimize_device(self, p0):
        """optimize() as one gpk_optimize_hypers (or, for "device_blocked", gpk_optimize_hypers_blocked) call on the
        training set of the handle's last set_data."""
        from robo_b200 import _lib
        from robo_b200.device_gp import TINY
        from robo_b200.kernels import load_kernel
        from robo_b200.models.gaussian_process_mcmc import _hyper_kernel, _hyper_prior
        prior_kind, prior_par, n_ls, n_lr = _hyper_prior(self.prior, "hyper_optimizer", self.hyper_optimizer)
        f = _hyper_kernel(self.gp.kernel, "hyper_optimizer", self.hyper_optimizer)
        if self._hyper_handle is None:
            self._hyper_handle = _lib.Handle(self.device)
        h = self._hyper_handle
        h.set_data(self.X, self.y)
        load_kernel(h, f)
        _lib.set_hyper_model(h, f["slots"], len(f["axis"]), float(self.mean), TINY, prior_kind, prior_par, n_ls, n_lr)
        run = _lib.optimize_hypers_blocked if self.hyper_optimizer == "device_blocked" else _lib.optimize_hypers
        self.hyper_result = run(h, p0)
        return self.hyper_result["theta"]

    # ------------------------------------------------------------------ posterior
    def predict_variance(self, x1, X2):
        """Covariance between x1 and every row of X2 (gaussian_process.py:221-248)."""
        if not self.is_trained:
            raise Exception('Model has to be trained first!')
        x_ = np.concatenate((x1, X2))
        _, var = self.predict(x_, full_cov=True)
        return var[-1, :-1, np.newaxis]

    @BaseModel._check_shapes_predict
    def predict(self, X_test, full_cov=False, **kwargs):
        """Predictive mean and variance (or full covariance), gaussian_process.py:251-296.
        Input scaling, output un-scaling and the eps clip happen on the device."""
        if not self.is_trained:
            raise Exception('Model has to be trained first!')
        if full_cov:
            return self.gp.predict_cov(X_test)
        return self.gp.predict_moments(X_test)

    def device_inputs(self, X_test):
        """What the device handle expects for the raw inputs X_test (the handle applies the [lower, upper] scaling
        itself); subclasses that transform inputs on the host (FabolasGP) return the transformed array."""
        return X_test

    def input_gradient(self, X_test, G):
        """A gradient G (M, D) with respect to device_inputs(X_test), taken back to the raw inputs X_test by the
        chain rule; the identity here, where the handle applies (and differentiates) the input scaling itself."""
        return G

    def score(self, X_test, kind, eta=None, par=0.0, want_values=True):
        """Fused predict -> acquisition -> arg-max used by robo_b200.acquisition_functions.
        ``kind``: one of 'ei', 'log_ei', 'pi', 'lcb'."""
        from robo_b200 import _lib
        if not self.is_trained:
            raise Exception('Model has to be trained first!')
        assert len(X_test.shape) == 2
        if eta is None:
            eta = 0.0 if kind == "lcb" else self.get_incumbent()[1]
        return self.gp.score(X_test, _lib.ACQ_KIND[kind], eta=float(eta), par=float(par),
                             want_values=want_values)

    def predictive_gradients(self, X_test):
        """d mu / d x and d var / d x at X_test, shapes (M, D) each.  This is the method the
        reference's acquisition functions call when ``derivative=True`` (ei.py:80-85, pi.py:65-71,
        lcb.py:66-69) and that none of its models provides (SURVEY.md section 8f rank 3)."""
        if not self.is_trained:
            raise Exception('Model has to be trained first!')
        assert len(X_test.shape) == 2
        r = self.gp.predict_grad(self.device_inputs(X_test))
        return self.input_gradient(X_test, r["dmu"]), self.input_gradient(X_test, r["dvar"])

    def score_with_gradient(self, X_test, kind, eta=None, par=0.0):
        """(f (M,), df (M, D)) for 'ei', 'pi', 'lcb' — value and input gradient of the acquisition."""
        from robo_b200 import _lib
        if not self.is_trained:
            raise Exception('Model has to be trained first!')
        if eta is None:
            eta = 0.0 if kind == "lcb" else self.get_incumbent()[1]
        r = self.gp.predict_grad(self.device_inputs(X_test), _lib.ACQ_KIND[kind], float(eta), float(par))
        return r["f"], self.input_gradient(X_test, r["df"])

    def sample_functions(self, X_test, n_funcs=1):
        """Posterior function samples at X_test (gaussian_process.py:298-332): mean and
        covariance from the device, the multivariate-normal draw with numpy like george."""
        if not self.is_trained:
            raise Exception('Model has to be trained first!')
        # the raw (unclipped) posterior covariance, like george's sample_conditional at :324: predict()'s eps clip
        # would erase every negative posterior correlation
        mu, cov = self.gp.posterior_cov(X_test)
        funcs = np.random.multivariate_normal(mu, cov, n_funcs) if n_funcs > 1 \
            else np.random.multivariate_normal(mu, cov)
        if len(funcs.shape) == 1:
            return funcs[None, :]
        return funcs

    def get_incumbent(self):
        """Best observed point, un-scaled (gaussian_process.py:334-352)."""
        inc, inc_value = super(GaussianProcess, self).get_incumbent()
        if self.normalize_input:
            inc = normalization.zero_one_unnormalization(inc, self.lower, self.upper)
        if self.normalize_output:
            inc_value = normalization.zero_mean_unit_var_unnormalization(inc_value, self.y_mean, self.y_std)
        return inc, inc_value
