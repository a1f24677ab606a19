"""BayesianLinearRegression — RoBO's Bayesian linear regression (robo/models/bayesian_linear_regression.py) on the GPU.

Same constructor, attributes (``X``, ``y``, ``X_transformed``, ``hypers``, ``p0``, ``burned``, ``models``) and methods
as the reference.  The hot path of ``train`` is the emcee run over theta = (log alpha, log beta): 20 walkers for 2000
burn-in plus 2000 chain steps, i.e. 80,000 marginal likelihoods on the first train and 40,000 on every later one.  Here
each run is one device call (gpk_blr_sample, robo_b200/csrc/gpk_blr.cuh): one launch per half-step evaluates every
proposal on chip (A = beta Phi^T Phi + alpha I, its Cholesky factor, the residual over all rows and the prior in one CTA
per walker) and takes the stretch move; the final walkers come back in one copy.  The sampler draws from a counter-based
Philox stream seeded from ``self.rng`` once per run, not from emcee's stream: the chain agrees with the reference in
law, not bit for bit.

The weight posteriors (m_i, L_i^-1) stay on the device (gpk_blr_fit); ``models`` holds the (m, S) pairs read back once
per train.  ``predict`` and every device acquisition score through one predictive pass over the candidates, features
made on the device: the basis must be one the device knows (linear, quadratic or none, recognised bit for bit on a
probe matrix), and the prior must be BayesianLinearRegressionPrior.  Divergences from the reference: where a pivot of A
is not positive the log-posterior is -inf (the reference's inv raises LinAlgError), and a NaN log-posterior is
reported as -inf (what the sampler sees in either implementation).
"""
import logging

import numpy as np
from scipy import optimize

from robo_b200 import _lib, priors
from robo_b200.models.base_model import BaseModel

logger = logging.getLogger(__name__)


def linear_basis_func(x):
    return np.append(x, np.ones([x.shape[0], 1]), axis=1)


def quadratic_basis_func(x):
    x = np.append(x ** 2, x, axis=1)
    return np.append(x, np.ones([x.shape[0], 1]), axis=1)


# a probe whose rows exercise signs, fractions and rounding: a basis is recognised by its bits on it
_PROBE = np.array([[0.0, 1.0, -0.5], [0.1, 1.0 / 3.0, 2.0 ** -20], [0.7, -3.25, 0.123456789],
                   [1.0 - 2.0 ** -30, 12.5, -0.9]])


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def basis_code(basis_func):
    """gpk_blr_basis code of a basis function: linear [x, 1], quadratic [x**2, x, 1] or none (None, or a function that
    returns its input).  Any other function raises TypeError: candidates the device maximizers generate get their
    features on the device."""
    if basis_func is None:
        return _lib.BLR_NONE
    try:
        v = np.ascontiguousarray(basis_func(_PROBE.copy()), dtype=np.float64)
    except Exception as e:
        raise TypeError("BayesianLinearRegression: the basis function could not be evaluated on a matrix: %s" % e)
    if _same_bits(v, linear_basis_func(_PROBE.copy())):
        return _lib.BLR_LINEAR
    if _same_bits(v, quadratic_basis_func(_PROBE.copy())):
        return _lib.BLR_QUADRATIC
    if _same_bits(v, _PROBE):
        return _lib.BLR_NONE
    raise TypeError("BayesianLinearRegression runs on the device for three bases only: linear [x, 1], quadratic "
                    "[x**2, x, 1] and none (basis_func=None)")


def prior_constants(prior):
    """(lognormal sigma, lognormal mean, horseshoe scale) of a BayesianLinearRegressionPrior (ours or the reference's
    class); TypeError for any other prior."""
    cls = type(prior)
    mod = cls.__module__ or ""
    if cls.__name__ == "BayesianLinearRegressionPrior" and (mod == priors.__name__ or mod.startswith("robo.priors")):
        return (float(prior.ln_prior_alpha.sigma), float(prior.ln_prior_alpha.mean), float(prior.horseshoe.scale))
    raise TypeError("BayesianLinearRegression restates BayesianLinearRegressionPrior on the device, not %s.%s"
                    % (mod, cls.__name__))


class BayesianLinearRegression(BaseModel):

    def __init__(self, alpha=1, beta=1000, basis_func=linear_basis_func, prior=None, do_mcmc=True, n_hypers=20,
                 chain_length=2000, burnin_steps=2000, rng=None, device=0):
        if rng is None:
            self.rng = np.random.RandomState(np.random.randint(0, 10000))
        else:
            self.rng = rng
        self.X = None
        self.y = None
        self.alpha = alpha
        self.beta = beta
        self.basis_func = basis_func
        if prior is None:
            self.prior = priors.BayesianLinearRegressionPrior(rng=self.rng)
        else:
            self.prior = prior
        prior_constants(self.prior)
        self.do_mcmc = do_mcmc
        self.n_hypers = n_hypers
        self.chain_length = chain_length
        self.burned = False
        self.burnin_steps = burnin_steps
        self.models = None
        self.device = int(device)
        self._handle = None
        self._fitted = False

    # ---- device state: handles do not survive pickling / deepcopy; _ready_handle rebuilds them from host state ------
    def __getstate__(self):
        st = self.__dict__.copy()
        st["_handle"] = None
        st["_fitted"] = False
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)

    def _upload(self):
        """A fresh handle holding the training set (a handle that held a BLR set cannot take a Gaussian process)."""
        code = basis_code(self.basis_func)
        F = _lib.blr_features(self.X.shape[1], code)
        if F > _lib.BLR_MAX_F:
            raise ValueError("BayesianLinearRegression: %d features exceed GPK_BLR_MAX_F = %d (linear basis: D <= %d, "
                             "quadratic: D <= %d)" % (F, _lib.BLR_MAX_F, _lib.BLR_MAX_F - 1, (_lib.BLR_MAX_F - 1) // 2))
        if self._handle is None:
            self._handle = _lib.Handle(self.device)
        self._fitted = False
        _lib.blr_set_data(self._handle, self.X, self.y, code, prior_constants(self.prior))
        return self._handle

    def _ready_handle(self):
        """The handle with the weight posteriors of ``hypers`` resident (scoring entry points take it)."""
        if self.X is None or getattr(self, "hypers", None) is None:
            raise ValueError("BayesianLinearRegression: train the model first")
        if self._handle is None or not self._fitted:
            h = self._upload()
            _lib.blr_fit(h, np.asarray(self.hypers, dtype=np.float64))
            self._fitted = True
        return self._handle

    def marginal_log_likelihood(self, theta):
        """Log likelihood of the data marginalised over the weights plus the prior (:76-113), one gpk_blr_lnpost
        call.  theta: (2,) = (log alpha, log beta)."""
        if self._handle is None:
            self._upload()
        return float(_lib.blr_lnpost(self._handle, np.asarray(theta, dtype=np.float64).reshape(1, 2))[0])

    def negative_mll(self, theta):
        return -self.marginal_log_likelihood(theta)

    @BaseModel._check_shapes_train
    def train(self, X, y, do_optimize=True):
        basis_code(self.basis_func)
        self.X = X
        if self.basis_func is not None:
            self.X_transformed = self.basis_func(X)
        else:
            self.X_transformed = self.X
        self.y = y
        h = self._upload()

        if do_optimize:
            if self.do_mcmc:
                # Do a burn-in in the first iteration
                if not self.burned:
                    # Initialize the walkers by sampling from the prior
                    self.p0 = self.prior.sample_from_prior(self.n_hypers)
                    seed = int(self.rng.randint(0, 2 ** 63, dtype=np.int64))
                    self.p0 = _lib.blr_sample(h, seed, self.p0, self.burnin_steps)["pos"]
                    self.burned = True
                seed = int(self.rng.randint(0, 2 ** 63, dtype=np.int64))
                pos = _lib.blr_sample(h, seed, self.p0, self.chain_length)["pos"]
                # Save the current position, it will be the start point in the next iteration
                self.p0 = pos
                # Take the last samples from each walker
                self.hypers = np.exp(pos)
            else:
                res = optimize.fmin(self.negative_mll, self.rng.rand(2))
                self.hypers = [[np.exp(res[0]), np.exp(res[1])]]
        else:
            self.hypers = [[self.alpha, self.beta]]

        for alpha, beta in self.hypers:
            logger.debug("Alpha=%f ; Beta=%f" % (alpha, beta))
        _lib.blr_fit(h, np.asarray(self.hypers, dtype=np.float64))
        self._fitted = True
        self.models = _lib.blr_models(h)

    @BaseModel._check_shapes_predict
    def predict(self, X_test):
        """Mean of the means and mean of the variances over the hyper-samples, clipped to eps (:213-254): one device
        pass."""
        return self._ready_handle().predict(np.asarray(X_test, dtype=np.float64))
