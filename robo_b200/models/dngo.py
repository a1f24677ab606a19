"""DNGO — pybnn's DNGO (Snoek et al., "Scalable Bayesian Optimization Using Deep Neural Networks", ICML 2015), the
surrogate robo/fmin/bayesian_optimization.py:105-109 builds for model_type="dngo", on the GPU without pybnn.

Same constructor as pybnn's, plus ``device``; ``train(X, y, do_optimize=True)``, ``predict(X_test)`` and
``get_incumbent``.  pybnn's source is not available, so the model is restated (robo_b200/csrc/gpk_dngo.cuh states it
step by step, DESIGN §1 row a29):

* a D -> 50 -> 50 -> 50 -> 1 tanh network with torch's nn.Linear initialisation, trained by Adam (torch's defaults,
  learning rate ``learning_rate``) on the mean squared error of minibatches of min(batch_size, N) rows for
  ``num_epochs`` epochs, each epoch a fresh order of the rows in full batches with the remainder dropped.  The device
  trains in fp64 where pybnn trains in float32.  ``train`` runs every epoch on the device in one launch;
* Bayesian linear regression over the last hidden layer's 50 features ``Theta``, exactly as BayesianLinearRegression
  with ``basis_func=None`` runs it on ``Theta`` and the (scaled) targets: the same log-posterior, prior and stretch-move
  sampler, ``p0`` from ``prior.sample_from_prior`` and ``burnin_steps`` on the first train, ``chain_length`` steps on
  every train, ``hypers`` the exponential of the final walkers; ``do_mcmc=False`` maximises the log-posterior with
  scipy's fmin from a uniform draw of ``rng``, and ``do_optimize=False`` takes ``[[alpha, beta]]``;
* predict: with mu_i = phi^T m_i and var_i = 1 / beta_i + phi^T S_i phi for each hyper-sample, m = mean mu_i and
  v = mean (mu_i^2 + var_i) - m^2, the mixture's full variance (robo's own BayesianLinearRegression averages the
  variances only; pybnn's DNGO may do the same), clipped to DBL_EPSILON, then de-normalised.  The device forms the
  mixture once per train (its mean m_bar and covariance factor R), so a candidate costs one forward pass and one 50 x 50
  quadratic form.

``n_units_1/2/3`` other than 50 raise ValueError (the device builds 50-wide layers only).  ``adapt_epoch`` is accepted
and has no effect: the network trains for ``num_epochs`` epochs whatever its value.  ``prior=None`` means
BayesianLinearRegressionPrior; any other prior raises TypeError.  With ``normalize_input`` / ``normalize_output`` the
inputs per column / the targets are scaled to zero mean and unit population std before training; ``X`` and ``y`` keep
the data as given.

Random numbers: ``__init__`` takes one draw from ``rng`` (np.random when None) to seed the network's Philox streams
(initial weights and epoch orders), and every ``train`` advances a counter, so each train starts a fresh network; the
sampler's seeds are drawn from ``rng`` per run, as BayesianLinearRegression draws them.

Pickling and deepcopy drop the device handle; the trained net is read back once per ``train``, and a copy re-uploads it
with the training set and refits ``hypers``, so it predicts bit-identically.
"""
import logging

import numpy as np
from scipy import optimize

from robo_b200 import _lib, priors
from robo_b200.models.base_model import BaseModel
from robo_b200.models.bayesian_linear_regression import prior_constants

logger = logging.getLogger(__name__)


class DNGO(BaseModel):

    def __init__(self, batch_size=10, num_epochs=500, learning_rate=0.01, adapt_epoch=5000, n_units_1=50, n_units_2=50,
                 n_units_3=50, alpha=1.0, beta=1000, prior=None, do_mcmc=True, n_hypers=20, chain_length=2000,
                 burnin_steps=2000, normalize_input=True, normalize_output=True, rng=None, device=0):
        if (n_units_1, n_units_2, n_units_3) != (_lib.DNGO_H,) * 3:
            raise ValueError("DNGO: the device builds layers of %d units only (n_units_1/2/3 = %s)"
                             % (_lib.DNGO_H, (n_units_1, n_units_2, n_units_3)))
        self.rng = rng if rng is not None else np.random
        if prior is None:
            prior = priors.BayesianLinearRegressionPrior(rng=self.rng)
        prior_constants(prior)
        self.prior = prior
        self.batch_size = int(batch_size)
        self.num_epochs = int(num_epochs)
        self.init_learning_rate = float(learning_rate)
        self.adapt_epoch = adapt_epoch
        self.n_units_1, self.n_units_2, self.n_units_3 = n_units_1, n_units_2, n_units_3
        self.alpha = alpha
        self.beta = beta
        self.do_mcmc = do_mcmc
        self.n_hypers = n_hypers
        self.chain_length = chain_length
        self.burnin_steps = burnin_steps
        self.burned = False
        self.normalize_input = normalize_input
        self.normalize_output = normalize_output
        self.seed = int(self.rng.randint(2 ** 31 - 1))
        self.counter = 0
        self.X = None
        self.y = None
        self.Theta = None
        self.hypers = None
        self.p0 = None
        self.models = None
        self.net = None
        self.device = int(device)
        self._handle = None

    # ---- device state: the handle does not survive pickling / deepcopy; _ready_handle re-uploads the net ------------
    def __getstate__(self):
        st = self.__dict__.copy()
        st["_handle"] = None
        return st

    def _upload(self):
        if self._handle is None:
            self._handle = _lib.Handle(self.device)
        _lib.dngo_set_data(self._handle, self.X, self.y, self.normalize_input, self.normalize_output,
                           prior_constants(self.prior))
        return self._handle

    def _ready_handle(self):
        """The handle with the net and the collapsed predictive resident (scoring entry points take it)."""
        if self.net is None or self.hypers is None:
            raise ValueError("DNGO: train the model first")
        if self._handle is None:
            h = self._upload()
            _lib.dngo_set_net(h, self.net)
            _lib.dngo_fit(h, np.asarray(self.hypers, dtype=np.float64))
        return self._handle

    def marginal_log_likelihood(self, theta):
        """The Bayesian linear regression's log-posterior of theta = (log alpha, log beta) on the features of the trained
        network (gpk_blr_lnpost on the DNGO handle)."""
        return float(_lib.blr_lnpost(self._handle, np.asarray(theta, dtype=np.float64).reshape(1, 2))[0])

    def negative_mll(self, theta):
        return -self.marginal_log_likelihood(theta)

    @BaseModel._check_shapes_train
    def train(self, X, y, do_optimize=True):
        """Train the network on X (N, D) and y (N,), then sample (or optimise) the regression's hyper-parameters over
        its features."""
        X = np.asarray(X, dtype=np.float64)
        y = np.asarray(y, dtype=np.float64)
        if X.shape[0] > _lib.DNGO_MAX_N:
            raise ValueError("DNGO: %d training points exceed GPK_DNGO_MAX_N = %d" % (X.shape[0], _lib.DNGO_MAX_N))
        if X.shape[1] > _lib.DNGO_MAX_D:
            raise ValueError("DNGO: %d input dimensions exceed GPK_DNGO_MAX_D = %d" % (X.shape[1], _lib.DNGO_MAX_D))
        self.X = X
        self.y = y
        self.net = None
        self.hypers = None
        h = self._upload()
        _lib.dngo_train(h, self.seed, self.counter, self.init_learning_rate, self.batch_size, self.num_epochs)
        self.counter += 1
        self.net = _lib.dngo_net(h)
        self.Theta = _lib.dngo_features(h, X)

        if do_optimize:
            if self.do_mcmc:
                if not self.burned:
                    p0 = self.prior.sample_from_prior(self.n_hypers)
                    seed = int(self.rng.randint(0, 2 ** 63, dtype=np.int64))
                    self.p0 = _lib.blr_sample(h, seed, p0, self.burnin_steps)["pos"]
                    self.burned = True
                seed = int(self.rng.randint(0, 2 ** 63, dtype=np.int64))
                pos = _lib.blr_sample(h, seed, self.p0, self.chain_length)["pos"]
                self.p0 = pos
                self.hypers = np.exp(pos)
            else:
                res = optimize.fmin(self.negative_mll, self.rng.rand(2))
                self.hypers = [[np.exp(res[0]), np.exp(res[1])]]
        else:
            self.hypers = [[self.alpha, self.beta]]

        for alpha, beta in self.hypers:
            logger.debug("Alpha=%f ; Beta=%f" % (alpha, beta))
        _lib.dngo_fit(h, np.asarray(self.hypers, dtype=np.float64))
        self.models = _lib.blr_models(h)

    @BaseModel._check_shapes_predict
    def predict(self, X_test):
        """The mixture's mean and full variance over the hyper-samples at every row: one device pass."""
        return self._ready_handle().predict(np.asarray(X_test, dtype=np.float64))
