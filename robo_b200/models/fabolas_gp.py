"""FabolasGP / FabolasGPMCMC (robo/models/fabolas_gp.py) on the GPU path.

The reference classes are thin wrappers: the last input column is the environment variable s (dataset
fraction), mapped through ``basis_func`` (``fabolas.py:96-102``: (1 - s)^2 for the objective, s for the
cost model), the configuration columns are scaled to [0, 1], and everything else is GaussianProcess /
GaussianProcessMCMC with ``normalize_input=False`` (fabolas_gp.py:28, :113).  Same here: the arithmetic (K build,
Cholesky, predictions, the batched likelihoods of the MCMC walkers, the fused multi-model marginalisation) is the
base classes' device path.  The environment factor of the reference's kernel is george's
BayesianLinearRegressionKernel from the automl fork (fabolas.py:111-117), whose source is not in the reference tree
(SURVEY.md section 8c: definition unrecoverable); any george-style kernel the caller passes is used as is — the
BASELINE config 4 shape is measured with a Matern-5/2 factor on the transformed column.
"""
from copy import deepcopy

import numpy as np

from robo_b200.models.gaussian_process import GaussianProcess
from robo_b200.models.gaussian_process_mcmc import GaussianProcessMCMC
from robo_b200.util import normalization


def _transform(X, lower, upper, basis_func):
    """fabolas_gp.py:122-126: scale the configuration columns, apply the basis function to the last column."""
    X_norm, _, _ = normalization.zero_one_normalization(X[:, :-1], lower, upper)
    s_ = basis_func(X[:, -1])[:, None]
    return np.concatenate((X_norm, s_), axis=1)


class FabolasGP(GaussianProcess):

    def __init__(self, kernel, basis_function, prior=None, noise=1e-3, use_gradients=False, normalize_output=False,
                 lower=None, upper=None, rng=None, device=0, hyper_optimizer="host"):
        self.basis_function = basis_function
        super(FabolasGP, self).__init__(kernel=kernel, prior=prior, noise=noise, use_gradients=use_gradients,
                                        normalize_output=normalize_output, normalize_input=False,
                                        lower=lower, upper=upper, rng=rng, device=device,
                                        hyper_optimizer=hyper_optimizer)

    def normalize(self, X):
        return _transform(X, self.lower, self.upper, self.basis_function)

    device_inputs = normalize

    def input_gradient(self, X_test, G):
        """The chain rule through normalize: 1 / (upper - lower) on the configuration columns, the basis function's
        derivative on s (-2 (1 - s) for (1 - s)^2, 1 for s).  NotImplementedError for any other basis function, whose
        derivative is not known here."""
        from robo_b200 import _lib
        from robo_b200.acquisition_functions.information_gain_per_unit_cost import basis_code
        try:
            code = basis_code(self.basis_function)
        except TypeError:
            raise NotImplementedError("input gradients of a FabolasGP need the basis function s or (1 - s) ** 2")
        lo, hi = normalization._column_range(X_test[:, :-1], self.lower, self.upper)
        s = X_test[:, -1]
        ds = np.ones_like(s) if code == _lib.BASIS_S else -2.0 * (1.0 - s)
        return np.concatenate((G[:, :-1] / (hi - lo), G[:, -1:] * ds[:, None]), axis=1)

    def train(self, X, y, do_optimize=True):
        self.original_X = X
        return super(FabolasGP, self).train(self.normalize(X), y, do_optimize)

    def train_begin(self, X, y):
        self.original_X = X
        return super(FabolasGP, self).train_begin(self.normalize(X), y)

    def predict(self, X_test, full_cov=False, **kwargs):
        return super(FabolasGP, self).predict(self.normalize(X_test), full_cov)

    def score(self, X_test, kind, eta=None, par=0.0, want_values=True):
        return super(FabolasGP, self).score(self.normalize(X_test), kind, eta=eta, par=par, want_values=want_values)

    def sample_functions(self, X_test, n_funcs=1):
        return super(FabolasGP, self).sample_functions(self.normalize(X_test), n_funcs)

    def get_incumbent(self):
        """fabolas_gp.py:140-162: the training configurations projected to the full data set (s = 1); the incumbent
        is the one with the lowest PREDICTED value there.  The reference normalises the projected points and then
        calls predict(), which normalises again (:155-157); that quirk decides which point wins, so it is kept."""
        projection = np.ones([self.original_X.shape[0], 1]) * 1
        X_projected = np.concatenate((self.original_X[:, :-1], projection), axis=1)
        X_norm = self.normalize(X_projected)
        m, _ = self.predict(X_norm)
        best = np.argmin(m)
        return X_projected[best], m[best]


class FabolasGPMCMC(GaussianProcessMCMC):

    def __init__(self, kernel, basis_func, prior=None, n_hypers=20, chain_length=2000, burnin_steps=2000,
                 normalize_output=False, rng=None, lower=None, upper=None, noise=-8, device=0, hyper_sampler="host"):
        self.basis_func = basis_func
        super(FabolasGPMCMC, self).__init__(kernel, prior, n_hypers, chain_length, burnin_steps,
                                            normalize_output=normalize_output, normalize_input=False, rng=rng,
                                            lower=lower, upper=upper, noise=noise, device=device,
                                            hyper_sampler=hyper_sampler)

    # fabolas_gp.py:33-100 is GaussianProcessMCMC.train with these two differences: the MCMC phase sees the transformed
    # inputs (:34-36), and every hyper-parameter sample becomes a FabolasGP trained on the raw inputs (:91-99).
    # The half-ensembles of walkers are evaluated concurrently on the device and predict() / the marginalised
    # acquisition are one fused multi-model call, exactly as for the base class.
    def _likelihood_inputs(self, X):
        return _transform(X, self.lower, self.upper, self.basis_func)

    def _hypers_without_optimisation(self):
        # fabolas_gp.py:77-81: earlier MCMC samples are kept when training without optimisation
        if getattr(self, "hypers", None) is not None and len(self.hypers) > 0:
            return self.hypers
        return super(FabolasGPMCMC, self)._hypers_without_optimisation()

    def _new_sub_model(self, kernel, noise):
        return FabolasGP(kernel, basis_function=self.basis_func, normalize_output=self.normalize_output, noise=noise,
                         lower=self.lower, upper=self.upper, rng=self.rng, device=self.device)
