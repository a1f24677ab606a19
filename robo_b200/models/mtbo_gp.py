"""MTBOGP / MTBOGPMCMC (robo/models/mtbo_gp.py) on the GPU path.

The reference classes are thin wrappers, like the Fabolas ones: the configuration columns are scaled to [0, 1], the last
input column is the task index, passed through np.rint and not scaled (mtbo_gp.py:12-15), and everything else is
GaussianProcess / GaussianProcessMCMC with ``normalize_input=False`` (:30, :117).  The task factor of the reference's
kernel is george's TaskKernel from the automl fork (mtbo.py:101), restated in robo_b200/kernels.py: TaskKernel.

Kept from the reference, on purpose:
  - MTBOGPMCMC sets each sample's parameters through ``kernel.vector = sample[:-1]`` (mtbo_gp.py:94).  The class also
    calls ``len(self.kernel.pars)`` (:53), which only george 0.2 has, and there the assignment sets the parameters; so
    it is restated that way (robo_b200.kernels.Kernel.vector has a setter);
  - training without optimisation keeps the earlier MCMC samples (:82-86);
  - MTBOGP.get_incumbent projects the training configurations to task 1, normalises them and then calls predict(),
    which normalises again (:148-153); that decides which point wins, so it is kept as FabolasGP keeps its twin.
"""
import numpy as np

from robo_b200.models.gaussian_process import GaussianProcess
from robo_b200.models.gaussian_process_mcmc import GaussianProcessMCMC
from robo_b200.util import normalization


def normalize(X, lower, upper):
    """mtbo_gp.py:12-15: scale the configuration columns, round the task column to the nearest integer (half to even)."""
    X_norm, _, _ = normalization.zero_one_normalization(X[:, :-1], lower, upper)
    return np.concatenate((X_norm, np.rint(X[:, None, -1])), axis=1)


class MTBOGP(GaussianProcess):

    def __init__(self, kernel, prior=None, noise=1e-3, use_gradients=False, normalize_output=False, lower=None,
                 upper=None, rng=None, device=0, hyper_optimizer="host"):
        super(MTBOGP, self).__init__(kernel=kernel, prior=prior, noise=noise, use_gradients=use_gradients,
                                     normalize_output=normalize_output, normalize_input=False,
                                     lower=lower, upper=upper, rng=rng, device=device,
                                     hyper_optimizer=hyper_optimizer)

    def normalize(self, X):
        return normalize(X, self.lower, self.upper)

    device_inputs = normalize

    def input_gradient(self, X_test, G):
        """The chain rule through normalize: 1 / (upper - lower) on the configuration columns, 0 on the task column
        (np.rint is piecewise constant)."""
        lo, hi = normalization._column_range(X_test[:, :-1], self.lower, self.upper)
        return np.concatenate((G[:, :-1] / (hi - lo), np.zeros_like(G[:, -1:])), axis=1)

    def train(self, X, y, do_optimize=True):
        self.original_X = X
        return super(MTBOGP, self).train(self.normalize(X), y, do_optimize)

    def train_begin(self, X, y):
        self.original_X = X
        return super(MTBOGP, self).train_begin(self.normalize(X), y)

    def predict(self, X_test, full_cov=False, **kwargs):
        return super(MTBOGP, self).predict(self.normalize(X_test), full_cov)

    def score(self, X_test, kind, eta=None, par=0.0, want_values=True):
        return super(MTBOGP, self).score(self.normalize(X_test), kind, eta=eta, par=par, want_values=want_values)

    def sample_functions(self, X_test, n_funcs=1):
        return super(MTBOGP, self).sample_functions(self.normalize(X_test), n_funcs)

    def get_incumbent(self):
        """mtbo_gp.py:136-159, with its double normalisation (see the module docstring)."""
        projection = np.ones([self.original_X.shape[0], 1]) * 1
        X_projected = np.concatenate((self.original_X[:, :-1], projection), axis=1)
        X_norm = self.normalize(X_projected)
        m, _ = self.predict(X_norm)
        best = np.argmin(m)
        return X_projected[best], m[best]


class MTBOGPMCMC(GaussianProcessMCMC):

    def __init__(self, kernel, prior=None, n_hypers=20, chain_length=2000, burnin_steps=2000, normalize_output=False,
                 rng=None, lower=None, upper=None, noise=-8, device=0, hyper_sampler="host"):
        self.hypers = None
        super(MTBOGPMCMC, self).__init__(kernel, prior, n_hypers, chain_length, burnin_steps,
                                         normalize_output=normalize_output, normalize_input=False, rng=rng,
                                         lower=lower, upper=upper, noise=noise, device=device,
                                         hyper_sampler=hyper_sampler)

    # mtbo_gp.py:37-105 is GaussianProcessMCMC.train with the MCMC phase on the mapped inputs (:38) and every sample a
    # MTBOGP trained on the raw inputs (:89-103)
    def _likelihood_inputs(self, X):
        return normalize(X, self.lower, self.upper)

    def _hypers_without_optimisation(self):
        if getattr(self, "hypers", None) is not None and len(self.hypers) > 0:
            return self.hypers
        return super(MTBOGPMCMC, self)._hypers_without_optimisation()

    def _new_sub_model(self, kernel, noise):
        return MTBOGP(kernel, normalize_output=self.normalize_output, noise=noise, lower=self.lower, upper=self.upper,
                      rng=self.rng, device=self.device)
