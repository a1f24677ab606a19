"""Hyper-priors used by the fmin facade: O(H) scalar host math added to the GPU log-likelihood
(SURVEY.md section 2 row 19: out of the hot path, stays Python).  Semantics — including the quirks —
follow robo/priors/base_prior.py, robo/priors/default_priors.py and robo/priors/env_priors.py."""
import numpy as np
import scipy.stats as sps


class TophatPrior(object):
    """base_prior.py:75-156."""

    def __init__(self, l_bound, u_bound, rng=None):
        self.rng = np.random.RandomState(np.random.randint(0, 10000)) if rng is None else rng
        self.min, self.max = l_bound, u_bound
        if not (self.max > self.min):
            raise Exception("Upper bound of Tophat prior must be greater than the lower bound!")

    def lnprob(self, theta):
        if np.any(theta < self.min) or np.any(theta > self.max):
            return -np.inf
        return 0

    def sample_from_prior(self, n_samples):
        p0 = self.min + self.rng.rand(n_samples) * (self.max - self.min)
        return p0[:, np.newaxis]

    def gradient(self, theta):
        return np.zeros([theta.shape[0]])


class HorseshoePrior(object):
    """base_prior.py:158-237 (returns +inf at theta == 0 like the reference, :194-196)."""

    def __init__(self, scale=0.1, rng=None):
        self.rng = np.random.RandomState(np.random.randint(0, 10000)) if rng is None else rng
        self.scale = scale

    def lnprob(self, theta):
        if np.any(theta == 0.0):
            return np.inf
        return np.log(np.log(1 + 3.0 * (self.scale / np.exp(theta)) ** 2))

    def sample_from_prior(self, n_samples):
        lamda = np.abs(self.rng.standard_cauchy(size=n_samples))
        p0 = np.log(np.abs(self.rng.randn() * lamda * self.scale))
        return p0[:, np.newaxis]

    def gradient(self, theta):
        a = -(6 * self.scale ** 2)
        b = (3 * self.scale ** 2 + np.exp(2 * theta))
        b *= np.log(3 * self.scale ** 2 * np.exp(- 2 * theta) + 1)
        return a / b


class LognormalPrior(object):
    """base_prior.py:239-316 (``mean`` is passed as scipy's ``loc``, :278, like the reference)."""

    def __init__(self, sigma, mean=0, rng=None):
        self.rng = np.random.RandomState(np.random.randint(0, 10000)) if rng is None else rng
        self.sigma, self.mean = sigma, mean

    def lnprob(self, theta):
        return sps.lognorm.logpdf(theta, self.sigma, loc=self.mean)

    def sample_from_prior(self, n_samples):
        p0 = self.rng.lognormal(mean=self.mean, sigma=self.sigma, size=n_samples)
        return p0[:, np.newaxis]

    def gradient(self, theta):
        return None


class NormalPrior(object):
    """base_prior.py:318-378 (lnprob returns the pdf, not its log, like the reference, :341-357)."""

    def __init__(self, sigma, mean=0, rng=None):
        self.rng = np.random.RandomState(np.random.randint(0, 10000)) if rng is None else rng
        self.sigma, self.mean = sigma, mean

    def lnprob(self, theta):
        return sps.norm.pdf(theta, scale=self.sigma, loc=self.mean)

    def sample_from_prior(self, n_samples):
        p0 = self.rng.normal(loc=self.mean, scale=self.sigma, size=n_samples)
        return p0[:, np.newaxis]


class DefaultPrior(object):
    """default_priors.py:8-53: lognormal on the amplitude, tophat(-10, 2) on the length scales,
    horseshoe(0.1) on the noise; gradient identically zero (:51-53)."""

    def __init__(self, n_dims, rng=None):
        self.rng = np.random.RandomState(np.random.randint(0, 10000)) if rng is None else rng
        self.n_dims = n_dims
        self.tophat = TophatPrior(-10, 2, rng=self.rng)
        self.ln_prior = LognormalPrior(mean=0.0, sigma=1.0, rng=self.rng)
        self.horseshoe = HorseshoePrior(scale=0.1, rng=self.rng)

    def lnprob(self, theta):
        lp = 0
        lp += self.ln_prior.lnprob(theta[0])
        lp += self.tophat.lnprob(theta[1:-1])
        lp += self.horseshoe.lnprob(theta[-1])
        return lp

    def sample_from_prior(self, n_samples):
        p0 = np.zeros([n_samples, self.n_dims])
        p0[:, 0] = self.ln_prior.sample_from_prior(n_samples)[:, 0]
        ls_sample = np.array([self.tophat.sample_from_prior(n_samples)[:, 0]
                              for _ in range(1, (self.n_dims - 1))]).T
        p0[:, 1:(self.n_dims - 1)] = ls_sample
        p0[:, -1] = self.horseshoe.sample_from_prior(n_samples)[:, 0]
        return p0

    def gradient(self, theta):
        return np.zeros([theta.shape[0]])


class EnvPrior(object):
    """env_priors.py:8-81 (the Fabolas prior): lognormal(mean -2) on the amplitude, tophat(-10, 2) on the n_ls length
    scales, NormalPrior(0, 1) on the n_lr parameters of the environment kernel (the pdf is added, as the reference
    does), horseshoe(0.001) on the noise."""

    def __init__(self, n_dims, n_ls, n_lr, rng=None):
        self.rng = np.random.RandomState(np.random.randint(0, 10000)) if rng is None else rng
        self.n_dims, self.n_ls, self.n_lr = n_dims, n_ls, n_lr
        self.bayes_lin_prior = NormalPrior(sigma=1, mean=0, rng=self.rng)
        self.tophat = TophatPrior(-10, 2, rng=self.rng)
        self.ln_prior = LognormalPrior(mean=-2, sigma=1.0, rng=self.rng)
        self.horseshoe = HorseshoePrior(scale=0.001, rng=self.rng)

    def lnprob(self, theta):
        lp = 0
        lp += self.ln_prior.lnprob(theta[0])
        lp += self.tophat.lnprob(theta[1:self.n_ls + 1])
        pos, end = self.n_ls + 1, self.n_ls + self.n_lr + 1
        for t in theta[pos:end]:
            lp += self.bayes_lin_prior.lnprob(t)
        lp += self.horseshoe.lnprob(theta[-1])
        return lp

    def sample_from_prior(self, n_samples):
        p0 = np.zeros([n_samples, self.n_dims])
        p0[:, 0] = self.ln_prior.sample_from_prior(n_samples)[:, 0]
        ls_sample = np.array([self.tophat.sample_from_prior(n_samples)[:, 0] for _ in range(0, self.n_ls)]).T
        p0[:, 1:(self.n_ls + 1)] = ls_sample
        pos, end = self.n_ls + 1, self.n_ls + self.n_lr + 1
        samples = np.array([self.bayes_lin_prior.sample_from_prior(n_samples)[:, 0] for _ in range(0, self.n_lr)]).T
        p0[:, pos:end] = samples
        p0[:, -1] = self.horseshoe.sample_from_prior(n_samples)[:, 0]
        return p0


class MTBOPrior(object):
    """env_priors.py:158-228 (the MTBO prior): lognormal(sigma 1, loc 0) on the amplitude, tophat(-10, 2) on the n_ls
    length scales, tophat(-1, 0) on the n_kt Cholesky entries of the task kernel as one vector test, horseshoe(0.1) on
    the noise.  sample_from_prior draws the task slice through numpy's (1, n, n_kt) broadcast, as the reference does."""

    def __init__(self, n_dims, n_ls, n_kt, rng=None):
        self.rng = np.random.RandomState(np.random.randint(0, 10000)) if rng is None else rng
        self.n_dims, self.n_ls, self.n_kt = n_dims, n_ls, n_kt
        self.tophat = TophatPrior(-10, 2, rng=self.rng)
        self.ln_prior = LognormalPrior(mean=0.0, sigma=1.0, rng=self.rng)
        self.horseshoe = HorseshoePrior(scale=0.1, rng=self.rng)
        self.tophat_task = TophatPrior(-1, 0, rng=self.rng)

    def lnprob(self, theta):
        lp = 0
        lp += self.ln_prior.lnprob(theta[0])
        lp += self.tophat.lnprob(theta[1:self.n_ls + 1])
        lp += self.tophat_task.lnprob(theta[self.n_ls + 1:self.n_ls + 1 + self.n_kt])
        lp += self.horseshoe.lnprob(theta[-1])
        return lp

    def sample_from_prior(self, n_samples):
        p0 = np.zeros([n_samples, self.n_dims])
        p0[:, 0] = self.ln_prior.sample_from_prior(n_samples)[:, 0]
        ls_sample = np.array([self.tophat.sample_from_prior(n_samples)[:, 0] for _ in range(0, self.n_ls)]).T
        p0[:, 1:(self.n_ls + 1)] = ls_sample
        pos, end = self.n_ls + 1, self.n_ls + self.n_kt + 1
        p0[:, pos:end] = np.array([self.tophat_task.sample_from_prior(n_samples) for _ in range(0, end - pos)]).T
        p0[:, -1] = self.horseshoe.sample_from_prior(n_samples)[:, 0]
        return p0


class BayesianLinearRegressionPrior(object):
    """bayesian_linear_regression_prior.py:8-60, with its quirks: lnprob adds LognormalPrior(sigma=0.1, mean=-10) of
    theta[0] (scipy's loc = -10) and HorseshoePrior(0.1) of 1 / theta[-1], one over log beta rather than the noise
    (:45-49); sample_from_prior draws a lognormal SAMPLE (about 4.5e-5) as log alpha and log beta = log(1 / exp(sigma))
    with the horseshoe's one randn() shared by all walkers (:51-60).  gpk_blr_lnpost restates lnprob on the device."""

    def __init__(self, rng=None):
        self.rng = np.random.RandomState(np.random.randint(0, 10000)) if rng is None else rng
        self.ln_prior_alpha = LognormalPrior(sigma=0.1, mean=-10, rng=self.rng)
        self.horseshoe = HorseshoePrior(scale=0.1, rng=self.rng)

    def lnprob(self, theta):
        lp = 0
        lp += self.ln_prior_alpha.lnprob(theta[0])
        lp += self.horseshoe.lnprob(1 / theta[-1])
        return lp

    def sample_from_prior(self, n_samples):
        p0 = np.zeros([n_samples, 2])
        p0[:, 0] = self.ln_prior_alpha.sample_from_prior(n_samples)[:, 0]
        sigmas = self.horseshoe.sample_from_prior(n_samples)[:, 0]
        p0[:, -1] = np.log(1 / np.exp(sigmas))
        return p0

    def gradient(self, theta):
        pass
