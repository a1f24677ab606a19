"""numpy restatement of the Fabolas kernel with the environment factor (include/gpk.h: gpk_set_env_factor) and an
oracle-backed stand-in handle that carries the factor — TEST INFRASTRUCTURE ONLY.

    k((x, z), (x', z')) = amp * prod_g f_g(r2_g) * (exp(log_a) + exp(log_b) * z * z')

The factor is a restatement from the Fabolas paper (arXiv:1605.07079), not checked against the george fork that
defines BayesianLinearRegressionKernel; env_value / env_gradient are the one place it is written down for the tests."""
import numpy as np
import scipy.linalg as spla

from oracle import george_oracle as G
from tests.fake_gpk import FAMILIES, FakeHandle


def env_value(z1, z2, log_a, log_b):
    """exp(log_a) + exp(log_b) z1 z2' for column vectors z1 (n1), z2 (n2) -> (n1, n2)."""
    return np.exp(log_a) + np.exp(log_b) * np.outer(z1, z2)


def env_gradient(z1, z2, log_a, log_b):
    """(d/dlog_a, d/dlog_b, d/dz1) of env_value, each (n1, n2)."""
    one = np.ones((len(z1), len(z2)))
    return np.exp(log_a) * one, np.exp(log_b) * np.outer(z1, z2), np.exp(log_b) * np.broadcast_to(z2, one.shape)


class EnvKernel(G.Kernel):
    """The factor in the oracle's kernel algebra (parameter vector (log_a, log_b), one axis)."""

    def __init__(self, log_a, log_b, ndim=1, axes=None):
        super(EnvKernel, self).__init__(ndim, axes)
        self.log_a, self.log_b = float(log_a), float(log_b)

    def get_parameter_vector(self, include_frozen=False):
        return np.array([self.log_a, self.log_b])

    def set_parameter_vector(self, vector, include_frozen=False):
        self.log_a, self.log_b = float(vector[0]), float(vector[1])

    def get_parameter_names(self, include_frozen=False):
        return ("log_a", "log_b")

    def _value(self, x1, x2):
        a = int(self.axes[0])
        return env_value(x1[:, a], x2[:, a], self.log_a, self.log_b)

    def _gradient(self, x1, x2):
        a = int(self.axes[0])
        ga, gb, _ = env_gradient(x1[:, a], x2[:, a], self.log_a, self.log_b)
        return np.stack([ga, gb], axis=-1)


def fabolas_kernel(D, log_amp, log_metric, log_a, log_b):
    """The oracle's 1 * prod_d Matern52(axes=d) * EnvKernel(axes=D) on D + 1 columns."""
    k = G.ConstantKernel(log_amp, ndim=D + 1)
    for d in range(D):
        k = G.Product(k, G.Matern52Kernel(np.exp([log_metric[d]]), ndim=D + 1, axes=[d]))
    return G.Product(k, EnvKernel(log_a, log_b, ndim=D + 1, axes=[D]))


class EnvFakeHandle(FakeHandle):
    """FakeHandle with gpk_set_env_factor: the factor multiplies the oracle kernel, the prior variance is per candidate
    and the marginal-likelihood gradient gains the (log_a, log_b) entries."""

    def set_kernel(self, family, log_amp, axis, group, log_metric):
        super(EnvFakeHandle, self).set_kernel(family, log_amp, axis, group, log_metric)
        self.env = None

    def set_env_factor(self, axis, log_a=0.0, log_b=0.0):
        if not (np.isfinite(log_a) and np.isfinite(log_b)) or axis < -1:
            raise ValueError("gpk_set_env_factor: bad argument")
        base = self.kernel if self.env is None else self.kernel.k1
        if axis >= base.ndim:                     # no data yet: the radial part was built on its own axes only
            family, log_amp, ax, group, lm = self.spec
            base = G.ConstantKernel(log_amp, ndim=axis + 1)
            for g in range(int(group.max()) + 1):
                sel = group == g
                base = G.Product(base, FAMILIES[int(family)](np.exp(lm[sel]), ndim=axis + 1, axes=ax[sel]))
        self.env = None if axis < 0 else (int(axis), float(log_a), float(log_b))
        self.kernel = base if self.env is None else G.Product(base, EnvKernel(log_a, log_b, ndim=base.ndim,
                                                                               axes=[axis]))
        self.fitted = self.linv_built = False

    def _moments(self, Xs, full=False, clip=True):
        if self.env is None or full:
            return super(EnvFakeHandle, self)._moments(Xs, full, clip)
        mu, _ = super(EnvFakeHandle, self)._moments(Xs, False, False)
        Xn = self._norm(Xs)
        Ks = self.kernel.get_value(Xn, self.X)
        V = spla.solve_triangular(self.L, Ks.T, lower=True)
        a, la, lb = self.env
        var = self.amp * (np.exp(la) + np.exp(lb) * Xn[:, a] ** 2) - np.einsum("ij,ij->j", V, V)
        on, ym, ys = self.out
        if on:
            var = var * ys ** 2
        return mu, np.clip(var, np.finfo(float).eps, np.inf) if clip else var

    def nll_grad(self, noise_var, n_terms, env=False):
        g = super(EnvFakeHandle, self).nll_grad(noise_var, n_terms)
        if not env:
            return g
        Kinv = spla.cho_solve((self.L, True), np.eye(len(self.y)))
        A = np.outer(self.alpha, self.alpha) - Kinv
        Kg = self.kernel.gradient(self.X)
        return np.concatenate([g[:-1], [-0.5 * np.sum(A * Kg[:, :, -2]), -0.5 * np.sum(A * Kg[:, :, -1])], g[-1:]])


def install(monkeypatch):
    """Route robo_b200 through EnvFakeHandle for the duration of a test."""
    from tests import fake_gpk
    from robo_b200 import _lib
    fake_gpk.install(monkeypatch)
    pool = {}
    monkeypatch.setattr(_lib, "Handle", EnvFakeHandle)
    monkeypatch.setattr(_lib, "moments_handle", lambda device=0: pool.setdefault(device, EnvFakeHandle(device)))
    return EnvFakeHandle
