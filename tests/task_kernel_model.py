"""numpy restatement of the MTBO kernel with the task factor (include/gpk.h: gpk_set_task_factor) and an oracle-backed
stand-in handle that carries the factor — TEST INFRASTRUCTURE ONLY.

    k((x, t), (x', t')) = amp * prod_g f_g(r2_g) * K_t[t, t'],   K_t = L L^T,   L_pq = exp(theta[p (p + 1) / 2 + q])

The factor is a restatement from Swersky, Snoek, Adams (NIPS 2013) and the reference's call sites, not checked against
the george fork that defines TaskKernel; task_matrix / task_value / task_gradient are the one place it is written down
for the tests.  K_t[a, b] sums L_aq L_bq in ascending q, multiply then add, with the C library's exp, as the host side of
gpk_task_matrix builds the table the device reads: the two agree bit for bit."""
import math

import numpy as np
import scipy.linalg as spla

from oracle import george_oracle as G
from tests.fake_gpk import FAMILIES, FakeHandle


def n_kt(n_tasks):
    return n_tasks * (n_tasks + 1) // 2


def cholesky_factor(theta, n_tasks):
    L = np.zeros((n_tasks, n_tasks))
    for p in range(n_tasks):
        for q in range(p + 1):
            L[p, q] = math.exp(theta[p * (p + 1) // 2 + q])      # the C library's exp, as the host helper calls it
    return L


def task_matrix(theta, n_tasks):
    """K_t (n_tasks x n_tasks) from the packed log-entries."""
    L = cholesky_factor(theta, n_tasks)
    K = np.zeros((n_tasks, n_tasks))
    for a in range(n_tasks):
        for b in range(a + 1):
            s = 0.0
            for q in range(b + 1):
                s = s + L[a, q] * L[b, q]
            K[a, b] = K[b, a] = s
    return K


def task_index(t, n_tasks):
    """The task a coordinate names, -1 when it is not an integer in [0, n_tasks)."""
    t = np.asarray(t, dtype=np.float64)
    ok = (t >= 0) & (t < n_tasks) & (t == np.floor(t))
    return np.where(ok, np.where(ok, t, 0).astype(int), -1)


def task_value(t1, t2, theta, n_tasks):
    """K_t[t1_i, t2_j] -> (n1, n2), NaN where a coordinate is not a task."""
    K = task_matrix(theta, n_tasks)
    i1, i2 = task_index(t1, n_tasks), task_index(t2, n_tasks)
    out = K[np.maximum(i1, 0)][:, np.maximum(i2, 0)]
    out[(i1 < 0)[:, None] | (i2 < 0)[None, :]] = np.nan
    return out


def task_gradient(t1, t2, theta, n_tasks):
    """d task_value / d theta_k -> (n1, n2, n_kt): dK_t[a, b] / dtheta_pq = L_pq (delta_ap L_bq + delta_bp L_aq)."""
    L = cholesky_factor(theta, n_tasks)
    i1, i2 = task_index(t1, n_tasks), task_index(t2, n_tasks)
    out = np.zeros((len(i1), len(i2), n_kt(n_tasks)))
    for p in range(n_tasks):
        for q in range(p + 1):
            dK = np.zeros((n_tasks, n_tasks))
            dK[p, :] += L[p, q] * L[:, q]
            dK[:, p] += L[p, q] * L[:, q]
            out[:, :, p * (p + 1) // 2 + q] = dK[i1][:, i2]
    return out


class TaskKernel(G.Kernel):
    """The factor in the oracle's kernel algebra (parameter vector: the packed log-entries of L, one axis)."""

    def __init__(self, theta, n_tasks, ndim=1, axes=None):
        super(TaskKernel, self).__init__(ndim, axes)
        self.n_tasks = int(n_tasks)
        self.theta = np.asarray(theta, dtype=np.float64).copy()

    def get_parameter_vector(self, include_frozen=False):
        return self.theta.copy()

    def set_parameter_vector(self, vector, include_frozen=False):
        self.theta = np.asarray(vector, dtype=np.float64).copy()

    def get_parameter_names(self, include_frozen=False):
        return tuple("L_%d" % k for k in range(len(self.theta)))

    def _value(self, x1, x2):
        a = int(self.axes[0])
        return task_value(x1[:, a], x2[:, a], self.theta, self.n_tasks)

    def _gradient(self, x1, x2):
        a = int(self.axes[0])
        return task_gradient(x1[:, a], x2[:, a], self.theta, self.n_tasks)


def mtbo_kernel(D, log_amp, log_metric, theta, n_tasks):
    """The oracle's amp * prod_d Matern52(axes=d) * TaskKernel(axes=D) on D + 1 columns."""
    k = G.ConstantKernel(log_amp, ndim=D + 1)
    for d in range(D):
        k = G.Product(k, G.Matern52Kernel(np.exp([log_metric[d]]), ndim=D + 1, axes=[d]))
    return G.Product(k, TaskKernel(theta, n_tasks, ndim=D + 1, axes=[D]))


class TaskFakeHandle(FakeHandle):
    """FakeHandle with gpk_set_task_factor: the factor multiplies the oracle kernel, the prior variance is
    amp K_t[t*, t*] and the marginal-likelihood gradient gains the n_kt task entries."""

    def set_kernel(self, family, log_amp, axis, group, log_metric):
        super(TaskFakeHandle, self).set_kernel(family, log_amp, axis, group, log_metric)
        self.task = None

    def set_task_factor(self, axis, n_tasks=1, theta=None):
        base = self.kernel if self.task is None else self.kernel.k1
        if axis >= 0:
            theta = np.asarray(theta, dtype=np.float64).ravel()
            if not (1 <= n_tasks <= 8) or theta.size != n_kt(n_tasks) or not np.all(np.isfinite(theta)):
                raise ValueError("gpk_set_task_factor: bad argument")
        if axis >= base.ndim:
            family, log_amp, ax, group, lm = self.spec
            base = G.ConstantKernel(log_amp, ndim=axis + 1)
            for g in range(int(group.max()) + 1):
                sel = group == g
                base = G.Product(base, FAMILIES[int(family)](np.exp(lm[sel]), ndim=axis + 1, axes=ax[sel]))
        self.task = None if axis < 0 else (int(axis), int(n_tasks), theta.copy())
        self.kernel = base if self.task is None else G.Product(base, TaskKernel(theta, n_tasks, ndim=base.ndim,
                                                                                axes=[axis]))
        self.fitted = self.linv_built = False

    def fit(self, diag_add, mean):
        if self.task is not None:
            a, nT, _ = self.task
            if np.any(task_index(self.X[:, a], nT) < 0):
                raise ValueError("gpk_fit: training column %d holds a value that is not a task index" % a)
        return super(TaskFakeHandle, self).fit(diag_add, mean)

    def _moments(self, Xs, full=False, clip=True):
        if self.task is None or full:
            return super(TaskFakeHandle, self)._moments(Xs, full, clip)
        mu, _ = super(TaskFakeHandle, self)._moments(Xs, False, False)
        Xn = self._norm(Xs)
        Ks = self.kernel.get_value(Xn, self.X)
        V = spla.solve_triangular(self.L, Ks.T, lower=True)
        a, nT, theta = self.task
        t = Xn[:, a]
        var = self.amp * np.diagonal(task_value(t, t, theta, nT)) - np.einsum("ij,ij->j", V, V)
        on, ym, ys = self.out
        if on:
            var = var * ys ** 2
        return mu, np.clip(var, np.finfo(float).eps, np.inf) if clip else var

    def nll_grad(self, noise_var, n_terms, env=False, n_kt=0):
        g = super(TaskFakeHandle, self).nll_grad(noise_var, n_terms)
        if not n_kt:
            return g
        Kinv = spla.cho_solve((self.L, True), np.eye(len(self.y)))
        A = np.outer(self.alpha, self.alpha) - Kinv
        Kg = self.kernel.gradient(self.X)[:, :, -n_kt:]
        return np.concatenate([g[:-1], -0.5 * np.einsum("ij,ijk->k", A, Kg), g[-1:]])


def install(monkeypatch):
    """Route robo_b200 through TaskFakeHandle for the duration of a test."""
    from tests import fake_gpk
    from robo_b200 import _lib
    fake_gpk.install(monkeypatch)
    pool = {}
    monkeypatch.setattr(_lib, "Handle", TaskFakeHandle)
    monkeypatch.setattr(_lib, "moments_handle", lambda device=0: pool.setdefault(device, TaskFakeHandle(device)))
    return TaskFakeHandle
