"""george-compatible kernel objects for the GPU path (host side: parameters only).

RoBO's callers build the covariance with george's kernel algebra
(robo/fmin/bayesian_optimization.py:79-81, robo/fmin/fabolas.py:104-110) and then only use
    len(kernel), kernel.get_parameter_vector(), kernel.set_parameter_vector(v), kernel[:],
    kernel.get_value(X1[, X2]), copy.deepcopy(kernel)
(gaussian_process.py:110,113,151,204; gaussian_process_mcmc.py:145,153;
test/test_models/test_gaussian_process.py:44-46).  These classes keep that surface and
*flatten* to the C ABI's kernel description (include/gpk.h: gpk_set_kernel):

    k(x, x') = exp(log_amp) * prod_g f( sum_{t in g} (x[axis_t] - x'[axis_t])^2 / exp(log_metric_t) )

Every value is computed on the GPU (gpk_kernel_matrix); nothing here evaluates a kernel on
the CPU.  Supported algebra: products of ConstantKernel and radial kernels of ONE family
(Matern-5/2, Matern-3/2 or ExpSquared), times at most one BayesianLinearRegressionKernel
(include/gpk.h: gpk_set_env_factor) or one TaskKernel (gpk_set_task_factor).  Sums are not representable on the device path and
raise NotImplementedError when flattened.
"""
import numpy as np

from . import _lib

__all__ = ["Kernel", "ConstantKernel", "Matern52Kernel", "Matern32Kernel", "ExpSquaredKernel",
           "BayesianLinearRegressionKernel", "TaskKernel", "Product", "Sum"]


class Kernel(object):
    is_kernel = True

    def __init__(self, ndim=1, axes=None):
        self.ndim = int(ndim)
        if axes is None:
            self.axes = np.arange(self.ndim)
        else:
            self.axes = np.atleast_1d(np.asarray(axes, dtype=int))
            if np.any(self.axes < 0) or np.any(self.axes >= self.ndim):
                raise ValueError("invalid axis for {0} dims".format(self.ndim))

    # ---- parameter protocol ----------------------------------------------------
    def __len__(self):
        return len(self.get_parameter_vector())

    def __getitem__(self, idx):
        return self.get_parameter_vector()[idx]

    def __setitem__(self, idx, value):
        v = self.get_parameter_vector()
        v[idx] = value
        self.set_parameter_vector(v)

    @property
    def vector(self):
        return self.get_parameter_vector()

    @vector.setter
    def vector(self, v):
        # george 0.2's kernel.vector assignment, which robo/models/mtbo_gp.py:94 uses to set the parameters
        self.set_parameter_vector(v)

    @property
    def pars(self):
        return np.exp(self.get_parameter_vector())

    # ---- algebra ------------------------------------------------------------------
    def _coerce(self, b):
        if hasattr(b, "is_kernel"):
            return b
        # george 0.3: a scalar c becomes ConstantKernel(log(c / ndim))
        return ConstantKernel(log_constant=np.log(float(b) / self.ndim), ndim=self.ndim)

    def __mul__(self, b):
        if not hasattr(b, "is_kernel"):
            return Product(self._coerce(b), self)
        return Product(self, b)

    __rmul__ = __mul__

    def __add__(self, b):
        if not hasattr(b, "is_kernel"):
            return Sum(self._coerce(b), self)
        return Sum(self, b)

    __radd__ = __add__

    # ---- device description --------------------------------------------------------
    def _collect(self, acc):
        raise NotImplementedError

    def flatten(self):
        """-> dict(family, log_amp, axis, group, log_metric, slots, env, task) for gpk_set_kernel.
        slots[i] = ('amp', None), ('metric', [term indices]), ('lin_a', None), ('lin_b', None) or ('task', k) for
        parameter i, used to map gradients back onto the george parameter vector.  env = None, or
        (axis, log_a, log_b) of the environment factor (gpk_set_env_factor); task = None, or (axis, n_tasks,
        theta tuple) of the task factor (gpk_set_task_factor), whose k-th packed entry is slot ('task', k)."""
        acc = dict(family=None, log_amp=0.0, axis=[], group=[], log_metric=[], slots=[], ngroups=0, env=None, task=None)
        self._collect(acc)
        if acc["env"] is not None and acc["task"] is not None:
            raise NotImplementedError("a kernel with both a BayesianLinearRegressionKernel and a TaskKernel factor is "
                                      "not supported on the device")
        if acc["family"] is None:
            raise NotImplementedError("the device path needs at least one radial kernel factor")
        return acc

    # ---- values (GPU) ------------------------------------------------------------------
    def _parse(self, x):
        x = np.atleast_1d(np.asarray(x, dtype=np.float64))
        if x.ndim == 1:
            x = np.atleast_2d(x).T
        if x.ndim != 2 or x.shape[1] != self.ndim:
            raise ValueError("Dimension mismatch")
        return x

    def get_value(self, x1, x2=None, device=0):
        x1 = self._parse(x1)
        x2 = x1 if x2 is None else self._parse(x2)
        h = _lib.moments_handle(device)
        load_kernel(h, self.flatten())
        return h.kernel_matrix(x1, x2)


def load_kernel(h, f):
    """Loads a flattened kernel (Kernel.flatten) onto a handle: gpk_set_kernel, then its environment or task factor."""
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    if f["env"] is not None:
        h.set_env_factor(*f["env"])
    if f["task"] is not None:
        h.set_task_factor(*f["task"])


class ConstantKernel(Kernel):
    def __init__(self, log_constant, ndim=1, axes=None):
        super(ConstantKernel, self).__init__(ndim, axes)
        self.log_constant = float(log_constant)

    def get_parameter_vector(self, include_frozen=False):
        return np.array([self.log_constant])

    def set_parameter_vector(self, vector, include_frozen=False):
        vector = np.atleast_1d(vector)
        if len(vector) != 1:
            raise ValueError("dimension mismatch")
        self.log_constant = float(vector[0])

    def get_parameter_names(self, include_frozen=False):
        return ("log_constant",)

    def _collect(self, acc):
        acc["log_amp"] += self.log_constant
        acc["slots"].append(("amp", None))


class _Radial(Kernel):
    family = None

    def __init__(self, metric, ndim=1, axes=None):
        super(_Radial, self).__init__(ndim, axes)
        metric = np.atleast_1d(np.asarray(metric, dtype=np.float64))
        if metric.ndim != 1:
            raise NotImplementedError("general (matrix) metrics are not supported")
        if len(metric) != 1 and len(metric) != len(self.axes):
            raise ValueError("Dimension mismatch")
        self.isotropic = len(metric) == 1
        self.log_metric = np.log(metric)

    def get_parameter_vector(self, include_frozen=False):
        return self.log_metric.copy()

    def set_parameter_vector(self, vector, include_frozen=False):
        vector = np.atleast_1d(np.asarray(vector, dtype=np.float64))
        if len(vector) != len(self.log_metric):
            raise ValueError("dimension mismatch")
        self.log_metric = vector.copy()

    def get_parameter_names(self, include_frozen=False):
        return tuple("metric:log_M_{0}_{0}".format(i) for i in range(len(self.log_metric)))

    def _collect(self, acc):
        if acc["family"] is not None and acc["family"] != self.family:
            raise NotImplementedError("products of different radial families are not supported on the device")
        acc["family"] = self.family
        g = acc["ngroups"]
        acc["ngroups"] += 1
        first = len(acc["axis"])
        for i, a in enumerate(self.axes):
            acc["axis"].append(int(a))
            acc["group"].append(g)
            acc["log_metric"].append(float(self.log_metric[0 if self.isotropic else i]))
        terms = list(range(first, len(acc["axis"])))
        if self.isotropic:
            acc["slots"].append(("metric", terms))
        else:
            for t in terms:
                acc["slots"].append(("metric", [t]))


class Matern52Kernel(_Radial):
    family = _lib.MATERN52


class Matern32Kernel(_Radial):
    family = _lib.MATERN32


class ExpSquaredKernel(_Radial):
    family = _lib.EXPSQUARED


class BayesianLinearRegressionKernel(Kernel):
    """The environment kernel of Fabolas (robo/fmin/fabolas.py:104-117) on one input column z:

        k(z, z') = exp(log_a) + exp(log_b) * z * z'

    a Bayesian linear regression in the features (1, z) with prior covariance diag(exp(log_a), exp(log_b)).
    Restated from the Fabolas paper (Klein et al., arXiv:1605.07079) and the reference's call sites: the george fork
    that defines this kernel is not public, so the definition has not been checked against it.  FabolasGP passes the
    basis-transformed dataset size as z.  Parameter vector (log_a, log_b)."""

    def __init__(self, log_a, log_b, ndim=1, axes=None):
        super(BayesianLinearRegressionKernel, self).__init__(ndim, axes)
        if len(self.axes) != 1:
            raise ValueError("BayesianLinearRegressionKernel takes exactly one axis")
        self.log_a, self.log_b = float(log_a), float(log_b)

    def get_parameter_vector(self, include_frozen=False):
        return np.array([self.log_a, self.log_b])

    def set_parameter_vector(self, vector, include_frozen=False):
        vector = np.atleast_1d(np.asarray(vector, dtype=np.float64))
        if len(vector) != 2:
            raise ValueError("dimension mismatch")
        self.log_a, self.log_b = float(vector[0]), float(vector[1])

    def get_parameter_names(self, include_frozen=False):
        return ("log_a", "log_b")

    def _collect(self, acc):
        if acc["env"] is not None:
            raise NotImplementedError("products of two BayesianLinearRegressionKernel factors are not supported on "
                                      "the device")
        acc["env"] = (int(self.axes[0]), self.log_a, self.log_b)
        acc["slots"].append(("lin_a", None))
        acc["slots"].append(("lin_b", None))


class TaskKernel(Kernel):
    """The task kernel of multi-task Bayesian optimisation (robo/fmin/mtbo.py:101, :134: george's
    TaskKernel(ndim, axis, num_tasks)) on input column ``axis``, whose values are task indices:

        k(t, t') = K_t[t, t'],   K_t = L L^T,   L_pq = exp(theta[p (p + 1) / 2 + q])   (q <= p)

    a free-form positive-definite task covariance (Swersky, Snoek, Adams, NIPS 2013) through its Cholesky factor, packed
    row by row (L00, L10, L11, L20, ...).  Restated from the paper and the reference's call sites: the george fork that
    defines this kernel is not public, so the definition has not been checked against it.  A coordinate that is not an
    integer in [0, num_tasks) has a NaN factor.  The parameter vector (num_tasks (num_tasks + 1) / 2 log-entries)
    starts at zeros, L all ones."""

    def __init__(self, ndim, axis, num_tasks):
        super(TaskKernel, self).__init__(ndim, axes=axis)
        if len(self.axes) != 1:
            raise ValueError("TaskKernel takes exactly one axis")
        self.num_tasks = int(num_tasks)
        if not 1 <= self.num_tasks <= _lib.MAX_TASKS:
            raise ValueError("TaskKernel supports 1 to %d tasks on the device" % _lib.MAX_TASKS)
        self.theta = np.zeros(self.num_tasks * (self.num_tasks + 1) // 2)

    def get_parameter_vector(self, include_frozen=False):
        return self.theta.copy()

    def set_parameter_vector(self, vector, include_frozen=False):
        vector = np.atleast_1d(np.asarray(vector, dtype=np.float64)).ravel()
        if len(vector) != len(self.theta):
            raise ValueError("dimension mismatch")
        self.theta = vector.copy()

    def get_parameter_names(self, include_frozen=False):
        return tuple("L_%d_%d" % (p, q) for p in range(self.num_tasks) for q in range(p + 1))

    def _collect(self, acc):
        if acc["task"] is not None:
            raise NotImplementedError("products of two TaskKernel factors are not supported on the device")
        acc["task"] = (int(self.axes[0]), self.num_tasks, tuple(float(v) for v in self.theta))
        for k in range(len(self.theta)):
            acc["slots"].append(("task", k))


class _Operator(Kernel):
    def __init__(self, k1, k2):
        if k1.ndim != k2.ndim:
            raise ValueError("Dimension mismatch")
        self.k1, self.k2 = k1, k2
        self.ndim = k1.ndim
        self.axes = np.arange(self.ndim)

    def get_parameter_vector(self, include_frozen=False):
        return np.concatenate((self.k1.get_parameter_vector(), self.k2.get_parameter_vector()))

    def set_parameter_vector(self, vector, include_frozen=False):
        vector = np.atleast_1d(np.asarray(vector, dtype=np.float64))
        n1 = len(self.k1)
        if len(vector) != n1 + len(self.k2):
            raise ValueError("dimension mismatch")
        self.k1.set_parameter_vector(vector[:n1])
        self.k2.set_parameter_vector(vector[n1:])

    def get_parameter_names(self, include_frozen=False):
        return tuple("k1:" + n for n in self.k1.get_parameter_names()) + \
            tuple("k2:" + n for n in self.k2.get_parameter_names())


class Product(_Operator):
    def _collect(self, acc):
        self.k1._collect(acc)
        self.k2._collect(acc)


class Sum(_Operator):
    def _collect(self, acc):
        raise NotImplementedError("sums of kernels are not supported on the device path")
