"""One table of kernel shapes shared by the int8 scoring tests and the predictive-gradient tests
(tests/test_gpu_kernel_shapes.py) and by the CPU check of the gradient reference (tests/test_grad_oracle_cpu.py).

Every case is a robo_b200 kernel plus its george-oracle twin, built by the same code from either module (both expose
ConstantKernel, Matern52Kernel, Matern32Kernel, ExpSquaredKernel and Product with the same constructors):

    m52        Constant x ARD Matern-5/2
    m32        Constant x ARD Matern-3/2
    rbf        Constant x ARD ExpSquared
    m52_iso    Constant x isotropic Matern-5/2 (one metric for all axes)
    prod1d     Constant x product of 1-D Matern-5/2 (Fabolas), D = 3: one group per axis
    m52_noamp  Matern-5/2 without a ConstantKernel (amplitude 1)
    m52_axis0  Constant x ARD Matern-5/2 x 1-D Matern-5/2 on axis 0: axis 0 in two groups
    terms64    Constant x ARD Matern-5/2 x ARD Matern-5/2, D = 32: 64 terms (GPK_MAX_TERMS) in two groups

and runs in two variants:

    raw        inputs in [0, 1]^D used as they are, no output transform
    scaled     inputs in the offset box [-5, 10]^D, normalize_input with that box, normalize_output=True

Metrics (squared length scales, in the unit cube the kernel sees) and the noise 1e-3 keep ||L^-1|| <= 1/sqrt(noise)
~ 32, inside the 8-slice budget of the int8 contraction (row exponents <= 7), so batches of >= 2048 candidates do take
that path.
"""
import numpy as np
from scipy.special import ndtr

from oracle import george_oracle as G
from oracle import robo_oracle as O
from robo_b200 import kernels as K

CASES = ["m52", "m32", "rbf", "m52_iso", "prod1d", "m52_noamp", "m52_axis0", "terms64"]
VARIANTS = ["raw", "scaled"]
NOISE = 1e-3
LOG_AMP = np.log(1.3)
BOX = (-5.0, 10.0)


def dim(case):
    return {"terms64": 32, "rbf": 2, "m52_noamp": 2}.get(case, 3)


def metrics(case, D):
    """ARD metrics of the case's first radial factor (and of the second, for the two-group cases)."""
    if case == "terms64":
        return np.linspace(6.0, 14.0, D), np.linspace(20.0, 9.0, D)
    if case == "rbf":           # shorter than the Matern cases: with 300 points in 2-D, longer RBF length scales make the
        return np.array([0.05, 0.12]), None      # float64 reference's own variance error near the data ~1e-10
    base = np.array([0.15, 0.4, 0.25])[:D]
    return base, np.array([0.6])


def build(mod, case, D=None):
    """The case's kernel from ``mod`` (robo_b200.kernels or oracle.george_oracle)."""
    D = dim(case) if D is None else D
    m1, m2 = metrics(case, D)
    amp = mod.ConstantKernel(LOG_AMP, ndim=D)
    if case == "m52":
        return mod.Product(amp, mod.Matern52Kernel(m1, ndim=D))
    if case == "m32":
        return mod.Product(amp, mod.Matern32Kernel(m1, ndim=D))
    if case == "rbf":
        return mod.Product(amp, mod.ExpSquaredKernel(m1, ndim=D))
    if case == "m52_iso":
        return mod.Product(amp, mod.Matern52Kernel([0.3], ndim=D))
    if case == "prod1d":
        k = amp
        for d in range(D):
            k = mod.Product(k, mod.Matern52Kernel(m1[d:d + 1], ndim=D, axes=d))
        return k
    if case == "m52_noamp":
        return mod.Matern52Kernel(m1, ndim=D)
    if case == "m52_axis0":
        return mod.Product(mod.Product(amp, mod.Matern52Kernel(m1, ndim=D)), mod.Matern52Kernel(m2, ndim=D, axes=0))
    if case == "terms64":
        return mod.Product(mod.Product(amp, mod.Matern52Kernel(m1, ndim=D)), mod.Matern52Kernel(m2, ndim=D))
    raise KeyError(case)


def amplitude(case):
    """k(x, x): the prior variance of the case's kernel (before the output transform)."""
    return 1.0 if case == "m52_noamp" else float(np.exp(LOG_AMP))


def box(variant, D):
    if variant == "raw":
        return np.zeros(D), np.ones(D)
    return np.full(D, BOX[0]), np.full(D, BOX[1])


def data(case, variant, N, M, seed=0):
    """(X (N, D), y (N,), Xs (M, D)) uniform in the variant's box; y a smooth function of the unit-cube inputs
    (affinely scaled in the ``scaled`` variant so that the output transform is not close to the identity)."""
    D = dim(case)
    rng = np.random.RandomState(1000 * CASES.index(case) + 17 * N + seed)
    lo, up = box(variant, D)
    U = rng.rand(N, D)
    y = np.sin(3.0 * U).sum(axis=1) / np.sqrt(D) + np.cos(5.0 * U[:, 0]) + 0.01 * rng.randn(N)
    if variant == "scaled":
        y = 40.0 * y + 7.0
    return lo + (up - lo) * U, y, lo + (up - lo) * rng.rand(M, D)


def model(case, variant):
    """Untrained robo_b200 GaussianProcess of the case."""
    from robo_b200.models.gaussian_process import GaussianProcess
    D = dim(case)
    if variant == "raw":
        return GaussianProcess(build(K, case, D), noise=NOISE, normalize_input=False, rng=np.random.RandomState(0))
    lo, up = box(variant, D)
    return GaussianProcess(build(K, case, D), noise=NOISE, normalize_input=True, normalize_output=True,
                           lower=lo, upper=up, rng=np.random.RandomState(0))


def oracle_state(case, variant, X, y):
    D = dim(case)
    if variant == "raw":
        return O.gp_fit(build(G, case, D), X, y, noise=NOISE, normalize_input=False)
    lo, up = box(variant, D)
    return O.gp_fit(build(G, case, D), X, y, noise=NOISE, normalize_input=True, normalize_output=True,
                    lower=lo, upper=up)


def prior_var(case, st):
    """k(x, x) in output units: the posterior variance far from the data."""
    return amplitude(case) * (st["y_std"] ** 2 if st["normalize_output"] else 1.0)


def acq_grad_scale(kind, mu, var, s_mu, s_var, eta, par):
    """Error scale of an acquisition's input gradient: the scales s_mu, s_var of d mu, d var (gp_predictive_gradients)
    carried through the closed form's partial derivatives in absolute value (df = f_mu dmu + f_s ds, ds = dvar / 2s).
    mu, var (m,); s_mu, s_var (m, D)."""
    s = np.sqrt(var)[:, None]
    if kind == "lcb":
        return s_mu + par * s_var / (2 * s)
    z = ((eta - mu - par) / np.sqrt(var))[:, None]
    if kind == "ei":
        return ndtr(z) * s_mu + O._pdf(z) * s_var / (2 * s)
    return O._pdf(z) / s * (s_mu + np.abs(z) * s_var / (2 * s))
