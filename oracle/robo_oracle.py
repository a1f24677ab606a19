"""numpy/scipy restatement of RoBO's GP-posterior + acquisition hot path.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Parity status: PINNED —
oracle/make_golden.py executes the reference's own classes
(/root/reference/robo/models/gaussian_process.py, robo/acquisition_functions/*)
on top of oracle.george_oracle and asserts that every function below returns
the same numbers; the resulting vectors are committed under tests/golden/.

The restatement is *functional* (explicit state dict instead of a model object)
so that it cannot be confused with, or imported as, the product classes.
"""
import numpy as np
import scipy.linalg as spla
from scipy.special import ndtr, log_ndtr

from oracle import george_oracle as G

EPS = np.finfo(np.float64).eps
LOG_SQRT_2PI = 0.5 * np.log(2.0 * np.pi)


# --------------------------------------------------------------------------- #
# robo/util/normalization.py
# --------------------------------------------------------------------------- #
def zero_one_normalization(X, lower=None, upper=None):
    """robo/util/normalization.py:4-13."""
    if lower is None:
        lower = np.min(X, axis=0)
    if upper is None:
        upper = np.max(X, axis=0)
    return np.true_divide((X - lower), (upper - lower)), lower, upper


def zero_one_unnormalization(Xn, lower, upper):
    """robo/util/normalization.py:16-17."""
    return lower + (upper - lower) * Xn


def zero_mean_unit_var_normalization(y):
    """robo/util/normalization.py:20-28 (population std, ddof=0)."""
    mean = np.mean(y, axis=0)
    std = np.std(y, axis=0)
    return (y - mean) / std, mean, std


# --------------------------------------------------------------------------- #
# robo/models/gaussian_process.py
# --------------------------------------------------------------------------- #
def gp_fit(kernel, X, y, noise=1e-3, normalize_input=True, normalize_output=False,
           lower=None, upper=None):
    """GaussianProcess.train(..., do_optimize=False): gaussian_process.py:70-124.

    Returns a state dict holding everything predict/nll need.  ``kernel`` is a
    george_oracle kernel; it is used as is (hyper-parameters are NOT optimised
    here, see gp_nll for the objective scipy minimises).
    """
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    assert X.shape[0] == y.shape[0] and X.ndim == 2 and y.ndim == 1   # base_model.py:66-72
    st = dict(kernel=kernel, normalize_input=normalize_input,
              normalize_output=normalize_output, lower=lower, upper=upper)
    if normalize_input:                                               # :89-93
        st["X"], st["lower"], st["upper"] = zero_one_normalization(X, lower, upper)
    else:
        st["X"] = X
    if normalize_output:                                              # :95-101
        st["y"], st["y_mean"], st["y_std"] = zero_mean_unit_var_normalization(y)
        if st["y_std"] == 0:
            raise ValueError("Cannot normalize output. All targets have the same value")
    else:
        st["y"] = y
    st["mean"] = np.mean(st["y"], axis=0)                             # :104
    gp = G.GP(kernel, mean=st["mean"])                                # :106
    st["hypers"] = np.append(kernel.get_parameter_vector(), np.log(noise))   # :113-114
    try:                                                              # :118-122
        gp.compute(st["X"], yerr=np.sqrt(noise))
    except np.linalg.LinAlgError:
        noise *= 10
        gp.compute(st["X"], yerr=np.sqrt(noise))
    st["noise"] = noise
    st["gp"] = gp
    return st


def gp_nll(st, theta, prior=None):
    """GaussianProcess.nll: gaussian_process.py:129-166 (mutates st['kernel'])."""
    theta = np.asarray(theta, dtype=np.float64)
    if np.any((-20 > theta) + (theta > 20)):                          # :147-148
        return 1e25
    gp = st["gp"]
    gp.kernel.set_parameter_vector(theta[:-1])                        # :151
    noise = np.exp(theta[-1])                                         # :152
    try:
        gp.compute(st["X"], yerr=np.sqrt(noise))                      # :155
    except np.linalg.LinAlgError:
        return 1e25
    ll = gp.log_likelihood(st["y"], quiet=True)                       # :159
    if prior is not None:
        ll += prior.lnprob(theta)                                     # :162-163
    return -ll if np.isfinite(ll) else 1e25                           # :166


def gp_loglik_terms(st):
    """(log-likelihood, log-determinant) of the current factorisation."""
    gp = st["gp"]
    return gp.log_likelihood(st["y"], quiet=True), gp.solver.log_determinant


def gp_predict(st, X_test, full_cov=False):
    """GaussianProcess.predict: gaussian_process.py:251-296.

    Faithful to the reference: george returns the full M x M covariance
    (:280), the diagonal is taken afterwards (:285-286), then the clip (:290-294).
    """
    X_test = np.asarray(X_test, dtype=np.float64)
    assert X_test.ndim == 2                                           # base_model.py:74-79
    if st["normalize_input"]:
        Xs, _, _ = zero_one_normalization(X_test, st["lower"], st["upper"])   # :276
    else:
        Xs = X_test
    mu, var = st["gp"].predict(st["y"], Xs)                           # :280
    if st["normalize_output"]:                                        # :282-284
        mu = mu * st["y_std"] + st["y_mean"]
        var = var * st["y_std"] ** 2
    if not full_cov:
        var = np.diag(var)                                            # :286
    var = np.clip(var, EPS, np.inf)                                   # :290-294 (the :294 zeroing is a no-op after the clip)
    return mu, var


def gp_predict_var_only(st, X_test):
    """CPU-optimised variant (BASELINE.md section 3 row ii): variance through one
    triangular solve, never forming the M x M covariance.  Same mean/variance as
    gp_predict up to rounding; used only as a second CPU baseline."""
    X_test = np.asarray(X_test, dtype=np.float64)
    if st["normalize_input"]:
        Xs, _, _ = zero_one_normalization(X_test, st["lower"], st["upper"])
    else:
        Xs = X_test
    gp = st["gp"]
    alpha = gp._compute_alpha(st["y"])
    Ks = gp.kernel.get_value(Xs, gp._x)
    mu = Ks @ alpha + st["mean"]
    U = gp.solver._factor[0]
    V = spla.solve_triangular(U, Ks.T, trans="T", lower=False, check_finite=False)
    var = gp.kernel.get_value(Xs[:1], Xs[:1])[0, 0] - np.einsum("ij,ij->j", V, V)
    if st["normalize_output"]:
        mu = mu * st["y_std"] + st["y_mean"]
        var = var * st["y_std"] ** 2
    return mu, np.clip(var, EPS, np.inf)


def flatten_kernel(kernel):
    """Product tree of ConstantKernels and radial kernels of ONE family -> the flat description oracle/kmat.c takes
    (family id, amplitude, per-term axis / metric / group-closing flag)."""
    fam_id = {G.Matern52Kernel: 0, G.ExpSquaredKernel: 1, G.Matern32Kernel: 2}
    amp, fams, axis, metric, last = [1.0], set(), [], [], []

    def walk(k):
        if isinstance(k, G.Product):
            walk(k.k1)
            walk(k.k2)
        elif isinstance(k, G.ConstantKernel):
            amp[0] = amp[0] * np.exp(k.log_constant)
        elif type(k) in fam_id:
            fams.add(fam_id[type(k)])
            m = k._axis_metric()
            for a, md in zip(k.axes, m):
                axis.append(int(a))
                metric.append(float(md))
                last.append(0)
            last[-1] = 1
        else:
            raise TypeError("flatten_kernel: unsupported kernel %r" % type(k))
    walk(kernel)
    if len(fams) != 1:
        raise TypeError("flatten_kernel: exactly one radial family expected")
    return dict(family=fams.pop(), amp=float(amp[0]), axis=np.array(axis, dtype=np.int32),
                last=np.array(last, dtype=np.int32), metric=np.array(metric, dtype=np.float64))


def kmat_fast(kernel, X1, X2):
    """kernel.get_value(X1, X2) through the threaded C restatement (oracle/kmat.c); equal to the numpy path to a few
    ulp (tests/test_oracle_golden.py)."""
    import ctypes as C
    from oracle import build_c
    lib = build_c.load()
    f = flatten_kernel(kernel)
    X1 = np.ascontiguousarray(X1, dtype=np.float64)
    X2 = np.ascontiguousarray(X2, dtype=np.float64)
    out = np.empty((len(X1), len(X2)))
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    lib.oracle_kmat(f["family"], f["amp"], len(f["axis"]), f["axis"].ctypes.data_as(ip), f["last"].ctypes.data_as(ip),
                    f["metric"].ctypes.data_as(dp), X1.ctypes.data_as(dp), len(X1), X2.ctypes.data_as(dp), len(X2),
                    X1.shape[1], out.ctypes.data_as(dp))
    return out


def gp_predict_var_only_fast(st, X_test, chunk=8192):
    """gp_predict_var_only for candidate batches of BASELINE size (2^20): K* from the threaded C restatement, chunked
    so that the working set stays bounded.  Same formulas, same clip."""
    X_test = np.asarray(X_test, dtype=np.float64)
    if st["normalize_input"]:
        Xs, _, _ = zero_one_normalization(X_test, st["lower"], st["upper"])
    else:
        Xs = X_test
    gp = st["gp"]
    alpha = gp._compute_alpha(st["y"])
    U = gp.solver._factor[0]
    kss = gp.kernel.get_value(Xs[:1], Xs[:1])[0, 0]
    mu, var = np.empty(len(Xs)), np.empty(len(Xs))
    for lo in range(0, len(Xs), chunk):
        Ks = kmat_fast(gp.kernel, Xs[lo:lo + chunk], gp._x)
        mu[lo:lo + chunk] = Ks @ alpha + st["mean"]
        V = spla.solve_triangular(U, Ks.T, trans="T", lower=False, check_finite=False)
        var[lo:lo + chunk] = kss - np.einsum("ij,ij->j", V, V)
    if st["normalize_output"]:
        mu = mu * st["y_std"] + st["y_mean"]
        var = var * st["y_std"] ** 2
    return mu, np.clip(var, EPS, np.inf)


def _kernel_input_grad(k, Xs, X):
    """(k(Xs, X) (m, n), d k(Xs, X) / d Xs (m, n, ndim)) of a george_oracle kernel, by the product rule over its tree:
    ConstantKernel -> 0; radial kernel f(r2) -> f'(r2) * 2 (x*_a - x_a) / metric_a on each of its axes."""
    if isinstance(k, G.Product):
        v1, g1 = _kernel_input_grad(k.k1, Xs, X)
        v2, g2 = _kernel_input_grad(k.k2, Xs, X)
        return v1 * v2, g1 * v2[:, :, None] + g2 * v1[:, :, None]
    if isinstance(k, G.ConstantKernel):
        return k._value(Xs, X), np.zeros((len(Xs), len(X), Xs.shape[1]))
    if isinstance(k, G._RadialKernel):
        r2 = k._r2(Xs, X)
        dfdr2 = k._dfdr2(r2)
        g = np.zeros((len(Xs), len(X), Xs.shape[1]))
        for a, md in zip(k.axes, k._axis_metric()):
            g[:, :, a] += dfdr2 * (2.0 * (Xs[:, a][:, None] - X[:, a][None, :]) / md)
        return k._f(r2), g
    raise TypeError("gp_predictive_gradients: unsupported kernel %r" % type(k))


def gp_predictive_gradients(st, X_test, chunk_elems=1 << 22):
    """Input gradients of GaussianProcess.predict's moments at the rows of X_test, in raw input coordinates:
        d mu / d x   = dk* . alpha                      (alpha = K^-1 (y - mean))
        d var / d x  = -2 dk* . w,   w = K^-1 k*        (k** is constant: stationary kernels)
    dk* from the george kernel tree (_kernel_input_grad), then the chain rules of zero_one_normalization
    (1 / (upper - lower)) and of the output un-normalisation (y_std, y_std^2).  The clip of var at DBL_EPSILON is not
    differentiated.  Returns dict(dmu, dvar, s_mu, s_var), each (m, D): s_mu = sum_j |dk_j| |alpha_j| and
    s_var = 2 sum_j |dk_j| |w_j| (same chain factors) are the magnitudes the sums cancel from, the natural error scale
    of any floating-point evaluation of them."""
    X_test = np.asarray(X_test, dtype=np.float64)
    if st["normalize_input"]:
        Xs, _, _ = zero_one_normalization(X_test, st["lower"], st["upper"])
        chain = 1.0 / (np.asarray(st["upper"], dtype=np.float64) - np.asarray(st["lower"], dtype=np.float64))
    else:
        Xs, chain = X_test, np.ones(X_test.shape[1])
    gp = st["gp"]
    alpha = gp._compute_alpha(st["y"])
    X = gp._x
    m, D = Xs.shape
    out = {k: np.empty((m, D)) for k in ("dmu", "dvar", "s_mu", "s_var")}
    step = max(1, chunk_elems // max(1, len(X) * D))
    for lo in range(0, m, step):
        Ks, dK = _kernel_input_grad(gp.kernel, Xs[lo:lo + step], X)
        W = gp.solver.apply_inverse(Ks.T)                                  # (n, mc)
        sl = slice(lo, lo + step)
        out["dmu"][sl] = np.einsum("cja,j->ca", dK, alpha)
        out["dvar"][sl] = -2.0 * np.einsum("cja,jc->ca", dK, W)
        out["s_mu"][sl] = np.einsum("cja,j->ca", np.abs(dK), np.abs(alpha))
        out["s_var"][sl] = 2.0 * np.einsum("cja,jc->ca", np.abs(dK), np.abs(W))
    ys = st["y_std"] if st["normalize_output"] else 1.0
    for k, f in (("dmu", ys), ("s_mu", ys), ("dvar", ys * ys), ("s_var", ys * ys)):
        out[k] *= chain[None, :] * f
    return out


def acq_gradients(mu, var, dmu, dvar, kind, eta=0.0, par=0.0):
    """(f (m,), df (m, D)): value and input gradient of EI / PI / LCB from the moments and their gradients, as the
    reference writes them with derivative=True (ei.py:80-85, pi.py:65-71, lcb.py:66-69); ds = dvar / (2 s)."""
    mu, var = np.asarray(mu, dtype=np.float64), np.asarray(var, dtype=np.float64)
    s = np.sqrt(var)
    dm, ds = np.asarray(dmu), np.asarray(dvar) / (2.0 * s[:, None])
    if kind == "lcb":
        return acq_lcb(mu, var, par), -(dm - par * ds)
    z = (eta - mu - par) / s
    if kind == "ei":
        f = s * (z * ndtr(z) + _pdf(z))
        return f, -dm * ndtr(z)[:, None] + ds * _pdf(z)[:, None]
    if kind == "pi":
        return ndtr(z), (-_pdf(z) / s)[:, None] * (dm + ds * z[:, None])
    raise ValueError("acq_gradients: %r has no input gradient" % kind)


def gp_predict_variance(st, x1, X2):
    """GaussianProcess.predict_variance: gaussian_process.py:221-248."""
    x_ = np.concatenate((x1, X2))
    _, var = gp_predict(st, x_, full_cov=True)
    return var[-1, :-1, np.newaxis]


def gp_get_incumbent(st):
    """gaussian_process.py:334-352 + base_model.py:94-106."""
    b = np.argmin(st["y"])
    inc, val = st["X"][b], st["y"][b]
    if st["normalize_input"]:
        inc = zero_one_unnormalization(inc, st["lower"], st["upper"])
    if st["normalize_output"]:
        val = val * st["y_std"] + st["y_mean"]
    return inc, val


def gp_grad_nll_correct(st, theta):
    """Mathematically correct gradient of -log-likelihood w.r.t. theta
    (log kernel parameters ..., log sigma^2).  The reference's grad_nll
    (gaussian_process.py:168-191) is dead code with a wrong noise slice
    (identity instead of sigma^2 I, :179-182); this is the corrected form,
    validated against finite differences of gp_nll in tests."""
    gp = st["gp"]
    gp.kernel.set_parameter_vector(theta[:-1])
    noise = np.exp(theta[-1])
    gp.compute(st["X"], yerr=np.sqrt(noise))
    alpha = gp._compute_alpha(st["y"])
    Kinv = gp.solver.get_inverse()
    A = np.outer(alpha, alpha) - Kinv
    Kg = gp.kernel.gradient(gp._x)
    g = 0.5 * np.einsum("ijk,ij", Kg, A)
    g_noise = 0.5 * noise * np.trace(A)
    return -np.append(g, g_noise)


def gp_grad_nll_terms_fast(st, theta, recompute=True):
    """gp_grad_nll_correct for BASELINE-size problems (config 5: N = 8192, D = 32, where the (N, N, H) array of
    gaussian_process.py:181 would need 18 GB): same formula, the einsum of :186 evaluated by the threaded C restatement
    without materialising dK/dtheta.  Returns d(-loglik)/d[log amp, log metric per kernel TERM ..., log sigma^2]
    (one entry per axis of every radial factor: isotropic kernels are the sum of their terms)."""
    import ctypes as C
    from oracle import build_c
    gp = st["gp"]
    noise = np.exp(theta[-1])
    if recompute:                       # False: st was fitted with exactly these hyper-parameters (saves a K build)
        gp.kernel.set_parameter_vector(theta[:-1])
        gp.compute(st["X"], yerr=np.sqrt(noise))
    alpha = gp._compute_alpha(st["y"])
    Kinv = gp.solver.get_inverse()
    A = np.ascontiguousarray(np.outer(alpha, alpha) - Kinv)
    f = flatten_kernel(gp.kernel)
    X = np.ascontiguousarray(gp._x, dtype=np.float64)
    g = np.zeros(len(f["axis"]) + 1)
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    build_c.load().oracle_grad_trace(f["family"], f["amp"], len(f["axis"]), f["axis"].ctypes.data_as(ip),
                                     f["last"].ctypes.data_as(ip), f["metric"].ctypes.data_as(dp), X.ctypes.data_as(dp),
                                     len(X), X.shape[1], A.ctypes.data_as(dp), g.ctypes.data_as(dp))
    return -np.append(0.5 * g, 0.5 * noise * np.trace(A))


def gp_grad_nll_reference_compat(st, theta):
    """gaussian_process.py:168-191 exactly (identity noise slice, no prior)."""
    gp = st["gp"]
    gp.kernel.set_parameter_vector(theta[:-1])
    noise = np.exp(theta[-1])
    gp.compute(st["X"], yerr=np.sqrt(noise))
    alpha = gp._compute_alpha(st["y"])
    Kinv = gp.solver.get_inverse()
    Kg = gp.kernel.gradient(gp._x)
    Kg = np.concatenate((Kg, np.eye(Kg.shape[0])[:, :, None]), axis=2)
    A = np.outer(alpha, alpha) - Kinv
    return -0.5 * np.einsum("ijk,ij", Kg, A)


# --------------------------------------------------------------------------- #
# robo/acquisition_functions/{ei,log_ei,pi,lcb}.py  (closed forms on moments)
# --------------------------------------------------------------------------- #
def _pdf(z):
    return np.exp(-0.5 * z * z) / np.sqrt(2.0 * np.pi)


def _logpdf(z):
    return -0.5 * z * z - LOG_SQRT_2PI


def acq_ei(m, v, eta, par=0.0):
    """EI.compute: ei.py:65-88 (whole-batch zero on any s==0; ValueError if f<0)."""
    s = np.sqrt(v)
    if (s == 0).any():
        return np.array([[0]])
    z = (eta - m - par) / s
    f = s * (z * ndtr(z) + _pdf(z))
    if (f < 0).any():
        raise ValueError
    return f


def acq_pi(m, v, eta, par=0.0):
    """PI.compute: pi.py:58-63."""
    s = np.sqrt(v)
    return ndtr((eta - m - par) / s)


def acq_lcb(m, v, par=1.0):
    """LCB.compute: lcb.py:62-65."""
    return -(m - par * np.sqrt(v))


def acq_log_ei(m, v, eta, par=0.0):
    """LogEI.compute: log_ei.py:67-122, branch order preserved
    (np.Infinity of the reference restated as np.inf: removed in numpy 2)."""
    f_min = eta - par
    s = np.sqrt(v)
    with np.errstate(divide="ignore", invalid="ignore"):
        z = (f_min - m) / s
    out = np.zeros([m.size])
    for i in range(m.size):
        mu, sigma = m[i], s[i]
        if abs(f_min - mu) == 0:                                       # :85-89
            out[i] = np.log(sigma) + _logpdf(z[i]) if sigma > 0 else -np.inf
        elif sigma == 0:                                               # :92-96
            out[i] = np.log(f_min - mu) if mu < f_min else -np.inf
        else:
            b = np.log(sigma) + _logpdf(z[i])                          # :99
            if f_min > mu:                                             # :101-107
                a = np.log(f_min - mu) + log_ndtr(z[i])
                out[i] = max(a, b) + np.log(1 + np.exp(-abs(b - a)))
            else:                                                      # :114-120
                a = np.log(mu - f_min) + log_ndtr(z[i])
                out[i] = -np.inf if a >= b else b + np.log(1 - np.exp(a - b))
    return out


ACQ = {"ei": acq_ei, "log_ei": acq_log_ei, "pi": acq_pi, "lcb": acq_lcb}


def acquisition(st, X_test, kind, par=None, eta=None):
    """acq.compute(X) on a fitted GP state: predict -> closed form."""
    m, v = gp_predict(st, X_test)
    if kind == "lcb":
        return acq_lcb(m, v, 1.0 if par is None else par)
    if eta is None:
        eta = gp_get_incumbent(st)[1]
    return ACQ[kind](m, v, eta, 0.0 if par is None else par)


def argmax_first(values):
    """numpy.argmax first-occurrence semantics (random_sampling.py:50)."""
    return int(np.argmax(values))


# --------------------------------------------------------------------------- #
# robo/models/gaussian_process_mcmc.py:230-247 / marginalization.py:115-121
# --------------------------------------------------------------------------- #
def mcmc_mixture_moments(mus, vars_):
    """GaussianProcessMCMC.predict: m = mean_i mu_i ; v = var_i(mu_i) + mean_i var_i,
    clipped (gaussian_process_mcmc.py:235-247).  mus/vars_: (n_models, M)."""
    m = mus.mean(axis=0)
    v = np.var(mus, axis=0) + np.mean(vars_, axis=0)
    return m, np.clip(v, EPS, np.inf)


def marginalised_acquisition(per_model_values):
    """MarginalizationGPMCMC.compute: marginalization.py:115-121."""
    return np.asarray(per_model_values).mean(axis=0)


# --------------------------------------------------------------------------- #
# synthetic workloads (SURVEY.md section 8d), shared by tests and bench.py
# --------------------------------------------------------------------------- #
def synthetic_problem(N, D, M, seed_train=1234, seed_cand=4321):
    """X ~ U[0,1]^(N x D), y = sum_d sinc(10 x_d - 5) + 0.01 N(0,1)
    (mirrors test/test_models/test_gaussian_process.py:14-15); candidates
    X* ~ U[0,1]^(M x D); theta: amplitude 1, metric_d = D/4, noise 1e-3."""
    rng = np.random.RandomState(seed_train)
    X = rng.rand(N, D)
    y = np.sinc(X * 10 - 5).sum(axis=1) + 0.01 * rng.randn(N)
    Xs = np.random.RandomState(seed_cand).rand(M, D)
    theta = np.concatenate(([0.0], np.full(D, np.log(D / 4.0))))
    return X, y, Xs, theta, 1e-3


def make_kernel(kind, D, theta):
    """kind in {'matern52','rbf'}: amp * ARD kernel with theta = [log amp, log metric_d...]."""
    cls = {"matern52": G.Matern52Kernel, "rbf": G.ExpSquaredKernel}[kind]
    k = G.Product(G.ConstantKernel(theta[0], ndim=D), cls(np.exp(theta[1:]), ndim=D))
    return k


# --------------------------------------------------------------------------- #
# counter-based candidate generator (checker for gpk_generate_candidates)
# --------------------------------------------------------------------------- #
def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11; Random123 constants), vectorised over numpy uint32 arrays."""
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    c0, c1, c2, c3 = [np.asarray(c, dtype=np.uint64) & np.uint64(0xFFFFFFFF) for c in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0 & 0xFFFFFFFF), np.uint64(k1 & 0xFFFFFFFF)
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & mask, p1 >> np.uint64(32), p1 & mask
        c0, c1, c2, c3 = (hi1 ^ c1 ^ k0) & mask, lo1, (hi0 ^ c3 ^ k1) & mask, lo0
        k0 = (k0 + np.uint64(0x9E3779B9)) & mask
        k1 = (k1 + np.uint64(0xBB67AE85)) & mask
    return c0, c1, c2, c3


def generate_candidates(seed, first, count, n_uniform, lower, upper, incumbent, scale):
    """Restatement of gpk_candidates_kernel: random_sampling.py:38-47 with a counter-based stream."""
    lower, upper, incumbent = [np.asarray(a, dtype=np.float64) for a in (lower, upper, incumbent)]
    d = lower.size
    npair = (d + 1) // 2
    gi = (np.arange(count, dtype=np.uint64) + np.uint64(first))[:, None] + np.zeros((1, npair), dtype=np.uint64)
    pb = np.zeros((count, 1), dtype=np.uint64) + np.arange(npair, dtype=np.uint64)[None, :]
    r0, r1, r2, r3 = philox4x32_10(gi & np.uint64(0xFFFFFFFF), gi >> np.uint64(32), pb, np.zeros_like(pb),
                                   seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    u0 = ((r1 << np.uint64(32) | r0) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    u1 = ((r3 << np.uint64(32) | r2) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    out = np.empty((count, 2 * npair))
    uni = (gi[:, 0] < np.uint64(n_uniform))
    lo2 = np.concatenate((lower, [0.0] * (2 * npair - d)))
    up2 = np.concatenate((upper, [1.0] * (2 * npair - d)))
    inc2 = np.concatenate((incumbent, [0.0] * (2 * npair - d)))
    a0, a1 = np.arange(0, 2 * npair, 2), np.arange(1, 2 * npair, 2)
    out[:, a0] = lo2[a0] + (up2[a0] - lo2[a0]) * u0
    out[:, a1] = lo2[a1] + (up2[a1] - lo2[a1]) * u1
    rad = np.sqrt(-2.0 * np.log(1.0 - u0))
    g0 = np.clip(inc2[a0] + scale * rad * np.cos(2 * np.pi * u1), lo2[a0], up2[a0])
    g1 = np.clip(inc2[a1] + scale * rad * np.sin(2 * np.pi * u1), lo2[a1], up2[a1])
    res = out.copy()
    res[np.ix_(~uni, a0)] = g0[~uni]
    res[np.ix_(~uni, a1)] = g1[~uni]
    return res[:, :d]
