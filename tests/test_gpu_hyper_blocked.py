"""GP hyper-parameters on the device at large N (gpk_hyper_lnpost_blocked / gpk_sample_hypers_blocked /
gpk_optimize_hypers_blocked, hyper_sampler / hyper_optimizer = "device_blocked").

- the log-likelihood against a reference that builds K in extended precision (tests/fit_reference.kernel_ld) and
  factors it in fp64, at N from 2 to 8192, every radial family, ARD and isotropic groups, the environment and the task
  factor; the log-prior bit for bit against gpk_hyper_lnpost's; the -inf cases;
- batch independence: a theta's bits alone, in a batch, reversed and in chunks of 1 and 3;
- the sampler and the optimiser bit for bit against tests/hyper_model.py and tests/hyperopt_model.py fed by
  gpk_hyper_lnpost_blocked;
- the models and facades end to end; every argument error."""
import numpy as np
import pytest

from tests import fit_reference as FR
from tests import hyper_model as HM
from tests import hyperopt_model as OM
from tests.test_de_es_cpu import LO, UP, branin

pytestmark = pytest.mark.gpu

TINY = 1.25e-12
# |ll_device - ll_ref| <= REL max(|ll_ref|, 1) for the thetas drawn here (noise >= e^-6, K well conditioned): the
# bound the small-N device likelihood is held to in tests/test_gpu_hyper.py
REL = 1e-10


def _kernel(case, D):
    from robo_b200 import kernels as K
    if case == "m52_ard":
        return 2.0 * K.Matern52Kernel(np.ones(D), ndim=D)
    if case == "rbf_iso":
        return 2.0 * K.ExpSquaredKernel(1.0, ndim=D)
    if case == "env":                                     # the Fabolas structure: the last column is the environment
        k = 1.0
        for d in range(D - 1):
            k = k * K.Matern52Kernel(np.ones(1), ndim=D, axes=d)
        return k * K.BayesianLinearRegressionKernel(log_a=0.1, log_b=0.1, ndim=D, axes=D - 1)
    if case == "task":                                    # the MTBO structure: the last column holds the task index
        k = 1.0 * K.Matern52Kernel(np.ones(D - 1), ndim=D, axes=list(range(D - 1)))
        return k * K.TaskKernel(D, D - 1, 3)
    raise ValueError(case)


def _prior(case, kernel):
    from robo_b200 import priors as PR
    dim = len(kernel) + 1
    rng = np.random.RandomState(0)
    if case == "env":
        return PR.EnvPrior(dim, len(kernel) - 3, 2, rng=rng)
    if case == "task":
        return PR.MTBOPrior(dim, len(kernel) - 7, 6, rng=rng)
    if case == "rbf_iso":
        return None
    return PR.DefaultPrior(dim, rng=rng)


def _data(case, N, D, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    if case == "env":
        X[:, -1] = (1 - rng.uniform(0.05, 1, N)) ** 2
    if case == "task":
        X[:, -1] = rng.randint(0, 3, N)
    y = np.sin(5 * X[:, :2]).sum(axis=1) + 0.1 * rng.randn(N)
    return X, y


def _handle(X, y, kernel, prior, batch_bytes=None):
    from robo_b200 import _lib
    from robo_b200.kernels import load_kernel
    from robo_b200.models.gaussian_process_mcmc import _hyper_prior
    f = kernel.flatten()
    h = _lib.Handle(0)
    if batch_bytes is not None:
        h.set_option("hyper_batch_bytes", batch_bytes)
    h.set_data(X, y)
    load_kernel(h, f)
    kind, par, n_ls, n_lr = _hyper_prior(prior)
    _lib.set_hyper_model(h, f["slots"], len(f["axis"]), float(np.mean(y)), TINY, kind, par, n_ls, n_lr)
    return h, f


def _flat_at(f, theta):
    """The flattened kernel with theta's parameters (the slot table's mapping)."""
    g = dict(f)
    log_amp, lm = 0.0, np.array(f["log_metric"], dtype=np.float64)
    env, task = [], []
    for p, (kind, terms) in enumerate(f["slots"]):
        if kind == "amp":
            log_amp += theta[p]
        elif kind == "metric":
            lm[terms] = theta[p]
        elif kind in ("lin_a", "lin_b"):
            env.append(theta[p])
        else:
            task.append(theta[p])
    g["log_amp"], g["log_metric"] = log_amp, lm
    if f["env"] is not None:
        g["env"] = (f["env"][0], env[0], env[1])
    if f["task"] is not None:
        g["task"] = (f["task"][0], f["task"][1], tuple(task))
    return g


def ref_ll(X, y, f, theta):
    """ll of theta: K in extended precision (kernel_ld, 512-row slabs), rounded to fp64, factored in fp64."""
    import scipy.linalg
    theta = np.asarray(theta, dtype=np.float64)
    if np.any(np.abs(theta) > 20):
        return -np.inf
    g = _flat_at(f, theta)
    N = len(X)
    K = np.empty((N, N))
    for i0 in range(0, N, 512):
        K[i0:i0 + 512] = FR.kernel_ld(g, X[i0:i0 + 512], X).astype(np.float64)
    yerr = np.sqrt(np.exp(theta[-1]))
    K[np.diag_indices(N)] += float(np.sqrt(np.float64(yerr) ** 2 + TINY) ** 2)
    try:
        L = np.linalg.cholesky(K)
    except np.linalg.LinAlgError:
        return -np.inf
    z = scipy.linalg.solve_triangular(L, y - np.mean(y), lower=True)
    return float(-0.5 * z @ z - np.sum(np.log(np.diag(L))) - 0.5 * N * np.log(2 * np.pi))


def _thetas(kernel, prior, rng, count):
    dim = len(kernel) + 1
    T = np.c_[rng.uniform(-1, 1, (count, dim - 1)), rng.uniform(-6, -2, count)]
    if prior is not None and hasattr(prior, "ln_prior"):
        T[:, 0] = rng.uniform(0.2, 1.5, count)                   # inside the lognormal's support
    return T


_SHAPES = ([(case, N) for N in (2, 31, 127, 128, 129, 232, 233, 1000, 2048, 4096) for case in ("m52_ard",)]
           + [(case, N) for N in (31, 129, 233, 1000) for case in ("rbf_iso", "env", "task")]
           + [("m52_ard_d8", N) for N in (233, 1000)] + [("m52_ard", 8192)])


@pytest.mark.parametrize("case,N", _SHAPES)
def test_lnpost_against_the_reference(case, N):
    from robo_b200 import _lib
    D = {"m52_ard": 3, "m52_ard_d8": 8, "rbf_iso": 4, "env": 3, "task": 3}[case]
    case = case.replace("_d8", "")
    kernel = _kernel(case, D)
    prior = _prior(case, kernel)
    X, y = _data(case, N, D, seed=N)
    h, f = _handle(X, y, kernel, prior)
    rng = np.random.RandomState(N + 7)
    T = _thetas(kernel, prior, rng, 2 if N >= 4096 else 5)
    dim = T.shape[1]
    special = np.array([np.r_[0.5, np.zeros(dim - 2), 21.0],           # |theta| > 20
                        np.r_[-20.5, np.zeros(dim - 2), -3.0],
                        np.r_[np.nan, np.zeros(dim - 2), -3.0]])       # NaN
    T = np.vstack([T, special])
    ll, lp = _lib.hyper_lnpost_blocked(h, T)
    assert np.all(np.isneginf(ll[-3:]))
    fin = slice(0, len(T) - 3)
    ref = np.array([ref_ll(X, y, f, t) for t in T[fin]])
    assert np.all(np.isfinite(ref)) and np.all(np.isfinite(ll[fin]))
    err = np.abs(ll[fin] - ref) / np.maximum(np.abs(ref), 1.0)
    assert np.max(err) < REL, (case, N, err)
    # the prior: gpk_hyper_lnpost's, bit for bit (on a small handle of the same model where N is above its limit)
    hs = h if N <= _lib.HYPER_MAX_N else _handle(X[:50], y[:50], kernel, prior)[0]
    ll_s, lp_s = _lib.hyper_lnpost(hs, T)
    assert lp.tobytes() == lp_s.tobytes()
    if N <= _lib.HYPER_MAX_N:
        assert np.all(np.isneginf(ll_s[-3:]))
        err = np.abs(ll[fin] - ll_s[fin]) / np.maximum(np.abs(ll_s[fin]), 1.0)
        assert np.max(err) < REL, (case, N, err)
    if hs is not h:
        hs.close()
    h.close()


@pytest.mark.parametrize("N", [40, 300])
def test_not_positive_definite_is_minus_inf(N):
    """Identical inputs: K = amp J exactly (the jitter is below half an ulp of amp = e^19.9), rank one."""
    from robo_b200 import _lib
    X = np.full((N, 2), 0.3)
    y = np.random.RandomState(0).rand(N)
    h, _ = _handle(X, y, _kernel("m52_ard", 2), None)
    ll, _ = _lib.hyper_lnpost_blocked(h, np.array([[19.9, 0.0, 0.0, -19.9], [19.9, 5.0, -5.0, -19.9],
                                                     [0.0, 0.0, 0.0, -2.0]]))
    assert np.all(np.isneginf(ll[:2])) and np.isfinite(ll[2])
    h.close()


def _per_theta_bytes(N):
    """A theta's matrix and P strip in a chunk (include/gpk.h, "hyper_batch_bytes"), without the few kB of the rest."""
    nb = -(-N // 128)
    return (nb + 2) * nb * 131072


def test_batch_independence():
    from robo_b200 import _lib
    N = 300
    kernel = _kernel("env", 3)
    prior = _prior("env", kernel)
    X, y = _data("env", N, 3)
    T = _thetas(kernel, prior, np.random.RandomState(3), 20)
    T[5, -1] = 20.5                                                  # -inf cases in the middle of the batch
    T[11, 0] = np.nan
    h, _ = _handle(X, y, kernel, prior)
    ll, lp = _lib.hyper_lnpost_blocked(h, T)
    alone = [_lib.hyper_lnpost_blocked(h, T[i:i + 1]) for i in range(len(T))]
    assert np.concatenate([a[0] for a in alone]).tobytes() == ll.tobytes()
    assert np.concatenate([a[1] for a in alone]).tobytes() == lp.tobytes()
    llr, lpr = _lib.hyper_lnpost_blocked(h, T[::-1])
    assert llr[::-1].tobytes() == ll.tobytes() and lpr[::-1].tobytes() == lp.tobytes()
    per = _per_theta_bytes(N)
    for chunk in (1, 3):
        h.set_option("hyper_batch_bytes", chunk * (per + 4096))
        llc, lpc = _lib.hyper_lnpost_blocked(h, T)
        assert llc.tobytes() == ll.tobytes() and lpc.tobytes() == lp.tobytes()
    assert np.isneginf(ll[5]) and np.isneginf(ll[11]) and np.sum(np.isfinite(ll)) == 18
    h.set_option("hyper_batch_bytes", per // 2)                      # one matrix does not fit
    with pytest.raises(ValueError, match="hyper_batch_bytes"):
        _lib.hyper_lnpost_blocked(h, T)
    h.close()


# ---- the sampler and the optimiser bit for bit ----------------------------------------------------------------------
@pytest.mark.parametrize("N,steps", [(100, 20), (2048, 3)])
def test_sampler_bit_for_bit(N, steps):
    from robo_b200 import _lib
    kernel = _kernel("env", 3)
    prior = _prior("env", kernel)
    X, y = _data("env", N, 3, seed=1)
    h, _ = _handle(X, y, kernel, prior)
    p0 = prior.sample_from_prior(20)
    r = _lib.sample_hypers_blocked(h, p0, steps, 987654321)
    ref = HM.run(lambda T: HM.post(*_lib.hyper_lnpost_blocked(h, T)), p0, steps, 987654321)
    assert r["pos"].tobytes() == ref["pos"].tobytes()
    assert r["lnpost"].tobytes() == ref["lnpost"].tobytes()
    assert np.array_equal(r["n_accepted"], ref["n_accepted"]) and np.any(ref["n_accepted"] > 0)
    h.close()


@pytest.mark.parametrize("N,D,maxiter", [(300, 2, 15000), (2048, 16, 12)])
def test_optimizer_bit_for_bit(N, D, maxiter):
    from robo_b200 import _lib
    kernel = _kernel("m52_ard", D)
    prior = _prior("m52_ard", kernel)
    X, y = _data("m52_ard", N, D, seed=2)
    h, _ = _handle(X, y, kernel, prior)
    p0 = np.r_[1.0, np.zeros(D), np.log(1e-3)]
    r = _lib.optimize_hypers_blocked(h, p0, maxiter=maxiter)
    ref = OM.run(lambda T: OM.objective(*_lib.hyper_lnpost_blocked(h, T), True), p0, maxiter=maxiter)
    assert r["theta"].tobytes() == ref["x"].tobytes()
    assert (r["f"], r["nit"], r["nfev"], r["status"]) == (ref["f"], ref["nit"], ref["nfev"], ref["status"])
    assert r["rounds"] == ref["rounds"] and r["noop_rounds"] == OM.noop_rounds(ref["rounds"])
    assert ref["nit"] >= 1
    h.close()


# ---- end to end ------------------------------------------------------------------------------------------------------
def test_fabolas_gp_mcmc_at_2048(monkeypatch):
    from robo_b200 import _lib
    from robo_b200.fmin.fabolas import _model, quadratic_bf
    seen = []
    real = _lib.sample_hypers_blocked

    def rec(h, p0, steps, seed):
        r = real(h, p0, steps, seed)
        seen.append(r)
        return r
    monkeypatch.setattr(_lib, "sample_hypers_blocked", rec)
    rng = np.random.RandomState(0)
    m = _model(2, quadratic_bf, 20, 4, 4, LO, UP, rng, "device_blocked")
    X = np.c_[LO + (UP - LO) * rng.rand(2048, 2), rng.uniform(0.05, 1, 2048)]
    y = np.log(np.array([branin(x) for x in X]) + 1) * (1 + 0.2 * X[:, 2])
    m.train(X, y)
    assert len(seen) == 2 and m.hypers.shape == (20, 6)
    assert np.all(np.isfinite(seen[-1]["lnpost"]))


@pytest.mark.parametrize("model_type,kw", [("gp_mcmc", dict(hyper_sampler="device_blocked")),
                                           ("gp", dict(hyper_optimizer="device_blocked"))])
def test_bayesian_optimization_facade(model_type, kw):
    from robo_b200.fmin.bayesian_optimization import bayesian_optimization
    res = bayesian_optimization(branin, LO, UP, num_iterations=30, model_type=model_type,
                                rng=np.random.RandomState(3), **kw)
    X = np.array(res["X"])
    assert len(X) == 30 and np.all(X >= LO) and np.all(X <= UP)
    assert np.all(np.isfinite(res["y"]))


# ---- argument errors -------------------------------------------------------------------------------------------------
def test_bad_arguments():
    from robo_b200 import _lib
    kernel = _kernel("m52_ard", 2)
    X, y = _data("m52_ard", 30, 2)
    h, _ = _handle(X, y, kernel, None)
    p0 = np.random.RandomState(0).rand(10, 4)
    with pytest.raises(ValueError, match="even"):
        _lib.sample_hypers_blocked(h, p0[:9], 5, 1)
    with pytest.raises(ValueError, match="dim"):
        _lib.hyper_lnpost_blocked(h, np.random.rand(2, 5))
    with pytest.raises(ValueError, match="steps"):
        _lib.sample_hypers_blocked(h, p0, -1, 1)
    with pytest.raises(ValueError, match="not finite"):
        _lib.optimize_hypers_blocked(h, np.r_[np.nan, 0, 0, 0])
    with pytest.raises(ValueError, match="maxcor"):
        _lib.optimize_hypers_blocked(h, np.zeros(4), maxcor=0)
    with pytest.raises(ValueError, match="hyper_batch_bytes"):
        h.set_option("hyper_batch_bytes", 0)
    h.set_data(X[:1], y[:1])
    with pytest.raises(ValueError, match="GPK_HYPER_BLOCKED_MAX_N"):
        _lib.hyper_lnpost_blocked(h, p0)
    Xb = np.random.RandomState(1).rand(_lib.HYPER_BLOCKED_MAX_N + 1, 2)
    h.set_data(Xb, Xb[:, 0])
    for call in (lambda: _lib.hyper_lnpost_blocked(h, p0), lambda: _lib.sample_hypers_blocked(h, p0, 1, 1),
                 lambda: _lib.optimize_hypers_blocked(h, p0[0])):
        with pytest.raises(ValueError, match="GPK_HYPER_BLOCKED_MAX_N"):
            call()
    h2 = _lib.Handle(0)
    with pytest.raises(ValueError, match="gpk_set_data"):
        _lib.hyper_lnpost_blocked(h2, p0)
    h.close()
    h2.close()
