"""The environment factor (Fabolas, gpk_set_env_factor) and the task factor (MTBO, gpk_set_task_factor) at every site
that applies them, against the extended-precision reference of tests/fit_reference.py and tests/es_reference.py:

  K           gpk_kernel_matrix with the factor == the same handle's K without it times the factor, bit for bit:
              fl(K0 fma(fl(c1 z), z', c0)) and fl(K0 K_t[a][b]); NaN off the tasks
  fit         factor, forward solve, log-det, log-likelihood and L^-1 (fit_reference) against that bit-checked K
  append      gpk_fit_append with a task or an environment value that only the appended rows hold
  nll_grad    grad_reference with the factor entries (the task entries with the host contraction's rounding)
  moments     gpk_predict, gpk_predict_cov / gpk_posterior_cov, gpk_predict_mean against cov_reference
  predict_grad   predict_grad_reference; the task axis exactly 0
  models      EI / PI / LCB with derivative=True through FabolasGP, MTBOGP and the sub-models of their MCMC classes:
              the value is the scoring path's, the gradient the device's taken through the model's input transform
  hyper       gpk_hyper_lnpost against hy_loglik_reference's first-order bound, -inf where K is not positive definite
  es          U and sigma of the entropy-search path against es_reference with the factor kernels

Every check prints its largest error-to-bound ratio ("ratio <check> <case> <value>").
"""
import math

import numpy as np
import pytest

from oracle import george_oracle as G
from robo_b200 import kernels as KM
from tests import es_reference as ER
from tests import fit_reference as R
from tests import kernel_cases as KC
from tests import task_kernel_model as TM

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not R.have_longdouble(), reason="np.longdouble is not an extended type here")]

NOISE = 1e-3
DIAG = NOISE + G.TINY
SHAPES = [1, 2, 31, 32, 33, 127, 128, 129, 255, 257, 640, 1153, 2049]
KINDS = ["env", "task"]
ENV = (0.1, -0.3)                              # log_a, log_b


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def gemm(A, B):
    import torch
    a = torch.from_numpy(np.ascontiguousarray(A, dtype=np.float64)).cuda()
    b = torch.from_numpy(np.ascontiguousarray(B, dtype=np.float64)).cuda()
    return (a @ b).cpu().numpy()


def report(check, case, r):
    print("ratio %-14s %-44s %.3e" % (check, case, r))
    assert r <= 1.0, "%s %s: error / bound = %.3g" % (check, case, r)


# ---- problems ----------------------------------------------------------------------------------------------------------
def task_theta(n_tasks, seed=0, diag=None):
    th = np.random.RandomState(200 + seed).uniform(-1.0, 0.3, TM.n_kt(n_tasks))
    if diag is not None:                        # log L_pp for p >= 1: K_t nearly rank 1 when very negative
        for p in range(1, n_tasks):
            th[p * (p + 1) // 2 + p] = diag
    return th


def flat_of(kind, case="m52", n_tasks=3, theta=None, env=ENV):
    f = KC.build(KM, case).flatten()
    D = KC.dim(case)
    if kind == "env":
        f["env"] = (D, env[0], env[1])
    elif kind == "task":
        f["task"] = (D, n_tasks, tuple(task_theta(n_tasks) if theta is None else theta))
    return f


def data(kind, case, N, seed=0, n_tasks=3, layout="shuffled", zclust=False):
    """KC's raw inputs plus the factor column: z = (1 - s)^2 of uniform s (clustered at 0 and 1 with zclust), or task
    indices in the given layout: 'shuffled', 'sorted', 'single' (the last task in one row), 'absent' (no row of the
    last task)."""
    X, y, _ = KC.data(case, "raw", N, 1, seed)
    rng = np.random.RandomState(N + 7 * seed)
    if kind == "env":
        s = rng.rand(N)
        if zclust:
            s = np.where(rng.rand(N) < 0.5, 1e-3 * rng.rand(N), 1 - 1e-3 * rng.rand(N))
        z = (1 - s) ** 2
    else:
        top = n_tasks - 1 if layout in ("single", "absent") and n_tasks > 1 else n_tasks
        z = rng.randint(0, top, N).astype(float)
        if N >= top:
            z[:top] = np.arange(top)            # every present task at least once
        if layout == "single" and n_tasks > 1:
            z[N // 2] = n_tasks - 1
        if layout == "sorted":
            z = np.sort(z)
        else:
            rng.shuffle(z)
    y = y + 0.3 * z
    return np.column_stack([X, z]), y


def set_factor(h, flat):
    if flat.get("env") is not None:
        h.set_env_factor(*flat["env"])
    if flat.get("task") is not None:
        h.set_task_factor(flat["task"][0], flat["task"][1], list(flat["task"][2]))


def new_handle(flat, X, y, factor=True):
    from robo_b200 import _lib
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(flat["family"], flat["log_amp"], flat["axis"], flat["group"], flat["log_metric"])
    if factor:
        set_factor(h, flat)
    return h


def expected_K(flat, X1, X2, K0):
    """gpk_factor_scale_kernel applied to the builder's K0: fl(K0 fma(fl(c1 z), z', c0)) or fl(K0 K_t[a][b])."""
    if flat.get("env") is not None:
        ax, la, lb = flat["env"]
        c0, c1 = math.exp(la), math.exp(lb)             # the C library's exp, as gpk_set_env_factor takes it
        F = ER.fma_exact((c1 * X1[:, ax])[:, None], X2[:, ax][None, :], c0)
        return K0 * F
    ax, nT, theta = flat["task"]
    return K0 * TM.task_value(X1[:, ax], X2[:, ax], np.asarray(theta), nT)


def device_K(flat, X1, X2=None, diag_add=None, check=True):
    """gpk_kernel_matrix with the factor; check: it equals the factor applied to the builder's K without it, bit for
    bit (NaN where the restatement has NaN)."""
    X2 = X1 if X2 is None else X2
    h = new_handle(flat, X1[:1], np.zeros(1), factor=False)
    K0 = h.kernel_matrix(X1, X2)
    set_factor(h, flat)
    K = h.kernel_matrix(X1, X2)
    h.close()
    if check:
        E = expected_K(flat, X1, X2, K0)
        assert np.array_equal(np.isnan(K), np.isnan(E))
        ok = ~np.isnan(E)
        bad = K[ok].view(np.int64) != E[ok].view(np.int64)
        assert not bad.any(), "%d of %d entries differ from the restated factor scaling" % (bad.sum(), bad.size)
    if diag_add is not None:
        K[np.diag_indices_from(K)] += diag_add
    return K


def state(h, n):
    return dict(L=h.get_factor(n), z=h.get_z(n), X=h.get_linv(n))


def check_fit(tag, flat, X, y, diag_add, mean, h, logdet, ll, panels=None, nodes=None):
    n = X.shape[0]
    s = state(h, n)
    K = device_K(flat, X, diag_add=diag_add)
    report("factor", tag, R.factor_check(s["L"], K, s["X"], gemm, panels=panels)[0])
    report("solve", tag, R.solve_check(s["L"], s["z"], y - mean, gemm)[0])
    report("logdet", tag, R.logdet_check(logdet, s["L"])[0])
    report("loglik", tag, R.loglik_check(ll, logdet, s["z"])[0])
    lc = R.linv_checks(s["L"], s["X"], gemm, nodes=nodes)
    assert lc["upper_zero"], tag
    report("linv_diag", tag, lc["diag"][0])
    report("linv_node", tag, lc["node"][0])
    return s


def fit_and_check(tag, flat, X, y, diag_add=DIAG):
    mean = float(np.mean(y))
    h = new_handle(flat, X, y)
    logdet, ll = h.fit(diag_add, mean)
    return h, check_fit(tag, flat, X, y, diag_add, mean, h, logdet, ll), mean


# ---- K bit for bit -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", SHAPES)
@pytest.mark.parametrize("kind", KINDS)
def test_kernel_matrix_bit_exact(kind, N):
    flat = flat_of(kind, n_tasks=5, theta=task_theta(5, N))
    X, _ = data(kind, "m52", N, n_tasks=5)
    if kind == "env":
        X[:min(N, 2), -1] = [0.0, 1.0][:min(N, 2)]        # z = 0 and z = 1
    device_K(flat, X)
    extra = np.repeat(X[:1], 4, axis=0)
    extra[:, -1] = [0.5, -1.0, 5.0, np.nan] if kind == "task" else [0.0, 1.0, 1e-300, 7.5]
    K = device_K(flat, np.vstack([X, extra]), X[:min(N, 300)])
    if kind == "task":                                     # coordinates that are not tasks give NaN
        assert np.all(np.isnan(K[N:]))
        assert not np.isnan(K[:N]).any()


# ---- the fit -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", SHAPES)
@pytest.mark.parametrize("kind", KINDS)
def test_fit_shapes(kind, N):
    X, y = data(kind, "m52", N)
    flat = flat_of(kind)
    h, s, mean = fit_and_check("%s m52 N=%d" % (kind, N), flat, X, y)
    h.close()


@pytest.mark.parametrize("case", KC.CASES)
@pytest.mark.parametrize("kind", KINDS)
def test_fit_kernel_cases(kind, case):
    """terms64 with the factor: 64 radial terms and the factor column, d = 33"""
    X, y = data(kind, case, 257)
    fit_and_check("%s %s N=257" % (kind, case), flat_of(kind, case), X, y)[0].close()


@pytest.mark.parametrize("kind", KINDS)
def test_fit_matern32(kind):
    X, y = data(kind, "m32", 1153)
    fit_and_check("%s m32 N=1153" % kind, flat_of(kind, "m32"), X, y)[0].close()


ILL = [("env", dict(env=(-6.0, 6.0), zclust=True)), ("env", dict(env=(-2.0, 9.5), zclust=True)),
       ("task", dict(diag=-8.0)), ("task", dict(diag=-4.0))]


@pytest.mark.parametrize("diag_add", [1e-6, G.TINY])
@pytest.mark.parametrize("ill", range(len(ILL)))
def test_fit_ill_conditioned(ill, diag_add):
    """log_b - log_a up to 12 with z clustered at 0 and 1; log L_pp down to -8 (K_t nearly rank 1); diag_add to TINY"""
    kind, kw = ILL[ill]
    N = 383
    if kind == "env":
        flat = flat_of("env", env=kw["env"])
        X, y = data("env", "m52", N, zclust=True)
    else:
        flat = flat_of("task", theta=task_theta(3, diag=kw["diag"]))
        X, y = data("task", "m52", N)
    K = device_K(flat, X, diag_add=diag_add)
    try:
        np.linalg.cholesky(K)
    except np.linalg.LinAlgError:
        pytest.skip("not positive definite in LAPACK either")
    print("kappa(K) = %.2e" % np.linalg.cond(K))
    fit_and_check("ill %d diag=%.0e" % (ill, diag_add), flat, X, y, diag_add)[0].close()


# ---- task layouts --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["shuffled", "sorted", "single", "absent"])
@pytest.mark.parametrize("n_tasks", [1, 2, 3, 5, 8])
def test_task_layouts(n_tasks, layout):
    N = 257
    flat = flat_of("task", n_tasks=n_tasks, theta=task_theta(n_tasks, n_tasks))
    X, y = data("task", "m52", N, n_tasks=n_tasks, layout=layout)
    tag = "task n=%d %s" % (n_tasks, layout)
    h, s, _ = fit_and_check(tag, flat, X, y)
    g = h.nll_grad(NOISE, len(flat["axis"]), n_kt=TM.n_kt(n_tasks))
    g_ref, bnd = R.grad_reference(flat, X, s["X"], s["z"], NOISE, gemm)
    report("grad", tag, R.ratio(np.abs(g - g_ref), bnd))
    if layout == "absent" and n_tasks > 1:                # row n_tasks - 1 of L touches only the absent task
        p = n_tasks - 1
        nr = len(flat["axis"]) + 1
        ent = [nr + p * (p + 1) // 2 + q for q in range(p + 1)]
        assert np.all(g[ent] == 0.0), g[ent]
    h.close()


# ---- gpk_fit_append -------------------------------------------------------------------------------------------------------
def append_panels(n, N1):
    return [(k, min(k + R.BM, n), min(k + R.BM, n), n) for k in range(0, N1, R.BM)] + [(0, N1, N1, n)]


@pytest.mark.parametrize("count", [1, 31, 33, 126])
@pytest.mark.parametrize("N1", [128, 256, 640])
@pytest.mark.parametrize("kind", KINDS)
def test_fit_append(kind, N1, count):
    n0 = N1 + 1
    n = n0 + count
    X, y = data(kind, "m52", n, seed=N1, n_tasks=3, layout="absent")
    if kind == "task":
        X[n0:, -1] = np.arange(count) % 3                  # task 2 appears in the appended rows only
        flat = flat_of("task")
    else:
        X[:n0, -1] = np.minimum(X[:n0, -1], 0.9)
        X[n - 1, -1] = 1.0                                  # z = 1 in an appended row only
        flat = flat_of("env")
    diag_add = DIAG
    h = new_handle(flat, X[:n0], y[:n0])
    h.fit(diag_add, float(np.mean(y[:n0])))
    h.get_linv(n0)
    mean = float(np.mean(y))
    r = h.fit_append(X, y, diag_add, mean)
    assert r is not None, "append not applicable at N1=%d n=%d" % (N1, n)
    nb = (n + R.BM - 1) // R.BM
    _, nodes = R.build_nodes(0, nb - 1)
    check_fit("%s append N1=%d n=%d" % (kind, N1, n), flat, X, y, diag_add, mean, h, r[0], r[1],
              panels=append_panels(n, N1), nodes=nodes + [(0, nb - 1, nb, 0)])
    h.close()


# ---- gpk_nll_grad ---------------------------------------------------------------------------------------------------------
def grad_check(tag, kind, case, N):
    flat = flat_of(kind, case)
    X, y = data(kind, case, N)
    mean = float(np.mean(y))
    h = new_handle(flat, X, y)
    h.fit(DIAG, mean)
    s = state(h, N)
    g = h.nll_grad(NOISE, len(flat["axis"]), env=kind == "env", n_kt=TM.n_kt(3) if kind == "task" else 0)
    g_ref, bnd = R.grad_reference(flat, X, s["X"], s["z"], NOISE, gemm)
    assert g.shape == g_ref.shape
    report("grad", tag, R.ratio(np.abs(g - g_ref), bnd))
    h.close()


@pytest.mark.parametrize("N", [96, 257])
@pytest.mark.parametrize("case", KC.CASES)
@pytest.mark.parametrize("kind", KINDS)
def test_nll_grad_kernel_cases(kind, case, N):
    grad_check("%s %s N=%d" % (kind, case, N), kind, case, N)


@pytest.mark.parametrize("N", [31, 32, 33, 127, 128, 129, 255, 256, 383, 640])
@pytest.mark.parametrize("kind", KINDS)
def test_nll_grad_shapes(kind, N):
    grad_check("%s m52 N=%d" % (kind, N), kind, "m52", N)


# ---- moments -------------------------------------------------------------------------------------------------------------
BOUNDS = (np.array([-1.0, 0.0, 0.0, 0.0]), np.array([2.0, 3.0, 1.0, 2.0]))


def candidates(kind, m, X, seed, bounds=None):
    rng = np.random.RandomState(seed)
    Xs = rng.rand(m, X.shape[1])
    Xs[:min(m, 8)] = X[:min(m, 8)]                           # on the data: the variance cancels, the clip engages
    if kind == "task":
        Xs[8:, -1] = rng.randint(0, 3, max(m - 8, 0))
    if bounds is not None:
        Xs = bounds[0] + Xs * (bounds[1] - bounds[0])
    return Xs


def scaled(Xs, bounds):
    return Xs if bounds is None else (Xs - bounds[0]) / (bounds[1] - bounds[0])


def kstar_err(flat, Ks, Kss_d, s, bounds):
    """Extra error where the device scales candidates on the fly and gpk_kernel_matrix is given host-scaled inputs:
    (n_terms + 16) u per K* / k** entry, carried through alpha (mean) and w (variance)."""
    if bounds is None:
        return 0.0, 0.0
    e = (len(flat["axis"]) + 16) * R.U
    a = np.abs(s["X"].T @ s["z"])
    W = np.abs(s["X"]).T @ gemm(np.abs(s["X"]), np.abs(Ks.T))
    return e * (np.abs(Ks) @ a), e * (2 * np.sum(np.abs(Ks) * W.T, axis=1) + np.abs(Kss_d))


@pytest.mark.parametrize("transform", [False, True])
@pytest.mark.parametrize("m", [1, 127, 128, 129, 383, 1000])
@pytest.mark.parametrize("kind", ["env", "env_bounds", "task"])
def test_posterior_cov(kind, m, transform):
    fk = kind[:3] if kind != "task" else "task"
    bounds = BOUNDS if kind == "env_bounds" else None
    flat = flat_of(fk)
    X, y = data(fk, "m52", 257)
    h, s, mean = fit_and_check("cov base %s" % kind, flat, X, y)
    if bounds is not None:
        h.set_input_bounds(*bounds)
    Xs = candidates(fk, m, scaled(X, None), m, bounds)
    if bounds is not None:
        Xs[:min(m, 8)] = bounds[0] + X[:min(m, 8)] * (bounds[1] - bounds[0])
    y_mean, y_std = (5.0, 37.0) if transform else (0.0, 1.0)
    h.set_output_transform(transform, y_mean, y_std)
    ys2 = y_std * y_std
    Xn = scaled(Xs, bounds)
    Ks, Kss = device_K(flat, Xn, X), device_K(flat, Xn)
    ref = R.cov_reference(s["X"], Ks, Kss, s["z"], mean, ys2, y_mean, y_std, gemm)
    em, ev = kstar_err(flat, Ks, np.diag(Kss), s, bounds)
    mb = ref["mu_bound"] + em * y_std
    tag = "%s m=%d transform=%s" % (kind, m, transform)
    for clip, fn in ((False, h.posterior_cov), (True, h.predict_cov)):
        mu, cov = fn(Xs)
        report("cov_mu", tag, R.ratio(np.abs(mu - ref["mu"]), mb))
        cb = ref["cov_bound"] + (np.sqrt(np.outer(ev, ev)) * ys2 if bounds is not None else 0.0)
        if clip:
            r, bad = ER.sigma_check(cov, ref["cov"], cb)
            assert not bad.any(), "%d entries outside the bound or not exactly the clip value" % bad.sum()
        else:
            r = R.ratio(np.abs(cov - ref["cov"]), cb)
        report("cov_clip" if clip else "cov_raw", tag, r)
    # gpk_predict (the scoring pass) and gpk_predict_mean (the mean-only builder) against the same reference
    mu, var = h.predict(Xs)
    report("pred_mu", tag, R.ratio(np.abs(mu - ref["mu"]), mb))
    r, bad = ER.sigma_check(var, np.diag(ref["cov"]), np.diag(ref["cov_bound"]) + ev * ys2)
    assert not bad.any()
    report("pred_var", tag, r)
    report("mean_only", tag, R.ratio(np.abs(h.predict_mean(Xs) - ref["mu"]), mb))
    h.close()


@pytest.mark.parametrize("opts", [{}, {"chunk": 1024}])
@pytest.mark.parametrize("kind", ["env", "env_bounds", "task"])
def test_predict_many_candidates(kind, opts):
    """m > 2048 rows: several pipelined chunks with chunk < m, and candidate counts that stride the factor kernel's grid"""
    from robo_b200 import _lib
    fk = kind[:3] if kind != "task" else "task"
    bounds = BOUNDS if kind == "env_bounds" else None
    flat = flat_of(fk)
    X, y = data(fk, "m52", 640)
    mean = float(np.mean(y))
    h = _lib.Handle(0)
    for k, v in opts.items():
        h.set_option(k, v)
    h.set_data(X, y)
    h.set_kernel(flat["family"], flat["log_amp"], flat["axis"], flat["group"], flat["log_metric"])
    set_factor(h, flat)
    h.fit(DIAG, mean)
    s = state(h, 640)
    if bounds is not None:
        h.set_input_bounds(*bounds)
    h.set_output_transform(True, 0.7, 1.9)
    m = 4099
    Xs = candidates(fk, m, X, 31, bounds)
    Xn = scaled(Xs, bounds)
    Ks = device_K(flat, Xn, X)
    # k(x*, x*): the diagonal of gpk_kernel_matrix, taken in 1 x 1 blocks of the same bits
    h2 = new_handle(flat, X[:1], np.zeros(1))
    kss = np.array([h2.kernel_matrix(Xn[i:i + 1], Xn[i:i + 1])[0, 0] for i in range(m)])
    h2.close()
    ref = R.cov_reference(s["X"], Ks, kss, s["z"], mean, 1.9 ** 2, 0.7, 1.9, gemm)
    em, ev = kstar_err(flat, Ks, kss, s, bounds)
    mu, var = h.predict(Xs)
    tag = "%s m=%d %s" % (kind, m, opts)
    report("pred_mu", tag, R.ratio(np.abs(mu - ref["mu"]), ref["mu_bound"] + em * 1.9))
    r, bad = ER.sigma_check(var, ref["cov"], ref["cov_bound"] + ev * 1.9 ** 2)
    assert not bad.any()
    report("pred_var", tag, r)
    report("mean_only", tag, R.ratio(np.abs(h.predict_mean(Xs) - ref["mu"]), ref["mu_bound"] + em * 1.9))
    h.close()


# ---- gpk_predict_grad ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [33, 129, 257, 640])
@pytest.mark.parametrize("kind", ["env", "env_bounds", "task"])
def test_predict_grad(kind, N):
    """N > 224: every warp of the gradient kernel holds a partial sum"""
    fk = kind[:3] if kind != "task" else "task"
    bounds = BOUNDS if kind == "env_bounds" else None
    flat = flat_of(fk)
    X, y = data(fk, "m52", N)
    h, s, mean = fit_and_check("pgrad base %s N=%d" % (kind, N), flat, X, y)
    if bounds is not None:
        h.set_input_bounds(*bounds)
    h.set_output_transform(True, 0.7, 1.9)
    Xs = candidates(fk, 64, X, N, bounds)
    r = h.predict_grad(Xs)
    lo, up = (None, None) if bounds is None else bounds
    dmu, dvar, bm, bv = R.predict_grad_reference(flat, X, s["X"], s["z"], Xs, lo, up, 1.9, gemm)
    tag = "%s N=%d" % (kind, N)
    report("pgrad_mu", tag, R.ratio(np.abs(r["dmu"] - dmu), bm))
    report("pgrad_var", tag, R.ratio(np.abs(r["dvar"] - dvar), bv))
    if fk == "task":
        assert np.all(r["dmu"][:, -1] == 0.0) and np.all(r["dvar"][:, -1] == 0.0)
    h.close()


# ---- EI / PI / LCB input gradients through the factor models ------------------------------------------------------------
LOWER, UPPER = np.array([-1.0, 0.5]), np.array([2.0, 4.0])


def _model(name):
    from robo_b200 import kernels
    from robo_b200.models.fabolas_gp import FabolasGP, FabolasGPMCMC
    from robo_b200.models.mtbo_gp import MTBOGP, MTBOGPMCMC
    if name.startswith("fabolas"):
        k = 1.3 * kernels.Matern52Kernel(np.ones(1) * 0.4, ndim=3, axes=0)
        k *= kernels.Matern52Kernel(np.ones(1) * 0.6, ndim=3, axes=1)
        k *= kernels.BayesianLinearRegressionKernel(0.1, -0.3, ndim=3, axes=2)
        basis = (lambda s: s) if name.endswith("linear") else (lambda s: (1 - s) ** 2)
        if "mcmc" in name:
            return FabolasGPMCMC(k, basis_func=basis, lower=LOWER, upper=UPPER, noise=np.log(NOISE),
                                 rng=np.random.RandomState(0))
        return FabolasGP(k, basis_function=basis, lower=LOWER, upper=UPPER, noise=NOISE, rng=np.random.RandomState(0))
    from robo_b200.fmin.mtbo import _mtbo_kernel
    k, task = _mtbo_kernel(2, 3)
    k.set_parameter_vector(np.r_[0.0, np.log([0.3, 0.5]), task_theta(3)])
    if "mcmc" in name:
        return MTBOGPMCMC(k, lower=LOWER, upper=UPPER, noise=np.log(NOISE), rng=np.random.RandomState(0))
    return MTBOGP(k, lower=LOWER, upper=UPPER, noise=NOISE, rng=np.random.RandomState(0))


def _raw(name, n, seed):
    rng = np.random.RandomState(seed)
    X = np.column_stack([LOWER + rng.rand(n, 2) * (UPPER - LOWER),
                         rng.randint(0, 3, n).astype(float) if name.startswith("mtbo") else rng.rand(n)])
    return X, np.sin(X[:, 0]) + np.cos(2 * X[:, 1]) + 0.5 * X[:, 2]


@pytest.mark.parametrize("acq", ["ei", "pi", "lcb"])
@pytest.mark.parametrize("name", ["fabolas", "fabolas_linear", "fabolas_mcmc", "mtbo", "mtbo_mcmc"])
def test_acquisition_gradients_through_the_models(name, acq):
    """compute(X, derivative=True) scores the same points as compute(X), and its gradient is the device's gradient at
    the model's transformed inputs taken back through the transform; central differences of compute(X) in the raw
    inputs confirm the chain rule"""
    from robo_b200.acquisition_functions import EI, LCB, PI
    X, y = _raw(name, 150, 3)
    model = _model(name)
    model.train(X, y, do_optimize=False)
    sub = model.models[0] if "mcmc" in name else model
    A = {"ei": EI, "pi": PI, "lcb": LCB}[acq](sub)
    Xc, _ = _raw(name, 40, 4)
    Xc[:, -1] = np.clip(Xc[:, -1], 0.05, 0.95) if name.startswith("fabolas") else Xc[:, -1]
    f, df = A.compute(Xc, derivative=True)
    f0 = A.compute(Xc)
    np.testing.assert_allclose(f, np.ravel(f0), rtol=1e-12, atol=1e-300)
    # the device gradient at the transformed inputs, and the transform's chain rule
    Xd = sub.normalize(Xc)
    eta = 0.0 if acq == "lcb" else sub.get_incumbent()[1]
    from robo_b200 import _lib
    r = sub.gp.predict_grad(Xd, _lib.ACQ_KIND[acq], float(eta), float(A.par))
    J = np.column_stack([np.tile(1.0 / (UPPER - LOWER), (len(Xc), 1)),
                         np.zeros(len(Xc)) if name.startswith("mtbo") else
                         (np.ones(len(Xc)) if name.endswith("linear") else -2.0 * (1.0 - Xc[:, -1]))])
    np.testing.assert_allclose(df, r["df"] * J, rtol=1e-14, atol=0)
    dmu, dvar = sub.predictive_gradients(Xc)
    np.testing.assert_allclose(dmu, r["dmu"] * J, rtol=1e-14, atol=0)
    np.testing.assert_allclose(dvar, r["dvar"] * J, rtol=1e-14, atol=0)
    step = 1e-6
    for a in range(3 if name.startswith("fabolas") else 2):
        Xp, Xm = Xc.copy(), Xc.copy()
        Xp[:, a] += step
        Xm[:, a] -= step
        fd = (np.ravel(A.compute(Xp)) - np.ravel(A.compute(Xm))) / (2 * step)
        np.testing.assert_allclose(df[:, a], fd, rtol=1e-5, atol=1e-6 * max(1.0, np.abs(fd).max()))
    if name.startswith("mtbo"):
        assert np.all(df[:, -1] == 0.0)


def test_unknown_basis_function_has_no_gradient():
    from robo_b200.acquisition_functions import EI
    from robo_b200.models.fabolas_gp import FabolasGP
    model = _model("fabolas")
    model = FabolasGP(model.kernel, basis_function=lambda s: np.sqrt(s), lower=LOWER, upper=UPPER, noise=NOISE)
    X, y = _raw("fabolas", 50, 5)
    model.train(X, y, do_optimize=False)
    with pytest.raises(NotImplementedError):
        EI(model).compute(X[:4], derivative=True)


# ---- gpk_hyper_lnpost ----------------------------------------------------------------------------------------------------
def _hyper_setup(prior_kind, N):
    from robo_b200 import _lib, kernels
    from robo_b200.device_gp import TINY
    from robo_b200.models.gaussian_process_mcmc import _hyper_prior
    from robo_b200.priors import DefaultPrior, EnvPrior, MTBOPrior
    rng = np.random.RandomState(N)
    X = rng.rand(N, 3)
    if prior_kind == "task":
        from robo_b200.fmin.mtbo import _mtbo_kernel
        kernel, task = _mtbo_kernel(2, 3)
        X[:, 2] = rng.randint(0, 3, N)
        prior = MTBOPrior(len(kernel) + 1, n_ls=2, n_kt=len(task), rng=np.random.RandomState(0))
    else:
        kernel = 1.3 * kernels.Matern52Kernel(np.ones(1) * 0.4, ndim=3, axes=0)
        kernel *= kernels.Matern52Kernel(np.ones(1) * 0.6, ndim=3, axes=1)
        if prior_kind == "env":
            X[:, 2] = (1 - X[:, 2]) ** 2
            kernel *= kernels.BayesianLinearRegressionKernel(0.1, 0.1, ndim=3, axes=2)
            prior = EnvPrior(len(kernel) + 1, n_ls=2, n_lr=2, rng=np.random.RandomState(0))
        else:
            prior = DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(0))
    y = np.sin(3 * X[:, 0]) + 0.3 * X[:, 2] + 0.05 * rng.randn(N)
    f = kernel.flatten()
    kind, par, n_ls, n_lr = _hyper_prior(prior)
    mean = float(np.mean(y))
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    set_factor(h, f)
    _lib.set_hyper_model(h, f["slots"], len(f["axis"]), mean, TINY, kind, par, n_ls, n_lr)
    return h, kernel, X, y, mean


def _thetas(prior_kind, dim, rng):
    """a moderate theta, and the ill-conditioned ones of the fit tests (log_b - log_a = 12; log L_pp = -8), small noise"""
    base = np.zeros(dim)
    base[-1] = -6.0
    out = [base.copy()]
    if prior_kind == "env":
        t = base.copy()
        t[3:5] = (-6.0, 6.0)
        out.append(t)
    if prior_kind == "task":
        t = base.copy()
        t[3:9] = task_theta(3, diag=-8.0)
        out.append(t)
    t = base.copy()
    t[-1] = -14.0
    out.append(t)
    out.append(base + rng.uniform(-0.5, 0.5, dim))
    return np.array(out)


@pytest.mark.parametrize("N", [1, 3, 31, 32, 33, 128, 129, 231, 232])
@pytest.mark.parametrize("prior_kind", ["none", "env", "task"])
def test_hyper_lnpost(prior_kind, N):
    from copy import deepcopy
    from robo_b200 import _lib
    from robo_b200.device_gp import TINY
    h, kernel, X, y, mean = _hyper_setup(prior_kind, N)
    dim = len(kernel) + 1
    T = _thetas(prior_kind, dim, np.random.RandomState(N))
    ll, _ = _lib.hyper_lnpost(h, T)
    worst = 0.0
    for t, l in zip(T, ll):
        k = deepcopy(kernel)
        k.set_parameter_vector(t[:-1])
        flat = k.flatten()
        yerr = np.sqrt(np.exp(t[-1]))
        diag = float(np.sqrt(np.float64(yerr) ** 2 + TINY) ** 2)
        ref = R.hy_loglik_reference(flat, X, y, mean, diag, n_tasks=3 if prior_kind == "task" else 0)
        if ref is None:
            assert l == -np.inf
            continue
        if ref["first_order"] > 0.1:
            print("first order %.2e: theta %s left out" % (ref["first_order"], t))
            continue
        worst = max(worst, abs(l - float(ref["ll"])) / ref["bound"])
    report("hy_ll", "%s N=%d" % (prior_kind, N), worst)
    h.close()


# ---- entropy search with a factor ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 129, 640])
@pytest.mark.parametrize("kind", KINDS)
def test_es_factor(kind, N):
    """U = K^-1 K(X, zb) and sigma from gpk_es_get_u / gpk_es_moments against es_reference with the factor kernel"""
    from oracle import robo_oracle as O
    from tests import env_kernel_model as EM
    flat = flat_of(kind, "prod1d")
    X, y = data(kind, "prod1d", N)
    if kind == "env":
        ok = EM.fabolas_kernel(3, flat["log_amp"], flat["log_metric"], *ENV)
    else:
        ok = TM.mtbo_kernel(3, flat["log_amp"], flat["log_metric"], np.asarray(flat["task"][2]), 3)
    st = O.gp_fit(ok, X, y, noise=NOISE, normalize_input=False)
    ref = ER.Reference(st)
    h = new_handle(flat, X, y)
    h.fit(DIAG, float(np.mean(y)))
    rng = np.random.RandomState(N)
    zb = rng.rand(20, 4)
    Xs = rng.rand(50, 4)
    if kind == "task":
        zb[:, -1] = rng.randint(0, 3, 20)
        Xs[:, -1] = rng.randint(0, 3, 50)
    lmb = np.log(np.full(20, 1.0 / 20))
    h.es_update(zb, lmb, NOISE, np.random.RandomState(1).randn(40), np.zeros(4), np.ones(4))
    U = h.es_get_u()
    U_ref, zs = ref.u(zb)
    dU = U - U_ref.astype(np.float64)
    tag = "%s N=%d" % (kind, N)
    report("es_u", tag, R.ratio(np.abs(dU), ref.u_bound(U_ref)))
    _, sig = h.es_moments(Xs)
    s_ref, mag, absK = ref.sigma(U_ref, zs, Xs)
    r, bad = ER.sigma_check(sig, s_ref, ref.sigma_bound(mag, absK, dU))
    assert not bad.any(), "%d sigma entries outside the bound" % bad.sum()
    report("es_sigma", tag, r)
    h.close()
