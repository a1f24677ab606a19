"""The fp64 fit path at every block shape, against the extended-precision reference of tests/fit_reference.py: backward
errors and per-stage errors taken against the device's OWN upstream outputs (its K from gpk_kernel_matrix + diag_add,
its L^, z^ and X^ = L^-1), so that the bounds depend on magnitudes only and stay tight where kappa(K) is large.

  fit         factor |L^ L^T - K|, forward solve |L^ z^ - (y - mean)|, log-det against 2 sum log L^_ii, log-likelihood
  L^-1        every diagonal tile, every node of the device's inversion tree, upper triangle exactly 0
  append      gpk_fit_append at every split-K position of the 512-column chunks: the appended factor within the backward
              bound of a fresh fit of the same rows (its block row by one explicit-inverse panel over N1 columns), the
              last diagonal tile, and P[b, :N1] as the node (0, b, nb)
  nll_grad    every kernel case and the noise entry against the gradient from the device's X^ and z^ in longdouble
  covariance  mu and every entry of gpk_predict_cov / gpk_posterior_cov, raw and with the output transform
  not PD      the failing pivot the device reports == LAPACK dpotrf's info - 1, and the handle refits to a fresh handle's
              bits
  reuse       one handle through set_data / fit with N, NP and d changing, a failed fit and fit_append: bit-identical to
              fresh handles

Every check prints its largest error-to-bound ratio ("ratio <check> <case> <value>").  The exact products of the
reference run as fp64 GEMMs on the GPU through torch (every slice product is exact in any summation order, see
fit_reference), the longdouble sums on the host.
"""
import re

import numpy as np
import pytest
import scipy.linalg as spla

from oracle import george_oracle as G
from robo_b200 import kernels as KM
from tests import es_reference as ER
from tests import fit_reference as R
from tests import kernel_cases as KC

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not R.have_longdouble(), reason="np.longdouble is not an extended type here")]

NOISE = 1e-3
SHAPES = [1, 2, 16, 17, 127, 128, 129, 255, 256, 257, 383, 640, 896, 1153, 1408, 2049, 6145]


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
    print("ratio %-14s %-40s %.3e" % (check, case, r))
    assert r <= 1.0, "%s %s: error / bound = %.3g" % (check, case, r)


# ---- problems ----------------------------------------------------------------------------------------------------------
def flat_of(case):
    return KC.build(KM, case).flatten()


def raw_data(case, N, seed=0):
    X, y, _ = KC.data(case, "raw", N, 1, seed)
    return X, y


def clustered(N, D, seed=0):
    """N points in N / 8 tight clusters (spread 1e-3 of the unit cube)"""
    rng = np.random.RandomState(N + seed)
    C = rng.rand(max(N // 8, 1), D)
    X = C[np.arange(N) % len(C)] + 1e-3 * rng.randn(N, D)
    return X, np.sin(3 * X).sum(axis=1)


def new_handle(flat, X, y):
    from robo_b200 import _lib
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(flat["family"], flat["log_amp"], flat["axis"], flat["group"], flat["log_metric"])
    return h


def device_K(flat, X1, X2=None, diag_add=None):
    from robo_b200 import _lib
    h = _lib.Handle(0)
    h.set_kernel(flat["family"], flat["log_amp"], flat["axis"], flat["group"], flat["log_metric"])
    K = h.kernel_matrix(X1, X1 if X2 is None else X2)
    h.close()
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


def fit_and_check(tag, flat, X, y, diag_add=NOISE + G.TINY):
    mean = float(np.mean(y))
    h = new_handle(flat, X, y)
    logdet, ll = h.fit(diag_add, mean)
    s = check_fit(tag, flat, X, y, diag_add, mean, h, logdet, ll)
    return h, s, mean


# ---- fit and L^-1 at every block shape ----------------------------------------------------------------------------------
@pytest.mark.parametrize("N", SHAPES)
def test_fit_shapes(N):
    X, y = raw_data("m52", N)
    h, s, mean = fit_and_check("m52 N=%d" % N, flat_of("m52"), X, y)
    if N > 1:                               # alpha through the posterior mean: mu - mean = K* X^T z
        Xs = np.random.RandomState(N).rand(64, X.shape[1])
        mu = h.predict(Xs)[0]
        ref = R.cov_reference(s["X"], device_K(flat_of("m52"), Xs, X), device_K(flat_of("m52"), Xs), s["z"], mean,
                              gemm=gemm)
        report("mean_alpha", "m52 N=%d" % N, R.ratio(np.abs(mu - ref["mu"]), ref["mu_bound"]))
    h.close()


@pytest.mark.parametrize("case", KC.CASES)
@pytest.mark.parametrize("N", [129, 640])
def test_fit_kernel_cases(case, N):
    X, y = raw_data(case, N)
    fit_and_check("%s N=%d" % (case, N), flat_of(case), X, y)[0].close()


@pytest.mark.parametrize("N", [257, 1153])
def test_fit_matern32(N):
    X, y = raw_data("m32", N)
    fit_and_check("m32 N=%d" % N, flat_of("m32"), X, y)[0].close()


@pytest.mark.parametrize("diag_add", [1e-6, 1e-9, G.TINY])
@pytest.mark.parametrize("N", [383, 1153])
def test_fit_ill_conditioned(N, diag_add):
    """clustered inputs, the diagonal term down to TINY: kappa(K) up to ~1e12, the same bounds"""
    flat = flat_of("m52")
    X, y = clustered(N, 3)
    K = device_K(flat, X, diag_add=diag_add)
    try:
        np.linalg.cholesky(K)
    except np.linalg.LinAlgError:
        pytest.skip("not positive definite in LAPACK either")
    print("kappa(K) = %.2e" % np.linalg.cond(K))
    fit_and_check("clustered N=%d diag=%.0e" % (N, diag_add), flat, X, y, diag_add)[0].close()


# ---- gpk_fit_append ------------------------------------------------------------------------------------------------------
def append_panels(n, N1):
    """the default 128-tile panels, plus the appended block row as one panel over the N1 leading columns"""
    return [(k, min(k + R.BM, n), min(k + R.BM, n), n) for k in range(0, N1, R.BM)] + [(0, N1, N1, n)]


@pytest.mark.parametrize("N1", [128, 256, 512, 640, 1024, 1152])
@pytest.mark.parametrize("counts", [(1,), (31,), (32,), (33,), (126,), (31, 32, 33)])
def test_fit_append(N1, counts):
    flat = flat_of("m52")
    n_all = N1 + 1 + sum(counts)
    X, y = raw_data("m52", n_all, seed=N1)
    n0 = N1 + 1
    diag_add = NOISE + G.TINY
    h = new_handle(flat, X[:n0], y[:n0])
    h.fit(diag_add, float(np.mean(y[:n0])))
    h.get_linv(n0)                          # L^-1 built: the precondition of the shortcut
    n = n0
    for c in counts:
        n += c
        mean = float(np.mean(y[:n]))
        r = h.fit_append(X[:n], y[:n], diag_add, mean)
        assert r is not None, "append not applicable at N1=%d n=%d" % (N1, n)
        nb = (n + R.BM - 1) // R.BM
        _, nodes = R.build_nodes(0, nb - 1)
        check_fit("append N1=%d n=%d" % (N1, n), flat, X[:n], y[:n], diag_add, mean, h, r[0], r[1],
                  panels=append_panels(n, N1), nodes=nodes + [(0, nb - 1, nb, 0)])
    h.close()


# ---- gpk_nll_grad ----------------------------------------------------------------------------------------------------------
def grad_check(tag, case, N, diag_add=NOISE + G.TINY, seed=0):
    flat = flat_of(case)
    X, y = raw_data(case, N, seed)
    mean = float(np.mean(y))
    h = new_handle(flat, X, y)
    h.fit(diag_add, mean)
    s = state(h, N)
    g = h.nll_grad(NOISE, len(flat["axis"]))
    g_ref, bnd = R.grad_reference(flat, X, s["X"], s["z"], NOISE, gemm)
    report("grad", tag, R.ratio(np.abs(g - g_ref), bnd))
    return h, g, flat, X, y, mean


@pytest.mark.parametrize("N", [31, 32, 33, 127, 128, 129, 255, 257, 383, 640])
def test_nll_grad_shapes(N):
    grad_check("m52 N=%d" % N, "m52", N)[0].close()


@pytest.mark.parametrize("case", KC.CASES)
@pytest.mark.parametrize("N", [96, 257])
def test_nll_grad_kernel_cases(case, N):
    grad_check("%s N=%d" % (case, N), case, N)[0].close()


def test_nll_grad_finite_differences():
    """well conditioned: the log-amplitude and noise entries against central differences of the device's loglik"""
    h, g, flat, X, y, mean = grad_check("fd m52 N=200", "m52", 200)
    step = 1e-5

    def ll(log_amp, noise):
        hh = new_handle(dict(flat, log_amp=log_amp), X, y)
        v = hh.fit(noise + G.TINY, mean)[1]
        hh.close()
        return v
    fd_amp = -(ll(flat["log_amp"] + step, NOISE) - ll(flat["log_amp"] - step, NOISE)) / (2 * step)
    fd_noise = -(ll(flat["log_amp"], NOISE * np.exp(step)) - ll(flat["log_amp"], NOISE * np.exp(-step))) / (2 * step)
    assert abs(g[0] - fd_amp) <= 1e-6 * max(1.0, abs(g[0]))
    assert abs(g[-1] - fd_noise) <= 1e-6 * max(1.0, abs(g[-1]))
    h.close()


# ---- gpk_predict_cov / gpk_posterior_cov -------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 127, 128, 129, 383, 1000])
@pytest.mark.parametrize("transform", [False, True])
def test_posterior_cov(m, transform):
    flat = flat_of("m52")
    N = 257
    X, y = raw_data("m52", N)
    h, s, mean = fit_and_check("cov base", flat, X, y)
    rng = np.random.RandomState(m)
    Xs = rng.rand(m, X.shape[1])
    Xs[:min(m, 8)] = X[:min(m, 8)]                 # on the data: the variance cancels to ~0 and the clip engages
    y_mean, y_std = (5.0, 37.0) if transform else (0.0, 1.0)
    h.set_output_transform(transform, y_mean, y_std)
    ys2 = y_std * y_std
    ref = R.cov_reference(s["X"], device_K(flat, Xs, X), device_K(flat, Xs), s["z"], mean, ys2, y_mean, y_std, gemm)
    tag = "m=%d transform=%s" % (m, transform)
    for clip, fn in ((False, h.posterior_cov), (True, h.predict_cov)):
        mu, cov = fn(Xs)
        report("cov_mu", tag, R.ratio(np.abs(mu - ref["mu"]), ref["mu_bound"]))
        if clip:
            r, bad = ER.sigma_check(cov, ref["cov"], ref["cov_bound"])
            assert not bad.any(), "%d entries outside the bound or not exactly the clip value" % bad.sum()
            assert np.all(cov >= R.EPS)
        else:
            r = R.ratio(np.abs(cov - ref["cov"]), ref["cov_bound"])
        report("cov_clip" if clip else "cov_raw", tag, r)
        np.testing.assert_array_equal(cov, cov.T)   # exactly symmetric: K** is, and tiles (a, b), (b, a) of V^T V
    h.close()


# ---- not positive definite ------------------------------------------------------------------------------------------------
def grid_inputs(N):
    g = int(np.ceil(np.sqrt(N)))
    pts = np.stack(np.meshgrid(np.arange(g), np.arange(g), indexing="ij"), -1).reshape(-1, 2)[:N] / g
    return pts + 0.1 / g


@pytest.mark.parametrize("pivot", [0, 15, 16, 127, 128, 129, 300])
def test_not_pd_pivot(pivot):
    """well-spaced inputs, row `pivot` a duplicate of an earlier row (of row 5 for a later block, so the GEMM updates
    carry the cancellation), diag_add = -1e-6: the pivot there is about -2e-6 and every earlier one clearly positive.
    Pivot 0: diag_add below -k(x, x), so the very first pivot is negative."""
    from robo_b200 import _lib
    flat = dict(family=_lib.MATERN52, log_amp=0.0, axis=[0, 1], group=[0, 0], log_metric=[np.log(5e-4)] * 2)
    N = 400
    X = grid_inputs(N)
    if pivot > 0:
        X[pivot] = X[5 if pivot >= 128 else pivot - 1]
    y = np.cos(5 * X).sum(axis=1)
    diag_add = -1.5 if pivot == 0 else -1e-6
    K = device_K(flat, X, diag_add=diag_add)
    _, info = spla.lapack.dpotrf(K, lower=1)
    assert info == pivot + 1
    h = new_handle(flat, X, y)
    with pytest.raises(np.linalg.LinAlgError) as ei:
        h.fit(diag_add, 0.0)
    got = int(re.search(r"pivot (-?\d+)", str(ei.value)).group(1))
    assert got == info - 1, (str(ei.value), info)
    # the same handle refits to the bits of a fresh one
    logdet, ll = h.fit(NOISE, 0.0)
    f = new_handle(flat, X, y)
    logdet2, ll2 = f.fit(NOISE, 0.0)
    assert (logdet, ll) == (logdet2, ll2)
    assert_same_state(h, f, N)
    h.close()
    f.close()


# ---- handle reuse ------------------------------------------------------------------------------------------------------------
def assert_same_state(h, f, n, Xs=None):
    a, b = state(h, n), state(f, n)
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    if Xs is not None:
        for x, y in zip(h.predict(Xs), f.predict(Xs)):
            np.testing.assert_array_equal(x, y)


def test_handle_reuse():
    """one handle through N shrinking and growing inside one NP and across NP, d changing, a not-PD failure and
    fit_append: after every step its factor, z, L^-1, log-det, log-likelihood and posterior equal a fresh handle's bits"""
    from robo_b200 import _lib
    h = _lib.Handle(0)
    diag_add = NOISE + G.TINY
    steps = [("m52", 300), ("m52", 260), ("m52", 383), ("m52", 700), ("m52", 129), ("m32", 200), ("terms64", 257),
             ("m52", 300)]
    for i, (case, N) in enumerate(steps):
        flat = flat_of(case)
        X, y = raw_data(case, N, seed=i)
        Xs = np.random.RandomState(i).rand(50, X.shape[1])
        h.set_data(X, y)
        h.set_kernel(flat["family"], flat["log_amp"], flat["axis"], flat["group"], flat["log_metric"])
        if i == 4:                                          # a failed fit first
            with pytest.raises(np.linalg.LinAlgError):
                h.fit(-2.0, 0.0)
        r = h.fit(diag_add, float(np.mean(y)))
        f = new_handle(flat, X, y)
        assert r == f.fit(diag_add, float(np.mean(y))), (case, N)
        assert_same_state(h, f, N, Xs)
        f.close()
        if i == 1:                                          # fit_append on the reused handle and on a fresh one
            X2, y2 = raw_data(case, 300, seed=99)
            X2[:N], y2[:N] = X, y
            for hh in (h, new_handle(flat, X, y)):
                if hh is not h:
                    hh.fit(diag_add, float(np.mean(y)))
                hh.get_linv(N)
                ra = hh.fit_append(X2, y2, diag_add, float(np.mean(y2)))
                assert ra is not None
                if hh is not h:
                    assert ra == rh
                    assert_same_state(h, hh, 300, Xs)
                    hh.close()
                else:
                    rh = ra
    h.close()
