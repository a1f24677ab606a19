"""tests/blr_reference.py checks itself without a GPU: the float64 restatement tests/blr_model.py (np.linalg.inv /
det, a different fp64 algorithm) lies inside the same bounds at the shapes of tests/test_gpu_blr_shapes.py, ill-conditioned
ones included, and a numpy emulation of the device's algorithms (gpk_blr_gram_kernel, gpk_blr_factor, gpk_blr_eval,
gpk_blr_score_kernel) lies inside them while each injected defect breaks them at the shapes where it bites."""
import numpy as np
import pytest

from tests import blr_model as BM
from tests import blr_reference as R
from tests.fit_reference import have_longdouble

pytestmark = pytest.mark.skipif(not have_longdouble(), reason="needs an 80-bit np.longdouble")


# ---- a numpy emulation of the device's algorithms, with the defects of DESIGN.md §2 ---------------------------------
def _tree256(parts, start=128):
    """gpk_blr_gram_kernel's / gpk_blr_eval's reduction over the 256 per-thread partial sums (axis 0)."""
    red = parts.copy()
    o = start
    while o > 0:
        red[:o] = red[:o] + red[o:2 * o]
        o >>= 1
    return red[0]


def _strided(terms, start=128):
    """Sum over rows of terms (N, ...) as 256 strided chains then the tree."""
    N = terms.shape[0]
    pad = (-N) % 256
    T = np.concatenate([terms, np.zeros((pad,) + terms.shape[1:])]) if pad else terms
    T = T.reshape((-1, 256) + terms.shape[1:])
    parts = np.zeros((256,) + terms.shape[1:])
    for r in range(T.shape[0]):
        parts = parts + T[r]
    return _tree256(parts, start)


def emulate_lnpost(Phi, y, theta, par, defect=None):
    """gpk_blr_eval in float64 (the defect: None, "lane", "gram_tree", "resid_tree" or "clamps")."""
    F = Phi.shape[1]
    tree = 64 if defect == "gram_tree" else 128
    G = _strided(Phi[:, :, None] * Phi[:, None, :], tree)
    b = _strided(Phi * y[:, None], tree)
    with np.errstate(all="ignore"):
        alpha, beta = np.exp(theta[0]), np.exp(theta[1])
        A = beta * G + alpha * np.eye(F)
        r = beta * b
        for k in range(F):
            p = A[k, k]
            if not p > 0:
                return -np.inf
            lkk = np.sqrt(p)
            col = A[k + 1:, k] / lkk
            ck = r[k] / lkk
            A[k, k] = lkk
            A[k + 1:, k] = col
            r[k] = ck
            w = F - (k + 1) if defect != "lane" else min(32, F - (k + 1))
            A[k + 1:, k + 1:k + 1 + w] -= np.outer(col, col[:w])
            r[k + 1:k + 1 + w] -= ck * col[:w]
        m = r.copy()
        for k in range(F - 1, -1, -1):
            m[k] = m[k] / A[k, k]
            m[:k] -= A[k, :k] * m[k]
        res = y - Phi @ m
        s = _strided(res * res, 64 if defect == "resid_tree" else 128)
        ld = 2.0 * np.sum(np.log(np.diag(A)))
        if defect == "clamps":
            logdet = -np.inf if ld > R.LOG_DBL_MAX else np.inf if ld < R.LOG_DET_ZERO else ld
        else:
            logdet = np.inf if ld > R.LOG_DBL_MAX else -np.inf if ld < R.LOG_DET_ZERO else ld
        N = Phi.shape[0]
        v = 0.5 * F * np.log(alpha) + 0.5 * N * np.log(beta) - 0.5 * N * R.LOG_2PI - beta / 2 * np.sqrt(s) \
            - alpha / 2 * np.dot(m, m) - 0.5 * logdet
        v = v + BM.prior_lnprob(theta, par)
    return -np.inf if np.isnan(v) else float(v)


def emulate_moments(Phi_t, Ms, Vs, ib, defect=None):
    """gpk_blr_score_kernel's moments in float64 from m_i, L_i^-1 and 1 / beta_i (the defect: None, "ib0" or
    "first16")."""
    k = len(Ms)
    smu = np.zeros(Phi_t.shape[0])
    svar = np.zeros(Phi_t.shape[0])
    for i in range(min(k, 16) if defect == "first16" else k):
        t = Phi_t @ Vs[i].T
        smu = smu + Phi_t @ Ms[i]
        svar = svar + ((ib[0] if defect == "ib0" else ib[i]) + np.sum(t * t, axis=1))
    return smu / k, np.maximum(svar / k, R.EPS)


@pytest.mark.parametrize("basis,D,N,clustered", R.LNPOST_CASES)
def test_restatement_inside_the_lnpost_bound(basis, D, N, clustered):
    X, y, Phi = R.case(basis, D, N, clustered=clustered)
    data = R.Data(Phi, y)
    checked = 0
    for th in R.theta_grid(data):
        ref = R.lnpost_reference(data, th, R.GRID_PAR, depth=R.numpy_depth(N, data.F))
        if ref is None or ref["eta"] > 0.1 or ref["near_threshold"]:
            continue
        v = BM.mll(Phi, y, th, R.GRID_PAR)
        assert R.err_ratio(v, ref["v"], ref["bound"]) <= 1.0, (th, v, float(ref["v"]), ref["bound"])
        checked += 1
    assert checked >= 4


@pytest.mark.parametrize("basis,D,N", [(0, 8, 50), (1, 31, 300), (2, 64, 63), (2, 34, 4097)])
def test_restatement_fit_and_moments_inside_the_bounds(basis, D, N):
    X, y, Phi = R.case(basis, D, N)
    data = R.Data(Phi, y)
    rng = np.random.RandomState(N)
    hypers = np.column_stack([np.exp(rng.uniform(-4, 1, 5)), np.exp(rng.uniform(0, 6, 5))])
    models = BM.fit(Phi, y, hypers)
    Vabs = []
    for (m, S), (a, bt) in zip(models, hypers):
        ref = R.fit_reference(data, a, bt, depth=R.numpy_depth(N, data.F))
        assert ref["eta"] <= 0.1
        assert R.err_ratio(m, ref["m"], ref["bound_m"]) <= 1.0
        assert R.err_ratio(S, ref["S"], ref["bound_S"]) <= 1.0
        Vabs.append(np.abs(ref["V"].astype(np.float64)))
    Xt = rng.uniform(-1.2, 1.2, (300, D))
    Pt = BM.features(Xt, basis)
    mu, var = BM.predict(Pt, hypers, models)
    mref = R.moments_reference(Pt, models, hypers[:, 1], Vabs)
    assert R.err_ratio(mu, mref["mu"], mref["bound_mu"]) <= 1.0
    r, clip_ok = R.var_check(var, mref["var"], mref["bound_var"])
    assert r <= 1.0 and clip_ok


LNPOST_DEFECTS = [("lane", (2, 34, 40)), ("lane", (0, 63, 300)), ("gram_tree", (0, 8, 129)),
                  ("gram_tree", (2, 64, 4097)), ("resid_tree", (1, 16, 129)), ("resid_tree", (2, 49, 257))]


def _defect_ratio(basis, D, N, defect):
    X, y, Phi = R.case(basis, D, N)
    data = R.Data(Phi, y)
    worst, clean = 0.0, 0.0
    for th in R.theta_grid(data, t1s=(-3.0, 4.0), n_cond=4):
        ref = R.lnpost_reference(data, th, R.GRID_PAR)
        if ref is None or ref["eta"] > 0.1 or ref["near_threshold"]:
            continue
        clean = max(clean, R.err_ratio(emulate_lnpost(Phi, y, th, R.GRID_PAR), ref["v"], ref["bound"]))
        worst = max(worst, R.err_ratio(emulate_lnpost(Phi, y, th, R.GRID_PAR, defect), ref["v"], ref["bound"]))
    return clean, worst


@pytest.mark.parametrize("defect,shape", LNPOST_DEFECTS)
def test_lnpost_defects_break_the_bound(defect, shape):
    clean, worst = _defect_ratio(*shape, defect)
    assert clean <= 1.0
    assert worst > 10.0, worst


@pytest.mark.parametrize("defect,shape", [("lane", (2, 33, 40)), ("gram_tree", (2, 64, 128)),
                                          ("resid_tree", (0, 8, 128))])
def test_lnpost_defects_are_invisible_below_their_threshold(defect, shape):
    """F <= 33 for the lane loop and N <= 128 for the trees: the shapes of the older tests cannot see them."""
    clean, worst = _defect_ratio(*shape, defect)
    assert clean <= 1.0 and worst <= 1.0


def test_swapped_clamps_give_the_wrong_infinity():
    X, y, Phi = R.case(2, 64, 300)
    data = R.Data(Phi, y)
    par = (1.0, -60.0, 0.1)
    for target, t1 in ((R.LOG_DBL_MAX + 15, 1.0), (R.LOG_DET_ZERO - 15, -40.0)):
        th = np.array([R.theta_for_logdet(data, target, t1), t1])
        ref = R.lnpost_reference(data, th, par)
        assert not np.isfinite(ref["v"])
        assert emulate_lnpost(Phi, y, th, par) == BM.mll(Phi, y, th, par) == float(ref["v"])
        assert emulate_lnpost(Phi, y, th, par, "clamps") == -float(ref["v"])


@pytest.mark.parametrize("defect,k", [("ib0", 3), ("ib0", 20), ("first16", 20), ("first16", 200)])
def test_moment_defects_break_the_bound(defect, k):
    basis, D, N = 0, 8, 60
    X, y, Phi = R.case(basis, D, N)
    data = R.Data(Phi, y)
    rng = np.random.RandomState(k)
    hypers = np.column_stack([np.exp(rng.uniform(-4, 1, k)), np.exp(rng.uniform(0, 6, k))])
    fits = [R.fit_reference(data, a, bt) for a, bt in hypers]
    models = [(f["m"].astype(np.float64), f["S"].astype(np.float64)) for f in fits]
    Vs = [f["V"].astype(np.float64) for f in fits]
    Pt = BM.features(rng.uniform(-1.2, 1.2, (200, D)), basis)
    mref = R.moments_reference(Pt, models, hypers[:, 1], [np.abs(V) for V in Vs])
    ib = 1.0 / hypers[:, 1]
    for d, expect_bad in ((None, False), (defect, True)):
        mu, var = emulate_moments(Pt, [m for m, _ in models], Vs, ib, d)
        r = max(R.err_ratio(mu, mref["mu"], mref["bound_mu"]), R.var_check(var, mref["var"], mref["bound_var"])[0])
        assert (r > 10.0) if expect_bad else (r <= 1.0), (d, r)
    mu, var = emulate_moments(Pt, [m for m, _ in models], Vs, ib, "first16")
    if k <= 16:
        assert R.var_check(var, mref["var"], mref["bound_var"])[0] <= 1.0
