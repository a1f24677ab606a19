"""The entropy-search candidate path at every shape, transform and branch, against the extended-precision reference of
tests/es_reference.py (U = K^-1 K(X, zb) and sigma in longdouble from the george oracle) and the dH restatement
tests/es_model.dh_folded.

Through gpk_es_get_u and gpk_es_moments (what gpk_es_dh_kernel reads) each stage is held on its own:
  U       per entry, within 4 N eps kappa(K) max|U[:, j]| (es_reference: normwise forward error of the solves);
  sigma   per entry, within [(N + 16) eps (|k(zb_j, x)| + sum_n |k(x, X_n)| |U_nj|) + sum_n |k(x, X_n)| |dU_nj|] y_std^2
          with dU the device's measured U error; entries below the clip by more than that must be exactly eps, entries
          within it of eps may land on either side (es_reference.sigma_check);
  var     against the oracle's fp64 variance at the project's 1e-10 (tests/product_cases.py);
  dH      against dh_folded fed the device's OWN var and sigma, within es_reference.dh_bound (term magnitudes: lane and
          tree order of the dot products, fma contraction, CUDA exp / log within 1 ulp); non-finite values exactly as
          compute_value maps them; plus a spot check of dH end to end against dh_folded on sigma_ref.
Every assertion prints its largest error-to-bound ratio.

The shapes cross the sigma kernel's 256-row tiles and the 128-row padding (N), the warp boundaries of the dH kernel's
lane loops (Nb), its per-thread W loop and reduction tree (Np), the int8 and fp64 variance paths (ozaki, batches on
both sides of 2048), the ES_CH = 16384 passes, gpk_es_multi over unlike handles, and U after gpk_fit_append.
"""
import numpy as np
import pytest

from oracle import robo_oracle as O
from tests import es_model as M
from tests import es_reference as R
from tests import kernel_cases as KC
from tests.product_cases import assert_var_close

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not R.have_longdouble(), reason="np.longdouble is not an extended type here")]

EPS = R.EPS
DMAX = float(np.finfo(float).max)
ES_CH = 16384
SN2 = 1e-3


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


# ---- fixtures: a fitted model, its reference, an update with chosen zb, lmb, W, sn2 --------------------------------
class Case(object):
    def __init__(self, case, variant, N, nb, Np, seed=0, m=240):
        X, y, Xs = KC.data(case, variant, N, m, seed)
        self.case, self.variant, self.X, self.y = case, variant, X, y
        D = X.shape[1]
        self.lo, self.up = KC.box(variant, D)
        rng = np.random.RandomState(7919 * N + 31 * nb + Np + seed)
        self.zb = self.lo + (self.up - self.lo) * rng.rand(nb, D)
        self.lmb = np.log(0.05 + rng.rand(nb))
        W = rng.randn(Np)
        self.W = W
        k = min(N, 6)
        Xs[:k] = X[:k]                                           # training inputs: sigma cancels, may clip
        Xs[k:k + 2] = self.zb[:2]                                # the representer points themselves
        self.Xs = Xs
        self.model = KC.model(case, variant)
        self.model.train(X, y, do_optimize=False)
        self.h = self.model.gp.handle
        self.st = KC.oracle_state(case, variant, X, y)
        self.ref = R.Reference(self.st)
        self.U_ref, self.zs = self.ref.u(self.zb)
        self.update(SN2)

    def update(self, sn2, W=None):
        W = self.W if W is None else W
        r = self.h.es_update(self.zb, self.lmb, sn2, W, self.lo, self.up)
        self.state = dict(logP=r["logP"], lmb=self.lmb, dlogPdMu=r["dlogPdMu"], dlogPdSigma=r["dlogPdSigma"],
                          dlogPdMudMu=r["dlogPdMudMu"], W=np.asarray(W, dtype=np.float64), sn2=sn2,
                          H=R.host_h(r["logP"], self.lmb))
        return self.state

    def kss(self):
        return KC.prior_var(self.case, self.st)

    def close(self):
        self.h.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def _ratio(a, b):
    return float(np.max(a / b)) if a.size else 0.0


def check_u(c):
    U = c.h.es_get_u()
    err = np.abs(U - c.U_ref.astype(np.float64))
    ub = c.ref.u_bound(c.U_ref)
    assert np.all(err <= ub), "U: max error / bound %.3g" % _ratio(err, ub)
    return U, _ratio(err, ub)


def check_sigma(c, U, Xs, sig):
    s, mag, absK = c.ref.sigma(c.U_ref, c.zs, Xs)
    bound = c.ref.sigma_bound(mag, absK, U - c.U_ref.astype(np.float64))
    ratio, bad = R.sigma_check(sig, s, bound)
    assert not bad.any(), "sigma: %d entries outside the bound (first %s)" % (bad.sum(), np.argwhere(bad)[:3].tolist())
    return s, ratio


def check_dh(c, Xs, dh, var, sig, rows=None):
    """dH of the in-box rows against dh_folded on the device's own var / sigma; returns the largest ratio and the bound
    relative to S = |H| + max |lmb| + 1 (the scale of the older 1e-7 S check)."""
    st = c.state
    worst, rel = 0.0, 0.0
    S = abs(st["H"]) + np.max(np.abs(st["lmb"])) + 1.0
    for i in (range(len(Xs)) if rows is None else rows):
        x = Xs[i]
        if np.any(x < c.lo) or np.any(x > c.up):
            assert dh[i] == EPS, (i, dh[i])
            continue
        r = M.dh_folded(st, var[i], sig[i])
        ref = M.compute_value(r, x, c.lo, c.up)
        if not np.isfinite(r) or ref == -DMAX:
            assert dh[i] == ref, (i, dh[i], ref)
            continue
        b, fin = R.dh_bound(st, var[i], sig[i], st["H"])
        assert fin and abs(dh[i] - ref) <= b, (i, dh[i], ref, b)
        worst = max(worst, abs(dh[i] - ref) / b)
        rel = max(rel, b / S)
    return worst, rel


def full_check(c, Xs=None, label=""):
    Xs = c.Xs if Xs is None else Xs
    U, ru = check_u(c)
    var, sig = c.h.es_moments(Xs)
    assert sig.shape == (len(Xs), len(c.zb))
    _, rs = check_sigma(c, U, Xs, sig)
    assert_var_close(var, O.gp_predict_var_only_fast(c.st, Xs)[1], c.kss())
    dh = c.h.es_compute(Xs)
    rd, rel = check_dh(c, Xs, dh, var, sig)
    print("%s: error / bound  U %.3g  sigma %.3g  dH %.3g (dH bound <= %.3g S)" % (label, ru, rs, rd, rel))
    return var, sig, dh


# ---- shapes --------------------------------------------------------------------------------------------------------
N_SHAPES = [1, 2, 127, 128, 129, 255, 256, 257, 511, 513, 1030]


@pytest.mark.parametrize("N", N_SHAPES)
@pytest.mark.parametrize("variant", KC.VARIANTS)
def test_training_sizes(N, variant):
    """N across the 256-row tiles of the sigma kernel and the 128-row padding of L^-1 (m52)."""
    if N == 1 and variant == "scaled":
        pytest.skip("one target has no standard deviation")
    with Case("m52", variant, N, 33, 257, seed=N) as c:
        full_check(c, label="m52-%s N=%d" % (variant, N))


@pytest.mark.parametrize("case", KC.CASES)
@pytest.mark.parametrize("variant", KC.VARIANTS)
def test_kernel_cases(case, variant):
    """Every kernel shape of tests/kernel_cases.py; 'scaled' runs normalize_input and normalize_output (out_scale =
    y_std^2 in the sigma kernel, v - sn2 in the reference's mixed units)."""
    with Case(case, variant, 300, 32, 256) as c:
        full_check(c, label="%s-%s" % (case, variant))


@pytest.mark.parametrize("nb,Np", [(2, 1), (2, 400), (31, 255), (32, 256), (33, 257), (33, 1), (64, 400), (64, 255),
                                   (31, 257), (64, 1)])
def test_representer_and_w_counts(nb, Np):
    """Nb at the warp boundaries of the lane loops (a += 32, i += 8 warps), Np = 1 and around the 256-thread W loop and
    its reduction tree."""
    with Case("m52", "scaled", 257, nb, Np, seed=nb + Np) as c:
        full_check(c, label="nb=%d Np=%d" % (nb, Np))


@pytest.mark.parametrize("ozaki", [0, 1])
@pytest.mark.parametrize("m", [1500, 2600])
def test_variance_paths(ozaki, m):
    """ozaki 0 / 1 with batches on both sides of 2048 (the int8 contraction needs >= 2048 candidates); sigma and dH on a
    sample of 400 rows, var on every row."""
    with Case("m52", "scaled", 513, 33, 256, seed=m, m=m) as c:
        c.h.set_option("ozaki", ozaki)
        var, sig = c.h.es_moments(c.Xs)
        assert_var_close(var, O.gp_predict_var_only_fast(c.st, c.Xs)[1], c.kss())
        rows = np.unique(np.r_[np.arange(10), np.random.RandomState(m).choice(m, 390, replace=False)])
        U, ru = check_u(c)
        _, rs = check_sigma(c, U, c.Xs[rows], sig[rows])
        dh = c.h.es_compute(c.Xs)
        rd, _ = check_dh(c, c.Xs, dh, var, sig, rows=rows)
        print("ozaki=%d m=%d: error / bound  U %.3g  sigma %.3g  dH %.3g" % (ozaki, m, ru, rs, rd))


# ---- forced branches and candidate edges ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def edge_case():
    c = Case("m52", "scaled", 300, 33, 257, seed=3)
    yield c
    c.close()


def test_sn2_above_every_v(edge_case):
    c = edge_case
    var, _ = c.h.es_moments(c.Xs)
    c.update(10.0 * float(np.max(var)))
    try:
        full_check(c, label="sn2 > v")
    finally:
        c.update(SN2)


def test_sn2_equal_to_v(edge_case):
    """v_ = 0 for one candidate: 1 / v_ = inf, and its value is exactly what dh_folded then compute_value give."""
    c = edge_case
    var, sig = c.h.es_moments(c.Xs)
    k = 20
    try:
        st = c.update(float(var[k]))
        dh = c.h.es_compute(c.Xs)
        ref = M.compute_value(M.dh_folded(st, var[k], sig[k]), c.Xs[k], c.lo, c.up)
        assert not np.isfinite(ref) or ref == -DMAX
        assert dh[k] == ref, (dh[k], ref)
        check_dh(c, c.Xs, dh, var, sig)
    finally:
        c.update(SN2)


@pytest.mark.parametrize("wp", [1e308, -1e308])
def test_huge_w_entry(edge_case, wp):
    """One W entry of +-1e308.  Where |g_i| > 1.8 the product overflows and the value is exactly what compute_value
    makes of dh_folded's NaN.  Otherwise that column's lPred is decided by g_i W_p alone, and dH is not determined to
    better than one lmb / Np by its inputs: the rows of dlogPdMu sum to zero, so where dm is nearly constant the g_i are
    rounding noise, and which entry the noise makes the column's maximum picks the column's value H + lmb_imax
    (es_reference.dh_interval_huge_column).  The device must lie in that interval, which is a single value up to the
    other columns' dh_bound wherever only one entry can be the maximum; where several can, the device's choice and
    dh_folded's may differ, and both must lie in it."""
    c = edge_case
    W = c.W.copy()
    W[7] = wp
    try:
        st = c.update(SN2, W)
        var, sig = c.h.es_moments(c.Xs)
        dh = c.h.es_compute(c.Xs)
        n_exact = n_one = n_amb = n_moved = 0
        for i, x in enumerate(c.Xs):
            if np.any(x < c.lo) or np.any(x > c.up):
                assert dh[i] == EPS
                continue
            r = M.dh_folded(st, var[i], sig[i])
            ref = M.compute_value(r, x, c.lo, c.up)
            if not np.isfinite(r) or ref == -DMAX:
                assert dh[i] == ref, (i, dh[i], ref)
                n_exact += 1
                continue
            iv = R.dh_interval_huge_column(st, var[i], sig[i], 7, st["H"])
            assert iv is not None, (i, var[i], sig[i].min(), sig[i].max())
            lo, hi, nA = iv
            assert lo <= dh[i] <= hi and lo <= ref <= hi, (i, dh[i], ref, iv)
            n_one += nA == 1
            n_amb += nA > 1
            n_moved += dh[i] != ref and nA > 1
        print("W_p = %g: %d non-finite (exact), %d decided, %d with an ambiguous maximum (%d where the device's choice "
              "differs from dh_folded's)" % (wp, n_exact, n_one, n_amb, n_moved))
        assert n_one > 0
    finally:
        c.update(SN2)


def test_candidate_edges(edge_case):
    """Outside the box: exactly DBL_EPSILON; on the lower and upper bounds: inside; at training inputs and at zb: the
    checked value; a NaN row: -DBL_MAX, and adding it changes no other value."""
    c = edge_case
    D = c.X.shape[1]
    rng = np.random.RandomState(5)
    C = c.lo + (c.up - c.lo) * rng.rand(40, D)
    C[0] = c.lo
    C[1] = c.up
    C[2, 0] = c.lo[0]
    C[3, 1] = c.up[1]
    C[4] = c.X[0]
    C[5] = c.zb[0]
    out = [c.lo - 1e-9 * (c.up - c.lo), c.up + np.spacing(c.up), np.r_[c.up[0] + 1.0, c.lo[1:]]]
    Cx = np.vstack([C, out])
    dh = c.h.es_compute(Cx)
    assert np.all(dh[len(C):] == EPS)
    assert np.all(dh[:4] != EPS)
    var, sig = c.h.es_moments(C)
    U = c.h.es_get_u()
    check_sigma(c, U, C, sig)
    check_dh(c, C, dh[:len(C)], var, sig)
    Cn = np.vstack([C[:17], np.full((1, D), np.nan), C[17:]])
    dn = c.h.es_compute(Cn)
    assert dn[17] == -DMAX
    assert np.array_equal(np.r_[dn[:17], dn[18:]], dh[:len(C)])


# ---- chunks and composition ----------------------------------------------------------------------------------------
def test_passes_over_es_ch():
    """m = 2 ES_CH + 37 with chunk = 2048 and the automatic chunk: equal to per-pass es_compute calls bit for bit; the
    rows at the pass boundaries and a sample against the reference."""
    m = 2 * ES_CH + 37
    with Case("m52", "scaled", 300, 33, 256, seed=11, m=m) as c:
        whole = c.h.es_compute(c.Xs)
        var, sig = c.h.es_moments(c.Xs)
        parts = np.concatenate([c.h.es_compute(c.Xs[a:a + ES_CH]) for a in range(0, m, ES_CH)])
        assert np.array_equal(whole, parts)
        vp = np.concatenate([c.h.es_moments(c.Xs[a:a + ES_CH])[0] for a in range(0, m, ES_CH)])
        assert np.array_equal(var, vp)
        c.h.set_option("chunk", 2048)
        assert np.array_equal(c.h.es_compute(c.Xs), whole)
        v2, s2 = c.h.es_moments(c.Xs)
        assert np.array_equal(v2, var) and np.array_equal(s2, sig)
        c.h.set_option("chunk", 0)
        rows = np.unique(np.r_[ES_CH - 1, ES_CH, 2 * ES_CH - 1, 2 * ES_CH, m - 1,
                               np.random.RandomState(2).choice(m, 507, replace=False)])
        U, ru = check_u(c)
        _, rs = check_sigma(c, U, c.Xs[rows], sig[rows])
        assert_var_close(var, O.gp_predict_var_only_fast(c.st, c.Xs)[1], c.kss())
        rd, _ = check_dh(c, c.Xs, whole, var, sig, rows=rows)
        print("m=%d: error / bound  U %.3g  sigma %.3g  dH %.3g" % (m, ru, rs, rd))


def test_es_multi_over_unlike_handles():
    """gpk_es_multi / gpk_es_multi_dev over handles with different N, Nb and Np: each handle's value is its own
    es_compute, the mean is MarginalizationGPMCMC's host reduction of those, bit for bit."""
    import torch
    from robo_b200 import _lib
    cases = [Case("m52", "scaled", 100, 8, 1, seed=1), Case("m52", "scaled", 257, 33, 256, seed=2),
             Case("m52", "scaled", 300, 64, 400, seed=3)]
    Xs = cases[0].Xs
    per = np.array([c.h.es_compute(Xs) for c in cases])
    handles = [c.h for c in cases]
    r = _lib.es_multi(handles, Xs)
    ref = _lib.moments_handle().reduce_models(per)
    assert np.array_equal(r["values"], ref)
    dX = torch.from_numpy(np.ascontiguousarray(Xs)).cuda()
    dout = torch.empty(len(Xs), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    _lib.es_multi_dev(handles, dX.data_ptr(), len(Xs), dout.data_ptr())
    handles[0].synchronize()
    assert np.array_equal(dout.cpu().numpy(), ref)
    for c, p in zip(cases, per):
        assert np.array_equal(c.h.es_compute(Xs), p)
        var, sig = c.h.es_moments(Xs)
        check_dh(c, Xs, p, var, sig)
        c.close()


def test_after_fit_append():
    """fit_append (260 -> 300 rows, inside the last 128-row block) patches L^-1; es_update then builds U from it: U and
    sigma against the reference of the appended training set."""
    X, y, Xs = KC.data("m52", "scaled", 300, 200, seed=4)
    model = KC.model("m52", "scaled")
    model.train(X[:260], y[:260], do_optimize=False)
    model.predict(Xs[:10])
    model.train(X, y, do_optimize=False)
    assert model.gp.n_appends == 1
    c = Case.__new__(Case)
    c.case, c.variant, c.X, c.y, c.Xs = "m52", "scaled", X, y, Xs
    c.lo, c.up = KC.box("scaled", X.shape[1])
    rng = np.random.RandomState(8)
    c.zb = c.lo + (c.up - c.lo) * rng.rand(33, X.shape[1])
    c.lmb = np.log(0.05 + rng.rand(33))
    c.W = rng.randn(256)
    c.model, c.h = model, model.gp.handle
    c.st = KC.oracle_state("m52", "scaled", X, y)
    c.ref = R.Reference(c.st)
    c.U_ref, c.zs = c.ref.u(c.zb)
    try:
        c.update(SN2)
        full_check(c, label="after fit_append")
    finally:
        c.close()


def test_end_to_end_against_reference_sigma(edge_case):
    """dH from the device against dh_folded on the device's var and the REFERENCE sigma (clipped), away from the
    cancellation regions: no sigma entry within its bound of the clip, v >= 2 sn2.  The bound is dh_bound plus the sigma
    bound carried through dH, 2 sum_j |d dH / d sigma_j| b_j (central differences of dh_folded)."""
    c = edge_case
    U = c.h.es_get_u()
    var, sig = c.h.es_moments(c.Xs)
    s, mag, absK = c.ref.sigma(c.U_ref, c.zs, c.Xs)
    bsig = c.ref.sigma_bound(mag, absK, U - c.U_ref.astype(np.float64))
    s = s.astype(np.float64)
    dh = c.h.es_compute(c.Xs)
    st = c.state
    S = abs(st["H"]) + np.max(np.abs(st["lmb"])) + 1.0
    n, worst, rel = 0, 0.0, 0.0
    for i in range(len(c.Xs)):
        if np.any(np.abs(s[i] - EPS) <= bsig[i]) or var[i] < 2 * st["sn2"]:
            continue
        sr = np.maximum(s[i], EPS)
        ref = M.dh_folded(st, var[i], sr)
        carried = 0.0
        for j in np.nonzero(s[i] > EPS)[0]:
            step = max(1e-6 * sr[j], bsig[i, j])
            up, dn = sr.copy(), sr.copy()
            up[j] += step
            dn[j] -= step
            carried += abs(M.dh_folded(st, var[i], up) - M.dh_folded(st, var[i], dn)) / (2 * step) * bsig[i, j]
        b = R.dh_bound(st, var[i], sr, st["H"])[0] + 2 * carried
        assert abs(dh[i] - ref) <= b, (i, dh[i], ref, b)
        worst = max(worst, abs(dh[i] - ref) / b)
        rel = max(rel, b / S)
        n += 1
    print("end to end: %d candidates, error / bound %.3g, bound <= %.3g S" % (n, worst, rel))
    assert n >= 20


def test_diagnostics_refuse_without_current_update():
    from robo_b200 import _lib
    X, y, Xs = KC.data("m52", "raw", 50, 5)
    model = KC.model("m52", "raw")
    model.train(X, y, do_optimize=False)
    h = model.gp.handle
    fresh = _lib.Handle()
    try:
        _refusals(model, h, fresh, X, y, Xs)
    finally:
        h.close()
        fresh.close()


def _refusals(model, h, fresh, X, y, Xs):
    with pytest.raises(ValueError, match="gpk_es_update first"):
        h.es_moments(Xs)
    with pytest.raises(ValueError, match="gpk_es_update first"):
        h.es_get_u()
    zb = np.random.RandomState(0).rand(4, X.shape[1])
    h.es_update(zb, np.zeros(4), SN2, np.linspace(-1, 1, 5), np.zeros(3), np.ones(3))
    assert h.es_dims() == (50, 4)
    assert h.es_get_u().shape == (50, 4)
    var, sig = h.es_moments(Xs)
    assert sig.shape == (5, 4) and np.all(sig >= EPS)
    model.train(X[:40], y[:40], do_optimize=False)                 # the model changed: U is stale
    with pytest.raises(ValueError, match="model changed"):
        h.es_moments(Xs)
    with pytest.raises(ValueError, match="model changed"):
        h.es_get_u()
    with pytest.raises(ValueError):
        h.es_moments(np.zeros((0, X.shape[1])))
    with pytest.raises((ValueError, RuntimeError)):
        fresh.es_moments(Xs)
