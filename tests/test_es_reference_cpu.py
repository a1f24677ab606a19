"""The extended-precision reference of the entropy-search candidate path (tests/es_reference.py) and its tolerances.

1. The reference against 50-digit mpmath on a tiny problem, and against robo_oracle.gp_predict_variance (the
   reference's own full-covariance formula) at fp64 rounding.
2. The bounds the GPU tests hold the device to, with injected defects: an fp64 emulation of gpk_es_sigma_kernel /
   gpk_es_dh_kernel in the kernels' order sits well inside the bound, and each defect falls outside it.  Each defect is
   also put through the older check of tests/test_gpu_es.py (dH at 1e-7 S with sigma from predict_variance) to show
   what that check could not see (DESIGN.md section 2 has the table these tests print).
"""
import math

import numpy as np
import pytest

from oracle import george_oracle as G
from oracle import robo_oracle as O
from tests import es_model as M
from tests import es_reference as R
from tests import kernel_cases as KC

pytestmark = pytest.mark.skipif(not R.have_longdouble(), reason="np.longdouble is not an extended type here")

EPS = R.EPS


def _problem(case, variant, N, nb, m, seed=0):
    X, y, Xs = KC.data(case, variant, N, m, seed)
    D = X.shape[1]
    lo, up = KC.box(variant, D)
    rng = np.random.RandomState(seed + 7)
    zb = lo + (up - lo) * rng.rand(nb, D)
    Xs[:5] = X[:5]                                   # training inputs: sigma cancels to rounding, clip either side
    Xs[5:8] = lo + (up - lo) * (0.5 + 0.5 * rng.rand(3, D))
    st = KC.oracle_state(case, variant, X, y)
    return st, X, zb, Xs


# ---- 1. the reference itself ---------------------------------------------------------------------------------------
def _mp_kernel(k, a, b, mp):
    if isinstance(k, G.Product):
        return _mp_kernel(k.k1, a, b, mp) * _mp_kernel(k.k2, a, b, mp)
    if isinstance(k, G.ConstantKernel):
        return mp.exp(mp.mpf(k.log_constant))
    r2 = mp.mpf(0)
    for ax, md in zip(k.axes, k._axis_metric()):
        d = mp.mpf(float(a[ax])) - mp.mpf(float(b[ax]))
        r2 += d * d / mp.mpf(float(md))
    if isinstance(k, G.Matern52Kernel):
        r = mp.sqrt(5 * r2)
        return (1 + r + 5 * r2 / 3) * mp.exp(-r)
    if isinstance(k, G.Matern32Kernel):
        r = mp.sqrt(3 * r2)
        return (1 + r) * mp.exp(-r)
    return mp.exp(-r2 / 2)


@pytest.mark.parametrize("case,variant", [("m52", "scaled"), ("rbf", "raw"), ("m52_axis0", "scaled")])
def test_reference_matches_mpmath(case, variant):
    mpmath = pytest.importorskip("mpmath")
    mp = mpmath.mp
    mp.dps = 50
    st, X, zb, Xs = _problem(case, variant, 12, 3, 10)
    ref = R.Reference(st)
    U, zs = ref.u(zb)
    s, mag, _ = ref.sigma(U, zs, Xs)
    Xn, xs = ref.X, R.scale_inputs(st, Xs)
    diag = mp.mpf(float(np.sqrt(st["gp"]._yerr2[0] + np.exp(st["gp"].white_noise)) ** 2))
    K = mp.matrix(12, 12)
    for i in range(12):
        for j in range(12):
            K[i, j] = _mp_kernel(ref.kernel, Xn[i], Xn[j], mp) + (diag if i == j else 0)
    eld = float(np.finfo(np.longdouble).eps)
    for j in range(3):
        kz = mp.matrix([_mp_kernel(ref.kernel, Xn[i], zs[j], mp) for i in range(12)])
        u = mp.lu_solve(K, kz)
        um = np.array([float(u[i]) for i in range(12)])
        tol_u = 64 * ref.kappa * eld * np.max(np.abs(um))
        assert np.max(np.abs(U[:, j].astype(np.float64) - um)) <= tol_u
        for c in range(len(Xs)):
            sm = (_mp_kernel(ref.kernel, xs[c], zs[j], mp)
                  - mp.fsum(_mp_kernel(ref.kernel, xs[c], Xn[i], mp) * u[i] for i in range(12))) * R.out_scale(st)
            err = abs(float(mp.mpf(np.format_float_scientific(s[c, j], unique=True)) - sm))     # round-trip digits
            assert err <= 64 * ref.kappa * eld * float(mag[c, j]), (j, c, err, float(mag[c, j]))


@pytest.mark.parametrize("case,variant", [("m52", "scaled"), ("m32", "raw"), ("prod1d", "scaled")])
def test_reference_matches_oracle_predict_variance(case, variant):
    """robo_oracle.gp_predict_variance (the full-covariance path, clipped, in output units) is an fp64 evaluation of
    the same quantity: within N eps kappa(K) of the term magnitudes, and on the same side of the clip."""
    st, X, zb, Xs = _problem(case, variant, 60, 5, 40)
    ref = R.Reference(st)
    U, zs = ref.u(zb)
    s, mag, _ = ref.sigma(U, zs, Xs)
    bound = len(X) * EPS * ref.kappa * mag.astype(np.float64)
    for c, x in enumerate(Xs):
        got = O.gp_predict_variance(st, zb, x[None]).ravel()
        ratio, bad = R.sigma_check(got, s[c], bound[c])
        assert not bad.any(), (c, got[bad], s[c][bad].astype(np.float64))


# ---- 2. the sigma bound against an emulation and injected defects -------------------------------------------------
def _old_check(st, zb, Xs, X, lo, up, sig_a, sig_b, v, nb, seed=0, dh_a=None, dh_b=None):
    """tests/test_gpu_es.py::test_compute_matches_model_on_device_moments's criterion: dH from sigma_a against dH from
    sigma_b at 1e-7 S on the candidates away from v = sn2 and from the training inputs.  True when it fails."""
    state = _ep_state(st, zb, nb, seed)
    S = abs(np.sum(np.exp(state["logP"]) * (state["logP"] + state["lmb"]))) + np.max(np.abs(state["lmb"])) + 1.0
    for i, x in enumerate(Xs):
        near = np.min(np.max(np.abs(X - x) / (up - lo), axis=1)) < 1e-2
        if near or abs(v[i] - state["sn2"]) < 1e-3 * v[i]:
            continue
        a = dh_a[i] if dh_a is not None else M.compute_value(M.dh_folded(state, v[i], sig_a[i]), x, lo, up)
        b = dh_b[i] if dh_b is not None else M.compute_value(M.dh_folded(state, v[i], sig_b[i]), x, lo, up)
        if np.isfinite(b) and abs(a - b) > 1e-7 * S:
            return True
    return False


_STATES = {}


def _ep_state(st, zb, nb, seed=0, Np=400):
    key = (id(st), nb, seed, Np)
    if key not in _STATES:
        mu, cov = O.gp_predict(st, zb, full_cov=True)
        ep = M.joint_min(mu, cov)
        rng = np.random.RandomState(seed)
        from scipy.stats import norm
        W = norm.ppf(np.linspace(1.0 / (Np + 1), 1.0 - 1.0 / (Np + 1), Np))
        rng.shuffle(W)
        lmb = np.log(0.05 + rng.rand(nb))
        _STATES[key] = dict(logP=ep["logP"], lmb=lmb, dlogPdMu=ep["dlogPdMu"], dlogPdSigma=ep["dlogPdSigma"],
                            dlogPdMudMu=ep["dlogPdMudMu"], W=W, sn2=st["noise"], H=R.host_h(ep["logP"], lmb))
    return _STATES[key]


@pytest.fixture(scope="module")
def sigma_problem():
    """N = 513 (three 256-row tiles), Nb = 33, scaled variant (y_std ~ 40): the emulated U and sigma."""
    st, X, zb, Xs = _problem("m52", "scaled", 513, 33, 120, seed=5)
    ref = R.Reference(st)
    U, zs = ref.u(zb)
    s, mag, absK = ref.sigma(U, zs, Xs)
    xs = R.scale_inputs(st, Xs)
    Kxs = R.kernel_ld(ref.kernel, xs, ref.X).astype(np.float64)
    kzx = R.kernel_ld(ref.kernel, xs, zs).astype(np.float64)
    Ue = R.device_u(ref.L64, R.kernel_ld(ref.kernel, ref.X, zs).astype(np.float64))
    dU = Ue - U.astype(np.float64)
    return dict(st=st, X=X, zb=zb, Xs=Xs, ref=ref, U=U, s=s, mag=mag, absK=absK, Kxs=Kxs, kzx=kzx, Ue=Ue, dU=dU,
                bound=ref.sigma_bound(mag, absK, dU), v=O.gp_predict_var_only(st, Xs)[1])


def test_emulated_u_inside_bound(sigma_problem):
    p = sigma_problem
    ub = p["ref"].u_bound(p["U"])
    ratio = np.max(np.abs(p["dU"]) / ub)
    print("U: emulation error / bound = %.3g (kappa %.3g)" % (ratio, p["ref"].kappa))
    assert ratio < 0.1


@pytest.mark.parametrize("defect", [None, "drop_tile_last", "u_row_off", "scale_ystd", "clip_first"])
def test_sigma_bound_separates_defects(sigma_problem, defect):
    p = sigma_problem
    ys2 = R.out_scale(p["st"])
    assert ys2 > 100.0
    got = R.sigma_emulate(p["Kxs"], p["kzx"], p["Ue"], ys2, defect)
    ratio, bad = R.sigma_check(got, p["s"], p["bound"])
    good = R.sigma_emulate(p["Kxs"], p["kzx"], p["Ue"], ys2)
    lo, up = KC.box("scaled", p["X"].shape[1])
    old = _old_check(p["st"], p["zb"], p["Xs"], p["X"], lo, up, got, good, p["v"], 33, seed=1) if defect else False
    print("sigma defect %s: max error / bound %.3g, entries outside %d, caught by the 1e-7 S dH check: %s"
          % (defect, ratio, int(bad.sum()), old))
    if defect is None:
        assert not bad.any() and ratio < 0.1
    else:
        assert bad.any()


# ---- 3. the dH bound against an emulation and injected defects ----------------------------------------------------
@pytest.fixture(scope="module")
def dh_problem(sigma_problem):
    p = sigma_problem
    state = _ep_state(p["st"], p["zb"], 33, seed=1)
    lo, up = KC.box("scaled", p["X"].shape[1])
    sig = R.sigma_emulate(p["Kxs"], p["kzx"], p["Ue"], R.out_scale(p["st"]))
    keep = [i for i in range(len(p["Xs"])) if np.all(p["Xs"][i] >= lo) and np.all(p["Xs"][i] <= up)
            and p["v"][i] > 2 * state["sn2"]][:24]
    return dict(state=state, sig=sig[keep], v=p["v"][keep], Xs=p["Xs"][keep], X=p["X"], st=p["st"], zb=p["zb"],
                lo=lo, up=up)


@pytest.mark.parametrize("defect", [None, "hs_diag_twice", "skip_w_256"])
def test_dh_bound_separates_defects(dh_problem, defect):
    q = dh_problem
    st_ = q["state"]
    worst, outside, dev, ref = 0.0, 0, [], []
    for v, s in zip(q["v"], q["sig"]):
        r = M.dh_folded(st_, v, s)
        b, fin = R.dh_bound(st_, v, s, st_["H"])
        assert fin
        e = R.dh_emulate(st_, v, s, defect=defect)
        worst = max(worst, abs(e - r) / b)
        outside += abs(e - r) > b
        dev.append(e)
        ref.append(r)
    S = abs(np.sum(np.exp(st_["logP"]) * (st_["logP"] + st_["lmb"]))) + np.max(np.abs(st_["lmb"])) + 1.0
    old = bool(np.any(np.abs(np.array(dev) - np.array(ref)) > 1e-7 * S))
    print("dH defect %s: max error / bound %.3g over %d candidates, outside %d, caught at 1e-7 S: %s"
          % (defect, worst, len(dev), outside, old))
    if defect is None:
        assert outside == 0 and worst < 0.1
    else:
        assert outside > 0


def test_dh_max_fallback_is_unreachable(dh_problem):
    """The all-columns max fall-back (information_gain.py:193-195) needs an infinite log-sum-exp, mx + log(sum exp(l -
    mx)).  With mx finite the sum lies in [1, Nb] and mx + log(Nb) cannot overflow; with mx = +-inf the largest entry
    gives inf - inf = NaN, so the log-sum-exp is NaN, not infinite.  So the branch is never taken in IEEE arithmetic and
    deciding it per column is indistinguishable: this pins that on the extreme inputs (a huge W entry, v == sn2, a
    huge sigma)."""
    q = dh_problem
    st_ = dict(q["state"])
    W = st_["W"].copy()
    W[3] = 1e308
    W[300] = -1e308
    for state in (st_, dict(st_, W=W)):
        for v, s in [(q["v"][0], q["sig"][0]), (state["sn2"], q["sig"][0]), (q["v"][1], q["sig"][1] * 1e150)]:
            a = R.dh_emulate(state, v, s)
            b = R.dh_emulate(state, v, s, defect="max_per_column")
            assert a == b or (math.isnan(a) and math.isnan(b))
            with np.errstate(all="ignore"):
                iv = np.float64(1.0) / np.float64(v - state["sn2"])
                dm = (s * iv) * math.sqrt(v + 1e-10)
                nb = s.size
                ia, ib = np.tril_indices(nb)
                base = state["logP"] + (state["dlogPdSigma"].dot(-((s[ia] * iv) * s[ib]))
                                        + 0.5 * M.fold(state["dlogPdMudMu"]).dot(dm[ia] * dm[ib]))
                L = base[:, None] + state["dlogPdMu"].dot(dm)[:, None] * state["W"][None, :]
                mx = np.max(L, axis=0)
                lse = mx + np.log(np.sum(np.exp(L - mx), axis=0))
            assert not np.any(np.isinf(lse))


def test_dlogpdmu_rows_sum_to_zero(dh_problem):
    """p_min does not change when every mean moves by the same amount, so each row of dlogPdMu sums to zero: g_i =
    dlogPdMu_i . dm is rounding noise wherever dm is (nearly) constant over the representer points."""
    D = dh_problem["state"]["dlogPdMu"]
    assert np.max(np.abs(D.sum(axis=1)) / np.abs(D).sum(axis=1)) < 1e-10


def test_huge_w_column_interval(dh_problem):
    """W_p = +-1e308: dh_folded and the kernel emulation both lie in es_reference.dh_interval_huge_column, which is one
    value (up to the other columns' bound) where a single entry can be the column's maximum."""
    q = dh_problem
    n_amb = n_one = 0
    for wp in (1e308, -1e308):
        W = q["state"]["W"].copy()
        W[7] = wp
        st_ = dict(q["state"], W=W)
        for v, s in zip(q["v"], q["sig"]):
            iv = R.dh_interval_huge_column(st_, v, s, 7, st_["H"])
            a = M.dh_folded(st_, v, s)
            if not np.isfinite(a):
                continue
            assert iv is not None
            lo, hi, nA = iv
            b = R.dh_emulate(st_, v, s)
            assert lo <= a <= hi and lo <= b <= hi, (a, b, iv)
            n_amb += nA > 1
            n_one += nA == 1
    print("huge W column: %d candidates decided, %d with an ambiguous maximum" % (n_one, n_amb))
    assert n_one > 0
