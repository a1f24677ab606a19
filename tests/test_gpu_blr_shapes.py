"""BayesianLinearRegression on the device (robo_b200/csrc/gpk_blr.cuh) against the extended-precision reference
tests/blr_reference.py at every feature-count threshold of the kernels (F in {1, 8, 9, 33, 34, 48, 49, 52, 53, 63, 64}
through the three bases), training sizes N in {1, 2, F - 1, 128, 129, 256, 257, 4097, 100000}, k in {1, 20, 200}
hyper-samples and batches M in {1, 127, 128, 129, 65536, 65537} (also chunked at 128 and 4096): the log-posterior on a
conditioning grid and across the det A overflow / underflow clamps, the weight posteriors, the moments and acquisitions,
the arg-max on planted ties, the GPK_NOT_PD refusal, handles of different F interleaved, and the model class end to
end.  Each check is a worst-case bound stated in tests/blr_reference.py; err / bound is in every failure message."""
import numpy as np
import pytest

from robo_b200 import _lib
from robo_b200.models.bayesian_linear_regression import BayesianLinearRegression, quadratic_basis_func
from tests import blr_model as BM
from tests import blr_reference as R
from tests.fit_reference import have_longdouble
from tests.test_gpu_bnn import _acq_interval

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_longdouble(), reason="needs an 80-bit np.longdouble")]

KINDS = (_lib.ACQ_EI, _lib.ACQ_LOG_EI, _lib.ACQ_PI, _lib.ACQ_LCB)


def _handle(X, y, basis, par=BM.PRIOR_PAR, chunk=0):
    h = _lib.Handle(0)
    if chunk:
        h.set_option("chunk", chunk)
    _lib.blr_set_data(h, X, y, basis, par)
    return h


def _lnpost_ratios(data, got, thetas, par):
    """(worst err / bound over the checked rows, rows checked); infinite references exactly."""
    worst, checked = 0.0, 0
    for g, th in zip(got, thetas):
        ref = R.lnpost_reference(data, th, par)
        if ref is None:
            assert g == BM.mll(data.Phi, data.y, th, par), th          # the float64 semantics: -inf
            continue
        if ref["eta"] > 0.1 or ref["near_threshold"]:
            continue
        worst = max(worst, R.err_ratio(g, ref["v"], ref["bound"]))
        checked += 1
    return worst, checked


@pytest.mark.parametrize("basis,D,N,clustered", R.LNPOST_CASES)
def test_lnpost_against_the_reference(basis, D, N, clustered):
    X, y, Phi = R.case(basis, D, N, clustered=clustered)
    data = R.Data(Phi, y)
    h = _handle(X, y, basis, R.GRID_PAR)
    T = R.theta_grid(data)
    got = _lib.blr_lnpost(h, T)
    worst, checked = _lnpost_ratios(data, got, T, R.GRID_PAR)
    assert worst <= 1.0, "lnpost err/bound = %.3g" % worst
    assert checked >= 4
    for i in (0, len(T) // 2, len(T) - 1):                             # alone and in a batch: the same bits
        assert np.array_equal(_lib.blr_lnpost(h, T[i:i + 1]).view(np.int64), got[i:i + 1].view(np.int64))


@pytest.mark.parametrize("basis,D", [(_lib.BLR_LINEAR, 63), (_lib.BLR_QUADRATIC, 31), (_lib.BLR_NONE, 64)])
def test_lnpost_overflow_and_underflow_branches(basis, D):
    """log det A 15 beyond each clamp gives exactly -inf (det overflows) / +inf (det underflows to 0), as numpy's det
    does; 15 inside it a finite value within the bound.  The underflow side needs the lognormal loc below theta_0."""
    X, y, Phi = R.case(basis, D, 300)
    data = R.Data(Phi, y)
    par = (1.0, -60.0, 0.1)
    h = _handle(X, y, basis, par)
    rows, expect = [], []
    for thr, t1, outside in ((R.LOG_DBL_MAX, 1.0, -np.inf), (R.LOG_DET_ZERO, -40.0, np.inf)):
        for side in (-15.0, 15.0):
            rows.append((R.theta_for_logdet(data, thr + side, t1), t1))
            beyond = (side > 0) == (outside == -np.inf)
            expect.append(outside if beyond else None)
    T = np.array(rows)
    got = _lib.blr_lnpost(h, T)
    for g, th, e in zip(got, T, expect):
        ref = R.lnpost_reference(data, th, par)
        assert ref is not None and not ref["near_threshold"]
        if e is not None:
            assert g == e == float(ref["v"]) == BM.mll(Phi, y, th, par), (th, g, e)
        else:
            assert np.isfinite(g) and ref["eta"] <= 0.1
            assert R.err_ratio(g, ref["v"], ref["bound"]) <= 1.0, (th, g, float(ref["v"]), ref["bound"])


def test_lnpost_nonfinite_theta():
    """NaN and infinite entries: -inf (NaN -> -inf, a failed pivot -> -inf), as tests/blr_model.py's float64
    restatement of the reference gives."""
    for basis, D, N in ((_lib.BLR_LINEAR, 8, 129), (_lib.BLR_NONE, 1, 1), (_lib.BLR_QUADRATIC, 31, 257)):
        X, y, Phi = R.case(basis, D, N)
        h = _handle(X, y, basis)
        vals = (np.nan, np.inf, -np.inf, 1.0, -9.0)
        T = np.array([(a, b) for a in vals for b in vals if not (np.isfinite(a) and np.isfinite(b))])
        got = _lib.blr_lnpost(h, T)
        ref = np.array([BM.mll(Phi, y, t) for t in T])
        assert np.array_equal(got, ref), (T[got != ref], got[got != ref], ref[got != ref])
        assert np.all(got == -np.inf)


def _fit_checks(data, h, hypers):
    """m_i and S_i of gpk_blr_get_models within their bounds (where the first-order bound applies), S_i symmetric to
    the bit; returns the models and |L_i^-1| of the reference."""
    models = _lib.blr_models(h)
    assert len(models) == len(hypers)
    Vabs, worst_m, worst_s = [], 0.0, 0.0
    for (m, S), (a, bt) in zip(models, hypers):
        assert np.array_equal(S.view(np.int64), S.T.view(np.int64))
        ref = R.fit_reference(data, a, bt)
        Vabs.append(np.abs(ref["V"].astype(np.float64)))
        if ref["eta"] <= 0.1:
            worst_m = max(worst_m, R.err_ratio(m, ref["m"], ref["bound_m"]))
            worst_s = max(worst_s, R.err_ratio(S, ref["S"], ref["bound_S"]))
    assert worst_m <= 1.0 and worst_s <= 1.0, "m err/bound = %.3g, S err/bound = %.3g" % (worst_m, worst_s)
    return models, Vabs


def _rows(M, k, chunk):
    """The candidate rows the moments are checked on: every row of a small batch, else the edges of the batch, of the
    128-row blocks and chunks, and a random sample; fewer with many hyper-samples (the longdouble sums)."""
    cap = max(256, 40000 // k)
    if M <= cap:
        return np.arange(M)
    pick = [np.arange(0, 130), np.arange(M - 130, M)]
    for c in (chunk, 65536):
        if c and c < M:
            pick.append(np.arange(c - 2, min(c + 2, M)))
    pick.append(np.random.RandomState(M).choice(M, max(cap - 270, 0), replace=False))
    return np.unique(np.concatenate(pick))


def _moment_ratios(mu, var, mref):
    rm = R.err_ratio(mu, mref["mu"], mref["bound_mu"])
    rv, clip_ok = R.var_check(var, mref["var"], mref["bound_var"])
    assert clip_ok
    return rm, rv


# (basis, D, N, k, M, chunk): every F threshold of the fit and scoring kernels, k in {1, 20, 200}, every batch edge
SCORE_CASES = [
    (_lib.BLR_NONE, 1, 1, 1, 129, 0),
    (_lib.BLR_LINEAR, 8, 256, 20, 1000, 128),
    (_lib.BLR_QUADRATIC, 16, 2, 200, 4099, 128),
    (_lib.BLR_LINEAR, 33, 129, 20, 127, 0),
    (_lib.BLR_NONE, 48, 4097, 3, 1, 0),
    (_lib.BLR_LINEAR, 48, 128, 20, 65536, 0),
    (_lib.BLR_QUADRATIC, 26, 257, 1, 128, 0),
    (_lib.BLR_NONE, 52, 4097, 20, 65537, 4096),
    (_lib.BLR_LINEAR, 62, 300, 200, 128, 0),
    (_lib.BLR_NONE, 64, 63, 20, 129, 0),
]


@pytest.mark.parametrize("basis,D,N,k,M,chunk", SCORE_CASES)
def test_fit_and_scoring_against_the_reference(basis, D, N, k, M, chunk):
    X, y, Phi = R.case(basis, D, N)
    data = R.Data(Phi, y)
    rng = np.random.RandomState(k + M)
    hypers = np.column_stack([np.exp(rng.uniform(-4, 1, k)), np.exp(rng.uniform(0, 6, k))])
    h = _handle(X, y, basis, chunk=chunk)
    _lib.blr_fit(h, hypers)
    models, Vabs = _fit_checks(data, h, hypers)
    Xt = rng.uniform(-1.2, 1.2, (M, D))
    rows = _rows(M, k, chunk)
    Pt = BM.features(Xt[rows], basis)
    mref = R.moments_reference(Pt, models, hypers[:, 1], Vabs)
    mu, var = h.predict(Xt)
    rm, rv = _moment_ratios(mu[rows], var[rows], mref)
    assert rm <= 1.0 and rv <= 1.0, "mu err/bound = %.3g, var err/bound = %.3g" % (rm, rv)
    multi = _lib.acq_multi([h], Xt, 1)
    assert np.array_equal(multi["mean"], mu) and np.array_equal(multi["var"], var)
    m64, v64 = mref["mu"].astype(np.float64), mref["var"].astype(np.float64)
    bm, bv = mref["bound_mu"], mref["bound_var"]
    eta = float(np.min(y))
    for kind in KINDS:
        e = 0.0 if kind == _lib.ACQ_LCB else eta
        r = h.acq(Xt, kind, e, 0.01)
        vals = r["values"]
        if kind in (_lib.ACQ_PI, _lib.ACQ_LCB):
            lo, hi = _acq_interval(m64, v64, bm, bv, kind, e, 0.01)
            tol = 1e-12 * np.maximum(np.abs(lo), np.abs(hi)) + 1e-300
            ok = (vals[rows] >= lo - tol) & (vals[rows] <= hi + tol)
            assert np.all(ok | ~np.isfinite(lo)), kind
        # EI and LogEI: the scoring epilogue on the moments just held to their bounds
        ref, _ = _lib.moments_handle().acq_moments(mu, var, kind, e, 0.01)
        fin = np.isfinite(ref)
        assert np.array_equal(np.isfinite(vals), fin)
        np.testing.assert_allclose(vals[fin], ref[fin], rtol=1e-12, atol=0)
        assert r["best_idx"] == int(np.argmax(vals)) and r["best_val"] == vals[r["best_idx"]]
        assert r["n_negative"] == (int(np.sum(vals < 0)) if kind == _lib.ACQ_EI else 0)
        one = _lib.acq_multi([h], Xt, 0, kind=kind, eta=[e], par=0.01, want_argmax=True)
        assert np.array_equal(one["values"], vals) and one["best_idx"] == r["best_idx"]
        assert one["n_negative"] == r["n_negative"]
    # the best row planted across the 128-candidate block edge and the chunk edge: the lowest index wins
    if M >= 130:
        r = h.acq(Xt, _lib.ACQ_EI, eta, 0.0)
        b = r["best_idx"]
        X2 = Xt.copy()
        spots = [127, 128] + ([chunk - 1, chunk] if chunk and chunk < M else [])
        X2[spots] = Xt[b]
        r2 = h.acq(X2, _lib.ACQ_EI, eta, 0.0)
        v2 = r2["values"]
        assert len(set(v2[spots].view(np.int64).tolist())) == 1
        assert r2["best_idx"] == int(np.argmax(v2)) <= min(spots + [b])
        assert v2[r2["best_idx"]] == v2[b] == r["best_val"]
        m2 = _lib.acq_multi([h], X2, 0, kind=_lib.ACQ_EI, eta=[eta], par=0.0, want_argmax=True)
        assert m2["best_idx"] == r2["best_idx"]


def test_fit_refuses_a_nonfinite_hyper_naming_its_index():
    X, y, Phi = R.case(_lib.BLR_LINEAR, 8, 129)
    h = _handle(X, y, _lib.BLR_LINEAR)
    good = np.array([[0.5, 10.0], [1.0, 20.0]])
    _lib.blr_fit(h, good)
    for bad in ([np.nan, 5.0], [2.0, np.nan], [-np.inf, 5.0]):
        H = np.array([[0.5, 10.0], [1.0, 20.0], bad, [np.nan, np.nan], [1.0, 1.0]])
        with pytest.raises(np.linalg.LinAlgError, match="hypers 2 "):
            _lib.blr_fit(h, H)
        with pytest.raises(RuntimeError, match="not fitted"):
            h.predict(X[:3])
        with pytest.raises(RuntimeError, match="not fitted"):
            _lib.blr_models(h)
    _lib.blr_fit(h, good)
    assert len(_lib.blr_models(h)) == 2


def _calls(h, X, thetas, hypers, Xt):
    """lnpost, fit, models, predict and acq on one handle, in that order."""
    out = [_lib.blr_lnpost(h, thetas)]
    _lib.blr_fit(h, hypers)
    out += [np.concatenate([np.concatenate([m, S.ravel()]) for m, S in _lib.blr_models(h)])]
    out += list(h.predict(Xt))
    r = h.acq(Xt, _lib.ACQ_EI, 0.0, 0.0)
    out += [r["values"], np.array([r["best_idx"]], dtype=np.float64)]
    return out


def test_handles_of_different_F_interleaved():
    """cudaFuncSetAttribute is per kernel and the latest blr_ready sets it: F = 3, 49 and 64 interleaved call by call
    give each handle's results alone bit for bit; then gpk_acq_multi over three handles of one D (F = 24, 25, 49)."""
    specs = [(_lib.BLR_LINEAR, 2, 300), (_lib.BLR_QUADRATIC, 24, 257), (_lib.BLR_NONE, 64, 129)]
    rng = np.random.RandomState(11)
    setup = []
    for basis, D, N in specs:
        X, y, _ = R.case(basis, D, N)
        setup.append((basis, X, y, rng.uniform(-1.2, 1.2, (1000, D))))
    thetas = np.array([[-2.0, 3.0], [0.5, 6.0], [-5.0, 1.0]])
    hypers = np.array([[0.1, 50.0], [1.0, 300.0], [0.02, 10.0]])
    alone = []
    for basis, X, y, Xt in setup:
        alone.append(_calls(_handle(X, y, basis), X, thetas, hypers, Xt))
    hs = [_handle(X, y, basis) for basis, X, y, _ in setup]
    got = [[] for _ in hs]
    for i, h in enumerate(hs):
        got[i].append(_lib.blr_lnpost(h, thetas))
    for i, h in enumerate(hs[::-1]):
        _lib.blr_fit(h, hypers)
    for i, h in enumerate(hs):
        got[i].append(np.concatenate([np.concatenate([m, S.ravel()]) for m, S in _lib.blr_models(h)]))
    for i, h in enumerate(hs):
        got[i] += list(h.predict(setup[i][3]))
    for i in (2, 0, 1):
        r = hs[i].acq(setup[i][3], _lib.ACQ_EI, 0.0, 0.0)
        got[i] += [r["values"], np.array([r["best_idx"]], dtype=np.float64)]
    for g, a in zip(got, alone):
        assert len(g) == len(a)
        for u, v in zip(g, a):
            assert np.array_equal(u.view(np.int64), v.view(np.int64))
    # one D, three bases
    D = 24
    X, y, _ = R.case(_lib.BLR_NONE, D, 200)
    Xt = rng.uniform(-1.2, 1.2, (4099, D))
    trio = [_handle(X, y, b) for b in (_lib.BLR_NONE, _lib.BLR_LINEAR, _lib.BLR_QUADRATIC)]
    for hh in trio:
        _lib.blr_fit(hh, hypers)
    etas = [0.1, -0.2, 0.3]
    per = [hh.acq(Xt, _lib.ACQ_EI, e, 0.0)["values"] for hh, e in zip(trio, etas)]
    mom = [hh.predict(Xt) for hh in trio]
    r = _lib.acq_multi(trio, Xt, 0, kind=_lib.ACQ_EI, eta=etas, par=0.0, want_argmax=True)
    ref = (per[0] + per[1] + per[2]) / 3
    tol = 4 * R.U * (np.abs(per[0]) + np.abs(per[1]) + np.abs(per[2])) / 3
    assert np.all(np.abs(r["values"] - ref) <= tol)
    assert r["best_idx"] == int(np.argmax(r["values"]))
    assert r["n_negative"] == sum(int(np.sum(p < 0)) for p in per)
    r1 = _lib.acq_multi(trio, Xt, 1)
    mus = np.array([m for m, _ in mom])
    vs = np.array([v for _, v in mom])
    mref = mus.mean(axis=0)
    vref = np.maximum(mus.var(axis=0) + vs.mean(axis=0), R.EPS)
    assert np.all(np.abs(r1["mean"] - mref) <= 8 * R.U * np.abs(mus).sum(axis=0))
    assert np.all(np.abs(r1["var"] - vref) <= 16 * R.U * (mus ** 2).sum(axis=0) + 8 * R.U * vs.sum(axis=0))


def test_model_class_quadratic_d31_end_to_end():
    """BayesianLinearRegression with the quadratic basis at D = 31 (F = 63), N = 300, a short chain; predict against
    the reference from the trained hypers (the moments from the device's own models)."""
    X, y, Phi = R.case(_lib.BLR_QUADRATIC, 31, 300)
    m = BayesianLinearRegression(basis_func=quadratic_basis_func, rng=np.random.RandomState(3), chain_length=20,
                                 burnin_steps=20)
    m.train(X, y, do_optimize=True)
    hypers = np.asarray(m.hypers, dtype=np.float64)
    assert hypers.shape == (20, 2)
    data = R.Data(Phi, y)
    Vabs, worst = [], 0.0
    for (mi, Si), (a, bt) in zip(m.models, hypers):
        ref = R.fit_reference(data, a, bt)
        assert ref is not None
        Vabs.append(np.abs(ref["V"].astype(np.float64)))
        if ref["eta"] <= 0.1:
            worst = max(worst, R.err_ratio(mi, ref["m"], ref["bound_m"]), R.err_ratio(Si, ref["S"], ref["bound_S"]))
    assert worst <= 1.0, worst
    Xt = np.random.RandomState(4).uniform(-1.2, 1.2, (500, 31))
    mu, var = m.predict(Xt)
    mref = R.moments_reference(BM.features(Xt, _lib.BLR_QUADRATIC), m.models, hypers[:, 1], Vabs)
    rm, rv = _moment_ratios(mu, var, mref)
    assert rm <= 1.0 and rv <= 1.0, "mu err/bound = %.3g, var err/bound = %.3g" % (rm, rv)
