"""Every kernel shape, input scaling and output transform of tests/kernel_cases.py on the two device paths that read the
flattened kernel description (KSpec: axis, group / last, inv_metric, scale, amp) on their own:

  (a) the int8 scoring path (batches of >= 2048 candidates: gpk_cov_oz_kernel builds K* with its own copy of the input
      scaling, the pre-scaled operands, the group reset and the amplitude), through the model classes and gpk_acq,
      against the oracle's moments and closed forms;
  (b) the other scoring entry points on the same cases (gpk_acq_dev, gpk_maximize_random, gpk_acq_multi);
  (c) the predictive gradients (gpk_predict_grad: K*, the two job tables V = L^-1 K*^T and Wt = (L^-T V)^T, and
      gpk_predict_grad_kernel) against oracle.robo_oracle.gp_predictive_gradients, which walks the george kernel tree
      and is itself pinned to mpmath in tests/test_grad_oracle_cpu.py.

Tolerances: moments at the north-star tolerances of tests/product_cases.py; EI / PI at rtol 1e-8; gradients at 1e-10
relative to s_mu = sum_j |dk_j| |alpha_j| and s_var = 2 sum_j |dk_j| |w_j| unless the conditioning of K says the
float64 solves cannot deliver that (then 16 kappa(K) eps, printed).
"""
import os

import numpy as np
import pytest
from scipy.special import log_ndtr, ndtr

from oracle import george_oracle as G
from oracle import robo_oracle as O
from tests import kernel_cases as KC
from tests.product_cases import assert_acq_close, assert_mean_close, assert_var_close

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
CASE_PARAMS = [pytest.param(c, v, id="%s-%s" % (c, v)) for c in KC.CASES for v in KC.VARIANTS]
# the int8 contraction is off under GPK_OZAKI=0
OZAKI_OFF = os.environ.get("GPK_OZAKI") == "0"


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _fit(case, variant, N, M, seed=0):
    X, y, Xs = KC.data(case, variant, N, M, seed)
    model = KC.model(case, variant)
    model.train(X, y, do_optimize=False)
    return model, KC.oracle_state(case, variant, X, y), X, y, Xs


def _ref_values(kind, mu, var, eta, par):
    """The reference's closed forms on the oracle moments (EI without the reference's raise on a negative value, so
    that negative values can be counted)."""
    if kind == "ei":
        s = np.sqrt(var)
        z = (eta - mu - par) / s
        return s * (z * ndtr(z) + O._pdf(z))
    if kind == "lcb":
        return O.acq_lcb(mu, var, par)
    return O.ACQ[kind](mu, var, eta, par)


def _moment_atol(kind, mu, var, eta, par, y, kss):
    """Absolute floor of EI / PI / LCB: 1e-13 (times std(y) for EI and LCB, which are in output units) plus the
    north-star moment tolerances carried through the closed form, |f_mu| dmu + |f_s| ds with ds = dvar / (2 s).  Near
    the data sigma^2 is at the noise level and a 1e-10 relative error of it moves EI by more than a bare 1e-13."""
    s = np.sqrt(var)
    dm = 1e-10 * np.maximum(np.abs(mu), np.std(y))
    ds = 1e-10 * np.maximum(var, 1e-6 * kss) / (2 * s)
    if kind == "lcb":
        return 1e-13 * max(1.0, np.std(y)) + dm + par * ds
    z = (eta - mu - par) / s
    if kind == "ei":
        return 1e-13 * max(1.0, np.std(y)) + ndtr(z) * dm + O._pdf(z) * ds
    return 1e-13 + O._pdf(z) / s * (dm + np.abs(z) * ds)


def _assert_best(best_idx, ref):
    """numpy.argmax semantics (first maximum); a different index only where the reference's top values tie to 1e-12."""
    i = O.argmax_first(ref)
    if best_idx != i:
        assert abs(ref[best_idx] - ref[i]) <= 1e-12 * max(abs(ref[i]), 1e-300), (best_idx, i, ref[best_idx], ref[i])


def _assert_log_ei_close(got, ref, mu, var, f_min, y, kss):
    """LogEI = log EI(mu, s) has no scale of its own: near the data sigma^2 is noisy relative to itself and log EI
    moves by orders of magnitude.  So its error is bounded by the moment tolerances carried through its derivative,
    taken in log space so that nothing under- or overflows:
        d logEI / d mu  = -Phi(z) / EI          = -exp(log Phi(z) - logEI)
        d logEI / d var = phi(z) / (2 s EI)     =  exp(log phi(z) - logEI) / (2 s)
        |got - ref| <= |d/d mu| dmu + |d/d var| dvar + 1e-8 max(1, |ref|)
    with z = (f_min - mu) / s, f_min = eta - par, dmu = 1e-10 max(|mu|, std y) and dvar = 1e-10 max(var, 1e-6 k(x, x))
    (tests/product_cases.py)."""
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(got), fin), "LogEI: finite pattern differs"
    assert np.all(got[~fin] == ref[~fin])
    g, r, m, v = got[fin], ref[fin], mu[fin], var[fin]
    s = np.sqrt(v)
    z = (f_min - m) / s
    dm = np.exp(log_ndtr(z) - r)
    dv = np.exp(O._logpdf(z) - r) / (2 * s)
    bound = dm * 1e-10 * np.maximum(np.abs(m), np.std(y)) + dv * 1e-10 * np.maximum(v, 1e-6 * kss) \
        + 1e-8 * np.maximum(1.0, np.abs(r))
    excess = np.abs(g - r) - bound
    assert np.all(excess <= 0), "LogEI: max excess error %.3g" % excess.max()


# --------------------------------------------------------------------------- (a) int8 scoring path
@pytest.mark.parametrize("case,variant", CASE_PARAMS)
def test_int8_scoring_matches_oracle(case, variant):
    """Model classes and gpk_acq on 2600+ candidates (the int8 contraction) against the oracle, with exact training
    inputs (the cancellation regime: sigma^2 at the noise level), points far from the data (sigma^2 = k(x, x)) and
    copies of every arg-max planted; then the same batch through gpk_acq_dev (identical results) and with ozaki = 0."""
    import torch
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    model, st, X, y, Xs = _fit(case, variant, 300, 2600)
    D = Xs.shape[1]
    lo, up = KC.box(variant, D)
    Xs[:8] = X[:8]                                                       # exact training inputs
    for i in range(4):                                                   # far from the data
        Xs[8 + i] = lo + (up - lo) * (6.0 + i)
    kss = KC.prior_var(case, st)
    mu_b, var_b = O.gp_predict_var_only_fast(st, Xs)
    eta_min, eta_med, eta_inc = float(np.min(y)), float(np.median(y)), float(O.gp_get_incumbent(st)[1])
    acqs = [("ei", 0.0, eta_min), ("ei", 0.1, eta_min), ("ei", 0.0, eta_med), ("ei", 0.1, eta_med),
            ("log_ei", 0.0, eta_inc), ("log_ei", 0.3, eta_inc), ("pi", 0.0, eta_inc), ("lcb", 1.0, 0.0), ("lcb", 2.5, 0.0)]
    # a copy of each reference arg-max at the end of the batch: the first index must win
    dups = sorted({O.argmax_first(_ref_values(k, mu_b, var_b, e, p)) for k, p, e in acqs})
    M0 = len(Xs)
    Xs = np.vstack([Xs, Xs[dups]])
    mu_ref, var_ref = np.concatenate([mu_b, mu_b[dups]]), np.concatenate([var_b, var_b[dups]])
    assert np.all(var_ref[8:12] >= kss * (1 - 1e-9))

    h = model.gp.handle
    oz0 = h.timings()["launches_ozaki"]
    mu, var = model.predict(Xs)
    assert_mean_close(mu, mu_ref, y)
    assert_var_close(var, var_ref, kss)
    cls = {"ei": EI, "log_ei": LogEI, "pi": PI, "lcb": LCB}
    for kind, par, eta in acqs:
        ref = _ref_values(kind, mu_ref, var_ref, eta, par)
        acq = cls[kind](model, par=par)
        vals = acq.compute(Xs, eta=eta) if kind == "ei" else acq.compute(Xs)
        r = h.acq(Xs, _lib.ACQ_KIND[kind], eta, par, want_values=True, want_moments=True)
        np.testing.assert_array_equal(vals, r["values"])
        np.testing.assert_array_equal(r["mu"], mu)
        np.testing.assert_array_equal(r["var"], var)
        if kind == "log_ei":
            _assert_log_ei_close(r["values"], ref, mu_ref, var_ref, eta - par, y, kss)
        else:
            assert_acq_close(r["values"], ref, rtol=1e-8 if kind != "lcb" else 1e-9,
                             atol=_moment_atol(kind, mu_ref, var_ref, eta, par, y, kss))
        _assert_best(r["best_idx"], ref)
        assert r["best_idx"] < M0
        np.testing.assert_array_equal(r["values"][M0:], r["values"][dups])       # position does not change a value
        if kind == "ei":
            assert r["n_negative"] == int(np.sum(ref < 0)) == 0
    if not OZAKI_OFF:
        assert h.timings()["launches_ozaki"] > oz0, "no int8 contraction ran: silent fp64 fallback"

    # gpk_acq_dev: the device-pointer entry point gives gpk_acq's results bit for bit
    r = h.acq(Xs, _lib.ACQ_EI, eta_min, 0.1, want_values=True, want_moments=True)
    dX = torch.from_numpy(np.ascontiguousarray(Xs)).cuda()
    out, dmu, dvar = (torch.empty(len(Xs), dtype=torch.float64, device="cuda") for _ in range(3))
    best = torch.empty(2, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    h.acq_dev(dX.data_ptr(), len(Xs), _lib.ACQ_EI, eta_min, 0.1, out.data_ptr(), dmu.data_ptr(), dvar.data_ptr(),
              best.data_ptr())
    h.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), r["values"])
    np.testing.assert_array_equal(dmu.cpu().numpy(), r["mu"])
    np.testing.assert_array_equal(dvar.cpu().numpy(), r["var"])
    b = best.cpu()
    assert b[0].item() == r["best_val"] and int(b.view(torch.int64)[1].item()) == r["best_idx"]

    # the fp64 contraction on the same batch agrees with the oracle at the same tolerances
    h.set_option("ozaki", 0)
    r0 = h.acq(Xs, _lib.ACQ_EI, eta_min, 0.0, want_values=True, want_moments=True)
    assert_mean_close(r0["mu"], mu_ref, y)
    assert_var_close(r0["var"], var_ref, kss)
    ref = _ref_values("ei", mu_ref, var_ref, eta_min, 0.0)
    assert_acq_close(r0["values"], ref, rtol=1e-8, atol=_moment_atol("ei", mu_ref, var_ref, eta_min, 0.0, y, kss))
    _assert_best(r0["best_idx"], ref)


# --------------------------------------------------------------------------- (b) other entry points
@pytest.mark.parametrize("case,variant", CASE_PARAMS)
def test_maximize_random_matches_oracle_argmax(case, variant):
    """gpk_maximize_random with the variant's box: 3000 device-generated candidates (int8 path), winner = the arg-max of
    the oracle's EI over the oracle's restatement of the same candidates."""
    from robo_b200 import _lib
    model, st, X, y, _ = _fit(case, variant, 300, 1, seed=3)
    D = X.shape[1]
    lo, up = KC.box(variant, D)
    inc, eta = model.get_incumbent()
    seed, M, nu = 0x5EED0000 + KC.CASES.index(case), 3000, 2100
    x, val, idx = model.gp.handle.maximize_random(seed, 0, M, nu, lo, up, inc, 0.1, _lib.ACQ_EI, float(eta), 0.0)
    cand = O.generate_candidates(seed, 0, M, nu, lo, up, inc, 0.1)
    mu_ref, var_ref = O.gp_predict_var_only_fast(st, cand)
    ref = _ref_values("ei", mu_ref, var_ref, float(eta), 0.0)
    _assert_best(idx, ref)
    assert abs(val - ref[idx]) <= 1e-8 * abs(ref[idx]) + 1e-13
    np.testing.assert_allclose(x, cand[idx], rtol=0, atol=1e-13 * np.max(np.abs(up)))


@pytest.mark.parametrize("kind", ["ei", "log_ei"])
def test_acq_multi_prod1d_models_match_oracle(kind):
    """gpk_acq_multi at m = 2500 over three fitted models of the Fabolas shape (product of 1-D Matern-5/2, input box,
    output transform), as GP-MCMC marginalisation uses it: mode 0 against the mean of the oracle's per-model values,
    mode 1 against the oracle's mixture moments."""
    from robo_b200 import _lib
    from robo_b200 import kernels as K
    case, variant = "prod1d", "scaled"
    X, y, Xs = KC.data(case, variant, 300, 2500, seed=11)
    models, states = [], []
    for i, shift in enumerate((0.0, 0.3, -0.4)):
        theta = KC.build(K, case).get_parameter_vector() + np.r_[0.2 * i, np.full(len(X[0]), shift)]
        km, kg = KC.build(K, case), KC.build(G, case)
        km.set_parameter_vector(theta)
        kg.set_parameter_vector(theta)
        m = KC.model(case, variant)
        m.kernel = km
        m.train(X, y, do_optimize=False)
        lo, up = KC.box(variant, X.shape[1])
        models.append(m)
        states.append(O.gp_fit(kg, X, y, noise=KC.NOISE, normalize_input=True, normalize_output=True, lower=lo, upper=up))
    handles = [m.gp.handle for m in models]
    moms = [O.gp_predict_var_only_fast(s, Xs) for s in states]
    etas = [float(O.gp_get_incumbent(s)[1]) for s in states]
    par = 0.0 if kind == "ei" else 0.3
    r = _lib.acq_multi(handles, Xs, 0, _lib.ACQ_KIND[kind], etas, par, want_argmax=True)
    per = [_ref_values(kind, mu, var, e, par) for (mu, var), e in zip(moms, etas)]
    ref = O.marginalised_acquisition(per)
    if kind == "ei":
        atol = np.mean([_moment_atol("ei", mu, var, e, par, y, KC.prior_var(case, s))
                        for (mu, var), e, s in zip(moms, etas, states)], axis=0)
        assert_acq_close(r["values"], ref, rtol=1e-8, atol=atol)
        assert r["n_negative"] == 0
    else:                                   # mean of three LogEI values: each error bounded as in the single-model test
        for k, (mu, var) in enumerate(moms):
            got_k = models[k].gp.handle.acq(Xs, _lib.ACQ_LOG_EI, etas[k], par)["values"]
            _assert_log_ei_close(got_k, per[k], mu, var, etas[k] - par, y, KC.prior_var(case, states[k]))
        fin = np.isfinite(ref)
        assert np.array_equal(np.isfinite(r["values"]), fin)
        per_dev = [m.gp.handle.acq(Xs, _lib.ACQ_LOG_EI, e, par)["values"] for m, e in zip(models, etas)]
        np.testing.assert_allclose(r["values"][fin], np.mean(per_dev, axis=0)[fin], rtol=1e-14, atol=0)
    _assert_best(r["best_idx"], ref)
    r1 = _lib.acq_multi(handles, Xs, 1)
    m_ref, v_ref = O.mcmc_mixture_moments(np.array([a for a, _ in moms]), np.array([b for _, b in moms]))
    assert_mean_close(r1["mean"], m_ref, y)
    assert_var_close(r1["var"], v_ref, max(KC.prior_var(case, s) for s in states))


# --------------------------------------------------------------------------- (c) predictive gradients
GRAD_SHAPES = [(1, 7), (129, 300), (300, 2049), (1100, 129), (129, 1)]    # 1, 2, 3, 9 row blocks; 1 .. 17 candidate blocks
                                                                          # (N = 2 instead of 1 with normalize_output)


def _kappa(st):
    gp = st["gp"]
    K = gp.kernel.get_value(gp._x)
    K[np.diag_indices_from(K)] += gp._yerr2 + np.exp(gp.white_noise)
    return float(np.linalg.cond(K))


def _grad_tol(st, label):
    """1e-10, or 16 kappa(K) eps where the conditioning of K caps what float64 solves (the device's L^-1 route and the
    oracle's Cholesky solve alike) can deliver."""
    kappa = _kappa(st)
    tol = max(1e-10, 16 * kappa * EPS)
    print("%s: kappa(K) = %.3g -> gradient tolerance %.3g" % (label, kappa, tol))
    return tol


def _assert_grads(dmu, dvar, ref, tol, what=""):
    emu = np.abs(dmu - ref["dmu"]) - tol * ref["s_mu"]
    evar = np.abs(dvar - ref["dvar"]) - tol * ref["s_var"]
    assert np.all(emu <= 0), "%s d mu: max excess %.3g (scaled %.3g)" % (
        what, emu.max(), np.max(np.abs(dmu - ref["dmu"]) / np.maximum(ref["s_mu"], 1e-300)))
    assert np.all(evar <= 0), "%s d var: max excess %.3g (scaled %.3g)" % (
        what, evar.max(), np.max(np.abs(dvar - ref["dvar"]) / np.maximum(ref["s_var"], 1e-300)))


def _acq_grad_bound(kind, mu, var, ref, eta, par, tol, y, kss):
    """Tolerance of df: the gradient tolerance through the closed form (KC.acq_grad_scale), plus the north-star moment
    tolerances carried through it (df re-evaluated at mu +- dmu and var +- dvar), plus 1e-300 for results that are
    subnormal (deep in the tails of Phi and phi)."""
    bound = tol * KC.acq_grad_scale(kind, mu, var, ref["s_mu"], ref["s_var"], eta, par) + 1e-300
    df0 = O.acq_gradients(mu, var, ref["dmu"], ref["dvar"], kind, eta, par)[1]
    dm = 1e-10 * np.maximum(np.abs(mu), np.std(y))
    dv = 1e-10 * np.maximum(var, 1e-6 * kss)
    for pair in (((mu + dm, var), (mu - dm, var)), ((mu, var + dv), (mu, np.maximum(var - dv, EPS)))):
        bound = bound + np.maximum(*[np.abs(O.acq_gradients(m2, v2, ref["dmu"], ref["dvar"], kind, eta, par)[1] - df0)
                                     for m2, v2 in pair])
    return df0, bound


@pytest.mark.parametrize("case,variant", CASE_PARAMS)
def test_predictive_gradients_match_oracle(case, variant):
    """dmu/dx, dvar/dx (model.predictive_gradients) and the EI / PI / LCB input gradients (derivative=True) against the
    oracle at 1, 2, 3 and 9 row blocks and 1 .. 17 candidate blocks (m = 2049: moments from the int8 path); predict_grad's
    moments equal gpk_predict's, and chunk = 128 < m changes no bit.  N > 224 pins all eight warps' partials of the
    gradient kernel; m > 128 pins the Wt job table beyond the first candidate block."""
    from robo_b200.acquisition_functions import EI, LCB, PI
    for N, m in GRAD_SHAPES:
        N = 2 if N == 1 and variant == "scaled" else N          # one target has no standard deviation
        model, st, X, y, Xs = _fit(case, variant, N, m, seed=m)
        tol = _grad_tol(st, "%s-%s N=%d m=%d" % (case, variant, N, m))
        kss = KC.prior_var(case, st)
        ref = O.gp_predictive_gradients(st, Xs)
        dmu, dvar = model.predictive_gradients(Xs)
        assert dmu.shape == dvar.shape == Xs.shape
        _assert_grads(dmu, dvar, ref, tol, "N=%d m=%d" % (N, m))
        h = model.gp.handle
        r = h.predict_grad(Xs)
        mu_p, var_p = h.predict(Xs)
        np.testing.assert_array_equal(r["mu"], mu_p)
        np.testing.assert_array_equal(r["var"], var_p)
        np.testing.assert_array_equal(r["dmu"], dmu)
        mu_ref, var_ref = O.gp_predict_var_only_fast(st, Xs)
        eta = float(O.gp_get_incumbent(st)[1])
        for cls, kind, par in ((EI, "ei", 0.0), (EI, "ei", 0.1), (PI, "pi", 0.0), (LCB, "lcb", 2.5)):
            f, df = cls(model, par=par).compute(Xs, derivative=True)
            e = 0.0 if kind == "lcb" else eta
            assert_acq_close(f, _ref_values(kind, mu_ref, var_ref, e, par), rtol=1e-8 if kind != "lcb" else 1e-9,
                             atol=_moment_atol(kind, mu_ref, var_ref, e, par, y, kss))
            df_ref, bound = _acq_grad_bound(kind, mu_ref, var_ref, ref, e, par, tol, y, kss)
            excess = np.abs(df - df_ref) - bound
            assert np.all(excess <= 0), "%s par %g N=%d m=%d: df max excess %.3g" % (kind, par, N, m, excess.max())
        if m > 128:
            h.set_option("chunk", 128)
            r2 = h.predict_grad(Xs)
            for k in ("mu", "var", "dmu", "dvar"):
                np.testing.assert_array_equal(r2[k], r[k])
        model.gp.handle.close()


@pytest.mark.parametrize("case,variant", CASE_PARAMS)
def test_predictive_gradients_after_fit_append(case, variant):
    """Gradients after the incremental refit (rows 650 -> 700 appended inside the last 128-row block) against a fresh
    full fit and the oracle."""
    X, y, Xs = KC.data(case, variant, 700, 300, seed=2)
    model = KC.model(case, variant)
    model.train(X[:650], y[:650], do_optimize=False)
    model.predict(Xs[:10])                                   # builds L^-1, which the shortcut extends
    model.train(X, y, do_optimize=False)
    assert model.gp.n_appends == 1
    fresh = KC.model(case, variant)
    fresh.train(X, y, do_optimize=False)
    assert fresh.gp.n_appends == 0
    st = KC.oracle_state(case, variant, X, y)
    tol = _grad_tol(st, "%s-%s append" % (case, variant))
    ref = O.gp_predictive_gradients(st, Xs)
    dmu_a, dvar_a = model.predictive_gradients(Xs)
    dmu_f, dvar_f = fresh.predictive_gradients(Xs)
    _assert_grads(dmu_a, dvar_a, ref, tol, "appended")
    _assert_grads(dmu_f, dvar_f, ref, tol, "fresh")
    _assert_grads(dmu_a, dvar_a, dict(ref, dmu=dmu_f, dvar=dvar_f), 2 * tol, "appended vs fresh")


def test_predict_grad_refusals():
    from robo_b200 import _lib
    model, st, X, y, Xs = _fit("m52", "raw", 50, 5)
    h = model.gp.handle
    with pytest.raises(ValueError):
        h.predict_grad(np.zeros((16385, X.shape[1])))
    with pytest.raises(ValueError):
        h.predict_grad(Xs, _lib.ACQ_LOG_EI, float(np.min(y)), 0.0)
    r = h.predict_grad(Xs)                                   # the handle is still usable
    assert np.all(np.isfinite(r["dmu"]))
