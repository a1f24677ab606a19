"""Pins the oracle's predictive-gradient reference (oracle.robo_oracle.gp_predictive_gradients, acq_gradients) to an
independent evaluation: the GP posterior written out in mpmath at 40 digits (kernel tree walked in mp arithmetic,
mp.cholesky / lu_solve for the solves) and differentiated by mpmath.diff, on every kernel case of tests/kernel_cases.py
with and without the input / output transforms; and, on one larger problem, against Richardson-extrapolated central
differences of the reference-faithful gp_predict.  No GPU and no compiled helper are needed."""
import mpmath as mp
import numpy as np
import pytest
from scipy.special import ndtr

from oracle import george_oracle as G
from oracle import robo_oracle as O
from tests import kernel_cases as KC

mp.mp.dps = 40


def _mp_kernel(k, x, xp):
    if isinstance(k, G.Product):
        return _mp_kernel(k.k1, x, xp) * _mp_kernel(k.k2, x, xp)
    if isinstance(k, G.ConstantKernel):
        return mp.exp(mp.mpf(k.log_constant))
    r2 = mp.mpf(0)
    for a, md in zip(k.axes, k._axis_metric()):
        r2 += (x[a] - xp[a]) ** 2 / mp.mpf(md)
    if isinstance(k, G.Matern52Kernel):
        r = mp.sqrt(5 * r2)
        return (1 + r + 5 * r2 / 3) * mp.exp(-r)
    if isinstance(k, G.Matern32Kernel):
        r = mp.sqrt(3 * r2)
        return (1 + r) * mp.exp(-r)
    if isinstance(k, G.ExpSquaredKernel):
        return mp.exp(-r2 / 2)
    raise TypeError(type(k))


class _MpPosterior(object):
    """mu(x), var(x) of a fitted oracle state, everything after the float64 inputs in 40-digit arithmetic."""

    def __init__(self, st):
        gp = st["gp"]
        self.k, self.st = gp.kernel, st
        self.X = [[mp.mpf(float(v)) for v in row] for row in gp._x]
        n = len(self.X)
        K = mp.matrix(n, n)
        for i in range(n):
            for j in range(n):
                K[i, j] = _mp_kernel(self.k, self.X[i], self.X[j])
            K[i, i] += mp.mpf(float(gp._yerr2[i])) + mp.exp(mp.mpf(float(gp.white_noise)))
        self.L = mp.cholesky(K)
        r = mp.matrix([mp.mpf(float(v)) - mp.mpf(float(st["mean"])) for v in st["y"]])
        self.alpha = mp.lu_solve(K, r)
        if st["normalize_input"]:
            self.lo = [mp.mpf(float(v)) for v in st["lower"]]
            self.span = [mp.mpf(float(u)) - mp.mpf(float(v)) for u, v in zip(st["upper"], st["lower"])]
        self.ys = mp.mpf(float(st["y_std"])) if st["normalize_output"] else mp.mpf(1)
        self.ym = mp.mpf(float(st["y_mean"])) if st["normalize_output"] else mp.mpf(0)

    def _unit(self, x):
        if not self.st["normalize_input"]:
            return x
        return [(v - l) / s for v, l, s in zip(x, self.lo, self.span)]

    def moments(self, x):
        u = self._unit(x)
        ks = [_mp_kernel(self.k, u, xj) for xj in self.X]
        mu = mp.fsum(a * b for a, b in zip(ks, self.alpha)) + mp.mpf(float(self.st["mean"]))
        v = []                                                         # v = L^-1 k*
        for i in range(len(ks)):
            v.append((ks[i] - mp.fsum(self.L[i, j] * v[j] for j in range(i))) / self.L[i, i])
        var = _mp_kernel(self.k, u, u) - mp.fsum(t * t for t in v)
        return mu * self.ys + self.ym, var * self.ys ** 2


def _mp_acq(kind, mu, var, eta, par):
    s = mp.sqrt(var)
    if kind == "lcb":
        return -(mu - par * s)
    z = (eta - mu - par) / s
    if kind == "ei":
        return s * (z * mp.ncdf(z) + mp.npdf(z))
    return mp.ncdf(z)


def _mp_acq_chain(kind, mu, var, dmu, dvar, eta, par):
    """d acq / d x = acq_mu dmu + acq_s dvar / (2 s), the partial derivatives written out independently of
    ei.py / pi.py / lcb.py."""
    s = mp.sqrt(var)
    ds = dvar / (2 * s)
    if kind == "lcb":
        return -dmu + par * ds
    z = (eta - mu - par) / s
    if kind == "ei":
        return -mp.ncdf(z) * dmu + mp.npdf(z) * ds
    return -mp.npdf(z) / s * dmu - mp.npdf(z) * z / s * ds


@pytest.mark.parametrize("variant", KC.VARIANTS)
@pytest.mark.parametrize("case", KC.CASES)
def test_predictive_gradients_match_mpmath(case, variant):
    N, M = 12, 3
    X, y, Xs = KC.data(case, variant, N, M, seed=5)
    st = KC.oracle_state(case, variant, X, y)
    g = O.gp_predictive_gradients(st, Xs)
    mu_o, var_o = O.gp_predict(st, Xs)
    post = _MpPosterior(st)
    D = Xs.shape[1]
    axes = range(D) if D <= 3 else (0, 1, D // 2, D - 1)
    eta = float(np.min(y)) + 0.1 * float(np.std(y))
    acqs = (("ei", eta, 0.0), ("ei", eta, 0.1), ("pi", eta, 0.0), ("lcb", 0.0, 2.5))
    ref_acq = {a: O.acq_gradients(mu_o, var_o, g["dmu"], g["dvar"], a[0], a[1], a[2]) for a in acqs}
    for c in range(M):
        x0 = [mp.mpf(float(v)) for v in Xs[c]]
        mu_mp, var_mp = post.moments(x0)
        assert abs(mu_o[c] - float(mu_mp)) <= 1e-12 * max(abs(float(mu_mp)), np.std(y))
        assert abs(var_o[c] - float(var_mp)) <= 1e-12 * float(var_mp)
        for a in axes:
            def along(t, i, a=a):
                x = list(x0)
                x[a] += t
                return post.moments(x)[i]
            dmu_mp, dvar_mp = mp.diff(lambda t: along(t, 0), 0), mp.diff(lambda t: along(t, 1), 0)
            dmu, dvar = float(dmu_mp), float(dvar_mp)
            assert abs(g["dmu"][c, a] - dmu) <= 1e-12 * g["s_mu"][c, a], (c, a, g["dmu"][c, a], dmu)
            assert abs(g["dvar"][c, a] - dvar) <= 1e-12 * g["s_var"][c, a], (c, a, g["dvar"][c, a], dvar)
            for (kind, e, par), (f, df) in ref_acq.items():
                e_, p_ = mp.mpf(e), mp.mpf(par)

                def acq_along(t):
                    m_, v_ = post.moments([v + (t if i == a else 0) for i, v in enumerate(x0)])
                    return _mp_acq(kind, m_, v_, e_, p_)
                # the closed-form derivative is the derivative of the closed form (all in 40 digits) ...
                chain_mp = _mp_acq_chain(kind, mu_mp, var_mp, dmu_mp, dvar_mp, e_, p_)
                assert abs(mp.diff(acq_along, 0) - chain_mp) <= mp.mpf(10) ** -25 * (abs(chain_mp) + 1e-300)
                # ... and acq_gradients evaluates it to rounding, on the oracle's own float moments and gradients
                m_o, v_o = mp.mpf(mu_o[c]), mp.mpf(var_o[c])
                ref_df = float(_mp_acq_chain(kind, m_o, v_o, mp.mpf(g["dmu"][c, a]), mp.mpf(g["dvar"][c, a]), e_, p_))
                sc = KC.acq_grad_scale(kind, mu_o[c:c + 1], var_o[c:c + 1], g["s_mu"][c:c + 1, a:a + 1],
                                g["s_var"][c:c + 1, a:a + 1], e, par)[0, 0]
                assert abs(df[c, a] - ref_df) <= 1e-12 * sc, (kind, c, a, df[c, a], ref_df, sc)
                if a == axes[0]:
                    # EI's closed form cancels in the lower tail: its error scale is s (|z| Phi(z) + phi(z))
                    s = np.sqrt(var_o[c])
                    z = (e - mu_o[c] - par) / s
                    fs = {"ei": s * (abs(z) * ndtr(z) + O._pdf(z)), "pi": ndtr(z), "lcb": abs(mu_o[c]) + par * s}[kind]
                    ref_f = float(_mp_acq(kind, m_o, v_o, e_, p_))
                    assert abs(f[c] - ref_f) <= 1e-12 * fs, (kind, c, f[c], ref_f)


def test_predictive_gradients_match_richardson_differences():
    """N = 300 (chunked evaluation of the reference, several chunks) against Richardson-extrapolated central
    differences of gp_predict (the reference-faithful path through george's full covariance)."""
    case, variant = "m52_axis0", "scaled"
    X, y, Xs = KC.data(case, variant, 300, 6, seed=9)
    st = KC.oracle_state(case, variant, X, y)
    g = O.gp_predictive_gradients(st, Xs, chunk_elems=300 * 3 * 2)
    D = Xs.shape[1]
    span = KC.box(variant, D)[1] - KC.box(variant, D)[0]
    for a in range(D):
        def cd(h):
            e = np.zeros(D)
            e[a] = h
            p, q = O.gp_predict(st, Xs + e), O.gp_predict(st, Xs - e)
            return (p[0] - q[0]) / (2 * h), (p[1] - q[1]) / (2 * h)
        h = 2e-3 * span[a]
        (m1, v1), (m2, v2) = cd(h), cd(h / 2)
        rm, rv = (4 * m2 - m1) / 3, (4 * v2 - v1) / 3
        # truncation O(h^4) and rounding ~ eps |f| / h leave ~1e-9 of the scale
        assert np.all(np.abs(g["dmu"][:, a] - rm) <= 1e-7 * g["s_mu"][:, a]), (a, g["dmu"][:, a], rm)
        assert np.all(np.abs(g["dvar"][:, a] - rv) <= 1e-7 * g["s_var"][:, a]), (a, g["dvar"][:, a], rv)


def test_acq_gradients_refuse_log_ei():
    with pytest.raises(ValueError):
        O.acq_gradients(np.zeros(2), np.ones(2), np.zeros((2, 1)), np.zeros((2, 1)), "log_ei", 0.0, 0.0)
