"""Numpy restatement of EPMGP joint_min with derivatives (the p_min belief of entropy search), written from its
semantics in the order gpk_es.cuh evaluates it.

The sweeps (min_faktor / lt_factor / log_relative_gauss) are restated step by step: every scalar is a numpy float64
and every vector step an elementwise numpy operation, so each rounding happens where the kernel rounds it, and the
kernel's sweep counts must equal these.  The device can differ in the last bits only through its libm functions
(erfc, log, exp).  The closed form uses the structure of R (two entries per column) and sums in index order, as the
kernel does; that is the reference's algebra in another summation order than numpy's dense products.

joint_min(mu, V) -> dict(logP, dlogPdMu, dlogPdSigma, dlogPdMudMu, sweeps, lt_calls)
  sweeps[k]   sweeps EP ran for problem k (at most 50)
  lt_calls[k] lt_factor steps it took (the last sweep may stop early on a NaN step)
"""
import math

import numpy as np
from scipy import special

SQ2 = float(np.sqrt(2))
ISQ2 = 1.0 / SQ2
EPS32 = float(np.finfo(np.float32).eps)
L2P = float(np.log(2) + np.log(np.pi))


class EPFailed(Exception):
    pass


def _npmax(a, b):
    """numpy.max([a, b]): NaN propagates, otherwise a unless b is larger."""
    return a if (a >= b or math.isnan(a)) else b


def _lt_factor(k, l, M, V, mp, p):
    """One EP step on the message of pair (k, l).  Returns (M, V, pnew, mpnew, logS, d, exit_flag); M and V are
    updated in place when exit_flag != -1."""
    f = np.float64
    cVc = ((V[l, l] - 2.0 * V[k, l]) + V[k, k]) / 2.0
    cM = (M[l] - M[k]) / SQ2
    cVnic = _npmax(cVc / (1.0 - p * cVc), f(0.0))
    cmni = cM + cVnic * (p * cM - mp)
    z = cmni / np.sqrt(cVnic + 1e-25)
    if np.isnan(z):
        z = f(-np.inf)
    if z < -6.0:
        return M, V, 0.0, 0.0, -math.inf, float("nan"), -1
    if z > 6.0:
        pnew, mpnew, lS = f(0.0), f(0.0), f(0.0)
        dp, dmp = -p, -mp
        d = dp if dp > dmp else dmp
        exit_flag = 1
    else:
        logphi = -0.5 * (z * z + L2P)
        lP = np.log(0.5 * special.erfc(-z / SQ2))
        e = np.exp(logphi - lP)
        alpha = e / np.sqrt(cVnic)
        beta = alpha * (alpha * cVnic + cmni)
        rr = beta / (1.0 - beta)
        pnew = rr / cVnic
        mpnew = rr * (alpha + cmni / cVnic) + alpha
        dp = _npmax(-p + EPS32, pnew - p)
        dmp = _npmax(-mp + EPS32, mpnew - mp)
        d = _npmax(dmp, dp)
        pnew = p + dp
        mpnew = mp + dmp
        lS = (lP - 0.5 * ((np.log(beta) - np.log(pnew)) - np.log(cVnic))) + ((alpha * alpha) / (2.0 * beta)) * cVnic
        exit_flag = 0
    Vc = (V[:, l] - V[:, k]) / SQ2
    den = 1.0 + dp * cVc
    cv = dp / den
    cm = (dmp - cM * dp) / den
    V -= cv * (Vc[:, None] * Vc[None, :])
    M += cm * Vc
    if exit_flag == 0 and np.isnan(V).any():
        raise EPFailed("an error occurs while running expectation propagation in entropy search. "
                       "Resulting variance contains NaN")
    return M, V, pnew, mpnew, lS, d, exit_flag


def _seqsum(a):
    s = 0.0
    for x in a:
        s = s + float(x)
    return s


def _cholesky(S):
    """Left-looking lower Cholesky in the kernel's order; None when a pivot is not positive."""
    n = S.shape[0]
    L = np.zeros_like(S)
    for j in range(n):
        s = S[j, j]
        for m in range(j):
            s = s - L[j, m] * L[j, m]
        if not s > 0.0:
            return None
        L[j, j] = math.sqrt(s)
        for i in range(j + 1, n):
            s = S[i, j]
            for m in range(j):
                s = s - L[i, m] * L[j, m]
            L[i, j] = s / L[j, j]
    return L


def min_factor(mu, Sig, k):
    """EP problem k: -> (logZ, dlogZdMu (D,), dlogZdMudMu (D, D), dlogZdSigma packed (T,), sweeps, lt_calls)."""
    D = mu.shape[0]
    D1 = D - 1
    T = D * (D + 1) // 2
    P, MP, logS = np.zeros(D1), np.zeros(D1), np.zeros(D1)
    M, V = mu.copy(), Sig.copy()
    d = 0.0
    sweeps = calls = 0
    for _ in range(50):
        sweeps += 1
        diff = 0.0
        for i in range(D1):
            l = i if i < k else i + 1
            calls += 1
            M, V, P[i], MP[i], logS[i], d, _ = _lt_factor(k, l, M, V, MP[i], P[i])
            if math.isnan(d):
                break
            diff = diff + abs(d)
        if math.isnan(d):
            break
        if abs(diff) < 0.001:
            break
    if math.isnan(d):
        return -math.inf, np.zeros(D), np.zeros((D, D)), np.zeros(T), sweeps, calls

    rho = np.sqrt(P) * ISQ2
    lidx = np.array([j if j < k else j + 1 for j in range(D1)], dtype=np.int64)
    r = np.empty(D)
    r[lidx] = MP * ISQ2
    r[k] = _seqsum(MP * -ISQ2)
    q = ((Sig[np.ix_(lidx, lidx)] - Sig[lidx, k][:, None]) - Sig[k, lidx][None, :]) + Sig[k, k]
    L = None
    for jitter in (0.0, 1e-10, 1e-6):
        S = np.eye(D1) + (rho[:, None] * rho[None, :]) * q
        S[np.diag_indices(D1)] += jitter
        L = _cholesky(S)
        if L is not None:
            break
    if L is None:
        raise np.linalg.LinAlgError("IRSR is not positive definite")
    Rt = np.zeros((D1, D))
    Rt[np.arange(D1), lidx] = rho
    Rt[:, k] = -rho
    G = np.zeros((D1, D))
    for j in range(D1):
        s = Rt[j].copy()
        for m in range(j):
            s = s - L[j, m] * G[m]
        G[j] = s / L[j, j]
    A = np.zeros((D, D))
    for m in range(D1):
        A = A + G[m][:, None] * G[m][None, :]
    Sr = np.zeros(D)
    for j in range(D):
        Sr = Sr + Sig[:, j] * r[j]
    b = mu + Sr
    Ab = np.zeros(D)
    for j in range(D):
        Ab = Ab + A[:, j] * b[j]
    rSr = _seqsum(r * Sr)
    bAb = _seqsum(b * Ab)
    Mur = _seqsum(mu * r)
    dts = 2.0 * _seqsum(np.log(np.diag(L)))
    s = _seqsum(logS)
    mpm = _seqsum([MP[j] * MP[j] / P[j] for j in range(D1) if MP[j] != 0.0])
    logZ = ((0.5 * ((rSr - bAb) - dts) + Mur) + s) - 0.5 * mpm
    X = ((-A - 2.0 * (r[:, None] * Ab[None, :])) + r[:, None] * r[None, :]) + Ab[:, None] * Ab[None, :]
    Ssym = 0.5 * (X + X.T)
    Ssym[np.diag_indices(D)] = 0.5 * np.diag(X)
    return logZ, r - Ab, -A, Ssym[np.tril_indices(D)], sweeps, calls


def joint_min(mu, V):
    mu = np.asarray(mu, dtype=np.float64).ravel()
    V = np.asarray(V, dtype=np.float64)
    D = mu.shape[0]
    T = D * (D + 1) // 2
    logP = np.zeros(D)
    dMu, dSig, dMuMu = np.zeros((D, D)), np.zeros((D, T)), np.zeros((D, D, D))
    sweeps, calls = np.zeros(D, dtype=np.int64), np.zeros(D, dtype=np.int64)
    with np.errstate(all="ignore"):
        for k in range(D):
            logP[k], dMu[k], dMuMu[k], dSig[k], sweeps[k], calls[k] = min_factor(mu, V, k)
    return dict(sweeps=sweeps, lt_calls=calls, **renormalise(logP, dMu, dSig, dMuMu))


def renormalise(logP, dMu, dSig, dMuMu):
    """joint_min's renormalisation, sums over k in index order.  Zij is the elementwise square of Zm broadcast
    along the rows (Zm.T * Zm of a 1-D Zm), as in the reference."""
    with np.errstate(all="ignore"):
        return _renormalise(logP, dMu, dSig, dMuMu)


def _renormalise(logP, dMu, dSig, dMuMu):
    D = logP.shape[0]
    lp = np.where(np.isinf(logP), -500.0, logP)
    e = np.exp(lp)
    Z = _seqsum(e)
    mx = lp[0]
    for x in lp[1:]:
        mx = _npmax(mx, x)
    s = mx + float(np.log(_seqsum(np.exp(lp - mx))))
    s = mx if math.isinf(s) else s
    Zm, Zs, gg = np.zeros(D), np.zeros(dSig.shape[1]), np.zeros((D, D))
    for k in range(D):
        Zm = Zm + e[k] * dMu[k]
        Zs = Zs + e[k] * dSig[k]
        gg = gg + (dMuMu[k] + dMu[k][:, None] * dMu[k][None, :]) * e[k]
    Zm, Zs, gg = Zm / Z, Zs / Z, gg / Z
    adds = -gg + (Zm * Zm)[None, :]
    return dict(logP=lp - s, dlogPdMu=dMu - Zm[None, :], dlogPdSigma=dSig - Zs[None, :],
                dlogPdMudMu=dMuMu + adds[None, :, :])


# ---- the entropy change of one candidate (InformationGain._dh_fun) ------------------------------------------------
def dh_matrix(state, v, sigma):
    """_dh_fun in the reference's matrix order.  state: dict(logP (Nb,), lmb (Nb,), dlogPdMu, dlogPdSigma,
    dlogPdMudMu, W (Np,), sn2); v: predictive variance at the candidate; sigma (Nb,) its covariance to zb."""
    with np.errstate(all="ignore"):
        nb = sigma.size
        v_ = np.array([[v - state["sn2"]]])
        s = sigma.reshape(-1, 1)
        norm_cov = s.dot(1.0 / v_)
        dm = norm_cov.dot(np.sqrt(np.array([[v + 1e-10]])))
        dv = -norm_cov.dot(s.T)
        dv = dv[np.triu(np.ones((nb, nb))).T.astype(bool), np.newaxis]
        dMM = dm.dot(dm.T)
        trterm = np.sum(np.sum(state["dlogPdMudMu"] * dMM[None], 2), 1)[:, None]
        logP = state["logP"].reshape(-1, 1)
        det = state["dlogPdSigma"].dot(dv) + 0.5 * trterm
        sto = state["dlogPdMu"].dot(dm).dot(state["W"].reshape(1, -1))
        lPred = (logP + det) + sto
        mx = np.amax(lPred, axis=0)
        sl = mx + np.log(np.sum(np.exp(lPred - mx), axis=0))
        lsel = mx if np.any(np.isinf(sl)) else sl
        lPred = lPred - lsel
        lmb = state["lmb"].reshape(-1, 1)
        H = -np.sum(np.exp(logP) * (logP + lmb))
        dHp = np.sum(np.exp(lPred) * (lPred + lmb), axis=0) + H
        return float(np.mean(dHp))


def fold(dlogPdMudMu):
    """dlogPdMudMu[i] folded to its lower triangle, row-major: H[a][b] + H[b][a] off the diagonal."""
    nb = dlogPdMudMu.shape[0]
    a, b = np.tril_indices(nb)
    return np.where(a == b, dlogPdMudMu[:, a, b], dlogPdMudMu[:, a, b] + dlogPdMudMu[:, b, a])


def dh_folded(state, v, sigma):
    """The same in the kernel's folded order (gpk_es_dh_kernel): quadratic forms over the packed lower triangle."""
    with np.errstate(all="ignore"):
        nb = sigma.size
        a, b = np.tril_indices(nb)
        iv = 1.0 / (v - state["sn2"])
        sq = np.sqrt(v + 1e-10)
        dm = (sigma * iv) * sq
        dv = -((sigma[a] * iv) * sigma[b])
        dmm = dm[a] * dm[b]
        base = state["logP"].ravel() + (state["dlogPdSigma"].dot(dv) + 0.5 * fold(state["dlogPdMudMu"]).dot(dmm))
        g = state["dlogPdMu"].dot(dm)
        lPred = base[:, None] + g[:, None] * state["W"].reshape(1, -1)
        mx = np.amax(lPred, axis=0)
        sl = mx + np.log(np.sum(np.exp(lPred - mx), axis=0))
        lsel = mx if np.any(np.isinf(sl)) else sl
        L = lPred - lsel
        lmb = state["lmb"].ravel()
        lp = state["logP"].ravel()
        H = -np.sum(np.exp(lp) * (lp + lmb))
        return float(np.mean(np.sum(np.exp(L) * (L + lmb[:, None]), axis=0) + H))


def compute_value(dh, x, lower, upper):
    """compute()'s replacements around one candidate's dH (information_gain.py:112-125, 219-222)."""
    if np.any(x < lower) or np.any(x > upper):
        return float(np.spacing(1))
    if np.isnan(dh) or dh == np.inf:
        return -np.finfo(float).max
    return dh
