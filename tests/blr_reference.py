"""Extended-precision reference of Bayesian linear regression on the device (robo_b200/csrc/gpk_blr.cuh): the marginal
log-likelihood and prior of gpk_blr_lnpost, the weight posteriors of gpk_blr_fit and the predictive moments of
gpk_blr_score_kernel, each with a worst-case bound on the device's fp64 error (CPU only).

The features Phi are exact: numpy's x * x rounds like __dmul_rn, so tests/blr_model.features gives the device's Phi bit
for bit.  From them, in np.longdouble (fit_reference.exact_matmul, cholesky_ld, forward_ld):
    G = Phi^T Phi, b = Phi^T y (exact products), A = beta G + alpha I, L = chol(A), z = L^-1 (beta b),
    m = L^-T z = beta A^-1 b, r = y - Phi m, ||r|| (the 2-norm, not its square), m^T m, log det A = 2 sum log L_ii,
    mll = F/2 log alpha + N/2 log beta - N/2 log 2 pi - beta/2 ||r|| - alpha/2 m^T m - 1/2 log det A
plus the prior lognorm.logpdf(theta_0, sigma, loc) + log(log(1 + 3 (scale / exp(1 / theta_1))^2)) in the same order
as gpk_hy_lognorm / gpk_hy_horseshoe, with alpha = exp(theta_0) and beta = exp(theta_1) taken exactly.

Bounds (u = 2^-53, gamma_n = n u / (1 - n u), C = 2 on every bound; worst cases, first order in the perturbations
E_A, E_c below, and valid while eta = || |A^-1| E_A ||_2 <= 0.1, which `lnpost_reference` reports):
  depth d_N     the summation depth of an N-term sum: ceil(N / 256) + 8 on the device (one fma chain per thread of
                the strided rows, then the 256-wide tree of gpk_blr_gram_kernel and gpk_blr_eval); N + F + 1 for the
                numpy restatement (BLAS in any order, and the F-term product with inv(A)).
  E_A           = beta (gamma_{d_N} |Phi|^T |Phi| + 3 u |G|) + 3 u alpha I + 2 gamma_{F+1} |L| |L^T|
                (the Gram sums; exp's 1 ulp and the product for beta G, the same and the add for alpha; the Cholesky
                backward error, Higham Thm 10.3, plus the back substitution L^T m = z taken onto A)
  E_c           = beta (gamma_{d_N} |Phi|^T |y| + 3 u |b|) + gamma_{F+1} |L| |z|    (beta b and the carried row)
  m             dm = |A^-1| (E_c + E_A |m|)
  log det A     E_ld = sum_ij |A^-1|_ij (E_A)_ij + 2 ((F + 2) u sum |log L_ii| + F u)   (tr(A^-1 dA), each log's
                ulp, the in-order sum, the sqrt of each pivot)
  ||r||         E_r = || gamma_F |Phi| |m| + u |r| ||_2 + || |Phi| dm ||_2 + (gamma_{d_N} / 2 + u) ||r||
                (the fma dot of each row and y - f, the perturbation of m through Phi, the tree sum and its sqrt)
  mll terms     E_1 = F/2 (3 u + 2 u |theta_0|) + u |T_1|, E_2 the same with N, theta_1; E_3 = 2 u |T_3|;
                E_4 = beta/2 E_r + 3 u |T_4|; E_5 = alpha/2 (gamma_F m^T m + 2 |m|^T dm) + 3 u |T_5|; E_6 = E_ld / 2;
                the five in-order adds 5 u sum |T_i|
  prior         lognorm: y = theta_0 - loc, l = log y: dl = 2 u |l| + u, d(l^2) = 2 |l| dl + u l^2,
                E = (d(l^2) + 3 u l^2) / (2 sigma^2) + 4 u + 2 u |log(sigma y sqrt(2 pi))|;
                horseshoe: x = 1 / theta_1, q = scale / exp(x): dq / q = 4 u + u |x|; w = 1 + 3 q^2:
                dw = 3 q^2 (2 dq / q + 2 u) + u w; lw = log w: dlw = dw / w + 2 u |lw|; E = dlw / |lw| + 2 u |log lw|;
                the two adds u (|mll| + |prior|) + u |prior|
  fit           m_i within C dm; S_i = L^-T L^-1 against A^-1 within
                C (|A^-1| E_A |A^-1| + gamma_F (|V|^T |L^T| |S| + |S| |L| |V|) + gamma_F |V|^T |V|), V = L^-1
                (the perturbation of A, the substitution L V = I, the product V^T V)
  moments       against the device's own m_i and S_i (gpk_blr_get_models), with phi the candidate's features:
                mu = 1/k sum_i phi^T m_i within C (1/k sum_i gamma_F |phi|^T |m_i| + gamma_{k+1} 1/k sum_i |mu_i|)
                var = 1/k sum_i (1 / beta_i + phi^T S_i phi) within
                C (1/k sum_i [4 gamma_{F+1} || |V_i| |phi| ||^2 + 2 u (1 / beta_i)] + gamma_{k+1} 1/k sum_i var_i)
                (the device forms ||L_i^-1 phi||^2 from L_i^-1: gamma_F per dot, its squares and sum, and S_i's own
                product rounding); var clipped at eps: below eps by more than the bound, the device gives eps exactly.
"""
import math

import numpy as np

from tests.blr_model import features
from tests.fit_reference import LD, U, cholesky_ld, exact_matmul, forward_ld, gamma

C_BLR = 2.0
EPS = float(np.finfo(np.float64).eps)
LOG_DBL_MAX = 709.782712893384            # gpk_blr.cuh's clamps: det A overflows above, underflows to 0 below
LOG_DET_ZERO = -745.1332191019412
LOG_2PI = 1.8378770664093453


def device_depth(N):
    """Summation depth of an N-term sum on the device: the strided fma chain of each of 256 threads, then the tree."""
    return -(-int(N) // 256) + 8


def numpy_depth(N, F):
    return int(N) + int(F) + 1


def back_ld(L, z):
    """L^T m = z in longdouble."""
    n = L.shape[0]
    m = np.zeros(n, dtype=LD)
    for i in range(n - 1, -1, -1):
        m[i] = (z[i] - L[i + 1:, i] @ m[i + 1:]) / L[i, i]
    return m


def inv_lower_ld(L):
    """L^-1 of a lower-triangular longdouble matrix (column by column forward substitution, vectorised)."""
    n = L.shape[0]
    V = np.zeros_like(L)
    for i in range(n):
        e = np.zeros(n, dtype=LD)
        e[i] = 1
        V[i] = (e - L[i, :i] @ V[:i]) / L[i, i]
    return V


class Data(object):
    """The exact Gram quantities of one training set (Phi exact fp64 features, y)."""

    def __init__(self, Phi, y):
        self.Phi = np.ascontiguousarray(Phi, dtype=np.float64)
        self.y = np.ascontiguousarray(y, dtype=np.float64)
        self.N, self.F = self.Phi.shape
        self.G = exact_matmul(self.Phi.T, self.Phi)
        self.b = exact_matmul(self.Phi.T, self.y[:, None])[:, 0]
        aP = np.abs(self.Phi)
        self.aG = aP.T @ aP
        self.ab = aP.T @ np.abs(self.y)
        self.PhiL = self.Phi.astype(LD)


def posterior(data, alpha, beta, depth=None):
    """dict(A, L, z, m, V = L^-1, Ainv, EA, Ec, dm, eta) for alpha, beta (longdouble), or None when the reference's own
    A is not positive definite.  depth: summation depth of the Gram sums (device_depth(N) by default)."""
    F = data.F
    alpha, beta = LD(alpha), LD(beta)
    A = beta * data.G + alpha * np.eye(F, dtype=LD)
    L = cholesky_ld(A)
    if L is None:
        return None
    c = beta * data.b
    z = forward_ld(L, c)
    m = back_ld(L, z)
    V = inv_lower_ld(L)
    Ainv = V.T @ V
    d = device_depth(data.N) if depth is None else depth
    a, bt = float(alpha), float(beta)
    aL = np.abs(L.astype(np.float64))
    absG = np.abs(data.G.astype(np.float64))
    EA = bt * (gamma(d) * data.aG + 3 * U * absG) + 3 * U * a * np.eye(F) + 2 * gamma(F + 1) * (aL @ aL.T)
    Ec = bt * (gamma(d) * data.ab + 3 * U * np.abs(data.b.astype(np.float64))) \
        + gamma(F + 1) * (aL @ np.abs(z.astype(np.float64)))
    aAi = np.abs(Ainv.astype(np.float64))
    am = np.abs(m.astype(np.float64))
    dm = aAi @ (Ec + EA @ am)
    eta = float(np.linalg.norm(aAi @ EA, 2))
    return dict(A=A, L=L, z=z, m=m, V=V, Ainv=Ainv, EA=EA, Ec=Ec, dm=dm, eta=eta)


def prior_ld(theta, par):
    """(prior, bound) of gpk_hy_lognorm(theta_0) + gpk_hy_horseshoe(1 / theta_1) in longdouble; the prior is None where
    either part is not finite (the float64 semantics of blr_model decide those)."""
    sig, loc, scale = (LD(p) for p in par)
    t0, t1 = LD(theta[0]), LD(theta[1])
    y = t0 - loc
    if not (y > 0) or t1 == 0 or not np.isfinite(t0) or not np.isfinite(t1):
        return None, None
    l = np.log(y)
    k2 = np.log(sig * y * np.sqrt(2 * LD(np.pi)))
    ln = -l * l / (2 * sig * sig) - k2
    fl, fsig = float(abs(l)), float(sig)
    dl = 2 * U * fl + U
    dl2 = 2 * fl * dl + U * fl * fl
    e_ln = (dl2 + 3 * U * fl * fl) / (2 * fsig * fsig) + 4 * U + 2 * U * float(abs(k2))
    x = 1 / t1
    q = scale / np.exp(x)
    w = 1 + 3 * q * q
    lw = np.log(w)
    if not lw > 0:
        return None, None
    hs = np.log(lw)
    rq = 4 * U + U * float(abs(x))
    dw = 3 * float(q * q) * (2 * rq + 2 * U) + U * float(w)
    dlw = dw / float(w) + 2 * U * float(abs(lw))
    e_hs = dlw / float(lw) + 2 * U * float(abs(hs))
    p = ln + hs
    return p, e_ln + e_hs + U * float(abs(p))


def lnpost_reference(data, theta, par, depth=None):
    """dict(v, bound, eta, logdet) of the log-posterior at theta (mll + prior), or None where the reference's A is not
    positive definite or the prior is not finite (module docstring for the bound)."""
    theta = np.asarray(theta, dtype=np.float64)
    if not np.all(np.isfinite(theta)):
        return None
    t0, t1 = LD(theta[0]), LD(theta[1])
    alpha, beta = np.exp(t0), np.exp(t1)
    P = posterior(data, alpha, beta, depth)
    pr, e_pr = prior_ld(theta, par)
    if P is None or pr is None:
        return None
    F, N = data.F, data.N
    d = device_depth(N) if depth is None else depth
    m, L = P["m"], P["L"]
    r = data.y.astype(LD) - data.PhiL @ m
    nrm = np.sqrt(np.sum(r * r))
    mtm = np.sum(m * m)
    logL = np.log(np.diag(L))
    logdet = 2 * np.sum(logL)
    T = [LD(F) / 2 * t0, LD(N) / 2 * t1, LD(N) / 2 * np.log(2 * LD(np.pi)), beta / 2 * nrm, alpha / 2 * mtm,
         logdet / 2]
    mll = T[0] + T[1] - T[2] - T[3] - T[4] - T[5]
    aT = [float(abs(t)) for t in T]
    a, bt = float(alpha), float(beta)
    aPhi = np.abs(data.Phi)
    am = np.abs(m.astype(np.float64))
    dm = P["dm"]
    rr = np.abs(r.astype(np.float64))
    E_r = np.linalg.norm(gamma(F) * (aPhi @ am) + U * rr) + np.linalg.norm(aPhi @ dm) \
        + (gamma(d) / 2 + U) * float(nrm)
    aAi = np.abs(P["Ainv"].astype(np.float64))
    E_ld = float(np.sum(aAi * P["EA"])) + 2 * ((F + 2) * U * float(np.sum(np.abs(logL))) + F * U)
    E = [F / 2 * (3 * U + 2 * U * abs(float(t0))) + U * aT[0],
         N / 2 * (3 * U + 2 * U * abs(float(t1))) + U * aT[1],
         2 * U * aT[2],
         bt / 2 * E_r + 3 * U * aT[3],
         a / 2 * (gamma(F) * float(mtm) + 2 * float(am @ dm)) + 3 * U * aT[4],
         E_ld / 2]
    bound = sum(E) + 5 * U * sum(aT) + e_pr + U * (float(abs(mll)) + float(abs(pr)))
    v = mll + pr
    ld = float(logdet)
    if ld > LOG_DBL_MAX:                      # det A overflows: mll = -inf
        v = LD(-np.inf)
    elif ld < LOG_DET_ZERO:                   # det A underflows to 0: mll = +inf
        v = LD(np.inf)
    near = min(abs(ld - LOG_DBL_MAX), abs(ld - LOG_DET_ZERO)) <= max(E_ld, 1e-6)
    return dict(v=v, mll=mll, bound=C_BLR * bound, eta=P["eta"], logdet=ld, near_threshold=near)


def logdet_ld(data, theta):
    """log det A at theta in longdouble (None where A is not positive definite)."""
    A = np.exp(LD(theta[1])) * data.G + np.exp(LD(theta[0])) * np.eye(data.F, dtype=LD)
    L = cholesky_ld(A)
    return None if L is None else float(2 * np.sum(np.log(np.diag(L))))


def fit_reference(data, alpha, beta, depth=None):
    """dict(m, S, bound_m, bound_S, V, eta) of the weight posterior at (alpha, beta) as gpk_blr_fit gives it
    (S = A^-1), or None where A is not positive definite."""
    P = posterior(data, alpha, beta, depth)
    if P is None:
        return None
    F = data.F
    aV = np.abs(P["V"].astype(np.float64))
    aL = np.abs(P["L"].astype(np.float64))
    aS = np.abs(P["Ainv"].astype(np.float64))
    bS = aS @ P["EA"] @ aS + gamma(F) * (aV.T @ aL.T @ aS + aS @ aL @ aV) + gamma(F) * (aV.T @ aV)
    return dict(m=P["m"], S=P["Ainv"], bound_m=C_BLR * P["dm"], bound_S=C_BLR * bS, V=P["V"], eta=P["eta"])


def moments_reference(Phi_t, models, betas, Vabs):
    """dict(mu, var (unclipped), bound_mu, bound_var) of the marginalised moments of the candidate features Phi_t
    (M, F) from the device's own (m_i, S_i) of gpk_blr_get_models; betas (k,) the fitted beta_i, Vabs[i] = |L_i^-1| of
    the reference (magnitudes for the bound)."""
    k = len(models)
    F = Phi_t.shape[1]
    P = Phi_t.astype(LD)
    aP = np.abs(Phi_t)
    smu = np.zeros(Phi_t.shape[0], dtype=LD)
    svar = np.zeros(Phi_t.shape[0], dtype=LD)
    bmu = np.zeros(Phi_t.shape[0])
    bvar = np.zeros(Phi_t.shape[0])
    amu = np.zeros(Phi_t.shape[0])
    avar = np.zeros(Phi_t.shape[0])
    for (m, S), beta, Va in zip(models, betas, Vabs):
        mu_i = P @ m.astype(LD)
        q_i = np.sum((P @ S.astype(LD)) * P, axis=1)
        ib = 1 / LD(beta)
        smu += mu_i
        svar += ib + q_i
        bmu += gamma(F) * (aP @ np.abs(m))
        t = aP @ Va.T
        bvar += 4 * gamma(F + 1) * np.sum(t * t, axis=1) + 2 * U * float(ib)
        amu += np.abs(mu_i.astype(np.float64))
        avar += np.abs((ib + q_i).astype(np.float64))
    bmu = (bmu + gamma(k + 1) * amu) / k
    bvar = (bvar + gamma(k + 1) * avar) / k
    return dict(mu=(smu / k), var=(svar / k), bound_mu=C_BLR * bmu, bound_var=C_BLR * bvar)


def var_check(got, ref, bound):
    """Largest |got - ref| / bound over the entries the eps clip does not decide, and whether every entry below eps by
    more than its bound is exactly eps; ref unclipped (longdouble)."""
    ref64 = ref.astype(np.float64)
    below = ref64 + bound < EPS
    free = ref64 - bound > EPS
    err = np.abs((got.astype(LD) - ref).astype(np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(free, err / bound, 0.0)
    return float(np.max(r)) if r.size else 0.0, bool(np.all(got[below] == EPS))


def err_ratio(got, ref, bound):
    """Largest |got - ref| / bound; infinite references must be matched exactly (ratio 0 or inf)."""
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=LD)
    inf = ~np.isfinite(ref)
    if np.any(inf):
        if not np.array_equal(got[inf], ref[inf].astype(np.float64)):
            return float("inf")
        got, ref, bound = got[~inf], ref[~inf], np.broadcast_to(bound, inf.shape)[~inf]
    err = np.abs((got.astype(LD) - ref).astype(np.float64))
    bound = np.asarray(bound, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.max(r)) if r.size else 0.0


def theta_for_logdet(data, target, t1, lo=-800.0, hi=800.0):
    """theta_0 with log det A(theta_0, t1) = target (bisection; log det is increasing in theta_0)."""
    for _ in range(200):
        mid = (lo + hi) / 2
        ld = logdet_ld(data, (mid, t1))
        if ld is None or ld < target:
            lo = mid
        else:
            hi = mid
    return (lo + hi) / 2


def cond_theta(data, cond, t1):
    """theta_0 with cond(A) ~ cond at theta_1 = t1 (A = beta G + alpha I: (beta l_max + alpha) / (beta l_min + alpha))."""
    lam = np.linalg.eigvalsh(data.G.astype(np.float64))
    lmax, lmin = max(lam[-1], 0.0), max(lam[0], 0.0)
    beta = math.exp(t1)
    # (beta lmax + a) / (beta lmin + a) = cond  ->  a = beta (lmax - cond lmin) / (cond - 1)
    a = beta * (lmax - cond * lmin) / (cond - 1.0)
    return math.log(a) if a > 0 else None


# a lognormal loc far below every grid theta_0, so that the prior stays finite while alpha / beta span the conditions
GRID_PAR = (1.0, -800.0, 0.1)


def theta_grid(data, t1s=(-3.0, 4.0, 11.0, 18.0), n_cond=8):
    """theta rows from well-conditioned A to cond(A) ~ 1 / (F u) (as far as the data allow) at each theta_1 in t1s."""
    F = data.F
    rows = []
    for t1 in t1s:
        for c in np.geomspace(2.0, 1.0 / (F * U), n_cond):
            t0 = cond_theta(data, c, t1)
            if t0 is not None and -700 < t0 < 700:
                rows.append((t0, t1))
        rows.append((t1 - 3.0, t1))
    return np.array(rows)


# ---- the shapes of tests/test_gpu_blr_shapes.py -------------------------------------------------------------------------------------------------------
# (basis, D, N, clustered): every F threshold through each basis at small and large N, and the clustered quadratic sets
LNPOST_CASES = [
    (0, 7, 2, False), (0, 8, 129, False), (0, 32, 32, False), (0, 33, 257, False), (0, 47, 1, False),
    (0, 48, 256, False), (0, 51, 51, False), (0, 52, 4097, False), (0, 62, 128, False), (0, 63, 63, False),
    (1, 4, 8, False), (1, 16, 129, False), (1, 24, 2, False), (1, 26, 257, False), (1, 31, 4097, False),
    (1, 2, 30, True), (1, 16, 128, True),
    (2, 1, 1, False), (2, 1, 4097, False), (2, 8, 7, False), (2, 9, 256, False), (2, 33, 1, False),
    (2, 34, 129, False), (2, 48, 2, False), (2, 49, 257, False), (2, 52, 51, False), (2, 53, 128, False),
    (2, 63, 62, False), (2, 64, 63, False), (2, 64, 4097, False), (2, 64, 100000, False),
]


def case(basis, D, N, seed=0, clustered=False):
    """(X, y, Phi) of one training set: inputs in [-1, 1], or clustered at 1 + 1e-3 [0, 1) (nearly collinear
    quadratic features)."""
    rng = np.random.RandomState(seed + 1000 * D + N)
    X = 1.0 + 1e-3 * rng.rand(N, D) if clustered else rng.uniform(-1.0, 1.0, (N, D))
    y = np.sin(3.0 * X).sum(axis=1) + 0.1 * rng.randn(N)
    return X, y, features(X, basis)
