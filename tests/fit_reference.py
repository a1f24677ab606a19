"""Extended-precision reference of the fp64 fit path (the blocked Cholesky, the forward solve, the log-determinant,
L^-1 by recursive block inversion, the K^-1 gradient and the full posterior covariance), as backward errors or per-stage
errors taken against the device's OWN upstream outputs (CPU only).

Exact products.  exact_matmul(A, B) cuts every row of A and every column of B, after scaling it by a power of two so
that its largest entry lies in [1/2, 1), into S slices of beta = floor((53 - ceil(log2 k)) / 2) bits by truncation: each
slice entry is an integer below 2^beta times a power of two, so each slice product A_a B_b is a sum of k integers below
2^(2 beta) on one grid, below 2^53 in total, and the fp64 GEMM returns it exactly whatever its summation order, blocking
or FMA use.  The slice products are added in np.longdouble (64-bit significand).  What is left out is bounded entrywise
by
    ref_err_ij = 2^(eA_i + eB_j) k 2^(3 - beta S) + 2^-60 (|A| |B|)_ij
(the dropped pairs a + b >= S and the truncated tails: k 2^(-beta S) (S + 2) of the row and column scales, S = 6 here;
then eight longdouble roundings of the partial sums).  With beta >= 20 that is 2^-117 of the scales: every bound below
carries it and it never matters unless an entry is 1e-20 of its row and column, which the GEMM can also not resolve.
The same idea as the int8 digit split of tests/ozaki_model.py, with fp64 slices instead of int8 digits.

Bounds (u = 2^-53, gamma_n = n u / (1 - n u); c fixed small constants; each is a worst case, not an estimate):
  factor         |L^ L^T - K|_ij <= C_FACTOR gamma_{N+1} (|L^| |L^T|)_ij + C_PANEL 128 u T_ij + ref_err
                 (Higham, Thm 10.3) where K is the device's own matrix (gpk_kernel_matrix + diag_add) and T the
                 explicit-inverse term of the panel solve: the panel of block (I, k) is L_Ik = S_Ik X_kk^T with the
                 device's inverse X_kk of the diagonal tile, not a substitution, so its residual carries
                 |S_Ik| (|X_kk^T| |L_kk^T|) with S_Ik = L_Ik L_kk^T: T_Ik = (|L_Ik| |L_kk^T|) |X_kk^T| |L_kk^T| on the
                 off-diagonal blocks, 0 on the diagonal tiles.
  forward solve  |L^ z^ - (y - mean)| <= C_SOLVE gamma_N |L^| |z^|
  log-det        |logdet - 2 sum log L^_ii| <= C_LOGDET (N + 16) u sum |2 log L^_ii|  (the per-tile partial sums, the
                 fixed-order sum of the tiles and 1 ulp of each log)
  L^-1 (per stage)
      diagonal tile   |X^_kk L^_kk - I| <= C_INV 128 u |X^_kk| |L^_kk|
      tree node       |X^_21 + X^_22 (L^_21 X^_11)| <= C_INV (hi - lo) 128 u |X^_22| |L^_21| |X^_11|  for every node
                      (lo, mid, hi) of build_nodes (gpk_api.cu), mid = lo + ceil((hi - lo) / 2), in 128-row blocks
      upper triangle  exactly 0
  gradient       g_p = -1/2 sum_ij (a_i a_j - (X^T X)_ij) dK_ij/dtheta_p with a = X^T z^ from the device's X^ and z^ in
                 longdouble; |g_dev - g_ref| <= C_GRAD [(N + 64 + nblk / 256) u sum_ij |dK_ij| (|a_i a_j| + (|X^|^T |X^|)_ij)
                 + sum_ij |dK_ij| |da_i| |a_j|] * s_p, da = gamma_N |X^T| |z^| (the device's alpha = Q z), s_p = 1 or the
                 noise variance for the noise entry
  covariance     V = X^ K*^T, cov = (K** - V^T V) y_std^2 per entry within
                 C_COV (N + 16) u (|K**| + (|X^| |K*^T|)^T (|X^| |K*^T|)) y_std^2; the clip exactly as
                 gpk_cov_finish_kernel states it (es_reference.sigma_check)
  mean           |mu - (K* X^T z^ + mean) y_std - y_mean| <= C_COV (N + 16) u ((|K*| |X^T|) |z^| + |mean|) y_std + u |mu|
"""
import math

import numpy as np

LD = np.longdouble
U = 2.0 ** -53
EPS = float(np.finfo(np.float64).eps)
BM = 128
SLICES = 6

C_FACTOR, C_PANEL, C_SOLVE, C_LOGDET, C_INV, C_GRAD, C_COV = 2.0, 2.0, 2.0, 2.0, 2.0, 2.0, 2.0


def have_longdouble():
    return float(np.finfo(np.longdouble).eps) <= 1e-18


def gamma(n):
    return n * U / (1.0 - n * U)


# ---- exact products ------------------------------------------------------------------------------------------------
def slice_bits(k):
    return (53 - int(math.ceil(math.log2(max(int(k), 1))))) // 2


def _slices(A, beta, nslices):
    """Rows of A scaled by 2^-e (largest entry in [1/2, 1)) and cut into nslices truncated beta-bit slices."""
    A = np.asarray(A, dtype=np.float64)
    mx = np.max(np.abs(A), axis=1) if A.shape[1] else np.zeros(A.shape[0])
    e = np.where(mx > 0, np.frexp(mx)[1], 0).astype(np.int64)
    T = np.ldexp(A, -e[:, None])
    out = []
    for s in range(nslices):
        f = 2.0 ** (beta * (s + 1))
        S = np.trunc(T * f) / f
        out.append(S)
        T = T - S
    return out, e


def _gemm_numpy(A, B):
    return A @ B


def exact_matmul(A, B, gemm=None, nslices=SLICES, with_err=False):
    """A @ B (longdouble) with every slice product exact (module docstring); gemm(A, B) -> fp64 product, numpy by
    default.  with_err: also the entrywise bound on what the reference leaves out (fp64)."""
    gemm = gemm or _gemm_numpy
    A = np.asarray(A, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    k = A.shape[1]
    beta = slice_bits(k)
    SA, eA = _slices(A, beta, nslices)
    SBt, eB = _slices(B.T, beta, nslices)
    pairs = sorted(((a, b) for a in range(nslices) for b in range(nslices) if a + b < nslices), key=lambda p: -sum(p))
    acc = np.zeros((A.shape[0], B.shape[1]), dtype=LD)
    for a, b in pairs:                                   # smallest terms first
        acc += gemm(SA[a], np.ascontiguousarray(SBt[b].T)).astype(LD)
    scale = eA[:, None] + eB[None, :]
    out = np.ldexp(acc, scale.astype(np.int32)) if acc.size else acc
    if not with_err:
        return out
    err = np.ldexp(np.full(out.shape, float(k) * 2.0 ** (3 - beta * nslices)), scale.astype(np.int32)) \
        + 2.0 ** -60 * gemm(np.abs(A), np.abs(B))
    return out, err


def split2(M):
    """longdouble M -> (hi, lo) fp64 with hi + lo = M to about 2^-106 |M|."""
    hi = M.astype(np.float64)
    return hi, (M - hi.astype(LD)).astype(np.float64)


def ratio(err, bound):
    """Largest err / bound (0 where both are 0; inf where err > 0 = bound)."""
    err = np.asarray(err, dtype=np.float64)
    bound = np.asarray(bound, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.max(r)) if r.size else 0.0


# ---- the device's tree ---------------------------------------------------------------------------------------------
def build_nodes(lo, hi, nodes=None):
    """build_nodes of gpk_api.cu over 128-row blocks: (lo, mid, hi, height), children before parents."""
    nodes = [] if nodes is None else nodes
    if hi - lo <= 1:
        return 0, nodes
    mid = lo + (hi - lo + 1) // 2
    hl, _ = build_nodes(lo, mid, nodes)
    hr, _ = build_nodes(mid, hi, nodes)
    ht = 1 + max(hl, hr)
    nodes.append((lo, mid, hi, ht))
    return ht, nodes


# ---- checks --------------------------------------------------------------------------------------------------------
def default_panels(N):
    """(c0, c1, r0, r1): rows [r0, r1) of block column [c0, c1) come from a panel solve by the inverse of the diagonal
    block [c0, c1); the blocked factorisation's 128-column panels."""
    return [(k, min(k + BM, N), min(k + BM, N), N) for k in range(0, N, BM) if k + BM < N]


def factor_check(L, K, X, gemm=None, panels=None):
    """(ratio, err, bound) of the factor's backward error; X the device's L^-1 (for the panel term), panels as
    default_panels (gpk_fit_append adds one panel of N1 columns for its block row)."""
    gemm = gemm or _gemm_numpy
    N = L.shape[0]
    LLt, rerr = exact_matmul(L, L.T, gemm, with_err=True)
    err = np.abs((LLt - K.astype(LD)).astype(np.float64))
    absL = np.abs(L)
    bound = C_FACTOR * gamma(N + 1) * gemm(absL, absL.T) + rerr
    T = np.zeros_like(L)
    for c0, c1, r0, r1 in (default_panels(N) if panels is None else panels):
        Lkk, Xkk = absL[c0:c1, c0:c1], np.abs(X[c0:c1, c0:c1])
        amp = gemm(Xkk.T, Lkk.T)                                     # |X_kk^T| |L_kk^T|
        T[r0:r1, c0:c1] += gemm(gemm(absL[r0:r1, c0:c1], Lkk.T), amp)
    T = T + T.T
    bound = bound + C_PANEL * 128 * U * T
    return ratio(err, bound), err, bound


def solve_check(L, z, r, gemm=None):
    Lz, rerr = exact_matmul(L, z[:, None], gemm, with_err=True)
    err = np.abs((Lz[:, 0] - r.astype(LD)).astype(np.float64))
    bound = C_SOLVE * gamma(L.shape[0]) * (np.abs(L) @ np.abs(z)) + rerr[:, 0]
    return ratio(err, bound), err, bound


def logdet_ref(L):
    return 2 * np.sum(np.log(np.diag(L).astype(LD)))


def logdet_check(logdet, L):
    ref = logdet_ref(L)
    err = abs(float(LD(logdet) - ref))
    bound = C_LOGDET * (L.shape[0] + 16) * U * float(np.sum(np.abs(2 * np.log(np.diag(L)))))
    return ratio(err, max(bound, 4 * U * abs(float(ref)))), err, bound


def loglik_check(ll, logdet, z):
    """ll = -z^T z / 2 - logdet / 2 - N log(2 pi) / 2 on the device's z and log-det."""
    N = z.size
    zz = np.sum(z.astype(LD) ** 2)
    ref = -zz / 2 - LD(logdet) / 2 - LD(N) * np.log(2 * LD(np.pi)) / 2
    err = abs(float(LD(ll) - ref))
    bound = C_LOGDET * ((N + 16) * U * float(zz) + 8 * U * (abs(logdet) + N * math.log(2 * math.pi)))
    return ratio(err, bound), err, bound


def linv_checks(L, X, gemm=None, nodes=None):
    """Per-stage checks of X = L^-1 (both n x n): dict(diag=(ratio, worst block), node=(ratio, worst node),
    upper_zero=bool).  nodes: (lo, mid, hi, _) in 128-row blocks, build_nodes(0, nb) by default."""
    gemm = gemm or _gemm_numpy
    N = L.shape[0]
    nb = (N + BM - 1) // BM
    out = dict(upper_zero=bool(np.all(np.triu(X, 1) == 0.0)))
    worst = (0.0, None)
    for k in range(nb):
        s = slice(k * BM, min((k + 1) * BM, N))
        Xk, Lk = X[s, s], L[s, s]
        P, rerr = exact_matmul(Xk, Lk, gemm, with_err=True)
        err = np.abs((P - np.eye(Xk.shape[0], dtype=LD)).astype(np.float64))
        bound = C_INV * 128 * U * gemm(np.abs(Xk), np.abs(Lk)) + rerr
        r = ratio(err, bound)
        if r >= worst[0]:
            worst = (r, k)
    out["diag"] = worst
    worst = (0.0, None)
    if nodes is None:
        _, nodes = build_nodes(0, nb)
    for lo, mid, hi, _ in nodes:
        a, b, c = lo * BM, mid * BM, min(hi * BM, N)
        X11, L21, X21, X22 = X[a:b, a:b], L[b:c, a:b], X[b:c, a:b], X[b:c, b:c]
        M = exact_matmul(L21, X11, gemm)
        Mh, Ml = split2(M)
        R = exact_matmul(X22, Mh, gemm) + gemm(X22, Ml).astype(LD) + X21.astype(LD)
        err = np.abs(R.astype(np.float64))
        mag = gemm(np.abs(X22), gemm(np.abs(L21), np.abs(X11)))
        bound = C_INV * (hi - lo) * 128 * U * mag + 2.0 ** -100 * mag
        r = ratio(err, bound)
        if r >= worst[0]:
            worst = (r, (lo, mid, hi))
    out["node"] = worst
    return out


# ---- gradient -------------------------------------------------------------------------------------------------------
def _radial(family, r2):
    if family == 1:                                   # ExpSquared
        return np.exp(-r2 / 2), np.full_like(r2, LD(-0.5))
    c = LD(5) if family == 0 else LD(3)
    s = np.sqrt(c * r2)
    if family == 0:                                   # Matern-5/2
        p = 1 + s + s * s / 3
        return p * np.exp(-s), -(LD(5) / 6) * (1 + s) / p
    return (1 + s) * np.exp(-s), -(LD(3) / 2) / (1 + s)   # Matern-3/2


def kernel_terms_ld(flat, X):
    """k(X, X) and dk/dtheta for theta = [log_amp, log_metric_t ...] of a flattened kernel (robo_b200.kernels
    flatten()), in longdouble: dk/dlog_amp = k, dk/dlog_metric_t = -k dlog f(r2_g)/dr2 (x_t - x'_t)^2 / metric_t."""
    X = np.asarray(X, dtype=np.float64)
    axis, group, lm = list(flat["axis"]), list(flat["group"]), list(flat["log_metric"])
    fam = int(flat["family"])
    amp = np.exp(LD(flat["log_amp"]))
    nt = len(axis)
    D2 = []
    for t in range(nt):
        d = X[:, axis[t]].astype(LD)[:, None] - X[:, axis[t]].astype(LD)[None, :]
        D2.append(d * d / np.exp(LD(lm[t])))
    k = np.full(D2[0].shape, amp, dtype=LD)
    dlog = {}
    for g in sorted(set(group)):
        ts = [t for t in range(nt) if group[t] == g]
        r2 = sum(D2[t] for t in ts)
        f, dl = _radial(fam, r2)
        k = k * f
        for t in ts:
            dlog[t] = dl
    grads = [k] + [-k * dlog[t] * D2[t] for t in range(nt)]
    return k, grads


def grad_reference(flat, X, Xinv, z, noise_var, gemm=None):
    """(g_ref (nt + 2,) float64, bound (nt + 2,)) from the device's X^ = L^-1 and z^."""
    gemm = gemm or _gemm_numpy
    N = X.shape[0]
    a = exact_matmul(Xinv.T, z[:, None], gemm)[:, 0]
    Kinv = exact_matmul(Xinv.T, Xinv, gemm)
    A = a[:, None] * a[None, :] - Kinv
    absX = np.abs(Xinv)
    mag0 = np.abs(a.astype(np.float64))[:, None] * np.abs(a.astype(np.float64))[None, :] + gemm(absX.T, absX)
    da = gamma(N) * (absX.T @ np.abs(z))
    dmag = da[:, None] * np.abs(a.astype(np.float64))[None, :]
    _, grads = kernel_terms_ld(flat, X)
    nblk = (((N + BM - 1) // BM) ** 2) * 4
    g, bnd = [], []
    for dK in grads + [np.eye(N, dtype=LD)]:
        g.append(float(-np.sum(A * dK) / 2))
        adK = np.abs(dK.astype(np.float64))
        bnd.append(C_GRAD * ((N + 64 + nblk / 256) * U * np.sum(adK * mag0) + np.sum(adK * dmag)) / 2)
    g, bnd = np.array(g), np.array(bnd)
    g[-1] *= noise_var
    bnd[-1] *= noise_var
    return g, bnd


# ---- posterior covariance --------------------------------------------------------------------------------------------
def cov_reference(Xinv, Ks, Kss, z, mean, ys2=1.0, y_mean=0.0, y_std=1.0, gemm=None):
    """dict(cov (unclipped, fp64), cov_bound, mu, mu_bound) from the device's X^, z^ and the kernel blocks
    K* (m, N) and K** (m, m)."""
    gemm = gemm or _gemm_numpy
    N = Xinv.shape[0]
    V = exact_matmul(Xinv, Ks.T, gemm)                    # (N, m)
    Vh, Vl = split2(V)
    VtV = exact_matmul(Vh.T, Vh, gemm) + (gemm(Vh.T, Vl) + gemm(Vl.T, Vh)).astype(LD)
    cov = ((Kss.astype(LD) - VtV) * LD(ys2)).astype(np.float64)
    W = gemm(np.abs(Xinv), np.abs(Ks.T))
    cb = C_COV * (N + 16) * U * (np.abs(Kss) + gemm(W.T, W)) * ys2
    ah, al = split2(exact_matmul(Xinv.T, z[:, None], gemm))         # a = X^T z
    mu_n = exact_matmul(Ks, ah, gemm)[:, 0] + gemm(Ks, al)[:, 0].astype(LD) + LD(mean)
    mu = (mu_n * LD(y_std) + LD(y_mean)).astype(np.float64)
    mb = C_COV * (N + 16) * U * ((W.T @ np.abs(z)) + abs(mean)) * y_std + 2 * U * np.abs(mu)
    return dict(cov=cov, cov_bound=cb, mu=mu, mu_bound=mb)
