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

C_FACTOR, C_PANEL, C_SOLVE, C_LOGDET, C_INV, C_GRAD, C_COV, C_PGRAD, C_HY = 2.0, 2.0, 2.0, 2.0, 2.0, 2.0, 2.0, 2.0, 2.0


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


def _radial_ld(flat, A, B):
    """amp prod_g f_g(r2_g) between the rows of A and B in longdouble, with the per-term (d log f / d r2_g) and the scaled
    squared distances D2_t = (a_t - b_t)^2 / metric_t."""
    axis, group, lm = list(flat["axis"]), list(flat["group"]), list(flat["log_metric"])
    k = np.full((len(A), len(B)), np.exp(LD(flat["log_amp"])), dtype=LD)
    D2 = []
    for t in range(len(axis)):
        d = A[:, axis[t]].astype(LD)[:, None] - B[:, axis[t]].astype(LD)[None, :]
        D2.append(d * d / np.exp(LD(lm[t])))
    dlog = {}
    for g in sorted(set(group)):
        ts = [t for t in range(len(axis)) if group[t] == g]
        f, dl = _radial(int(flat["family"]), sum(D2[t] for t in ts))
        k = k * f
        for t in ts:
            dlog[t] = dl
    return k, dlog, D2


def task_factor_ld(theta, n_tasks):
    """(K_t, [dK_t / dtheta_k in packed order]) in longdouble: K_t = L L^T, L_pq = exp(theta_k), k = p (p + 1) / 2 + q,
    dK_t / dtheta_pq = L_pq (e_p L_q^T + L_q e_p^T)."""
    L = np.zeros((n_tasks, n_tasks), dtype=LD)
    for p in range(n_tasks):
        for q in range(p + 1):
            L[p, q] = np.exp(LD(theta[p * (p + 1) // 2 + q]))
    dK = []
    for p in range(n_tasks):
        for q in range(p + 1):
            D = np.zeros((n_tasks, n_tasks), dtype=LD)
            D[p, :] += L[p, q] * L[:, q]
            D[:, p] += L[p, q] * L[:, q]
            dK.append(D)
    return L @ L.T, dK


def factor_ld(flat, A, B):
    """The single-column factor of a flattened kernel between the rows of A and B in longdouble, and its parameter
    derivatives [d/dlog_a, d/dlog_b] or [dK_t[t, t'] / dtheta_k ...]; (None, []) without a factor.  Task coordinates
    that are not tasks give NaN (as the device)."""
    env, task = flat.get("env"), flat.get("task")
    if env is not None:
        ax, la, lb = env
        c0, c1 = np.exp(LD(la)), np.exp(LD(lb))
        zz = A[:, ax].astype(LD)[:, None] * B[:, ax].astype(LD)[None, :]
        return c0 + c1 * zz, [np.full(zz.shape, c0, dtype=LD), c1 * zz]
    if task is not None:
        ax, nT, theta = task
        Kt, dKt = task_factor_ld(theta, nT)
        ia, ib = _task_index(A[:, ax], nT), _task_index(B[:, ax], nT)
        bad = (ia < 0)[:, None] | (ib < 0)[None, :]
        sel = np.ix_(np.maximum(ia, 0), np.maximum(ib, 0))
        F = Kt[sel]
        F[bad] = np.nan
        return F, [D[sel] for D in dKt]
    return None, []


def _task_index(t, n):
    t = np.asarray(t, dtype=np.float64)
    ok = (t >= 0) & (t < n) & (t == np.floor(t))
    return np.where(ok, np.where(ok, t, 0), -1).astype(int)


def kernel_terms_ld(flat, X):
    """k(X, X) and dk/dtheta in the device's order, in longdouble: theta = [log_amp, log_metric_t ...] then, with the
    environment factor, [log_a, log_b], with the task factor the n_kt packed entries of L.  Radial part R (amp
    included): dR/dlog_amp = R, dR/dlog_metric_t = -R dlog f(r2_g)/dr2 (x_t - x'_t)^2 / metric_t; each is multiplied by
    the factor F, and the factor's own derivatives are R dF/dtheta (env: R c0, R c1 z z'; task: R dK_t[t, t']/dtheta)."""
    X = np.asarray(X, dtype=np.float64)
    k, dlog, D2 = _radial_ld(flat, X, X)
    grads = [k] + [-k * dlog[t] * D2[t] for t in range(len(D2))]
    F, dF = factor_ld(flat, X, X)
    if F is None:
        return k, grads
    return k * F, [g * F for g in grads] + [k * d for d in dF]


def grad_reference(flat, X, Xinv, z, noise_var, gemm=None):
    """(g_ref, bound) in the device's layout (n_terms + 2 entries, + 2 with the environment factor, + n_kt with the task
    factor, the noise entry last) from the device's X^ = L^-1 and z^.  The task entries are contracted on the host
    from the per-pair sums G_ab = sum_{t_i = a, t_j = b} A_ij R_ij; their bound gains that contraction's rounding,
    (2 n_tasks) u sum_ab |G_ab| |dK_t[a, b]|."""
    gemm = gemm or _gemm_numpy
    X = np.asarray(X, dtype=np.float64)
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
    if flat.get("task") is not None:
        ax, nT, theta = flat["task"]
        R, _, _ = _radial_ld(flat, X, X)
        ti = _task_index(X[:, ax], nT)
        onehot = (ti[:, None] == np.arange(nT)[None, :]).astype(LD)
        Gab = np.abs((onehot.T @ (A * R) @ onehot).astype(np.float64))
        _, dKt = task_factor_ld(theta, nT)
        nterm = len(flat["axis"]) + 1
        for k, D in enumerate(dKt):
            bnd[nterm + k] += C_GRAD * 2 * nT * U * np.sum(Gab * np.abs(D.astype(np.float64))) / 2
    g[-1] *= noise_var
    bnd[-1] *= noise_var
    return g, bnd


# ---- predictive gradients ----------------------------------------------------------------------------------------------
def kernel_ld(flat, A, B):
    """k(A, B) of a flattened kernel, factor included, in longdouble (A, B float64 rows as the device reads them)."""
    k, _, _ = _radial_ld(flat, np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64))
    F, _ = factor_ld(flat, np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64))
    return k if F is None else k * F


def predict_grad_reference(flat, X, Xinv, z, Xs, lower=None, upper=None, y_std=None, gemm=None):
    """(dmu, dvar, bound_mu, bound_var), each (m, d), of gpk_predict_grad restated in longdouble from the device's
    X^ = L^-1 and z^ (cov_reference's way): alpha = X^T z^, w = X^T (X^ k*), and for candidate x*, scaled
    xn = (x* - lower) / (upper - lower) in fp64 as the device scales it,
        dmu_a  = y_std / (upper_a - lower_a) sum_j alpha_j dk_j/dxn_a
        dvar_a = y_std^2 / (upper_a - lower_a) (dk**/dxn_a - 2 sum_j w_j dk_j/dxn_a)
    with k_j = R_j F_j: dk_j/dxn_a = F_j dR_j/dxn_a on the radial axes, R_j c1 z_j on the environment axis (and
    dk**/dz* = 2 amp c1 z*), exactly 0 on the task axis.  Bound per entry (the same scaling):
        C_PGRAD [(N + n_terms + 16) u sum_j |dk_j| (|alpha_j| + 2 |w_j|) + sum_j |dk_j| (|dalpha_j| + 2 |dw_j|)
                 + 8 u |dk**|]
    with dalpha = gamma_N |X^T| |z^| (alpha = Q z^) and dw = (2 gamma_N + (n_terms + 16) u) |X^T| (|X^| |k*|) (the two
    products and the device's own K* entries), the error alpha^ and w^ carry, as grad_reference carries it."""
    gemm = gemm or _gemm_numpy
    X = np.asarray(X, dtype=np.float64)
    Xs = np.asarray(Xs, dtype=np.float64)
    N, d = X.shape
    m = Xs.shape[0]
    Xn = Xs if lower is None else (Xs - lower) / (upper - lower)
    span = np.ones(d) if lower is None else (np.asarray(upper, dtype=np.float64) - lower)
    ys = 1.0 if y_std is None else float(y_std)
    nt = len(flat["axis"])
    alpha = exact_matmul(Xinv.T, z[:, None], gemm)[:, 0]
    R, dlog, D2 = _radial_ld(flat, Xn, X)
    F, _ = factor_ld(flat, Xn, X)
    Ks = R if F is None else R * F
    ah, al = split2(exact_matmul(Xinv, Ks.T.astype(np.float64), gemm))
    w = exact_matmul(Xinv.T, ah, gemm) + gemm(Xinv.T, al).astype(LD)        # (N, m)
    absX = np.abs(Xinv)
    dal = gamma(N) * (absX.T @ np.abs(z))
    dw = (2 * gamma(N) + (nt + 16) * U) * gemm(absX.T, gemm(absX, np.abs(Ks.T.astype(np.float64))))
    Fm = np.ones_like(R) if F is None else F
    dk = [np.zeros((m, N), dtype=LD) for _ in range(d)]
    axis, lm = list(flat["axis"]), list(flat["log_metric"])
    for t in range(nt):
        diff = Xn[:, axis[t]].astype(LD)[:, None] - X[:, axis[t]].astype(LD)[None, :]
        dk[axis[t]] = dk[axis[t]] + Fm * R * dlog[t] * 2 * diff / np.exp(LD(lm[t]))
    dkss = np.zeros((m, d), dtype=LD)
    env = flat.get("env")
    if env is not None:
        ax, la, lb = env
        c1 = np.exp(LD(lb))
        dk[ax] = R * c1 * X[:, ax].astype(LD)[None, :]
        dkss[:, ax] = 2 * np.exp(LD(flat["log_amp"])) * c1 * Xn[:, ax].astype(LD)
    dmu, dvar = np.zeros((m, d)), np.zeros((m, d))
    bmu, bvar = np.zeros((m, d)), np.zeros((m, d))
    for a in range(d):
        s = LD(ys) / LD(span[a])
        dmu[:, a] = ((dk[a] @ alpha.astype(LD)) * s).astype(np.float64)
        dvar[:, a] = ((dkss[:, a] - 2 * np.sum(dk[a] * w.T, axis=1)) * s * LD(ys)).astype(np.float64)
        adk = np.abs(dk[a].astype(np.float64))
        aw, aal = np.abs(w.T.astype(np.float64)), np.abs(alpha.astype(np.float64))
        cm = (N + nt + 16) * U * (adk @ aal) + adk @ dal
        cv = (N + nt + 16) * U * 2 * np.sum(adk * aw, axis=1) + 2 * np.sum(adk * dw.T, axis=1) \
            + 8 * U * np.abs(dkss[:, a].astype(np.float64))
        bmu[:, a] = C_PGRAD * cm * ys / span[a]
        bvar[:, a] = C_PGRAD * cv * ys * ys / span[a]
    return dmu, dvar, bmu, bvar


# ---- the hyper sampler's log-likelihood (gpk_hy_eval) ------------------------------------------------------------------
def cholesky_ld(K):
    """Lower Cholesky factor of a longdouble matrix in longdouble (None when a pivot is not positive)."""
    K = np.array(K, dtype=LD)
    n = K.shape[0]
    L = np.zeros_like(K)
    for j in range(n):
        s = K[j:, j] - L[j:, :j] @ L[j, :j]
        if not s[0] > 0:
            return None
        L[j, j] = np.sqrt(s[0])
        L[j + 1:, j] = s[1:] / L[j, j]
    return L


def forward_ld(L, r):
    z = np.zeros(L.shape[0], dtype=LD)
    for i in range(L.shape[0]):
        z[i] = (r[i] - L[i, :i] @ z[:i]) / L[i, i]
    return z


def hy_loglik_reference(flat, X, y, mean, diag_add, n_tasks=0):
    """dict(ll, bound, first_order) of the log-likelihood gpk_hy_eval computes for one theta, or None when the reference's
    own K is not positive definite.  gpk_hyper_lnpost returns only ll, so the device's L^ cannot be read back: the bound
    is first order, stated from the reference's K, L and alpha = K^-1 (y - mean) in longdouble.  With ll(K) =
    -r^T K^-1 r / 2 - log det K / 2 - n log(2 pi) / 2, a perturbation dK moves it by (alpha^T dK alpha - tr(K^-1 dK)) / 2
    to first order, so
        |ll_dev - ll_ref| <= C_HY ( [sum_ij |K^-1|_ij E_ij + sum_ij |alpha_i| E_ij |alpha_j|] / 2
                                    + (n + 8) u (sum_i |log L_ii| + z^T z) )
        E = (gamma_{n+1} + 2 gamma_n) |L| |L^T| + E_build
    where gamma_{n+1} |L| |L^T| is the backward error of the column-by-column Cholesky (Higham, Thm 10.3), 2 gamma_n
    |L| |L^T| that of the forward solve taken onto K ((L + dL)(L + dL)^T), and E_build = (n_terms + 2 n_tasks + 24) u
    |K| the per-entry error of the inline build (the radial evaluation, amp, the factor's fma or the K_t table the
    kernel forms from theta, and the diagonal fl(sqrt(yerr^2 + tiny))^2); the last term is the rounding of the sums
    of z^2 and log L_ii.  first_order = ||K^-1||_2 ||E||_F, which must be small (the test asserts <= 0.1) for the
    neglected second-order terms not to matter."""
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[0]
    K = kernel_ld(flat, X, X)
    K[np.diag_indices(n)] += LD(diag_add)
    L = cholesky_ld(K)
    if L is None:
        return None
    r = np.asarray(y, dtype=np.float64).astype(LD) - LD(mean)
    z = forward_ld(L, r)
    Linv = np.linalg.inv(L.astype(np.float64))
    Kinv = exact_matmul(Linv.T, Linv)
    alpha = (Kinv @ r).astype(np.float64)
    logL = np.log(np.diag(L))
    ll = -np.sum(z * z) / 2 - np.sum(logL) - LD(n) * np.log(2 * LD(np.pi)) / 2
    aL = np.abs(L.astype(np.float64))
    E = (gamma(n + 1) + 2 * gamma(n)) * (aL @ aL.T) \
        + (len(flat["axis"]) + 2 * n_tasks + 24) * U * np.abs(K.astype(np.float64))
    aK = np.abs(Kinv.astype(np.float64))
    bound = C_HY * ((np.sum(aK * E) + np.abs(alpha) @ E @ np.abs(alpha)) / 2
                    + (n + 8) * U * float(np.sum(np.abs(logL)) + np.sum(z * z)))
    first = float(np.linalg.norm(aK, 2) * np.linalg.norm(E))
    return dict(ll=ll, bound=float(bound), first_order=first)


# ---- posterior covariance --------------------------------------------------------------------------------------------
def cov_reference(Xinv, Ks, Kss, z, mean, ys2=1.0, y_mean=0.0, y_std=1.0, gemm=None):
    """dict(cov (unclipped, fp64), cov_bound, mu, mu_bound) from the device's X^, z^ and the kernel blocks
    K* (m, N) and K** (m, m); K** as a vector (m,) gives the variances (m,) instead of the covariance."""
    gemm = gemm or _gemm_numpy
    N = Xinv.shape[0]
    V = exact_matmul(Xinv, Ks.T, gemm)                    # (N, m)
    W = gemm(np.abs(Xinv), np.abs(Ks.T))
    if np.ndim(Kss) == 1:                                 # K** given as its diagonal: the variances alone
        cov = ((Kss.astype(LD) - np.sum(V * V, axis=0)) * LD(ys2)).astype(np.float64)
        cb = C_COV * (N + 16) * U * (np.abs(Kss) + np.sum(W * W, axis=0)) * ys2
    else:
        Vh, Vl = split2(V)
        VtV = exact_matmul(Vh.T, Vh, gemm) + (gemm(Vh.T, Vl) + gemm(Vl.T, Vh)).astype(LD)
        cov = ((Kss.astype(LD) - VtV) * LD(ys2)).astype(np.float64)
        cb = C_COV * (N + 16) * U * (np.abs(Kss) + gemm(W.T, W)) * ys2
    ah, al = split2(exact_matmul(Xinv.T, z[:, None], gemm))         # a = X^T z
    mu_n = exact_matmul(Ks, ah, gemm)[:, 0] + gemm(Ks, al)[:, 0].astype(LD) + LD(mean)
    mu = (mu_n * LD(y_std) + LD(y_mean)).astype(np.float64)
    mb = C_COV * (N + 16) * U * ((W.T @ np.abs(z)) + abs(mean)) * y_std + 2 * U * np.abs(mu)
    return dict(cov=cov, cov_bound=cb, mu=mu, mu_bound=mb)
