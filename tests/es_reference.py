"""Extended-precision reference of the entropy-search candidate path (gpk_es_update's U, gpk_es_sigma_kernel's sigma,
gpk_es_dh_kernel's dH), and fp64 emulations of the two kernels in their own summation order (CPU only).

Reference.  The kernel is the george oracle's tree (oracle/george_oracle.py) evaluated in np.longdouble (80-bit x87 on
x86-64, eps 1.1e-19): squared distances, radial functions and products in longdouble, on inputs scaled in float64 as
robo_oracle.gp_predict scales them (zero_one_normalization), with george's diagonal fl(sqrt(fl(yerr^2 + tiny)))^2.
    U_ref = K^-1 K(X, zb)       fp64 Cholesky, then iterative refinement with the residuals in longdouble
    sigma_ref_j(x) = (k(zb_j, x) - k(x, X) U_ref[:, j]) * y_std^2      (longdouble; unclipped: the clip is applied by
                                                                        the caller, see sigma_bound)
Refinement converges by a factor kappa(K) eps_64 per step, to about kappa(K) eps_ld relative: for the kappa <= 1e6
of the cases here that is 1e-13 of |U|, three orders below the fp64 error it is used to measure.

Bounds.
    sigma:  |sigma_dev - sigma_ref| <= [gamma eps (|k(zb_j, x)| + sum_n |k(x, X_n)| |U_nj|) + sum_n |k(x, X_n)| |dU_nj|]
                                       * y_std^2
            gamma = N + 16: the N fma steps of the sequential sum (each at most one rounding of the running sum, bounded
            by the sum of the term magnitudes), 8 ulp for each fp64 kernel value (a product of <= 2 radial factors of
            exp, sqrt and a short distance sum) and the subtraction and the scaling; dU = U_dev - U_ref, the measured
            error of the U the kernel reads, carried through the sum exactly by the triangle inequality.
    U:      |U_dev - U_ref|_col <= 4 N eps kappa_2(K) max|U_ref[:, j]|: the normwise forward error of a backward-stable
            solve (Cholesky, triangular inverse, two triangular products), each column on its own.
    dH:     dh_bound below.
"""
import math

import numpy as np

from oracle import george_oracle as G
from oracle import robo_oracle as O

LD = np.longdouble
EPS = float(np.finfo(np.float64).eps)
TILE = 256                                   # GPK_ES_THREADS: training rows per tile of gpk_es_sigma_kernel


def have_longdouble():
    return float(np.finfo(np.longdouble).eps) <= 1e-18


def kernel_ld(k, A, B):
    """k(A, B) of a george_oracle kernel tree in longdouble; A (n1, D), B (n2, D) float64 inputs.  The factor kernels of
    tests/env_kernel_model.py (EnvKernel) and tests/task_kernel_model.py (TaskKernel) are understood too."""
    if isinstance(k, G.Product):
        return kernel_ld(k.k1, A, B) * kernel_ld(k.k2, A, B)
    if isinstance(k, G.Sum):
        return kernel_ld(k.k1, A, B) + kernel_ld(k.k2, A, B)
    if isinstance(k, G.ConstantKernel):
        return np.full((len(A), len(B)), np.exp(LD(k.log_constant)), dtype=LD)
    if isinstance(k, G._RadialKernel):
        r2 = np.zeros((len(A), len(B)), dtype=LD)
        for a, md in zip(k.axes, k._axis_metric()):
            d = A[:, a].astype(LD)[:, None] - B[:, a].astype(LD)[None, :]
            r2 += d * d / LD(md)
        return k._f(r2)
    from tests import env_kernel_model as EM
    from tests import task_kernel_model as TM
    if isinstance(k, EM.EnvKernel):                 # c0 + c1 z z'
        a = int(k.axes[0])
        return np.exp(LD(k.log_a)) + np.exp(LD(k.log_b)) * (A[:, a].astype(LD)[:, None] * B[:, a].astype(LD)[None, :])
    if isinstance(k, TM.TaskKernel):                # K_t[t, t'], K_t = L L^T in longdouble, NaN off the tasks
        from tests import fit_reference as FR
        a = int(k.axes[0])
        Kt, _ = FR.task_factor_ld(k.theta, k.n_tasks)
        ia, ib = TM.task_index(A[:, a], k.n_tasks), TM.task_index(B[:, a], k.n_tasks)
        out = Kt[np.ix_(np.maximum(ia, 0), np.maximum(ib, 0))]
        out[(ia < 0)[:, None] | (ib < 0)[None, :]] = np.nan
        return out
    raise TypeError("kernel_ld: unsupported kernel %r" % type(k))


def scale_inputs(st, X):
    X = np.asarray(X, dtype=np.float64)
    if st["normalize_input"]:
        return O.zero_one_normalization(X, st["lower"], st["upper"])[0]
    return X


def out_scale(st):
    return float(st["y_std"]) ** 2 if st["normalize_output"] else 1.0


class Reference(object):
    """The extended-precision state of one fitted oracle model (robo_oracle.gp_fit's st)."""

    def __init__(self, st):
        self.st = st
        gp = st["gp"]
        self.kernel = gp.kernel
        self.X = np.asarray(gp._x, dtype=np.float64)              # scaled training inputs
        diag = float(np.sqrt(gp._yerr2[0] + np.exp(gp.white_noise)) ** 2)
        self.K = kernel_ld(self.kernel, self.X, self.X)
        self.K[np.diag_indices_from(self.K)] += LD(diag)
        self.K64 = self.K.astype(np.float64)
        self.L64 = np.linalg.cholesky(self.K64)
        self.kappa = float(np.linalg.cond(self.K64))
        self.ys2 = out_scale(st)

    def _solve64(self, R):
        import scipy.linalg as spla
        return spla.cho_solve((self.L64, True), R.astype(np.float64))

    def solve(self, B, steps=4):
        """K^-1 B with longdouble residuals (iterative refinement)."""
        B = np.asarray(B, dtype=LD)
        Xs = self._solve64(B).astype(LD)
        for _ in range(steps):
            Xs = Xs + self._solve64(B - self.K @ Xs).astype(LD)
        return Xs

    def u(self, zb):
        """(U_ref (N, nb) longdouble, scaled zb) for raw representer points zb (nb, D)."""
        zs = scale_inputs(self.st, zb)
        return self.solve(kernel_ld(self.kernel, self.X, zs)), zs

    def sigma(self, U, zs, Xs):
        """Unclipped sigma_ref (m, nb) and the term magnitudes |k(zb, x)| + |k(x, X)| |U| (m, nb), both times y_std^2,
        and |k(x, X)| (m, N) for the U error term."""
        xs = scale_inputs(self.st, Xs)
        Kxs = kernel_ld(self.kernel, xs, self.X)
        kzx = kernel_ld(self.kernel, xs, zs)
        s = (kzx - Kxs @ U) * LD(self.ys2)
        mag = (np.abs(kzx) + np.abs(Kxs) @ np.abs(U)) * LD(self.ys2)
        return s, mag, np.abs(Kxs).astype(np.float64)

    def u_bound(self, U):
        col = 4.0 * U.shape[0] * EPS * self.kappa * np.max(np.abs(U.astype(np.float64)), axis=0)
        return np.broadcast_to(col, U.shape)

    def sigma_bound(self, mag, absK, dU):
        N = absK.shape[1]
        return (N + 16) * EPS * mag.astype(np.float64) + (absK @ np.abs(dU)) * self.ys2


def sigma_check(got, ref, bound):
    """Per-entry check of a device (or emulated) sigma against the unclipped reference.  Above eps + bound: within the
    bound; below eps - bound: exactly eps (the clip); within the bound of eps: either side of the clip.  Returns the
    largest error-to-bound ratio over the unclipped entries and a boolean mask of the failing entries."""
    ref = ref.astype(np.float64)
    hi = ref > EPS + bound
    lo = ref < EPS - bound
    mid = ~hi & ~lo
    bad = np.zeros(got.shape, dtype=bool)
    bad[hi] = np.abs(got[hi] - ref[hi]) > bound[hi]
    bad[lo] = got[lo] != EPS
    bad[mid] = ~((got[mid] == EPS) | (np.abs(got[mid] - ref[mid]) <= bound[mid]))
    ratio = float(np.max(np.abs(got[hi] - ref[hi]) / bound[hi])) if hi.any() else 0.0
    return ratio, bad


# ---- fp64 emulations in the kernels' order -----------------------------------------------------------------------
def fma(a, b, c):
    """fl(a b + c), the product and sum taken in longdouble (64-bit significand) and rounded once to fp64; differs
    from a true fma only by a rare double rounding."""
    return (np.asarray(a, dtype=LD) * np.asarray(b, dtype=LD) + np.asarray(c, dtype=LD)).astype(np.float64)


def fma_exact(a, b, c):
    """fl(a b + c) correctly rounded (a true fma), elementwise.  The longdouble result of fma() is rounded a second time
    to fp64; that double rounding can only go wrong where the longdouble value is exactly halfway between two fp64
    numbers (rounding to 64 bits is monotone and every fp64 midpoint is a 64-bit number).  Those entries are recomputed
    exactly with fractions.Fraction, so the result is the true fma's bits everywhere."""
    from fractions import Fraction
    a, b, c = np.broadcast_arrays(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64),
                                  np.asarray(c, dtype=np.float64))
    v = np.asarray(a, dtype=LD) * np.asarray(b, dtype=LD) + np.asarray(c, dtype=LD)
    out = v.astype(np.float64)
    rest = np.abs((v - out.astype(LD)).astype(np.float64))
    sp = np.spacing(np.abs(out))
    tie = np.isfinite(out) & (rest > 0) & ((rest == sp / 2) | (rest == sp / 4))
    out = np.array(out)
    for idx in zip(*np.nonzero(tie)):
        exact = Fraction(float(a[idx])) * Fraction(float(b[idx])) + Fraction(float(c[idx]))
        lo = float(exact)                    # Fraction -> float rounds to nearest, ties to even
        out[idx] = lo
    return out


def device_u(L64, Kxz):
    """U as gpk_es_update builds it: P = L^-1 in fp64, then P^T (P K(X, zb)) in fp64."""
    import scipy.linalg as spla
    P = spla.solve_triangular(L64, np.eye(L64.shape[0]), lower=True)
    return P.T @ (P @ Kxz)


def sigma_emulate(Kxs, kzx, U, ys2, defect=None):
    """gpk_es_sigma_kernel in fp64: Kxs (m, N), kzx (m, nb), U (N, nb) fp64.  acc = fma(k_n, U_n, acc) in index
    order over 256-row tiles, then clip((kzx - acc) * ys2, eps).  Defects:
        'drop_tile_last'  row 255 of every tile skipped (cnt - 1);
        'u_row_off'       the first row of every tile after the first reads U one row back;
        'scale_ystd'      scaled by y_std instead of y_std^2;
        'clip_first'      the clip applied before the scale."""
    m, N = Kxs.shape
    acc = np.zeros((m, U.shape[1]))
    for n0 in range(0, N, TILE):
        cnt = min(TILE, N - n0)
        if defect == "drop_tile_last":
            cnt -= 1
        for q in range(cnt):
            r = n0 + q
            ur = U[r - 1] if (defect == "u_row_off" and q == 0 and n0 > 0) else U[r]
            acc = fma(Kxs[:, r][:, None], ur[None, :], acc)
    d = kzx - acc
    if defect == "clip_first":
        return np.maximum(d, EPS) * ys2
    v = d * (math.sqrt(ys2) if defect == "scale_ystd" else ys2)
    return np.where(v < EPS, EPS, v)


# ---- dH ------------------------------------------------------------------------------------------------------------
def host_h(logP, lmb):
    """H as gpk_es_update sums it: -sum_i exp(logP_i) (logP_i + lmb_i) in index order."""
    H = 0.0
    for p, l in zip(np.ravel(logP), np.ravel(lmb)):
        H += math.exp(p) * (p + l)
    return -H


def _warp_dot(A, b):
    """A (nb, T) . b (T,) row by row as the warps of gpk_es_dh_kernel: lane l fma-accumulates x = l, l + 32, ...; then
    the xor-shuffle tree (offsets 16, 8, 4, 2, 1); lane 0's value."""
    nb, T = A.shape
    lanes = np.zeros((nb, 32))
    for x0 in range(0, T, 32):
        k = min(32, T - x0)
        lanes[:, :k] = fma(A[:, x0:x0 + k], b[None, x0:x0 + k], lanes[:, :k])
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    return lanes[:, 0]


def dh_emulate(state, v, sigma, Hs=None, defect=None):
    """gpk_es_dh_kernel in fp64 for one in-bounds candidate: state as tests/es_model.dh_folded takes it plus H
    (gpk_es_update's host value).  Defects:
        'hs_diag_twice'    the Hs diagonal folded twice (2 H[a][a]);
        'skip_w_256'       the columns p >= 256 of W skipped (the thread loop runs once);
        'max_per_column'   the max fall-back decided per column instead of over every column."""
    from tests.es_model import fold
    nb = sigma.size
    a, b = np.tril_indices(nb)
    Hs = fold(state["dlogPdMudMu"]) if Hs is None else Hs
    if defect == "hs_diag_twice":
        Hs = Hs.copy()
        Hs[:, a == b] *= 2.0
    W = np.asarray(state["W"], dtype=np.float64).ravel()
    lmb = np.asarray(state["lmb"], dtype=np.float64).ravel()
    H = state["H"] if "H" in state else host_h(state["logP"], lmb)
    npn = W.size
    with np.errstate(all="ignore"):
        iv = np.float64(1.0) / np.float64(v - state["sn2"])
        sq = np.sqrt(np.float64(v) + 1e-10)
        dm = (sigma * iv) * sq
        dv = -((sigma[a] * iv) * sigma[b])
        dmm = dm[a] * dm[b]
        g = _warp_dot(state["dlogPdMu"], dm)
        base = np.asarray(state["logP"], dtype=np.float64).ravel() + fma(0.5, _warp_dot(Hs, dmm),
                                                                          _warp_dot(state["dlogPdSigma"], dv))
        L = fma(g[:, None], W[None, :], base[:, None])                       # (nb, np)
        mx = L[0].copy()
        for i in range(1, nb):
            mx = np.where((mx >= L[i]) | np.isnan(mx), mx, L[i])
        se = np.zeros(npn)
        for i in range(nb):
            se = se + np.exp(L[i] - mx)
        lse = mx + np.log(se)
        inf_col = np.isinf(lse)
        sel = np.where(inf_col if defect == "max_per_column" else np.any(inf_col), mx, lse)
        col = np.zeros(npn)
        for i in range(nb):
            l = L[i] - sel
            col = fma(np.exp(l), l + lmb[i], col)
        vals = col + H
        acc = np.zeros(256)
        for p in range(npn):
            if defect == "skip_w_256" and p >= 256:
                break
            acc[p % 256] += vals[p]
        s2 = 128
        while s2 > 0:
            acc[:s2] = acc[:s2] + acc[s2:2 * s2]
            s2 //= 2
        dH = acc[0] / npn
    return -np.finfo(float).max if (math.isnan(dH) or dH == math.inf) else float(dH)


def _dh_terms(state, v, sigma):
    """base_i, g_i of the kernel (numpy order) and the bounds d_i, e_i on their rounding (see dh_bound)."""
    from tests.es_model import fold
    nb = sigma.size
    T = nb * (nb + 1) // 2
    a, b = np.tril_indices(nb)
    lp = np.asarray(state["logP"], dtype=np.float64).ravel()
    with np.errstate(all="ignore"):
        iv = np.float64(1.0) / np.float64(v - state["sn2"])
        sq = np.sqrt(np.float64(v) + 1e-10)
        dm = (sigma * iv) * sq
        dv = -((sigma[a] * iv) * sigma[b])
        dmm = dm[a] * dm[b]
        Hs = fold(state["dlogPdMudMu"])
        base = lp + (state["dlogPdSigma"].dot(dv) + 0.5 * Hs.dot(dmm))
        g = state["dlogPdMu"].dot(dm)
        d = (T + 40) * EPS * (np.abs(state["dlogPdSigma"]).dot(np.abs(dv)) + 0.5 * np.abs(Hs).dot(np.abs(dmm))
                              + np.abs(lp))
        e = (nb + 40) * EPS * np.abs(state["dlogPdMu"]).dot(np.abs(dm))
    return base, g, d, e


def dh_bound(state, v, sigma, H=None):
    """Bound on |dH_dev - dh_folded(state, v, sigma)| when both are fed the same v and sigma (and the device H).

    dm, dv, dmm, 1 / v_ and sqrt are single IEEE operations in the same order in both, so they agree bit for bit.  The
    rest is derived step by step, each step's constant rounded up:
      - a dot product of T terms, in the kernel's lane partials (T / 32 fma each) and 5-step shuffle tree or in numpy's
        order, is within (T + 5) eps of sum |terms| either way; the two orders together within 2 (T + 5) eps, taken as
        (T + 40) eps for the Sigma and Hs sums and (nb + 40) eps for g (with the 1 / 2 and the add of logP_i folded in):
        d_i = (T + 40) eps (sum |dSig_i| |dv| + 0.5 sum |Hs_i| |dmm| + |logP_i|),  e_i = (nb + 40) eps sum |dMu_i| |dm|;
      - l_ip = base_i + g_i w_p - sel_p: the product and the sum (fma-contracted on the device, not in numpy) add at most
        2 roundings of |base_i| + |g_i w_p| each (4 eps), so lPred is within d_i + e_i |w_p| + 4 eps (|base_i| +
        |g_i w_p|); sel_p = mx_p + log(sum exp(l - mx_p)) moves by at most the largest of those (exp and log within
        1 ulp each of a value <= log nb), hence the factor 2 and the 4 eps |sel_p|:
        dl_p = 2 max_i (d_i + e_i |w_p| + 4 eps (|base_i| + |g_i w_p|)) + 4 eps |sel_p|;
      - the column value sum_i exp(l)(l + lmb) moves by sum_i |d/dl| dl = sum_i exp(l_ip) (|l_ip + lmb_i| + 1) dl_p,
        plus its own rounding: exp within 1 ulp, the product, the add of lmb and the nb-term sum, (nb + 8) eps of
        sum_i exp(l) (|l + lmb| + |l| + 2); and H (C++ in index order against numpy's pairwise sum), within 8 eps of
        |H| + sum_i exp(logP_i) |logP_i + lmb_i|;
      - the mean over p: the per-thread sums of Np / 256 columns and the 8-step tree, (Np / 256 + 10) eps of
        mean |col_p + H|.
    It is a worst case over every rounding at once.  On the device the error sits 1e3 to 1e8 below it (DESIGN.md
    section 2), so the bound is not a measure of the kernel's accuracy, only a ceiling that a wrong term breaks.
    Returns (bound, finite flag)."""
    base, g, d, e = _dh_terms(state, v, sigma)
    nb = sigma.size
    lp = np.asarray(state["logP"], dtype=np.float64).ravel()
    lmb = np.asarray(state["lmb"], dtype=np.float64).ravel()
    W = np.asarray(state["W"], dtype=np.float64).ravel()
    with np.errstate(all="ignore"):
        Lr = base[:, None] + g[:, None] * W[None, :]
        mx = np.max(Lr, axis=0)
        lse = mx + np.log(np.sum(np.exp(Lr - mx), axis=0))
        sel = mx if np.any(np.isinf(lse)) else lse
        dli = d[:, None] + e[:, None] * np.abs(W)[None, :] + 4 * EPS * (np.abs(base)[:, None] + np.abs(g[:, None] * W))
        dl = 2 * np.max(dli, axis=0) + 4 * EPS * np.abs(sel)
        l = Lr - sel
        ex = np.exp(l)
        Hh = -np.sum(np.exp(lp) * (lp + lmb)) if H is None else H
        colerr = np.sum(ex * (np.abs(l + lmb[:, None]) + 1.0), axis=0) * dl \
            + (nb + 8) * EPS * np.sum(ex * (np.abs(l + lmb[:, None]) + np.abs(l) + 2.0), axis=0) \
            + 8 * EPS * (abs(Hh) + np.sum(np.exp(lp) * np.abs(lp + lmb)))
        col = np.sum(ex * (l + lmb[:, None]), axis=0) + Hh
        bound = float(np.mean(colerr) + (W.size / 256 + 10) * EPS * np.mean(np.abs(col)))
    return bound, bool(np.isfinite(bound))


def dh_interval_huge_column(state, v, sigma, p, H):
    """The values dH may take when column p of W is so large (|W_p| ~ 1e300) that the column's lPred = base + g W_p is
    decided by g alone, and the rounding of g decides which entry is the column's maximum.

    The rows of dlogPdMu sum to zero (p_min does not change when every mean moves by the same amount), so where dm is
    nearly constant over the representer points (sigma clipped at eps in most columns, v far above sn2) every g_i is
    rounding noise of size e_i, and g_i W_p is noise of size e_i |W_p| ~ 1e280.  Whichever entry comes out largest has
    l = 0 exactly and the others exp(l) = 0 exactly, so the column is H + lmb_imax (or H + the sum over entries that tie
    bit for bit): a last-bit difference in g moves dH by |lmb| / Np.  Neither the kernel's summation order nor numpy's is
    the right one; dH is simply not determined by its inputs there.

    With u_i = d_i + e_i |W_p| + 4 eps (|base_i| + |g_i W_p|) the bound on the rounding of lPred_i, the entries that can
    be the maximum are A = {i : lPred_i + u_i >= max_j (lPred_j - u_j)}; every other entry lies at least 1e4 below them
    (else None is returned), so its exp(l) is exactly 0.  What the entries of A come out as decides the rest:
      - one of them largest by more than 745: the column is H + lmb_i;
      - several equal to the last bit at a magnitude that absorbs log(count) into sel: each has l = 0, and the column is
        H + the sum of their lmb;
      - several within 745 of each other (g_i exactly 0, say): softmax weights p_i, and the column is
        H + sum p_i lmb_i + sum p_i log p_i, within [min_A lmb - log |A|, max_A lmb].
    So the column lies between H + min(the most negative subset sum of lmb over A, min_A lmb - log |A|) and H + the
    largest subset sum (nonempty subsets), which is exactly H + lmb_i when A = {i}.  The other columns are dh_folded on W without column p, within dh_bound.
    Returns (lo, hi, |A|), or None when the column is not in that regime."""
    from tests.es_model import dh_folded
    base, g, d, e = _dh_terms(state, v, sigma)
    lmb = np.asarray(state["lmb"], dtype=np.float64).ravel()
    W = np.asarray(state["W"], dtype=np.float64).ravel()
    w = W[p]
    with np.errstate(all="ignore"):
        L = base + g * w
        u = d + e * abs(w) + 4 * EPS * (np.abs(base) + np.abs(g * w))
    if not (np.all(np.isfinite(L)) and np.all(np.isfinite(u))):
        return None
    A = L + u >= np.max(L - u)
    if np.any(~A) and np.max(L[~A] + u[~A]) > np.min(L[A] - u[A]) - 1e4:
        return None
    rest = dict(state, W=np.delete(W, p))
    r = dh_folded(rest, v, sigma)
    b, fin = dh_bound(rest, v, sigma, H)
    if not (np.isfinite(r) and fin):
        return None
    n = W.size
    s_rest = r * (n - 1)
    slack = b * (n - 1) + 16 * EPS * (abs(H) + np.sum(np.abs(lmb)) + abs(s_rest))
    la = lmb[A]
    c_lo = min(np.sum(la[la < 0]) if np.any(la < 0) else np.min(la), np.min(la) - math.log(la.size))
    c_hi = np.sum(la[la > 0]) if np.any(la > 0) else np.max(la)
    lo = (s_rest + H + c_lo - slack) / n
    hi = (s_rest + H + c_hi + slack) / n
    return lo, hi, int(A.sum())
