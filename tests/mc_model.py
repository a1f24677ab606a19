"""Numpy restatement of the sampling-based entropy search kernels (robo_b200/csrc/gpk_esmc.cuh) — TEST INFRASTRUCTURE
ONLY.

Every product and sum follows the kernels' stated order; numpy's elementwise float64 operations round each once, like
the kernels' __dmul_rn / __dadd_rn.  Given the device's draws F, the counts equal gpk_mc_pmin_kernel's bit for bit.  The
draws themselves are restated with numpy's log and cos / sin (the device uses log and sincospi), so they agree to a few
ulp, not bit for bit.  Columns whose two smallest values lie within a few ulp are flagged as near ties, where an input
that differs in the last bits (numpy's LAPACK factor, a restated draw) may pick another winner."""
import numpy as np

from tests.de_model import _philox
from tests.es_model import _cholesky

TAG = 0x4D430001
NOISE_LAST = 10000.0
DBL_MAX = np.finfo(np.float64).max
TIE_ULPS = 8


def draws(seed, nb, nf):
    """F (nb, nf): Philox (q, k, 0, TAG) and Box-Muller, F[k][2q] = r cos(2 pi u2), F[k][2q + 1] = r sin(2 pi u2)."""
    nq = (nf + 1) // 2
    k = np.arange(nb, dtype=np.uint64)[:, None]
    q = np.arange(nq, dtype=np.uint64)[None, :]
    w0, w1, w2, w3 = _philox(seed, q, k, 0, TAG)
    u1 = (((w1 << np.uint64(32)) | w0) >> np.uint64(11)).astype(np.float64) + 1.0
    u1 = u1 * 2.0 ** -53
    u2 = (((w3 << np.uint64(32)) | w2) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    r = np.sqrt(-2.0 * np.log(u1))
    F = np.empty((nb, 2 * nq))
    F[:, 0::2] = r * np.cos(2.0 * np.pi * u2)
    F[:, 1::2] = r * np.sin(2.0 * np.pi * u2)
    return F[:, :nf].copy()


def ladder():
    """The noise of every rung of mc_part.joint_pmin's jitter ladder, in order: 0, 1e-9, ..., 10000.0."""
    out, noise = [0.0], 0.0
    while True:
        if noise == 0.0:
            noise = 1e-10
        if noise == NOISE_LAST:
            return out
        noise = noise * 10.0
        out.append(noise)


def factorise(A):
    """The left-looking factor of A + noise I on the ladder -> (L, rung); LinAlgError past the last rung.  Only the
    lower triangle of A is read."""
    for r, noise in enumerate(ladder()):
        S = np.array(A, dtype=np.float64)
        if r > 0:
            S[np.diag_indices_from(S)] = S[np.diag_indices_from(S)] + noise
        L = _cholesky(S)
        if L is not None:
            return L, r
    raise np.linalg.LinAlgError("Cholesky decomposition failed.")


def funcs(L, F):
    """funcs[a][f] = sum_{k <= a} L[a][k] F[k][f], summed for k = 0, 1, ... from 0.0."""
    nb = L.shape[0]
    out = np.empty((nb, F.shape[1]))
    for a in range(nb):
        s = np.zeros(F.shape[1])
        for k in range(a + 1):
            s = s + L[a, k] * F[k]
        out[a] = s
    return out


def count(M, fu):
    """Arg-min counts over the columns (f, p) of fl(M[a][p] + funcs[a][f]) -> (counts (nb,), near-tie columns)."""
    nb = M.shape[0]
    vals = M[:, None, :] + fu[:, :, None]                    # (nb, nf, np)
    arg = np.argmin(vals, axis=0)
    counts = np.bincount(arg.ravel(), minlength=nb)
    if nb > 1:
        two = np.partition(vals, 1, axis=0)[:2]
        gap = two[1] - two[0]
        scale = np.maximum(np.abs(two[0]), np.abs(two[1]))
        near = int(np.count_nonzero(gap <= TIE_ULPS * np.spacing(scale)))
    else:
        near = 0
    return counts, near


def pmin_from_counts(counts, total):
    p = counts.astype(np.float64) / float(total)
    p[p < 1e-70] = 1e-70
    return p


def joint_pmin(m, V, F):
    """gpk_mc_pmin: m (nb,) or (nb, np), V (nb, nb), F (nb, nf) -> dict(pmin, counts, near, rung)."""
    m = np.asarray(m, dtype=np.float64)
    if m.ndim == 1:
        m = m[:, None]
    L, rung = factorise(V)
    counts, near = count(m, funcs(L, F))
    return dict(pmin=pmin_from_counts(counts, F.shape[1] * m.shape[1]), counts=counts, near=near, rung=rung)


def H_of(logP, lmb):
    """H = -sum_i exp(logP_i) (logP_i + lmb_i), summed in index order (gpk_esmc_update)."""
    H = 0.0
    for lp, lm in zip(np.ravel(logP), np.ravel(lmb)):
        H += float(np.exp(lp)) * (float(lp) + float(lm))
    return -H


def value_of(pmin, lmb, H):
    acc = 0.0
    for p, lm in zip(pmin, np.ravel(lmb)):
        acc = acc + p * (np.log(p) + lm)
    v = acc + H
    return -DBL_MAX if (np.isnan(v) or v == np.inf) else float(v)


def candidate(Mb, Vb, W, F, v, sigma, sn2, lmb, H):
    """One candidate of gpk_mc_pmin_kernel from its variance v and clipped covariance sigma (nb,) to zb
    -> dict(value, pmin, counts, near, rung)."""
    W = np.ravel(W)
    iv = 1.0 / (v - sn2)
    nc = sigma * iv
    dm = nc * np.sqrt(v + 1e-10)
    M = Mb[:, None] + dm[:, None] * W[None, :]
    A = Vb + -(nc[:, None] * sigma[None, :])
    L, rung = factorise(A)
    counts, near = count(M, funcs(L, F))
    p = pmin_from_counts(counts, F.shape[1] * W.size)
    return dict(value=value_of(p, lmb, H), pmin=p, counts=counts, near=near, rung=rung)
