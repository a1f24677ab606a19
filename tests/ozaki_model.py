"""Exact CPU model of the int8 variance contraction (gpk_ozaki.cuh, gpk_oz_vargemm_kernel) and of the finish kernel's
variance (gpk_kernels.cuh, gpk_finish_kernel).

Fed the same fp64 operands, it reproduces the device's row exponents, per-row-block partial sums part_ssq and the
variance BIT FOR BIT, because every step of the device computation is either exact or a fixed sequence of roundings:
  * digits: e = oz_exponent(max |row|), X = rint(v 2^56) with v = x 2^-e, the bytes of X + 0x0080..80 minus 128
    (oz_digits: 7 balanced base-256 digits, most significant first);
  * level sums: acc[lvl] = sum_{s + t = lvl} <Pq[s][i][:], Kq[t][c][:]> over k < 128 (ib + 1), the block-lower
    triangle the kernel reads; exact int32 sums on the device, exact fp64 sums of integers here (|sum| <= 7 K 128^2 <
    2^53, and < 2^31 or the device's int32 accumulator would wrap: asserted);
  * the epilogue order of gpk_ozaki.cuh (its comment states it as a contract, see tile_colsum below) and the
    finish kernel's order (finish below).
Anyone who changes the kernel's digit rule or reduction order changes this file in the same commit.

Candidates are independent (one exponent eK for all of Ks), so a sample of rows of Ks is modelled by passing just
those rows: contract(P, Ks[idx], amp)["part_ssq"] equals the device's part_ssq[:, idx].
"""
import numpy as np

S = 7                 # digits per operand
TM = 128              # rows of a tile (row block of P)
_BIAS = sum(128 << (8 * j) for j in range(S))


def oz_exponent(amax):
    """oz_exponent of gpk_ozaki.cuh, elementwise: frexp's exponent + 1, one more when the mantissa is >= 127.49 / 128;
    0 for a zero maximum."""
    amax = np.asarray(amax, dtype=np.float64)
    m, ex = np.frexp(amax)
    e = ex.astype(np.int64) + 1 + (m * 128.0 >= 127.49)
    return np.where(amax > 0.0, e, 0).astype(np.int64)


def digits(A, e):
    """The S balanced base-256 digits of A 2^-e (e broadcast against A) as float64 integers in [-128, 127],
    shape (S,) + A.shape, most significant first (oz_digits / oz_digit_of)."""
    v = np.ldexp(np.asarray(A, dtype=np.float64), -np.asarray(e, dtype=np.int64))
    X = np.rint(v * 72057594037927936.0).astype(np.int64)                 # 2^56, round half to even
    Y = X + _BIAS
    return np.stack([(((Y >> (8 * (S - 1 - s))) & 0xFF) - 128).astype(np.float64) for s in range(S)])


def pad(P, Ks):
    """Zero padding of gpk_oz_contract / the fitted layout: P to NP x NP, Ks to NP columns (rows of Ks need none: the
    padded candidates are not read back)."""
    n = P.shape[0]
    NP = -(-n // TM) * TM
    Pp = np.zeros((NP, NP))
    Pp[:n, :n] = P
    Kp = np.zeros((Ks.shape[0], NP))
    Kp[:, :n] = Ks
    return Pp, Kp


def level_sums(QP, QK):
    """acc[lvl] (S x rows x cands) = sum_{s + t = lvl} QP[s] QK[t]^T for digit stacks QP (S x rows x k), QK (S x cands
    x k): float64 GEMMs on integers, exact."""
    acc = np.zeros((S, QP.shape[1], QK.shape[1]))
    for s in range(S):
        prod = QP[s] @ QK[:S - s].transpose(0, 2, 1)                     # (S - s) x rows x cands
        acc[s:] += prod
    assert np.all(np.abs(acc) < 2.0 ** 31), "a level sum leaves the int32 accumulator"
    return acc


def fold(acc):
    """V / 2^(eP + eK) of one tile from its level sums: v = 0, then v = v + acc[lvl] 2^(-8 (lvl + 2)) for lvl = 6 .. 0
    (the product is a power-of-two scaling, so the kernel's fma rounds once, like this sum)."""
    v = np.zeros(acc.shape[1:])
    for lvl in range(S - 1, -1, -1):
        v = v + acc[lvl] * np.ldexp(1.0, -8 * (lvl + 2))
    return v


def _fma_exact(x, y, z):
    from fractions import Fraction
    r = Fraction(x) * Fraction(y) + Fraction(z)
    return float(r.numerator / r.denominator) if r else 0.0   # int / int is correctly rounded, subnormals included


def fma(x, y, z):
    """x y + z with one rounding (the device's fused multiply-add), elementwise.  Boldo and Melquiond's emulation
    ("Emulation of FMA and correctly rounded sums", IEEE TC 2008): exact product (Veltkamp / Dekker), TwoSum with z,
    the two low parts added with rounding to odd, one final rounding to nearest.  Where a splitting step could
    underflow or overflow, the element is computed exactly with fractions."""
    x, y, z = np.broadcast_arrays(*(np.asarray(a, dtype=np.float64) for a in (x, y, z)))
    with np.errstate(over="ignore", invalid="ignore"):
        p = x * y

        def split(a):
            c = 134217729.0 * a                                             # 2^27 + 1
            hi = c - (c - a)
            return hi, a - hi
        xh, xl = split(x)
        yh, yl = split(y)
        e = ((xh * yh - p) + xh * yl + xl * yh) + xl * yl                    # p + e = x y exactly
        s = z + p
        b = s - z
        t = (z - (s - b)) + (p - b)                                         # s + t = z + p exactly
        w = t + e
        b2 = w - t
        err = (t - (w - b2)) + (e - b2)
        even = (w.view(np.int64) & 1) == 0
        w = np.where((err != 0) & even, np.nextafter(w, np.copysign(np.inf, err)), w)      # round to odd
        r = s + w
    big, small = 2.0 ** 500, 2.0 ** -450
    risky = ~(np.isfinite(x) & np.isfinite(y) & np.isfinite(z))
    risky |= (np.abs(x) > big) | (np.abs(y) > big) | (np.abs(z) > big)
    risky |= ((np.abs(x) < small) & (x != 0)) | ((np.abs(y) < small) & (y != 0)) | ((np.abs(p) < small ** 2) & (p != 0))
    risky |= (np.abs(z) < small ** 2) & (z != 0)
    if risky.any():
        r = np.array(r, copy=True)
        for i in zip(*np.nonzero(risky)):
            r[i] = _fma_exact(x[i], y[i], z[i]) if np.isfinite(x[i] * y[i] + z[i]) else x[i] * y[i] + z[i]
    return r


def tile_colsum(acc, e_rows, eK):
    """The epilogue of one 128-row tile: x = v 2^(eP[row] + eK); per consumer warp w (rows 16 w .. 16 w + 15) and row
    pair g = 0 .. 7, c_g = fma(x(16 w + g + 8), x(16 w + g + 8), x(16 w + g)^2) (the compiler contracts the kernel's
    col += x * x); the butterfly gives ((c0 + c1) + (c2 + c3)) + ((c4 + c5) + (c6 + c7)); the column sum adds the
    warps w = 0 .. 7 in sequence from 0.0."""
    v = fold(acc)
    x = (v * np.ldexp(1.0, np.asarray(e_rows, dtype=np.int64) + int(eK))[:, None]).reshape(8, 2, 8, -1)   # [w][b][g]
    c = fma(x[:, 1], x[:, 1], x[:, 0] * x[:, 0])                        # [w][g]
    bw = ((c[:, 0] + c[:, 1]) + (c[:, 2] + c[:, 3])) + ((c[:, 4] + c[:, 5]) + (c[:, 6] + c[:, 7]))
    s = np.zeros(acc.shape[2])
    for w in range(8):
        s = s + bw[w]
    return s


def contract(P, Ks, amp, defect_digits=None, defect_acc=None):
    """gpk_oz_contract: -> dict(eP (n,), eK, part_ssq (nb x m)).  P: n x n (only its block-lower triangle enters the
    level sums; its full rows set the row exponents), Ks: m x n with |entries| <= amp.
    defect_digits(QK) / defect_acc(acc) return altered K* digits / level sums of a tile: the self-test injects kernel
    defects through them."""
    P, Ks = np.asarray(P, dtype=np.float64), np.asarray(Ks, dtype=np.float64)
    n = P.shape[0]
    Pp, Kp = pad(P, Ks)
    NP = Pp.shape[0]
    eP = oz_exponent(np.max(np.abs(Pp), axis=1))
    eK = int(oz_exponent(float(amp)))
    QK = digits(Kp, eK)
    if defect_digits is not None:
        QK = defect_digits(QK)
    part = np.empty((NP // TM, Ks.shape[0]))
    for ib in range(NP // TM):
        rows = slice(ib * TM, (ib + 1) * TM)
        kmax = (ib + 1) * TM
        QP = digits(Pp[rows, :kmax], eP[rows, None])
        acc = level_sums(QP, QK[:, :, :kmax])
        if defect_acc is not None:
            acc = defect_acc(acc)
        part[ib] = tile_colsum(acc, eP[rows], eK)
    return dict(eP=eP[:n], eK=eK, part_ssq=part)


def V(P, Ks, amp):
    """V = P Ks^T (n x m) through the same digits and fold, before squaring (the whole lower triangle of P)."""
    P, Ks = np.asarray(P, dtype=np.float64), np.asarray(Ks, dtype=np.float64)
    eP = oz_exponent(np.max(np.abs(P), axis=1))
    eK = int(oz_exponent(float(amp)))
    v = fold(level_sums(digits(P, eP[:, None]), digits(Ks, eK)))
    return v * np.ldexp(1.0, eP + eK)[:, None]


def finish(part_ssq, kss, y_std=None):
    """The variance of gpk_finish_kernel: ssq = sum over ib = 0 .. nb - 1 in sequence from 0.0, var = kss - ssq, times
    y_std^2 under the output transform, clipped at DBL_EPSILON (NaN stays NaN)."""
    ssq = np.zeros(part_ssq.shape[1])
    for p in range(part_ssq.shape[0]):
        ssq = ssq + part_ssq[p]
    var = kss - ssq
    if y_std is not None:
        var = var * (y_std * y_std)
    return np.where(var < np.finfo(np.float64).eps, np.finfo(np.float64).eps, var)
