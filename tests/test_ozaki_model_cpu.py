"""CPU checks of tests/ozaki_model.py, the exact model of the int8 variance contraction that the GPU tests
(test_gpu_ozaki_exact.py) hold the kernel to bit for bit: it is tied to the split already pinned in
tools/ozaki_study.py, its accuracy against an extended-precision reference is bounded and recorded, and equality with
it detects kernel defects that the 1e-10 parity tolerance lets through."""
import os
import sys

import numpy as np
import scipy.linalg as spla

from oracle import robo_oracle as O
from tests import ozaki_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import ozaki_study as Z                                       # noqa: E402

U = 2.0 ** -53


def _problem(N, D, Mc, seed, log_amp):
    """L^-1 of a Matern-5/2 GP with noise 1e-3 (fp64, scipy) and K* of Mc candidates: the operands of scoring."""
    rng = np.random.RandomState(seed)
    X, Xs = rng.rand(N, D), rng.rand(Mc, D)
    theta = np.concatenate(([log_amp], rng.uniform(-0.5, 0.5, D)))
    k = O.make_kernel("matern52", D, theta)
    K = k.get_value(X)
    K[np.diag_indices_from(K)] += 1e-3 + 1.25e-12
    L = spla.cholesky(K, lower=True)
    P = spla.solve_triangular(L, np.eye(N), lower=True)
    return P, k.get_value(Xs, X), float(np.exp(log_amp))


def test_digits_and_V_equal_the_pinned_split_bit_for_bit():
    rng = np.random.RandomState(3)
    n, m = 300, 70
    P = np.tril(rng.randn(n, n) * np.exp(rng.uniform(-8, 3, (n, 1))))
    P[17] = 0.0                                                   # all-zero row: exponent 0
    amp = 1.7
    Ks = rng.uniform(0.0, amp, (m, n))
    eP = M.oz_exponent(np.abs(P).max(axis=1))
    QP, eP_ref = Z.split256(P, 7, axis=1)
    np.testing.assert_array_equal(eP, eP_ref.ravel())
    np.testing.assert_array_equal(M.digits(P, eP[:, None]), np.stack(QP))
    V_ref, pairs = Z.ozaki_matmul(P, Ks.T, 7, amp, base=256)
    assert pairs == 28
    np.testing.assert_array_equal(M.V(P, Ks, amp), V_ref)


def test_fma_is_correctly_rounded():
    """The model's fused multiply-add against exact rational arithmetic, on random operands, ties, cancellation and
    products that underflow."""
    rng = np.random.RandomState(9)
    x = rng.randn(4000) * np.exp2(rng.randint(-30, 30, 4000))
    y = rng.randn(4000) * np.exp2(rng.randint(-30, 30, 4000))
    z = rng.randn(4000) * np.exp2(rng.randint(-60, 60, 4000))
    z[:500] = -x[:500] * y[:500]                                        # cancellation
    x[500:600], y[500:600] = 1.0 + 2.0 ** -52, 1.0 - 2.0 ** -53         # products just off representable
    x[600:700], y[600:700], z[600:700] = 3e-160, 2e-160, 1e-320         # subnormal range
    x[700:800] = y[700:800]                                             # squares, as in the epilogue
    r = M.fma(x, y, z)
    for i in range(len(x)):
        assert r[i] == M._fma_exact(x[i], y[i], z[i]), i
    assert np.any(r != x * y + z)                                       # the test has teeth


def test_tile_reduction_order_is_the_documented_one():
    # part_ssq of one tile against a plain loop written from the contract in gpk_ozaki.cuh
    rng = np.random.RandomState(5)
    n, m = 128, 9
    P = np.tril(rng.randn(n, n))
    Ks = rng.rand(m, n)
    r = M.contract(P, Ks, 1.0)
    x = M.V(P, Ks, 1.0)
    for c in range(m):
        s = 0.0
        for w in range(8):
            cg = [M._fma_exact(x[16 * w + g + 8, c], x[16 * w + g + 8, c], x[16 * w + g, c] * x[16 * w + g, c])
                  for g in range(8)]
            s += ((cg[0] + cg[1]) + (cg[2] + cg[3])) + ((cg[4] + cg[5]) + (cg[6] + cg[7]))
        assert r["part_ssq"][0, c] == s


def test_model_variance_error_is_within_the_split_bound():
    """Accuracy of the int8 path itself, against an 80-bit reference of k** - ||P k*||^2 with the same fp64 P.

    Per entry V_i = sum_k P_ik K_ck (k <= i): the digits are exact to half a unit of 2^(e - 56) per operand, |P_ik| <
    2^(eP_i - 1), |K_ck| < 2^(eK - 1), so one product is off by at most 2^(eP_i + eK - 57) (1 + 2^-56); the 28-pair
    triangle drops the levels s + t >= 7, at most 6 128^2 2^-72 (1 + 2^-6) 2^(eP_i + eK) = 3.05 2^(eP_i + eK - 57) per k.
    Hence |dV_i| <= 4.1 (i + 1) 2^(eP_i + eK - 57) + 8 u sum_k |P_ik K_ck| (the 7 fp64 additions of the fold, u =
    2^-53), and |dvar| <= sum_i (2 |V_i| |dV_i| + dV_i^2) + (N + 3) u sum_i V_i^2 + u k** (squares, the sums over rows
    and row blocks, the subtraction).

    Observed on this C2-like problem (N = 1024, D = 16, 128 candidates): the error is at most 8.3e-4 of the bound; the
    scaled error |dvar| / max(var, 1e-6 k**) is 1.9e-14 for the int8 path, 2.0e-14 for the split alone (exact level
    sums, fold and squares in 80 bits) and 2.3e-14 for the plain fp64 product P K*^T.  The split costs no accuracy
    against fp64 here, and the path sits four orders of magnitude inside the 1e-10 the parity tests allow."""
    P, Ks, amp = _problem(1024, 16, 128, 11, 0.0)
    N = P.shape[0]
    r = M.contract(P, Ks, amp)
    var = M.finish(r["part_ssq"], amp)
    Pl, Kl = P.astype(np.longdouble), Ks.astype(np.longdouble)
    Vl = Pl @ Kl.T
    var_ref = amp - (Vl * Vl).sum(axis=0)
    err = np.abs(var.astype(np.longdouble) - var_ref).astype(np.float64)
    eP, eK = r["eP"], r["eK"]
    V = P @ Ks.T
    absdot = np.abs(P) @ np.abs(Ks).T
    dV = 4.1 * (np.arange(N) + 1.0)[:, None] * np.ldexp(1.0, eP + eK - 57)[:, None] + 8 * U * absdot
    bound = (2 * np.abs(V) * dV + dV * dV).sum(axis=0) + (N + 3) * U * (V * V).sum(axis=0) + U * amp
    assert np.all(err <= bound), (err / bound).max()
    assert (err / bound).max() < 0.05
    den = np.maximum(var_ref.astype(np.float64), 1e-6 * amp)
    scaled = err / den
    # the split alone: exact level sums, folded and squared in 80 bits
    QP, QK = M.digits(P, eP[:, None]), M.digits(Ks, eK)
    acc = M.level_sums(QP, QK).astype(np.longdouble)
    vs = sum(acc[l] * np.longdouble(2.0) ** (-8 * (l + 2)) for l in range(M.S))
    vs = vs * (np.longdouble(2.0) ** (eP + eK).astype(np.longdouble))[:, None]
    split_err = np.abs(amp - (vs * vs).sum(axis=0) - var_ref).astype(np.float64) / den
    fp64_err = np.abs(amp - np.einsum("ij,ij->j", V, V) - var_ref).astype(np.float64) / den
    assert scaled.max() < 1e-11 and split_err.max() < 1e-11 and fp64_err.max() < 1e-11
    print("scaled variance error: int8 path %.2e, split alone %.2e, fp64 product %.2e; error / bound <= %.1e"
          % (scaled.max(), split_err.max(), fp64_err.max(), (err / bound).max()))


def test_equality_detects_defects_the_tolerance_misses():
    """Kernel defects injected into the model on the shape of test_int8_scoring_edge_shapes (N = 640, D = 5, M = 512).
    Every one changes part_ssq, so bit equality with the model catches it, while the first two move the scaled
    variance error by ~1e-11 and stay inside the 1e-10 parity tolerance."""
    P, Ks, amp = _problem(640, 5, 512, 640 * 7 + 5, 0.2)
    ref = M.contract(P, Ks, amp)["part_ssq"]
    var_ref = M.finish(ref, amp)

    def slice6_is_slice5(QK):
        QK = QK.copy()
        QK[6] = QK[5]
        return QK

    def slice6_chunks_swizzled(QK):
        QK = QK.copy()
        m, NP = QK.shape[1:]
        QK[6] = QK[6].reshape(m, NP // 64, 4, 16)[:, :, [1, 0, 3, 2], :].reshape(m, NP)
        return QK

    def kblock_lost_in_slices_5_6(QK):
        QK = QK.copy()
        QK[5:, :, 64:128] = 0.0
        return QK

    def level6_dropped(acc):
        acc = acc.copy()
        acc[6] = 0.0
        return acc

    scaled = {}
    for name, kw in (("slice6_is_slice5", dict(defect_digits=slice6_is_slice5)),
                     ("slice6_chunks_swizzled", dict(defect_digits=slice6_chunks_swizzled)),
                     ("level6_dropped", dict(defect_acc=level6_dropped)),
                     ("kblock_lost_in_slices_5_6", dict(defect_digits=kblock_lost_in_slices_5_6))):
        part = M.contract(P, Ks, amp, **kw)["part_ssq"]
        assert not np.array_equal(part, ref), name
        var = M.finish(part, amp)
        scaled[name] = np.max(np.abs(var - var_ref) / np.maximum(var_ref, 1e-6 * amp))
    assert scaled["slice6_is_slice5"] < 1e-10 and scaled["slice6_chunks_swizzled"] < 1e-10, scaled
    print(scaled)


def test_finish_sums_row_blocks_in_order_and_clips():
    part = np.array([[1e-17, 0.25, np.nan], [0.5, 0.75, 0.0], [1.0, 1.0, 0.0]])
    var = M.finish(part, 2.0, y_std=2.0)
    assert var[0] == (2.0 - ((1e-17 + 0.5) + 1.0)) * 4.0
    assert var[1] == np.finfo(np.float64).eps                     # 2 - 2 = 0, clipped
    assert np.isnan(var[2])
