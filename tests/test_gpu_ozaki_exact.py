"""The int8 variance contraction (gpk_oz_vargemm_kernel) against its exact CPU model, tests/ozaki_model.py, BIT FOR BIT.

The digits follow a fixed integer rule, the level sums are exact int32 sums, and the epilogue and the finish kernel
reduce in a fixed order, so the device's row exponents, per-row-block partial sums and variances must equal the model's
exactly.  Equality sees what the 1e-10 parity tolerance cannot: a wrong descriptor or swizzle on the last digit slice,
a dropped digit level, a lost k-block, a tile written twice or never (tests/test_ozaki_model_cpu.py shows the power on
the CPU).  gpk_oz_contract runs the contraction alone on caller-supplied operands; the last test goes through gpk_acq."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from robo_b200 import kernels as K
from tests import ozaki_model as M

pytestmark = pytest.mark.gpu

SCHEDULES = [(cs, persist, grid) for cs in (1, 2, 4) for persist, grid in ((0, 0), (1, 0), (1, 1), (1, 2))]
CODE = {1: 0, 2: 16, 4: 32}


@pytest.fixture(scope="module")
def handle():
    from robo_b200 import _lib
    h = _lib.Handle(0)
    yield h
    h.close()


def _run(h, P, Ks, amp, cs=4, persist=3, grid=0):
    h.set_option("ozcluster", cs)
    h.set_option("ozpersist", persist)
    h.set_option("ozgrid", grid)
    r = h.oz_contract(P, Ks, amp)
    if persist != 3:
        assert int(h.timings()["ozaki_kernel_variant"]) == 1 + 8 * persist + CODE[cs]
    return r


def _assert_matches(r, P, Ks, amp, cols=None):
    cols = np.arange(Ks.shape[0]) if cols is None else cols
    ref = M.contract(P, Ks[cols], amp)
    np.testing.assert_array_equal(r["eP"], ref["eP"])
    assert r["eK"] == ref["eK"]
    np.testing.assert_array_equal(r["part_ssq"][:, cols], ref["part_ssq"])


def _sample(m, rng, chunk=None, extra=96):
    """Candidates the model covers when all of them would cost too much: the first and the last cluster tile (128
    candidates) of every chunk, the ragged tail, and `extra` random ones."""
    chunk = chunk or m
    idx = [np.arange(lo, min(lo + 128, m)) for lo in range(0, m, chunk)]
    idx += [np.arange(max(min(lo + chunk, m) - 128, lo), min(lo + chunk, m)) for lo in range(0, m, chunk)]
    idx.append(rng.choice(m, min(extra, m), replace=False))
    return np.unique(np.concatenate(idx))


def _operands(n, m, seed):
    rng = np.random.RandomState(seed)
    P = np.tril(rng.randn(n, n)) * np.exp(rng.uniform(-3.0, 2.0, (n, 1)))
    amp = 1.3
    Ks = rng.uniform(-0.2, 1.0, (m, n)) * amp
    return P, Ks, amp, rng


# (N, m): 1, 2, 3 and 5 row blocks, 32 and 33 (just above the automatic persistent switch); m ragged around the 32-,
# 128- and 4 x 32-candidate tiles.  At N = 4096 and 4224 the L2 group (24 or 26 candidate blocks) does not divide the
# 32 / 36 candidate blocks.
SHAPES = [(100, 45), (129, 161), (256, 33), (384, 257), (640, 1000), (4096, 900), (4224, 1100)]


@pytest.mark.parametrize("N,m", SHAPES)
def test_contraction_equals_model_for_every_schedule(handle, N, m):
    P, Ks, amp, rng = _operands(N, m, N + m)
    cols = _sample(m, rng) if N > 1024 else None
    cs_ref = None
    for cs, persist, grid in SCHEDULES:
        r = _run(handle, P, Ks, amp, cs, persist, grid)
        if cs_ref is None:
            _assert_matches(r, P, Ks, amp, cols)                 # the model once per shape
            cs_ref = r
        else:
            # every schedule, every candidate: bit-identical to the first, which equals the model
            np.testing.assert_array_equal(r["part_ssq"], cs_ref["part_ssq"], err_msg=str((cs, persist, grid)))
            np.testing.assert_array_equal(r["eP"], cs_ref["eP"])


def test_digit_edge_inputs(handle):
    n, m = 384, 160
    rng = np.random.RandomState(7)
    P = np.tril(rng.randn(n, n))
    specials = {
        130: 127.48 / 128 * 4.0,        # largest mantissa just below the 127.49 / 128 bump
        131: 127.5 / 128 * 2.0,         # just above: one more exponent
        132: 127.49 / 128,              # exactly at the bump
        133: 2.0,                       # exact power of two
        134: -3.75,                     # negative row maximum
        135: 63.7,                      # eP = 7: |P| just below 64, the int8 path's limit
        136: 63.99,                     # ... one more with the bump
        137: 1e-300,                    # very small exponents
        138: 3e-160,                    # squares land in the subnormal range
    }
    for i, v in specials.items():
        P[i, : i + 1] *= abs(v) / np.abs(P[i, : i + 1]).max() * 0.5
        P[i, i // 2] = v
    P[140, :] = 0.0                     # all-zero rows: eP = 0
    P[300, :] = 0.0
    # rounding ties of rint(v 2^56): odd multiples of 2^(e - 57) in a row with e = 0 (row maximum 0.4)
    tie = (2 * rng.randint(0, 2 ** 40, 200) + 1) * 2.0 ** -57 * rng.choice([-1.0, 1.0], 200)
    P[250, :] = 0.0
    P[250, :200] = tie
    P[250, 7] = 0.4
    for amp in (0.75, 127.5 / 128 * 2.0, 2.0):
        eK = int(M.oz_exponent(amp))
        Ks = rng.uniform(-1.0, 1.0, (m, n)) * amp
        Ks[0, :] = amp                                                 # entries equal to amp
        Ks[1, :] = -amp
        Ks[2, ::2] = 2.0 ** (eK - 58)                                  # below 2^(eK - 57): all digits zero
        Ks[3, :] = 1e-30
        Ks[4, :100] = (2 * rng.randint(0, 2 ** 40, 100) + 1) * 2.0 ** (eK - 57)       # ties
        assert not M.digits(Ks[2, ::2], eK).any()
        r = _run(handle, P, Ks, amp)
        _assert_matches(r, P, Ks, amp)
        # the inputs sit where they were meant to: both sides of the bump, eP = 7 and 8, zero rows, tiny exponents
        np.testing.assert_array_equal(r["eP"][[130, 131, 132, 133, 134, 135, 136, 137, 138, 140, 250, 300]],
                                      [3, 3, 2, 3, 3, 7, 8, -995, -528, 0, 0, 0])


def test_accumulator_headroom_at_k_16384(handle):
    """Constant P (lower triangle) and Ks with balanced digits [-126, -128 x 6]: every pair product has the same sign, so
    the level sums of the last rows reach their largest magnitude; level 6 of row 16383 is 16384 x 114176 =
    1 870 659 584, 87 % of 2^31.  The level sums have a closed form, so the model needs no 16384^2 GEMM."""
    n, m = 16384, 128
    amp = 0.988296568627451
    v = -amp
    e = int(M.oz_exponent(amp))
    d = M.digits(np.array(v), e)
    np.testing.assert_array_equal(d, [-126] + [-128] * 6)
    lvl = np.array([sum(d[s] * d[l - s] for s in range(l + 1)) for l in range(M.S)])
    assert lvl[6] == 114176 and lvl[6] * n == 1870659584 and lvl[6] * n < 2 ** 31
    P = np.full((n, n), v)
    for i in range(0, n, 1024):
        P[i:i + 1024] = np.tril(P[i:i + 1024], k=i)
    Ks = np.full((m, n), v)
    r = _run(handle, P, Ks, amp)
    del P
    assert r["eK"] == e and np.all(r["eP"] == e)
    for ib in range(n // M.TM):
        cnt = ib * M.TM + np.arange(M.TM) + 1.0                        # nonzeros of each row of the block
        acc = lvl[:, None, None] * cnt[None, :, None] * np.ones((1, 1, m))
        ref = M.tile_colsum(acc, np.full(M.TM, e), e)
        np.testing.assert_array_equal(r["part_ssq"][ib], ref, err_msg="row block %d" % ib)
    # one row more pads to 16512 > 16384 rows: refused before any operand is read
    small = np.zeros(4)
    out = np.zeros(4)
    eP, eK = np.zeros(4, dtype=np.int32), C.c_int()
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    rc = handle.lib.gpk_oz_contract(handle._h, small.ctypes.data_as(dp), 16385, small.ctypes.data_as(dp), 1, 1.0,
                                    out.ctypes.data_as(dp), eP.ctypes.data_as(ip), C.byref(eK))
    assert rc == 2                                                     # GPK_BAD_ARG


def test_bad_operands_are_refused(handle):
    P, Ks, amp, _ = _operands(130, 40, 1)
    Ks[3, 5] = amp * (1 + 2.0 ** -52)
    with pytest.raises(ValueError):
        handle.oz_contract(P, Ks, amp)
    with pytest.raises(ValueError):
        handle.oz_contract(P, Ks[:, :100], amp)


def _fitted(N, D, seed, transform):
    from robo_b200 import _lib
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    y = np.sin(3 * X.sum(axis=1)) + 0.5
    log_amp = 0.2
    h = _lib.Handle(0)
    h.set_data(X, y)
    f = K.Product(K.ConstantKernel(log_amp, ndim=D), K.Matern52Kernel(np.exp(rng.uniform(-0.5, 0.5, D)), ndim=D)).flatten()
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    if transform:
        h.set_output_transform(True, 0.3, 1.7)
    h.fit(1e-3, float(np.mean(y)))
    return h, X, y, rng, math.exp(log_amp)


def test_contract_leaves_a_fitted_model_untouched():
    from robo_b200 import _lib
    h, X, y, rng, amp = _fitted(300, 4, 21, False)
    Xs = rng.rand(2500, 4)
    before = h.acq(Xs, _lib.ACQ_EI, float(np.min(y)), 0.0, want_values=True, want_moments=True)
    P, Ks, a, _ = _operands(500, 300, 2)
    h.oz_contract(P, Ks, a)
    after = h.acq(Xs, _lib.ACQ_EI, float(np.min(y)), 0.0, want_values=True, want_moments=True)
    h.close()
    for k in ("values", "mu", "var"):
        np.testing.assert_array_equal(after[k], before[k])


@pytest.mark.skipif(os.environ.get("GPK_OZAKI") == "0", reason="GPK_OZAKI=0 runs the fp64 contraction in gpk_acq")
@pytest.mark.parametrize("transform", [False, True])
def test_acq_variance_equals_model_with_and_without_lookahead(transform):
    """The production path: L^-1 from get_linv and K* from kernel_matrix (the same covariance builder and train operand
    as scoring; the model splits that fp64 K* into the digits the int8 builder writes itself) through the model give
    gpk_acq's variances bit for bit, over several chunks with both K* buffers, the look-ahead builder on the side stream
    and the serial schedule, and the output transform."""
    from robo_b200 import _lib
    N, D, m, chunk = 640, 5, 10000, 2048
    h, X, y, rng, amp = _fitted(N, D, 640 + transform, transform)
    Xs = rng.rand(m, D)
    Linv = h.get_linv(N)
    Ks = h.kernel_matrix(Xs, X)
    cols = _sample(m, rng, chunk, extra=256)
    var_ref = M.finish(M.contract(Linv, Ks[cols], amp)["part_ssq"], amp, 1.7 if transform else None)
    h.set_option("chunk", chunk)
    launches = 0
    for overlap in (0, 1):
        h.set_option("overlap", overlap)
        r = h.acq(Xs, _lib.ACQ_EI, float(np.min(y)), 0.0, want_values=True, want_moments=True)
        t = h.timings()
        assert t["launches_ozaki"] >= launches + 5, t                        # one int8 launch per chunk, no fall-back
        launches = t["launches_ozaki"]
        np.testing.assert_array_equal(r["var"][cols], var_ref, err_msg="overlap %d" % overlap)
    h.close()
