"""CPU checks of tests/fit_reference.py: the exact product against mpmath and longdouble matmul, the bounds on a
numpy emulation of the device's fp64 algorithms (blocked Cholesky with explicit diagonal-block inverses, the recursive
block inversion over build_nodes, the split-K append, the gradient from Q = P^T), and the defect table of DESIGN.md
section 2: defects a kernel bug would produce, injected into those correct results, fail the new checks where the
older tolerances of tests/test_gpu_parity.py pass."""
import numpy as np
import pytest
import scipy.linalg as spla

from oracle import robo_oracle as O
from tests import fit_reference as R

pytestmark = pytest.mark.skipif(not R.have_longdouble(), reason="np.longdouble is not an extended type here")

BM = R.BM


# ---- exact product ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,k,n", [(1, 1, 1), (3, 7, 5), (24, 24, 24), (9, 17, 2)])
def test_exact_matmul_against_mpmath(m, k, n):
    mpmath = pytest.importorskip("mpmath")
    rng = np.random.RandomState(m * 100 + k)
    A = rng.randn(m, k) * np.exp(rng.randn(m, k) * 8)          # entries over ~20 orders of magnitude
    B = rng.randn(k, n) * np.exp(rng.randn(k, n) * 8)
    got, err = R.exact_matmul(A, B, with_err=True)
    mpmath.mp.prec = 300
    for i in range(m):
        for j in range(n):
            ref = mpmath.fsum(mpmath.mpf(float(A[i, t])) * mpmath.mpf(float(B[t, j])) for t in range(k))
            dev = abs(mpmath.mpf(got[i, j].astype(np.float64)) + mpmath.mpf(float(got[i, j] - LDf(got[i, j]))) - ref)
            assert dev <= mpmath.mpf(float(err[i, j])), (i, j, dev, err[i, j])


def LDf(x):
    return np.longdouble(np.float64(x))


@pytest.mark.parametrize("N", [1, 2, 31, 128, 129, 256])
def test_exact_matmul_against_longdouble_matmul(N):
    rng = np.random.RandomState(N)
    A = rng.randn(N, N)
    B = rng.randn(N, N + 3)
    got, err = R.exact_matmul(A, B, with_err=True)
    ref = A.astype(np.longdouble) @ B.astype(np.longdouble)
    ref_err = N * 2.0 ** -63 * (np.abs(A) @ np.abs(B))           # longdouble matmul's own rounding
    assert np.all(np.abs((got - ref).astype(np.float64)) <= err + ref_err)
    # and the fp64 product is not exact: the reference resolves what it gets wrong
    assert np.any(A @ B != got.astype(np.float64)) or N < 8


def test_exact_matmul_with_a_gemm_that_reorders():
    """any summation order gives the same slice products: a blocked GEMM summing k in reverse gives the same bits"""
    rng = np.random.RandomState(3)
    A, B = rng.randn(40, 300), rng.randn(300, 20)

    def rev(X, Y):
        return sum(X[:, t:t + 7] @ Y[t:t + 7] for t in reversed(range(0, X.shape[1], 7)))
    np.testing.assert_array_equal(R.exact_matmul(A, B), R.exact_matmul(A, B, gemm=rev))


# ---- numpy emulations of the device's algorithms ---------------------------------------------------------------------
def problem(N=700, D=16, noise=1e-3, seed=700):
    X, y, _, theta, _ = O.synthetic_problem(N, D, 1, seed_train=seed)
    K = O.make_kernel("matern52", D, theta).get_value(X)
    K[np.diag_indices_from(K)] += noise
    return X, y - np.mean(y), K, theta


def blocked_cholesky(K, defect=None):
    """Right-looking 128-block Cholesky, the panel by the explicit inverse of the diagonal tile (as the device).
    'update_twice': at step 1 the first 16 columns of the panel update tile (5, 4) once more."""
    N = K.shape[0]
    S = np.tril(K).copy()
    L = np.zeros_like(K)
    nb = (N + BM - 1) // BM
    for k in range(nb):
        a, b = k * BM, min((k + 1) * BM, N)
        Skk = S[a:b, a:b]
        L[a:b, a:b] = np.linalg.cholesky(np.tril(Skk) + np.tril(Skk, -1).T)
        Xkk = spla.solve_triangular(L[a:b, a:b], np.eye(b - a), lower=True)
        L[b:, a:b] = S[b:, a:b] @ Xkk.T
        for i in range(k + 1, nb):
            i0, i1 = i * BM, min((i + 1) * BM, N)
            for j in range(k + 1, i + 1):
                j0, j1 = j * BM, min((j + 1) * BM, N)
                S[i0:i1, j0:j1] -= L[i0:i1, a:b] @ L[j0:j1, a:b].T
                if defect == "update_twice" and (k, i, j) == (1, 5, 4):
                    S[i0:i1, j0:j1] -= L[i0:i1, a:a + 16] @ L[j0:j1, a:a + 16].T
    return L


def tree_inverse(L):
    """L^-1 as build_linv: diagonal tiles inverted, then for every node X21 = -X22 (L21 X11)."""
    N = L.shape[0]
    nb = (N + BM - 1) // BM
    X = np.zeros_like(L)
    for k in range(nb):
        s = slice(k * BM, min((k + 1) * BM, N))
        X[s, s] = spla.solve_triangular(L[s, s], np.eye(s.stop - s.start), lower=True)
    _, nodes = R.build_nodes(0, nb)
    for lo, mid, hi, _ in nodes:
        a, b, c = lo * BM, mid * BM, min(hi * BM, N)
        X[b:c, a:b] = -(X[b:c, b:c] @ (L[b:c, a:b] @ X[a:b, a:b]))
    return X


def append_rows(L, X, K, N1, defect=None):
    """gpk_fit_append on the emulated factor of the first N1 rows: L_row = K[b, :N1] P11^T summed over 512-column
    chunks, the Schur complement, the last block, P[b, :N1] = -P_bb (L_row P11).  'drop_chunk': the last chunk of
    L_row's contraction is lost."""
    N = K.shape[0]
    L2, X2 = np.zeros((N, N)), np.zeros((N, N))
    L2[:N1, :N1], X2[:N1, :N1] = L[:N1, :N1], X[:N1, :N1]
    Kb = K[N1:, :N1]
    Lrow = np.zeros((N - N1, N1))
    for j in range(N1 // BM):
        cols = slice(j * BM, (j + 1) * BM)
        chunks = list(range(0, (j + 1) * BM, 512))
        if defect == "drop_chunk" and len(chunks) > 1:
            chunks = chunks[:-1]
        for k0 in chunks:
            k1 = min(k0 + 512, (j + 1) * BM)
            Lrow[:, cols] += Kb[:, k0:k1] @ X[cols, k0:k1].T
    S = K[N1:, N1:] - Lrow @ Lrow.T
    Lbb = np.linalg.cholesky(S)
    Pbb = spla.solve_triangular(Lbb, np.eye(N - N1), lower=True)
    L2[N1:, :N1], L2[N1:, N1:] = Lrow, Lbb
    X2[N1:, N1:] = Pbb
    X2[N1:, :N1] = -(Pbb @ (Lrow @ X[:N1, :N1]))
    return L2, X2


def device_grad(X, z, Xin, theta, noise, Q=None, drop_tile=None):
    """The gradient of gpk_nll_grad in fp64 from Q (default X^T): alpha = Q z, K^-1 = Q Q^T, g = -1/2 sum A dK.
    drop_tile = (r, c): the 32-row trace tile r of 128-column block c is missing."""
    Q = Xin.T if Q is None else Q
    a = Q @ z
    A = np.outer(a, a) - Q @ Q.T
    flat = dict(family=0, log_amp=theta[0], axis=list(range(X.shape[1])), group=[0] * X.shape[1],
                log_metric=list(theta[1:]))
    _, grads = R.kernel_terms_ld(flat, X)
    W = A.copy()
    if drop_tile is not None:
        r, c = drop_tile
        blk = np.zeros_like(W, dtype=bool)
        blk[32 * r:32 * r + 32, 128 * c:128 * c + 128] = True
        blk &= np.tril(np.ones_like(blk))
        W[blk | blk.T] = 0.0
    g = [-0.5 * np.sum(W * dK.astype(np.float64)) for dK in grads]
    g.append(-0.5 * np.trace(W) * noise)
    return np.array(g), flat


def old_linv_ok(Xin, Lref):
    return np.abs(Xin @ Lref - np.eye(Lref.shape[0])).max() < 1e-9


def old_factor_ok(L, Lref):
    return np.abs(L - Lref).max() <= 2e-12 * np.abs(Lref).max()


# ---- the checks hold on correct results --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emulated():
    Xd, r, K, theta = problem()
    L = blocked_cholesky(K)
    Xin = tree_inverse(L)
    z = spla.solve_triangular(L, r, lower=True)
    return dict(Xd=Xd, r=r, K=K, theta=theta, L=L, Xin=Xin, z=z, Lref=spla.cholesky(K, lower=True))


def test_checks_pass_on_the_emulated_algorithms(emulated):
    e = emulated
    rf, _, _ = R.factor_check(e["L"], e["K"], e["Xin"])
    rs, _, _ = R.solve_check(e["L"], e["z"], e["r"])
    lc = R.linv_checks(e["L"], e["Xin"])
    assert rf <= 1 and rs <= 1, (rf, rs)
    assert lc["diag"][0] <= 1 and lc["node"][0] <= 1 and lc["upper_zero"], lc
    ld = 2 * np.sum(np.log(np.diag(e["L"])))
    assert R.logdet_check(ld, e["L"])[0] <= 1
    ll = -0.5 * e["z"] @ e["z"] - 0.5 * ld - 0.5 * len(e["z"]) * np.log(2 * np.pi)
    assert R.loglik_check(ll, ld, e["z"])[0] <= 1
    g, flat = device_grad(e["Xd"], e["z"], e["Xin"], e["theta"], 1e-3)
    g_ref, bnd = R.grad_reference(flat, e["Xd"], e["Xin"], e["z"], 1e-3)
    assert np.all(np.abs(g - g_ref) <= bnd)


def test_tree_nodes_match_the_device_table():
    """build_nodes restated: every block below the diagonal is produced by exactly one node; unbalanced for nb = 5"""
    for nb in (1, 2, 3, 5, 9, 17, 48):
        _, nodes = R.build_nodes(0, nb)
        seen = np.zeros((nb, nb), dtype=int)
        for lo, mid, hi, _ in nodes:
            assert mid == lo + (hi - lo + 1) // 2
            seen[mid:hi, lo:mid] += 1
        assert np.array_equal(seen, np.tril(np.ones((nb, nb), dtype=int), -1))


# ---- the defect table ------------------------------------------------------------------------------------------------
def defect_rows(e):
    """[(defect, old check passes?, new check ratio)] on the N = 700, D = 16 problem."""
    rows = []
    Lref = e["Lref"]
    # one 128 x 128 tile of L^-1 (block row 4, column 1) off by a relative 1e-12
    X = e["Xin"].copy()
    X[512:640, 128:256] *= 1 + 1e-12
    lc = R.linv_checks(e["L"], X)
    rows.append(("L^-1 tile (4, 1) x (1 + 1e-12)", old_linv_ok(X, Lref), max(lc["diag"][0], lc["node"][0])))
    # one tile of L off by a relative 1e-11 (its entries are below 0.15: the older 2e-12 max|L| does not see it)
    L = e["L"].copy()
    L[384:512, 128:256] *= 1 + 1e-11
    rows.append(("L tile (3, 1) x (1 + 1e-11)", old_factor_ok(L, Lref), R.factor_check(L, e["K"], e["Xin"])[0]))
    # one trailing-update tile applied twice for one 16-column panel
    try:                                # far too large for noise 1e-3: the last diagonal block stops being PD
        L = blocked_cholesky(e["K"], defect="update_twice")
        row = (old_factor_ok(L, Lref), R.factor_check(L, e["K"], e["Xin"])[0])
    except np.linalg.LinAlgError:
        row = (False, np.inf)
    rows.append(("trailing tile (5, 4) updated twice by 16 columns of panel 1",) + row)
    # the append with one split-K chunk dropped (N1 = 640 -> 700)
    try:                                # the Schur complement of the last block is no longer PD
        L2, X2 = append_rows(e["L"], e["Xin"], e["K"], 640, defect="drop_chunk")
        row = (old_append_ok(L2, e), R.factor_check(L2, e["K"], X2)[0])
    except np.linalg.LinAlgError:
        row = (False, np.inf)
    rows.append(("append: last 512-column chunk of L_row dropped",) + row)
    # Q != P^T in one tile (seen through alpha and K^-1 in the gradient; the gradient bound is looser than the factor's,
    # a relative 1e-12 sits at 0.09 of it)
    Q = e["Xin"].T.copy()
    Q[128:256, 512:640] *= 1 + 1e-10
    g, flat = device_grad(e["Xd"], e["z"], e["Xin"], e["theta"], 1e-3, Q=Q)
    g_ref, bnd = R.grad_reference(flat, e["Xd"], e["Xin"], e["z"], 1e-3)
    rows.append(("Q tile (1, 4) != P^T x (1 + 1e-10)", old_grad_ok(g, e), float(np.max(np.abs(g - g_ref) / bnd))))
    # one 32-row tile of the gradient trace missing
    g, _ = device_grad(e["Xd"], e["z"], e["Xin"], e["theta"], 1e-3, drop_tile=(9, 2))
    rows.append(("gradient trace tile (rows 288..319, block 2) missing", old_grad_ok(g, e),
                 float(np.max(np.abs(g - g_ref) / bnd))))
    return rows


def old_append_ok(L2, e):
    return np.abs(L2 - e["Lref"]).max() <= 1e-11 * np.abs(e["Lref"]).max()


def old_grad_ok(g, e):
    g0, _ = device_grad(e["Xd"], e["z"], e["Xin"], e["theta"], 1e-3)
    return bool(np.all(np.abs(g - g0) <= 1e-8 * np.abs(g0) + 1e-8 * np.abs(g0).max()))


def test_defect_table(emulated):
    """every defect is caught by the new checks (ratio > 1); the ones the older tolerances miss are the point"""
    rows = defect_rows(emulated)
    for name, old_ok, r in rows:
        print("%-62s old check passes: %-5s new ratio: %.3g" % (name, old_ok, r))
        assert r > 1, name
    assert sum(old_ok for _, old_ok, _ in rows) >= 3


def test_append_emulation_passes(emulated):
    e = emulated
    L2, X2 = append_rows(e["L"], e["Xin"], e["K"], 640)
    assert R.factor_check(L2, e["K"], X2)[0] <= 1
    lc = R.linv_checks(L2, X2)
    assert lc["diag"][0] <= 1 and lc["node"][0] <= 1
