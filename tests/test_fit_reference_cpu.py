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


# ---- the single-column factors: environment (Fabolas) and task (MTBO) ---------------------------------------------------
ENV_FLAT = dict(family=0, log_amp=0.2, axis=[0, 1], group=[0, 1], log_metric=[-1.0, -0.5], env=(2, 0.1, -0.3),
                task=None)
TASK_THETA = (-0.2, 0.3, -0.6, 0.1, -0.4, -1.0)


def task_flat(n_tasks=3, theta=TASK_THETA):
    return dict(family=0, log_amp=0.2, axis=[0, 1], group=[0, 1], log_metric=[-1.0, -0.5], env=None,
                task=(2, n_tasks, tuple(theta[:n_tasks * (n_tasks + 1) // 2])))


def factor_data(kind, N, seed=0, n_tasks=3):
    rng = np.random.RandomState(seed)
    X = rng.rand(N, 3)
    if kind == "env":
        X[:, 2] = (1 - rng.rand(N)) ** 2
    else:
        X[:, 2] = rng.randint(0, n_tasks, N)
    y = np.sin(3 * X[:, 0]) + 0.3 * X[:, 2] + 0.1 * rng.randn(N)
    return X, y - np.mean(y)


def _mp_kernel(mpmath, flat, x1, x2, theta):
    """k(x1, x2) in mpmath, theta = [log_amp, log_metric..., factor parameters] (Matern-5/2 per group)."""
    nt = len(flat["axis"])
    k = mpmath.exp(theta[0])
    for g in sorted(set(flat["group"])):
        r2 = mpmath.mpf(0)
        for t in range(nt):
            if flat["group"][t] == g:
                ax = flat["axis"][t]
                r2 += (mpmath.mpf(float(x1[ax])) - mpmath.mpf(float(x2[ax]))) ** 2 / mpmath.exp(theta[1 + t])
        s = mpmath.sqrt(5 * r2)
        k *= (1 + s + s * s / 3) * mpmath.exp(-s)
    fp = theta[1 + nt:]
    if flat["env"] is not None:
        ax = flat["env"][0]
        return k * (mpmath.exp(fp[0]) + mpmath.exp(fp[1]) * mpmath.mpf(float(x1[ax])) * mpmath.mpf(float(x2[ax])))
    ax, nT, _ = flat["task"]
    a, b = int(x1[ax]), int(x2[ax])
    Lm = [[mpmath.exp(fp[p * (p + 1) // 2 + q]) if q <= p else 0 for q in range(nT)] for p in range(nT)]
    return k * mpmath.fsum(Lm[a][q] * Lm[b][q] for q in range(nT))


@pytest.mark.parametrize("kind", ["env", "task"])
def test_factor_terms_against_mpmath(kind):
    """K and every dK/dtheta of kernel_terms_ld, the factor entries included, against mpmath derivatives of the kernel
    written out independently (300-bit, numerical differentiation at that precision)"""
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.prec = 300
    flat = ENV_FLAT if kind == "env" else task_flat()
    X, _ = factor_data(kind, 4, seed=3)
    K, grads = R.kernel_terms_ld(flat, X)
    fp = list(flat["env"][1:]) if kind == "env" else list(flat["task"][2])
    theta0 = [mpmath.mpf(flat["log_amp"])] + [mpmath.mpf(v) for v in flat["log_metric"]] + [mpmath.mpf(v) for v in fp]
    assert len(grads) == len(theta0)
    for i in range(4):
        for j in range(4):
            ref = _mp_kernel(mpmath, flat, X[i], X[j], theta0)
            assert abs(mpmath.mpf(float(K[i, j])) - ref) <= 4e-16 * abs(ref) + 1e-300
            for p in range(len(theta0)):
                def f(v, p=p):
                    th = list(theta0)
                    th[p] = v
                    return _mp_kernel(mpmath, flat, X[i], X[j], th)
                d = mpmath.diff(f, theta0[p])
                got = grads[p][i, j]
                # to longdouble precision (the reference's own rounding): 1e-17 of the largest term
                assert abs(mpmath.mpf(float(got)) + mpmath.mpf(float(got - np.longdouble(float(got)))) - d) \
                    <= 1e-17 * max(abs(ref), 1e-300), (kind, i, j, p)


def test_fma_exact_where_double_rounding_bites():
    """the longdouble fma of es_reference rounds twice; fma_exact must return the correctly rounded bits on the cases
    where that goes wrong, and agree with it everywhere else"""
    from fractions import Fraction
    from tests import es_reference as ER
    t = 2.0 ** -53
    a = np.array([t * (1 + 2.0 ** -17), t * (1 + 2.0 ** -17), 1 + 2.0 ** -30, 3.0])
    b = np.array([1.0, -1.0, 1 + 2.0 ** -30, 1.0 / 3.0])
    c = np.array([1.0, -1.0, -1.0, -1.0])
    got = ER.fma_exact(a, b, c)
    for i in range(len(a)):
        exact = float(Fraction(a[i]) * Fraction(b[i]) + Fraction(c[i]))
        assert got[i] == exact, (i, got[i], exact)
    # the first two: 1 + 2^-53 + 2^-70 is just above a midpoint, rounded to it in longdouble, then to even (1.0)
    assert ER.fma(a[:2], b[:2], c[:2])[0] == 1.0 and got[0] == 1.0 + 2.0 ** -52 and got[1] == -(1.0 + 2.0 ** -52)
    rng = np.random.RandomState(0)
    a, b, c = rng.rand(3, 20000)
    got = ER.fma_exact(a, b, c)
    ref = np.array([float(Fraction(x) * Fraction(y) + Fraction(w)) for x, y, w in zip(a[:2000], b[:2000], c[:2000])])
    assert np.array_equal(got[:2000], ref)


def factor_problem(kind, N=300, seed=11, n_tasks=3):
    flat = ENV_FLAT if kind == "env" else task_flat(n_tasks)
    X, r = factor_data(kind, N, seed, n_tasks)
    K = R.kernel_terms_ld(flat, X)[0].astype(np.float64)
    K[np.diag_indices_from(K)] += 1e-2
    L = np.linalg.cholesky(K)
    Xin = spla.solve_triangular(L, np.eye(N), lower=True)
    z = spla.solve_triangular(L, r, lower=True)
    return dict(flat=flat, X=X, r=r, K=K, L=L, Xin=Xin, z=z)


def factor_grad(e, dK_override=None, task_defect=None):
    """gpk_nll_grad emulated in fp64: A = alpha alpha^T - K^-1 from X^, the radial and environment entries as
    -1/2 sum A dK, the task entries contracted on the host from the per-pair sums G_ab (held for a >= b only).
    dK_override: {entry: dK}.  task_defect: 'diag_once' (the a = b = p term of G counted once), ('drop', a, b)."""
    flat, X = e["flat"], e["X"]
    a = e["Xin"].T @ e["z"]
    A = np.outer(a, a) - e["Xin"].T @ e["Xin"]
    _, grads = R.kernel_terms_ld(flat, X)
    nr = len(flat["axis"]) + 1
    g = []
    for p, dK in enumerate(grads):
        if task_defect is not None and p >= nr:
            break
        dK = (dK_override or {}).get(p, dK)
        g.append(-0.5 * np.sum(A * np.asarray(dK, dtype=np.float64)))
    if task_defect is not None:
        ax, nT, theta = flat["task"]
        Rm = R._radial_ld(flat, X, X)[0].astype(np.float64)
        t = X[:, ax].astype(int)
        G = np.zeros((nT, nT))
        for p in range(nT):
            for q in range(p + 1):
                G[p, q] = np.sum((A * Rm)[np.ix_(t == p, t == q)])
        if isinstance(task_defect, tuple):
            G[task_defect[1], task_defect[2]] = 0.0
        Lt = np.array([[np.exp(theta[p * (p + 1) // 2 + q]) if q <= p else 0.0 for q in range(nT)] for p in range(nT)])
        for p in range(nT):
            for q in range(p + 1):
                # dK_ab/dtheta_pq = L_pq (d_ap L_bq + d_bp L_aq): the row sum over b and the column sum over a
                row = sum((G[p, b] if p >= b else G[b, p]) * Lt[b, q] for b in range(nT))
                col = sum((G[a_, p] if a_ >= p else G[p, a_]) * Lt[a_, q] for a_ in range(nT))
                if task_defect == "diag_once":
                    col -= G[p, p] * Lt[p, q]
                g.append(-0.5 * Lt[p, q] * (row + col))
    g.append(-0.5 * np.trace(A) * 1e-2)
    return np.array(g)


def old_fd_ok(g, g0):
    """the older central-difference check: rel = 1e-5, abs = 1e-6 per entry"""
    return bool(np.all(np.abs(g - g0) <= 1e-5 * np.abs(g0) + 1e-6))


@pytest.mark.parametrize("kind", ["env", "task"])
def test_factor_checks_pass_on_the_emulation(kind):
    e = factor_problem(kind)
    g = factor_grad(e, task_defect="none" if kind == "task" else None)
    g_ref, bnd = R.grad_reference(e["flat"], e["X"], e["Xin"], e["z"], 1e-2)
    assert g.shape == g_ref.shape == (len(e["flat"]["axis"]) + (4 if kind == "env" else 2 + 6),)
    assert np.all(np.abs(g - g_ref) <= bnd), np.abs(g - g_ref) / bnd
    assert R.factor_check(e["L"], e["K"], e["Xin"])[0] <= 1
    Xs = np.random.RandomState(5).rand(40, 3)
    lo, up = np.array([0.0, 0.0, 0.0]), np.array([1.0, 1.0, 1.0])
    Xs[:, 2] = np.random.RandomState(6).randint(0, 3, 40) if kind == "task" else Xs[:, 2]
    dmu, dvar, bm, bv = R.predict_grad_reference(e["flat"], e["X"], e["Xin"], e["z"], Xs)
    em, ev = emulate_predict_grad(e, Xs)
    assert np.all(np.abs(em - dmu) <= bm) and np.all(np.abs(ev - dvar) <= bv)
    if kind == "task":
        assert np.all(dmu[:, 2] == 0) and np.all(dvar[:, 2] == 0)


def emulate_predict_grad(e, Xs, lower=None, upper=None, drop_env_chain=False):
    """gpk_predict_grad in fp64 (no output transform), from central differences-free closed forms"""
    flat, X = e["flat"], e["X"]
    Xn = Xs if lower is None else (Xs - lower) / (upper - lower)
    span = np.ones(3) if lower is None else upper - lower
    Ks = R.kernel_ld(flat, Xn, X).astype(np.float64)
    alpha = e["Xin"].T @ e["z"]
    W = (e["Xin"].T @ (e["Xin"] @ Ks.T)).T
    Rm = R._radial_ld(flat, Xn, X)[0].astype(np.float64)
    F = Ks / Rm
    dmu, dvar = np.zeros(Xs.shape), np.zeros(Xs.shape)
    for t, ax in enumerate(flat["axis"]):
        s = np.sqrt(5 * (Xn[:, ax][:, None] - X[:, ax][None, :]) ** 2 / np.exp(flat["log_metric"][t]))
        dl = -(5.0 / 6) * (1 + s) / (1 + s + s * s / 3)
        dk = Ks * dl * 2 * (Xn[:, ax][:, None] - X[:, ax][None, :]) / np.exp(flat["log_metric"][t])
        dmu[:, ax] = dk @ alpha / span[ax]
        dvar[:, ax] = -2 * np.sum(dk * W, axis=1) / span[ax]
    if flat["env"] is not None:
        ax, la, lb = flat["env"]
        dk = Rm * np.exp(lb) * X[:, ax][None, :]
        sc = 1.0 if drop_env_chain else span[ax]
        dmu[:, ax] = dk @ alpha / sc
        dvar[:, ax] = (2 * np.exp(flat["log_amp"]) * np.exp(lb) * Xn[:, ax] - 2 * np.sum(dk * W, axis=1)) / sc
    return dmu, dvar


def factor_defect_rows():
    """[(defect, old check passes?, new error / bound)] on N = 300, D = 2 + the factor column, diag 1e-2"""
    rows = []
    e = factor_problem("env")
    flat, X = e["flat"], e["X"]
    g_ref, bnd = R.grad_reference(flat, X, e["Xin"], e["z"], 1e-2)
    g0 = factor_grad(e)
    nr = len(flat["axis"]) + 1
    # genvb accumulated with z_c z_c instead of z_c z_j
    Rm = R._radial_ld(flat, X, X)[0]
    z = X[:, 2].astype(np.longdouble)
    g = factor_grad(e, {nr + 1: Rm * np.exp(np.longdouble(flat["env"][2])) * (z * z)[:, None]})
    rows.append(("genvb with z_c z_c instead of z_c z_j", old_fd_ok(g, g0), R.ratio(np.abs(g - g_ref), bnd)))
    # the factor scale skips the last, ragged 128-column tile (N = 300: columns 256..299) of the fit's K
    N = X.shape[0]
    Rk = R._radial_ld(flat, X, X)[0].astype(np.float64)
    Kd = e["K"].copy()
    Kd[:, 256:] = Rk[:, 256:] + 1e-2 * np.eye(N)[:, 256:]
    Kd = np.tril(Kd) + np.tril(Kd, -1).T
    try:
        Ld = np.linalg.cholesky(Kd)
        Xd = spla.solve_triangular(Ld, np.eye(N), lower=True)
        ll = lambda L, r: -0.5 * np.sum(spla.solve_triangular(L, r, lower=True) ** 2) - np.sum(np.log(np.diag(L)))
        old = abs(ll(Ld, e["r"]) - ll(e["L"], e["r"])) <= 1e-9 * abs(ll(e["L"], e["r"]))
        rows.append(("factor scale skips the last ragged column tile", old, R.factor_check(Ld, e["K"], Xd)[0]))
    except np.linalg.LinAlgError:
        rows.append(("factor scale skips the last ragged column tile", False, np.inf))
    # k** with the raw z* instead of the scaled one (environment axis bounds [0, 2])
    lo, up = np.zeros(3), np.array([1.0, 1.0, 2.0])
    Xs = np.random.RandomState(4).rand(50, 3) * up
    Xn = (Xs - lo) / (up - lo)
    Ks = R.kernel_ld(flat, Xn, X).astype(np.float64)
    Kss = R.kernel_ld(flat, Xn, Xn).astype(np.float64)
    ref = R.cov_reference(e["Xin"], Ks, Kss, e["z"], 0.0)
    V = e["Xin"] @ Ks.T
    amp, c0, c1 = np.exp(flat["log_amp"]), np.exp(flat["env"][1]), np.exp(flat["env"][2])
    var_ok = np.diag(Kss) - np.sum(V * V, axis=0)
    var_bad = amp * (c0 + c1 * Xs[:, 2] ** 2) - np.sum(V * V, axis=0)
    vref = np.clip(np.diag(ref["cov"]), R.EPS, np.inf)
    old = bool(np.max(np.abs(var_bad - vref) / np.maximum(vref, 1e-6)) < 1e-8)
    assert R.ratio(np.abs(var_ok - np.diag(ref["cov"])), np.diag(ref["cov_bound"])) <= 1
    rows.append(("k** from the raw z* instead of the scaled one", old,
                 R.ratio(np.abs(var_bad - np.diag(ref["cov"])), np.diag(ref["cov_bound"]))))
    # the 1 / (upper - lower) chain factor missing on the environment axis of predict_grad
    dmu, dvar, bm, bv = R.predict_grad_reference(flat, X, e["Xin"], e["z"], Xs, lo, up)
    em, ev = emulate_predict_grad(e, Xs, lo, up)
    assert np.all(np.abs(em - dmu) <= bm) and np.all(np.abs(ev - dvar) <= bv)
    dm, dv = emulate_predict_grad(e, Xs, lo, up, drop_env_chain=True)
    old = bool(np.allclose(dm, em, rtol=1e-5, atol=1e-6) and np.allclose(dv, ev, rtol=1e-5, atol=1e-6))
    rows.append(("predict_grad without 1 / (upper - lower) on the env axis", old,
                 max(R.ratio(np.abs(dm - dmu), bm), R.ratio(np.abs(dv - dvar), bv))))
    # the task factor
    e = factor_problem("task")
    flat, X = e["flat"], e["X"]
    g_ref, bnd = R.grad_reference(flat, X, e["Xin"], e["z"], 1e-2)
    g0 = factor_grad(e, task_defect="none")
    assert np.all(np.abs(g0 - g_ref) <= bnd)
    g = factor_grad(e, task_defect="diag_once")
    rows.append(("task contraction: the a = b = p term of G counted once", old_fd_ok(g, g0),
                 R.ratio(np.abs(g - g_ref), bnd)))
    g = factor_grad(e, task_defect=("drop", 2, 0))
    rows.append(("task contraction: the pair G_20 dropped", old_fd_ok(g, g0), R.ratio(np.abs(g - g_ref), bnd)))
    # gpk_hy_eval reading K_t[t_i][t_i] for both indices
    yv = e["r"][:120]
    Xh = X[:120]
    ref = R.hy_loglik_reference(flat, Xh, yv, 0.0, 1e-2, n_tasks=3)
    assert ref["first_order"] <= 0.1
    Rh = R._radial_ld(flat, Xh, Xh)[0].astype(np.float64)
    Kt = R.task_factor_ld(flat["task"][2], 3)[0].astype(np.float64)
    t = Xh[:, 2].astype(int)
    Kb = Rh * Kt[t, t][:, None] + 1e-2 * np.eye(120)
    Kb = np.tril(Kb) + np.tril(Kb, -1).T
    try:
        Lb = np.linalg.cholesky(Kb)
        zb = spla.solve_triangular(Lb, yv, lower=True)
        llb = -0.5 * zb @ zb - np.sum(np.log(np.diag(Lb))) - 60 * np.log(2 * np.pi)
        old = abs(llb - float(ref["ll"])) <= 1e-9 * abs(float(ref["ll"])) + 1e-9
        rows.append(("hy_eval: K_t[t_i][t_i] for both indices", old, abs(llb - float(ref["ll"])) / ref["bound"]))
    except np.linalg.LinAlgError:
        rows.append(("hy_eval: K_t[t_i][t_i] for both indices", False, np.inf))
    return rows


def test_factor_defect_table():
    """every injected factor defect fails the new bounds (ratio > 1); the table printed is DESIGN.md section 2's"""
    rows = factor_defect_rows()
    for name, old_ok, r in rows:
        print("%-58s old check passes: %-5s new error / bound: %.3g" % (name, old_ok, r))
        assert r > 1, name
    assert len(rows) == 7


def test_hy_loglik_reference_on_fp64():
    """the bound holds for an fp64 Cholesky of the same K (the device's algorithm class) at every factor"""
    for kind in ("env", "task"):
        flat = ENV_FLAT if kind == "env" else task_flat()
        X, y = factor_data(kind, 60, seed=2)
        ref = R.hy_loglik_reference(flat, X, y, 0.1, 1e-3, n_tasks=3 if kind == "task" else 0)
        K = R.kernel_ld(flat, X, X).astype(np.float64) + 1e-3 * np.eye(60)
        L = np.linalg.cholesky(K)
        zz = spla.solve_triangular(L, y - 0.1, lower=True)
        ll = -0.5 * zz @ zz - np.sum(np.log(np.diag(L))) - 30 * np.log(2 * np.pi)
        assert ref["first_order"] <= 0.1
        assert abs(ll - float(ref["ll"])) <= ref["bound"], (kind, abs(ll - float(ref["ll"])), ref["bound"])
