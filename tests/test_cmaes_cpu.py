"""CMA-ES without a GPU: the constants, the bound transform, gpk_cmaes_exp, the Jacobi sweeps and the ranking of the
exact restatement (tests/cmaes_model.py); the strategy in law on standard test functions; the stop reasons, the budget
and IPOP; the CMAES class on the oracle-backed fake handle (tests/fake_cmaes.py)."""
import math

import numpy as np
import pytest

from robo_b200 import _lib
from tests import cmaes_model as M


@pytest.fixture
def fake(monkeypatch):
    from tests import fake_cmaes
    return fake_cmaes.install(monkeypatch)


@pytest.mark.parametrize("d,lam,mueff", [(2, 6, 2.0286), (3, 7, 2.2548), (16, 12, 3.7295), (64, 16, 4.8409)])
def test_constants_match_the_tutorial(d, lam, mueff):
    assert _lib.cmaes_lambda(d) == lam == 4 + math.floor(3 * math.log(d))
    c = _lib.cmaes_run_constants(d, lam)
    mu = lam // 2
    assert c["mu"] == mu and c["w"].size == mu
    np.testing.assert_allclose(c["w"].sum(), 1.0, rtol=0, atol=1e-15)
    assert np.all(np.diff(c["w"]) < 0) and np.all(c["w"] > 0)
    raw = np.log((lam + 1) / 2.0) - np.log(np.arange(1, mu + 1))
    np.testing.assert_allclose(c["w"], raw / raw.sum(), rtol=1e-15)
    assert c["mueff"] == pytest.approx(1.0 / np.sum(c["w"] ** 2)) and c["mueff"] == pytest.approx(mueff, abs=1e-4)
    me = c["mueff"]
    assert c["cs"] == pytest.approx((me + 2) / (d + me + 5))
    assert c["ds"] == pytest.approx(1 + 2 * max(0, math.sqrt((me - 1) / (d + 1)) - 1) + c["cs"])
    assert c["cc"] == pytest.approx((4 + me / d) / (d + 4 + 2 * me / d))
    assert c["c1"] == pytest.approx(2 / ((d + 1.3) ** 2 + me))
    assert c["cmu"] == pytest.approx(min(1 - c["c1"], 2 * (me - 2 + 1 / me) / ((d + 2) ** 2 + me)))
    assert c["chi"] == pytest.approx(math.sqrt(d) * (1 - 1 / (4 * d) + 1 / (21 * d * d)))
    assert 0 < c["c1"] + c["cmu"] <= 1 and c["hist"] <= _lib.CMA_HIST and 0 <= c["flat"] < lam
    tab = _lib.cmaes_constants(d, 2)
    assert tab.shape == (3, _lib.CMA_NCONST) and list(tab[:, 0]) == [lam, 2 * lam, 4 * lam]
    np.testing.assert_array_equal(tab[0, _lib.CMA_C_W:_lib.CMA_C_W + mu], c["w"])


def test_bound_transform():
    lower, upper = np.array([-5.0, 0.0, 2.0]), np.array([10.0, 15.0, 2.5])
    al, au = M.margins(lower, upper)
    rs = np.random.RandomState(0)
    x = rs.standard_normal((20000, 3)) * 40.0
    y = M.transform(x, lower, upper)
    assert np.all(y >= lower) and np.all(y <= upper)
    inner = lower + al + (upper - au - lower - al) * rs.rand(2000, 3)
    np.testing.assert_array_equal(M.transform(inner, lower, upper), inner)
    box = lower + (upper - lower) * rs.rand(5000, 3)
    box[:3] = lower
    box[3:6] = upper
    np.testing.assert_allclose(M.transform(M.genotype(box, lower, upper), lower, upper), box, rtol=0, atol=1e-12)
    # mirror symmetry at the ends of the invertible range and periodicity far outside
    np.testing.assert_allclose(M.transform(lower - al - 0.3 * al, lower, upper),
                               M.transform(lower - al + 0.3 * al, lower, upper), rtol=1e-12)
    per = 2 * (upper - lower + al + au)
    np.testing.assert_allclose(M.transform(x[:100] + 3 * per, lower, upper), M.transform(x[:100], lower, upper),
                               rtol=0, atol=1e-9)


def test_exp_within_one_ulp():
    x = np.concatenate([np.linspace(-50, 50, 200001), np.random.RandomState(1).uniform(-2, 2, 100000)])
    y, ref = M.exp(x), np.exp(x)
    assert np.max(np.abs(y - ref) / np.spacing(ref)) <= 1.0
    assert M.exp(0.0) == 1.0 and M.exp(800.0) == np.inf and M.exp(-800.0) == 0.0 and np.isnan(M.exp(np.nan))


@pytest.mark.parametrize("d", [2, 3, 7, 16, 64])
def test_jacobi(d):
    rs = np.random.RandomState(d)
    A = rs.standard_normal((d, d))
    Q = np.linalg.qr(A)[0]
    C = (Q * np.logspace(-6, 2, d)) @ Q.T
    trace = []
    ev, B, sweeps = M.jacobi(C, trace)
    Cs = np.triu(C) + np.triu(C, 1).T
    assert sweeps <= M.SWEEPS
    np.testing.assert_allclose(B.T @ B, np.eye(d), rtol=0, atol=1e-13)
    np.testing.assert_allclose((B * ev) @ B.T, Cs, rtol=0, atol=1e-13 * np.abs(Cs).max())
    np.testing.assert_allclose(np.sort(ev), np.linalg.eigvalsh(Cs), rtol=1e-10, atol=1e-13 * np.abs(ev).max())
    # the rotation order is fixed: every round pairs each index at most once, and a sweep visits every pair once
    rounds = M.round_robin(d)
    assert len(rounds) == d - 1 + (d & 1)
    pairs = set()
    for p, q in rounds:
        assert len(set(p) | set(q)) == 2 * p.size and np.all(p < q)
        pairs |= set(zip(p.tolist(), q.tolist()))
    assert pairs == {(i, j) for i in range(d) for j in range(i + 1, d)}
    again = []
    M.jacobi(C, again)
    assert len(again) == len(trace) and all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
                                            for a, b in zip(again, trace))


def test_rank_matches_numpy_stable_argsort():
    rs = np.random.RandomState(3)
    for _ in range(200):
        n = rs.randint(2, 40)
        e = rs.choice([0.0, -0.0, 1.0, -1.0, np.nan, np.inf, -np.inf, 2.5], n) if rs.rand() < 0.5 \
            else rs.standard_normal(n)
        np.testing.assert_array_equal(M.rank(e), np.argsort(e, kind="stable"))
    np.testing.assert_array_equal(M.rank(np.array([0.0, -0.0, np.nan, -0.0, 0.0])), [0, 1, 3, 4, 2])


def _sphere(P):
    return -np.sum((P - 0.3) ** 2, axis=1)


def _ellipsoid(d, seed):
    Q = np.linalg.qr(np.random.RandomState(seed).standard_normal((d, d)))[0]
    scale = 1e3 ** (np.arange(d) / max(d - 1, 1))

    def f(P):
        Z = (P - 0.3) @ Q
        return -np.sum(scale * Z * Z, axis=1)
    return f


def _rosenbrock(P):
    return -np.sum(100.0 * (P[:, 1:] - P[:, :-1] ** 2) ** 2 + (1.0 - P[:, :-1]) ** 2, axis=1)


@pytest.mark.parametrize("name,d,budget", [("sphere", 2, 2000), ("sphere", 8, 6000), ("sphere", 16, 12000),
                                           ("ellipsoid", 2, 3000), ("ellipsoid", 8, 20000),
                                           ("rosenbrock", 2, 6000), ("rosenbrock", 4, 20000)])
def test_reaches_the_optimum_in_law(name, d, budget):
    lower, upper = -3.0 * np.ones(d), 3.0 * np.ones(d)
    for seed in range(3):
        fn = {"sphere": _sphere, "ellipsoid": _ellipsoid(d, seed), "rosenbrock": _rosenbrock}[name]
        x0 = np.random.RandomState(seed).uniform(lower, upper)
        trace = []
        r = M.run(fn, M.numpy_normals(seed), x0, lower, upper, n_func_evals=budget, restarts=2, trace=trace)
        assert r["energy"] < 1e-10, (name, d, seed, r["energy"], r["stop"])
        assert np.all(r["x"] >= lower) and np.all(r["x"] <= upper)
        # C stays symmetric positive definite
        np.testing.assert_array_equal(r["C"], r["C"].T)
        assert np.all(np.linalg.eigvalsh(r["C"]) > 0)


def test_stop_reasons_budget_and_ipop():
    d = 4
    lower, upper = np.zeros(d), np.ones(d)
    x0 = np.full(d, 0.4)
    lam = _lib.cmaes_lambda(d)
    # maxfevals: the budget ends every run, and the overshoot stays below lambda
    r = M.run(_sphere, M.numpy_normals(1), x0, lower, upper, n_func_evals=50, restarts=3)
    assert r["stop"][0] == _lib.CMA_MAXFEVALS and r["nit"][1:].sum() == 0 and r["nfev_total"] - 50 < lam
    # tolfun: a flat surface; tolfun ends run 0 and IPOP doubles lambda for run 1
    r = M.run(lambda P: np.zeros(len(P)), M.numpy_normals(2), x0, lower, upper, n_func_evals=100000, restarts=1)
    assert list(r["stop"]) == [_lib.CMA_TOLFUN, _lib.CMA_TOLFUN]
    assert r["nfev"][0] == lam * r["nit"][0] and r["nfev"][1] == 2 * lam * r["nit"][1]
    assert r["nit"][0] == _lib.cmaes_run_constants(d, lam)["hist"]
    # tolx: a surface whose energies keep a spread of |x - 0.5| (scaled so that tolfun cannot fire first) is approached
    # until the step size vanishes
    r = M.run(lambda P: -np.sum(np.abs(P - 0.5), axis=1) * 1e12, M.numpy_normals(3), x0, lower, upper,
              n_func_evals=200000)
    assert r["stop"][0] == _lib.CMA_TOLX
    assert r["sigma"] * np.max(np.fmax(np.fabs(r["pc"]), np.sqrt(np.diag(r["C"])))) < 1e-11
    # numerical: a NaN step size
    with np.errstate(over="ignore", invalid="ignore"):
        r = M.run(lambda P: np.full(len(P), np.nan), M.numpy_normals(5), x0, lower, upper, n_func_evals=100000,
                  sigma0=1e308)
    assert r["stop"][0] == _lib.CMA_NUMERICAL and not r["found"] and np.isnan(r["energy"])


@pytest.mark.parametrize("seed", range(4))
def test_forced_conditioncov(seed):
    """An axis-parallel ellipsoid of condition 1e18: C learns the inverse Hessian, and the run stops on conditioncov
    as soon as the ratio of C's largest to smallest eigenvalue exceeds 1e14, long before tolfun or tolx could fire
    (a test on the ratio of D = sqrt(eigenvalues) would need 1e28 and never stop this way)."""
    r = M.run(lambda P: -(1e18 * (P[:, 0] - 0.5) ** 2 + (P[:, 1] - 0.5) ** 2), M.numpy_normals(seed),
              np.array([0.3, 0.6]), np.zeros(2), np.ones(2), n_func_evals=10 ** 6)
    assert r["stop"].tolist() == [_lib.CMA_CONDITIONCOV]
    ev = M.jacobi(r["C"])[0]
    assert 1e14 < ev.max() / ev.min() < 1e16


def _gp(d, n=8, seed=0):
    from robo_b200 import kernels as K
    from robo_b200.models.gaussian_process import GaussianProcess
    rng = np.random.RandomState(seed)
    lower, upper = np.zeros(d), np.ones(d)
    X = rng.rand(n, d)
    y = np.sin(3 * X).sum(axis=1)
    model = GaussianProcess(2 * K.Matern52Kernel(np.ones(d) * 0.3, ndim=d), normalize_input=True, lower=lower,
                            upper=upper, rng=np.random.RandomState(1))
    model.train(X, y, do_optimize=False)
    return model, lower, upper


@pytest.mark.parametrize("kind", ["ei", "log_ei", "pi", "lcb"])
def test_maximizer_shape_bounds_and_seed(fake, kind):
    """test/test_maximizers/test_maximizers_two_dim.py: shape (D,), inside the bounds; the seed advances per call."""
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    from robo_b200.maximizers import CMAES
    model, lower, upper = _gp(2)
    acq = {"ei": EI, "log_ei": LogEI, "pi": PI, "lcb": LCB}[kind](model)
    cm = CMAES(acq, lower, upper, n_func_evals=200, rng=np.random.RandomState(3))
    x = cm.maximize()
    assert x.shape == (2,) and np.all(x >= lower) and np.all(x <= upper)
    assert cm.last["nfev"] >= 200 or cm.last["stop"][0] != _lib.CMA_MAXFEVALS
    np.testing.assert_allclose(-acq.compute(x[None, :]).ravel()[0], cm.last["best_energy"], rtol=1e-12)
    seed0 = cm.last["seed"]
    cm.maximize()
    assert cm.last["seed"] != seed0


def test_one_dim_raises_before_base_init(fake):
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import CMAES
    model, lower, upper = _gp(1)
    with pytest.raises(RuntimeError):
        CMAES(EI(model), lower, upper)


def test_refuses_host_acquisitions(fake):
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import CMAES
    from robo_b200.models.base_model import BaseModel

    class HostModel(BaseModel):
        def train(self, X, y, **kwargs):
            self.X, self.y = X, y

        def predict(self, X_test, **kwargs):
            return np.zeros(len(X_test)), np.ones(len(X_test))
    hm = HostModel()
    hm.train(np.zeros((2, 2)), np.zeros(2))
    with pytest.raises(TypeError, match="CMAES"):
        CMAES(EI(hm), np.zeros(2), np.ones(2), rng=np.random.RandomState(0)).maximize()


def test_falls_back_to_the_start_point_without_a_finite_energy(fake, monkeypatch):
    from robo_b200.acquisition_functions import LCB
    from robo_b200.maximizers import CMAES
    from robo_b200.maximizers import cmaes as mod
    model, lower, upper = _gp(2)
    cm = CMAES(LCB(model), lower, upper, n_func_evals=30, rng=np.random.RandomState(7))
    monkeypatch.setattr(mod, "maximize_cmaes", lambda *a: dict(x=np.full(2, 0.5), energy=np.nan, nfev_total=30,
                                                              nit=np.array([5]), stop=np.array([1])))
    rs = np.random.RandomState(7)
    rs.randint(0, 2 ** 31 - 1)                                   # the seed CMAES draws at construction
    start = mod.init_random_uniform(lower, upper, 1, rs)
    x = cm.maximize()
    assert x.shape == (1, 2)                                  # the reference returns init_random_uniform's (1, D) array
    np.testing.assert_array_equal(x, start)
