"""RandomForest's host layer and the forest restatement tests/rf_model.py, without a GPU: the restatement against
scikit-learn's CART, its invariants, the reference's contracts and rng consumption, pickling, argument errors, the
zero-std rules and the device dispatch, on the numpy stand-in of the device entry points (tests/fake_rf.py)."""
import copy
import os
import pickle

import numpy as np
import pytest

from robo_b200 import _lib
from robo_b200.models import RandomForest
from tests import fake_rf
from tests import rf_model as RM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def fake(monkeypatch):
    return fake_rf.install(monkeypatch)


def _grid(N, D, seed):
    """Inputs on a 2^-16 grid (scikit-learn's 1e-7 feature threshold never bites) and smooth noisy responses."""
    rng = np.random.RandomState(seed)
    X = np.floor(rng.rand(N, D) * 2 ** 16) / 2 ** 16
    return X, np.sin(3 * X).sum(axis=1) + 0.1 * rng.randn(N)


def test_header_constants_match_the_binding():
    src = open(os.path.join(ROOT, "include", "gpk.h")).read()
    for name, v in (("N", _lib.RF_MAX_N), ("D", _lib.RF_MAX_D), ("T", _lib.RF_MAX_T)):
        assert "#define GPK_RF_MAX_%s %d " % (name, v) in src
    cuh = open(os.path.join(ROOT, "robo_b200", "csrc", "gpk_rf.cuh")).read()
    assert "GPK_RF_TAG_BOOT 0x%08Xu" % RM.TAG_BOOT in cuh and "GPK_RF_TAG_PERM 0x%08Xu" % RM.TAG_PERM in cuh
    assert "GPK_RF_PURITY 1e-8\n" in cuh and RM.PURITY == 1e-8


@pytest.mark.parametrize("N,seed", [(2, 0), (15, 1), (60, 2), (300, 3)])
def test_each_tree_equals_sklearn_at_one_dimension(N, seed):
    from sklearn.tree import DecisionTreeRegressor
    X, y = _grid(N, 1, seed)
    Xt = np.vstack([X, _grid(500, 1, seed + 100)[0]])
    forest = RM.fit(X, y, 7 + seed, 2, 6)
    m, _ = RM.each_tree(forest, Xt)
    for t in range(6):
        cnt = RM.multiplicities(7 + seed, 2, t, N, N, True)
        rep = np.repeat(np.arange(N), cnt)
        sk = DecisionTreeRegressor(random_state=0).fit(X[rep], y[rep])
        np.testing.assert_allclose(m[t], sk.predict(Xt), rtol=0, atol=1e-12)
        assert len(forest[t]["feat"]) == sk.tree_.node_count


def test_draws():
    for N in (1, 2, 7, 1000):
        cnt = RM.multiplicities(3, 0, 5, N, 3 * N, True)
        assert cnt.sum() == 3 * N and cnt.min() >= 0
        c = RM.multiplicities(3, 0, 5, N, N, False)
        assert np.all(c == 1)
        if N > 2:
            c = RM.multiplicities(3, 0, 5, N, N - 2, False)
            assert c.sum() == N - 2 and c.max() == 1
    assert np.all(RM.index(np.array([0, 1, 2 ** 32 - 1], dtype=np.uint64), 7) == [0, 0, 6])
    assert not np.array_equal(RM.multiplicities(3, 0, 0, 50, 50, True), RM.multiplicities(3, 1, 0, 50, 50, True))
    assert not np.array_equal(RM.multiplicities(3, 0, 0, 50, 50, True), RM.multiplicities(3, 0, 1, 50, 50, True))
    with pytest.raises(ValueError):
        RM.multiplicities(3, 0, 0, 5, 6, False)


def test_without_bootstrap_every_tree_reproduces_the_data():
    X, y = _grid(40, 3, 4)
    forest = RM.fit(X, y, 1, 0, 5, 0, False)
    for t in forest[1:]:
        for k in RM.FIELDS:
            assert np.array_equal(t[k], forest[0][k])
    m, v = RM.each_tree(forest, X)
    assert np.all(m == y[None, :]) and np.all(v == 0)
    mu, var = RM.predict(forest[:2], X)
    assert np.array_equal(mu, y) and np.all(var == 0)


def test_law_of_total_variance():
    X, y = _grid(80, 2, 5)
    forest = RM.fit(X, y, 9, 0, 30)
    Xt = _grid(200, 2, 6)[0]
    m, v = RM.each_tree(forest, Xt)
    mu, var = RM.predict(forest, Xt)
    _, explained = RM.predict(forest, Xt, total_variance=False)
    np.testing.assert_allclose(mu, m.mean(axis=0), rtol=1e-14)
    np.testing.assert_allclose(explained, m.var(axis=0), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(var, m.var(axis=0) + v.mean(axis=0), rtol=1e-12, atol=1e-15)
    # the leaves' W, mean and var are those of the tree's samples in the leaf
    cnt = RM.multiplicities(9, 0, 0, 80, 80, True)
    leaf = RM.leaves(forest[0], X)
    for l in np.flatnonzero(forest[0]["feat"] < 0)[:10]:
        ys = np.repeat(y, cnt)[np.repeat(leaf, cnt) == l]
        assert forest[0]["W"][l] == len(ys)
        np.testing.assert_allclose([forest[0]["mean"][l], forest[0]["var"][l]], [ys.mean(), ys.var()],
                                   rtol=1e-13, atol=1e-16)


def test_constant_y_and_duplicated_rows():
    X, _ = _grid(30, 2, 7)
    forest = RM.fit(X, np.full(30, -1.5), 2, 0, 3)
    assert all(len(t["feat"]) == 1 and t["mean"][0] == -1.5 and t["var"][0] == 0 for t in forest)
    # duplicated rows with different responses cannot be separated: one leaf holds them with their spread
    Xd = np.repeat(X[:5], 4, axis=0)
    yd = np.arange(20, dtype=np.float64)
    tree = RM.fit(Xd, yd, 2, 0, 1, 0, False)[0]
    leaf = RM.leaves(tree, X[:5])
    for i in range(5):
        np.testing.assert_allclose(tree["mean"][leaf[i]], yd[4 * i:4 * i + 4].mean())
        np.testing.assert_allclose(tree["var"][leaf[i]], yd[4 * i:4 * i + 4].var())
    # ties between features: the lowest feature wins
    Xt = np.column_stack([X[:, 0], X[:, 0]])
    tree = RM.fit(Xt, X[:, 0], 2, 0, 1, 0, False)[0]
    assert np.all(tree["feat"][tree["feat"] >= 0] == 0)


def test_reference_contracts(fake):
    # test/test_models/test_random_forest.py
    X, y = _grid(10, 2, 8)
    model = RandomForest(rng=np.random.RandomState(1))
    model.train(X, y)
    m, v = model.predict(_grid(20, 2, 9)[0])
    assert m.shape == (20,) and v.shape == (20,)
    inc, inc_val = model.get_incumbent()
    b = np.argmin(y)
    assert np.all(inc == X[b]) and inc_val == y[b]
    assert model.predict_each_tree(X) is None and model.sample_functions(X) is None
    assert model.X is X and model.y is y and model.n_points_per_tree == 0


def test_rng_consumption_equals_the_reference(fake):
    rng, ref = np.random.RandomState(5), np.random.RandomState(5)
    m = RandomForest(rng=rng)
    assert m.seed == ref.randint(1000)
    X, y = _grid(20, 2, 10)
    m.train(X, y)
    m.train(X, y)
    assert rng.randint(2 ** 30) == ref.randint(2 ** 30)              # train draws nothing from rng
    h = m._handle
    assert [c[:2] for c in h.fit_calls] == [(m.seed, 0), (m.seed, 1)]
    c = copy.deepcopy(m)
    r2 = copy.deepcopy(ref)
    assert c.seed == r2.randint(1000) and c.counter == 0             # __setstate__: a new engine from the copy's rng


def test_pickle_and_deepcopy_predict_bit_identically(fake):
    X, y = _grid(50, 3, 11)
    m = RandomForest(num_trees=7, rng=np.random.RandomState(2))
    m.train(X, y)
    Xt = _grid(100, 3, 12)[0]
    mu, var = m.predict(Xt)
    for c in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        assert c._handle is None
        cm, cv = c.predict(Xt)
        assert np.array_equal(cm, mu) and np.array_equal(cv, var)


def test_argument_errors(fake):
    with pytest.raises(ValueError, match="GPK_RF_MAX_T"):
        RandomForest(num_trees=0)
    with pytest.raises(ValueError, match="n_points_per_tree"):
        RandomForest(n_points_per_tree=-1)
    with pytest.raises(ValueError, match="GPK_RF_MAX_N = 16384"):
        RandomForest().train(np.zeros((_lib.RF_MAX_N + 1, 1)), np.zeros(_lib.RF_MAX_N + 1))
    with pytest.raises(ValueError, match="GPK_RF_MAX_D = 64"):
        RandomForest().train(np.zeros((3, 65)), np.zeros(3))
    with pytest.raises(ValueError, match="without bootstrapping"):
        RandomForest(do_bootstrapping=False, n_points_per_tree=11).train(*_grid(10, 1, 0))
    with pytest.raises(ValueError, match="train the model first"):
        RandomForest().predict(np.zeros((2, 1)))


def test_zero_std_rules(fake):
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    X = np.array([[0.0], [1.0]])
    m = RandomForest(num_trees=2, do_bootstrapping=False, rng=np.random.RandomState(0))
    m.train(X, np.array([1.0, 0.0]))
    Xt = np.array([[0.2], [0.9]])
    assert np.all(m.predict(Xt)[1] == 0)
    h = m._ready_handle()
    eta = 0.0
    assert np.array_equal(h.acq(Xt, _lib.ACQ_EI, eta)["values"], [0.0, 0.0])
    assert np.array_equal(h.acq(Xt, _lib.ACQ_PI, eta)["values"], [0.0, np.nan], equal_nan=True)
    assert np.array_equal(h.acq(Xt, _lib.ACQ_PI, 0.5)["values"], [0.0, 1.0])
    assert np.array_equal(h.acq(Xt, _lib.ACQ_LCB)["values"], [-1.0, 0.0])
    assert np.array_equal(EI(m).compute(Xt), [[0]])                  # the whole-batch quirk (ei.py:72-74)
    assert LCB(m).compute(Xt).shape == (2,) and PI(m).compute(Xt).shape == (2,) and LogEI(m) is not None


def test_device_spec_and_random_sampling_dispatch(fake):
    from robo_b200.acquisition_functions import EI, LCB, PI, LogEI
    from robo_b200.maximizers import DeviceRandomSampling
    from robo_b200.maximizers.device_spec import device_spec
    X, y = _grid(20, 2, 13)
    m = RandomForest(rng=np.random.RandomState(0))
    m.train(X, y)
    for cls, kind in ((EI, "ei"), (LogEI, "log_ei"), (PI, "pi"), (LCB, "lcb")):
        which, (k, etas, par, hs) = device_spec(cls(m), "test")
        assert which == "acq" and k == kind and hs == [m._handle]
        assert etas == [0.0 if kind == "lcb" else float(np.min(y))]
    x = DeviceRandomSampling(EI(m), np.zeros(2), np.ones(2), n_samples=40, rng=np.random.RandomState(1)).maximize()
    assert x.shape == (2,)
    with pytest.raises(ValueError, match="one GPU"):
        DeviceRandomSampling(EI(m), np.zeros(2), np.ones(2), world=2, rank=0).maximize()
    # a zero std anywhere returns the first candidate, as the reference's batch RandomSampling does
    z = RandomForest(num_trees=2, do_bootstrapping=False, rng=np.random.RandomState(0))
    z.train(np.array([[0.0], [1.0]]), np.array([1.0, 0.0]))
    s = DeviceRandomSampling(EI(z), np.zeros(1), np.ones(1), n_samples=30, rng=np.random.RandomState(3))
    x = s.maximize()
    cands = z._handle.generate_candidates(s.last["seed"], 0, 30, 21, np.zeros(1), np.ones(1), [1.0], 0.1)
    assert np.array_equal(x, cands[0]) and s.last["best_idx"] == 0


def test_facade_still_refuses_rf():
    from robo_b200 import compat
    assert "pyrfr" in open(compat.__file__).read()
