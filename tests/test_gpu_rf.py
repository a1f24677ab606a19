"""RandomForest on the device (robo_b200/csrc/gpk_rf.cuh) against its exact restatement tests/rf_model.py: the trees,
the predictive moments and the acquisition values bit for bit, every device maximizer over a forest, BayesianOptimization
end to end, and the refusals between model kinds."""
import copy
import pickle

import numpy as np
import pytest

from robo_b200 import _lib
from robo_b200.models import RandomForest
from tests import rf_model as RM

pytestmark = pytest.mark.gpu

KINDS = (_lib.ACQ_EI, _lib.ACQ_LOG_EI, _lib.ACQ_PI, _lib.ACQ_LCB)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int64) if a.dtype == np.float64 else a


def _data(N, D, seed, kind="grid"):
    rng = np.random.RandomState(seed)
    if kind == "ties":             # a coarse grid: duplicated rows, tied features and repeated responses
        X = rng.randint(0, 5, size=(N, D)) / 4.0
        y = np.round(rng.randn(N), 1)
    else:
        X = np.floor(rng.rand(N, D) * 2 ** 16) / 2 ** 16
        y = np.sin(3 * X).sum(axis=1) + 0.1 * rng.randn(N)
    return X, y


def _device_forest(X, y, seed, counter, T, n_per_tree, bootstrap, total=True):
    h = _lib.Handle(0)
    _lib.rf_set_data(h, X, y)
    _lib.rf_fit(h, seed, counter, T, n_per_tree, bootstrap, total)
    return h


def _check_trees(h, X, y, seed, counter, T, n_per_tree, bootstrap):
    got = _lib.rf_trees(h)
    ref = RM.pack(RM.fit(X, y, seed, counter, T, n_per_tree, bootstrap), 2 * len(y))
    assert np.array_equal(got["n_nodes"], ref["n_nodes"])
    for k in RM.FIELDS:
        assert np.array_equal(_bits(got[k]), _bits(ref[k])), k
    return RM.unpack(got)


def _check_scores(h, forest, Xt, total=True):
    mu, var = h.predict(Xt)
    rm, rv = RM.predict(forest, Xt, total)
    assert np.array_equal(_bits(mu), _bits(rm)) and np.array_equal(_bits(var), _bits(rv))
    eta = float(np.min(rm)) + 0.05
    for kind in KINDS:
        r = h.acq(Xt, kind, eta, 0.01)
        ref, _ = _lib.moments_handle().acq_moments(rm, rv, kind, eta, 0.01)
        if kind == _lib.ACQ_EI:
            ref = np.where(rv == 0, 0.0, ref)
        assert np.array_equal(_bits(r["values"]), _bits(ref)), kind
        assert r["best_idx"] == int(np.argmax(ref))


# (D, N, T, n_per_tree, bootstrap, data)
CASES = [(1, 1, 1, 0, True, "grid"), (2, 3, 30, 0, True, "grid"), (8, 30, 33, 0, True, "grid"),
         (64, 200, 3, 0, True, "grid"), (2, 200, 100, 150, False, "grid"), (2, 200, 33, 0, False, "grid"),
         (1, 2000, 33, 500, True, "grid"), (8, 2000, 2, 0, True, "grid"), (16, 2000, 1, 3000, True, "grid"),
         (3, 200, 30, 0, True, "ties"), (8, 2000, 2, 0, False, "ties"),
         (1, _lib.RF_MAX_N, 1, 0, True, "grid"), (2, _lib.RF_MAX_N, 1, 0, False, "ties")]


@pytest.mark.parametrize("D,N,T,npt,boot,kind", CASES)
def test_trees_moments_and_acquisitions_bit_for_bit(D, N, T, npt, boot, kind):
    X, y = _data(N, D, 10 * D + N, kind)
    seed, counter = 17 * N + D, 3
    h = _device_forest(X, y, seed, counter, T, npt, boot)
    forest = _check_trees(h, X, y, seed, counter, T, npt, boot)
    Xt = np.vstack([X[:500], _data(700, D, 5, kind)[0]])
    _check_scores(h, forest, Xt)
    h.close()


def test_explained_variance_and_constant_y():
    X, y = _data(60, 3, 1)
    h = _device_forest(X, y, 5, 0, 30, 0, True, total=False)
    forest = RM.unpack(_lib.rf_trees(h))
    _check_scores(h, forest, _data(300, 3, 2)[0], total=False)
    h = _device_forest(X, np.full(60, 2.5), 5, 0, 4, 0, True)
    trees = _lib.rf_trees(h)
    assert np.all(trees["n_nodes"] == 1) and np.all(trees["mean"][:, 0] == 2.5) and np.all(trees["var"][:, 0] == 0)


def test_many_candidates_and_batches_beyond_one_chunk():
    X, y = _data(200, 4, 3)
    h = _device_forest(X, y, 11, 1, 30, 0, True)
    forest = RM.unpack(_lib.rf_trees(h))
    for M in (65536, 2 * 65536 + 5):
        Xt = np.random.RandomState(M).rand(M, 4)
        _check_scores(h, forest, Xt)
    big = np.random.RandomState(9).rand(1 << 20, 4)
    r = _lib.acq_multi([h], big, 0, kind=_lib.ACQ_EI, eta=[float(y.min())], par=0.0, want_argmax=True)
    rm, rv = RM.predict(forest, big)
    ref, _ = _lib.moments_handle().acq_moments(rm, rv, _lib.ACQ_EI, float(y.min()), 0.0)
    ref = np.where(rv == 0, 0.0, ref)
    assert np.array_equal(_bits(r["values"]), _bits(ref)) and r["best_idx"] == int(np.argmax(ref))


def test_deterministic_for_a_seed():
    X, y = _data(300, 5, 4)
    a = _lib.rf_trees(_device_forest(X, y, 42, 7, 30, 0, True))
    b = _lib.rf_trees(_device_forest(X, y, 42, 7, 30, 0, True))
    c = _lib.rf_trees(_device_forest(X, y, 42, 8, 30, 0, True))
    for k in RM.FIELDS:
        assert np.array_equal(_bits(a[k]), _bits(b[k]))
    assert not np.array_equal(a["thr"], c["thr"])


def test_model_train_copy_and_pickle():
    X, y = _data(100, 2, 6)
    m = RandomForest(rng=np.random.RandomState(3))
    m.train(X, y)
    m.train(X, y)
    forest = RM.fit(X, y, m.seed, 1, 30)
    Xt = _data(400, 2, 7)[0]
    mu, var = m.predict(Xt)
    rm, rv = RM.predict(forest, Xt)
    assert np.array_equal(_bits(mu), _bits(rm)) and np.array_equal(_bits(var), _bits(rv))
    for c in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        cm, cv = c.predict(Xt)
        assert np.array_equal(_bits(cm), _bits(mu)) and np.array_equal(_bits(cv), _bits(var))


def _trained(d=2, n=40, seed=0, **kw):
    X, y = _data(n, d, seed)
    m = RandomForest(rng=np.random.RandomState(seed), **kw)
    m.train(X, y)
    return m


def test_device_maximizers_return_their_energy():
    from robo_b200.acquisition_functions import EI, LogEI
    from robo_b200.maximizers import device_spec as DS
    for acq_cls in (EI, LogEI):
        m = _trained()
        acq = acq_cls(m)
        lo, up = np.zeros(2), np.ones(2)
        spec = DS.device_spec(acq, "test")
        assert spec[0] == "acq"
        runs = [DS.maximize_de(*spec, 5, 30, 20, (0.5, 1.0), 0.7, 0.01, 0.0, lo, up),
                DS.maximize_cmaes(*spec, 9, np.full(2, 0.5), lo, up, 400, 0),
                DS.maximize_direct(*spec, lo, up, 400, 200)]
        r = DS.maximize_lbfgs(*spec, np.random.RandomState(2).rand(4, 2), lo, up)
        best = int(np.argmin(r["energy"]))
        runs.append(dict(x=r["x"][best], energy=r["energy"][best]))
        for r in runs:
            x = np.asarray(r["x"]).ravel()
            assert np.all(x >= lo) and np.all(x <= up)
            host = float(np.ravel(acq.compute(x[None]))[0])
            if np.isfinite(host):
                assert r["energy"] == -host


def test_maximizer_classes():
    from robo_b200.acquisition_functions import EI, LCB, PI
    from robo_b200.maximizers import (CMAES, DeviceRandomSampling, DifferentialEvolution, Direct, GridSearch,
                                      RandomSampling, SciPyOptimizer)
    for d, classes in ((1, (GridSearch, DifferentialEvolution, DeviceRandomSampling, RandomSampling)),
                       (2, (DifferentialEvolution, SciPyOptimizer, CMAES, Direct, DeviceRandomSampling,
                            RandomSampling))):
        for acq_cls in (EI, PI, LCB):
            m = _trained(d=d)
            acq = acq_cls(m)
            lo, up = np.zeros(d), np.ones(d)
            for cls in classes:
                kw = dict(verbose=False) if cls in (CMAES, Direct) else {}
                x = np.asarray(cls(acq, lo, up, rng=np.random.RandomState(1), **kw).maximize()).ravel()
                assert x.shape == (d,) and np.all((lo <= x) & (x <= up)), cls.__name__
                assert np.isfinite(acq.compute(x[None])).all()


def test_device_random_sampling_keeps_the_zero_std_batch_rule():
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DeviceRandomSampling
    # without bootstrapping every tree is the same, so the variance is 0 wherever the trees' leaves are pure
    X = np.array([[0.0], [1.0]])
    m = RandomForest(num_trees=4, do_bootstrapping=False, rng=np.random.RandomState(0))
    m.train(X, np.array([1.0, 0.0]))
    s = DeviceRandomSampling(EI(m), np.zeros(1), np.ones(1), n_samples=50, rng=np.random.RandomState(2))
    x = s.maximize()
    h = m._ready_handle()
    cands = h.generate_candidates(s.last["seed"], 0, 50, 35, np.zeros(1), np.ones(1), X[1], 0.1)
    assert np.array_equal(x, cands[0]) and s.last["best_idx"] == 0
    assert np.all(m.predict(cands)[1] == 0)


def test_bayesian_optimization_end_to_end_on_branin():
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DifferentialEvolution
    from robo_b200.solver.bayesian_optimization import BayesianOptimization

    def branin(x):
        a, b, c, r, s, t = 1, 5.1 / (4 * np.pi ** 2), 5 / np.pi, 6, 10, 1 / (8 * np.pi)
        return float(a * (x[1] - b * x[0] ** 2 + c * x[0] - r) ** 2 + s * (1 - t) * np.cos(x[0]) + s)
    lo, up = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
    rng = np.random.RandomState(4)
    m = RandomForest(rng=rng)
    acq = EI(m)
    bo = BayesianOptimization(branin, lo, up, acq, m, DifferentialEvolution(acq, lo, up, rng=rng), rng=rng)
    x, fval = bo.run(num_iterations=8)
    assert len(bo.X) == 8 and np.all((np.asarray(bo.X) >= lo) & (np.asarray(bo.X) <= up))
    assert np.isfinite(fval) and m.counter >= 1


def test_refusals_and_limits():
    X, y = _data(30, 2, 8)
    h = _lib.Handle(0)
    with pytest.raises(ValueError, match="gpk_rf_set_data has not been called"):
        _lib.rf_fit(h, 1, 0, 3, 0, True, True)
    with pytest.raises(ValueError, match="GPK_RF_MAX_N = 16384"):
        _lib.rf_set_data(h, np.zeros((_lib.RF_MAX_N + 1, 1)), np.zeros(_lib.RF_MAX_N + 1))
    with pytest.raises(ValueError, match="GPK_RF_MAX_D = 64"):
        _lib.rf_set_data(h, np.zeros((3, 65)), np.zeros(3))
    with pytest.raises(ValueError, match="finite"):
        _lib.rf_set_data(h, np.array([[np.nan]]), np.zeros(1))
    _lib.rf_set_data(h, X, y)
    with pytest.raises(RuntimeError, match="not fitted"):
        h.predict(X[:3])
    with pytest.raises(ValueError, match="GPK_RF_MAX_T"):
        _lib.rf_fit(h, 1, 0, _lib.RF_MAX_T + 1, 0, True, True)
    with pytest.raises(ValueError, match="without bootstrapping"):
        _lib.rf_fit(h, 1, 0, 3, 31, False, True)
    _lib.rf_fit(h, 1, 0, 3, 0, True, True)
    refuse = "random forest"
    for call in (lambda: h.set_data(X, y), lambda: h.set_kernel(0, 0.0, [0], [0], [0.0]), lambda: h.fit(1e-6, 0.0),
                 lambda: h.predict_grad(X[:3]), lambda: h.predict_cov(X[:3]),
                 lambda: _lib.hyper_lnpost(h, np.zeros((1, 3))), lambda: _lib.es_multi([h], X[:3]),
                 lambda: _lib.esmc_multi([h], X[:3]),
                 lambda: _lib.blr_set_data(h, X, y, _lib.BLR_LINEAR, (0.1, -10.0, 0.1)),
                 lambda: _lib.blr_lnpost(h, np.zeros((1, 2)))):
        with pytest.raises(ValueError, match=refuse):
            call()
    gp = _lib.Handle(0)
    gp.set_data(X, y)
    with pytest.raises(ValueError, match="Gaussian-process model"):
        _lib.rf_set_data(gp, X, y)
    blr = _lib.Handle(0)
    _lib.blr_set_data(blr, X, y, _lib.BLR_LINEAR, (0.1, -10.0, 0.1))
    with pytest.raises(ValueError, match="Bayesian linear regression"):
        _lib.rf_set_data(blr, X, y)
    with pytest.raises(ValueError, match="Bayesian linear regression"):
        _lib.rf_trees(blr)
    with pytest.raises(ValueError, match="GPK_RF_MAX_N"):
        RandomForest().train(np.zeros((_lib.RF_MAX_N + 1, 1)), np.zeros(_lib.RF_MAX_N + 1))
