"""DifferentialEvolution over the information-gain acquisitions without a GPU, on the oracle-backed fake
(tests/fake_de_es.py): dispatch per acquisition type, the TypeErrors that stay, the entropy_search facade's maximizers
and the polish through compute()."""
import numpy as np
import pytest

from tests import fabolas_acq_model as F

LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
EXT_LO, EXT_UP = np.append(LO, 0.0), np.append(UP, 1.0)
IS_ENV = np.array([0, 0, 1])


@pytest.fixture
def fake(monkeypatch):
    from tests import fake_de_es
    return fake_de_es.install(monkeypatch)


@pytest.fixture
def calls(fake, monkeypatch):
    """Counts the _lib entry point every DifferentialEvolution.maximize takes."""
    from robo_b200 import _lib
    seen = []
    for name in ("maximize_de", "maximize_de_es", "maximize_de_es_cost"):
        def wrap(*a, _fn=getattr(_lib, name), _name=name, **k):
            seen.append(_name)
            return _fn(*a, **k)
        monkeypatch.setattr(_lib, name, wrap)
    return seen


def branin(x):
    x1, x2 = x[0], x[1]
    return (x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x1) + 10


def _data(n=10, seed=0):
    rng = np.random.RandomState(seed)
    X = LO + (UP - LO) * rng.rand(n, 2)
    return X, np.array([branin(x) for x in X])


def _gp():
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    X, y = _data()
    gp = GaussianProcess(2 * K.Matern52Kernel(np.ones(2), ndim=2), normalize_input=True, lower=LO, upper=UP,
                         rng=np.random.RandomState(1))
    gp.train(X, y, do_optimize=False)
    return gp


def _mcmc():
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    X, y = _data()
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)), n_hypers=8,
                                chain_length=5, burnin_steps=5, normalize_input=True, lower=LO, upper=UP,
                                rng=np.random.RandomState(2))
    model.train(X, y, do_optimize=True)
    return model


def _ig(model):
    from robo_b200.acquisition_functions import InformationGain
    ig = InformationGain(model, LO, UP, Nb=10, sampling_acquisition=F.ConstantSampling, rng=np.random.RandomState(3))
    return ig


def _fabolas_pair(seed=0):
    from robo_b200 import kernels as K
    from robo_b200.models import FabolasGP
    rng = np.random.RandomState(seed)
    X = np.concatenate((LO + (UP - LO) * rng.rand(12, 2), rng.uniform(0.05, 1.0, (12, 1))), axis=1)
    models = []
    for basis, y in ((lambda s: (1 - s) ** 2, np.sin(X[:, 0]) + X[:, 2]), (lambda s: s, -1.0 + 2.0 * X[:, 2])):
        k = 1.3 * K.Matern52Kernel(np.ones(1) * 0.4, ndim=3, axes=0)
        k *= K.Matern52Kernel(np.ones(1) * 0.6, ndim=3, axes=1)
        k *= K.Matern52Kernel(np.ones(1) * 0.9, ndim=3, axes=2)
        m = FabolasGP(k, basis_function=basis, noise=1e-3, lower=LO, upper=UP, rng=np.random.RandomState(1))
        m.train(X, y, do_optimize=False)
        models.append(m)
    return models


def _puc(obj, cost):
    from robo_b200.acquisition_functions import InformationGainPerUnitCost
    return InformationGainPerUnitCost(obj, cost, EXT_LO, EXT_UP, IS_ENV, sampling_acquisition=F.ConstantSampling,
                                      n_representer=10, rng=np.random.RandomState(3))


class _Ensemble(object):
    def __init__(self, models):
        self.models = models


def _acquisitions():
    """name -> (updated acquisition, lower, upper, expected entry point, expected number of handles)."""
    from robo_b200.acquisition_functions import EI, MarginalizationGPMCMC
    gp = _gp()
    ig = _ig(gp)
    ig.update(gp)
    mcmc = _mcmc()
    mig = MarginalizationGPMCMC(_ig(mcmc))
    mig.update(mcmc)
    obj, cost = _fabolas_pair()
    puc = _puc(obj, cost)
    np.random.seed(0)
    puc.update(obj, cost, overhead=0.1)
    pairs = [_fabolas_pair(s) for s in (1, 2)]
    om, cm = _Ensemble([p[0] for p in pairs]), _Ensemble([p[1] for p in pairs])
    mpuc = MarginalizationGPMCMC(_puc(om, cm))
    mpuc.update(om, cm, overhead=0.1)
    return dict(ig=(ig, LO, UP, "maximize_de_es", 1), marg_ig=(mig, LO, UP, "maximize_de_es", len(mcmc.models)),
                puc=(puc, EXT_LO, EXT_UP, "maximize_de_es_cost", 1), marg_puc=(mpuc, EXT_LO, EXT_UP, "maximize_de_es_cost", 2),
                ei=(EI(gp), LO, UP, "maximize_de", 1))


def test_dispatch_per_acquisition_type(calls):
    from robo_b200.maximizers import DifferentialEvolution
    for name, (acq, lower, upper, entry, n) in _acquisitions().items():
        de = DifferentialEvolution(acq, lower, upper, n_iters=3, rng=np.random.RandomState(0), polish=False)
        which, spec = de._device_spec()
        # InformationGainPerUnitCost is an InformationGain: it must go to the per-unit-cost evolution
        assert which == {"maximize_de_es": "es", "maximize_de_es_cost": "es_cost", "maximize_de": "acq"}[entry], name
        handles = spec if which == "es" else spec[0] if which == "es_cost" else spec[3]
        assert len(handles) == n, name
        del calls[:]
        x = de.maximize()
        assert calls == [entry], name
        assert x.shape == lower.shape and np.all(x >= lower) and np.all(x <= upper), name
        # the device winner is the maximiser of compute over the evaluated population
        np.testing.assert_allclose(-np.asarray(acq.compute(x[None, :])).ravel()[0], de.last["device_energy"],
                                   rtol=1e-12)


def test_marginalised_information_gain_takes_the_fused_call(fake, monkeypatch):
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import MarginalizationGPMCMC
    mcmc = _mcmc()
    acq = MarginalizationGPMCMC(_ig(mcmc))
    with pytest.raises(ValueError, match="update"):            # the per-estimator error before update()
        acq.compute(LO[None, :])
    acq.update(mcmc)
    C = LO + (UP - LO) * np.random.RandomState(0).rand(50, 2)
    loop = np.mean([e.compute(C) for e in acq.estimators], axis=0)
    seen = []
    monkeypatch.setattr(_lib, "es_multi", lambda hs, X, want_values=True: seen.append(len(hs)) or
                        dict(values=loop, best_val=loop.max(), best_idx=int(np.argmax(loop))))
    assert np.array_equal(acq.compute(C), loop) and acq.argmax(C) == int(np.argmax(loop))
    assert seen == [len(mcmc.models)] * 2
    with pytest.raises(NotImplementedError):                  # derivative=True keeps the loop
        acq.compute(C, derivative=True)
    acq.estimators[1].lmb = acq.estimators[1].lmb.copy()
    acq.estimators[1].lmb[0] = -np.inf
    with pytest.raises(ValueError, match="lmb should not be infinite."):
        acq.compute(C)


def test_type_errors_stay(fake):
    from robo_b200.acquisition_functions import EI
    from robo_b200.maximizers import DifferentialEvolution
    from robo_b200.models.base_model import BaseModel
    obj, _ = _fabolas_pair()
    with pytest.raises(TypeError):
        DifferentialEvolution(EI(obj), EXT_LO, EXT_UP, rng=np.random.RandomState(0)).maximize()

    class HostModel(BaseModel):
        def train(self, X, y, **kwargs):
            self.X, self.y = X, y

        def predict(self, X_test, **kwargs):
            return np.zeros(len(X_test)), np.ones(len(X_test))
    hm = HostModel()
    hm.train(np.zeros((2, 2)), np.zeros(2))
    with pytest.raises(TypeError):
        DifferentialEvolution(EI(hm), np.zeros(2), np.ones(2), rng=np.random.RandomState(0)).maximize()
    with pytest.raises(ValueError):                           # InformationGain before update()
        DifferentialEvolution(_ig(_gp()), LO, UP, rng=np.random.RandomState(0)).maximize()


def test_polish_goes_through_compute(fake):
    from robo_b200.maximizers import DifferentialEvolution
    acqs = _acquisitions()
    for name in ("ig", "marg_ig", "puc", "marg_puc"):
        acq, lower, upper = acqs[name][:3]
        seen = []
        compute = acq.compute

        def recording(X, *a, **k):
            seen.append(np.array(X))
            return compute(X, *a, **k)
        acq.compute = recording
        de = DifferentialEvolution(acq, lower, upper, n_iters=3, rng=np.random.RandomState(2))
        x = de.maximize()
        assert len(seen) >= 1 and all(s.shape == (1, lower.size) for s in seen), name
        assert np.all(x >= lower) and np.all(x <= upper)
        assert de.last["best_energy"] <= de.last["device_energy"]


def test_entropy_search_maximizers(fake):
    from robo_b200.fmin import entropy_search
    np.random.seed(1)
    res = entropy_search(branin, LO, UP, num_iterations=4, n_init=3, model="gp", maximizer="differential_evolution",
                         rng=np.random.RandomState(1))
    X = np.array(res["X"])
    assert len(X) == 4 and np.all(X >= LO) and np.all(X <= UP) and res["f_opt"] == min(res["y"])
    with pytest.raises(ValueError, match="scipy"):
        entropy_search(branin, LO, UP, maximizer="scipy")
