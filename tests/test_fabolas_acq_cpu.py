"""InformationGainPerUnitCost's host logic (robo/acquisition_functions/information_gain_per_unit_cost.py): basis
recognition for the device transform, the representer-point projection and its environment-coordinate quirk, the
restart loop and its error, the overhead default, the derivative error, the ratio's overflow, and the pairing of
objective and cost sub-models in MarginalizationGPMCMC.  No GPU needed."""
import numpy as np
import pytest

from tests import fabolas_acq_model as F

LO = np.array([-5.0, 0.0, 0.0])
UP = np.array([10.0, 15.0, 1.0])
IS_ENV = np.array([0, 0, 1])


def _ig(value=0.5, lower=LO, upper=UP, is_env=IS_ENV, nb=10):
    from robo_b200.acquisition_functions import InformationGainPerUnitCost

    def sampling(model, **kw):
        return F.ConstantSampling(model, value=value)
    return InformationGainPerUnitCost(F.HostModel(), F.HostModel(), lower, upper, is_env, sampling_acquisition=sampling,
                                      n_representer=nb, rng=np.random.RandomState(0))


def test_basis_recognition():
    from robo_b200 import _lib
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import basis_code
    assert basis_code(lambda s: s) == _lib.BASIS_S
    assert basis_code(lambda s: (1 - s) ** 2) == _lib.BASIS_ONE_MINUS_S_SQ      # robo/fmin/fabolas.py:96-98

    def objective_basis(s):
        return (1 - s) ** 2
    assert basis_code(objective_basis) == _lib.BASIS_ONE_MINUS_S_SQ
    for other in (lambda s: 1 - s, lambda s: s ** 2, lambda s: (1 - s) * (1 - s) + 0.0 * s + 1e-300,
                  lambda s: np.sqrt(s), lambda s: 1.0):
        with pytest.raises(TypeError):
            basis_code(other)


def test_representer_points_projection_and_env_coordinate():
    ig = _ig()
    ig.sample_representer_points()
    assert ig.zb.shape == (10, 3) and ig.lmb.shape == (10, 1)
    assert np.all(ig.zb[:, :2] >= LO[:2]) and np.all(ig.zb[:, :2] <= UP[:2])
    # the sampling acquisition saw the configuration part extended by the environment's upper bound
    seen = np.concatenate(ig.sampling_acquisition.seen)
    assert seen.shape[1] == 3 and np.all(seen[:, 2] == UP[2])
    assert ig.sampling_acquisition.updates == 1
    # information_gain_per_unit_cost.py:151-153: the environment coordinate is the NUMBER of environment dimensions
    assert np.all(ig.zb[:, 2] == 1.0)


def test_env_coordinate_quirk_with_two_env_dimensions():
    lo, up, env = np.array([0.0, 0.0, 0.0]), np.array([1.0, 3.0, 5.0]), np.array([0, 1, 1])
    ig = _ig(lower=lo, upper=up, is_env=env)
    ig.sample_representer_points()
    assert ig.zb.shape == (10, 3)
    assert np.all(ig.zb[:, 1:] == 2.0)                        # not the upper bounds 3 and 5
    seen = np.concatenate(ig.sampling_acquisition.seen)
    assert np.all(seen[:, 1] == 3.0) and np.all(seen[:, 2] == 5.0)


def test_wrapper_and_batch_agree_and_test_config_bounds_only():
    ig = _ig()
    ig.sampling_acquisition.update(None)
    X = np.array([[0.0, 1.0], [11.0, 1.0], [-5.0, 15.0], [3.0, -0.1]])
    one = np.array([ig.sampling_acquisition_wrapper(x) for x in X])
    assert np.array_equal(ig._sampling_batch(X), one)
    assert np.array_equal(np.isinf(one), [False, True, False, True])


def test_restart_loop_and_error(monkeypatch):
    from robo_b200.acquisition_functions import information_gain_per_unit_cost as mod
    runs = []
    real = mod.EnsembleSampler

    class Counting(real):
        def run_mcmc(self, *a, **kw):
            runs.append(1)
            return real.run_mcmc(self, *a, **kw)
    monkeypatch.setattr(mod, "EnsembleSampler", Counting)
    ig = _ig(value=-np.inf)
    with pytest.raises(ValueError, match="Could not sample valid representer points! LogEI is -infinity"):
        ig.sample_representer_points()
    assert len(runs) == 5
    runs.clear()
    ig = _ig(value=0.25)
    ig.sample_representer_points()
    assert len(runs) == 1


def test_overhead_default_and_derivative_error():
    ig = _ig()
    ig.overhead = 7
    with pytest.raises(TypeError):                           # host models do not go to the device
        ig.update(F.HostModel(), F.HostModel())
    assert ig.overhead == 0
    with pytest.raises(TypeError):
        ig.update(F.HostModel(), F.HostModel(), overhead=0.25)
    assert ig.overhead == 0.25
    with pytest.raises(TypeError):                           # the reference's `raise "Not implemented"` under Python 3
        ig.compute(np.zeros((2, 3)), derivative=True)


def test_information_gain_still_refuses_fabolas_models():
    from robo_b200.acquisition_functions.information_gain import _device_model
    from robo_b200.models import FabolasGP
    fab = FabolasGP(None, basis_function=lambda s: s, lower=LO[:2], upper=UP[:2])
    with pytest.raises(TypeError):
        _device_model(fab)


def test_ratio_and_overflow_quirks():
    dh = np.array([2.0, F.EPS, -F.DBL_MAX, -F.DBL_MAX, -np.inf, 1.0])
    log_cost = np.array([0.0, np.log(4.0), 1.0, -1.0, 0.0, 800.0])
    v = F.per_unit_cost(dh, log_cost, 0.0)
    assert v[0] == 2.0
    assert v[1] == F.EPS / np.exp(np.log(4.0))
    assert np.isfinite(v[2]) and v[2] < 0                    # cost > 1: -DBL_MAX / c stays finite
    assert v[3] == -np.inf                                   # cost < 1: overflows to -inf
    assert v[4] == -np.inf
    assert v[5] == 0.0                                       # exp overflows to inf: dh / inf
    assert F.per_unit_cost(-F.DBL_MAX, -1.0, 1.0) == -F.DBL_MAX / (np.exp(-1.0) + 1.0)


def test_marginalisation_pairs_estimators():
    from robo_b200.acquisition_functions import InformationGainPerUnitCost, MarginalizationGPMCMC
    calls = []

    class Recording(InformationGainPerUnitCost):
        def update(self, model, cost_model, overhead=None):
            calls.append((model, cost_model, overhead))

    obj, cost = F.Ensemble(4), F.Ensemble(4)
    acq = MarginalizationGPMCMC(Recording(obj, cost, LO, UP, IS_ENV, sampling_acquisition=F.ConstantSampling,
                                          rng=np.random.RandomState(0)))
    assert acq.cost_model is cost and len(acq.estimators) == 4
    assert [e.cost_model for e in acq.estimators] == cost.models
    acq.update(obj, cost, overhead=0.5)
    assert [c[0] for c in calls] == obj.models
    assert [c[1] for c in calls] == cost.models
    assert all(c[2] == 0.5 for c in calls)
