"""What scores an acquisition on the device, shared by the device maximizers (DifferentialEvolution, SciPyOptimizer,
CMAES, Direct, GridSearch), and the differential-evolution, multi-start L-BFGS, CMA-ES and DIRECT calls over it
(gpk_maximize_de*, gpk_maximize_lbfgs*, gpk_maximize_cmaes*, gpk_maximize_direct*) and the one-shot scoring of a
batch (gpk_acq_multi, gpk_es_multi, gpk_esmc_multi, gpk_es_cost_multi)."""
import numpy as np

from robo_b200 import _lib
from robo_b200.models.bayesian_linear_regression import BayesianLinearRegression
from robo_b200.models.dngo import DNGO
from robo_b200.models.gaussian_process import GaussianProcess
from robo_b200.models.random_forest import RandomForest
from robo_b200.models.wrapper_bohamiann import WrapperBohamiann

KINDS = ("ei", "log_ei", "pi", "lcb")
# the models other than GaussianProcess that score on the device: each holds one handle of its own (_ready_handle)
DEVICE_SURROGATES = (BayesianLinearRegression, RandomForest, WrapperBohamiann, DNGO)


def raw_inputs(model):
    """The model hands its raw inputs to the handle (no host-side transform such as FabolasGP's)."""
    return model is not None and getattr(type(model), "device_inputs", None) is GaussianProcess.device_inputs


def device_spec(acq, who):
    """What scores the acquisition ``acq`` on the device:
        ("es_cost", device_spec's tuple)   InformationGainPerUnitCost, alone or marginalised (gpk_es_cost_multi)
        ("esmc", handles)                  InformationGainMC, alone or marginalised (gpk_esmc_compute / gpk_esmc_multi)
        ("es", handles)                    InformationGain, alone or marginalised (gpk_es_compute / gpk_es_multi)
        ("acq", (kind, etas, par, handles)) EI / LogEI / PI / LCB (gpk_acq_multi)
    TypeError, naming the maximizer ``who``, when the acquisition does not run on device models."""
    from robo_b200.acquisition_functions.information_gain import InformationGain
    from robo_b200.acquisition_functions.information_gain_mc import InformationGainMC
    from robo_b200.acquisition_functions.information_gain_per_unit_cost import (InformationGainPerUnitCost,
                                                                                device_spec as es_cost_spec)
    estimators = acq.estimators if hasattr(acq, "_fused_spec") else [acq]
    # InformationGainPerUnitCost is an InformationGain: it is recognised first
    if estimators and all(isinstance(e, InformationGainPerUnitCost) for e in estimators):
        return "es_cost", es_cost_spec(estimators)
    # so is InformationGainMC: recognised before InformationGain, whose EP path it must not take
    if estimators and all(isinstance(e, InformationGainMC) for e in estimators):
        if not all(raw_inputs(e.model) for e in estimators):
            raise TypeError("%s needs InformationGainMC on robo_b200 GaussianProcess models" % who)
        return "esmc", [e._ready_handle() for e in estimators]
    if estimators and all(isinstance(e, InformationGain) for e in estimators):
        if not all(raw_inputs(e.model) for e in estimators):
            raise TypeError("%s needs InformationGain on robo_b200 GaussianProcess models" % who)
        return "es", [e._ready_handle() for e in estimators]
    return "acq", acq_spec(acq, who)


def acq_spec(acq, who):
    """(kind, eta per model, par, handles) of the acquisition, or TypeError when it does not run on device GPs whose
    inputs go to the handle untransformed or on a BayesianLinearRegression, RandomForest, WrapperBohamiann or DNGO (eta: its
    min observed y)."""
    if hasattr(acq, "_fused_spec"):                          # MarginalizationGPMCMC
        fused = acq._fused_spec()
        if fused is None or not all(raw_inputs(m) for m in acq.model.models):
            raise TypeError("%s needs a marginalised EI / LogEI / PI / LCB over device GaussianProcess sub-models" % who)
        kind, etas, par, handles = fused
        return kind, etas, par, handles
    model = getattr(acq, "model", None)
    kind = getattr(acq, "kind", None)
    if isinstance(model, DEVICE_SURROGATES) and kind in KINDS and getattr(acq, "cost_model", None) is None:
        eta = 0.0 if kind == "lcb" else float(model.get_incumbent()[1])
        return kind, [eta], float(acq.par), [model._ready_handle()]
    if kind not in KINDS or getattr(acq, "cost_model", None) is not None or not raw_inputs(model) \
            or not hasattr(getattr(model, "gp", None), "handle"):
        raise TypeError("%s needs EI / LogEI / PI / LCB on a robo_b200 GaussianProcess model" % who)
    eta = 0.0 if kind == "lcb" else float(model.get_incumbent()[1])
    model.gp._restore()
    model.gp._push_cfg()
    return kind, [eta], float(acq.par), [model.gp.handle]


def is_sampling_based(acq):
    """The acquisition is InformationGainMC, alone or marginalised: its surface is piecewise constant in x."""
    from robo_b200.acquisition_functions.information_gain_mc import InformationGainMC
    estimators = acq.estimators if hasattr(acq, "_fused_spec") else [acq]
    return len(estimators) > 0 and all(isinstance(e, InformationGainMC) for e in estimators)


def _run(which, spec, es_cost, es, acq, esmc=None):
    """Calls the maximizer of ``which`` over ``spec`` (what ``device_spec`` returned): es_cost(ho, hc, **configuration),
    es(handles), esmc(handles) or acq(handles, kind code, etas, par).  ValueError as ei.py:86-88 when EI came out
    negative; TypeError when the maximizer has no ``esmc``."""
    if which == "esmc":
        if esmc is None:
            raise TypeError("the sampling-based information gain has no device path for this maximizer")
        return esmc(spec)
    if which == "es_cost":
        ho, hc, lo, up, bo, bc, oh = spec
        return es_cost(ho, hc, cfg_lower=lo, cfg_upper=up, basis_objective=bo, basis_cost=bc, overhead=oh)
    if which == "es":
        return es(spec)
    kind, etas, par, handles = spec
    r = acq(handles, _lib.ACQ_KIND[kind], etas, par)
    if kind == "ei" and r["n_negative"] > 0:
        raise ValueError("Expected Improvement is smaller than 0!")
    return r


def maximize_de(which, spec, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper):
    """Differential evolution on the device over what ``device_spec`` returned -> _lib's result dict (x, energy, nit,
    nfev)."""
    args = (seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper)
    return _run(which, spec,
                lambda ho, hc, **cfg: _lib.maximize_de_es_cost(ho, hc, *args, **cfg),
                lambda hs: _lib.maximize_de_es(hs, *args),
                lambda hs, kind, etas, par: _lib.maximize_de(hs, *args, kind=kind, eta=etas, par=par),
                lambda hs: _lib.maximize_de_esmc(hs, *args))


def maximize_lbfgs(which, spec, x0, lower, upper):
    """Multi-start L-BFGS on the device from the rows of x0 over what ``device_spec`` returned, scipy's L-BFGS-B
    defaults -> _lib's result dict (x, energy, nit, nfev, status per start)."""
    return _run(which, spec,
                lambda ho, hc, **cfg: _lib.maximize_lbfgs_es_cost(ho, hc, x0, lower, upper, **cfg),
                lambda hs: _lib.maximize_lbfgs_es(hs, x0, lower, upper),
                lambda hs, kind, etas, par: _lib.maximize_lbfgs(hs, kind, etas, par, x0, lower, upper))


def maximize_cmaes(which, spec, seed, x0, lower, upper, n_func_evals, restarts):
    """CMA-ES on the device from x0 over what ``device_spec`` returned, sigma0 = 0.6 as the reference passes it ->
    _lib's result dict (x, energy, nfev_total, nit / nfev / stop per run, the last run's state)."""
    args = (seed, x0, lower, upper, n_func_evals, restarts)
    return _run(which, spec,
                lambda ho, hc, **cfg: _lib.maximize_cmaes_es_cost(ho, hc, seed, x0, lower, upper, n_func_evals=n_func_evals,
                                                                  restarts=restarts, **cfg),
                lambda hs: _lib.maximize_cmaes_es(hs, *args),
                lambda hs, kind, etas, par: _lib.maximize_cmaes(hs, kind, etas, par, *args),
                lambda hs: _lib.maximize_cmaes_esmc(hs, *args))


def maximize_direct(which, spec, lower, upper, n_func_evals, n_iters):
    """DIRECT on the device in the box lower / upper over what ``device_spec`` returned -> _lib's result dict (x,
    energy, nit, nfev, stop, rows)."""
    args = (lower, upper, n_func_evals, n_iters)
    return _run(which, spec,
                lambda ho, hc, **cfg: _lib.maximize_direct_es_cost(ho, hc, lower, upper, n_func_evals=n_func_evals,
                                                                   n_iters=n_iters, **cfg),
                lambda hs: _lib.maximize_direct_es(hs, *args),
                lambda hs, kind, etas, par: _lib.maximize_direct(hs, kind, etas, par, *args),
                lambda hs: _lib.maximize_direct_esmc(hs, *args))


def score_batch(which, spec, X):
    """The one-shot value of every row of X (m, d) over what ``device_spec`` returned, with numpy's first arg-max ->
    dict(values (m,), best_idx)."""
    return _run(which, spec,
                lambda ho, hc, **cfg: _lib.es_cost_multi(ho, hc, X, cfg["cfg_lower"], cfg["cfg_upper"],
                                                         cfg["basis_objective"], cfg["basis_cost"], cfg["overhead"]),
                lambda hs: _lib.es_multi(hs, X),
                lambda hs, kind, etas, par: _lib.acq_multi(hs, X, 0, kind=kind, eta=etas, par=par, want_argmax=True),
                lambda hs: _lib.esmc_multi(hs, X))


def lbfgs_success(status):
    """scipy's ``res.success`` for a gpk_lb_status: converged by ftol or pgtol."""
    return np.isin(status, (_lib.LB_FTOL, _lib.LB_PGTOL))
