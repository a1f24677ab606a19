"""MarginalizationGPMCMC (robo/acquisition_functions/marginalization.py): averages an acquisition
function over the hyper-parameter samples of a GaussianProcessMCMC model.  One estimator
(deep copy of the acquisition function) per sub-model exactly like the reference (:33-47,
:64-78); every estimator's compute() is the fused GPU path of its sub-model, and the mean over
models (:121) is reduced on the GPU as well."""
from copy import deepcopy

import numpy as np

from robo_b200 import _lib
from robo_b200.acquisition_functions.base_acquisition import BaseAcquisitionFunction


class MarginalizationGPMCMC(BaseAcquisitionFunction):

    def __init__(self, acquisition_func):
        self.acquisition_func = acquisition_func
        self.model = acquisition_func.model
        self.cost_model = acquisition_func.cost_model if hasattr(acquisition_func, "cost_model") else None
        self.estimators = []
        self._make_estimators()

    def _make_estimators(self):
        for i in range(len(self.model.models)):
            estimator = deepcopy(self.acquisition_func)
            estimator.model = self.model.models[i]
            if hasattr(estimator, "stream"):         # InformationGainMC: its own draws per sub-model
                estimator.stream = i
            if self.cost_model is not None and len(self.cost_model.models) > 0:
                estimator.cost_model = self.cost_model.models[i]
            self.estimators.append(estimator)

    def update(self, model, cost_model=None, **kwargs):
        if len(self.estimators) == 0:
            self._make_estimators()
        self.model = model
        if cost_model is not None:
            self.cost_model = cost_model
        if len(self.estimators) != len(self.model.models):
            self.estimators = []
            self._make_estimators()
        from robo_b200.acquisition_functions.information_gain import InformationGain, sample_representers_device
        if all(isinstance(e, InformationGain) and e.representer_sampler == "device" for e in self.estimators):
            # the representer points of every estimator in one device call (gpk_sample_representers), then each
            # estimator's EP and U as in its own update()
            handles = []
            for i, e in enumerate(self.estimators):
                if cost_model is not None:
                    e._set_cost(self.cost_model.models[i], **kwargs)
                handles.append(e._begin_update(self.model.models[i]))
            sample_representers_device(self.estimators)
            for e, h in zip(self.estimators, handles):
                e._end_update(h)
            return
        for i in range(len(self.model.models)):
            if cost_model is not None:
                self.estimators[i].update(self.model.models[i], self.cost_model.models[i], **kwargs)
            else:
                self.estimators[i].update(self.model.models[i], **kwargs)

    def compute(self, X_test, derivative=False):
        n = len(self.model.models)
        es = self._es_cost_spec() if not derivative else None
        if es is not None:
            # information gain per unit cost over the (objective, cost) sub-model pairs as ONE call (gpk_es_cost_multi)
            ho, hc, lo, up, bo, bc, oh = es
            return _lib.es_cost_multi(ho, hc, np.asarray(X_test, dtype=np.float64), lo, up, bo, bc, oh)["values"]
        handles = self._esmc_spec() if not derivative else None
        if handles is not None:
            # the sampling-based information gain of every estimator and the mean over them as ONE call (gpk_esmc_multi)
            return _lib.esmc_multi(handles, np.asarray(X_test, dtype=np.float64))["values"]
        handles = self._es_spec() if not derivative else None
        if handles is not None:
            # the information gain of every estimator and the mean over them as ONE call (gpk_es_multi)
            return _lib.es_multi(handles, np.asarray(X_test, dtype=np.float64))["values"]
        fused = self._fused_spec() if not derivative else None
        if fused is not None:
            # marginalization.py:115-121 as ONE call: the batch goes to the device once, the n sub-models score it
            # concurrently and the mean over models is taken there (gpk_acq_multi mode 0); M doubles come back
            kind, etas, par, handles = fused
            X_dev = self.model.models[0].device_inputs(np.asarray(X_test, dtype=np.float64))
            r = _lib.acq_multi(handles, X_dev, 0, _lib.ACQ_KIND[kind], etas, par)
            if kind == "ei" and r["n_negative"] > 0:
                raise ValueError("Expected Improvement is smaller than 0!")      # ei.py:86-88
            return r["values"]
        acquisition_values = np.zeros([n, X_test.shape[0]])
        for i in range(n):
            acquisition_values[i] = self.estimators[i].compute(X_test, derivative=derivative)
        return _lib.moments_handle().reduce_models(acquisition_values)

    def argmax(self, X_test):
        """numpy.argmax of compute(X_test) taken on the device when the fused path applies."""
        es = self._es_cost_spec()
        if es is not None:
            ho, hc, lo, up, bo, bc, oh = es
            r = _lib.es_cost_multi(ho, hc, np.asarray(X_test, dtype=np.float64), lo, up, bo, bc, oh, want_values=False)
            return int(r["best_idx"])
        handles = self._esmc_spec()
        if handles is not None:
            return int(_lib.esmc_multi(handles, np.asarray(X_test, dtype=np.float64), want_values=False)["best_idx"])
        handles = self._es_spec()
        if handles is not None:
            return int(_lib.es_multi(handles, np.asarray(X_test, dtype=np.float64), want_values=False)["best_idx"])
        fused = self._fused_spec()
        if fused is None:
            return int(np.argmax(self.compute(X_test)))
        kind, etas, par, handles = fused
        X_dev = self.model.models[0].device_inputs(np.asarray(X_test, dtype=np.float64))
        r = _lib.acq_multi(handles, X_dev, 0, _lib.ACQ_KIND[kind], etas, par, want_argmax=True)
        if kind == "ei" and r["n_negative"] > 0:
            raise ValueError("Expected Improvement is smaller than 0!")
        return int(r["best_idx"])

    def _es_cost_spec(self):
        """The fused call's arguments (information_gain_per_unit_cost.device_spec) when every estimator is an
        InformationGainPerUnitCost; estimator i pairs objective sub-model i with cost sub-model i."""
        from robo_b200.acquisition_functions.information_gain_per_unit_cost import (InformationGainPerUnitCost,
                                                                                    device_spec)
        if self.cost_model is None or len(self.estimators) == 0 or \
                not all(isinstance(e, InformationGainPerUnitCost) for e in self.estimators):
            return None
        return device_spec(self.estimators)

    def _es_spec(self):
        """The objective handles of the fused call (gpk_es_multi) when every estimator is an InformationGain, neither
        per unit cost nor sampling-based, on a device GaussianProcess sub-model; raises the estimators' own ValueErrors
        (before update(), an infinite lmb)."""
        from robo_b200.acquisition_functions.information_gain import InformationGain
        from robo_b200.acquisition_functions.information_gain_mc import InformationGainMC
        from robo_b200.acquisition_functions.information_gain_per_unit_cost import InformationGainPerUnitCost
        from robo_b200.maximizers.device_spec import raw_inputs as _raw_inputs
        if len(self.estimators) == 0 or not all(isinstance(e, InformationGain) and
                                                not isinstance(e, (InformationGainPerUnitCost, InformationGainMC))
                                                and _raw_inputs(e.model) for e in self.estimators):
            return None
        return [e._ready_handle() for e in self.estimators]

    def _esmc_spec(self):
        """The objective handles of the fused call (gpk_esmc_multi) when every estimator is an InformationGainMC on a
        device GaussianProcess sub-model; raises the estimators' own ValueErrors."""
        from robo_b200.acquisition_functions.information_gain_mc import InformationGainMC
        from robo_b200.maximizers.device_spec import raw_inputs as _raw_inputs
        if len(self.estimators) == 0 or not all(isinstance(e, InformationGainMC) and _raw_inputs(e.model)
                                                for e in self.estimators):
            return None
        return [e._ready_handle() for e in self.estimators]

    def _fused_spec(self):
        """(kind, eta per model, par, handles) when every estimator is a closed-form acquisition on a device GP."""
        if self.cost_model is not None or len(self.estimators) == 0 or not hasattr(self.model, "sub_model_handles"):
            return None
        kinds = set(getattr(e, "kind", None) for e in self.estimators)
        pars = set(float(getattr(e, "par", 0.0)) for e in self.estimators)
        if len(kinds) != 1 or len(pars) != 1 or list(kinds)[0] not in ("ei", "log_ei", "pi", "lcb"):
            return None
        if any(e.model is not m or not hasattr(m, "device_inputs") for e, m in zip(self.estimators, self.model.models)):
            return None
        handles = self.model.sub_model_handles()
        if handles is None or len(handles) != len(self.estimators):
            return None
        kind = list(kinds)[0]
        etas = [0.0 if kind == "lcb" else float(e.model.get_incumbent()[1]) for e in self.estimators]
        return kind, etas, list(pars)[0], handles
