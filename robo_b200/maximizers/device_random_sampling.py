"""DeviceRandomSampling — RandomSampling (robo/maximizers/random_sampling.py) with the candidates
generated on the GPU (SURVEY.md section 8f rank 2).

Same proposal distribution as the reference: 70 % uniform over the box, 30 % clipped Gaussian
(std 0.1 per coordinate) around the incumbent, uniform part first.  The reference draws from numpy's
global RNG (it ignores its own ``rng`` argument), so its stream cannot be reproduced by anyone; here
candidate i comes from Philox4x32-10 keyed by (seed, i), which makes the result independent of
chunking and of the number of GPUs: with ``world > 1`` every rank scores a contiguous index range and
one 16-byte all_gather settles the arg-max (robo_b200/distributed.py).  Nothing but the winning point
crosses PCIe.

Over a RandomForest, whose predictive std can be exactly 0, EI keeps the reference's batch rule (ei.py:72-74: a zero
std anywhere makes the whole batch [[0]], so RandomSampling's arg-max is row 0): when any candidate has a zero
variance, the first candidate is returned.
"""
import numpy as np

from robo_b200 import _lib
from robo_b200.distributed import allgather_best, pack_pair, shard_bounds
from robo_b200.maximizers.base_maximizer import BaseMaximizer
from robo_b200.maximizers.device_spec import DEVICE_SURROGATES
from robo_b200.models.random_forest import RandomForest


class DeviceRandomSampling(BaseMaximizer):

    def __init__(self, objective_function, lower, upper, n_samples=500, rng=None, rank=0, world=1, group=None):
        self.n_samples = int(n_samples)
        self.rank, self.world, self.group = rank, world, group
        self.calls = 0
        super(DeviceRandomSampling, self).__init__(objective_function, lower, upper, rng)
        self.seed = int(self.rng.randint(0, 2 ** 31 - 1))

    def maximize(self):
        acq = self.objective_func
        model = acq.model
        es = self._es_cost_spec(acq)
        if es is not None:
            return self._maximize_es_cost(acq, es)
        surrogate = isinstance(model, DEVICE_SURROGATES)
        if not surrogate and (not hasattr(model, "gp") or not hasattr(model.gp, "handle")):
            raise TypeError("DeviceRandomSampling needs a robo_b200 GaussianProcess, BayesianLinearRegression, "
                            "RandomForest, WrapperBohamiann or DNGO model")
        if surrogate and self.world > 1:
            raise ValueError("DeviceRandomSampling of a %s runs on one GPU" % type(model).__name__)
        kind = _lib.ACQ_KIND[acq.kind]
        inc_x, inc_y = model.get_incumbent()
        eta = 0.0 if acq.kind == "lcb" else float(inc_y)
        seed = (self.seed + 0x9E3779B97F4A7C15 * self.calls) & 0xFFFFFFFFFFFFFFFF
        self.calls += 1
        # random_sampling.py:38-47: int(0.7 n) uniform points followed by int(0.3 n) Gaussian ones (n = 5 gives 3 + 1)
        n_uniform = int(self.n_samples * .7)
        n_total = n_uniform + int(self.n_samples * .3)
        if surrogate:
            handle = model._ready_handle()
        else:
            model.gp._restore()
            model.gp._push_cfg()
            handle = model.gp.handle
        if self.world > 1 and handle.comm_info()["world"] == self.world:
            # candidates, scoring, exchange and merge behind one C-ABI call (gpk_maximize_random_sharded)
            x, val, idx = handle.maximize_random_sharded(seed, n_total, n_uniform, self.lower, self.upper, inc_x, 0.1,
                                                         kind, eta, acq.par)
        else:
            lo, hi = shard_bounds(n_total, self.rank, self.world)
            if hi > lo:
                x, val, idx = handle.maximize_random(seed, lo, hi - lo, n_uniform, self.lower, self.upper, inc_x, 0.1,
                                                     kind, eta, acq.par)
            else:
                x, val, idx = None, 0.0, -1             # empty shard (world > n_samples): still joins the exchange
            if self.world > 1:
                import torch
                dev = "cuda:%d" % torch.cuda.current_device() if torch.cuda.is_available() else "cpu"
                val, idx = allgather_best(pack_pair(val, idx, dev), self.group)
                x = handle.generate_candidates(seed, idx, 1, n_uniform, self.lower, self.upper, inc_x, 0.1)[0]
        if isinstance(model, RandomForest) and acq.kind == "ei":
            X = handle.generate_candidates(seed, 0, n_total, n_uniform, self.lower, self.upper, inc_x, 0.1)
            if (np.sqrt(model.predict(X)[1]) == 0).any():
                x, val, idx = X[0], 0.0, 0
        self.last = dict(seed=seed, best_idx=idx, best_val=val)
        return x

    def _next_seed(self):
        seed = (self.seed + 0x9E3779B97F4A7C15 * self.calls) & 0xFFFFFFFFFFFFFFFF
        self.calls += 1
        return seed

    @staticmethod
    def _es_cost_spec(acq):
        """The fused call's arguments when acq is an InformationGainPerUnitCost, or a MarginalizationGPMCMC of them."""
        from robo_b200.acquisition_functions.information_gain_per_unit_cost import (InformationGainPerUnitCost,
                                                                                    device_spec)
        if isinstance(acq, InformationGainPerUnitCost):
            return device_spec([acq])
        if hasattr(acq, "_es_cost_spec"):
            return acq._es_cost_spec()
        return None

    def _maximize_es_cost(self, acq, es):
        """Candidates, information gain per unit cost, mean over the model pairs and arg-max in one device call
        (gpk_maximize_random_es_cost); the incumbent as random_sampling.py:42 takes it.  One GPU only."""
        if self.world > 1:
            raise ValueError("DeviceRandomSampling of InformationGainPerUnitCost runs on one GPU")
        ho, hc, lo, up, bo, bc, oh = es
        inc_x = acq.model.get_incumbent()[0]
        seed = self._next_seed()
        n_uniform = int(self.n_samples * .7)
        n_total = n_uniform + int(self.n_samples * .3)
        x, val, idx = _lib.maximize_random_es_cost(ho, hc, seed, n_total, n_uniform, self.lower, self.upper, inc_x, 0.1,
                                                   lo, up, bo, bc, oh)
        self.last = dict(seed=seed, best_idx=idx, best_val=val)
        return x
