#!/usr/bin/env python
"""Information gain per unit cost at the BASELINE config 4 shape: N = 2048 training points with two configuration
columns and the environment column, 20 objective + 20 cost FabolasGP sub-models (FabolasGPMCMC, short chains),
MarginalizationGPMCMC(InformationGainPerUnitCost).  Prints one JSON line with the card and its power limit.

  update     one acq.update(objective, cost) after a warm-up update, split into the representer sampling (the EI
             ensemble sampler of the 20 estimators) and the rest (es_update: predict(zb, full_cov), EP, U)
  maximize   the candidate batch (500, the reference's RandomSampling default, and 65,536) scored in three arms:
             (a) fused: one gpk_es_cost_multi call over the 20 pairs
             (b) the reference's per-estimator loop with the device models: es_compute + cost predict + numpy ratio
             (c) fused, but the cost models' mean through the full scoring pass (option "meanonly" = 0)
             Each arm is warmed up, then the arms alternate for `reps` rounds; the median and the spread (min, max) of
             the wall time per call are reported.  The outputs are compared across the arms.

    python tools/fabolas_acq_bench.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LO, UP = np.array([0.0, 0.0]), np.array([1.0, 1.0])
EXT_LO, EXT_UP = np.append(LO, 0.0), np.append(UP, 1.0)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, limit = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return "unknown", "unknown"


class _Prior(object):
    def __init__(self, r):
        self.r = r

    def lnprob(self, t):
        return 0.0 if np.all(np.abs(t) < 6) else -np.inf

    def sample_from_prior(self, n):
        return self.r.uniform(-2, 1, size=(n, 5))


def _kernel(amp, ls):
    from robo_b200 import kernels as K
    k = amp * K.Matern52Kernel(np.ones(1) * ls[0], ndim=3, axes=0)
    k *= K.Matern52Kernel(np.ones(1) * ls[1], ndim=3, axes=1)
    k *= K.Matern52Kernel(np.ones(1) * ls[2], ndim=3, axes=2)
    return k


def _models(n=2048, n_hypers=20):
    from robo_b200.models import FabolasGPMCMC
    rng = np.random.RandomState(0)
    X = np.concatenate((rng.rand(n, 2), rng.uniform(0.05, 1.0, (n, 1))), axis=1)
    y = np.sin(6 * X[:, 0]) + X[:, 1] ** 2 + (1 - X[:, 2]) ** 2 + 0.01 * rng.randn(n)
    c = -1.0 + 2.5 * X[:, 2] + 0.2 * X[:, 0] + 0.01 * rng.randn(n)
    objm = FabolasGPMCMC(_kernel(1.0, (0.3, 0.3, 0.5)), basis_func=lambda s: (1 - s) ** 2,
                         prior=_Prior(np.random.RandomState(1)), n_hypers=n_hypers, chain_length=4, burnin_steps=3,
                         lower=LO, upper=UP, rng=np.random.RandomState(2))
    objm.train(X, y, do_optimize=True)
    costm = FabolasGPMCMC(_kernel(1.0, (0.4, 0.4, 0.5)), basis_func=lambda s: s, prior=_Prior(np.random.RandomState(3)),
                          n_hypers=n_hypers, chain_length=4, burnin_steps=3, lower=LO, upper=UP,
                          rng=np.random.RandomState(4))
    costm.train(X, c, do_optimize=True)
    return objm, costm


def _stats(ts):
    ts = np.array(ts) * 1e3
    return dict(median_ms=float(np.median(ts)), min_ms=float(ts.min()), max_ms=float(ts.max()), n=int(ts.size))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from robo_b200 import _lib
    from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost, MarginalizationGPMCMC
    name, limit = _card()
    objm, costm = _models()
    acq = MarginalizationGPMCMC(InformationGainPerUnitCost(objm, costm, EXT_LO, EXT_UP, np.array([0, 0, 1]),
                                                           sampling_acquisition=EI, rng=np.random.RandomState(0)))
    np.random.seed(0)
    acq.update(objm, costm)                                    # warm-up
    sampling = []
    for e in acq.estimators:
        def timed(e=e, f=e.sample_representer_points):
            t = time.perf_counter()
            f()
            sampling.append(time.perf_counter() - t)
        e.sample_representer_points = timed
    t0 = time.perf_counter()
    acq.update(objm, costm)
    t_update = time.perf_counter() - t0
    t_sampling = float(np.sum(sampling))
    ho, hc, lo, up, bo, bc, oh = acq._es_cost_spec()

    def arm_a(C):
        return _lib.es_cost_multi(ho, hc, C, lo, up, bo, bc, oh)["values"]

    def arm_b(C):
        inside = np.all((C >= EXT_LO) & (C <= EXT_UP), axis=1)
        vals = np.zeros((len(acq.estimators), len(C)))
        for i, e in enumerate(acq.estimators):
            dh = e.model.gp.handle.es_compute(e.model.normalize(C))
            dh[~inside] = np.spacing(1)
            vals[i] = dh / (np.exp(e.cost_model.predict(C)[0]) + e.overhead)
        return vals.mean(axis=0)

    def arm_c(C):
        for h in hc:
            h.set_option("meanonly", 0)
        try:
            return arm_a(C)
        finally:
            for h in hc:
                h.set_option("meanonly", 1)

    arms = dict(fused=arm_a, per_estimator_loop=arm_b, fused_cost_full_pass=arm_c)
    rng = np.random.RandomState(5)
    maximize = {}
    for m in (500, 65536):
        C = EXT_LO + (EXT_UP - EXT_LO) * rng.rand(m, 3)
        out = {k: f(C) for k, f in arms.items()}               # warm-up, and the outputs compared below
        times = {k: [] for k in arms}
        for _ in range(a.reps):
            for k, f in arms.items():
                torch.cuda.synchronize()
                t = time.perf_counter()
                f(C)
                times[k].append(time.perf_counter() - t)
        ref = out["fused"]
        ok = np.isfinite(ref)
        scale = np.maximum(np.abs(ref), 1e-300)
        maximize[str(m)] = dict(
            {k: _stats(v) for k, v in times.items()},
            argmax_equal=all(int(np.argmax(v)) == int(np.argmax(ref)) for v in out.values()),
            max_rel_diff_loop=float(np.max(np.abs(out["per_estimator_loop"][ok] - ref[ok]) / scale[ok])),
            max_rel_diff_cost_full_pass=float(np.max(np.abs(out["fused_cost_full_pass"][ok] - ref[ok]) / scale[ok])),
            finite=int(ok.sum()))
    print(json.dumps(dict(card=name, power_limit=limit, n_train=2048, n_models=len(acq.estimators), nb=acq.estimators[0].Nb,
                          np=acq.estimators[0].Np,
                          update=dict(total_ms=t_update * 1e3, representer_sampling_ms=t_sampling * 1e3,
                                      es_update_ms=(t_update - t_sampling) * 1e3),
                          maximize=maximize)))


if __name__ == "__main__":
    main()
