#!/usr/bin/env python
"""One acquisition update() with the representer points drawn on the host (EnsembleSampler, one scoring call per
estimator and half-step) against the device (gpk_sample_representers, one call for all estimators), at two shapes:

  fabolas   the BASELINE config 4 shape of tools/fabolas_acq_bench.py: N = 2048, 20 objective + 20 cost FabolasGP
            sub-models, MarginalizationGPMCMC(InformationGainPerUnitCost), EI sampling, Nb = 50
  es        the entropy_search default: Branin, 20 training points, a 10-model GP-MCMC ensemble,
            MarginalizationGPMCMC(InformationGain), EI sampling, Nb = 50

Both samplers are warmed up by one update, then `reps` rounds alternate host and device.  Reported per sampler: the
sampling time and the whole update time (median, min, max in ms), and as a quality check the mean and the finite
fraction of the final lmb over all estimators.  Prints one JSON line with the card and its power limit.

    python tools/representer_bench.py [--reps 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import fabolas_acq_bench as FB  # noqa: E402

LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])


def _branin(x):
    return (x[1] - 5.1 / (4 * np.pi ** 2) * x[0] ** 2 + 5 / np.pi * x[0] - 6) ** 2 \
        + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x[0]) + 10


def _es_model():
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    rng = np.random.RandomState(4)
    X = LO + (UP - LO) * rng.rand(20, 2)
    y = np.array([_branin(x) for x in X])
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)),
                                n_hypers=10, chain_length=200, burnin_steps=100, normalize_input=True,
                                normalize_output=False, lower=LO, upper=UP, rng=np.random.RandomState(2))
    model.train(X, y, do_optimize=True)
    return model


def _shape(which, sampler, models):
    from robo_b200.acquisition_functions import EI, InformationGain, InformationGainPerUnitCost, MarginalizationGPMCMC
    if which == "fabolas":
        objm, costm = models
        acq = MarginalizationGPMCMC(InformationGainPerUnitCost(objm, costm, FB.EXT_LO, FB.EXT_UP, np.array([0, 0, 1]),
                                                               sampling_acquisition=EI, rng=np.random.RandomState(0),
                                                               representer_sampler=sampler))
        return acq, lambda: acq.update(objm, costm)
    acq = MarginalizationGPMCMC(InformationGain(models, LO, UP, sampling_acquisition=EI, rng=np.random.RandomState(0),
                                                representer_sampler=sampler))
    return acq, lambda: acq.update(models)


def _timed_update(acq, update, sampling):
    """One update(); the time spent drawing representer points is added to sampling[-1]."""
    import robo_b200.acquisition_functions.information_gain as IG
    sampling.append(0.0)
    real_dev = IG.sample_representers_device
    real_host = {}

    def dev(estimators):
        t = time.perf_counter()
        try:
            return real_dev(estimators)
        finally:
            sampling[-1] += time.perf_counter() - t
    IG.sample_representers_device = dev
    for e in acq.estimators:
        if e.representer_sampler == "host":
            real_host[id(e)] = e.sample_representer_points

            def host(e=e):
                t = time.perf_counter()
                try:
                    return real_host[id(e)]()
                finally:
                    sampling[-1] += time.perf_counter() - t
            e.sample_representer_points = host
    try:
        t0 = time.perf_counter()
        update()
        return time.perf_counter() - t0
    finally:
        IG.sample_representers_device = real_dev
        for e in acq.estimators:
            e.__dict__.pop("sample_representer_points", None)


def _stats(ts):
    ts = np.array(ts) * 1e3
    return dict(median_ms=float(np.median(ts)), min_ms=float(ts.min()), max_ms=float(ts.max()), n=int(ts.size))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="fabolas,es")
    a = ap.parse_args()
    name, limit = FB._card()
    out = dict(card=name, power_limit=limit, reps=a.reps)
    for which in a.shapes.split(","):
        models = FB._models() if which == "fabolas" else _es_model()
        arms = {s: _shape(which, s, models) for s in ("host", "device")}
        for acq, update in arms.values():
            np.random.seed(0)
            update()                                             # warm-up
        upd = {s: [] for s in arms}
        smp = {s: [] for s in arms}
        for _ in range(a.reps):
            for s, (acq, update) in arms.items():
                upd[s].append(_timed_update(acq, update, smp[s]))
        res = {}
        for s, (acq, _) in arms.items():
            lmb = np.concatenate([np.ravel(e.lmb) for e in acq.estimators])
            fin = np.isfinite(lmb)
            res[s] = dict(update=_stats(upd[s]), sampling=_stats(smp[s]), lmb_mean=float(np.mean(lmb[fin])),
                          lmb_finite_fraction=float(fin.mean()))
        res["sampling_speedup"] = res["host"]["sampling"]["median_ms"] / res["device"]["sampling"]["median_ms"]
        res["n_models"] = len(arms["host"][0].estimators)
        out[which] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
