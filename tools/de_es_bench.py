#!/usr/bin/env python
"""Differential evolution over the information-gain acquisitions: the device maximizer
(robo_b200.maximizers.DifferentialEvolution -> gpk_maximize_de_es / gpk_maximize_de_es_cost) with and without its
L-BFGS-B polish, against scipy.optimize.differential_evolution(maxiter=20) driven by the reference's per-point objective
(robo/maximizers/differential_evolution.py:27-34: one clipped row per call, -acq, infinities -> DBL_MAX, scipy's other
defaults) over the SAME acquisition object.  Two shapes:
  es      the entropy_search facade default: Branin, D = 2, gp_mcmc with 10 sub-models,
          MarginalizationGPMCMC(InformationGain), Nb = 50, Np = 400
  fabolas the config 4 Fabolas shape: N = 2048, two configuration columns and the environment column, 20 objective +
          20 cost sub-models, MarginalizationGPMCMC(InformationGainPerUnitCost) (models of tools/fabolas_acq_bench.py)
For the es shape also the marginalised entropy change of a candidate batch (500, the reference's RandomSampling
default, and 65,536): one gpk_es_multi call against the per-estimator loop (gpk_es_compute per sub-model, then
gpk_reduce_models), with the outputs compared bit for bit.
Every arm is warmed up, then the arms alternate for `rounds` rounds (one seed per round); medians and spreads (min, max)
of the wall time, ending in a device synchronise, are reported, with the acquisition value of the returned point and the
polish's share of the polished arm's time (same seed, so the device part is identical).  Prints one JSON line with the
card's name and power limit read in the same run.  Needs a GPU.

    python tools/de_es_bench.py [--rounds 5] [--shapes es,fabolas] [--no-scipy]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import scipy.optimize

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import fabolas_acq_bench as FB                                         # noqa: E402
from de_bench import card                                              # noqa: E402

LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])


def branin(x):
    return (x[1] - 5.1 / (4 * np.pi ** 2) * x[0] ** 2 + 5 / np.pi * x[0] - 6) ** 2 \
        + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x[0]) + 10


def make_problem(shape):
    """-> (updated acquisition, lower, upper, description)."""
    from robo_b200 import kernels as K
    from robo_b200.acquisition_functions import EI, InformationGain, InformationGainPerUnitCost, MarginalizationGPMCMC
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    if shape == "es":
        rng = np.random.RandomState(4)
        X = LO + (UP - LO) * rng.rand(20, 2)
        y = np.array([branin(x) for x in X])
        kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)           # robo/fmin/entropy_search.py's kernel and prior
        model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)),
                                    n_hypers=10, chain_length=200, burnin_steps=100, normalize_input=True,
                                    normalize_output=False, lower=LO, upper=UP, rng=np.random.RandomState(2))
        model.train(X, y, do_optimize=True)
        acq = MarginalizationGPMCMC(InformationGain(model, LO, UP, sampling_acquisition=EI,
                                                    rng=np.random.RandomState(0)))
        np.random.seed(0)
        acq.update(model)
        return acq, LO, UP, dict(N=20, D=2, models=len(acq.estimators), nb=50, np=400)
    objm, costm = FB._models()
    acq = MarginalizationGPMCMC(InformationGainPerUnitCost(objm, costm, FB.EXT_LO, FB.EXT_UP, np.array([0, 0, 1]),
                                                           sampling_acquisition=EI, rng=np.random.RandomState(0)))
    np.random.seed(0)
    acq.update(objm, costm)
    return acq, FB.EXT_LO, FB.EXT_UP, dict(N=2048, D=3, models=len(acq.estimators), nb=50, np=400)


def sync():
    import torch
    torch.cuda.synchronize()


def acq_value(acq, x):
    return float(np.asarray(acq.compute(np.asarray(x, dtype=np.float64)[None, :])).ravel()[0])


def run_device(acq, lower, upper, seed, polish):
    from robo_b200.maximizers import DifferentialEvolution
    de = DifferentialEvolution(acq, lower, upper, rng=np.random.RandomState(seed), polish=polish)
    sync()
    t0 = time.perf_counter()
    x = de.maximize()
    sync()
    t = time.perf_counter() - t0
    return dict(s=t, nfev=de.last["nfev"], nit=de.last["nit"], acq=acq_value(acq, x), polished=de.last["polished"])


def run_scipy(acq, lower, upper, seed):
    def objective(x):                                                  # differential_evolution.py:27-34
        a = -np.asarray(acq(np.array([np.clip(x, lower, upper)])), dtype=np.float64)
        if np.any(np.isinf(a)):
            return sys.float_info.max
        return float(a.ravel()[0])
    sync()
    t0 = time.perf_counter()
    res = scipy.optimize.differential_evolution(objective, list(zip(lower, upper)), maxiter=20,
                                                rng=np.random.default_rng(seed))
    x = np.clip(res.x, lower, upper)
    sync()
    t = time.perf_counter() - t0
    return dict(s=t, nfev=int(res.nfev), nit=int(res.nit), acq=acq_value(acq, x))


def stats(rows, key="s"):
    v = np.array([r[key] for r in rows], dtype=np.float64)
    return dict(median=float(np.median(v)), min=float(v.min()), max=float(v.max()), n=int(v.size))


def batch_arms(acq, rounds):
    """gpk_es_multi against the per-estimator loop at 500 and 65,536 candidates."""
    from robo_b200 import _lib
    handles = acq._es_spec()
    arms = dict(fused=lambda C: _lib.es_multi(handles, C)["values"],
                per_estimator_loop=lambda C: _lib.moments_handle().reduce_models(np.array([h.es_compute(C)
                                                                                           for h in handles])))
    rng = np.random.RandomState(5)
    out = {}
    for m in (500, 65536):
        C = LO + (UP - LO) * rng.rand(m, 2)
        vals = {k: f(C) for k, f in arms.items()}                      # warm-up, and the outputs compared below
        times = {k: [] for k in arms}
        for _ in range(rounds):
            for k, f in arms.items():
                sync()
                t = time.perf_counter()
                f(C)
                times[k].append(dict(s=time.perf_counter() - t))
        out[str(m)] = dict({k: stats(v) for k, v in times.items()},
                           bit_identical=vals["fused"].tobytes() == vals["per_estimator_loop"].tobytes())
        out[str(m)]["speedup"] = out[str(m)]["per_estimator_loop"]["median"] / out[str(m)]["fused"]["median"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--shapes", default="es,fabolas")
    ap.add_argument("--no-scipy", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("de_es_bench.py needs a CUDA device")
    name, power = card()
    out = dict(tool="de_es_bench", gpu=name, power_limit=power, rounds=args.rounds, shapes={})
    for shape in args.shapes.split(","):
        acq, lower, upper, desc = make_problem(shape)
        run_device(acq, lower, upper, 12345, False)                    # warm-up: module load, scratch
        arms = {"device_nopolish": [], "device_polish": [], "scipy_reference": []}
        for s in range(args.rounds):
            arms["device_nopolish"].append(run_device(acq, lower, upper, s, False))
            arms["device_polish"].append(run_device(acq, lower, upper, s, True))
            if not args.no_scipy:
                arms["scipy_reference"].append(run_scipy(acq, lower, upper, s))
        res = dict(desc, pop=15 * desc["D"])
        for arm, rows in arms.items():
            if rows:
                res[arm] = dict(wall_s=stats(rows), nfev=stats(rows, "nfev")["median"], nit=stats(rows, "nit")["median"],
                                best_acq=stats(rows, "acq"))
        pol = [(p["s"] - n["s"]) / p["s"] for p, n in zip(arms["device_polish"], arms["device_nopolish"])]
        res["polish_share"] = float(np.median(pol))
        res["polish_accepted"] = int(sum(r["polished"] for r in arms["device_polish"]))
        if arms["scipy_reference"]:
            res["speedup_vs_scipy_polished"] = res["scipy_reference"]["wall_s"]["median"] / \
                res["device_polish"]["wall_s"]["median"]
        if shape == "es":
            res["batch"] = batch_arms(acq, args.rounds)
        out["shapes"][shape] = res
        print(json.dumps({shape: res}), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
