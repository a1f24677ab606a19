"""Differential evolution over the acquisition surface: the device maximizer (robo_b200.maximizers.DifferentialEvolution,
gpk_maximize_de) with and without its L-BFGS-B polish, against scipy.optimize.differential_evolution driven by the
reference's per-point objective (robo/maximizers/differential_evolution.py:27-51: one clipped row per call, -acq,
infinities -> DBL_MAX, scipy's defaults: popsize 15, updating 'immediate', polish) over the SAME robo_b200 acquisition
object.  Three shapes:
  small   N = 30,   D = 2,  gp_mcmc, 10 sub-models, marginalised LogEI
  default N = 200,  D = 16, gp_mcmc, 52 sub-models, marginalised LogEI (the facade default)
  int8    N = 4096, D = 16, one GP, LogEI, popsize 4096 -> P = 65,536 (scoring on the int8 contraction)
Per arm: wall time of maximize() ending in a device synchronise, evaluations, nit, the acquisition value of the
returned point (medians over seeds), and the polish's share of the polished arm's time (same seeds, so the device part
is identical).  Prints one JSON line with the card's name and power limit read in the same run.  Needs a GPU.

    python tools/de_bench.py [--seeds 3] [--shapes small,default,int8] [--no-scipy]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.optimize

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import robo_oracle as O                                    # noqa: E402
from robo_b200 import kernels as K                                     # noqa: E402
from robo_b200.acquisition_functions import LogEI, MarginalizationGPMCMC  # noqa: E402
from robo_b200.maximizers import DifferentialEvolution                 # noqa: E402
from robo_b200.models import GaussianProcess, GaussianProcessMCMC      # noqa: E402
from robo_b200.priors import DefaultPrior                              # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as e:                                             # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def make_problem(shape):
    """-> (acquisition object, lower, upper, popsize of the device arm, description)."""
    N, D = {"small": (30, 2), "default": (200, 16), "int8": (4096, 16)}[shape]
    X, y, _, theta, noise = O.synthetic_problem(N, D, 16, seed_train=7)
    lower, upper = np.zeros(D), np.ones(D)
    if shape == "int8":
        kernel = K.Product(K.ConstantKernel(theta[0], ndim=D), K.Matern52Kernel(np.exp(theta[1:]), ndim=D))
        model = GaussianProcess(kernel, noise=noise, normalize_input=True, lower=lower, upper=upper)
        model.train(X, y, do_optimize=False)
        return LogEI(model), lower, upper, 4096, dict(N=N, D=D, models=1)
    # facade kernel, prior and n_hypers rule (robo/fmin/bayesian_optimization.py:75-87); short chains: the hypers only
    # set the surface
    kernel = 2 * K.Matern52Kernel(np.ones(D), ndim=D)
    n_hypers = 3 * len(kernel)
    n_hypers += n_hypers % 2
    model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)),
                                n_hypers=n_hypers, chain_length=10, burnin_steps=10, normalize_input=True,
                                normalize_output=False, lower=lower, upper=upper, rng=np.random.RandomState(2))
    model.train(X, y, do_optimize=True)
    return MarginalizationGPMCMC(LogEI(model)), lower, upper, 15, dict(N=N, D=D, models=len(model.models))


def sync():
    import torch
    torch.cuda.synchronize()


def acq_value(acq, x):
    return float(np.asarray(acq.compute(np.asarray(x, dtype=np.float64)[None, :])).ravel()[0])


def run_device(acq, lower, upper, popsize, seed, polish):
    de = DifferentialEvolution(acq, lower, upper, popsize=popsize, rng=np.random.RandomState(seed), polish=polish)
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


def median(rows, key):
    return float(np.median([r[key] for r in rows]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=3)
    ap.add_argument("--shapes", default="small,default,int8")
    ap.add_argument("--no-scipy", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("de_bench.py needs a CUDA device")
    name, power = card()
    out = dict(tool="de_bench", gpu=name, power_limit=power, seeds=args.seeds, shapes={})
    for shape in args.shapes.split(","):
        acq, lower, upper, popsize, desc = make_problem(shape)
        run_device(acq, lower, upper, popsize, 12345, False)             # warm-up: module load, scratch, int8 slices
        arms = {"device_nopolish": [], "device_polish": [], "scipy_reference": []}
        for s in range(args.seeds):
            arms["device_nopolish"].append(run_device(acq, lower, upper, popsize, s, False))
            arms["device_polish"].append(run_device(acq, lower, upper, popsize, s, True))
            if not args.no_scipy:
                arms["scipy_reference"].append(run_scipy(acq, lower, upper, s))
        res = dict(desc, pop=max(5, popsize * desc["D"]))
        for arm, rows in arms.items():
            if rows:
                res[arm] = dict(wall_s=median(rows, "s"), nfev=median(rows, "nfev"), nit=median(rows, "nit"),
                                best_acq=median(rows, "acq"))
        pol = [(p["s"] - n["s"]) / p["s"] for p, n in zip(arms["device_polish"], arms["device_nopolish"])]
        res["polish_share"] = float(np.median(pol))
        res["polish_accepted"] = int(sum(r["polished"] for r in arms["device_polish"]))
        if arms["scipy_reference"]:
            res["speedup_vs_scipy_polished"] = res["scipy_reference"]["wall_s"] / res["device_polish"]["wall_s"]
        out["shapes"][shape] = res
        print(json.dumps({shape: res}), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
