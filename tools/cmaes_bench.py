"""CMA-ES over the acquisition surface: the device maximizer (robo_b200.maximizers.CMAES, gpk_maximize_cmaes) against
the reference's cost structure, the same restated algorithm (tests/cmaes_model.py) on the host with one single-row
acquisition call per evaluation, as robo/maximizers/cmaes.py:66-68 hands cma.fmin.  Both arms run the reference's
defaults (n_func_evals = 1000, restarts = 0, sigma0 = 0.6) over the SAME robo_b200 acquisition object, on the shapes of
tools/lbfgs_bench.py:
  bo       Branin, gp_mcmc, 10 sub-models, marginalised LogEI (the bayesian_optimization default)
  default  N = 200, D = 16, gp_mcmc, 52 sub-models, marginalised LogEI (the facade default)
  es       InformationGain over 10 sub-models (the entropy_search default)
  fabolas  InformationGainPerUnitCost over 20 (objective, cost) pairs (config 4 Fabolas)
Rounds alternate the arms; per arm: median [min, max] wall time of one maximize() ending in a device synchronise,
evaluations, generations and the best energy.
The kernel arm (--kernels) runs the device maximizer alone on one GP at D = 2, 16 and 64 (LCB, the reference
defaults) under torch.profiler and reports the mean device time of each CMA-ES kernel per launch: at these D purecma's
eigendecomposition gap is below lambda, so every gpk_cmaes_update_kernel launch runs the Jacobi sweeps, and its time
at D = 64 against D = 16 is their cost.  Prints one JSON line with the card's name and power limit read in the same
run.  Needs a GPU.

    python tools/cmaes_bench.py [--rounds 3] [--shapes bo,default,es,fabolas] [--kernels]
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

import de_bench                                                        # noqa: E402
import lbfgs_bench                                                     # noqa: E402
from robo_b200.maximizers import CMAES                                 # noqa: E402
from tests import cmaes_model                                          # noqa: E402


def _sync():
    import torch
    torch.cuda.synchronize()


def device_arm(acq, lower, upper, seed):
    cm = CMAES(acq, lower, upper, verbose=False, rng=np.random.RandomState(seed))
    _sync()
    t = time.perf_counter()
    cm.maximize()
    _sync()
    return time.perf_counter() - t, cm.last["nfev"], int(cm.last["nit"].sum()), cm.last["best_energy"]


def host_arm(acq, lower, upper, seed):
    rng = np.random.RandomState(seed)
    rng.randint(0, 2 ** 31 - 1)
    x0 = lower + (upper - lower) * rng.uniform(size=lower.size)
    calls = [0]

    def per_row(P):
        calls[0] += len(P)
        return np.array([float(np.asarray(acq.compute(p[None, :])).ravel()[0]) for p in P])
    _sync()
    t = time.perf_counter()
    r = cmaes_model.run(per_row, cmaes_model.numpy_normals(seed), x0, lower, upper, 1000, 0)
    _sync()
    return time.perf_counter() - t, calls[0], int(r["nit"].sum()), r["energy"]


def kernel_arm(d):
    """Mean device time per launch of each CMA-ES kernel in one maximize() on a single GP of input dimension d."""
    from torch.profiler import ProfilerActivity, profile
    from oracle import robo_oracle as O
    from robo_b200.acquisition_functions import LCB
    from robo_b200.models import GaussianProcess
    from tests.product_cases import product_kernel
    X, y, _, theta, noise = O.synthetic_problem(200, d, 16, seed_train=3)
    model = GaussianProcess(product_kernel("matern52", theta, d), noise=noise, normalize_input=False)
    model.train(X, y, do_optimize=False)
    lower, upper = np.zeros(d), np.ones(d)
    device_arm(LCB(model), lower, upper, 98)                           # warm-up
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cm = CMAES(LCB(model), lower, upper, verbose=False, rng=np.random.RandomState(0))
        cm.maximize()
        _sync()
    out = dict(D=d, generations=int(cm.last["nit"].sum()), nfev=int(cm.last["nfev"]))
    for ev in prof.key_averages():
        if "gpk_cmaes" in ev.key:
            name = ev.key.split("(")[0].replace("void ", "")
            total = getattr(ev, "device_time_total", None)
            if total is None:
                total = ev.cuda_time_total
            out[name] = dict(launches=int(ev.count), us_per_launch=float(total) / max(ev.count, 1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="bo,default,es,fabolas")
    ap.add_argument("--kernels", action="store_true")
    args = ap.parse_args()
    name, power = de_bench.card()
    out = dict(tool="cmaes_bench", gpu=name, power_limit=power, shapes={})
    if args.kernels:
        out["kernels"] = [kernel_arm(d) for d in (2, 16, 64)]
    for shape in [s for s in args.shapes.split(",") if s]:
        acq, lower, upper, desc = lbfgs_bench.make_problem(shape)
        device_arm(acq, lower, upper, 99)                              # warm-up: module load, buffer sizing
        res = {"device": [], "host_single_row": []}
        for r in range(args.rounds):
            res["device"].append(device_arm(acq, lower, upper, r))
            res["host_single_row"].append(host_arm(acq, lower, upper, r))
        summary = dict(desc)
        for arm, rows in res.items():
            t = np.array([row[0] for row in rows]) * 1e3
            summary[arm] = dict(ms_median=float(np.median(t)), ms_min=float(t.min()), ms_max=float(t.max()),
                                nfev=[int(row[1]) for row in rows], generations=[row[2] for row in rows],
                                best_energy=[float(row[3]) for row in rows])
        summary["speedup_median"] = summary["host_single_row"]["ms_median"] / summary["device"]["ms_median"]
        out["shapes"][shape] = summary
    print(json.dumps(out))


if __name__ == "__main__":
    main()
