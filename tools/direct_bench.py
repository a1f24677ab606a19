"""DIRECT over the acquisition surface: the device maximizer (robo_b200.maximizers.Direct, gpk_maximize_direct) against
the reference's cost structure, scipy.optimize.direct (a C translation of the same Gablonsky DIRECT 2.0.4 code) with
locally_biased=False, eps=1e-4, vol_tol=0, len_tol=0, f_min=-inf, driven by the one-point objective of
robo/maximizers/direct.py:50-54 (-acq of a single row per call) over the SAME robo_b200 acquisition object.  Both arms
run the reference's defaults (n_func_evals = 400, n_iters = 200) on the shapes of tools/cmaes_bench.py:
  bo       Branin, gp_mcmc, 10 sub-models, marginalised LogEI (the bayesian_optimization default)
  default  N = 200, D = 16, gp_mcmc, 52 sub-models, marginalised LogEI (the facade default)
  es       InformationGain over 10 sub-models (the entropy_search default)
  fabolas  InformationGainPerUnitCost over 20 (objective, cost) pairs (config 4 Fabolas)
Rounds alternate the arms; per arm: median [min, max] wall time of one maximize() ending in a device synchronise,
evaluations, iterations and the best energy, and whether the two arms made the same run (the same evaluations,
iterations and returned x; a batched pass and a single-row call may differ in the last bits, which can change a
choice).  Prints one JSON line with the card's name and
power limit read in the same run.  Needs a GPU.

    python tools/direct_bench.py [--rounds 3] [--shapes bo,default,es,fabolas]
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
from robo_b200.maximizers import Direct                                # noqa: E402


def _sync():
    import torch
    torch.cuda.synchronize()


def device_arm(acq, lower, upper):
    dr = Direct(acq, lower, upper, verbose=False)
    _sync()
    t = time.perf_counter()
    x = dr.maximize()
    _sync()
    return time.perf_counter() - t, dr.last["nfev"], dr.last["nit"], dr.last["best_energy"], x


def host_arm(acq, lower, upper):
    from scipy.optimize import direct
    pts = []

    def one_row(x):
        pts.append(np.array(x))
        return -float(np.asarray(acq.compute(np.array([x]))).ravel()[0])
    _sync()
    t = time.perf_counter()
    r = direct(one_row, list(zip(lower, upper)), eps=1e-4, maxfun=400, maxiter=200, locally_biased=False,
               vol_tol=0.0, len_tol=0.0, f_min=-np.inf)
    _sync()
    return time.perf_counter() - t, int(r.nfev), int(r.nit), float(r.fun), np.asarray(r.x)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="bo,default,es,fabolas")
    args = ap.parse_args()
    name, power = de_bench.card()
    out = dict(tool="direct_bench", gpu=name, power_limit=power, shapes={})
    for shape in [s for s in args.shapes.split(",") if s]:
        acq, lower, upper, desc = lbfgs_bench.make_problem(shape)
        device_arm(acq, lower, upper)                                  # warm-up: module load, buffer sizing
        res = {"device": [], "host_single_row": []}
        for _ in range(args.rounds):
            res["device"].append(device_arm(acq, lower, upper))
            res["host_single_row"].append(host_arm(acq, lower, upper))
        summary = dict(desc)
        for arm, rows in res.items():
            t = np.array([row[0] for row in rows]) * 1e3
            summary[arm] = dict(ms_median=float(np.median(t)), ms_min=float(t.min()), ms_max=float(t.max()),
                                nfev=[int(row[1]) for row in rows], nit=[int(row[2]) for row in rows],
                                best_energy=[float(row[3]) for row in rows])
        dev, host = res["device"][-1], res["host_single_row"][-1]
        summary["same_run"] = bool(dev[1] == host[1] and dev[2] == host[2] and np.array_equal(dev[4], host[4]))
        summary["speedup_median"] = summary["host_single_row"]["ms_median"] / summary["device"]["ms_median"]
        out["shapes"][shape] = summary
    print(json.dumps(out))


if __name__ == "__main__":
    main()
