"""Multi-start L-BFGS on the device (robo_b200.maximizers.SciPyOptimizer, gpk_maximize_lbfgs*) against the reference's
loop: scipy's L-BFGS-B from the same starts, one after the other, on the single-point objective
(robo/maximizers/scipy_optimizer.py:39-82) over the SAME robo_b200 acquisition object.  Shapes:
  bo       the bayesian_optimization default: Branin, gp_mcmc with 10 sub-models, marginalised LogEI
  default  N = 200, D = 16, gp_mcmc, 52 sub-models, marginalised LogEI (tools/de_bench.py's default shape)
  es       the entropy_search default: marginalised InformationGain (tools/de_es_bench.py)
  fabolas  config 4 Fabolas: marginalised InformationGainPerUnitCost (tools/de_es_bench.py)
Then DifferentialEvolution with polish=True (scipy's L-BFGS-B on the host) against polish="device" at the
tools/de_bench.py shapes.  Every arm is warmed up, then the arms alternate for `rounds` rounds (one seed per round);
wall times end in a device synchronise; medians and spreads (min, max) of the wall time and the best energy.  Prints
one JSON line with the card's name and power limit read in the same run.  Needs a GPU.

    python tools/lbfgs_bench.py [--rounds 3] [--shapes bo,default,es,fabolas] [--de-shapes small,default,int8]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import de_bench as DB                                                  # noqa: E402
import de_es_bench as DEB                                              # noqa: E402
from robo_b200.maximizers import DifferentialEvolution, SciPyOptimizer  # noqa: E402


def make_problem(shape):
    if shape == "bo":
        return _branin_problem()
    if shape == "default":
        acq, lower, upper, _, desc = DB.make_problem("default")
        return acq, lower, upper, desc
    return DEB.make_problem(shape)


def _branin_problem():
    from robo_b200 import kernels as K
    from robo_b200.acquisition_functions import LogEI, MarginalizationGPMCMC
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    rng = np.random.RandomState(4)
    X = DEB.LO + (DEB.UP - DEB.LO) * rng.rand(20, 2)
    y = np.array([DEB.branin(x) for x in X])
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)), n_hypers=10,
                                chain_length=200, burnin_steps=100, normalize_input=True, normalize_output=False,
                                lower=DEB.LO, upper=DEB.UP, rng=np.random.RandomState(2))
    model.train(X, y, do_optimize=True)
    return MarginalizationGPMCMC(LogEI(model)), DEB.LO, DEB.UP, dict(N=20, D=2, models=len(model.models))


def run_scipy_optimizer(acq, lower, upper, seed, device):
    opt = SciPyOptimizer(acq, lower, upper, rng=np.random.RandomState(seed))
    DB.sync()
    t0 = time.perf_counter()
    if device:
        opt.maximize()
    else:
        opt._maximize_host(opt._starts())
    DB.sync()
    return dict(s=time.perf_counter() - t0, energy=float(np.min(opt.last["energy"])))


def run_de(acq, lower, upper, popsize, seed, polish):
    de = DifferentialEvolution(acq, lower, upper, popsize=popsize, rng=np.random.RandomState(seed), polish=polish)
    DB.sync()
    t0 = time.perf_counter()
    de.maximize()
    DB.sync()
    return dict(s=time.perf_counter() - t0, energy=float(de.last["best_energy"]), polished=de.last["polished"])


def stats(rows, key):
    v = [r[key] for r in rows]
    return dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v)))


def arms_result(arms):
    return {a: dict(wall_s=stats(rows, "s"), best_energy=stats(rows, "energy")) for a, rows in arms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="bo,default,es,fabolas")
    ap.add_argument("--de-shapes", default="small,default,int8")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lbfgs_bench.py needs a CUDA device")
    name, power = DB.card()
    out = dict(tool="lbfgs_bench", gpu=name, power_limit=power, rounds=args.rounds, scipy_optimizer={},
               de_polish={})
    for shape in [s for s in args.shapes.split(",") if s]:
        acq, lower, upper, desc = make_problem(shape)
        run_scipy_optimizer(acq, lower, upper, 12345, True)               # warm-up
        arms = {"device": [], "reference_loop": []}
        for s in range(args.rounds):
            arms["device"].append(run_scipy_optimizer(acq, lower, upper, s, True))
            arms["reference_loop"].append(run_scipy_optimizer(acq, lower, upper, s, False))
        res = dict(desc, **arms_result(arms))
        res["speedup"] = res["reference_loop"]["wall_s"]["median"] / res["device"]["wall_s"]["median"]
        out["scipy_optimizer"][shape] = res
        print(json.dumps({shape: res}), file=sys.stderr, flush=True)
    for shape in [s for s in args.de_shapes.split(",") if s]:
        acq, lower, upper, popsize, desc = DB.make_problem(shape)
        run_de(acq, lower, upper, popsize, 12345, "device")               # warm-up
        arms = {"polish_host": [], "polish_device": []}
        for s in range(args.rounds):
            arms["polish_host"].append(run_de(acq, lower, upper, popsize, s, True))
            arms["polish_device"].append(run_de(acq, lower, upper, popsize, s, "device"))
        res = dict(desc, **arms_result(arms))
        res["speedup"] = res["polish_host"]["wall_s"]["median"] / res["polish_device"]["wall_s"]["median"]
        out["de_polish"][shape] = res
        print(json.dumps({"de_" + shape: res}), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
