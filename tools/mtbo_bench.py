"""MTBO on the device: one JSON line with the card's name and power limit.

  mtbo:      mtbo() at the shape of the reference's experiments/fabolas/run_mtbo.py (D = 2, n_init = 5, n_hypers = 50,
             two tasks) on a cheap synthetic two-task objective, once with the host samplers (the default) and once
             with hyper_sampler = representer_sampler = "device".  Per BO iteration after the initial design: the wall
             time of train (objective and cost models), the acquisition's update and maximize; median and min / max.
  cost_multi: gpk_es_cost_multi (InformationGainPerUnitCost over the marginalised MTBO models, BASIS_TASK input map)
             over 500 and 65,536 candidates; median and min / max over --reps calls.

    python tools/mtbo_bench.py [--iterations 20] [--reps 20] [--arms mtbo,cost_multi]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.fabolas_bench import card, stats, sync  # noqa: E402


def objective(x, task):
    # task 1 is the expensive target, task 0 a cheaper, shifted auxiliary
    shift = 0.1 * (1 - task)
    return float(np.sum((x - 0.3 - shift) ** 2) + 0.01), float(1.0 + 9.0 * task)


def bench_mtbo(iterations, sampler):
    import importlib
    F = importlib.import_module("robo_b200.fmin.mtbo")
    from robo_b200.acquisition_functions import MarginalizationGPMCMC
    from robo_b200.maximizers import RandomSampling
    from robo_b200.models.mtbo_gp import MTBOGPMCMC
    parts = {"train": [], "update": [], "maximize": []}
    pending = {}

    def timed(name, fn, accumulate=False):
        def wrap(*a, **k):
            sync()
            t = time.perf_counter()
            r = fn(*a, **k)
            sync()
            dt = time.perf_counter() - t
            if accumulate:
                pending[name] = pending.get(name, 0.0) + dt
            else:
                parts[name].append(dt)
            return r
        return wrap

    orig = (MTBOGPMCMC.train, MarginalizationGPMCMC.update, RandomSampling.maximize)
    MTBOGPMCMC.train = timed("train", orig[0], accumulate=True)
    MarginalizationGPMCMC.update = timed("update", orig[1])

    def maximize(self):
        parts["train"].append(pending.pop("train", 0.0))
        return timed("maximize", orig[2])(self)
    RandomSampling.maximize = maximize
    try:
        np.random.seed(1)
        t = time.perf_counter()
        F.mtbo(objective, np.zeros(2), np.ones(2), n_tasks=2, n_init=5, num_iterations=iterations, n_hypers=50,
               rng=np.random.RandomState(1), hyper_sampler=sampler, representer_sampler=sampler)
        total = time.perf_counter() - t
    finally:
        MTBOGPMCMC.train, MarginalizationGPMCMC.update, RandomSampling.maximize = orig
    out = {k: stats(v) for k, v in parts.items()}
    out["total_s"] = total
    return out


def bench_cost_multi(reps):
    from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost, MarginalizationGPMCMC
    from robo_b200.fmin.mtbo import _mtbo_kernel
    from robo_b200.models import MTBOGPMCMC
    from robo_b200.priors import MTBOPrior
    rng = np.random.RandomState(0)
    n = 40
    X = np.hstack([rng.rand(n, 2), rng.randint(0, 2, (n, 1))])
    y = np.log(np.array([objective(x[:2], x[2])[0] for x in X]))
    c = np.log(np.array([objective(x[:2], x[2])[1] for x in X]))
    models = []
    for i, t in enumerate((y, c)):
        k, task = _mtbo_kernel(2, 2)
        m = MTBOGPMCMC(k, prior=MTBOPrior(len(k) + 1, 2, len(task), rng=np.random.RandomState(1 + i)), n_hypers=50,
                       chain_length=200, burnin_steps=100, lower=np.zeros(2), upper=np.ones(2),
                       rng=np.random.RandomState(2 + i), hyper_sampler="device")
        m.train(X, t, do_optimize=True)
        models.append(m)
    lo, up = np.zeros(3), np.array([1.0, 1.0, 1.0])
    acq = MarginalizationGPMCMC(InformationGainPerUnitCost(models[0], models[1], lo, up, np.array([0, 0, 1]),
                                                           sampling_acquisition=EI, rng=np.random.RandomState(0),
                                                           representer_sampler="device"))
    np.random.seed(0)
    acq.update(models[0], models[1])
    out = {}
    for m in (500, 65536):
        C = lo + (up - lo) * rng.rand(m, 3)
        for _ in range(3):
            acq.compute(C)
        ts = []
        for _ in range(reps):
            sync()
            t = time.perf_counter()
            acq.compute(C)
            sync()
            ts.append(time.perf_counter() - t)
        out["m%d" % m] = stats(ts)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=20)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--arms", default="mtbo,cost_multi")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mtbo_bench needs a CUDA device")
    name, power = card()
    res = dict(tool="mtbo_bench", gpu=name, power_limit=power)
    arms = args.arms.split(",")
    if "cost_multi" in arms:
        res["es_cost_multi_50x2_models_n40"] = bench_cost_multi(args.reps)
    if "mtbo" in arms:
        res["mtbo_host_samplers"] = bench_mtbo(args.iterations, "host")
        res["mtbo_device_samplers"] = bench_mtbo(args.iterations, "device")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
