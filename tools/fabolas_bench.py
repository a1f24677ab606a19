"""Fabolas on the device: one JSON line with the card's name and power limit.

  fabolas: fabolas() at the reference example's shape (D = 2, s in [100, 50000], default subsets, n_init = 10,
           50 iterations) on a cheap synthetic objective, once with the host samplers (the default) and once with
           hyper_sampler = representer_sampler = "device".  Per BO iteration after the initial design: the wall time
           of train (objective and cost models), the incumbent estimate, the acquisition's update and maximize; median
           and min / max over the iterations.
  ei:      EI + arg-max over 65,536 candidates at N = 2048 (D = 2 plus the environment column) on a model with the
           environment factor, which scores on the fp64 contraction, against the same model with a Matern-5/2 factor
           on the environment column, which takes the int8 contraction; median and min / max over --reps calls.

    python tools/fabolas_bench.py [--iterations 50] [--reps 20] [--arms fabolas,ei]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:
        return "unknown (%s)" % e, "unknown"


def sync():
    import torch
    torch.cuda.synchronize()


def stats(v):
    v = np.asarray(v, dtype=np.float64) * 1e3
    return dict(median_ms=float(np.median(v)), min_ms=float(v.min()), max_ms=float(v.max()), n=int(v.size))


def objective(x, s):
    # the loss grows toward small subsets, the cost with log s
    return float(np.sum((x - 0.3) ** 2) + 50.0 / s + 0.01), float(1.0 + 0.1 * np.log(s))


def bench_fabolas(iterations, sampler):
    import importlib
    F = importlib.import_module("robo_b200.fmin.fabolas")
    from robo_b200.acquisition_functions import MarginalizationGPMCMC
    from robo_b200.maximizers import RandomSampling
    from robo_b200.models.fabolas_gp import FabolasGPMCMC
    parts = {"train": [], "incumbent": [], "update": [], "maximize": []}
    pending = {}

    def timed(name, fn, accumulate=False):
        def wrap(*a, **k):
            sync()
            t = time.perf_counter()
            r = fn(*a, **k)
            sync()
            dt = time.perf_counter() - t
            if accumulate:                          # train: the objective's and the cost's model of one iteration
                pending[name] = pending.get(name, 0.0) + dt
            else:
                parts[name].append(dt)
            return r
        return wrap

    orig = (FabolasGPMCMC.train, F.projected_incumbent_estimation, MarginalizationGPMCMC.update,
            RandomSampling.maximize)
    FabolasGPMCMC.train = timed("train", orig[0], accumulate=True)
    F.projected_incumbent_estimation = timed("incumbent", orig[1])
    MarginalizationGPMCMC.update = timed("update", orig[2])

    def maximize(self):
        parts["train"].append(pending.pop("train", 0.0))
        return timed("maximize", orig[3])(self)
    RandomSampling.maximize = maximize
    try:
        np.random.seed(1)
        t = time.perf_counter()
        F.fabolas(objective, np.zeros(2), np.ones(2), 100, 50000, n_init=10, num_iterations=iterations,
                  rng=np.random.RandomState(1), hyper_sampler=sampler, representer_sampler=sampler)
        total = time.perf_counter() - t
    finally:
        FabolasGPMCMC.train, F.projected_incumbent_estimation, MarginalizationGPMCMC.update, RandomSampling.maximize = orig
    # the last train (the final incumbent's) has no maximize after it
    out = {k: stats(v) for k, v in parts.items()}
    out["total_s"] = total
    return out


def bench_ei(reps):
    from robo_b200 import _lib
    rng = np.random.RandomState(0)
    N, m = 2048, 65536
    X = rng.rand(N, 3)
    X[:, 2] = (1 - X[:, 2]) ** 2
    y = np.sin(3 * X[:, 0]) + X[:, 2] + 0.05 * rng.randn(N)
    C = rng.rand(m, 3)
    out = {}
    for arm in ("env_factor_fp64", "matern_env_int8"):
        h = _lib.Handle(0)
        h.set_data(X, y)
        if arm == "env_factor_fp64":
            h.set_kernel(_lib.MATERN52, 0.0, [0, 1], [0, 1], [-1.0, -1.0])
            h.set_env_factor(2, 0.1, 0.1)
        else:
            h.set_kernel(_lib.MATERN52, 0.0, [0, 1, 2], [0, 1, 2], [-1.0, -1.0, -1.0])
        h.fit(1e-2, float(np.mean(y)))
        eta = float(np.min(y))
        for _ in range(3):
            h.acq(C, _lib.ACQ_EI, eta, 0.0, want_values=False)
        sync()
        before = h.timings()["launches_ozaki"]
        ts = []
        for _ in range(reps):
            sync()
            t = time.perf_counter()
            h.acq(C, _lib.ACQ_EI, eta, 0.0, want_values=False)
            sync()
            ts.append(time.perf_counter() - t)
        r = stats(ts)
        r["int8_contractions"] = h.timings()["launches_ozaki"] - before
        out[arm] = r
        h.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=50)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--arms", default="fabolas,ei")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("fabolas_bench needs a CUDA device")
    name, power = card()
    res = dict(tool="fabolas_bench", gpu=name, power_limit=power)
    arms = args.arms.split(",")
    if "ei" in arms:
        res["ei_65536_n2048"] = bench_ei(args.reps)
    if "fabolas" in arms:
        res["fabolas_host_samplers"] = bench_fabolas(args.iterations, "host")
        res["fabolas_device_samplers"] = bench_fabolas(args.iterations, "device")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
