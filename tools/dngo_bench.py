"""DNGO on the device, at three shapes:

  ref       D = 2, N = 10 (the reference test's size)
  branin    Branin, D = 2, N = 30
  d8        D = 8, N = 200

Rows, each timing ending in a device synchronise:
  train     DNGO.train at the defaults (500 epochs of batches of 10, 20 walkers, 2000 burn-in + 2000 chain steps): the
            first train (network + burn-in + chain) and a later one (one more row: network + chain)
  ei        EI over 65,536 and over 2^20 candidates with the arg-max (gpk_acq_multi)
  de        DifferentialEvolution.maximize, 20 generations
  kernel    gpk_dngo_score_kernel's time per 2^20 candidates under torch.profiler (a separate run, EI with the arg-max)
Host arm (--host, the ref shape only): tests/dngo_model.torch_train (pybnn's loop restated in torch, float64, CPU) and the
host EnsembleSampler over tests/blr_model's log-posterior of the features, the burn-in and the chain, as a first train.
One untimed warm-up of every device row per shape, then --rounds rounds; median, [min, max].  Prints one JSON line per round and a
summary line, each with the card's name and power limit read in the same call.

    python tools/dngo_bench.py [--rounds 3] [--shapes ref,branin,d8] [--host] [--out dngo_bench.json]
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

from robo_b200 import _lib  # noqa: E402
from robo_b200.acquisition_functions import EI  # noqa: E402
from robo_b200.maximizers import DifferentialEvolution  # noqa: E402
from robo_b200.models import DNGO  # noqa: E402

SHAPES = {"ref": (2, 10), "branin": (2, 30), "d8": (8, 200)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:
        return "unknown (%s)" % e, "unknown"


def data(shape):
    d, n = SHAPES[shape]
    rng = np.random.RandomState(42)
    if shape == "branin":
        X = rng.rand(n + 1, 2) * [15, 15] - [5, 0]
        x1, x2 = X[:, 0], X[:, 1]
        y = (x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x1) + 10
        return X, y, np.array([-5.0, 0.0]), np.array([10.0, 15.0])
    X = rng.rand(n + 1, d)
    return X, np.sinc(X * 10 - 5).sum(axis=1), np.zeros(d), np.ones(d)


def sync():
    import torch
    torch.cuda.synchronize()


def device_train(shape, seed):
    X, y, _, _ = data(shape)
    m = DNGO(rng=np.random.RandomState(seed))
    times = []
    for rows in (len(X) - 1, len(X)):
        t0 = time.perf_counter()
        m.train(X[:rows], y[:rows])
        sync()
        times.append(time.perf_counter() - t0)
    return times, m


def device_ei(model, Xc, eta):
    h = model._ready_handle()
    t0 = time.perf_counter()
    r = _lib.acq_multi([h], Xc, 0, kind=_lib.ACQ_EI, eta=[eta], par=0.0, want_argmax=True)
    sync()
    return time.perf_counter() - t0, int(r["best_idx"])


def device_de(model, lo, up, seed):
    acq = EI(model)
    mx = DifferentialEvolution(acq, lo, up, n_iters=20, rng=np.random.RandomState(seed))
    t0 = time.perf_counter()
    x = mx.maximize()
    sync()
    return time.perf_counter() - t0, float(np.ravel(acq.compute(np.atleast_2d(x)))[0])


def kernel_time(model, Xc, eta, reps=5):
    """gpk_dngo_score_kernel's mean time per call over reps EI passes, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    h = model._ready_handle()
    _lib.acq_multi([h], Xc, 0, kind=_lib.ACQ_EI, eta=[eta], par=0.0, want_argmax=True)
    sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            _lib.acq_multi([h], Xc, 0, kind=_lib.ACQ_EI, eta=[eta], par=0.0, want_argmax=True)
        torch.cuda.synchronize()
    total, count = 0.0, 0
    for ev in prof.events():
        if "gpk_dngo_score_kernel" in ev.name:
            total += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            count += 1
    return total / max(count, 1) / 1e3, count              # ms per launch (a 2^20 batch may span several launches)


def host_train(shape, seed):
    """pybnn's network loop in torch (float64, CPU) and the host ensemble sampler over the features, as a first train."""
    import torch
    from robo_b200.priors import BayesianLinearRegressionPrior
    from robo_b200.util.ensemble_sampler import EnsembleSampler
    from tests import blr_model as LM
    from tests import dngo_model as DM
    torch.set_num_threads(os.cpu_count() or 1)
    X, y, _, _ = data(shape)
    X, y = X[:-1], y[:-1]
    rng = np.random.RandomState(seed)
    t0 = time.perf_counter()
    theta, Theta, (xm, xs, ym, ysd) = DM.torch_train(X, y, seed)
    t_net = time.perf_counter() - t0
    ys = (y - ym) / ysd
    s = EnsembleSampler(20, 2, None, batch_lnpostfn=LM.lnpost(Theta, ys))
    p0 = BayesianLinearRegressionPrior(rng=rng).sample_from_prior(20)
    p0, _, _ = s.run_mcmc(p0, 2000, rstate0=rng)
    s.run_mcmc(p0, 2000, rstate0=rng)
    return t_net, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="ref,branin,d8")
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    name, power = card()
    summary = dict(card=name, power_limit=power, shapes={})
    for shape in args.shapes.split(","):
        rows = []
        X, y, lo, up = data(shape)
        eta = float(np.min(y))
        _, warm = device_train(shape, 99)              # warm-up (module load, first launches) of every timed call
        for M in (65536, 1 << 20):
            device_ei(warm, lo + (up - lo) * np.random.RandomState(M).rand(M, len(lo)), eta)
        device_de(warm, lo, up, 99)
        for rnd in range(1, args.rounds + 1):
            seed = 100 + rnd
            res = {}
            res["train"], model = device_train(shape, seed)
            rs = np.random.RandomState(seed)
            for M in (65536, 1 << 20):
                Xc = lo + (up - lo) * rs.rand(M, len(lo))
                res["ei_%d" % M], _ = device_ei(model, Xc, eta)
            res["de"], res["de_value"] = device_de(model, lo, up, seed)
            if args.host and shape == "ref":
                res["host_net"], res["host_train"] = host_train(shape, seed)
            line = dict(card=name, power_limit=power, shape=shape, round=rnd, **res)
            print(json.dumps(line), flush=True)
            rows.append(res)
        Xc = lo + (up - lo) * np.random.RandomState(7).rand(1 << 20, len(lo))
        kt, launches = kernel_time(model, Xc, eta)

        def stat(key, i=None):
            v = np.array([r[key][i] if i is not None else r[key] for r in rows])
            return dict(median=float(np.median(v)), min=float(v.min()), max=float(v.max()))
        out = dict(train_first=stat("train", 0), train_later=stat("train", 1), ei_65536=stat("ei_65536"),
                   ei_1048576=stat("ei_1048576"), de_20=stat("de"),
                   score_kernel_ms_per_launch=kt, score_kernel_launches_per_2p20=launches / 5.0)
        if "host_train" in rows[0]:
            out["host_net"], out["host_train_first"] = stat("host_net"), stat("host_train")
        summary["shapes"][shape] = out
    print(json.dumps(dict(summary=summary)), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
