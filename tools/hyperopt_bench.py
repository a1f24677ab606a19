"""GaussianProcess.train with hyper_optimizer "host" (scipy L-BFGS-B, one gpk_fit per nll) against "device"
(gpk_optimize_hypers), one JSON line per row on stdout.

Rows: the bayesian_optimization(model_type="gp") default (Branin, D = 2, N = 30, DefaultPrior, cov_amp = 2), N = 200
at D = 8, N = 232 at D = 16, and an MTBOGP with the task factor; each timed at the first train and at a later one
(N + 1 points, starting from the previous optimum), arms alternating after a warm-up, every timing ending in a device
synchronise.  Then one whole bayesian_optimization(model_type="gp", num_iterations=30) per arm.  --profile times the
round kernel alone with torch.profiler (a separate run: tracing slows the host)."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    import torch
    p = torch.cuda.get_device_properties(0)
    try:
        import subprocess
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True).stdout.strip().splitlines()[0]
    except Exception:
        pl = "unknown"
    return p.name, pl


def _branin(x):
    x1, x2 = x[..., 0], x[..., 1]
    return (x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x1) + 10


def _case(name):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    from robo_b200.priors import DefaultPrior
    rng = np.random.RandomState(0)
    if name == "mtbo":
        from robo_b200.models.mtbo_gp import MTBOGP
        from robo_b200.priors import MTBOPrior
        k = 3.0
        for d in range(2):
            k *= K.Matern52Kernel(np.ones([1]) * 0.1, ndim=3, axes=d)
        task = K.TaskKernel(3, 2, 2)
        k = k * task
        X = np.hstack([rng.rand(61, 2), rng.randint(0, 2, (61, 1))])
        y = np.sin(5 * X[:, 0]) + X[:, 1] + 0.5 * X[:, 2]

        def make(opt):
            return MTBOGP(deepcopy_k(k), prior=MTBOPrior(len(k) + 1, 2, len(task), rng=np.random.RandomState(1)),
                          lower=np.zeros(2), upper=np.ones(2), rng=np.random.RandomState(2), hyper_optimizer=opt)
        return make, X[:60], y[:60], X, y
    D, N = {"fmin": (2, 30), "n200_d8": (8, 200), "n232_d16": (16, 232)}[name]
    lo, up = (np.array([-5.0, 0.0]), np.array([10.0, 15.0])) if D == 2 else (np.zeros(D), np.ones(D))
    X = lo + (up - lo) * rng.rand(N + 1, D)
    y = _branin(X) if D == 2 else np.sin(3 * X).sum(axis=1) + 0.1 * rng.randn(N + 1)

    # the facade's cov_amp = 2 at D = 2; at larger D the amplitude is raised to 4 D, so that the lognormal prior on the
    # log amplitude (george divides the constant by ndim) is finite at the start
    amp = 2.0 if D == 2 else 4.0 * D

    def make(opt):
        k = amp * K.Matern52Kernel(np.ones(D), ndim=D)
        return GaussianProcess(k, prior=DefaultPrior(len(k) + 1, rng=np.random.RandomState(1)), normalize_input=True,
                               lower=lo, upper=up, rng=np.random.RandomState(2), hyper_optimizer=opt)
    return make, X[:N], y[:N], X, y


def deepcopy_k(k):
    from copy import deepcopy
    return deepcopy(k)


def _timed(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def _stats(v):
    v = np.array(v)
    return dict(median=float(np.median(v)), min=float(v.min()), max=float(v.max()))


def bench_row(name, reps, card):
    make, X1, y1, X2, y2 = _case(name)
    res = {}
    times = {(a, s): [] for a in ("host", "device") for s in ("first", "later")}
    for rep in range(reps + 1):                              # rep 0 is the warm-up
        for arm in ("host", "device"):
            m = make(arm)
            t1 = _timed(lambda: m.train(X1, y1))
            r1 = dict(m.hyper_result or {})
            t2 = _timed(lambda: m.train(X2, y2))
            r2 = dict(m.hyper_result or {})
            if rep:
                times[(arm, "first")].append(t1)
                times[(arm, "later")].append(t2)
            for stage, r in (("first", r1), ("later", r2)):
                res[(arm, stage)] = dict(nit=r.get("nit"), nfev=r.get("nfev"), rounds=r.get("rounds"),
                                         noop_rounds=r.get("noop_rounds"),
                                         nll=float(m.nll(m.hypers)) if stage == "later" else None)
    for stage in ("first", "later"):
        row = dict(row=name, stage=stage, card=card[0], power_limit=card[1])
        for arm in ("host", "device"):
            row[arm] = dict(time_s=_stats(times[(arm, stage)]), **res[(arm, stage)])
        print(json.dumps(row), flush=True)


def bench_bo(card, iters=30):
    from robo_b200.fmin import bayesian_optimization
    lo, up = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
    out = dict(row="bayesian_optimization_gp_30", card=card[0], power_limit=card[1])
    for arm in ("host", "device"):
        t = _timed(lambda: out.__setitem__(arm, bayesian_optimization(
            lambda x: float(_branin(np.asarray(x))), lo, up, num_iterations=iters, model_type="gp",
            rng=np.random.RandomState(0), hyper_optimizer=arm)))
        r = out[arm]
        tt = np.array(r["time_train"], dtype=float)
        out[arm] = dict(total_s=t, train_per_iter_s=_stats(tt[tt > 0]) if np.any(tt > 0) else None,
                        f_opt=float(r["f_opt"]))
    print(json.dumps(out), flush=True)


def profile(card):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    rows = []
    for name in ("fmin", "n200_d8", "n232_d16"):
        make, X1, y1, _, _ = _case(name)
        m = make("device")
        m.train(X1, y1)
        with tprof(activities=[ProfilerActivity.CUDA]) as p:
            m = make("device")
            m.train(X1, y1)
            torch.cuda.synchronize()
        ev = [e for e in p.key_averages() if "gpk_ho_round_kernel" in e.key]
        if ev:
            e = ev[0]
            rows.append(dict(row=name, kernel="gpk_ho_round_kernel", calls=e.count,
                             us_per_round=e.device_time_total / max(e.count, 1), rounds=m.hyper_result["rounds"],
                             card=card[0], power_limit=card[1]))
    for r in rows:
        print(json.dumps(r), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rows", default="fmin,n200_d8,n232_d16,mtbo")
    ap.add_argument("--bo", action="store_true", help="also time one bayesian_optimization run per arm")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("hyperopt_bench needs a CUDA device")
    card = _card()
    if a.profile:
        profile(card)
        return
    for name in a.rows.split(","):
        bench_row(name, a.reps, card)
    if a.bo:
        bench_bo(card)


if __name__ == "__main__":
    main()
