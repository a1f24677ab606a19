"""Hyper-parameter inference at large N: "host" against "device_blocked" (gpk_sample_hypers_blocked /
gpk_optimize_hypers_blocked), and "device" against "device_blocked" at N = 232, one JSON line per row on stdout.

Rows (--rows picks a subset):
  fabolas2048  one FabolasGPMCMC.train (N = 2048, 20 walkers, EnvPrior, 100 burn-in + 200 chain steps)
  mcmc1000     one GaussianProcessMCMC.train (N = 1000, D = 8, DefaultPrior, 20 walkers, 100 + 200 steps)
  gp2048       one GaussianProcess.train (N = 2048, D = 16, no prior, L-BFGS-B from the kernel's start)
  gp8192       one GaussianProcess.train (N = 8192, D = 32, no prior: the marginal-likelihood shape of BASELINE config 5)
  crossover232 GaussianProcessMCMC (N = 232, D = 16, 36 walkers, 100 + 200 steps): "device" against "device_blocked"
Each row runs its two arms in alternating rounds (--rounds, default 3) after one warm-up train per arm on the first
300 points, every timing
ending in a device synchronise, and reports the median and the spread (min, max) of the seconds per train, with the
mean, median and range of the final walkers' log-posteriors (MCMC rows) or the final nll (GP rows) of each arm's last round.  The card's
name and power limit are read in the same run."""
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


def _sync():
    import torch
    torch.cuda.synchronize()


def _mcmc_lnpost(m):
    """The final walkers' log-posteriors (the prior plus the likelihood, as the host sampler sees it): mean, median,
    min and max."""
    v = np.array([m.loglikelihood(t) for t in m.hypers])
    return dict(mean=float(np.mean(v)), median=float(np.median(v)), min=float(v.min()), max=float(v.max()))


def _row_mcmc(name, arms, N, D, n_hypers, burnin, chain, fabolas):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    from robo_b200.fmin.fabolas import _model, quadratic_bf
    rng = np.random.RandomState(N)
    if fabolas:
        X = np.c_[rng.rand(N, D), rng.uniform(0.05, 1, N)]
        y = np.sin(5 * X[:, :D]).sum(axis=1) * (1 + 0.2 * X[:, D]) + 0.05 * rng.randn(N)
    else:
        X = rng.rand(N, D)
        y = np.sin(5 * X).sum(axis=1) + 0.05 * rng.randn(N)

    def make(arm):
        if fabolas:
            return _model(D, quadratic_bf, n_hypers, burnin, chain, np.zeros(D), np.ones(D), np.random.RandomState(1),
                          arm)
        k = 2.0 * K.Matern52Kernel(np.ones(D), ndim=D)
        return GaussianProcessMCMC(k, prior=DefaultPrior(len(k) + 1, rng=np.random.RandomState(1)), n_hypers=n_hypers,
                                   chain_length=chain, burnin_steps=burnin, lower=np.zeros(D), upper=np.ones(D),
                                   rng=np.random.RandomState(2), hyper_sampler=arm)
    return _alternate(name, arms, make, X, y, _mcmc_lnpost, dict(N=N, D=D, n_hypers=n_hypers, burnin=burnin,
                                                                   chain=chain))


def _row_gp(name, arms, N, D):
    from robo_b200 import kernels as K
    from robo_b200.models import GaussianProcess
    rng = np.random.RandomState(N)
    X = rng.rand(N, D)
    y = np.sin(5 * X[:, :4]).sum(axis=1) + 0.05 * rng.randn(N)

    def make(arm):
        k = 2.0 * K.Matern52Kernel(np.ones(D), ndim=D)
        return GaussianProcess(k, prior=None, lower=np.zeros(D), upper=np.ones(D), rng=np.random.RandomState(0),
                               hyper_optimizer=arm)
    return _alternate(name, arms, make, X, y, lambda m: float(m.nll(m.hypers)), dict(N=N, D=D))


def _alternate(name, arms, make, X, y, quality, shape):
    times = {a: [] for a in arms}
    last = {}
    for a in arms:                                           # warm-up: one train per arm on the first 300 points
        make(a).train(X[:300], y[:300])
    for r in range(ROUNDS):
        for a in (arms if r % 2 == 0 else arms[::-1]):
            m = make(a)
            _sync()
            t0 = time.perf_counter()
            m.train(X, y)
            _sync()
            times[a].append(time.perf_counter() - t0)
            last[a] = m
    out = dict(row=name, shape=shape, rounds=ROUNDS)
    for a in arms:
        t = np.array(times[a])
        out[a] = dict(median_s=float(np.median(t)), min_s=float(t.min()), max_s=float(t.max()),
                      quality=quality(last[a]))
    out["speedup_median"] = out[arms[0]]["median_s"] / out[arms[1]]["median_s"]
    return out


ROUNDS = 3


def main():
    global ROUNDS
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="fabolas2048,mcmc1000,gp2048,gp8192,crossover232")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    ROUNDS = a.rounds
    name, pl = _card()
    rows = {
        "fabolas2048": lambda: _row_mcmc("fabolas2048", ["host", "device_blocked"], 2048, 2, 20, 100, 200, True),
        "mcmc1000": lambda: _row_mcmc("mcmc1000", ["host", "device_blocked"], 1000, 8, 20, 100, 200, False),
        "gp2048": lambda: _row_gp("gp2048", ["host", "device_blocked"], 2048, 16),
        "gp8192": lambda: _row_gp("gp8192", ["host", "device_blocked"], 8192, 32),
        "crossover232": lambda: _row_mcmc("crossover232", ["device", "device_blocked"], 232, 16, 36, 100, 200, False),
    }
    for r in a.rows.split(","):
        res = rows[r]()
        res.update(card=name, power_limit=pl)
        line = json.dumps(res)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
