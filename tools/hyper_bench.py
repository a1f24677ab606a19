"""One GaussianProcessMCMC.train() with the hyper-parameters sampled on the host (EnsembleSampler over the likelihood
pool) against the device (gpk_sample_hypers), at three shapes:

  (a) the bayesian_optimization default: Branin, N = 30, 10 walkers; the first train (100 burn-in + 200 chain steps)
      and a later train (200 steps, N = 31)
  (b) N = 200, 6 input columns (theta of dimension 8), 18 walkers, 100 + 200 steps
  (c) the Fabolas-shaped FabolasGPMCMC: N = 120, 12 walkers, EnvPrior, 100 + 200 steps

Each timed train ends in a device synchronise.  One untimed warm-up round, then alternating host / device rounds;
median, min and max per shape.  The final walkers of both samplers are scored by gpk_hyper_lnpost: their mean
log-posterior (over the finite ones) and finite fraction.  Prints one JSON line with the card and its power limit.

    python tools/hyper_bench.py [--rounds 3] [--out hyper_bench.json]
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
from robo_b200 import kernels as K  # noqa: E402
from robo_b200.device_gp import TINY  # noqa: E402
from robo_b200.models import GaussianProcessMCMC  # noqa: E402
from robo_b200.models.fabolas_gp import FabolasGPMCMC  # noqa: E402
from robo_b200.models.gaussian_process_mcmc import _hyper_prior  # noqa: E402
from robo_b200.priors import DefaultPrior, EnvPrior  # noqa: E402

LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])


def branin(x):
    x1, x2 = x[..., 0], x[..., 1]
    return (x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x1) + 10


def shape_a(sampler):
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    m = GaussianProcessMCMC(kernel, prior=DefaultPrior(4, rng=np.random.RandomState(1)), n_hypers=10, chain_length=200,
                            burnin_steps=100, normalize_input=True, lower=LO, upper=UP, rng=np.random.RandomState(2),
                            hyper_sampler=sampler)
    rng = np.random.RandomState(0)
    X = LO + (UP - LO) * rng.rand(31, 2)
    return m, [(X[:30], branin(X[:30])), (X, branin(X))]


def shape_b(sampler):
    kernel = 2 * K.Matern52Kernel(np.ones(6), ndim=6)
    m = GaussianProcessMCMC(kernel, prior=DefaultPrior(8, rng=np.random.RandomState(3)), n_hypers=18, chain_length=200,
                            burnin_steps=100, normalize_input=True, lower=np.zeros(6), upper=np.ones(6),
                            rng=np.random.RandomState(4), hyper_sampler=sampler)
    rng = np.random.RandomState(8)
    X = rng.rand(200, 6)
    return m, [(X, np.sin(5 * X).sum(axis=1) + 0.05 * rng.randn(200))]


def shape_c(sampler):
    kernel = K.Product(K.ConstantKernel(0.0, ndim=3), K.Product(K.Matern52Kernel(np.ones(2), ndim=3, axes=[0, 1]),
                                                                K.Matern52Kernel(np.ones(1), ndim=3, axes=[2])))
    m = FabolasGPMCMC(kernel, basis_func=lambda s: (1 - s) ** 2,
                      prior=EnvPrior(len(kernel) + 1, 2, 1, rng=np.random.RandomState(6)), n_hypers=12,
                      chain_length=200, burnin_steps=100, lower=LO, upper=UP, rng=np.random.RandomState(5),
                      hyper_sampler=sampler)
    rng = np.random.RandomState(0)
    X = np.c_[LO + (UP - LO) * rng.rand(120, 2), rng.uniform(0.05, 1, 120)]
    return m, [(X, np.log(branin(X) + 1) * (1 + 0.2 * X[:, 2]))]


def final_lnpost(m):
    """gpk_hyper_lnpost of the model's final walkers on its own likelihood inputs."""
    f = m.kernel.flatten()
    h = _lib.Handle(m.device)
    h.set_data(m.X, m.y)
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    kind, par, n_ls, n_lr = _hyper_prior(m.prior)
    _lib.set_hyper_model(h, f["slots"], len(f["axis"]), float(m.mean), TINY, kind, par, n_ls, n_lr)
    ll, lp = _lib.hyper_lnpost(h, m.hypers)
    h.close()
    v = np.where(np.isfinite(ll), ll if kind == _lib.PRIOR_NONE else lp + ll, -np.inf)
    return v


def timed_trains(make, sampler, sync):
    m, data = make(sampler)
    out = []
    for X, y in data:
        t0 = time.perf_counter()
        m.train(X, y)
        sync()
        out.append(time.perf_counter() - t0)
    return out, final_lnpost(m)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, power = [s.strip() for s in q.splitlines()[0].split(",")]
        return name, power
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("hyper_bench.py measures on the GPU; no CUDA device is visible")
    sync = torch.cuda.synchronize
    shapes = {"a_bo_default": (shape_a, ["first_train", "later_train"]), "b_n200_dim8": (shape_b, ["first_train"]),
              "c_fabolas_n120": (shape_c, ["first_train"])}
    res = {}
    for name, (make, labels) in shapes.items():
        for sampler in ("host", "device"):                    # warm-up: modules, handles, buffers of every shape
            timed_trains(make, sampler, sync)
        t = {s: [] for s in ("host", "device")}
        lnp = {}
        for _ in range(a.rounds):
            for sampler in ("host", "device"):
                tt, lnp[sampler] = timed_trains(make, sampler, sync)
                t[sampler].append(tt)
        r = {}
        for sampler in ("host", "device"):
            arr = np.array(t[sampler])
            for j, lab in enumerate(labels):
                r["%s_%s_s" % (sampler, lab)] = dict(median=float(np.median(arr[:, j])), min=float(arr[:, j].min()),
                                                     max=float(arr[:, j].max()))
            v = lnp[sampler]
            fin = np.isfinite(v)
            r["%s_final_lnpost_mean" % sampler] = float(v[fin].mean()) if fin.any() else None
            r["%s_final_lnpost_finite" % sampler] = float(fin.mean())
        for lab in labels:
            r["speedup_" + lab] = r["host_%s_s" % lab]["median"] / r["device_%s_s" % lab]["median"]
        res[name] = r
        print(name, json.dumps(r), file=sys.stderr)
    gpu, power = card()
    line = json.dumps(dict(tool="hyper_bench", gpu=gpu, power_limit=power, rounds=a.rounds, shapes=res))
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
