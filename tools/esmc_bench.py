#!/usr/bin/env python
"""Benchmark of the sampling-based entropy search (InformationGainMC) on the device against a host restatement.

Shape: the entropy_search default on Branin: a GP-MCMC ensemble of 10 sub-models, Nb = 50, Np = 50, Nf = 500,
marginalised by MarginalizationGPMCMC.  Arms, run in alternating rounds after a warm-up, each timing ending in a device
synchronise; the JSON line reports the median and the spread (min, max) of every arm:
    update        MarginalizationGPMCMC.update (representer points by the device sampler, then gpk_esmc_update x 10)
    compute_500   compute() of 500 candidates on the device (gpk_esmc_multi)
    compute_65536 compute() of 65,536 candidates on the device
    host_500      the reference's joint_pmin per candidate in numpy (Cholesky with the jitter ladder, Nf draws, the
                  arg-min over Nf Np columns) on ONE sub-model, fed the device's v and sigma; x 10 for the ensemble is
                  reported as host_500_ensemble_estimate, which is an extrapolation, not a measurement
    de_device     DifferentialEvolution (maxiter 20, popsize 15, no polish) on the device
    de_scipy      scipy.optimize.differential_evolution(maxiter=20, polish=False) on the one-point objective, every
                  row one compute() call on the device
With --profile the run instead takes torch.profiler's CUDA time of gpk_mc_pmin_kernel over compute_65536 and sets it
against the fp64-pipe bound of the operation counts (every product and sum of the kernel is one fp64 instruction):
    per candidate: Nb (Nb + 1) / 2 Nf (multiply, add) for the draws + Nb Nf Np (add, compare) for the arg-min.
Usage: python tools/esmc_bench.py [--rounds 5] [--profile] [--out results/esmc_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

LO, UP = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
NB, NP, NF = 50, 50, 500
FP64_INSTR_PER_S = 132 * 64 * 1.98e9        # H100 SXM data sheet: 34 TFLOPS fp64 = 132 SMs x 64 fp64 lanes x 1.98 GHz x 2


def _branin(x):
    return (x[1] - 5.1 / (4 * np.pi ** 2) * x[0] ** 2 + 5 / np.pi * x[0] - 6) ** 2 \
        + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x[0]) + 10


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:                                    # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def _sync():
    import torch
    torch.cuda.synchronize()


def _setup():
    from robo_b200 import kernels as K
    from robo_b200.acquisition_functions import EI, InformationGainMC, MarginalizationGPMCMC
    from robo_b200.models import GaussianProcessMCMC
    from robo_b200.priors import DefaultPrior
    rng = np.random.RandomState(4)
    X = LO + (UP - LO) * rng.rand(20, 2)
    y = np.array([_branin(x) for x in X])
    kernel = 2 * K.Matern52Kernel(np.ones(2), ndim=2)
    model = GaussianProcessMCMC(kernel, prior=DefaultPrior(len(kernel) + 1, rng=np.random.RandomState(1)),
                                n_hypers=10, chain_length=200, burnin_steps=100, normalize_input=True,
                                normalize_output=False, lower=LO, upper=UP, rng=np.random.RandomState(2))
    model.train(X, y, do_optimize=True)
    acq = MarginalizationGPMCMC(InformationGainMC(model, LO, UP, Nb=NB, Np=NP, Nf=NF, sampling_acquisition=EI,
                                                  rng=np.random.RandomState(0), representer_sampler="device"))
    acq.update(model)
    return model, acq


def _host_values(est, C):
    """The reference's compute per candidate in numpy (information_gain_mc.py:67-156 with mc_part.joint_pmin), on the
    estimator's Mb, Vb and the device's v and sigma; fresh numpy draws per candidate, as the reference takes them."""
    h = est._ready_handle()
    var, sig = h.es_moments(C)
    Mb, Vb = h.esmc_get_state()
    W = est.W.ravel()
    lmb = est.lmb.ravel()
    H = -np.sum(np.exp(est.logP.ravel()) * (est.logP.ravel() + lmb))
    out = np.empty(C.shape[0])
    rng = np.random.RandomState(0)
    for i in range(C.shape[0]):
        nc = sig[i] / (var[i] - est.sn2)
        M = Mb[:, None] + (nc * np.sqrt(var[i] + 1e-10))[:, None] * W[None, :]
        V = Vb - np.outer(nc, sig[i])
        noise = 0
        while True:
            try:
                cV = np.linalg.cholesky(V + noise * np.eye(NB))
                break
            except np.linalg.LinAlgError:
                if noise == 0:
                    noise = 1e-10
                if noise == 10000:
                    raise
                noise *= 10
        funcs = cV @ rng.randn(NF, NB).T
        mins = np.argmin((M[:, None, :] + funcs[:, :, None]).reshape(NB, -1), axis=0)
        p = np.bincount(mins, minlength=NB) / float(NF * NP)
        p[p < 1e-70] = 1e-70
        out[i] = np.sum(p * (np.log(p) + lmb)) + H
    return out


def _timed(fn):
    _sync()
    t = time.perf_counter()
    fn()
    _sync()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import scipy.optimize
    import torch
    from robo_b200.maximizers import DifferentialEvolution
    name, power = _card()
    model, acq = _setup()
    rng = np.random.RandomState(7)
    C500 = LO + (UP - LO) * rng.rand(500, 2)
    C64k = LO + (UP - LO) * rng.rand(65536, 2)
    n_models = len(acq.estimators)
    ops = (NB * (NB + 1) // 2 * NF * 2 + NB * NF * NP * 2) * 65536 * n_models
    if a.profile:
        acq.compute(C64k)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            acq.compute(C64k)
            _sync()
        kern = sum(e.device_time_total for e in prof.key_averages() if "gpk_mc_pmin_kernel" in e.key) * 1e-6
        other = sum(e.device_time_total for e in prof.key_averages() if "gpk_mc_pmin_kernel" not in e.key) * 1e-6
        res = dict(bench="esmc_profile", card=name, power_limit=power, candidates=65536, models=n_models,
                   pmin_kernel_s=kern, other_kernels_s=other, fp64_instructions=ops,
                   fp64_bound_s=ops / FP64_INSTR_PER_S, share_of_fp64_bound=(ops / FP64_INSTR_PER_S) / kern)
    else:
        arms = {
            "update": lambda: acq.update(model),
            "compute_500": lambda: acq.compute(C500),
            "compute_65536": lambda: acq.compute(C64k),
            "host_500": lambda: _host_values(acq.estimators[0], C500),
            "de_device": lambda: DifferentialEvolution(acq, LO, UP, n_iters=20, rng=np.random.RandomState(1),
                                                       polish=False).maximize(),
            "de_scipy": lambda: scipy.optimize.differential_evolution(
                lambda x: -float(acq.compute(np.clip(x, LO, UP)[None, :])[0]), list(zip(LO, UP)), maxiter=20,
                polish=False, seed=1),
        }
        for fn in arms.values():                                    # warm-up of every shape
            fn()
        times = {k: [] for k in arms}
        for r in range(a.rounds):
            for k in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                if k == "host_500" and len(times[k]) >= 2:
                    continue                                        # seconds per round: two rounds suffice
                times[k].append(_timed(arms[k]))
        res = dict(bench="esmc", card=name, power_limit=power, shape=dict(models=n_models, Nb=NB, Np=NP, Nf=NF),
                   rounds=a.rounds)
        for k, v in times.items():
            res[k] = dict(median_s=float(np.median(v)), min_s=float(np.min(v)), max_s=float(np.max(v)), n=len(v))
        res["host_500_ensemble_estimate_s"] = res["host_500"]["median_s"] * n_models
        res["compute_65536_per_candidate_model_us"] = res["compute_65536"]["median_s"] / (65536 * n_models) * 1e6
        res["fp64_bound_65536_s"] = ops / FP64_INSTR_PER_S
        torch.cuda.synchronize()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
