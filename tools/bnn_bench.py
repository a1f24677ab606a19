"""WrapperBohamiann on the device against the reference's cost structure restated on the host, at three shapes:

  ref       D = 2, N = 10    (the reference test, test_wrapper_bohamiann.py)
  branin    D = 2, N = 30
  d8        D = 8, N = 200

pybnn is not available, so the host arm is tests/bnn_model.torch_train: pybnn's training loop restated in torch on the
CPU (float64, a shuffled batch loader, the loss and adaptive SGHMC per parameter tensor, one round of small torch ops
per step), at the wrapper's settings (100 N burn-in steps, 100 N + 10,000 steps, 99 networks kept).

Arms, each timing ending in a device synchronise:
  train1 / train2   the first train() on a fresh model and a later one on the same model (host: one torch_train)
  ei65k / ei1m      predict + EI + arg-max over 65,536 and 2^20 candidates (device: gpk_acq; host at 65,536 only: the
                    99 networks' forward passes batched in torch, the moments, EI, argmax)
  de                DifferentialEvolution.maximize at 20 generations (device only)
One untimed device warm-up per shape, then alternating host / device rounds; median, [min, max].  Prints one JSON line
per round and a summary line, each with the card's name and power limit read in the same call.

--profile runs a separate pass under torch.profiler and derives the scoring kernel's FMA rate: 99 networks x
(50 D + 2,550) FMAs per candidate over the kernel time of gpk_bnn_score_kernel, against the fp64 vector-pipe rate the
library measures on the same card (gpk_measure_fp64_peaks) and labelled as such.  The 100 tanh per network are not
counted in that rate.

    python tools/bnn_bench.py [--rounds 3] [--shapes ref,branin,d8] [--no-host] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
from scipy.stats import norm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from robo_b200 import _lib  # noqa: E402
from robo_b200.acquisition_functions import EI  # noqa: E402
from robo_b200.maximizers import DifferentialEvolution  # noqa: E402
from robo_b200.models import WrapperBohamiann  # noqa: E402
from tests import bnn_model as BM  # noqa: E402

SHAPES = {"ref": (2, 10), "branin": (2, 30), "d8": (8, 200)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:
        return "unknown (%s)" % e, "unknown"


def problem(D, N, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    return X, np.sinc(X * 10 - 5).sum(axis=1)


def timed(fn, handle=None):
    t = time.perf_counter()
    out = fn()
    if handle is not None:
        handle.synchronize()
    return time.perf_counter() - t, out


def host_ei(samples, stats, X, eta):
    """Host predict + EI + argmax: the networks' forward passes batched in torch (float64)."""
    import torch
    xm, xs, ym, ysd = stats
    D = X.shape[1]
    L = BM.layout(D)
    x = torch.as_tensor((X - xm) / xs)
    F = []
    for th in torch.as_tensor(samples):
        h1 = torch.tanh(x @ th[L["W1"]].reshape(50, D).T + th[L["b1"]])
        h2 = torch.tanh(h1 @ th[L["W2"]].reshape(50, 50).T + th[L["b2"]])
        F.append(h2 @ th[L["W3"]] + th[L["b3"]])
    F = torch.stack(F).numpy()
    m = F.mean(axis=0)
    v = ((F - m) ** 2).mean(axis=0) + np.exp(samples[:, L["lv"]]).mean()
    m, v = m * ysd + ym, v * ysd * ysd
    s = np.sqrt(v)
    z = (eta - m) / s
    ei = s * (z * norm.cdf(z) + norm.pdf(z))
    return int(np.argmax(ei))


def profile_rate(name, power, D=2, N=30, M=1 << 20):
    import torch
    from torch.profiler import ProfilerActivity, profile
    X, y = problem(D, N)
    m = WrapperBohamiann(rng=np.random.RandomState(0))
    m.train(X, y)
    h = m._ready_handle()
    Xc = np.random.RandomState(1).rand(M, D)
    h.acq(Xc, _lib.ACQ_EI, float(y.min()))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            h.acq(Xc, _lib.ACQ_EI, float(y.min()))
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "gpk_bnn_score_kernel" in e.key]
    total_us = sum(e.device_time_total for e in ev)
    launches = sum(e.count for e in ev)
    kernel_s = total_us / 1e6 / 3                           # three passes of 2^20 candidates
    S = m.samples.shape[0]
    fma = float(M) * S * (50 * D + 2550)
    _, dfma_tflops = h.measure_fp64_peaks()
    rate = fma / kernel_s
    print(json.dumps(dict(arm="score_rate", card=name, power_limit=power, D=D, S=S, candidates=M,
                          kernel_ms_per_pass=kernel_s * 1e3, launches=launches, fma_per_s=rate,
                          fp64_vector_peak_measured_tflops=dfma_tflops,
                          share_of_measured_fp64_vector_rate=2 * rate / (dfma_tflops * 1e12))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="ref,branin,d8")
    ap.add_argument("--no-host", action="store_true")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    name, power = card()
    if a.profile:
        profile_rate(name, power)
        return
    summary = {}
    for shape in a.shapes.split(","):
        D, N = SHAPES[shape]
        X, y = problem(D, N)
        eta = float(y.min())
        rng = np.random.RandomState(2)
        C65, C1m = rng.rand(65536, D), rng.rand(1 << 20, D)
        warm = WrapperBohamiann(rng=np.random.RandomState(9))
        warm.train(X, y)
        warm._ready_handle().acq(C1m, _lib.ACQ_EI, eta)
        for r in range(a.rounds):
            rec = dict(shape=shape, D=D, N=N, round=r, card=name, power_limit=power)
            if not a.no_host:
                t, (S, stats) = timed(lambda: BM.torch_train(X, y, r))
                rec["host_train_s"] = t
                rec["host_ei65k_s"] = timed(lambda: host_ei(S, stats, C65, eta))[0]
            m = WrapperBohamiann(rng=np.random.RandomState(r))
            rec["dev_train1_s"] = timed(lambda: m.train(X, y))[0]
            rec["dev_train2_s"] = timed(lambda: m.train(X, y))[0]
            h = m._ready_handle()
            rec["dev_ei65k_s"] = timed(lambda: h.acq(C65, _lib.ACQ_EI, eta), h)[0]
            rec["dev_ei1m_s"] = timed(lambda: h.acq(C1m, _lib.ACQ_EI, eta), h)[0]
            acq = EI(m)
            de = DifferentialEvolution(acq, np.zeros(D), np.ones(D), n_iters=20, rng=np.random.RandomState(r))
            rec["dev_de20_s"] = timed(lambda: de.maximize(), h)[0]
            print(json.dumps(rec), flush=True)
            for k, v in rec.items():
                if k.endswith("_s"):
                    summary.setdefault((shape, k), []).append(v)
    out = {"%s:%s" % k: dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v)))
           for k, v in summary.items()}
    print(json.dumps(dict(summary=out, card=name, power_limit=power)), flush=True)


if __name__ == "__main__":
    main()
