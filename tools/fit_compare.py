#!/usr/bin/env python
"""Fit time of the look-ahead Cholesky schedule (automatic depth-2 trailing updates, and depth2 = 0) at the BASELINE
sizes, next to cuSOLVER's dense potrf on the same GPU (torch.linalg.cholesky -> cusolverDnDpotrf / cusolverDnXpotrf;
SURVEY.md section 7 step 4 asked for that baseline).  Prints one JSON line per size.  python tools/fit_compare.py"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from robo_b200 import _lib                                   # noqa: E402
from robo_b200 import kernels as K                           # noqa: E402


def ours(N, D, reps=6, depth2=2):
    rng = np.random.RandomState(1234)
    X = rng.rand(N, D)
    y = np.sinc(X * 10 - 5).sum(axis=1) + 0.01 * rng.randn(N)
    theta = np.concatenate(([0.0], np.full(D, np.log(D / 4.0))))
    h = _lib.Handle(0)
    h.set_option("depth2", depth2)
    h.set_data(X, y)
    f = K.Product(K.ConstantKernel(theta[0], ndim=D), K.Matern52Kernel(np.exp(theta[1:]), ndim=D)).flatten()
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    dadd = float(np.sqrt(np.float64(np.sqrt(1e-3)) ** 2 + 1.25e-12) ** 2)
    ts, ks, ps = [], [], []
    for _ in range(reps):
        h.fit(dadd, float(np.mean(y)))
        t = h.timings()
        ts.append(t["fit_ms"]); ks.append(t["kbuild_ms"]); ps.append(t["potrf_ms"])
    h.predict(X[:128])
    linv = h.timings()["linv_ms"]
    h.close()
    return float(np.median(ts[1:])), float(np.median(ks[1:])), float(np.median(ps[1:])), linv


def cusolver(N, reps=6):
    g = torch.Generator(device="cuda").manual_seed(0)
    A = torch.randn(N, N, dtype=torch.float64, device="cuda", generator=g)
    A = A @ A.T + N * torch.eye(N, dtype=torch.float64, device="cuda")
    b = torch.randn(N, 1, dtype=torch.float64, device="cuda", generator=g)
    ts, ss = [], []
    for _ in range(reps):
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        L = torch.linalg.cholesky(A)
        e1.record()
        torch.linalg.solve_triangular(L, b, upper=False)
        e2.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1)); ss.append(e1.elapsed_time(e2))
    return float(np.median(ts[1:])), float(np.median(ss[1:]))


for N, D in ((1024, 8), (2048, 3), (4096, 16), (8192, 32)):
    b = ours(N, D)
    b0 = ours(N, D, depth2=0)
    c = cusolver(N)
    flop = N ** 3 / 3.0
    print(json.dumps({"N": N, "D": D,
                      "plain_lookahead": {"fit_ms": b[0], "kbuild_ms": b[1], "potrf_incl_forward_solve_logdet_ms": b[2],
                                          "linv_ms": b[3], "potrf_tflops": flop / (b[2] * 1e-3) / 1e12},
                      "plain_lookahead_depth1": {"fit_ms": b0[0], "potrf_incl_forward_solve_logdet_ms": b0[2]},
                      "cusolver_torch_linalg_cholesky": {"potrf_ms": c[0], "forward_solve_ms": c[1],
                                                         "potrf_tflops": flop / (c[0] * 1e-3) / 1e12}}))
