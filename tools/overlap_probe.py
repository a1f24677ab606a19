#!/usr/bin/env python
"""How well does the K* builder of chunk i+1 (low-priority side stream) hide behind the int8 contraction of chunk i?
Scores M = 131072 device-resident candidates at N = 4096, D = 16 with option "overlap" on and off and prints the time
per pass, next to the per-kernel figures of the handle.      python tools/overlap_probe.py"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from robo_b200 import _lib                                   # noqa: E402
from robo_b200 import kernels as K                           # noqa: E402

N, D, M = 4096, 16, 131072
rng = np.random.RandomState(1234)
X = rng.rand(N, D)
y = np.sinc(X * 10 - 5).sum(axis=1) + 0.01 * rng.randn(N)
theta = np.concatenate(([0.0], np.full(D, np.log(D / 4.0))))
dX = torch.rand(M, D, dtype=torch.float64, device="cuda")
out = {}
for label, opts in (("overlap", {}), ("no_overlap", {"overlap": 0}),
                    ("fp64_overlap", {"ozaki": 0}), ("fp64_no_overlap", {"ozaki": 0, "overlap": 0})):
    h = _lib.Handle(0)
    for k, v in opts.items():
        h.set_option(k, v)
    h.set_data(X, y)
    f = K.Product(K.ConstantKernel(theta[0], ndim=D), K.Matern52Kernel(np.exp(theta[1:]), ndim=D)).flatten()
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    h.fit(1e-3 + 1.25e-12, float(np.mean(y)))
    best = torch.zeros(2, dtype=torch.float64, device="cuda")
    for _ in range(3):
        h.acq_dev(dX.data_ptr(), M, _lib.ACQ_EI, float(np.min(y)), 0.0, 0, 0, 0, best.data_ptr())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 5
    st = torch.cuda.ExternalStream(h.stream_ptr()) if hasattr(h, "stream_ptr") else None
    t = []
    for _ in range(reps):
        torch.cuda.synchronize()
        import time
        t0 = time.perf_counter()
        h.acq_dev(dX.data_ptr(), M, _lib.ACQ_EI, float(np.min(y)), 0.0, 0, 0, 0, best.data_ptr())
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    tim = h.timings()
    out[label] = {"pass_ms_wall_min": min(t), "score_ms_events": tim["score_ms"], "kstar_ms_last_chunk": tim["kstar_ms"],
                  "vargemm_ms_avg": tim["vargemm_ms"], "finish_ms": tim["finish_ms"], "launches_ozaki": tim["launches_ozaki"]}
    h.close()
print(json.dumps(out))
