#!/usr/bin/env python
"""Scoring time per pass with and without the persistent tile walk, per training-set size: options "ozpersist" and
"ozcluster" of the int8 contraction (which N should the automatic mode switch at, for which cluster size?), next to
the fp64 contraction ("ozaki" = 0, one CTA per tile).    python tools/persist_threshold.py"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from robo_b200 import _lib                                   # noqa: E402
from robo_b200 import kernels as K                           # noqa: E402

D = 8
out = {}
for N, M in ((512, 524288), (1024, 524288), (1536, 262144), (2048, 262144), (3072, 131072), (4096, 131072), (6144, 65536)):
    rng = np.random.RandomState(N)
    X = rng.rand(N, D)
    y = np.sinc(X * 10 - 5).sum(axis=1) + 0.01 * rng.randn(N)
    theta = np.concatenate(([0.0], np.full(D, np.log(D / 4.0))))
    dX = torch.rand(M, D, dtype=torch.float64, device="cuda")
    row = {}
    configs = [("int8_cluster%d_%s" % (cs, "persistent" if p else "one_tile_per_cta"), {"ozcluster": cs, "ozpersist": p})
               for cs in (1, 2, 4) for p in (0, 1)]
    configs += [("fp64_one_tile_per_cta", {"ozaki": 0})]
    for name, opts in configs:
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
        t = []
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            h.acq_dev(dX.data_ptr(), M, _lib.ACQ_EI, float(np.min(y)), 0.0, 0, 0, 0, best.data_ptr())
            torch.cuda.synchronize()
            t.append((time.perf_counter() - t0) * 1e3)
        tim = h.timings()
        row[name] = {"pass_ms_min": min(t), "pass_ms_median": float(np.median(t)),
                     "contraction_ms_per_chunk": tim["vargemm_ms"], "int8_launches": tim["launches_ozaki"]}
        h.close()
    out["N=%d M=%d" % (N, M)] = row
print(json.dumps(out, indent=1))
