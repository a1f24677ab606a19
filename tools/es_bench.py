#!/usr/bin/env python
"""Times EPMGP p_min on the device (gpk_ep_joint_min) against the numpy restatement in the reference's loop order
(tests/es_model.py, the host path), at the entropy-search default Nb = 50 on a GP posterior.  Prints one JSON line
with the card and its power limit, read in the same call.

    python tools/es_bench.py [--nb 50] [--reps 20] [--host-reps 3]

The device figure is the wall time of the blocking call (operands in, EP, renormalisation, results out), median over
--reps calls after two warm-up calls.  The host figure is the median over --host-reps runs of the restatement.
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


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, limit = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, limit
    except Exception:
        return "unknown", "unknown"


def _posterior(nb, seed=0):
    rng = np.random.RandomState(seed)
    X, Z = rng.rand(30, 2), rng.rand(nb, 2)

    def k(A, B):
        r2 = (((A[:, None, :] - B[None, :, :]) / 0.3) ** 2).sum(-1)
        r = np.sqrt(5.0 * r2)
        return 2.0 * (1.0 + r + 5.0 * r2 / 3.0) * np.exp(-r)

    K = k(X, X) + 1e-3 * np.eye(30)
    Ks = k(Z, X)
    mu = Ks @ np.linalg.solve(K, np.sin(6 * X[:, 0]) + X[:, 1])
    return mu, np.clip(k(Z, Z) - Ks @ np.linalg.solve(K, Ks.T), np.finfo(float).eps, np.inf)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nb", type=int, default=50)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=3)
    a = ap.parse_args()
    from robo_b200 import _lib
    from tests import es_model

    mu, V = _posterior(a.nb)
    h = _lib.moments_handle()
    for _ in range(2):
        dev = h.ep_joint_min(mu, V)
    t_dev = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        h.ep_joint_min(mu, V)
        t_dev.append(time.perf_counter() - t0)
    t_host = []
    for _ in range(a.host_reps):
        t0 = time.perf_counter()
        ref = es_model.joint_min(mu, V)
        t_host.append(time.perf_counter() - t0)
    name, limit = _card()
    scale = np.max(np.abs(ref["logP"]))
    print(json.dumps(dict(
        card=name, power_limit=limit, nb=a.nb, sweeps_total=int(dev["sweeps"].sum()),
        sweeps_equal=bool(np.array_equal(dev["sweeps"], ref["sweeps"])),
        logP_max_abs_diff_rel=float(np.max(np.abs(dev["logP"] - ref["logP"])) / scale),
        ep_device_ms=1e3 * float(np.median(t_dev)), ep_host_ms=1e3 * float(np.median(t_host)),
        update_ms="not measured", maximize_ms="not measured", candidates_per_s="not measured")))


if __name__ == "__main__":
    main()
