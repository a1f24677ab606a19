#!/usr/bin/env python
"""Diagonal-block kernel (gpk_potrf_diag_dmma_kernel): agreement of the factor, the inverse and the log-likelihood
with scipy at a size the host finishes in a second, the non-PD status, fit-time timing at N = 4096 (and N = 2048 / 8192
with SIZES=...) and the kernel's per-phase clock64() profile ("diagprof").  Prints one line per check; exits non-zero
on a mismatch."""
import os
import sys

import numpy as np
import scipy.linalg as sla

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from robo_b200 import _lib                     # noqa: E402
from robo_b200 import kernels as K             # noqa: E402

SIZES = [int(s) for s in os.environ.get("SIZES", "4096").split(",")]
TINY = 1.25e-12
bad = 0


def problem(n, d, seed=1234):
    rng = np.random.RandomState(seed)
    X = rng.rand(n, d)
    y = np.sinc(X * 10 - 5).sum(axis=1) + 0.01 * rng.randn(n)
    theta = np.concatenate(([0.0], np.full(d, np.log(d / 4.0))))
    f = K.Product(K.ConstantKernel(theta[0], ndim=d), K.Matern52Kernel(np.exp(theta[1:]), ndim=d)).flatten()
    return X, y, f


def handle(X, y, f):
    h = _lib.Handle(0)
    h.set_data(X, y)
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    return h


da = float(np.sqrt(np.float64(np.sqrt(1e-3)) ** 2 + TINY) ** 2)

# ---- 1. agreement with scipy (N = 700: five full blocks + a ragged one)
for n in (100, 700):
    X, y, f = problem(n, 5, seed=11)
    h = handle(X, y, f)
    logdet, ll = h.fit(da, float(np.mean(y)))
    L, Li = h.get_factor(n), h.get_linv(n)
    Kd = h.kernel_matrix(X, X) + da * np.eye(n)
    Lr = sla.cholesky(Kd, lower=True)
    eL = np.abs(L - Lr).max() / np.abs(Lr).max()
    eI = np.abs(Li @ Lr - np.eye(n)).max()
    eU = max(np.abs(np.triu(L, 1)).max(), np.abs(np.triu(Li, 1)).max())
    eld = abs(logdet - 2 * np.log(np.diag(Lr)).sum()) / abs(logdet)
    ok = eL < 1e-12 and eI < 1e-9 and eU == 0.0 and eld < 1e-12
    bad += not ok
    print("agree n=%d  |L-Lref| %.2e  |Linv L - I| %.2e  upper %.1e  logdet rel %.2e  %s"
          % (n, eL, eI, eU, eld, "ok" if ok else "MISMATCH"))
    h.close()

# ---- 2. not positive definite: status = first failing pivot
X = np.zeros((6, 2))
h = handle(X, np.arange(6.0), *problem(6, 2)[2:])
try:
    h.fit(0.0, 0.0)
    print("notpd: no error  MISMATCH")
    bad += 1
except Exception as e:                          # noqa: BLE001
    print("notpd: %s: %s" % (type(e).__name__, e))
h.close()

# ---- 3. timing
for n in SIZES:
    X, y, f = problem(n, 16)
    h = handle(X, y, f)
    ts = []
    for _ in range(8):
        logdet, ll = h.fit(da, float(np.mean(y)))
        ts.append(h.timings()["fit_ms"])
    print("time n=%d  fit_ms median %.3f min %.3f  ll=%.12f" % (n, np.median(ts[2:]), min(ts), ll))
    h.close()
    # cycle stamps of the last diagonal block (clock64, SM clock)
    h = handle(X, y, f)
    h.set_option("diagprof", int(os.environ.get("DIAGPROF", 1)))
    for _ in range(3):
        try:
            h.fit(da, float(np.mean(y)))
        except Exception as e:                  # noqa: BLE001  (DIAGPROF=2 leaves garbage in K)
            print("  (fit under diagprof raised %s)" % type(e).__name__)
    t = h.diag_profile()
    ph = np.array([[t[2 + 2 * p] - t[1 + 2 * p], (t[3 + 2 * p] - t[2 + 2 * p]) if p < 7 else 0]
                   for p in range(8)])
    print("diagprof n=%d total %d cycles (init %d); per panel [factor+solve, update+publish]:"
          % (n, t[33] - t[0], t[1] - t[0]))
    print(ph.T)
    print("sums", ph.sum(axis=0))
    if t[34]:
        print("panel 3 fine stamps: S loads %d, pivots 0-3 %d, 4-7 %d, 8-11 %d, 12-15 %d, smem stores %d, barrier %d; "
              "U global stores %d, update+publish %d, barrier %d"
              % (t[34] - t[7], t[35] - t[34], t[36] - t[35], t[37] - t[36], t[38] - t[37], t[39] - t[38],
                 t[8] - t[39], t[40] - t[8], t[41] - t[40], t[9] - t[41]))
        print("panel 3 factorising warp: pivots 0-3 %d, 4-7 %d, 8-11 %d, 12-14 + rsqrt %d cycles"
              % (t[42] - t[46], t[43] - t[42], t[44] - t[43], t[45] - t[44]))
    h.close()
sys.exit(1 if bad else 0)
