#!/usr/bin/env python
"""Write tests/golden/es_ep.npz by running the reference's own robo/util/epmgp.joint_min(with_derivatives=True).

Run where the reference tree is available (ROBO_REFERENCE, default /root/reference):

    python tools/make_es_golden.py

Only the outputs are kept; no reference code enters the repository.  Two numpy-2 shims: np.Infinity and np.NAN
(removed in numpy 2.0) are aliased to np.inf and np.nan.  lt_factor is wrapped to count the EP steps of every
problem k, which pins the sweep counts of tests/es_model.py.

Cases
  uniform  m = 1, V = I, Nb = 50 (the reference test's known answer: p_min near 1 / Nb)
  dirac    m = 1000 except m[0] = 1, V = I, Nb = 50 (p_min[0] == 1 exactly; every k > 0 leaves EP through z < -6,
           logZ = -inf, replaced by -500)
  mixed    Nb = 6, two far points: their problems take the z < -6 exit while the others converge
  branin   the posterior of a Matern-5/2 GP on 20 Branin evaluations (fixed hyper-parameters) at Nb = 50 points,
           clipped at DBL_EPSILON as GaussianProcess.predict(full_cov=True) returns it
  rand2, rand17  random posteriors

For Nb >= 50 only the derivatives of problems k < 2 are stored (the fixture stays small); logP, the renormalisation
inputs of every k, is stored in full.
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("ROBO_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "es_ep.npz")


def _matern52(A, B, ls, amp):
    r2 = (((A[:, None, :] - B[None, :, :]) / ls) ** 2).sum(-1)
    r = np.sqrt(5.0 * r2)
    return amp * (1.0 + r + 5.0 * r2 / 3.0) * np.exp(-r)


def _posterior(Z, X, y, ls, amp, noise):
    K = _matern52(X, X, ls, amp) + noise * np.eye(len(X))
    Ks = _matern52(Z, X, ls, amp)
    mu = Ks @ np.linalg.solve(K, y)
    V = _matern52(Z, Z, ls, amp) - Ks @ np.linalg.solve(K, Ks.T)
    return mu, np.clip(V, np.finfo(float).eps, np.inf)


def cases():
    rng = np.random.RandomState(20261015)
    out = {}
    out["uniform"] = (np.ones(50), np.eye(50))
    m = np.ones(50) * 1000.0
    m[0] = 1.0
    out["dirac"] = (m, np.eye(50))
    out["mixed"] = (np.array([0.0, 0.3, 40.0, -0.2, 55.0, 0.1]), 0.05 * np.eye(6) + 0.01)

    def branin(x):
        return (x[:, 1] - 5.1 / (4 * np.pi ** 2) * x[:, 0] ** 2 + 5 / np.pi * x[:, 0] - 6) ** 2 \
            + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x[:, 0]) + 10
    lo, up = np.array([-5.0, 0.0]), np.array([10.0, 15.0])
    X = rng.rand(20, 2)
    y = branin(lo + (up - lo) * X)
    y = (y - y.mean()) / y.std()
    Z = rng.rand(50, 2)
    out["branin"] = _posterior(Z, X, y, np.array([0.3, 0.4]), 2.0, 1e-3)
    for nb in (2, 17):
        X = rng.rand(8, 3)
        Z = rng.rand(nb, 3)
        out["rand%d" % nb] = _posterior(Z, X, rng.randn(8), np.array([0.5, 0.5, 0.5]), 1.5, 1e-2)
    return out


def main():
    if not hasattr(np, "Infinity"):
        np.Infinity = np.inf
    if not hasattr(np, "NAN"):
        np.NAN = np.nan
    sys.modules.setdefault("emcee", types.ModuleType("emcee"))
    sys.path.insert(0, REF)
    from robo.util import epmgp

    orig = epmgp.lt_factor
    calls = {}

    def counting(s, *a, **kw):
        calls[s] = calls.get(s, 0) + 1
        return orig(s, *a, **kw)

    epmgp.lt_factor = counting
    data = {}
    for name, (mu, V) in cases().items():
        calls.clear()
        logP, dMu, dSig, dMuMu = epmgp.joint_min(mu, V, with_derivatives=True)
        nb = mu.shape[0]
        keep = 2 if nb >= 50 else nb
        data[name + "_mu"] = mu
        data[name + "_V"] = V
        data[name + "_logP"] = logP
        data[name + "_dlogPdMu"] = dMu[:keep]
        data[name + "_dlogPdSigma"] = dSig[:keep]
        data[name + "_dlogPdMudMu"] = dMuMu[:keep]
        data[name + "_lt_calls"] = np.array([calls.get(k, 0) for k in range(nb)], dtype=np.int64)
        print(name, "Nb =", nb, "lt_factor steps", int(data[name + "_lt_calls"].sum()))
    epmgp.lt_factor = orig
    np.savez(OUT, names=np.array(sorted({k.rsplit("_", 1)[0] for k in data if k.endswith("_mu")})), **data)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
