#!/usr/bin/env python
"""Write tests/golden/fabolas_ig.npz by running the reference's own InformationGainPerUnitCost
(robo/acquisition_functions/information_gain_per_unit_cost.py) over the reference's own FabolasGP models.

Run where the reference tree is available (ROBO_REFERENCE, default /root/reference):

    python tools/make_fabolas_ig_golden.py

Only outputs are kept; no reference code enters the repository.  What is restated underneath the reference:
  - george, by oracle/george_oracle.py (as oracle/make_golden.py:case_fabolas does);
  - emcee, absent here, by robo_b200/util/ensemble_sampler.py's stretch move.  The reference calls run_mcmc without a
    random state, so the shim seeds each run from numpy's global stream: the file is reproducible byte for byte under the
    np.random.seed below.  The representer points and their log-probabilities are stored as sampled; the GPU test
    injects them, so MCMC parity with emcee does not matter.
  - two numpy-2 aliases (np.Infinity, np.NAN) used by robo/util/epmgp.py.

Models: objective with basis (1 - s)^2, cost with basis s (robo/fmin/fabolas.py:96-102), products of three 1-D
Matern-5/2 kernels with fixed hyper-parameters, noise 1e-3, trained with do_optimize=False.  The acquisition: EI as the
sampling acquisition, 50 representer points, Np = 400, overhead 0.1.  Candidates: 120 uniform in the extended box, 10
outside it, 10 training inputs, 10 at small s where the predicted cost is below 1.

Outside the extended box the reference's compute raises (dh_fun returns a (value, gradient) pair there, which
InformationGain.compute cannot store); for those candidates the entropy change is dh_fun's own DBL_EPSILON, divided by
the cost as compute divides it.
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("ROBO_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "fabolas_ig.npz")

LOWER, UPPER = np.array([-1.0, 2.0]), np.array([3.0, 5.0])
OBJ_K = (1.3, (0.4, 0.6, 0.9))
COST_K = (0.8, (0.5, 0.7, 0.6))
NOISE = 1e-3
OVERHEAD = 0.1


def _install_shims():
    sys.path.insert(0, ROOT)
    from oracle import george_oracle as G
    from robo_b200.util.ensemble_sampler import EnsembleSampler
    G.install_as_george()

    class SeededSampler(EnsembleSampler):
        def run_mcmc(self, p0, N, rstate0=None, lnprob0=None):
            if rstate0 is None:
                rstate0 = np.random.RandomState(np.random.randint(0, 2 ** 31 - 1))
            return EnsembleSampler.run_mcmc(self, p0, N, rstate0=rstate0, lnprob0=lnprob0)

    emcee = types.ModuleType("emcee")
    emcee.EnsembleSampler = SeededSampler
    sys.modules["emcee"] = emcee
    if not hasattr(np, "Infinity"):
        np.Infinity = np.inf
    if not hasattr(np, "NAN"):
        np.NAN = np.nan
    sys.path.insert(0, REF)
    return G


def data():
    rng = np.random.RandomState(20261016)
    X = np.concatenate((LOWER + (UPPER - LOWER) * rng.rand(30, 2), rng.uniform(0.05, 1.0, (30, 1))), axis=1)
    y = np.sin(X[:, 0]) + 0.3 * X[:, 1] + (1 - X[:, 2]) ** 2
    c = -1.2 + 2.5 * X[:, 2] + 0.1 * X[:, 0]                  # log cost, below 0 for small s
    lo, up = np.append(LOWER, 0.0), np.append(UPPER, 1.0)
    Xt = lo + (up - lo) * rng.rand(150, 3)
    Xt[120:125] = up + 0.1 + rng.rand(5, 3)                   # outside the extended box
    Xt[125:128] = lo - 0.2
    Xt[128, 2], Xt[129, 0] = 1.2, -1.5
    Xt[130:140] = X[:10]                                      # training inputs
    Xt[140:150, 2] = 0.02 * rng.rand(10)                      # small s: predicted cost below 1
    return X, y, c, Xt, lo, up


def main():
    G = _install_shims()
    from robo.acquisition_functions.ei import EI
    from robo.acquisition_functions.information_gain_per_unit_cost import InformationGainPerUnitCost
    from robo.models.fabolas_gp import FabolasGP

    def kernel(spec):
        amp, ls = spec
        k = amp * G.kernels.Matern52Kernel(np.ones(1) * ls[0], ndim=3, axes=0)
        k *= G.kernels.Matern52Kernel(np.ones(1) * ls[1], ndim=3, axes=1)
        k *= G.kernels.Matern52Kernel(np.ones(1) * ls[2], ndim=3, axes=2)
        return k

    X, y, c, Xt, lo, up = data()
    obj = FabolasGP(kernel(OBJ_K), basis_function=lambda s: (1 - s) ** 2, noise=NOISE, lower=LOWER, upper=UPPER,
                    rng=np.random.RandomState(0))
    obj.train(X, y, do_optimize=False)
    cost = FabolasGP(kernel(COST_K), basis_function=lambda s: s, noise=NOISE, lower=LOWER, upper=UPPER,
                     rng=np.random.RandomState(1))
    cost.train(X, c, do_optimize=False)
    is_env = np.array([0, 0, 1])
    np.random.seed(7)
    ig = InformationGainPerUnitCost(obj, cost, lo, up, is_env_variable=is_env, sampling_acquisition=EI, n_representer=50)
    ig.update(obj, cost, overhead=OVERHEAD)
    log_cost = cost.predict(Xt)[0]
    inside = np.all((Xt >= lo) & (Xt <= up), axis=1)
    values = np.empty(len(Xt))
    values[inside] = ig.compute(Xt[inside])
    # Outside the box the reference's dh_fun returns the pair (dH, gradient) even for derivative=False, which
    # InformationGain.compute cannot store (ValueError).  dH is taken from dh_fun itself and divided as compute divides.
    for i in np.where(~inside)[0]:
        dh = float(ig.dh_fun(Xt[i][None, :])[0][0, 0])
        values[i] = dh / (np.exp(log_cost[i]) + ig.overhead)
    np.savez(OUT, X=X, y=y, c=c, lower=LOWER, upper=UPPER, extend_lower=lo, extend_upper=up, is_env=is_env,
             obj_amp=OBJ_K[0], obj_ls=np.array(OBJ_K[1]), cost_amp=COST_K[0], cost_ls=np.array(COST_K[1]),
             noise=NOISE, overhead=OVERHEAD, zb=np.array(ig.zb), lmb=np.array(ig.lmb), Np=ig.Np, Xt=Xt,
             values=values, log_cost=log_cost)
    print("wrote", OUT, "finite", int(np.isfinite(values).sum()), "cost < 1", int(np.sum(np.exp(log_cost) < 1)))


if __name__ == "__main__":
    main()
