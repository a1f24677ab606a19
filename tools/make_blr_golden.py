#!/usr/bin/env python
"""Write tests/golden/blr.npz by running the reference's own BayesianLinearRegression
(robo/models/bayesian_linear_regression.py) and BayesianLinearRegressionPrior, with robo_b200's EnsembleSampler
registered as sys.modules["emcee"] (emcee is not installed; oracle/make_golden.py registers the george restatement the
same way).

Run where the reference tree is available, with ROBO_REFERENCE naming its root (the directory that holds robo/):
    ROBO_REFERENCE=/path/to/RoBO python tools/make_blr_golden.py
Only inputs and outputs are kept; no reference code enters the repository.

Cases (key prefixes):
  unit_*     the reference unit test's data (D = 1, y = 2 x), trained with do_optimize=False: models and predict
  lin_* / quad_* / none_*   D = 4 linear (N = 50), D = 3 quadratic (N = 40), D = 2 with basis_func=None (N = 30):
             the mll on a theta grid (prior -inf for theta_0 <= -10, the det overflow to +inf, theta_1 <= 0 for the
             horseshoe of 1 / theta_1), (m, S) at three (alpha, beta) pairs, predict over all three at test points
  fmin_*     the do_mcmc=False path from RandomState(3) on the lin_ data: hypers
  mcmc_*     the reference example's data (D = 1, N = 20, linear), three seeds at the default chain (20 walkers, 2000
             burn-in + 2000 steps): final walkers, the mean and sd of log alpha / log beta, predict at test points
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("ROBO_REFERENCE")
OUT = os.path.join(ROOT, "tests", "golden", "blr.npz")
HYPERS = np.array([[1.0, 1000.0], [0.5, 200.0], [2.0, 50.0]])
MCMC_SEEDS = (11, 12, 13)


def _reference():
    if not REF:
        raise SystemExit("set ROBO_REFERENCE to the root of the reference tree (the directory that holds robo/)")
    sys.path.insert(0, ROOT)
    from robo_b200.util import ensemble_sampler
    em = types.ModuleType("emcee")
    em.EnsembleSampler = ensemble_sampler.EnsembleSampler
    sys.modules["emcee"] = em
    sys.path.insert(0, REF)
    from robo.models import bayesian_linear_regression as R
    return R


def _grid():
    t0 = np.array([-12.0, -9.5, -3.0, 0.0, 1.5, 150.0])
    t1 = np.array([-2.0, 0.0, 0.5, 3.0, 7.0])
    return np.array([[a, b] for a in t0 for b in t1])


def main():
    R = _reference()
    out = {}
    # the reference unit test (test/test_models/test_bayesian_linear_regression.py)
    rng = np.random.RandomState(5)
    X = rng.rand(10, 1)
    y = (X * 2)[:, 0]
    Xt = rng.rand(10, 1)
    m = R.BayesianLinearRegression(alpha=1, beta=1000, rng=np.random.RandomState(0))
    m.train(X, y, do_optimize=False)
    mu, var = m.predict(Xt)
    out.update(unit_X=X, unit_y=y, unit_Xt=Xt, unit_m=m.models[0][0], unit_S=m.models[0][1], unit_mu=mu, unit_var=var,
               unit_mll=m.marginal_log_likelihood(np.array([np.log(1), np.log(1000)])))

    grid = _grid()
    for name, d, n, basis in (("lin", 4, 50, R.linear_basis_func), ("quad", 3, 40, R.quadratic_basis_func),
                              ("none", 2, 30, None)):
        rng = np.random.RandomState(100 + d)
        X = rng.rand(n, d)
        y = np.sin(3 * X).sum(axis=1) + 0.1 * rng.randn(n)
        Xt = rng.rand(25, d)
        m = R.BayesianLinearRegression(basis_func=basis, rng=np.random.RandomState(1))
        m.train(X, y, do_optimize=False)
        with np.errstate(all="ignore"):
            mll = np.array([m.marginal_log_likelihood(t) for t in grid])
        Phi = m.X_transformed
        cond = []
        for t in grid:
            with np.errstate(all="ignore"):
                A = np.exp(t[1]) * Phi.T @ Phi + np.exp(t[0]) * np.eye(Phi.shape[1])
                cond.append(np.linalg.cond(A) if np.all(np.isfinite(A)) else np.inf)
        models = []
        for a, b in HYPERS:
            mm = R.BayesianLinearRegression(alpha=a, beta=b, basis_func=basis, rng=np.random.RandomState(1))
            mm.train(X, y, do_optimize=False)
            models.append(mm.models[0])
        m.hypers = [list(h) for h in HYPERS]
        m.models = models
        mu, var = m.predict(Xt)
        out.update({name + "_X": X, name + "_y": y, name + "_Xt": Xt, name + "_grid": grid, name + "_mll": mll,
                    name + "_cond": np.array(cond), name + "_hypers": HYPERS,
                    name + "_m": np.array([a for a, _ in models]), name + "_S": np.array([s for _, s in models]),
                    name + "_mu": mu, name + "_var": var})

    # do_mcmc=False: optimize.fmin(negative_mll, rng.rand(2)) from a fixed rng
    m = R.BayesianLinearRegression(do_mcmc=False, rng=np.random.RandomState(3))
    m.train(out["lin_X"], out["lin_y"], do_optimize=True)
    out.update(fmin_hypers=np.array(m.hypers, dtype=np.float64))

    # the reference example (examples/example_blr.py): f(x) = 10 x - 5 + noise, 20 uniform points
    rng = np.random.RandomState(42)
    X = rng.uniform(0, 1, (20, 1))
    y = (10 * X - 5 + 0.001 * rng.randn(20, 1))[:, 0]
    Xt = np.linspace(0, 1, 11)[:, None]
    walkers, mus, vars_ = [], [], []
    for s in MCMC_SEEDS:
        m = R.BayesianLinearRegression(rng=np.random.RandomState(s))
        m.train(X, y, do_optimize=True)
        walkers.append(m.p0.copy())
        mu, var = m.predict(Xt)
        mus.append(mu)
        vars_.append(var)
        print("seed %d: mean log alpha %.4f, log beta %.4f" % (s, m.p0[:, 0].mean(), m.p0[:, 1].mean()))
    W = np.array(walkers)
    out.update(mcmc_X=X, mcmc_y=y, mcmc_Xt=Xt, mcmc_seeds=np.array(MCMC_SEEDS), mcmc_walkers=W,
               mcmc_mean=W.reshape(-1, 2).mean(axis=0), mcmc_sd=W.reshape(-1, 2).std(axis=0, ddof=1),
               mcmc_mu=np.array(mus), mcmc_var=np.array(vars_))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
