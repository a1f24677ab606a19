"""BayesianLinearRegression on the device against the reference's cost structure restated on the host, at three shapes:

  example   the reference example (examples/example_blr.py): D = 1, N = 20, linear basis
  d8        D = 8, N = 200, quadratic basis (F = 17)
  d32       D = 32, N = 2000, linear basis (F = 33)

Arms, each timing ending in a device synchronise:
  train     train() with 20 walkers, the first train (burn-in + chain) and a later one (one more row, chain only), at
            the reference defaults (2000 + 2000 steps) for example and d8; d32 runs 200 + 200 steps on both arms,
            because one host train at the defaults there takes minutes.  Host: robo_b200's EnsembleSampler over the
            numpy mll in the reference's order (tests/blr_model.py, the code the CPU tests use) and the reference's
            (m, S) loop.  Device:
            BayesianLinearRegression.train (gpk_blr_sample + gpk_blr_fit)
  ei        EI of 65,536 candidates and its arg-max: host numpy predict in the reference's order (on pieces of 1024
            rows: the reference forms an M x M matrix per hyper-sample) + scipy EI + argmax; device gpk_acq_multi
  de        DifferentialEvolution.maximize (20 generations) against scipy's differential_evolution(maxiter=20) on the
            one-point acquisition the reference's maximizer calls
One untimed device warm-up train per shape, then alternating host / device rounds; median, [min, max].  The final
walkers of both samplers are scored by gpk_blr_lnpost: their mean log-posterior over the finite ones and the finite fraction.  Prints
one JSON line per round and a summary line, each with the card's name and power limit read in the same call.

    python tools/blr_bench.py [--rounds 3] [--shapes example,d8,d32] [--out blr_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
from scipy import optimize
from scipy.stats import norm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from robo_b200 import _lib  # noqa: E402
from robo_b200.acquisition_functions import EI  # noqa: E402
from robo_b200.maximizers import DifferentialEvolution  # noqa: E402
from robo_b200.models.bayesian_linear_regression import (BayesianLinearRegression, linear_basis_func,  # noqa: E402
                                                         quadratic_basis_func)
from robo_b200.priors import BayesianLinearRegressionPrior  # noqa: E402
from robo_b200.util.ensemble_sampler import EnsembleSampler  # noqa: E402
from tests import blr_model as BM  # noqa: E402

SHAPES = {"example": (1, 20, _lib.BLR_LINEAR), "d8": (8, 200, _lib.BLR_QUADRATIC), "d32": (32, 2000, _lib.BLR_LINEAR)}
STEPS = {"example": 2000, "d8": 2000, "d32": 200}      # burn-in steps = chain steps of both arms
FUNCS = {_lib.BLR_LINEAR: linear_basis_func, _lib.BLR_QUADRATIC: quadratic_basis_func}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:
        return "unknown (%s)" % e, "unknown"


def data(shape):
    d, n, _ = SHAPES[shape]
    rng = np.random.RandomState(42)
    X = rng.rand(n + 1, d)
    y = 10 * X.sum(axis=1) - 5 + 0.1 * np.sin(7 * X).sum(axis=1) + 0.001 * rng.randn(n + 1)
    return X, y


def sync():
    import torch
    torch.cuda.synchronize()


def host_train(shape, seed):
    """The reference's train() twice (first + later), its emcee run restated over the numpy mll."""
    X, y = data(shape)
    basis = SHAPES[shape][2]
    rng = np.random.RandomState(seed)
    prior = BayesianLinearRegressionPrior(rng=rng)
    times, p0 = [], None
    for rows in (len(X) - 1, len(X)):
        t0 = time.perf_counter()
        Phi = BM.features(X[:rows], basis)
        f = BM.lnpost(Phi, y[:rows])
        s = EnsembleSampler(20, 2, None, batch_lnpostfn=f)
        if p0 is None:
            p0 = prior.sample_from_prior(20)
            p0, _, _ = s.run_mcmc(p0, STEPS[shape], rstate0=rng)
        pos, _, _ = s.run_mcmc(p0, STEPS[shape], rstate0=rng)
        p0 = pos
        hypers = np.exp(s.chain[:, -1])
        models = BM.fit(Phi, y[:rows], hypers)
        times.append(time.perf_counter() - t0)
    return times, p0, (hypers, models)


def device_train(shape, seed):
    X, y = data(shape)
    m = BayesianLinearRegression(basis_func=FUNCS[SHAPES[shape][2]], rng=np.random.RandomState(seed),
                                 chain_length=STEPS[shape], burnin_steps=STEPS[shape])
    times = []
    for rows in (len(X) - 1, len(X)):
        t0 = time.perf_counter()
        m.train(X[:rows], y[:rows], do_optimize=True)
        sync()
        times.append(time.perf_counter() - t0)
    return times, m.p0, m


def walker_stats(shape, P):
    X, y = data(shape)
    h = _lib.Handle(0)
    _lib.blr_set_data(h, X, y, SHAPES[shape][2], BM.PRIOR_PAR)
    v = _lib.blr_lnpost(h, P)
    fin = np.isfinite(v)
    return float(v[fin].mean()) if fin.any() else float("-inf"), float(fin.mean())


def host_ei(shape, hm, Xc, eta):
    hypers, models = hm
    t0 = time.perf_counter()
    Phi = BM.features(Xc, SHAPES[shape][2])
    # the reference's predict forms np.dot(np.dot(X, S), X.T), an M x M matrix per hyper-sample (34 GB at M = 65,536):
    # the host arm runs it on pieces of 1024 rows
    parts = [BM.predict(Phi[i:i + 1024], hypers, models) for i in range(0, len(Phi), 1024)]
    m, v = np.concatenate([a for a, _ in parts]), np.concatenate([b for _, b in parts])
    s = np.sqrt(v)
    z = (eta - m) / s
    f = s * (z * norm.cdf(z) + norm.pdf(z))
    best = int(np.argmax(f))
    return time.perf_counter() - t0, best


def device_ei(model, Xc, eta):
    h = model._ready_handle()
    t0 = time.perf_counter()
    r = _lib.acq_multi([h], Xc, 0, kind=_lib.ACQ_EI, eta=[eta], par=0.0, want_argmax=True)
    sync()
    return time.perf_counter() - t0, int(r["best_idx"])


def host_de(shape, hm, eta, seed):
    hypers, models = hm
    d = SHAPES[shape][0]

    def neg_ei(x):
        m, v = BM.predict(BM.features(x[None], SHAPES[shape][2]), hypers, models)
        s = np.sqrt(v[0])
        z = (eta - m[0]) / s
        return -(s * (z * norm.cdf(z) + norm.pdf(z)))
    t0 = time.perf_counter()
    r = optimize.differential_evolution(neg_ei, [(0.0, 1.0)] * d, maxiter=20, seed=seed, polish=False)
    return time.perf_counter() - t0, float(-r.fun)


def device_de(model, seed):
    d = model.X.shape[1]
    acq = EI(model)
    mx = DifferentialEvolution(acq, np.zeros(d), np.ones(d), n_iters=20, rng=np.random.RandomState(seed))
    t0 = time.perf_counter()
    x = mx.maximize()
    sync()
    return time.perf_counter() - t0, float(np.ravel(acq.compute(np.atleast_2d(x)))[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="example,d8,d32")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    name, power = card()
    summary = dict(card=name, power_limit=power, shapes={})
    for shape in args.shapes.split(","):
        rows = []
        device_train(shape, 99)                        # warm-up of the device arm (module load, first launches)
        for rnd in range(1, args.rounds + 1):
            seed = 100 + rnd
            order = ("host", "device") if rnd % 2 == 0 else ("device", "host")
            res = {}
            for arm in order:
                print("# %s round %d: %s arm" % (shape, rnd, arm), flush=True)
                if arm == "host":
                    res["host_train"], P, hm = host_train(shape, seed)
                    res["host_walkers"] = walker_stats(shape, P)
                else:
                    res["device_train"], P, model = device_train(shape, seed)
                    res["device_walkers"] = walker_stats(shape, P)
            X, y = data(shape)
            eta = float(np.min(y))
            Xc = np.random.RandomState(seed).rand(65536, SHAPES[shape][0])
            res["host_ei"], hb = host_ei(shape, hm, Xc, eta)
            res["device_ei"], db = device_ei(model, Xc, eta)
            res["host_de"], hv = host_de(shape, hm, eta, seed)
            res["device_de"], dv = device_de(model, seed)
            res["de_values"] = (hv, dv)
            line = dict(card=name, power_limit=power, shape=shape, steps=STEPS[shape], round=rnd, **res)
            print(json.dumps(line), flush=True)
            rows.append(res)

        def stat(key, i=None):
            v = np.array([r[key][i] if i is not None else r[key] for r in rows])
            return dict(median=float(np.median(v)), min=float(v.min()), max=float(v.max()))
        summary["shapes"][shape] = dict(
            steps=STEPS[shape],
            train_first=dict(host=stat("host_train", 0), device=stat("device_train", 0)),
            train_later=dict(host=stat("host_train", 1), device=stat("device_train", 1)),
            ei_65536=dict(host=stat("host_ei"), device=stat("device_ei")),
            de=dict(host=stat("host_de"), device=stat("device_de")),
            walkers_mean_lnpost=dict(host=stat("host_walkers", 0), device=stat("device_walkers", 0)),
            walkers_finite=dict(host=stat("host_walkers", 1), device=stat("device_walkers", 1)))
    print(json.dumps(dict(summary=summary)), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
