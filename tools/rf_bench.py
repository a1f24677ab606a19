"""RandomForest on the device against the reference's cost structure restated on the host, at three shapes (T = 30):

  branin    D = 2, N = 30
  d8        D = 8, N = 200
  d16       D = 16, N = 2000

pyrfr is not available, so the host arm is scikit-learn's RandomForestRegressor(n_estimators=30, max_features=None,
bootstrap=True, n_jobs=-1) on all of this machine's cores (the count is printed): the same kind of forest from a
compiled library, predicted the way the reference's wrapper predicts (random_forest.py:106-107 calls
predict_mean_var once per row; the batch arms use one batched sklearn predict, which is cheaper than that loop).

Arms, each timing ending in a device synchronise:
  train1 / train2   the first train() on a fresh model and a later one on the same model
  ei65k / ei1m      predict + EI + arg-max over 65,536 and 2^20 candidates (host: batched predict, per-tree variance
                    by the law of total variance over the trees' predictions, scipy EI, argmax; device: gpk_acq_multi)
  de                DifferentialEvolution.maximize (20 generations, 20 x D members) against scipy's
                    differential_evolution(maxiter=20), polish on as the reference maximizer runs it, on the one-row
                    acquisition (one sklearn predict per row)
  direct            Direct.maximize at its defaults against scipy.optimize.direct with the same budget on the one-row
                    acquisition
One untimed device warm-up per shape, then alternating host / device rounds; median, [min, max].  Prints one JSON line
per round and a summary line, each with the card's name and power limit read in the same call.

    python tools/rf_bench.py [--rounds 3] [--shapes branin,d8,d16] [--arms train,ei,de,direct]
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
from robo_b200.maximizers import DifferentialEvolution, Direct  # noqa: E402
from robo_b200.models import RandomForest  # noqa: E402

SHAPES = {"branin": (2, 30), "d8": (8, 200), "d16": (16, 2000)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:
        return "unknown (%s)" % e, "unknown"


def sync():
    import torch
    if torch.cuda.is_available():
        torch.cuda.synchronize()


def problem(D, N, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.rand(N, D)
    return X, np.sin(3 * X).sum(axis=1) + 0.1 * rng.randn(N)


def host_forest(X, y):
    from sklearn.ensemble import RandomForestRegressor
    return RandomForestRegressor(n_estimators=30, max_features=None, bootstrap=True, n_jobs=-1,
                                 random_state=0).fit(X, y)


def host_moments(f, X):
    P = np.array([t.predict(X) for t in f.estimators_])
    return P.mean(axis=0), P.var(axis=0)


def host_ei(f, X, eta):
    m, v = host_moments(f, X)
    s = np.sqrt(v)
    with np.errstate(divide="ignore", invalid="ignore"):
        z = (eta - m) / s
        e = s * (z * norm.cdf(z) + norm.pdf(z))
    return np.where(s == 0, 0.0, e)


def timed(fn):
    sync()
    t0 = time.perf_counter()
    out = fn()
    sync()
    return time.perf_counter() - t0, out


def arms(shape, which, rounds, name, power):
    D, N = SHAPES[shape]
    X, y = problem(D, N)
    eta = float(y.min())
    lo, up = np.zeros(D), np.ones(D)
    dev = RandomForest(rng=np.random.RandomState(1))
    dev.train(X, y)                                           # warm-up
    hf = host_forest(X, y)
    rows = []
    cands = {k: np.random.RandomState(k).rand(k, D) for k in (65536, 1 << 20)}

    def one_row(x):
        return -float(host_ei(hf, np.atleast_2d(x), eta)[0])
    for r in range(rounds):
        res = {}
        if "train" in which:
            res["train1_host"] = timed(lambda: host_forest(X, y))[0]
            m = RandomForest(rng=np.random.RandomState(r))
            res["train1_dev"] = timed(lambda: m.train(X, y))[0]
            res["train2_host"] = timed(lambda: host_forest(X, y))[0]
            res["train2_dev"] = timed(lambda: m.train(X, y))[0]
        if "ei" in which:
            for k, C in cands.items():
                tag = "ei65k" if k == 65536 else "ei1m"
                res[tag + "_host"] = timed(lambda: int(np.argmax(host_ei(hf, C, eta))))[0]
                h = dev._ready_handle()
                res[tag + "_dev"] = timed(lambda: _lib.acq_multi([h], C, 0, kind=_lib.ACQ_EI, eta=[eta], par=0.0,
                                                                 want_argmax=True)["best_idx"])[0]
        if "de" in which:
            res["de_host"] = timed(lambda: optimize.differential_evolution(one_row, list(zip(lo, up)), maxiter=20,
                                                                           seed=r))[0]
            res["de_dev"] = timed(lambda: DifferentialEvolution(EI(dev), lo, up, n_iters=20,
                                                                rng=np.random.RandomState(r)).maximize())[0]
        if "direct" in which:
            mx = Direct(EI(dev), lo, up, verbose=False)
            res["direct_host"] = timed(lambda: optimize.direct(one_row, list(zip(lo, up)), maxiter=mx.n_iters,
                                                               maxfun=mx.n_func_evals, locally_biased=False))[0]
            res["direct_dev"] = timed(lambda: mx.maximize())[0]
        line = dict(shape=shape, round=r, card=name, power_limit=power, cores=os.cpu_count(), seconds=res)
        print(json.dumps(line), flush=True)
        rows.append(res)
    keys = rows[0].keys()
    summary = {k: dict(median=float(np.median([x[k] for x in rows])), min=float(min(x[k] for x in rows)),
                       max=float(max(x[k] for x in rows))) for k in keys}
    name, power = card()
    print(json.dumps(dict(shape=shape, summary=summary, card=name, power_limit=power, cores=os.cpu_count())),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="branin,d8,d16")
    ap.add_argument("--arms", default="train,ei,de,direct")
    a = ap.parse_args()
    for s in a.shapes.split(","):
        name, power = card()
        arms(s, a.arms.split(","), a.rounds, name, power)


if __name__ == "__main__":
    main()
