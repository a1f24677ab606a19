"""``fabolas`` facade with the signature, object wiring and result dict of robo/fmin/fabolas.py:31-312, built from the
robo_b200 classes: the kernel 1 * prod_d Matern52(axes=d) * BayesianLinearRegressionKernel(axes=D) for the objective
and the cost, EnvPrior(n_ls=D, n_lr=2), FabolasGPMCMC with the quadratic (1 - s)^2 and the linear basis, and
MarginalizationGPMCMC(InformationGainPerUnitCost(..., sampling_acquisition=EI, n_representer=50)) maximised by
RandomSampling.  Every model fit, prediction and acquisition runs on the device.

The environment kernel is a restatement (robo_b200/kernels.py: BayesianLinearRegressionKernel): the george fork that
defines it is not public.

Kept from the reference, on purpose:
  - ``n_init * len(subsets) <= num_iterations`` is asserted, and the defaults (40 * 3 > 100) fail it;
  - the initial design evaluates configuration i on every subset s_max / subset (integer division by truncation), and
    its output files are written as fabolas_iter_<i>.json with the entries of position i, once per subset: the file of
    configuration i is rewritten len(subsets) times and ends with entries that belong to evaluation i, not to it;
  - the incumbents of the initial design are argmin of the observed y so far, the env column dropped;
  - ``results["c"]`` holds the log-costs, ``results["y"]`` exp of the log-objective;
  - the final incumbent is estimated by a fresh ``train`` and projected_incumbent_estimation, whatever inc_estimation is.

RandomSampling is built without ``rng`` as in the reference, so it, its incumbent perturbations and
InformationGainPerUnitCost's representer restarts draw from numpy's global state: two runs evaluate the same
configurations when both ``rng`` and ``np.random.seed`` are fixed.  hyper_sampler and representer_sampler select the
device samplers as in the sibling facades ("host", the default, keeps the reference's host samplers).
"""
import json
import logging
import os
import time

import numpy as np

from robo_b200 import kernels
from robo_b200.acquisition_functions import EI, InformationGainPerUnitCost, MarginalizationGPMCMC
from robo_b200.initial_design import init_latin_hypercube_sampling
from robo_b200.maximizers import RandomSampling
from robo_b200.models.fabolas_gp import FabolasGPMCMC
from robo_b200.priors import EnvPrior
from robo_b200.util.incumbent_estimation import projected_incumbent_estimation

logger = logging.getLogger(__name__)


def transform(s, s_min, s_max):
    """Subset size s -> its position in [0, 1] on the log2 scale between s_min and s_max."""
    lo, hi = np.log2(s_min), np.log2(s_max)
    return (np.log2(s) - lo) / (hi - lo)


def retransform(s_transform, s_min, s_max):
    """Inverse of transform, rounded to the nearest integer subset size."""
    lo, hi = np.log2(s_min), np.log2(s_max)
    return int(np.rint(2 ** (s_transform * (hi - lo) + lo)))


def quadratic_bf(x):
    return (1 - x) ** 2


def linear_bf(x):
    return x


def _fabolas_kernel(n_dims):
    """1 * prod_d Matern52 on configuration column d * the environment factor on column n_dims."""
    k = 1
    for d in range(n_dims):
        k *= kernels.Matern52Kernel(np.ones([1]) * 0.01, ndim=n_dims + 1, axes=d)
    return k * kernels.BayesianLinearRegressionKernel(log_a=0.1, log_b=0.1, ndim=n_dims + 1, axes=n_dims)


def _model(n_dims, basis, n_hypers, burnin, chain_length, lower, upper, rng, hyper_sampler):
    kernel = _fabolas_kernel(n_dims)
    prior = EnvPrior(len(kernel) + 1, n_ls=n_dims, n_lr=2, rng=rng)
    return FabolasGPMCMC(kernel, prior=prior, burnin_steps=burnin, chain_length=chain_length, n_hypers=n_hypers,
                         normalize_output=False, basis_func=basis, lower=lower, upper=upper, rng=rng,
                         hyper_sampler=hyper_sampler)


def fabolas(objective_function, lower, upper, s_min, s_max,
            n_init=40, num_iterations=100, subsets=[256, 128, 64], inc_estimation="mean",
            burnin=100, chain_length=100, n_hypers=12, output_path=None, rng=None,
            hyper_sampler="host", representer_sampler="host"):
    """Fast Bayesian Optimization of Machine Learning Hyperparameters on Large Datasets (Klein et al.,
    arXiv:1605.07079).  objective_function(x, s) -> (loss, cost) on a training subset of s points; the loss and the
    cost are modelled on a log scale.  Returns dict(x_opt, incumbents, runtime, overhead, time_func_eval, X, y, c)."""
    assert n_init * len(subsets) <= num_iterations, \
        "the initial design (n_init * len(subsets) evaluations) must fit into num_iterations"
    assert lower.shape[0] == upper.shape[0], "lower and upper bounds differ in dimension"

    t0 = time.time()
    if rng is None:
        rng = np.random.RandomState(np.random.randint(0, 10000))
    n_dims = lower.shape[0]

    # the objective's kernel decides n_hypers: three samples per parameter, even, when 12 is too few
    if n_hypers < 2 * len(_fabolas_kernel(n_dims)):
        n_hypers = 3 * len(_fabolas_kernel(n_dims))
        n_hypers += n_hypers % 2
    model_objective = _model(n_dims, quadratic_bf, n_hypers, burnin, chain_length, lower, upper, rng, hyper_sampler)
    model_cost = _model(n_dims, linear_bf, n_hypers, burnin, chain_length, lower, upper, rng, hyper_sampler)

    ext_lower, ext_upper = np.append(lower, 0), np.append(upper, 1)
    is_env = np.zeros(n_dims + 1)
    is_env[-1] = 1
    acquisition_func = MarginalizationGPMCMC(InformationGainPerUnitCost(
        model_objective, model_cost, ext_lower, ext_upper, sampling_acquisition=EI, is_env_variable=is_env,
        n_representer=50, representer_sampler=representer_sampler))
    maximizer = RandomSampling(acquisition_func, ext_lower, ext_upper)

    evals, overhead, incumbents, runtime = [], [], [], []
    X, y, c = [], [], []

    def evaluate(x, s):
        tic = time.time()
        loss, cost = objective_function(x, s)
        evals.append(time.time() - tic)
        logger.info("f(%s, s=%d) = %f at cost %f (%f s)", str(x), s, loss, cost, evals[-1])
        return np.log(loss), np.log(cost)

    def save(i):
        # file i holds the i-th entry of every list, as the reference writes it (see the module docstring)
        if output_path is None:
            return
        record = {"optimization_overhead": overhead[i], "runtime": runtime[i], "incumbent": incumbents[i].tolist(),
                  "time_func_eval": evals[i], "iteration": i}
        with open(os.path.join(output_path, "fabolas_iter_%d.json" % i), "w") as fh:
            json.dump(record, fh)

    logger.info("Initial Design")
    x_init = init_latin_hypercube_sampling(lower, upper, n_init, rng)
    for i in range(n_init):
        for subset in subsets:
            tic = time.time()
            s = int(s_max / float(subset))
            ly, lc = evaluate(x_init[i], s)
            X.append(np.append(x_init[i], transform(s, s_min, s_max)))
            y.append(ly)
            c.append(lc)
            incumbents.append(X[int(np.argmin(y))][:-1])       # the best observation so far, env column dropped
            overhead.append(time.time() - tic)
            runtime.append(time.time() - t0)
            save(i)

    X, y, c = np.array(X), np.array(y), np.array(c)
    for it in range(len(X), num_iterations):
        logger.info("Start iteration %d ... ", it)
        tic = time.time()
        model_objective.train(X, y, do_optimize=True)
        model_cost.train(X, c, do_optimize=True)

        if inc_estimation == "last_seen":
            best = int(np.argmin(y))
            incumbent, incumbent_value = np.append(X[best][:-1], 1), y[best]
        else:
            incumbent, incumbent_value = projected_incumbent_estimation(model_objective, X[:, :-1], proj_value=1)
        incumbents.append(incumbent[:-1])
        logger.info("Current incumbent %s with estimated performance %f", str(incumbent), np.exp(incumbent_value))

        acquisition_func.update(model_objective, model_cost)
        new_x = maximizer.maximize()
        s = retransform(new_x[-1], s_min, s_max)
        overhead.append(time.time() - tic)

        ly, lc = evaluate(new_x[:-1], s)
        X = np.concatenate((X, new_x[None, :]), axis=0)
        y = np.append(y, ly)
        c = np.append(c, lc)
        runtime.append(time.time() - t0)
        save(it)

    model_objective.train(X, y, do_optimize=True)
    incumbent, incumbent_value = projected_incumbent_estimation(model_objective, X[:, :-1], proj_value=1)
    logger.info("Final incumbent %s with estimated performance %f", str(incumbent), incumbent_value)

    return {"x_opt": incumbent[:-1].tolist(),
            "incumbents": [v.tolist() for v in incumbents],
            "runtime": runtime,
            "overhead": overhead,
            "time_func_eval": evals,
            "X": [row.tolist() for row in X],
            "y": [np.exp(v).tolist() for v in y],         # back from the log scale
            "c": [v.tolist() for v in c]}                 # left on the log scale, as the reference returns it
