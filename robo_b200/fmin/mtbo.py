"""``mtbo`` facade with the signature, object wiring and result dict of robo/fmin/mtbo.py:34-280, built from the
robo_b200 classes: the kernel 1 * prod_d Matern52(axes=d) * TaskKernel(D + 1, D, n_tasks) for the objective and the
cost, MTBOPrior(n_ls=D, n_kt=len(task kernel)), MTBOGPMCMC, and MarginalizationGPMCMC(InformationGainPerUnitCost(...,
sampling_acquisition=EI, n_representer=50)) over the box extended by the task column [0, n_tasks - 1], maximised by
RandomSampling.  Every model fit, prediction and acquisition runs on the device.

The task kernel is a restatement (robo_b200/kernels.py: TaskKernel): the george fork that defines it is not public.

Kept from the reference, on purpose:
  - n_hypers becomes 3 * len(kernel), made even, when it is below 2 * len(kernel);
  - the cost prior is built with the objective task kernel's n_kt;
  - the initial design evaluates one Latin-hypercube point per iteration, each on task 0, and its incumbents are argmin
    of the observed y so far, the task column dropped;
  - the loop incumbent is the best observation projected to task 1 (its estimated value is y, not a prediction); the
    final one is estimated by a fresh train and projected_incumbent_estimation to task n_tasks - 1;
  - the task the maximizer returns is rounded with np.rint before the evaluation;
  - ``results["X"]``, ``["y"]`` and ``["c"]`` are numpy arrays, y and c on the log scale.

RandomSampling is built without ``rng`` as in the reference, so it and InformationGainPerUnitCost's representer restarts
draw from numpy's global state: two runs evaluate the same configurations when both ``rng`` and ``np.random.seed`` are
fixed.  hyper_sampler and representer_sampler select the device samplers as in the sibling facades ("host", the
default, keeps the reference's host samplers).
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
from robo_b200.models.mtbo_gp import MTBOGPMCMC
from robo_b200.priors import MTBOPrior
from robo_b200.util.incumbent_estimation import projected_incumbent_estimation

logger = logging.getLogger(__name__)


def _mtbo_kernel(n_dims, n_tasks):
    """(1 * prod_d Matern52 on configuration column d * the task kernel on column n_dims, the task kernel)."""
    k = 1
    for d in range(n_dims):
        k *= kernels.Matern52Kernel(np.ones([1]) * 0.01, ndim=n_dims + 1, axes=d)
    task_kernel = kernels.TaskKernel(n_dims + 1, n_dims, n_tasks)
    return k * task_kernel, task_kernel


def mtbo(objective_function, lower, upper, n_tasks=2, n_init=2, num_iterations=30,
         burnin=100, chain_length=200, n_hypers=20, output_path=None, rng=None,
         hyper_sampler="host", representer_sampler="host"):
    """Multi-Task Bayesian Optimization (Swersky, Snoek, Adams, NIPS 2013): an auxiliary cheaper task speeds up the
    optimisation of a more expensive, similar one.  objective_function(x, task) -> (loss, cost); the loss and the cost
    are modelled on a log scale.  Returns dict(x_opt, incumbents, runtime, overhead, time_func_eval, X, y, c)."""
    assert n_init <= num_iterations, "Number of initial design point has to be <= than the number of iterations"
    assert lower.shape[0] == upper.shape[0], "Dimension miss match between upper and lower bound"

    time_start = time.time()
    if rng is None:
        rng = np.random.RandomState(np.random.randint(0, 10000))
    n_dims = lower.shape[0]

    time_func_eval, time_overhead, incumbents, runtime = [], [], [], []
    X, y, c = [], [], []

    kernel, task_kernel = _mtbo_kernel(n_dims, n_tasks)
    if n_hypers < 2 * len(kernel):
        n_hypers = 3 * len(kernel)
        if n_hypers % 2 == 1:
            n_hypers += 1
    prior = MTBOPrior(len(kernel) + 1, n_ls=n_dims, n_kt=len(task_kernel), rng=rng)
    model_objective = MTBOGPMCMC(kernel, prior=prior, burnin_steps=burnin, chain_length=chain_length,
                                 n_hypers=n_hypers, lower=lower, upper=upper, rng=rng, hyper_sampler=hyper_sampler)

    cost_kernel, _ = _mtbo_kernel(n_dims, n_tasks)
    cost_prior = MTBOPrior(len(cost_kernel) + 1, n_ls=n_dims, n_kt=len(task_kernel), rng=rng)
    model_cost = MTBOGPMCMC(cost_kernel, prior=cost_prior, burnin_steps=burnin, chain_length=chain_length,
                            n_hypers=n_hypers, lower=lower, upper=upper, rng=rng, hyper_sampler=hyper_sampler)

    extend_lower, extend_upper = np.append(lower, 0), np.append(upper, n_tasks - 1)
    is_env = np.zeros(extend_lower.shape[0])
    is_env[-1] = 1
    ig = InformationGainPerUnitCost(model_objective, model_cost, extend_lower, extend_upper, sampling_acquisition=EI,
                                    is_env_variable=is_env, n_representer=50, representer_sampler=representer_sampler)
    acquisition_func = MarginalizationGPMCMC(ig)
    maximizer = RandomSampling(acquisition_func, extend_lower, extend_upper)

    def save(it):
        if output_path is None:
            return
        data = {"optimization_overhead": time_overhead[it], "runtime": runtime[it],
                "incumbent": incumbents[it].tolist(), "time_func_eval": time_func_eval[it], "iteration": it}
        with open(os.path.join(output_path, "mtbo_iter_%d.json" % it), "w") as fh:
            json.dump(data, fh)

    logger.info("Initial Design")
    for it in range(n_init):
        start_time_overhead = time.time()
        task = 0                                   # the initial design evaluates the auxiliary task only
        x = init_latin_hypercube_sampling(lower, upper, 1, rng)[0]
        st = time.time()
        func_val, cost = objective_function(x, task)
        time_func_eval.append(time.time() - st)
        logger.info("f(%s, task=%d) = %f at cost %f (%f s)", str(x), task, func_val, cost, time_func_eval[-1])
        X.append(np.append(x, task))
        y.append(np.log(func_val))
        c.append(np.log(cost))
        incumbents.append(X[int(np.argmin(y))][:-1])
        time_overhead.append(time.time() - start_time_overhead)
        runtime.append(time.time() - time_start)
        save(it)

    X, y, c = np.array(X), np.array(y), np.array(c)
    for it in range(n_init, num_iterations):
        logger.info("Start iteration %d ... ", it)
        start_time = time.time()
        model_objective.train(X, y, do_optimize=True)
        model_cost.train(X, c, do_optimize=True)

        best_idx = np.argmin(y)
        incumbent = np.append(X[best_idx][:-1], 1)
        incumbent_value = y[best_idx]
        incumbents.append(incumbent[:-1])
        logger.info("Current incumbent %s with estimated performance %f", str(incumbent), np.exp(incumbent_value))

        acquisition_func.update(model_objective, model_cost)
        new_x = maximizer.maximize()
        new_x[-1] = np.rint(new_x[-1])             # the continuous task coordinate to a task index
        time_overhead.append(time.time() - start_time)

        start_time = time.time()
        new_y, new_c = objective_function(new_x[:-1], new_x[-1])
        time_func_eval.append(time.time() - start_time)
        logger.info("f(%s) = %f at cost %f (%f s)", str(new_x), new_y, new_c, time_func_eval[-1])

        X = np.concatenate((X, new_x[None, :]), axis=0)
        y = np.concatenate((y, np.log(np.array([new_y]))), axis=0)
        c = np.concatenate((c, np.log(np.array([new_c]))), axis=0)
        runtime.append(time.time() - time_start)
        save(it)

    model_objective.train(X, y)
    incumbent, incumbent_value = projected_incumbent_estimation(model_objective, X[:, :-1], proj_value=n_tasks - 1)
    logger.info("Final incumbent %s with estimated performance %f", str(incumbent), incumbent_value)

    return {"x_opt": incumbent[:-1].tolist(),
            "incumbents": [inc.tolist() for inc in incumbents],
            "runtime": runtime,
            "overhead": time_overhead,
            "time_func_eval": time_func_eval,
            "X": X,
            "y": y,
            "c": c}
