#!/usr/bin/env python
"""Write tests/golden/mtbo_ref.npz and tests/golden/mtbo_ig.npz by running the reference's own MTBO wrapper code
(robo/models/mtbo_gp.py: MTBOGP, MTBOGPMCMC; robo/priors/env_priors.py: MTBOPrior;
robo/acquisition_functions/information_gain_per_unit_cost.py: InformationGainPerUnitCost) on the oracle.

Run where the reference tree is available (ROBO_REFERENCE, default /root/reference), CPU only:

    python tools/make_mtbo_golden.py

Only outputs are kept; no reference code enters the repository.  What is restated underneath the reference:
  - george, by oracle/george_oracle.py, with two additions made here at run time: george.kernels.TaskKernel(ndim, axis,
    num_tasks) is the restated task kernel of tests/task_kernel_model.py (the fork's source is not public), and the
    kernels' ``vector`` gets george 0.2's setter, which mtbo_gp.py:94 assigns;
  - emcee, absent here, by robo_b200/util/ensemble_sampler.py's stretch move, seeded from numpy's global stream (as
    tools/make_fabolas_ig_golden.py does); the representer points are stored as sampled and injected by the GPU test;
  - two numpy-2 aliases (np.Infinity, np.NAN) used by robo/util/epmgp.py.

So the files pin the reference's wrapper code (input maps, the get_incumbent projection, sample handling of
MTBOGPMCMC, the prior, the acquisition over MTBO models), not the kernel.

mtbo_ref.npz: MTBOPrior.lnprob at chosen theta and sample_from_prior under a seeded rng; MTBOGP predictions and its
get_incumbent winner; MTBOGPMCMC(do_optimize=False) predictions, once on the kernel's own parameters and once on
earlier hyper-parameter samples (kept when training without optimisation).
mtbo_ig.npz: InformationGainPerUnitCost over an objective and a cost MTBOGP, candidates inside the extended box (task
values continuous in [0, n_tasks - 1], rint ties at 0.5 and 1.5 included) and outside it (there the value is dh_fun's
own DBL_EPSILON divided by the cost, as tools/make_fabolas_ig_golden.py explains).  Outside candidates keep a task
value that rounds to a task: the restated kernel is NaN elsewhere, and the oracle's solver refuses NaN.
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("ROBO_REFERENCE", "/root/reference")
OUT_REF = os.path.join(ROOT, "tests", "golden", "mtbo_ref.npz")
OUT_IG = os.path.join(ROOT, "tests", "golden", "mtbo_ig.npz")

N_TASKS = 3
LOWER, UPPER = np.array([-1.0, 2.0]), np.array([3.0, 5.0])
OBJ_K = (1.3, (0.4, 0.6), (-0.2, -0.7, 0.1, -0.4, -0.9, 0.2))
COST_K = (0.8, (0.5, 0.7), (0.1, -0.3, -0.5, -0.1, 0.0, -0.6))
NOISE = 1e-3
OVERHEAD = 0.1


def _install_shims():
    sys.path.insert(0, ROOT)
    from oracle import george_oracle as G
    from robo_b200.util.ensemble_sampler import EnsembleSampler
    from tests import task_kernel_model as T
    G.install_as_george()

    class TaskKernel(T.TaskKernel):
        def __init__(self, ndim, axis, num_tasks):
            super(TaskKernel, self).__init__(np.zeros(T.n_kt(num_tasks)), num_tasks, ndim=ndim, axes=[axis])
    G.kernels.TaskKernel = TaskKernel
    G.Kernel.vector = property(G.Kernel.get_parameter_vector, lambda self, v: self.set_parameter_vector(v))

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


def kernel(G, spec):
    amp, ls, theta = spec
    k = amp * G.kernels.Matern52Kernel(np.ones(1) * ls[0], ndim=3, axes=0)
    k *= G.kernels.Matern52Kernel(np.ones(1) * ls[1], ndim=3, axes=1)
    task = G.kernels.TaskKernel(3, 2, N_TASKS)
    task.set_parameter_vector(np.array(theta))
    return k * task


def data():
    rng = np.random.RandomState(20261017)
    X = np.concatenate((LOWER + (UPPER - LOWER) * rng.rand(30, 2), rng.randint(0, N_TASKS, (30, 1))), axis=1)
    y = np.sin(X[:, 0]) + 0.3 * X[:, 1] + 0.4 * X[:, 2]
    c = -1.2 + 1.1 * X[:, 2] + 0.1 * X[:, 0]                  # log cost, below 0 on task 0
    lo, up = np.append(LOWER, 0.0), np.append(UPPER, N_TASKS - 1.0)
    Xt = lo + (up - lo) * rng.rand(150, 3)
    Xt[120:125, :2] = UPPER + 0.1 + rng.rand(5, 2)            # outside the extended box in the configuration columns
    Xt[125:128, :2] = LOWER - 0.2
    Xt[128, 2], Xt[129, 0] = N_TASKS - 0.5, -1.5              # outside in the task column only: rint(2.5) = 2
    Xt[130:136, 2] = [0.5, 1.5, 0.5, 1.5, 0.49999999, 1.50000001]   # rint ties (half to even) and their neighbours
    Xt[136:146] = X[:10]                                      # training inputs
    return X, y, c, Xt, lo, up


def main():
    G = _install_shims()
    from robo.acquisition_functions.ei import EI
    from robo.acquisition_functions.information_gain_per_unit_cost import InformationGainPerUnitCost
    from robo.models.mtbo_gp import MTBOGP, MTBOGPMCMC
    from robo.priors.env_priors import MTBOPrior

    X, y, c, Xt, lo, up = data()
    n_kt = N_TASKS * (N_TASKS + 1) // 2

    # ---- mtbo_ref.npz ----
    prior = MTBOPrior(1 + 2 + n_kt + 1, n_ls=2, n_kt=n_kt, rng=np.random.RandomState(11))
    theta = np.array([[0.7, -3.0, 1.0, -0.5, -0.2, -0.9, -0.1, -0.6, -0.3, -4.0],
                      [2.0, 0.5, -9.0, 0.0, -1.0, -0.5, -0.5, -0.5, -0.5, -2.0],
                      [0.7, -3.0, 1.0, 0.1, -0.2, -0.9, -0.1, -0.6, -0.3, -4.0],      # task entry above 0
                      [0.7, -3.0, 3.0, -0.5, -0.2, -0.9, -0.1, -0.6, -0.3, -4.0],     # length scale above 2
                      [-0.5, -3.0, 1.0, -0.5, -0.2, -0.9, -0.1, -0.6, -1.2, -4.0]])
    lnprob = np.array([prior.lnprob(t) for t in theta])
    samples = prior.sample_from_prior(7)

    gp = MTBOGP(kernel(G, OBJ_K), noise=NOISE, lower=LOWER, upper=UPPER, rng=np.random.RandomState(0))
    gp.train(X, y, do_optimize=False)
    gp_mu, gp_var = gp.predict(Xt[:120])
    inc, inc_val = gp.get_incumbent()

    mc = MTBOGPMCMC(kernel(G, OBJ_K), lower=LOWER, upper=UPPER, rng=np.random.RandomState(0))
    mc.train(X, y, do_optimize=False)
    mc_mu, mc_var = mc.predict(Xt[:120])
    hypers = np.array([np.r_[np.log(1.3 / 3), np.log([0.4, 0.6]), OBJ_K[2], -6.0],
                       np.r_[np.log(0.9 / 3), np.log([0.8, 0.3]), np.array(OBJ_K[2]) - 0.3, -5.0],
                       np.r_[np.log(2.0 / 3), np.log([0.2, 0.9]), np.array(OBJ_K[2]) + 0.1, -7.0]])
    mc2 = MTBOGPMCMC(kernel(G, OBJ_K), lower=LOWER, upper=UPPER, rng=np.random.RandomState(0))
    mc2.hypers = hypers
    mc2.train(X, y, do_optimize=False)
    mc2_mu, mc2_var = mc2.predict(Xt[:120])
    np.savez(OUT_REF, X=X, y=y, Xt=Xt[:120], lower=LOWER, upper=UPPER, n_tasks=N_TASKS, obj_amp=OBJ_K[0],
             obj_ls=np.array(OBJ_K[1]), obj_theta=np.array(OBJ_K[2]), noise=NOISE,
             prior_theta=theta, prior_lnprob=lnprob, prior_seed=11, prior_samples=samples,
             gp_mu=gp_mu, gp_var=gp_var, inc=inc, inc_val=inc_val, mc_mu=mc_mu, mc_var=mc_var,
             hypers=hypers, mc2_mu=mc2_mu, mc2_var=mc2_var)

    # ---- mtbo_ig.npz ----
    obj = MTBOGP(kernel(G, OBJ_K), noise=NOISE, lower=LOWER, upper=UPPER, rng=np.random.RandomState(0))
    obj.train(X, y, do_optimize=False)
    cost = MTBOGP(kernel(G, COST_K), noise=NOISE, lower=LOWER, upper=UPPER, rng=np.random.RandomState(1))
    cost.train(X, c, do_optimize=False)
    is_env = np.array([0, 0, 1])
    np.random.seed(7)
    ig = InformationGainPerUnitCost(obj, cost, lo, up, is_env_variable=is_env, sampling_acquisition=EI, n_representer=50)
    ig.update(obj, cost, overhead=OVERHEAD)
    log_cost = cost.predict(Xt)[0]
    inside = np.all((Xt >= lo) & (Xt <= up), axis=1)
    values = np.empty(len(Xt))
    values[inside] = ig.compute(Xt[inside])
    for i in np.where(~inside)[0]:
        dh = float(ig.dh_fun(Xt[i][None, :])[0][0, 0])
        values[i] = dh / (np.exp(log_cost[i]) + ig.overhead)
    np.savez(OUT_IG, X=X, y=y, c=c, lower=LOWER, upper=UPPER, extend_lower=lo, extend_upper=up, is_env=is_env,
             n_tasks=N_TASKS, obj_amp=OBJ_K[0], obj_ls=np.array(OBJ_K[1]), obj_theta=np.array(OBJ_K[2]),
             cost_amp=COST_K[0], cost_ls=np.array(COST_K[1]), cost_theta=np.array(COST_K[2]), noise=NOISE,
             overhead=OVERHEAD, zb=np.array(ig.zb), lmb=np.array(ig.lmb), Np=ig.Np, Xt=Xt, values=values,
             log_cost=log_cost)
    print("wrote", OUT_REF, OUT_IG, "finite", int(np.isfinite(values).sum()), "outside", int((~inside).sum()),
          "lnprob", lnprob)


if __name__ == "__main__":
    main()
