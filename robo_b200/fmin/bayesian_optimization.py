"""``bayesian_optimization`` facade with the signature and object wiring of
robo/fmin/bayesian_optimization.py:27-158 for the GP model types (``gp``, ``gp_mcmc``): same kernel
(cov_amp * Matern52, :75-81), DefaultPrior, n_hypers rule (:85-87), acquisition switch (:114-129),
MarginalizationGPMCMC wrapping (:126-129) and result dict (:149-157) — built from the robo_b200
classes so BASELINE.json configs[0] runs on the GPU box.  Orchestration only."""
import numpy as np

from robo_b200 import kernels
from robo_b200.acquisition_functions import EI, LCB, PI, LogEI, MarginalizationGPMCMC
from robo_b200.initial_design import init_latin_hypercube_sampling
from robo_b200.maximizers import DifferentialEvolution, RandomSampling
from robo_b200.models import GaussianProcess, GaussianProcessMCMC
from robo_b200.priors import DefaultPrior
from robo_b200.solver import BayesianOptimization


def bayesian_optimization(objective_function, lower, upper, num_iterations=30, X_init=None, Y_init=None,
                          maximizer="random", acquisition_func="log_ei", model_type="gp_mcmc",
                          n_init=3, rng=None, output_path=None, n_candidates=500,
                          chain_length=200, burnin_steps=100, hyper_sampler="host", hyper_optimizer="host"):
    assert upper.shape[0] == lower.shape[0], "Dimension miss match"
    assert np.all(lower < upper), "Lower bound >= upper bound"
    assert n_init <= num_iterations, "Number of initial design point has to be <= than the number of iterations"
    if rng is None:
        rng = np.random.RandomState(np.random.randint(0, 10000))

    cov_amp = 2
    n_dims = lower.shape[0]
    kernel = cov_amp * kernels.Matern52Kernel(np.ones([n_dims]), ndim=n_dims)
    prior = DefaultPrior(len(kernel) + 1)
    n_hypers = 3 * len(kernel)
    if n_hypers % 2 == 1:
        n_hypers += 1

    if model_type == "gp":
        # hyper_optimizer="device" runs each train's L-BFGS-B over the marginal likelihood on the device
        # (gpk_optimize_hypers), "host" with scipy
        model = GaussianProcess(kernel, prior=prior, rng=rng, normalize_output=False, normalize_input=True,
                                lower=lower, upper=upper, hyper_optimizer=hyper_optimizer)
    elif model_type == "gp_mcmc":
        # hyper_sampler="device" samples the hyper-parameters on the device (gpk_sample_hypers), "host" with
        # EnsembleSampler; the two agree in law, not bit for bit
        model = GaussianProcessMCMC(kernel, prior=prior, n_hypers=n_hypers, chain_length=chain_length,
                                    burnin_steps=burnin_steps, normalize_input=True, normalize_output=False,
                                    rng=rng, lower=lower, upper=upper, hyper_sampler=hyper_sampler)
    else:
        raise ValueError("'{}' is not a valid model on the GPU path (gp, gp_mcmc)".format(model_type))

    acq_cls = {"ei": EI, "log_ei": LogEI, "pi": PI, "lcb": LCB}.get(acquisition_func)
    if acq_cls is None:
        raise ValueError("'{}' is not a valid acquisition function".format(acquisition_func))
    a = acq_cls(model)
    acq = MarginalizationGPMCMC(a) if model_type == "gp_mcmc" else a

    if maximizer == "random":
        max_func = RandomSampling(acq, lower, upper, n_samples=n_candidates, rng=rng)
    elif maximizer == "differential_evolution":
        max_func = DifferentialEvolution(acq, lower, upper, rng=rng)
    else:
        raise ValueError("'{}' is not accelerated on the GPU path; use 'random', 'differential_evolution' or pass the robo_b200 "
                         "objects to the reference's own maximizers".format(maximizer))

    bo = BayesianOptimization(objective_function, lower, upper, acq, model, max_func, initial_points=n_init,
                              rng=rng, initial_design=init_latin_hypercube_sampling, output_path=output_path)
    x_best, f_min = bo.run(num_iterations, X=X_init, y=Y_init)

    results = dict()
    results["x_opt"] = x_best
    results["f_opt"] = f_min
    results["incumbents"] = [inc for inc in bo.incumbents]
    results["incumbent_values"] = [val for val in bo.incumbents_values]
    results["runtime"] = bo.runtime
    results["overhead"] = bo.time_overhead
    results["X"] = [x.tolist() for x in bo.X]
    results["y"] = [y for y in bo.y]
    results["time_train"] = bo.time_train
    results["time_maximize"] = bo.time_maximize
    return results
