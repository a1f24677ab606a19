"""``entropy_search`` facade with the signature and object wiring of robo/fmin/entropy_search.py:20-131: same kernel
(cov_amp * Matern52), DefaultPrior, n_hypers rule, ``InformationGain(gp, lower, upper, sampling_acquisition=EI)``,
MarginalizationGPMCMC wrapping for ``gp_mcmc`` and result dict, built from the robo_b200 classes.  Maximizers:
"random" (RandomSampling) and "differential_evolution" (the evolution on the device, gpk_maximize_de_es, with the
reference's L-BFGS-B polish on the host); "scipy" needs a derivative of the entropy change, which the device path does
not have."""
import numpy as np

from robo_b200 import kernels
from robo_b200.acquisition_functions import EI, InformationGain, MarginalizationGPMCMC
from robo_b200.initial_design import init_latin_hypercube_sampling
from robo_b200.maximizers import DifferentialEvolution, RandomSampling
from robo_b200.models import GaussianProcess, GaussianProcessMCMC
from robo_b200.priors import DefaultPrior
from robo_b200.solver import BayesianOptimization


def entropy_search(objective_function, lower, upper, num_iterations=30, maximizer="random", model="gp_mcmc",
                   X_init=None, Y_init=None, n_init=3, output_path=None, rng=None, representer_sampler="host",
                   hyper_sampler="host", hyper_optimizer="host"):
    assert upper.shape[0] == lower.shape[0], "Dimension miss match"
    assert np.all(lower < upper), "Lower bound >= upper bound"
    assert n_init <= num_iterations, "Number of initial design point has to be <= than the number of iterations"
    if rng is None:
        rng = np.random.RandomState(np.random.randint(0, 10000))
    if maximizer not in ("random", "differential_evolution"):
        raise ValueError("'{}' is not a maximizer of entropy search on the GPU path: InformationGain has no device "
                         "derivative for 'scipy'; use 'random' or 'differential_evolution'".format(maximizer))

    cov_amp = 2
    n_dims = lower.shape[0]
    kernel = cov_amp * kernels.Matern52Kernel(np.ones([n_dims]), ndim=n_dims)
    prior = DefaultPrior(len(kernel) + 1)
    n_hypers = 3 * len(kernel)
    if n_hypers % 2 == 1:
        n_hypers += 1

    if model == "gp":
        # hyper_optimizer="device" runs each train's L-BFGS-B over the marginal likelihood on the device
        # (gpk_optimize_hypers), "host" with scipy
        gp = GaussianProcess(kernel, prior=prior, rng=rng, normalize_output=False, normalize_input=True,
                             lower=lower, upper=upper, hyper_optimizer=hyper_optimizer)
    elif model == "gp_mcmc":
        # hyper_sampler="device" samples the hyper-parameters on the device (gpk_sample_hypers), "host" with
        # EnsembleSampler; the two agree in law, not bit for bit
        gp = GaussianProcessMCMC(kernel, prior=prior, n_hypers=n_hypers, chain_length=200, burnin_steps=100,
                                 normalize_input=True, normalize_output=False, rng=rng, lower=lower, upper=upper,
                                 hyper_sampler=hyper_sampler)
    else:
        raise ValueError("'{}' is not a valid model on the GPU path (gp, gp_mcmc)".format(model))

    # representer_sampler="device" draws the representer points on the device (gpk_sample_representers)
    a = InformationGain(gp, lower=lower, upper=upper, sampling_acquisition=EI, representer_sampler=representer_sampler)
    acquisition_func = a if model == "gp" else MarginalizationGPMCMC(a)
    if maximizer == "random":
        max_func = RandomSampling(acquisition_func, lower, upper, rng=rng)
    else:
        max_func = DifferentialEvolution(acquisition_func, lower, upper, rng=rng)

    bo = BayesianOptimization(objective_function, lower, upper, acquisition_func, gp, max_func,
                              initial_design=init_latin_hypercube_sampling, initial_points=n_init, rng=rng,
                              output_path=output_path)
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
    return results
