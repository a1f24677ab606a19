"""Host-side helpers of the GPU path (training-data scaling, the ensemble sampler used by GP-MCMC)."""
from .posterior_optimization import posterior_mean_optimization, posterior_mean_plus_std_optimization  # noqa: F401
