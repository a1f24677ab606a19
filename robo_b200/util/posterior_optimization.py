"""posterior_mean_optimization and posterior_mean_plus_std_optimization (robo/util/posterior_optimization.py) with
the restarts on the GPU.

The reference runs scipy's L-BFGS-B from n_restarts uniform starts on mu(x) (or mu(x) + sqrt(v(x))), one predict call
per point.  For a GaussianProcess or a GaussianProcessMCMC whose sub-models take raw inputs, all starts run in lockstep
on the device (gpk_maximize_lbfgs with GPK_OBJ_MEAN / GPK_OBJ_MEAN_STD over the mixture moments of gpk_acq_multi
mode 1), with the same projected L-BFGS and forward differences as SciPyOptimizer.  ``with_gradients`` does not change
the device path: the reference's with_gradients=True calls predictive_gradients, which none of its models has.  Any
other model, Fabolas models included (their inputs are transformed on the host), takes the reference's host loop.
"""
import numpy as np
from scipy import optimize

from robo_b200 import _lib
from robo_b200.initial_design.init_random_uniform import init_random_uniform


def _device_handles(model):
    """The fitted handles whose mixture moments are the model's predict, or None when the model does not run on the
    device with raw inputs."""
    from robo_b200.maximizers.device_spec import raw_inputs
    from robo_b200.models.gaussian_process import GaussianProcess
    from robo_b200.models.gaussian_process_mcmc import GaussianProcessMCMC
    if isinstance(model, GaussianProcess) and raw_inputs(model) and getattr(model, "is_trained", False):
        model.gp._restore()
        model.gp._push_cfg()
        return [model.gp.handle]
    if isinstance(model, GaussianProcessMCMC) and model.is_trained and all(raw_inputs(m) for m in model.models):
        return model.sub_model_handles()
    return None


def _optimize(model, lower, upper, n_restarts, with_gradients, objective, f, df):
    startpoints = init_random_uniform(lower, upper, n_restarts)
    handles = _device_handles(model)
    if handles is not None:
        r = _lib.maximize_lbfgs(handles, objective, None, 0.0, startpoints, lower, upper)
        return r["x"][int(np.argmin(r["energy"]))]
    x_opt = np.zeros([len(startpoints), lower.shape[0]])
    fval = np.zeros([len(startpoints)])
    for i, startpoint in enumerate(startpoints):
        if with_gradients:
            res = optimize.fmin_l_bfgs_b(f, startpoint, df, bounds=list(zip(lower, upper)))
            x_opt[i] = res[0]
            fval[i] = res[1]
        else:
            res = optimize.minimize(f, startpoint, bounds=list(zip(lower, upper)), method="L-BFGS-B")
            x_opt[i] = res["x"]
            fval[i] = res["fun"]
    return x_opt[np.argmin(fval)]


def posterior_mean_optimization(model, lower, upper, n_restarts=10, with_gradients=False):
    """The point of the box with the lowest posterior mean found from n_restarts uniform starts
    (posterior_optimization.py:8-58)."""

    def f(x):
        return model.predict(x[np.newaxis, :])[0][0]

    def df(x):
        return model.predictive_gradients(x[np.newaxis, :])[0]

    return _optimize(model, lower, upper, n_restarts, with_gradients, _lib.OBJ_MEAN, f, df)


def posterior_mean_plus_std_optimization(model, lower, upper, n_restarts=10, with_gradients=False):
    """The point of the box with the lowest posterior mean + standard deviation found from n_restarts uniform starts
    (posterior_optimization.py:61-118)."""

    def f(x):
        mu, var = model.predict(x[np.newaxis, :])
        return (mu + np.sqrt(var))[0]

    def df(x):
        dmu, dvar = model.predictive_gradients(x[np.newaxis, :])
        _, var = model.predict(x[np.newaxis, :])
        dstd = 0.5 * dvar / np.sqrt(var)
        return dmu[:, :, 0] + dstd

    return _optimize(model, lower, upper, n_restarts, with_gradients, _lib.OBJ_MEAN_STD, f, df)
