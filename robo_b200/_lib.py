"""ctypes binding of include/gpk.h — the stub a RoBO maintainer would add (INTEGRATION.md).

There is deliberately NO CPU fallback: if libgpk.so cannot be loaded, or no CUDA device is
present, every compute call raises.  Status codes map to the exceptions the reference's
callers already handle (SURVEY.md section 8b "Error conventions"):
    GPK_NOT_PD     -> numpy.linalg.LinAlgError   (gaussian_process.py:120,156)
    GPK_BAD_ARG    -> ValueError
    GPK_CUDA_ERROR -> RuntimeError
    GPK_EP_FAILED  -> Exception with the reference's message (robo/util/epmgp.py:204-207)
"""
import ctypes as C
import os

import numpy as np

from . import _build

GPK_OK, GPK_NOT_PD, GPK_BAD_ARG, GPK_CUDA_ERROR, GPK_NOT_FITTED, GPK_NOT_APPLICABLE, GPK_EP_FAILED = range(7)
MATERN52, EXPSQUARED, MATERN32 = 0, 1, 2
ACQ_NONE, ACQ_EI, ACQ_LOG_EI, ACQ_PI, ACQ_LCB = range(5)
ACQ_KIND = {"ei": ACQ_EI, "log_ei": ACQ_LOG_EI, "pi": ACQ_PI, "lcb": ACQ_LCB, "none": ACQ_NONE}
OBJ_MEAN, OBJ_MEAN_STD = 5, 6                  # GPK_OBJ_MEAN / GPK_OBJ_MEAN_STD: posterior objectives of gpk_maximize_lbfgs
LB_MAX_D = 64                                  # GPK_LB_MAX_D: largest input dimension of gpk_maximize_lbfgs*
# gpk_lb_status: why a start of gpk_maximize_lbfgs* stopped (FTOL and PGTOL are scipy's success)
LB_FTOL, LB_PGTOL, LB_MAXITER, LB_MAXFUN, LB_ABNORMAL, LB_INVALID = range(6)
BASIS_S, BASIS_ONE_MINUS_S_SQ, BASIS_TASK = range(3)   # gpk_basis: the last column's map of a Fabolas / MTBO model
PRIOR_NONE, PRIOR_DEFAULT, PRIOR_ENV, PRIOR_MTBO = range(4)   # gpk_prior_kind: the hyper-priors gpk_sample_hypers restates
MAX_TASKS = 8                                 # GPK_MAX_TASKS
HYPER_MAX_N = 232                              # GPK_HYPER_MAX_N: most training points of gpk_sample_hypers
HYPER_MAX_DIM = 96                             # GPK_HYPER_MAX_DIM: most entries of theta (log noise included)
HO_CHUNK = 16                                  # GPK_HO_CHUNK: rounds of gpk_optimize_hypers between two status reads
HYPER_BLOCKED_MAX_N = 8192                     # GPK_HYPER_BLOCKED_MAX_N: most training points of gpk_*_blocked
HYPER_BATCH_BYTES = 4294967296                 # GPK_HYPER_BATCH_BYTES: default chunk budget of gpk_*_blocked
BLR_LINEAR, BLR_QUADRATIC, BLR_NONE = range(3)  # gpk_blr_basis: the features of a BayesianLinearRegression handle
BLR_MAX_F = 64                                 # GPK_BLR_MAX_F: most features of a BayesianLinearRegression handle
RF_MAX_N, RF_MAX_D, RF_MAX_T = 16384, 64, 512  # GPK_RF_MAX_N / GPK_RF_MAX_D / GPK_RF_MAX_T: the largest forest
BNN_MAX_N, BNN_MAX_D, BNN_MAX_BATCH = 4096, 64, 32   # GPK_BNN_MAX_N / GPK_BNN_MAX_D / GPK_BNN_MAX_BATCH
DNGO_MAX_N, DNGO_MAX_D, DNGO_MAX_BATCH = 4096, 64, 16   # GPK_DNGO_MAX_N / GPK_DNGO_MAX_D / GPK_DNGO_MAX_BATCH
DNGO_H = 50                                    # units per hidden layer of a DNGO net: the features per row
CMA_MAX_D, CMA_MAX_LAMBDA, CMA_HIST = 64, 2048, 160   # GPK_CMA_MAX_D / GPK_CMA_MAX_LAMBDA / GPK_CMA_HIST
CMA_C_W = 20                                   # GPK_CMA_C_W: where a run's weights start in its constant row
CMA_NCONST = CMA_C_W + CMA_MAX_LAMBDA // 2     # GPK_CMA_NCONST: doubles per run in the constant table
# gpk_cmaes_stop: why a CMA-ES run stopped (RUNNING: not stopped, or never started)
CMA_RUNNING, CMA_MAXFEVALS, CMA_TOLFUN, CMA_TOLX, CMA_CONDITIONCOV, CMA_NUMERICAL = range(6)
CMA_STOP_NAMES = ("running", "maxfevals", "tolfun", "tolx", "conditioncov", "numerical")
DIRECT_MAX_D, DIRECT_MAXDEEP, DIRECT_MAXDIV = 64, 600, 5000   # GPK_DIRECT_MAX_D / _MAXDEEP / _MAXDIV
DIRECT_MAX_RECTS = 1 << 22                     # GPK_DIRECT_MAX_RECTS: most rectangles of one run's store
# gpk_direct_stop: why a DIRECT run stopped
DIRECT_RUNNING, DIRECT_MAXF, DIRECT_MAXT, DIRECT_FGLOBAL, DIRECT_MAXDEEP_HIT, DIRECT_MAXDIV_HIT = range(6)
DIRECT_STOP_NAMES = ("running", "maxf", "maxT", "fglobal", "maxdeep", "maxdiv")

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_lp = C.POINTER(C.c_long)
_vp = C.c_void_p

_SIGNATURES = {
    "gpk_create": [C.POINTER(_vp), C.c_int],
    "gpk_destroy": [_vp],
    "gpk_set_option": [_vp, C.c_char_p, C.c_long],
    "gpk_set_stream": [_vp, _vp],
    "gpk_synchronize": [_vp],
    "gpk_set_data": [_vp, _dp, _dp, C.c_int, C.c_int],
    "gpk_set_input_bounds": [_vp, _dp, _dp, C.c_int],
    "gpk_set_output_transform": [_vp, C.c_int, C.c_double, C.c_double],
    "gpk_set_kernel": [_vp, C.c_int, C.c_double, C.c_int, _ip, _ip, _dp],
    "gpk_set_env_factor": [_vp, C.c_int, C.c_double, C.c_double],
    "gpk_set_task_factor": [_vp, C.c_int, C.c_int, _dp],
    "gpk_fit": [_vp, C.c_double, C.c_double, _dp, _dp],
    "gpk_fit_begin": [_vp, C.c_double, C.c_double],
    "gpk_fit_end": [_vp, _dp, _dp],
    "gpk_fit_append": [_vp, _dp, _dp, C.c_int, C.c_int, C.c_double, C.c_double, _dp, _dp],
    "gpk_predict": [_vp, _dp, C.c_long, _dp, _dp],
    "gpk_predict_cov": [_vp, _dp, C.c_long, _dp, _dp],
    "gpk_posterior_cov": [_vp, _dp, C.c_long, _dp, _dp],
    "gpk_acq": [_vp, _dp, C.c_long, C.c_int, C.c_double, C.c_double, _dp, _dp, _dp, _dp, _lp, _lp],
    "gpk_acq_dev": [_vp, _vp, C.c_long, C.c_int, C.c_double, C.c_double, _vp, _vp, _vp, _vp],
    "gpk_predict_grad": [_vp, _dp, C.c_long, C.c_int, C.c_double, C.c_double, _dp, _dp, _dp, _dp, _dp, _dp],
    "gpk_maximize_random": [_vp, C.c_ulonglong, C.c_long, C.c_long, C.c_long, _dp, _dp, _dp, C.c_double, C.c_int,
                            C.c_double, C.c_double, _dp, _dp, _lp],
    "gpk_generate_candidates": [_vp, C.c_ulonglong, C.c_long, C.c_long, C.c_long, C.c_int, _dp, _dp, _dp, C.c_double, _dp],
    "gpk_acq_moments": [_vp, _dp, _dp, C.c_long, C.c_int, C.c_double, C.c_double, _dp, _lp],
    "gpk_kernel_matrix": [_vp, _dp, C.c_long, _dp, C.c_long, C.c_int, _dp],
    "gpk_reduce_models": [_vp, _dp, _dp, C.c_int, C.c_long, C.c_int, _dp, _dp],
    "gpk_acq_multi": [C.POINTER(_vp), C.c_int, _dp, C.c_long, C.c_int, C.c_int, _dp, C.c_double, _dp, _dp, _lp, _dp, _lp],
    "gpk_maximize_de": [C.POINTER(_vp), C.c_int, C.c_ulonglong, C.c_long, C.c_int, C.c_double, C.c_double, C.c_double,
                        C.c_double, C.c_double, _dp, _dp, C.c_int, _dp, C.c_double, _dp, _dp, _ip, _lp, _lp, _dp, _dp],
    "gpk_comm_unique_id": [_vp],
    "gpk_comm_init": [_vp, C.c_int, C.c_int, _vp],
    "gpk_comm_destroy": [_vp],
    "gpk_comm_info": [_vp, _ip, _ip, _ip],
    "gpk_shard_bounds": [C.c_long, C.c_int, C.c_int, _lp, _lp],
    "gpk_comm_argmax_pair": [_vp, C.c_double, C.c_long, _dp, _lp],
    "gpk_acq_argmax_sharded": [_vp, _dp, C.c_long, C.c_int, C.c_double, C.c_double, _dp, _lp],
    "gpk_acq_argmax_sharded_dev": [_vp, _vp, C.c_long, C.c_long, C.c_int, C.c_double, C.c_double, _vp],
    "gpk_maximize_random_sharded": [_vp, C.c_ulonglong, C.c_long, C.c_long, _dp, _dp, _dp, C.c_double, C.c_int,
                                    C.c_double, C.c_double, _dp, _dp, _lp],
    "gpk_nll_grad": [_vp, C.c_double, _dp],
    "gpk_measure_fp64_peaks": [_vp, _dp, _dp],
    "gpk_measure_int8_peak": [_vp, _dp],
    "gpk_measure_int8_peak_sustained": [_vp, C.c_double, C.c_int, _dp],
    "gpk_get_factor": [_vp, _dp],
    "gpk_get_linv": [_vp, _dp],
    "gpk_get_z": [_vp, _dp],
    "gpk_oz_contract": [_vp, _dp, C.c_int, _dp, C.c_long, C.c_double, _dp, _ip, _ip],
    "gpk_ep_joint_min": [_vp, _dp, _dp, C.c_int, _dp, _dp, _dp, _dp, _ip],
    "gpk_es_update": [_vp, _dp, C.c_int, _dp, C.c_double, _dp, C.c_int, _dp, _dp, _dp, _dp, _dp, _dp],
    "gpk_es_compute": [_vp, _dp, C.c_long, _dp],
    "gpk_es_compute_dev": [_vp, _vp, C.c_long, _vp],
    "gpk_es_moments": [_vp, _dp, C.c_long, _dp, _dp],
    "gpk_es_get_u": [_vp, _dp],
    "gpk_es_dims": [_vp, _ip, _ip],
    "gpk_mc_pmin": [_vp, _dp, C.c_int, _dp, C.c_int, C.c_int, C.c_ulonglong, _dp, _ip],
    "gpk_mc_draws": [_vp, C.c_ulonglong, C.c_int, C.c_int, _dp],
    "gpk_esmc_update": [_vp, _dp, C.c_int, _dp, C.c_double, _dp, C.c_int, C.c_int, C.c_ulonglong, _dp, _dp],
    "gpk_esmc_compute": [_vp, _dp, C.c_long, _dp],
    "gpk_esmc_compute_dev": [_vp, _vp, C.c_long, _vp],
    "gpk_esmc_multi": [C.POINTER(_vp), C.c_int, _dp, C.c_long, _dp, _dp, _lp],
    "gpk_esmc_multi_dev": [C.POINTER(_vp), C.c_int, _vp, C.c_long, _vp, _vp],
    "gpk_maximize_de_esmc": [C.POINTER(_vp), C.c_int, C.c_ulonglong, C.c_long, C.c_int, C.c_double, C.c_double,
                             C.c_double, C.c_double, C.c_double, _dp, _dp, _dp, _dp, _ip, _lp, _dp, _dp],
    "gpk_esmc_get_draws": [_vp, _dp],
    "gpk_esmc_get_state": [_vp, _dp, _dp],
    "gpk_esmc_last_jitter": [_vp, _lp],
    "gpk_predict_mean": [_vp, _dp, C.c_long, _dp],
    "gpk_predict_mean_dev": [_vp, _vp, C.c_long, _vp],
    "gpk_es_cost_multi": [C.POINTER(_vp), C.POINTER(_vp), C.c_int, _dp, C.c_long, _dp, _dp, C.c_int, C.c_int, C.c_int,
                          C.c_double, _dp, _dp, _lp],
    "gpk_es_cost_multi_dev": [C.POINTER(_vp), C.POINTER(_vp), C.c_int, _vp, C.c_long, _dp, _dp, C.c_int, C.c_int, C.c_int,
                              C.c_double, _vp, _vp],
    "gpk_maximize_random_es_cost": [C.POINTER(_vp), C.POINTER(_vp), C.c_int, C.c_ulonglong, C.c_long, C.c_long, _dp, _dp,
                                    _dp, C.c_double, _dp, _dp, C.c_int, C.c_int, C.c_int, C.c_double, _dp, _dp, _lp],
    "gpk_es_multi": [C.POINTER(_vp), C.c_int, _dp, C.c_long, _dp, _dp, _lp],
    "gpk_es_multi_dev": [C.POINTER(_vp), C.c_int, _vp, C.c_long, _vp, _vp],
    "gpk_maximize_de_es": [C.POINTER(_vp), C.c_int, C.c_ulonglong, C.c_long, C.c_int, C.c_double, C.c_double, C.c_double,
                           C.c_double, C.c_double, _dp, _dp, _dp, _dp, _ip, _lp, _dp, _dp],
    "gpk_maximize_de_es_cost": [C.POINTER(_vp), C.POINTER(_vp), C.c_int, C.c_ulonglong, C.c_long, C.c_int, C.c_double,
                                C.c_double, C.c_double, C.c_double, C.c_double, _dp, _dp, _dp, _dp, C.c_int, C.c_int,
                                C.c_int, C.c_double, _dp, _dp, _ip, _lp, _dp, _dp],
    "gpk_maximize_lbfgs": [C.POINTER(_vp), C.c_int, C.c_int, _dp, C.c_double, C.c_long, _dp, _dp, _dp, C.c_int, C.c_int,
                           C.c_long, C.c_double, C.c_double, _dp, _dp, _ip, _lp, _ip, _lp],
    "gpk_maximize_lbfgs_es": [C.POINTER(_vp), C.c_int, C.c_long, _dp, _dp, _dp, C.c_int, C.c_int, C.c_long, C.c_double,
                              C.c_double, _dp, _dp, _ip, _lp, _ip],
    "gpk_maximize_lbfgs_es_cost": [C.POINTER(_vp), C.POINTER(_vp), C.c_int, C.c_long, _dp, _dp, _dp, _dp, _dp, C.c_int,
                                   C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_long, C.c_double, C.c_double,
                                   _dp, _dp, _ip, _lp, _ip],
    "gpk_maximize_cmaes": [C.POINTER(_vp), C.c_int, C.c_int, _dp, C.c_double, C.c_ulonglong, _dp, C.c_double, _dp, _dp,
                           C.c_long, C.c_int, _dp, _vp, _lp],
    "gpk_maximize_cmaes_es": [C.POINTER(_vp), C.c_int, C.c_ulonglong, _dp, C.c_double, _dp, _dp, C.c_long, C.c_int, _dp,
                              _vp],
    "gpk_maximize_cmaes_esmc": [C.POINTER(_vp), C.c_int, C.c_ulonglong, _dp, C.c_double, _dp, _dp, C.c_long, C.c_int,
                                _dp, _vp],
    "gpk_maximize_cmaes_es_cost": [C.POINTER(_vp), C.POINTER(_vp), C.c_int, C.c_ulonglong, _dp, C.c_double, _dp, _dp,
                                   C.c_long, C.c_int, _dp, _dp, _dp, C.c_int, C.c_int, C.c_int, C.c_double, _vp],
    "gpk_maximize_direct": [C.POINTER(_vp), C.c_int, C.c_int, _dp, C.c_double, _dp, _dp, C.c_long, C.c_int, _vp, _lp],
    "gpk_maximize_direct_es": [C.POINTER(_vp), C.c_int, _dp, _dp, C.c_long, C.c_int, _vp],
    "gpk_maximize_direct_esmc": [C.POINTER(_vp), C.c_int, _dp, _dp, C.c_long, C.c_int, _vp],
    "gpk_maximize_direct_es_cost": [C.POINTER(_vp), C.POINTER(_vp), C.c_int, _dp, _dp, C.c_long, C.c_int, _dp, _dp,
                                    C.c_int, C.c_int, C.c_int, C.c_double, _vp],
    "gpk_cmaes_draws": [_vp, C.c_ulonglong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _dp],
    "gpk_sample_representers": [C.POINTER(_vp), C.c_int, C.POINTER(C.c_ulonglong), C.c_int, C.c_int, C.c_int, C.c_int,
                                _dp, C.c_double, _dp, _dp, C.c_int, C.c_int, _dp, _dp, C.c_int, C.c_double, _dp, _dp,
                                _ip, _lp, _lp],
    "gpk_set_hyper_model": [_vp, C.c_int, _ip, _ip, C.c_int, C.c_double, C.c_double, C.c_int, _dp, C.c_int, C.c_int],
    "gpk_hyper_lnpost": [_vp, _dp, C.c_int, C.c_int, _dp, _dp],
    "gpk_sample_hypers": [_vp, _dp, C.c_int, C.c_int, C.c_int, C.c_ulonglong, _dp, _dp, _lp],
    "gpk_optimize_hypers": [_vp, _dp, C.c_int, C.c_int, C.c_int, C.c_long, C.c_double, C.c_double, C.c_double, C.c_int,
                            _dp, _dp, _ip, _lp, _ip],
    "gpk_optimize_hypers_blocked": [_vp, _dp, C.c_int, C.c_int, C.c_int, C.c_long, C.c_double, C.c_double, C.c_double, C.c_int,
                            _dp, _dp, _ip, _lp, _ip],
    "gpk_hyper_lnpost_blocked": [_vp, _dp, C.c_int, C.c_int, _dp, _dp],
    "gpk_sample_hypers_blocked": [_vp, _dp, C.c_int, C.c_int, C.c_int, C.c_ulonglong, _dp, _dp, _lp],
    "gpk_blr_set_data": [_vp, _dp, _dp, C.c_int, C.c_int, C.c_int, _dp],
    "gpk_blr_lnpost": [_vp, _dp, C.c_int, _dp],
    "gpk_blr_sample": [_vp, C.c_ulonglong, C.c_int, _dp, C.c_int, _dp, _dp, _lp],
    "gpk_blr_fit": [_vp, _dp, C.c_int],
    "gpk_blr_get_models": [_vp, _dp, _dp],
    "gpk_blr_dims": [_vp, _ip, _ip, _ip],
    "gpk_rf_set_data": [_vp, _dp, _dp, C.c_int, C.c_int],
    "gpk_rf_fit": [_vp, C.c_ulonglong, C.c_uint, C.c_int, C.c_int, C.c_int, C.c_int],
    "gpk_rf_dims": [_vp, _ip, _ip, _ip, _ip],
    "gpk_rf_get_trees": [_vp, _ip, _ip, _dp, _ip, _dp, _dp, _dp],
    "gpk_rf_set_trees": [_vp, C.c_int, C.c_int, _ip, _ip, _dp, _ip, _dp, _dp, _dp],
    "gpk_bnn_set_data": [_vp, _dp, _dp, C.c_int, C.c_int],
    "gpk_bnn_train": [_vp, C.c_ulonglong, C.c_uint, C.c_double, C.c_double, C.c_double, C.c_long, C.c_long, C.c_long,
                      C.c_int],
    "gpk_bnn_dims": [_vp, _ip, _ip, _ip, _ip],
    "gpk_bnn_get_samples": [_vp, _dp],
    "gpk_bnn_set_samples": [_vp, C.c_int, _dp],
    "gpk_bnn_get_state": [_vp, _dp, _dp, _dp, _dp, _dp],
    "gpk_bnn_draws": [_vp, C.c_ulonglong, C.c_uint, C.c_int, C.c_int, _dp],
    "gpk_dngo_set_data": [_vp, _dp, _dp, C.c_int, C.c_int, C.c_int, C.c_int, _dp],
    "gpk_dngo_train": [_vp, C.c_ulonglong, C.c_uint, C.c_double, C.c_int, C.c_int],
    "gpk_dngo_fit": [_vp, _dp, C.c_int],
    "gpk_dngo_dims": [_vp, _ip, _ip, _ip, _ip],
    "gpk_dngo_get_net": [_vp, _dp],
    "gpk_dngo_set_net": [_vp, _dp],
    "gpk_dngo_features": [_vp, _dp, C.c_long, _dp],
    "gpk_dngo_get_state": [_vp, _dp, _dp, C.POINTER(C.c_longlong)],
    "gpk_get_timings": [_vp, _dp],
    "gpk_get_diag_profile": [_vp, C.POINTER(C.c_longlong)],
}

_lib = None


def library_path():
    return _build.LIB


def load(build_if_missing=True):
    """dlopen libgpk.so (building it first if the sources are newer). Raises if impossible."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if build_if_missing and os.environ.get("GPK_NO_BUILD") != "1":
        try:
            _build.build()
        except Exception as e:
            if not os.path.exists(path):
                raise
            # sources are newer than the binary and cannot be rebuilt (no nvcc on this box): the binary that travelled
            # with the tree is used, loudly; the ABI check below still refuses a library that lacks a declared symbol
            import warnings
            warnings.warn("libgpk.so is older than its sources and could not be rebuilt (%s); using the existing binary"
                          % str(e).splitlines()[0])
    if not os.path.exists(path):
        raise RuntimeError("libgpk.so is missing (%s) and could not be built; there is no CPU fallback" % path)
    lib = C.CDLL(path)
    for name, argtypes in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if a declared symbol is not exported
        fn.argtypes = argtypes
        fn.restype = C.c_int
    lib.gpk_last_error.argtypes = [_vp]
    lib.gpk_last_error.restype = C.c_char_p
    lib.gpk_version.argtypes = []
    lib.gpk_version.restype = C.c_char_p
    _lib = lib
    return lib


def exported_symbols():
    return sorted(list(_SIGNATURES) + ["gpk_last_error", "gpk_version"])


def _as_dp(a):
    return a.ctypes.data_as(_dp)


def f64(a):
    """C-contiguous float64 view/copy (the ABI takes plain double*)."""
    return np.ascontiguousarray(a, dtype=np.float64)


class Handle(object):
    """Owns one gpk_handle (one fitted GP on one GPU)."""

    def __init__(self, device=0):
        self.lib = load()
        self.device = int(device)
        h = _vp()
        rc = self.lib.gpk_create(C.byref(h), self.device)
        if rc != GPK_OK:
            raise RuntimeError("gpk_create failed on device %d (status %d): no usable CUDA device; "
                               "robo_b200 has no CPU fallback" % (self.device, rc))
        self._h = h
        # test/diagnostic override: GPK_CHUNK=<multiple of 128>
        if os.environ.get("GPK_CHUNK"):
            self.set_option("chunk", int(os.environ["GPK_CHUNK"]))
        # schedule and contraction switches: GPK_OZAKI=0|1 (fp64 | int8 variance contraction), GPK_DEPTH2,
        # GPK_OZPERSIST, GPK_OZCLUSTER, GPK_OZGRID (see gpk_set_option in include/gpk.h)
        for env, key in (("GPK_OZAKI", "ozaki"), ("GPK_DEPTH2", "depth2"), ("GPK_OZPERSIST", "ozpersist"),
                         ("GPK_OZCLUSTER", "ozcluster"), ("GPK_OZGRID", "ozgrid")):
            if os.environ.get(env):
                self.set_option(key, int(os.environ[env]))

    # -- plumbing -----------------------------------------------------------------
    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self.lib.gpk_destroy(h)
            except Exception:
                pass

    def __del__(self):
        self.close()

    def _check(self, rc):
        if rc == GPK_OK:
            return
        msg = self.lib.gpk_last_error(self._h)
        msg = msg.decode("utf-8", "replace") if msg else ""
        if rc == GPK_NOT_PD:
            raise np.linalg.LinAlgError(msg or "Matrix is not positive definite")
        if rc == GPK_BAD_ARG:
            raise ValueError(msg)
        if rc == GPK_NOT_FITTED:
            raise RuntimeError(msg or "model not fitted")
        if rc == GPK_EP_FAILED:
            raise Exception(msg)
        raise RuntimeError("gpk: " + msg)

    def set_option(self, key, value):
        self._check(self.lib.gpk_set_option(self._h, key.encode(), int(value)))

    def set_stream(self, cuda_stream_ptr):
        self._check(self.lib.gpk_set_stream(self._h, _vp(cuda_stream_ptr or 0)))

    def synchronize(self):
        self._check(self.lib.gpk_synchronize(self._h))

    # -- model state ----------------------------------------------------------------
    def set_data(self, X, y):
        X, y = f64(X), f64(y)
        n, d = X.shape
        self._check(self.lib.gpk_set_data(self._h, _as_dp(X), _as_dp(y), n, d))

    def set_input_bounds(self, lower, upper):
        if lower is None or upper is None:
            self._check(self.lib.gpk_set_input_bounds(self._h, None, None, 0))
            return
        lo, up = f64(lower).ravel(), f64(upper).ravel()
        self._check(self.lib.gpk_set_input_bounds(self._h, _as_dp(lo), _as_dp(up), lo.size))

    def set_output_transform(self, enabled, y_mean=0.0, y_std=1.0):
        self._check(self.lib.gpk_set_output_transform(self._h, int(bool(enabled)), float(y_mean), float(y_std)))

    def set_kernel(self, family, log_amp, axis, group, log_metric):
        axis = np.ascontiguousarray(axis, dtype=np.int32)
        group = np.ascontiguousarray(group, dtype=np.int32)
        lm = f64(log_metric)
        self._check(self.lib.gpk_set_kernel(self._h, int(family), float(log_amp), axis.size,
                                            axis.ctypes.data_as(_ip), group.ctypes.data_as(_ip), _as_dp(lm)))

    def set_env_factor(self, axis, log_a=0.0, log_b=0.0):
        """gpk_set_env_factor: multiply the kernel by exp(log_a) + exp(log_b) z z' on column axis (-1: remove)."""
        self._check(self.lib.gpk_set_env_factor(self._h, int(axis), float(log_a), float(log_b)))

    def set_task_factor(self, axis, n_tasks=1, theta=None):
        """gpk_set_task_factor: multiply the kernel by K_t[t, t'] = (L L^T)[t, t'] on column axis, L_pq =
        exp(theta[p (p + 1) / 2 + q]) (-1: remove)."""
        th = None
        if int(axis) >= 0:
            th = np.ascontiguousarray(np.asarray(theta, dtype=np.float64).ravel())
            if th.size != int(n_tasks) * (int(n_tasks) + 1) // 2:
                raise ValueError("set_task_factor: need n_tasks (n_tasks + 1) / 2 entries")
        self._check(self.lib.gpk_set_task_factor(self._h, int(axis), int(n_tasks), _as_dp(th) if th is not None else None))

    def fit(self, diag_add, mean):
        logdet, ll = C.c_double(), C.c_double()
        self._check(self.lib.gpk_fit(self._h, float(diag_add), float(mean), C.byref(logdet), C.byref(ll)))
        return logdet.value, ll.value

    def fit_append(self, X, y, diag_add, mean):
        """Incremental refit after rows were appended (gpk_fit_append).  Returns (logdet, loglik), or None when the
        library reports that the shortcut does not apply (the model is untouched: run set_data + fit)."""
        X, y = f64(X), f64(y)
        n, d = X.shape
        logdet, ll = C.c_double(), C.c_double()
        rc = self.lib.gpk_fit_append(self._h, _as_dp(X), _as_dp(y), n, d, float(diag_add), float(mean),
                                     C.byref(logdet), C.byref(ll))
        if rc == GPK_NOT_APPLICABLE:
            return None
        self._check(rc)
        return logdet.value, ll.value

    def fit_begin(self, diag_add, mean):
        self._check(self.lib.gpk_fit_begin(self._h, float(diag_add), float(mean)))

    def fit_end(self):
        logdet, ll = C.c_double(), C.c_double()
        self._check(self.lib.gpk_fit_end(self._h, C.byref(logdet), C.byref(ll)))
        return logdet.value, ll.value

    # -- scoring ----------------------------------------------------------------------
    def predict(self, Xs):
        Xs = f64(Xs)
        m = Xs.shape[0]
        mu, var = np.empty(m), np.empty(m)
        self._check(self.lib.gpk_predict(self._h, _as_dp(Xs), m, _as_dp(mu), _as_dp(var)))
        return mu, var

    def predict_cov(self, Xs):
        Xs = f64(Xs)
        m = Xs.shape[0]
        mu, cov = np.empty(m), np.empty((m, m))
        self._check(self.lib.gpk_predict_cov(self._h, _as_dp(Xs), m, _as_dp(mu), _as_dp(cov)))
        return mu, cov

    def posterior_cov(self, Xs):
        """(mu, cov) with the raw, unclipped posterior covariance (sampling; gpk_posterior_cov)."""
        Xs = f64(Xs)
        m = Xs.shape[0]
        mu, cov = np.empty(m), np.empty((m, m))
        self._check(self.lib.gpk_posterior_cov(self._h, _as_dp(Xs), m, _as_dp(mu), _as_dp(cov)))
        return mu, cov

    def acq(self, Xs, kind, eta=0.0, par=0.0, want_values=True, want_moments=False):
        """-> dict(values, mu, var, best_val, best_idx, n_negative)"""
        Xs = f64(Xs)
        m = Xs.shape[0]
        out = np.empty(m) if want_values else None
        mu = np.empty(m) if want_moments else None
        var = np.empty(m) if want_moments else None
        bv, bi, nn = C.c_double(), C.c_long(-1), C.c_long(0)
        self._check(self.lib.gpk_acq(self._h, _as_dp(Xs), m, int(kind), float(eta), float(par),
                                     _as_dp(out) if want_values else None,
                                     _as_dp(mu) if want_moments else None,
                                     _as_dp(var) if want_moments else None,
                                     C.byref(bv), C.byref(bi), C.byref(nn)))
        return dict(values=out, mu=mu, var=var, best_val=bv.value, best_idx=bi.value, n_negative=nn.value)

    def acq_dev(self, d_Xs_ptr, m, kind, eta, par, d_out_ptr=0, d_mu_ptr=0, d_var_ptr=0, d_best_ptr=0):
        """Device-pointer variant (asynchronous on the handle's stream)."""
        self._check(self.lib.gpk_acq_dev(self._h, _vp(d_Xs_ptr), int(m), int(kind), float(eta), float(par),
                                         _vp(d_out_ptr or 0), _vp(d_mu_ptr or 0), _vp(d_var_ptr or 0),
                                         _vp(d_best_ptr or 0)))

    def predict_grad(self, Xs, kind=ACQ_NONE, eta=0.0, par=0.0):
        """-> dict(mu, var, dmu (m,d), dvar (m,d)[, f, df]) — moments and their input gradients."""
        Xs = f64(Xs)
        m, d = Xs.shape
        mu, var, dmu, dvar = np.empty(m), np.empty(m), np.empty((m, d)), np.empty((m, d))
        f = np.empty(m) if kind != ACQ_NONE else None
        df = np.empty((m, d)) if kind != ACQ_NONE else None
        self._check(self.lib.gpk_predict_grad(self._h, _as_dp(Xs), m, int(kind), float(eta), float(par), _as_dp(mu),
                                              _as_dp(var), _as_dp(dmu), _as_dp(dvar),
                                              _as_dp(f) if f is not None else None,
                                              _as_dp(df) if df is not None else None))
        return dict(mu=mu, var=var, dmu=dmu, dvar=dvar, f=f, df=df)

    def maximize_random(self, seed, first, count, n_uniform, lower, upper, incumbent, scale, kind, eta=0.0, par=0.0):
        """-> (best_x (d,), best_val, best_global_idx) over device-generated candidates [first, first+count)."""
        lo, up, inc = f64(lower).ravel(), f64(upper).ravel(), f64(incumbent).ravel()
        bx = np.empty(lo.size)
        bv, bi = C.c_double(), C.c_long(-1)
        self._check(self.lib.gpk_maximize_random(self._h, int(seed), int(first), int(count), int(n_uniform), _as_dp(lo),
                                                 _as_dp(up), _as_dp(inc), float(scale), int(kind), float(eta), float(par),
                                                 _as_dp(bx), C.byref(bv), C.byref(bi)))
        return bx, bv.value, bi.value

    def generate_candidates(self, seed, first, count, n_uniform, lower, upper, incumbent, scale):
        lo, up, inc = f64(lower).ravel(), f64(upper).ravel(), f64(incumbent).ravel()
        out = np.empty((count, lo.size))
        self._check(self.lib.gpk_generate_candidates(self._h, int(seed), int(first), int(count), int(n_uniform), lo.size,
                                                     _as_dp(lo), _as_dp(up), _as_dp(inc), float(scale), _as_dp(out)))
        return out

    # -- multi-GPU (gpk_comm_*) -----------------------------------------------------------
    def comm_init(self, rank, world, unique_id=None):
        """Collective over all ranks.  unique_id: the 128 bytes of comm_unique_id() made on rank 0."""
        buf = C.create_string_buffer(bytes(unique_id), 128) if unique_id is not None else None
        self._check(self.lib.gpk_comm_init(self._h, int(rank), int(world), C.cast(buf, _vp) if buf is not None else None))

    def comm_destroy(self):
        self._check(self.lib.gpk_comm_destroy(self._h))

    def comm_info(self):
        r, w, v = C.c_int(), C.c_int(), C.c_int()
        self._check(self.lib.gpk_comm_info(self._h, C.byref(r), C.byref(w), C.byref(v)))
        return dict(rank=r.value, world=w.value, nccl_version=v.value)

    def comm_argmax_pair(self, val, idx):
        """Exchange only: this rank's (value, global index) -> the merged winner on every rank."""
        bv, bi = C.c_double(), C.c_long(-1)
        self._check(self.lib.gpk_comm_argmax_pair(self._h, float(val), int(idx), C.byref(bv), C.byref(bi)))
        return bv.value, bi.value

    def acq_argmax_sharded(self, Xs_all, kind, eta=0.0, par=0.0):
        """Xs_all: the full batch, identical on every rank -> (best value, best GLOBAL index) on every rank."""
        Xs_all = f64(Xs_all)
        bv, bi = C.c_double(), C.c_long(-1)
        self._check(self.lib.gpk_acq_argmax_sharded(self._h, _as_dp(Xs_all), Xs_all.shape[0], int(kind), float(eta),
                                                    float(par), C.byref(bv), C.byref(bi)))
        return bv.value, bi.value

    def acq_argmax_sharded_dev(self, d_Xs_ptr, m_shard, first_global, kind, eta, par, d_best_ptr=0):
        self._check(self.lib.gpk_acq_argmax_sharded_dev(self._h, _vp(d_Xs_ptr or 0), int(m_shard), int(first_global),
                                                        int(kind), float(eta), float(par), _vp(d_best_ptr or 0)))

    def maximize_random_sharded(self, seed, n_total, n_uniform, lower, upper, incumbent, scale, kind, eta=0.0, par=0.0):
        lo, up, inc = f64(lower).ravel(), f64(upper).ravel(), f64(incumbent).ravel()
        bx = np.empty(lo.size)
        bv, bi = C.c_double(), C.c_long(-1)
        self._check(self.lib.gpk_maximize_random_sharded(self._h, int(seed), int(n_total), int(n_uniform), _as_dp(lo),
                                                         _as_dp(up), _as_dp(inc), float(scale), int(kind), float(eta),
                                                         float(par), _as_dp(bx), C.byref(bv), C.byref(bi)))
        return bx, bv.value, bi.value

    def acq_moments(self, mu, var, kind, eta=0.0, par=0.0):
        mu, var = f64(mu).ravel(), f64(var).ravel()
        out = np.empty(mu.size)
        nn = C.c_long(0)
        self._check(self.lib.gpk_acq_moments(self._h, _as_dp(mu), _as_dp(var), mu.size, int(kind), float(eta),
                                             float(par), _as_dp(out), C.byref(nn)))
        return out, nn.value

    def nll_grad(self, noise_var, n_terms, env=False, n_kt=0):
        """d(-loglik)/d[log_amp, log_metric_t..., (log_a, log_b with the environment factor, or the n_kt task entries
        with the task factor,) log sigma^2] of the current fit."""
        g = np.empty(n_terms + (4 if env else 2) + int(n_kt))
        self._check(self.lib.gpk_nll_grad(self._h, float(noise_var), _as_dp(g)))
        return g

    def reduce_models(self, A, B=None):
        """mean over models (B None) or GP-MCMC mixture moments (mean, var) (B = per-model variances)."""
        A = f64(A)
        n, m = A.shape
        out1 = np.empty(m)
        if B is None:
            self._check(self.lib.gpk_reduce_models(self._h, _as_dp(A), None, n, m, 0, _as_dp(out1), None))
            return out1
        B = f64(B)
        out2 = np.empty(m)
        self._check(self.lib.gpk_reduce_models(self._h, _as_dp(A), _as_dp(B), n, m, 1, _as_dp(out1), _as_dp(out2)))
        return out1, out2

    def kernel_matrix(self, X1, X2):
        X1, X2 = f64(X1), f64(X2)
        out = np.empty((X1.shape[0], X2.shape[0]))
        self._check(self.lib.gpk_kernel_matrix(self._h, _as_dp(X1), X1.shape[0], _as_dp(X2), X2.shape[0],
                                               X1.shape[1], _as_dp(out)))
        return out

    def measure_fp64_peaks(self):
        """-> (DMMA tensor-pipe TFLOP/s, DFMA vector-pipe TFLOP/s) measured on this GPU."""
        a, b = C.c_double(), C.c_double()
        self._check(self.lib.gpk_measure_fp64_peaks(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def measure_int8_peak(self):
        """-> int8 tensor-pipe issue-rate peak in TOP/s (wgmma s8) measured on this GPU."""
        a = C.c_double()
        self._check(self.lib.gpk_measure_int8_peak(self._h, C.byref(a)))
        return a.value

    def measure_int8_peak_sustained(self, seconds=0.4, random_operands=True):
        """-> the same issue rate held for `seconds` (second half timed): what the power limit leaves of the burst figure.
        random_operands: pseudo-random operand bytes (switching activity of real digit slices) instead of a constant pattern."""
        a = C.c_double()
        self._check(self.lib.gpk_measure_int8_peak_sustained(self._h, float(seconds), 1 if random_operands else 0, C.byref(a)))
        return a.value

    # -- introspection ----------------------------------------------------------------
    def get_factor(self, n):
        L = np.empty((n, n))
        self._check(self.lib.gpk_get_factor(self._h, _as_dp(L)))
        return L

    def get_linv(self, n):
        L = np.empty((n, n))
        self._check(self.lib.gpk_get_linv(self._h, _as_dp(L)))
        return L

    def get_z(self, n):
        z = np.empty(n)
        self._check(self.lib.gpk_get_z(self._h, _as_dp(z)))
        return z

    def oz_contract(self, P, Ks, amp):
        """The int8 variance contraction alone (gpk_oz_contract) on P (n x n, lower triangular) and Ks (m x n,
        |entries| <= amp) -> dict(part_ssq (nb x m), eP (n,) int32, eK)."""
        P, Ks = f64(P), f64(Ks)
        n = P.shape[0]
        if P.ndim != 2 or P.shape[1] != n or Ks.ndim != 2 or Ks.shape[1] != n:
            raise ValueError("oz_contract: P must be n x n and Ks m x n")
        m = Ks.shape[0]
        part = np.empty(((n + 127) // 128, m))
        eP = np.empty(n, dtype=np.int32)
        eK = C.c_int()
        self._check(self.lib.gpk_oz_contract(self._h, _as_dp(P), n, _as_dp(Ks), m, float(amp), _as_dp(part),
                                             eP.ctypes.data_as(_ip), C.byref(eK)))
        return dict(part_ssq=part, eP=eP, eK=eK.value)

    def ep_joint_min(self, mu, V, derivatives=True):
        """EPMGP p_min on caller operands (gpk_ep_joint_min) -> dict(logP (nb,)[, dlogPdMu (nb, nb), dlogPdSigma
        (nb, nb (nb + 1) / 2), dlogPdMudMu (nb, nb, nb), sweeps (nb,) int32])."""
        mu, V = f64(mu).ravel(), f64(V)
        nb = mu.size
        if V.shape != (nb, nb):
            raise ValueError("ep_joint_min: V must be %d x %d" % (nb, nb))
        logP = np.empty(nb)
        if not derivatives or not 2 <= nb <= 64:          # nb is checked by the library before any buffer is used
            self._check(self.lib.gpk_ep_joint_min(self._h, _as_dp(mu), _as_dp(V), nb, _as_dp(logP), None, None, None, None))
            return dict(logP=logP)
        dMu, dSig, dMuMu = np.empty((nb, nb)), np.empty((nb, nb * (nb + 1) // 2)), np.empty((nb, nb, nb))
        sweeps = np.empty(nb, dtype=np.int32)
        self._check(self.lib.gpk_ep_joint_min(self._h, _as_dp(mu), _as_dp(V), nb, _as_dp(logP), _as_dp(dMu), _as_dp(dSig),
                                              _as_dp(dMuMu), sweeps.ctypes.data_as(_ip)))
        return dict(logP=logP, dlogPdMu=dMu, dlogPdSigma=dSig, dlogPdMudMu=dMuMu, sweeps=sweeps)

    def es_update(self, zb, lmb, sn2, W, lower, upper):
        """gpk_es_update -> dict(logP (nb,), dlogPdMu, dlogPdSigma, dlogPdMudMu)."""
        zb, lmb, W = f64(zb), f64(lmb).ravel(), f64(W).ravel()
        lo, up = f64(lower).ravel(), f64(upper).ravel()
        nb = zb.shape[0]
        if lmb.size != nb:
            raise ValueError("es_update: lmb needs one value per representer point")
        if not 2 <= nb <= 64:
            self._check(self.lib.gpk_es_update(self._h, _as_dp(zb), nb, _as_dp(lmb), float(sn2), _as_dp(W), W.size,
                                               _as_dp(lo), _as_dp(up), None, None, None, None))
        logP = np.empty(nb)
        dMu, dSig, dMuMu = np.empty((nb, nb)), np.empty((nb, nb * (nb + 1) // 2)), np.empty((nb, nb, nb))
        self._check(self.lib.gpk_es_update(self._h, _as_dp(zb), nb, _as_dp(lmb), float(sn2), _as_dp(W), W.size,
                                           _as_dp(lo), _as_dp(up), _as_dp(logP), _as_dp(dMu), _as_dp(dSig),
                                           _as_dp(dMuMu)))
        return dict(logP=logP, dlogPdMu=dMu, dlogPdSigma=dSig, dlogPdMudMu=dMuMu)

    def es_compute(self, Xs):
        """gpk_es_compute: the entropy change of every row of Xs (m, d) -> (m,)."""
        Xs = f64(Xs)
        out = np.empty(Xs.shape[0])
        self._check(self.lib.gpk_es_compute(self._h, _as_dp(Xs), Xs.shape[0], _as_dp(out)))
        return out

    def es_compute_dev(self, d_Xs_ptr, m, d_out_ptr):
        self._check(self.lib.gpk_es_compute_dev(self._h, _vp(d_Xs_ptr), int(m), _vp(d_out_ptr)))

    def es_dims(self):
        """gpk_es_dims: (n, nb) of the last es_update."""
        n, nb = C.c_int(), C.c_int()
        self._check(self.lib.gpk_es_dims(self._h, C.byref(n), C.byref(nb)))
        return n.value, nb.value

    def es_moments(self, Xs):
        """gpk_es_moments (diagnostic): what gpk_es_compute's dH kernel reads for the rows of Xs (m, d) -> (var (m,),
        sigma (m, nb))."""
        Xs = f64(Xs)
        m = Xs.shape[0]
        _, nb = self.es_dims()
        var, sigma = np.empty(m), np.empty((m, nb))
        self._check(self.lib.gpk_es_moments(self._h, _as_dp(Xs), m, _as_dp(var), _as_dp(sigma)))
        return var, sigma

    def es_get_u(self):
        """gpk_es_get_u (diagnostic): U = K^-1 K(X, zb) of the last es_update -> (n, nb)."""
        U = np.empty(self.es_dims())
        self._check(self.lib.gpk_es_get_u(self._h, _as_dp(U)))
        return U

    # -- sampling-based entropy search (gpk_esmc.cuh) --------------------------------------------------------------
    def mc_pmin(self, m, V, nf, seed):
        """gpk_mc_pmin: joint_pmin on caller operands, m (nb,) or (nb, np), V (nb, nb) -> (pmin (nb,), n_jitter)."""
        m, V = f64(m), f64(V)
        if m.ndim == 1:
            m = m[:, None]
        nb, np_ = m.shape
        if V.shape != (nb, nb):
            raise ValueError("mc_pmin: V must be %d x %d" % (nb, nb))
        pmin, nj = np.empty(nb), C.c_int(0)
        self._check(self.lib.gpk_mc_pmin(self._h, _as_dp(m), np_, _as_dp(V), nb, int(nf),
                                         int(seed) & 0xFFFFFFFFFFFFFFFF, _as_dp(pmin), C.byref(nj)))
        return pmin, nj.value

    def mc_draws(self, seed, nb, nf):
        """gpk_mc_draws: the draws F (nb, nf) a seed gives."""
        F = np.empty((int(nb), int(nf)))
        self._check(self.lib.gpk_mc_draws(self._h, int(seed) & 0xFFFFFFFFFFFFFFFF, int(nb), int(nf), _as_dp(F)))
        return F

    def esmc_update(self, zb, lmb, sn2, W, nf, seed):
        """gpk_esmc_update -> dict(logP (nb,), pmin (nb,), n_jitter)."""
        zb, lmb, W = f64(zb), f64(lmb).ravel(), f64(W).ravel()
        nb = zb.shape[0]
        if lmb.size != nb:
            raise ValueError("esmc_update: lmb needs one value per representer point")
        logP, pmin = np.empty(nb), np.empty(nb)
        self._check(self.lib.gpk_esmc_update(self._h, _as_dp(zb), nb, _as_dp(lmb), float(sn2), _as_dp(W), W.size,
                                             int(nf), int(seed) & 0xFFFFFFFFFFFFFFFF, _as_dp(logP), _as_dp(pmin)))
        self._esmc_nf = int(nf)
        return dict(logP=logP, pmin=pmin, n_jitter=self.esmc_last_jitter())

    def esmc_compute(self, Xs):
        """gpk_esmc_compute: the sampling-based entropy change of every row of Xs (m, d) -> (m,)."""
        Xs = f64(Xs)
        out = np.empty(Xs.shape[0])
        self._check(self.lib.gpk_esmc_compute(self._h, _as_dp(Xs), Xs.shape[0], _as_dp(out)))
        return out

    def esmc_compute_dev(self, d_Xs_ptr, m, d_out_ptr):
        self._check(self.lib.gpk_esmc_compute_dev(self._h, _vp(d_Xs_ptr), int(m), _vp(d_out_ptr)))

    def esmc_get_draws(self):
        """gpk_esmc_get_draws (diagnostic): the current update's F (nb, nf)."""
        F = np.empty((self.es_dims()[1], self._esmc_nf))
        self._check(self.lib.gpk_esmc_get_draws(self._h, _as_dp(F)))
        return F

    def esmc_get_state(self):
        """gpk_esmc_get_state (diagnostic): the current update's (Mb (nb,), Vb (nb, nb))."""
        nb = self.es_dims()[1]
        Mb, Vb = np.empty(nb), np.empty((nb, nb))
        self._check(self.lib.gpk_esmc_get_state(self._h, _as_dp(Mb), _as_dp(Vb)))
        return Mb, Vb

    def esmc_last_jitter(self):
        """gpk_esmc_last_jitter: factorisations that needed jitter in the last synchronised p_min call."""
        n = C.c_long(0)
        self._check(self.lib.gpk_esmc_last_jitter(self._h, C.byref(n)))
        return n.value

    def predict_mean(self, Xs):
        """gpk_predict_mean: the predictive mean alone of every row of Xs (m, d) -> (m,)."""
        Xs = f64(Xs)
        mu = np.empty(Xs.shape[0])
        self._check(self.lib.gpk_predict_mean(self._h, _as_dp(Xs), Xs.shape[0], _as_dp(mu)))
        return mu

    def predict_mean_dev(self, d_Xs_ptr, m, d_mu_ptr):
        self._check(self.lib.gpk_predict_mean_dev(self._h, _vp(d_Xs_ptr), int(m), _vp(d_mu_ptr)))

    def diag_profile(self):
        t = np.zeros(64, dtype=np.int64)
        self._check(self.lib.gpk_get_diag_profile(self._h, t.ctypes.data_as(C.POINTER(C.c_longlong))))
        return t

    def timings(self):
        t = np.zeros(16)
        self._check(self.lib.gpk_get_timings(self._h, _as_dp(t)))
        keys = ["fit_ms", "kbuild_ms", "potrf_ms", "linv_ms", "score_ms", "kstar_ms", "vargemm_ms", "finish_ms",
                "launches_vargemm", "launches_total", "launches_ozaki", "ozaki_max_row_exponent", "reserved",
                "ozaki_slice_pairs", "ozaki_kernel_variant"]
        return dict(zip(keys, t.tolist()))


def comm_unique_id():
    """128-byte NCCL id (rank 0 makes it and ships it to the other ranks by any means: file, pipe, MPI, a
    torch.distributed store ...)."""
    lib = load()
    buf = C.create_string_buffer(128)
    if lib.gpk_comm_unique_id(C.cast(buf, _vp)) != GPK_OK:
        raise RuntimeError("gpk_comm_unique_id failed: NCCL (libnccl.so.2) is not available")
    return buf.raw


def shard_bounds(m, rank, world):
    lib = load()
    lo, hi = C.c_long(), C.c_long()
    if lib.gpk_shard_bounds(int(m), int(rank), int(world), C.byref(lo), C.byref(hi)) != GPK_OK:
        raise ValueError("shard_bounds: bad arguments")
    return lo.value, hi.value


def _handles(handles):
    """The C array of the handles' pointers, the first argument of every entry point over several models."""
    return (_vp * len(handles))(*[h._h for h in handles])


def _etas(eta, n):
    """eta (a scalar or one value per model; None: zeros) as n contiguous doubles."""
    return f64(np.zeros(n) if eta is None else np.broadcast_to(np.asarray(eta, dtype=np.float64), (n,)))


def acq_multi(handles, Xs, mode, kind=ACQ_NONE, eta=None, par=0.0, want_argmax=False):
    """gpk_acq_multi over ``handles`` (all fitted, same device).  mode 0 -> dict(values, n_negative, best_val,
    best_idx); mode 1 -> dict(mean, var)."""
    h0 = handles[0]
    Xs = f64(Xs)
    m = Xs.shape[0]
    arr = _handles(handles)
    out1 = np.empty(m)
    out2 = np.empty(m) if mode == 1 else None
    etas = _etas(eta, len(handles))
    nn, bv, bi = C.c_long(0), C.c_double(), C.c_long(-1)
    h0._check(h0.lib.gpk_acq_multi(arr, len(handles), _as_dp(Xs), m, int(mode), int(kind), _as_dp(etas), float(par),
                                   _as_dp(out1), _as_dp(out2) if out2 is not None else None, C.byref(nn),
                                   C.byref(bv) if want_argmax else None, C.byref(bi) if want_argmax else None))
    if mode == 1:
        return dict(mean=out1, var=out2)
    return dict(values=out1, n_negative=nn.value, best_val=bv.value, best_idx=bi.value)


def maximize_de(handles, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper, kind, eta, par=0.0,
                want_population=False):
    """gpk_maximize_de over ``handles`` (all fitted, same device): differential evolution minimising -acq, acq the
    mean over the handles.  -> dict(x (D,), energy, nit, nfev, n_negative[, population (pop, D), energies (pop,)])."""
    h0 = handles[0]
    lo, up = f64(lower).ravel(), f64(upper).ravel()
    arr = _handles(handles)
    etas = _etas(eta, len(handles))
    x = np.empty(lo.size)
    pop = int(pop)
    P = np.empty((pop, lo.size)) if want_population and pop > 0 else None
    E = np.empty(pop) if want_population and pop > 0 else None
    be, nit, nfev, nn = C.c_double(), C.c_int(), C.c_long(), C.c_long()
    h0._check(h0.lib.gpk_maximize_de(arr, len(handles), int(seed) & 0xFFFFFFFFFFFFFFFF, pop, int(maxiter),
                                     float(mutation[0]), float(mutation[1]), float(recombination), float(tol),
                                     float(atol), _as_dp(lo), _as_dp(up), int(kind), _as_dp(etas), float(par),
                                     _as_dp(x), C.byref(be), C.byref(nit), C.byref(nfev), C.byref(nn),
                                     _as_dp(P) if P is not None else None, _as_dp(E) if E is not None else None))
    r = _de_result(x, be, nit, nfev, P, E, want_population)
    r["n_negative"] = nn.value
    return r


def _es_cost_args(objective, cost, lower, upper):
    if len(objective) == 0 or len(objective) != len(cost):
        raise ValueError("information gain per unit cost: need as many cost handles as objective handles (>= 1)")
    ho = _handles(objective)
    hc = _handles(cost)
    lo, up = f64(lower).ravel(), f64(upper).ravel()
    if lo.size != up.size:
        raise ValueError("information gain per unit cost: lower and upper differ in length")
    return ho, hc, lo, up


def es_cost_multi(objective, cost, Xs, lower, upper, basis_objective, basis_cost, overhead, want_values=True):
    """gpk_es_cost_multi over the (objective[i], cost[i]) pairs: raw candidates Xs (m, d), configuration bounds
    lower / upper (d - 1) -> dict(values (m,) or None, best_val, best_idx)."""
    ho, hc, lo, up = _es_cost_args(objective, cost, lower, upper)
    h0 = objective[0]
    Xs = f64(Xs)
    m = Xs.shape[0]
    out = np.empty(m) if want_values else None
    bv, bi = C.c_double(), C.c_long(-1)
    h0._check(h0.lib.gpk_es_cost_multi(ho, hc, len(objective), _as_dp(Xs), m, _as_dp(lo), _as_dp(up), lo.size,
                                       int(basis_objective), int(basis_cost), float(overhead),
                                       _as_dp(out) if want_values else None, C.byref(bv), C.byref(bi)))
    return dict(values=out, best_val=bv.value, best_idx=bi.value)


def es_cost_multi_dev(objective, cost, d_Xs_ptr, m, lower, upper, basis_objective, basis_cost, overhead, d_out_ptr,
                      d_best_ptr=0):
    """Device-batch variant, asynchronous on objective[0]'s stream."""
    ho, hc, lo, up = _es_cost_args(objective, cost, lower, upper)
    h0 = objective[0]
    h0._check(h0.lib.gpk_es_cost_multi_dev(ho, hc, len(objective), _vp(d_Xs_ptr), int(m), _as_dp(lo), _as_dp(up),
                                           lo.size, int(basis_objective), int(basis_cost), float(overhead), _vp(d_out_ptr or 0),
                                           _vp(d_best_ptr or 0)))


def maximize_random_es_cost(objective, cost, seed, count, n_uniform, box_lower, box_upper, incumbent, scale, lower,
                            upper, basis_objective, basis_cost, overhead):
    """gpk_maximize_random_es_cost -> (best_x (d,), best_val, best_idx)."""
    ho, hc, lo, up = _es_cost_args(objective, cost, lower, upper)
    h0 = objective[0]
    blo, bup, inc = f64(box_lower).ravel(), f64(box_upper).ravel(), f64(incumbent).ravel()
    if not blo.size == bup.size == inc.size == lo.size + 1:
        raise ValueError("maximize_random_es_cost: the box and the incumbent need d entries, the configuration bounds d - 1")
    bx = np.empty(blo.size)
    bv, bi = C.c_double(), C.c_long(-1)
    h0._check(h0.lib.gpk_maximize_random_es_cost(ho, hc, len(objective), int(seed) & 0xFFFFFFFFFFFFFFFF, int(count),
                                                 int(n_uniform), _as_dp(blo), _as_dp(bup), _as_dp(inc), float(scale),
                                                 _as_dp(lo), _as_dp(up), lo.size, int(basis_objective), int(basis_cost),
                                                 float(overhead), _as_dp(bx), C.byref(bv), C.byref(bi)))
    return bx, bv.value, bi.value


def es_multi(objective, Xs, want_values=True):
    """gpk_es_multi: the entropy change of every row of Xs (m, d) under each handle, averaged over the handles ->
    dict(values (m,) or None, best_val, best_idx)."""
    h0 = objective[0]
    ho = _handles(objective)
    Xs = f64(Xs)
    m = Xs.shape[0]
    out = np.empty(m) if want_values else None
    bv, bi = C.c_double(), C.c_long(-1)
    h0._check(h0.lib.gpk_es_multi(ho, len(objective), _as_dp(Xs), m, _as_dp(out) if want_values else None,
                                  C.byref(bv), C.byref(bi)))
    return dict(values=out, best_val=bv.value, best_idx=bi.value)


def es_multi_dev(objective, d_Xs_ptr, m, d_out_ptr, d_best_ptr=0):
    """Device-batch variant, asynchronous on objective[0]'s stream."""
    h0 = objective[0]
    ho = _handles(objective)
    h0._check(h0.lib.gpk_es_multi_dev(ho, len(objective), _vp(d_Xs_ptr), int(m), _vp(d_out_ptr or 0),
                                      _vp(d_best_ptr or 0)))


def esmc_multi(objective, Xs, want_values=True):
    """gpk_esmc_multi: the sampling-based entropy change of every row of Xs (m, d) under each handle, averaged over the
    handles -> dict(values (m,) or None, best_val, best_idx)."""
    h0 = objective[0]
    ho = _handles(objective)
    Xs = f64(Xs)
    m = Xs.shape[0]
    out = np.empty(m) if want_values else None
    bv, bi = C.c_double(), C.c_long(-1)
    h0._check(h0.lib.gpk_esmc_multi(ho, len(objective), _as_dp(Xs), m, _as_dp(out) if want_values else None,
                                    C.byref(bv), C.byref(bi)))
    return dict(values=out, best_val=bv.value, best_idx=bi.value)


def esmc_multi_dev(objective, d_Xs_ptr, m, d_out_ptr, d_best_ptr=0):
    """Device-batch variant, asynchronous on objective[0]'s stream."""
    h0 = objective[0]
    h0._check(h0.lib.gpk_esmc_multi_dev(_handles(objective), len(objective), _vp(d_Xs_ptr), int(m), _vp(d_out_ptr or 0),
                                        _vp(d_best_ptr or 0)))


def _de_result(x, be, nit, nfev, P, E, want_population):
    r = dict(x=x, energy=be.value, nit=nit.value, nfev=nfev.value)
    if want_population:
        r.update(population=P, energies=E)
    return r


def maximize_de_es(objective, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper,
                   want_population=False):
    """gpk_maximize_de_es: differential evolution minimising minus the entropy change (one handle: gpk_es_compute's
    value; several: gpk_es_multi's mean) -> dict(x (D,), energy, nit, nfev[, population (pop, D), energies (pop,)])."""
    h0 = objective[0]
    ho = _handles(objective)
    lo, up = f64(lower).ravel(), f64(upper).ravel()
    x = np.empty(lo.size)
    pop = int(pop)
    P = np.empty((pop, lo.size)) if want_population and pop > 0 else None
    E = np.empty(pop) if want_population and pop > 0 else None
    be, nit, nfev = C.c_double(), C.c_int(), C.c_long()
    h0._check(h0.lib.gpk_maximize_de_es(ho, len(objective), int(seed) & 0xFFFFFFFFFFFFFFFF, pop, int(maxiter),
                                        float(mutation[0]), float(mutation[1]), float(recombination), float(tol),
                                        float(atol), _as_dp(lo), _as_dp(up), _as_dp(x), C.byref(be), C.byref(nit),
                                        C.byref(nfev), _as_dp(P) if P is not None else None,
                                        _as_dp(E) if E is not None else None))
    return _de_result(x, be, nit, nfev, P, E, want_population)


def maximize_de_esmc(objective, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper,
                     want_population=False):
    """gpk_maximize_de_esmc: differential evolution minimising minus the sampling-based entropy change (one handle:
    gpk_esmc_compute's value; several: gpk_esmc_multi's mean) -> as maximize_de_es."""
    h0 = objective[0]
    ho = _handles(objective)
    lo, up = f64(lower).ravel(), f64(upper).ravel()
    x = np.empty(lo.size)
    pop = int(pop)
    P = np.empty((pop, lo.size)) if want_population and pop > 0 else None
    E = np.empty(pop) if want_population and pop > 0 else None
    be, nit, nfev = C.c_double(), C.c_int(), C.c_long()
    h0._check(h0.lib.gpk_maximize_de_esmc(ho, len(objective), int(seed) & 0xFFFFFFFFFFFFFFFF, pop, int(maxiter),
                                          float(mutation[0]), float(mutation[1]), float(recombination), float(tol),
                                          float(atol), _as_dp(lo), _as_dp(up), _as_dp(x), C.byref(be), C.byref(nit),
                                          C.byref(nfev), _as_dp(P) if P is not None else None,
                                          _as_dp(E) if E is not None else None))
    return _de_result(x, be, nit, nfev, P, E, want_population)


def maximize_de_es_cost(objective, cost, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper,
                        cfg_lower, cfg_upper, basis_objective, basis_cost, overhead, want_population=False):
    """gpk_maximize_de_es_cost: differential evolution over the extended box lower / upper (d) minimising minus the
    information gain per unit cost of gpk_es_cost_multi (configuration bounds cfg_lower / cfg_upper, d - 1) -> as
    maximize_de_es."""
    ho, hc, clo, cup = _es_cost_args(objective, cost, cfg_lower, cfg_upper)
    h0 = objective[0]
    lo, up = f64(lower).ravel(), f64(upper).ravel()
    if not lo.size == up.size == clo.size + 1:
        raise ValueError("maximize_de_es_cost: the box needs d entries, the configuration bounds d - 1")
    x = np.empty(lo.size)
    pop = int(pop)
    P = np.empty((pop, lo.size)) if want_population and pop > 0 else None
    E = np.empty(pop) if want_population and pop > 0 else None
    be, nit, nfev = C.c_double(), C.c_int(), C.c_long()
    h0._check(h0.lib.gpk_maximize_de_es_cost(ho, hc, len(objective), int(seed) & 0xFFFFFFFFFFFFFFFF, pop, int(maxiter),
                                             float(mutation[0]), float(mutation[1]), float(recombination), float(tol),
                                             float(atol), _as_dp(lo), _as_dp(up), _as_dp(clo), _as_dp(cup), clo.size,
                                             int(basis_objective), int(basis_cost), float(overhead), _as_dp(x),
                                             C.byref(be), C.byref(nit), C.byref(nfev),
                                             _as_dp(P) if P is not None else None, _as_dp(E) if E is not None else None))
    return _de_result(x, be, nit, nfev, P, E, want_population)


LB_DEFAULTS = dict(maxcor=10, maxiter=15000, maxfun=15000, ftol=2.220446049250313e-09, pgtol=1e-5)   # scipy's


def _lb_io(x0, lower, upper):
    lo, up = f64(lower).ravel(), f64(upper).ravel()
    x0 = f64(np.atleast_2d(x0))
    if lo.size != up.size or x0.ndim != 2 or x0.shape[1] != lo.size:
        raise ValueError("maximize_lbfgs: x0 needs shape (n_starts, d) with d = len(lower) = len(upper)")
    R = x0.shape[0]
    outs = (np.empty((R, lo.size)), np.empty(R), np.empty(R, dtype=np.intc), np.empty(R, dtype=np.int_),
            np.empty(R, dtype=np.intc))
    return x0, lo, up, outs


def _lb_opts(kw):
    o = dict(LB_DEFAULTS, **kw)
    return int(o["maxcor"]), int(o["maxiter"]), int(o["maxfun"]), float(o["ftol"]), float(o["pgtol"])


def _lb_out_ptrs(outs):
    x, e, nit, nfev, st = outs
    return _as_dp(x), _as_dp(e), nit.ctypes.data_as(_ip), nfev.ctypes.data_as(_lp), st.ctypes.data_as(_ip)


def _lb_result(outs):
    x, e, nit, nfev, st = outs
    return dict(x=x, energy=e, nit=nit.astype(np.int64), nfev=nfev.astype(np.int64), status=st.astype(np.int64))


def maximize_lbfgs(handles, kind, eta, par, x0, lower, upper, **options):
    """gpk_maximize_lbfgs over ``handles`` (all fitted, same device): multi-start bounded L-BFGS from the rows of x0
    (n_starts, d) minimising -acq (kind ACQ_EI ... ACQ_LCB, acq the mean over the handles) or the posterior objective
    (OBJ_MEAN, OBJ_MEAN_STD; eta ignored).  options: maxcor, maxiter, maxfun, ftol, pgtol (scipy's defaults) ->
    dict(x (n_starts, d), energy, nit, nfev, status (n_starts each), n_negative)."""
    h0 = handles[0]
    x0, lo, up, outs = _lb_io(x0, lower, upper)
    arr = _handles(handles)
    etas = _etas(eta, len(handles))
    nn = C.c_long()
    h0._check(h0.lib.gpk_maximize_lbfgs(arr, len(handles), int(kind), _as_dp(etas), float(par), x0.shape[0], _as_dp(x0),
                                        _as_dp(lo), _as_dp(up), *_lb_opts(options), *_lb_out_ptrs(outs), C.byref(nn)))
    r = _lb_result(outs)
    r["n_negative"] = nn.value
    return r


def maximize_lbfgs_es(objective, x0, lower, upper, **options):
    """gpk_maximize_lbfgs_es: the same minimising minus the entropy change (one handle: gpk_es_compute's value;
    several: gpk_es_multi's mean) -> dict(x, energy, nit, nfev, status)."""
    h0 = objective[0]
    ho = _handles(objective)
    x0, lo, up, outs = _lb_io(x0, lower, upper)
    h0._check(h0.lib.gpk_maximize_lbfgs_es(ho, len(objective), x0.shape[0], _as_dp(x0), _as_dp(lo), _as_dp(up),
                                           *_lb_opts(options), *_lb_out_ptrs(outs)))
    return _lb_result(outs)


def maximize_lbfgs_es_cost(objective, cost, x0, lower, upper, cfg_lower, cfg_upper, basis_objective, basis_cost,
                           overhead, **options):
    """gpk_maximize_lbfgs_es_cost: the same over the extended box lower / upper (d) minimising minus the information
    gain per unit cost of gpk_es_cost_multi (configuration bounds cfg_lower / cfg_upper, d - 1) -> as
    maximize_lbfgs_es."""
    ho, hc, clo, cup = _es_cost_args(objective, cost, cfg_lower, cfg_upper)
    h0 = objective[0]
    x0, lo, up, outs = _lb_io(x0, lower, upper)
    if lo.size != clo.size + 1:
        raise ValueError("maximize_lbfgs_es_cost: the box needs d entries, the configuration bounds d - 1")
    h0._check(h0.lib.gpk_maximize_lbfgs_es_cost(ho, hc, len(objective), x0.shape[0], _as_dp(x0), _as_dp(lo),
                                                _as_dp(up), _as_dp(clo), _as_dp(cup), clo.size, int(basis_objective),
                                                int(basis_cost), float(overhead), *_lb_opts(options),
                                                *_lb_out_ptrs(outs)))
    return _lb_result(outs)


def cmaes_run_constants(d, lam):
    """The constants of one CMA-ES run of population lam in dimension d (Hansen's tutorial, Table 1, positive weights
    only; purecma's lazy eigendecomposition gap; cma's tolfun history length) as a dict.  gpk_maximize_cmaes* and
    tests/cmaes_model.py both take them from here, so no log runs on the device."""
    import math
    d, lam = int(d), int(lam)
    mu = lam // 2
    w = math.log((lam + 1) / 2.0) - np.log(np.arange(1, mu + 1, dtype=np.float64))
    w = w / np.sum(w)
    mueff = 1.0 / np.sum(w * w)
    cs = (mueff + 2.0) / (d + mueff + 5.0)
    ds = 1.0 + 2.0 * max(0.0, math.sqrt((mueff - 1.0) / (d + 1.0)) - 1.0) + cs
    cc = (4.0 + mueff / d) / (d + 4.0 + 2.0 * mueff / d)
    c1 = 2.0 / ((d + 1.3) ** 2 + mueff)
    cmu = min(1.0 - c1, 2.0 * (mueff - 2.0 + 1.0 / mueff) / ((d + 2.0) ** 2 + mueff))
    chi = math.sqrt(d) * (1.0 - 1.0 / (4.0 * d) + 1.0 / (21.0 * d * d))
    return dict(lam=lam, mu=mu, w=w, mueff=float(mueff), cs=cs, ds=ds, cc=cc, c1=c1, cmu=cmu, chi=chi,
                hist=10 + int(math.ceil(30.0 * d / lam)), eig_gap=lam / (c1 + cmu) / d / 10.0,
                flat=int(math.ceil(0.7 * lam)) - 1, omcs=1.0 - cs, cps=math.sqrt(cs * (2.0 - cs) * mueff),
                omcc=1.0 - cc, ccc=math.sqrt(cc * (2.0 - cc) * mueff), ccd=cc * (2.0 - cc), a0=1.0 - c1 - cmu,
                hth=(1.4 + 2.0 / (d + 1.0)) * chi, csds=cs / ds)


def cmaes_lambda(d, run=0):
    """The population of IPOP run ``run``: (4 + floor(3 ln d)) 2^run."""
    import math
    return (4 + int(3.0 * math.log(d))) << int(run)


def cmaes_constants(d, restarts):
    """The constant table of gpk_maximize_cmaes*: (restarts + 1, CMA_NCONST), one GPK_CMA_C_* row per run.  A run whose
    lambda exceeds CMA_MAX_LAMBDA keeps its lambda but no weights; the library refuses it."""
    keys = ("lam", "mu", "mueff", "cs", "ds", "cc", "c1", "cmu", "chi", "hist", "eig_gap", "flat", "omcs", "cps", "omcc",
            "ccc", "ccd", "a0", "hth", "csds")
    tab = np.zeros((int(restarts) + 1, CMA_NCONST))
    for r in range(int(restarts) + 1):
        c = cmaes_run_constants(d, cmaes_lambda(d, r))
        tab[r, :CMA_C_W] = [c[k] for k in keys]
        if c["mu"] <= CMA_MAX_LAMBDA // 2:
            tab[r, CMA_C_W:CMA_C_W + c["mu"]] = c["w"]
    return tab


class _CmaesResult(C.Structure):
    _fields_ = [(name, _vp) for name in ("best_x", "best_energy", "nfev_total", "nit", "nfev", "stop", "m", "sigma",
                                         "ps", "pc", "C")]


def _cmaes_io(x0, lower, upper, restarts):
    lo, up, x0 = f64(lower).ravel(), f64(upper).ravel(), f64(x0).ravel()
    if not lo.size == up.size == x0.size:
        raise ValueError("maximize_cmaes: x0, lower and upper need d entries each")
    d, runs = lo.size, int(restarts) + 1
    if runs < 1:
        raise ValueError("maximize_cmaes: need restarts >= 0")
    outs = dict(best_x=np.empty(d), best_energy=np.empty(1), nfev_total=np.zeros(1, dtype=np.int_),
                nit=np.zeros(runs, dtype=np.intc), nfev=np.zeros(runs, dtype=np.int_), stop=np.zeros(runs, dtype=np.intc),
                m=np.empty(d), sigma=np.empty(1), ps=np.empty(d), pc=np.empty(d), C=np.empty((d, d)))
    res = _CmaesResult(*[outs[k].ctypes.data for k, _ in _CmaesResult._fields_])
    return x0, lo, up, f64(cmaes_constants(d, restarts)), outs, res


def _cmaes_result(outs):
    return dict(x=outs["best_x"], energy=float(outs["best_energy"][0]), nfev_total=int(outs["nfev_total"][0]),
                nit=outs["nit"].astype(np.int64), nfev=outs["nfev"].astype(np.int64),
                stop=outs["stop"].astype(np.int64), m=outs["m"], sigma=float(outs["sigma"][0]), ps=outs["ps"],
                pc=outs["pc"], C=outs["C"])


def maximize_cmaes(handles, kind, eta, par, seed, x0, lower, upper, n_func_evals=1000, restarts=0, sigma0=0.6):
    """gpk_maximize_cmaes over ``handles`` (all fitted, same device): CMA-ES from x0 (d,) minimising -acq (kind ACQ_EI
    ... ACQ_LCB, acq the mean over the handles) -> dict(x (d,), energy, nfev_total, nit / nfev / stop per run, the last
    run's final m, sigma, ps, pc and C, n_negative)."""
    h0 = handles[0]
    x0, lo, up, tab, outs, res = _cmaes_io(x0, lower, upper, restarts)
    nn = C.c_long()
    h0._check(h0.lib.gpk_maximize_cmaes(_handles(handles), len(handles), int(kind), _as_dp(_etas(eta, len(handles))),
                                        float(par), int(seed) & 0xFFFFFFFFFFFFFFFF, _as_dp(x0), float(sigma0),
                                        _as_dp(lo), _as_dp(up), int(n_func_evals), int(restarts), _as_dp(tab),
                                        C.byref(res), C.byref(nn)))
    r = _cmaes_result(outs)
    r["n_negative"] = nn.value
    return r


def maximize_cmaes_es(objective, seed, x0, lower, upper, n_func_evals=1000, restarts=0, sigma0=0.6):
    """gpk_maximize_cmaes_es: the same minimising minus the entropy change (one handle: gpk_es_compute's value;
    several: gpk_es_multi's mean) -> as maximize_cmaes without n_negative."""
    h0 = objective[0]
    x0, lo, up, tab, outs, res = _cmaes_io(x0, lower, upper, restarts)
    h0._check(h0.lib.gpk_maximize_cmaes_es(_handles(objective), len(objective), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                           _as_dp(x0), float(sigma0), _as_dp(lo), _as_dp(up), int(n_func_evals),
                                           int(restarts), _as_dp(tab), C.byref(res)))
    return _cmaes_result(outs)


def maximize_cmaes_esmc(objective, seed, x0, lower, upper, n_func_evals=1000, restarts=0, sigma0=0.6):
    """gpk_maximize_cmaes_esmc: the same minimising minus the sampling-based entropy change -> as maximize_cmaes_es."""
    h0 = objective[0]
    x0, lo, up, tab, outs, res = _cmaes_io(x0, lower, upper, restarts)
    h0._check(h0.lib.gpk_maximize_cmaes_esmc(_handles(objective), len(objective), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                             _as_dp(x0), float(sigma0), _as_dp(lo), _as_dp(up), int(n_func_evals),
                                             int(restarts), _as_dp(tab), C.byref(res)))
    return _cmaes_result(outs)


def maximize_cmaes_es_cost(objective, cost, seed, x0, lower, upper, cfg_lower, cfg_upper, basis_objective, basis_cost,
                           overhead, n_func_evals=1000, restarts=0, sigma0=0.6):
    """gpk_maximize_cmaes_es_cost: the same over the extended box lower / upper (d) minimising minus the information
    gain per unit cost of gpk_es_cost_multi (configuration bounds cfg_lower / cfg_upper, d - 1) -> as
    maximize_cmaes_es."""
    ho, hc, clo, cup = _es_cost_args(objective, cost, cfg_lower, cfg_upper)
    h0 = objective[0]
    x0, lo, up, tab, outs, res = _cmaes_io(x0, lower, upper, restarts)
    if lo.size != clo.size + 1:
        raise ValueError("maximize_cmaes_es_cost: the box needs d entries, the configuration bounds d - 1")
    h0._check(h0.lib.gpk_maximize_cmaes_es_cost(ho, hc, len(objective), int(seed) & 0xFFFFFFFFFFFFFFFF, _as_dp(x0),
                                                float(sigma0), _as_dp(lo), _as_dp(up), int(n_func_evals),
                                                int(restarts), _as_dp(tab), _as_dp(clo), _as_dp(cup), clo.size,
                                                int(basis_objective), int(basis_cost), float(overhead), C.byref(res)))
    return _cmaes_result(outs)


def cmaes_draws(handle, seed, run, g0, g1, lam, d):
    """gpk_cmaes_draws: the normals of generations g0 .. g1 - 1 of run ``run`` -> ((g1 - g0), lam, d)."""
    out = np.empty((int(g1) - int(g0), int(lam), int(d)))
    handle._check(handle.lib.gpk_cmaes_draws(handle._h, int(seed) & 0xFFFFFFFFFFFFFFFF, int(run), int(g0), int(g1),
                                             int(lam), int(d), _as_dp(out)))
    return out


class _DirectResult(C.Structure):
    _fields_ = [(name, _vp) for name in ("best_x", "best_energy", "nit", "nfev", "stop", "rows")]


def _direct_io(lower, upper, n_iters):
    lo, up = f64(lower).ravel(), f64(upper).ravel()
    if lo.size != up.size:
        raise ValueError("maximize_direct: lower and upper need d entries each")
    outs = dict(best_x=np.empty(lo.size), best_energy=np.empty(1), nit=np.zeros(1, dtype=np.intc),
                nfev=np.zeros(1, dtype=np.int_), stop=np.zeros(1, dtype=np.intc),
                rows=np.zeros(max(int(n_iters) - 1, 1), dtype=np.int_))
    res = _DirectResult(*[outs[k].ctypes.data for k, _ in _DirectResult._fields_])
    return lo, up, outs, res


def _direct_result(outs):
    nit, stop = int(outs["nit"][0]), int(outs["stop"][0])
    sampled = max(nit - 1 - (stop == DIRECT_MAXT), 0)            # iterations 2 .. nit, the last one not under maxT
    return dict(x=outs["best_x"], energy=float(outs["best_energy"][0]), nit=nit, nfev=int(outs["nfev"][0]),
                stop=stop, rows=outs["rows"][:sampled].astype(np.int64))


def maximize_direct(handles, kind, eta, par, lower, upper, n_func_evals=400, n_iters=200):
    """gpk_maximize_direct over ``handles`` (all fitted, same device): DIRECT in the box lower / upper (d,) minimising
    -acq (kind ACQ_EI ... ACQ_LCB, acq the mean over the handles) -> dict(x (d,), energy, nit, nfev, stop, rows (the
    rows of iterations 2 .. nit), n_negative)."""
    h0 = handles[0]
    lo, up, outs, res = _direct_io(lower, upper, n_iters)
    nn = C.c_long()
    h0._check(h0.lib.gpk_maximize_direct(_handles(handles), len(handles), int(kind), _as_dp(_etas(eta, len(handles))),
                                         float(par), _as_dp(lo), _as_dp(up), int(n_func_evals), int(n_iters),
                                         C.byref(res), C.byref(nn)))
    r = _direct_result(outs)
    r["n_negative"] = nn.value
    return r


def maximize_direct_es(objective, lower, upper, n_func_evals=400, n_iters=200):
    """gpk_maximize_direct_es: the same minimising minus the entropy change -> as maximize_direct without n_negative."""
    h0 = objective[0]
    lo, up, outs, res = _direct_io(lower, upper, n_iters)
    h0._check(h0.lib.gpk_maximize_direct_es(_handles(objective), len(objective), _as_dp(lo), _as_dp(up),
                                            int(n_func_evals), int(n_iters), C.byref(res)))
    return _direct_result(outs)


def maximize_direct_esmc(objective, lower, upper, n_func_evals=400, n_iters=200):
    """gpk_maximize_direct_esmc: the same minimising minus the sampling-based entropy change."""
    h0 = objective[0]
    lo, up, outs, res = _direct_io(lower, upper, n_iters)
    h0._check(h0.lib.gpk_maximize_direct_esmc(_handles(objective), len(objective), _as_dp(lo), _as_dp(up),
                                              int(n_func_evals), int(n_iters), C.byref(res)))
    return _direct_result(outs)


def maximize_direct_es_cost(objective, cost, lower, upper, cfg_lower, cfg_upper, basis_objective, basis_cost,
                            overhead, n_func_evals=400, n_iters=200):
    """gpk_maximize_direct_es_cost: the same over the extended box lower / upper (d) minimising minus the information
    gain per unit cost of gpk_es_cost_multi (configuration bounds cfg_lower / cfg_upper, d - 1)."""
    ho, hc, clo, cup = _es_cost_args(objective, cost, cfg_lower, cfg_upper)
    h0 = objective[0]
    lo, up, outs, res = _direct_io(lower, upper, n_iters)
    if lo.size != clo.size + 1:
        raise ValueError("maximize_direct_es_cost: the box needs d entries, the configuration bounds d - 1")
    h0._check(h0.lib.gpk_maximize_direct_es_cost(ho, hc, len(objective), _as_dp(lo), _as_dp(up), int(n_func_evals),
                                                 int(n_iters), _as_dp(clo), _as_dp(cup), clo.size,
                                                 int(basis_objective), int(basis_cost), float(overhead),
                                                 C.byref(res)))
    return _direct_result(outs)


def sample_representers(models, seeds, nb, steps, max_runs, kind, eta, par, lower, upper, fabolas=None):
    """gpk_sample_representers: the stretch-move representer points of one estimator per handle in ``models``.
    seeds (n,) 64-bit, eta (n,), lower / upper (dw,) the walker box; fabolas = None or dict(cfg_lower, cfg_upper, basis,
    env_value) (the scored row is [walker, env_value] under the model's Fabolas transform) -> dict(zb (n, nb, dw),
    lmb (n, nb), runs (n,), n_accepted (n, nb), n_negative)."""
    n = len(models)
    if n < 1:
        raise ValueError("sample_representers: need at least one model")
    h0 = models[0]
    hs = _handles(models)
    sd = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint64).ravel())
    etas = _etas(eta, n)
    lo, up = f64(lower).ravel(), f64(upper).ravel()
    if sd.size != n or lo.size != up.size:
        raise ValueError("sample_representers: need one seed per model and lower / upper of one length")
    dw, nb = lo.size, int(nb)
    if fabolas is not None:
        clo, cup = f64(fabolas["cfg_lower"]).ravel(), f64(fabolas["cfg_upper"]).ravel()
        if clo.size != dw or cup.size != dw:
            raise ValueError("sample_representers: the configuration bounds need dw = d - 1 entries")
        basis, env = int(fabolas["basis"]), float(fabolas["env_value"])
    else:
        clo = cup = None
        basis, env = 0, 0.0
    zb = np.empty((n, max(nb, 0), dw))
    lmb = np.empty((n, max(nb, 0)))
    acc = np.zeros((n, max(nb, 0)), dtype=np.int64)
    runs = np.zeros(n, dtype=np.int32)
    nn = C.c_long(0)
    h0._check(h0.lib.gpk_sample_representers(hs, n, sd.ctypes.data_as(C.POINTER(C.c_ulonglong)), nb, int(steps),
                                             int(max_runs), int(kind), _as_dp(etas), float(par), _as_dp(lo), _as_dp(up),
                                             dw, int(fabolas is not None), _as_dp(clo) if clo is not None else None,
                                             _as_dp(cup) if cup is not None else None, basis, env, _as_dp(zb),
                                             _as_dp(lmb), runs.ctypes.data_as(_ip), acc.ctypes.data_as(_lp),
                                             C.byref(nn)))
    return dict(zb=zb, lmb=lmb, runs=runs, n_accepted=acc, n_negative=nn.value)


def set_hyper_model(handle, slots, n_terms, mean, tiny, prior_kind=PRIOR_NONE, prior_par=None, n_ls=0, n_lr=0):
    """gpk_set_hyper_model: theta -> the handle's kernel (set_kernel first; its structure is used, not its values).
    slots: kernels.py flatten()["slots"] (one ("amp", None), ("metric", [terms]), ("lin_a", None), ("lin_b", None) or
    ("task", k) per kernel parameter; lin_a / lin_b need the environment factor set on the handle, the task slots (in
    packed order) its task factor); n_terms: the kernel's metric
    terms; mean / tiny: the constant mean and the jitter added to yerr^2; prior_par: the 7 constants of include/gpk.h
    (None without a prior)."""
    kinds = {"metric": 0, "amp": 1, "lin_a": 2, "lin_b": 3, "task": 4}
    amp = np.array([kinds[kind] for kind, _ in slots], dtype=np.int32)
    term = np.full(int(n_terms), -1, dtype=np.int32)
    for p, (kind, terms) in enumerate(slots):
        if kind == "metric":
            for t in terms:
                if not 0 <= t < n_terms:
                    raise ValueError("set_hyper_model: slot %d names term %d of %d" % (p, t, n_terms))
                term[t] = p
    par = f64(prior_par).ravel() if prior_par is not None else None
    if par is not None and par.size != 7:
        raise ValueError("set_hyper_model: the prior needs 7 constants")
    handle._check(handle.lib.gpk_set_hyper_model(handle._h, amp.size, amp.ctypes.data_as(_ip), term.ctypes.data_as(_ip),
                                                 term.size, float(mean), float(tiny), int(prior_kind),
                                                 _as_dp(par) if par is not None else None, int(n_ls), int(n_lr)))


def hyper_lnpost(handle, thetas, _fn="gpk_hyper_lnpost"):
    """gpk_hyper_lnpost: (log-likelihood, log-prior) of every row of thetas (count, dim), as gpk_sample_hypers computes
    them."""
    T = f64(np.atleast_2d(thetas))
    count, dim = T.shape
    ll, lp = np.empty(count), np.empty(count)
    handle._check(getattr(handle.lib, _fn)(handle._h, _as_dp(T), count, dim, _as_dp(ll), _as_dp(lp)))
    return ll, lp


def hyper_lnpost_blocked(handle, thetas):
    """gpk_hyper_lnpost_blocked: hyper_lnpost for 2 <= N <= HYPER_BLOCKED_MAX_N, as gpk_sample_hypers_blocked and
    gpk_optimize_hypers_blocked compute it (a batched blocked Cholesky per chunk of thetas)."""
    return hyper_lnpost(handle, thetas, _fn="gpk_hyper_lnpost_blocked")


def sample_hypers(handle, p0, steps, seed, _fn="gpk_sample_hypers"):
    """gpk_sample_hypers: one stretch-move run of the walkers p0 (nwalkers, dim) for `steps` steps ->
    dict(pos (nwalkers, dim), lnpost (nwalkers,), n_accepted (nwalkers,))."""
    P = f64(np.atleast_2d(p0))
    nw, dim = P.shape
    pos, lnp = np.empty((nw, dim)), np.empty(nw)
    acc = np.zeros(nw, dtype=np.int64)
    handle._check(getattr(handle.lib, _fn)(handle._h, _as_dp(P), nw, dim, int(steps), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                           _as_dp(pos), _as_dp(lnp), acc.ctypes.data_as(_lp)))
    return dict(pos=pos, lnpost=lnp, n_accepted=acc)


def sample_hypers_blocked(handle, p0, steps, seed):
    """gpk_sample_hypers_blocked: sample_hypers over the log-posteriors of hyper_lnpost_blocked (N up to
    HYPER_BLOCKED_MAX_N)."""
    return sample_hypers(handle, p0, steps, seed, _fn="gpk_sample_hypers_blocked")


def optimize_hypers(handle, p0, maxcor=10, maxiter=15000, maxfun=15000, ftol=2.220446049250313e-09, gtol=1e-5,
                    eps=1e-8, maxls=20, _fn="gpk_optimize_hypers"):
    """gpk_optimize_hypers: scipy.optimize.minimize(nll, p0, method='L-BFGS-B') with scipy's default options, on the
    device -> dict(theta (dim,), f, nit, nfev, status (LB_*), rounds, noop_rounds).  rounds: the points scored (dim + 1
    evaluations each); noop_rounds: the launches after the final round that returned at once (the rest of the last
    chunk of HO_CHUNK)."""
    x0 = f64(np.ravel(p0)).copy()
    dim = x0.size
    theta = np.empty(dim)
    f, nfev = C.c_double(), C.c_long()
    nit, status = C.c_int(), C.c_int()
    handle._check(getattr(handle.lib, _fn)(handle._h, _as_dp(x0), dim, int(maxcor), int(maxiter), int(maxfun),
                                           float(ftol), float(gtol), float(eps), int(maxls), _as_dp(theta),
                                           C.byref(f), C.byref(nit), C.byref(nfev), C.byref(status)))
    rounds = nfev.value // (dim + 1)
    return dict(theta=theta, f=f.value, nit=nit.value, nfev=nfev.value, status=status.value, rounds=rounds,
                noop_rounds=-(-rounds // HO_CHUNK) * HO_CHUNK - rounds)


def optimize_hypers_blocked(handle, p0, **opt):
    """gpk_optimize_hypers_blocked: optimize_hypers over the objective of hyper_lnpost_blocked (N up to
    HYPER_BLOCKED_MAX_N); the same options and result."""
    return optimize_hypers(handle, p0, _fn="gpk_optimize_hypers_blocked", **opt)


def blr_features(n_dims, basis):
    """F, the number of features of a BayesianLinearRegression handle on n_dims inputs."""
    return {BLR_LINEAR: n_dims + 1, BLR_QUADRATIC: 2 * n_dims + 1, BLR_NONE: n_dims}[basis]


def blr_set_data(handle, X, y, basis, prior_par):
    """gpk_blr_set_data: the training set and its features (basis: BLR_*) on the handle, which becomes a
    BayesianLinearRegression handle; prior_par = (lognormal sigma, lognormal mean, horseshoe scale)."""
    X, y, par = f64(X), f64(y).ravel(), f64(prior_par).ravel()
    n, d = X.shape
    if par.size != 3:
        raise ValueError("blr_set_data: the prior needs 3 constants")
    handle._check(handle.lib.gpk_blr_set_data(handle._h, _as_dp(X), _as_dp(y), n, d, int(basis), _as_dp(par)))


def blr_lnpost(handle, thetas):
    """gpk_blr_lnpost: the log-posterior (marginal log-likelihood plus prior, NaN -> -inf) of every row of thetas
    (count, 2) = (log alpha, log beta), as gpk_blr_sample computes it."""
    T = f64(np.atleast_2d(thetas))
    if T.ndim != 2 or T.shape[1] != 2:
        raise ValueError("blr_lnpost: thetas must have shape (count, 2)")
    out = np.empty(T.shape[0])
    handle._check(handle.lib.gpk_blr_lnpost(handle._h, _as_dp(T), T.shape[0], _as_dp(out)))
    return out


def blr_sample(handle, seed, p0, steps):
    """gpk_blr_sample: one stretch-move run of the walkers p0 (nwalkers, 2) for `steps` steps ->
    dict(pos (nwalkers, 2), lnpost (nwalkers,), n_accepted (nwalkers,))."""
    P = f64(np.atleast_2d(p0))
    if P.ndim != 2 or P.shape[1] != 2:
        raise ValueError("blr_sample: p0 must have shape (nwalkers, 2)")
    nw = P.shape[0]
    pos, lnp = np.empty((nw, 2)), np.empty(nw)
    acc = np.zeros(nw, dtype=np.int64)
    handle._check(handle.lib.gpk_blr_sample(handle._h, int(seed) & 0xFFFFFFFFFFFFFFFF, nw, _as_dp(P), int(steps),
                                            _as_dp(pos), _as_dp(lnp), acc.ctypes.data_as(_lp)))
    return dict(pos=pos, lnpost=lnp, n_accepted=acc)


def blr_fit(handle, hypers):
    """gpk_blr_fit: the weight posteriors of the (alpha, beta) rows of hypers, resident on the handle."""
    H = f64(np.atleast_2d(hypers))
    if H.ndim != 2 or H.shape[1] != 2:
        raise ValueError("blr_fit: hypers must have shape (k, 2)")
    handle._check(handle.lib.gpk_blr_fit(handle._h, _as_dp(H), H.shape[0]))


def blr_models(handle):
    """gpk_blr_get_models: [(m (F,), S (F, F))] of the last gpk_blr_fit."""
    n, F, k = C.c_int(), C.c_int(), C.c_int()
    handle._check(handle.lib.gpk_blr_dims(handle._h, C.byref(n), C.byref(F), C.byref(k)))
    M, S = np.empty((k.value, F.value)), np.empty((k.value, F.value, F.value))
    handle._check(handle.lib.gpk_blr_get_models(handle._h, _as_dp(M), _as_dp(S)))
    return [(M[i].copy(), S[i].copy()) for i in range(k.value)]


RF_FIELDS = ("feat", "thr", "left", "W", "mean", "var")     # gpk_rf_get_trees' node arrays, in its argument order


def rf_set_data(handle, X, y):
    """gpk_rf_set_data: the training set on the handle, which becomes a random-forest handle."""
    X, y = f64(X), f64(y).ravel()
    if X.ndim != 2 or X.shape[0] != y.size:
        raise ValueError("rf_set_data: X must be (n, d) and y (n,)")
    n, d = X.shape
    handle._check(handle.lib.gpk_rf_set_data(handle._h, _as_dp(X), _as_dp(y), n, d))


def rf_fit(handle, seed, counter, num_trees, n_per_tree, bootstrap, total_variance):
    """gpk_rf_fit: grow the forest on the device (draws keyed by seed and the fit counter)."""
    handle._check(handle.lib.gpk_rf_fit(handle._h, int(seed) & 0xFFFFFFFFFFFFFFFF, int(counter) & 0xFFFFFFFF,
                                        int(num_trees), int(n_per_tree), int(bool(bootstrap)),
                                        int(bool(total_variance))))


def rf_trees(handle):
    """gpk_rf_get_trees: dict(n_nodes (T,), feat, thr, left, W, mean, var (T, 2 n) each, breadth-first node order;
    right child = left + 1, feat -1 at a leaf; slots past n_nodes are zero)."""
    n, d, T, S = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    handle._check(handle.lib.gpk_rf_dims(handle._h, C.byref(n), C.byref(d), C.byref(T), C.byref(S)))
    T, S = T.value, S.value
    if T == 0:
        raise RuntimeError("rf_trees: model is not fitted (gpk_rf_fit)")
    nn = np.empty(T, dtype=np.int32)
    out = {k: np.empty((T, S), dtype=np.int32 if k in ("feat", "left") else np.float64) for k in RF_FIELDS}
    ptrs = [out[k].ctypes.data_as(_ip if out[k].dtype == np.int32 else _dp) for k in RF_FIELDS]
    handle._check(handle.lib.gpk_rf_get_trees(handle._h, nn.ctypes.data_as(_ip), *ptrs))
    pad = np.arange(S)[None, :] >= nn[:, None]
    for k in RF_FIELDS:
        out[k][pad] = 0
    out["n_nodes"] = nn
    return out


def rf_set_trees(handle, trees, total_variance):
    """gpk_rf_set_trees: the arrays of rf_trees back onto a handle that holds the same training set."""
    nn = np.ascontiguousarray(trees["n_nodes"], dtype=np.int32)
    arr = {k: np.ascontiguousarray(trees[k], dtype=np.int32 if k in ("feat", "left") else np.float64)
           for k in RF_FIELDS}
    ptrs = [arr[k].ctypes.data_as(_ip if arr[k].dtype == np.int32 else _dp) for k in RF_FIELDS]
    handle._check(handle.lib.gpk_rf_set_trees(handle._h, nn.size, int(bool(total_variance)), nn.ctypes.data_as(_ip),
                                              *ptrs))


def bnn_params(n_dims):
    """P, the parameters of one network of a BNN handle on n_dims inputs."""
    return 50 * int(n_dims) + 2652


def bnn_set_data(handle, X, y):
    """gpk_bnn_set_data: the training set on the handle (normalised there), which becomes a BNN handle."""
    X, y = f64(X), f64(y).ravel()
    if X.ndim != 2 or X.shape[0] != y.size:
        raise ValueError("bnn_set_data: X must be (n, d) and y (n,)")
    n, d = X.shape
    handle._check(handle.lib.gpk_bnn_set_data(handle._h, _as_dp(X), _as_dp(y), n, d))


def bnn_train(handle, seed, counter, lr, mdecay, eps, burn_in, num_steps, keep_every, batch):
    """gpk_bnn_train: one adaptive-SGHMC chain in one launch (draws keyed by seed and the train counter)."""
    handle._check(handle.lib.gpk_bnn_train(handle._h, int(seed) & 0xFFFFFFFFFFFFFFFF, int(counter) & 0xFFFFFFFF,
                                           float(lr), float(mdecay), float(eps), int(burn_in), int(num_steps),
                                           int(keep_every), int(batch)))


def bnn_dims(handle):
    """gpk_bnn_dims -> (n, d, P, S)."""
    n, d, P, S = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    handle._check(handle.lib.gpk_bnn_dims(handle._h, C.byref(n), C.byref(d), C.byref(P), C.byref(S)))
    return n.value, d.value, P.value, S.value


def bnn_samples(handle):
    """gpk_bnn_get_samples: the (S, P) kept networks."""
    _, _, P, S = bnn_dims(handle)
    if S == 0:
        raise RuntimeError("bnn_samples: model is not trained (gpk_bnn_train)")
    out = np.empty((S, P))
    handle._check(handle.lib.gpk_bnn_get_samples(handle._h, _as_dp(out)))
    return out


def bnn_set_samples(handle, samples):
    """gpk_bnn_set_samples: the (S, P) networks of bnn_samples back onto a handle that holds the same training set."""
    Z = f64(samples)
    if Z.ndim != 2 or Z.shape[1] != bnn_dims(handle)[2]:
        raise ValueError("bnn_set_samples: samples must be (S, P)")
    handle._check(handle.lib.gpk_bnn_set_samples(handle._h, Z.shape[0], _as_dp(Z)))


def bnn_state(handle):
    """gpk_bnn_get_state -> dict(theta, p, tau, g, vhat) of the last chain (P each)."""
    P = bnn_dims(handle)[2]
    out = {k: np.empty(P) for k in ("theta", "p", "tau", "g", "vhat")}
    handle._check(handle.lib.gpk_bnn_get_state(handle._h, *[_as_dp(out[k]) for k in ("theta", "p", "tau", "g", "vhat")]))
    return out


def bnn_draws(handle, seed, counter, step0, ns):
    """gpk_bnn_draws: the (ns, P) normals of chain steps step0 .. step0 + ns - 1 (step -1: the initial weights)."""
    P = bnn_dims(handle)[2]
    Z = np.empty((int(ns), P))
    handle._check(handle.lib.gpk_bnn_draws(handle._h, int(seed) & 0xFFFFFFFFFFFFFFFF, int(counter) & 0xFFFFFFFF,
                                           int(step0), int(ns), _as_dp(Z)))
    return Z


def dngo_params(n_dims):
    """P, the parameters of the net of a DNGO handle on n_dims inputs."""
    return 50 * int(n_dims) + 5201


def dngo_set_data(handle, X, y, normalize_input, normalize_output, prior_par):
    """gpk_dngo_set_data: the training set on the handle (normalised there under the flags), which becomes a DNGO
    handle; prior_par = (lognormal sigma, lognormal mean, horseshoe scale) of its Bayesian linear regression."""
    X, y, par = f64(X), f64(y).ravel(), f64(prior_par).ravel()
    if X.ndim != 2 or X.shape[0] != y.size:
        raise ValueError("dngo_set_data: X must be (n, d) and y (n,)")
    if par.size != 3:
        raise ValueError("dngo_set_data: the prior needs 3 constants")
    n, d = X.shape
    handle._check(handle.lib.gpk_dngo_set_data(handle._h, _as_dp(X), _as_dp(y), n, d, int(bool(normalize_input)),
                                               int(bool(normalize_output)), _as_dp(par)))


def dngo_train(handle, seed, counter, lr, batch, epochs):
    """gpk_dngo_train: train a fresh net by Adam in one launch (draws keyed by seed and the train counter), then the
    features and the regression's products."""
    handle._check(handle.lib.gpk_dngo_train(handle._h, int(seed) & 0xFFFFFFFFFFFFFFFF, int(counter) & 0xFFFFFFFF,
                                            float(lr), int(batch), int(epochs)))


def dngo_fit(handle, hypers):
    """gpk_dngo_fit: the weight posteriors of the (alpha, beta) rows of hypers and the collapsed predictive."""
    H = f64(np.atleast_2d(hypers))
    if H.ndim != 2 or H.shape[1] != 2:
        raise ValueError("dngo_fit: hypers must have shape (k, 2)")
    handle._check(handle.lib.gpk_dngo_fit(handle._h, _as_dp(H), H.shape[0]))


def dngo_dims(handle):
    """gpk_dngo_dims -> (n, d, P, k)."""
    n, d, P, k = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    handle._check(handle.lib.gpk_dngo_dims(handle._h, C.byref(n), C.byref(d), C.byref(P), C.byref(k)))
    return n.value, d.value, P.value, k.value


def dngo_net(handle):
    """gpk_dngo_get_net: the (P,) trained net."""
    out = np.empty(dngo_dims(handle)[2])
    handle._check(handle.lib.gpk_dngo_get_net(handle._h, _as_dp(out)))
    return out


def dngo_set_net(handle, net):
    """gpk_dngo_set_net: the net of dngo_net back onto a handle that holds the same training set."""
    w = f64(net).ravel()
    if w.size != dngo_dims(handle)[2]:
        raise ValueError("dngo_set_net: the net must have P entries")
    handle._check(handle.lib.gpk_dngo_set_net(handle._h, _as_dp(w)))


def dngo_features(handle, X):
    """gpk_dngo_features: the (m, 50) features of the rows X (m, d)."""
    X = f64(np.atleast_2d(X))
    out = np.empty((X.shape[0], DNGO_H))
    handle._check(handle.lib.gpk_dngo_features(handle._h, _as_dp(X), X.shape[0], _as_dp(out)))
    return out


def dngo_state(handle):
    """gpk_dngo_get_state -> dict(m, v (P each), t) of Adam after the last train."""
    P = dngo_dims(handle)[2]
    m, v, t = np.empty(P), np.empty(P), C.c_longlong()
    handle._check(handle.lib.gpk_dngo_get_state(handle._h, _as_dp(m), _as_dp(v), C.byref(t)))
    return dict(m=m, v=v, t=t.value)


_moments_handle = {}


def moments_handle(device=0):
    """Shared handle for gpk_acq_moments (acquisition on non-GPU models)."""
    if device not in _moments_handle:
        _moments_handle[device] = Handle(device)
    return _moments_handle[device]
