"""robo/util/epmgp.py on the GPU: the EPMGP approximation of p_min, the probability of each of Nb points to be the
minimum of a Gaussian N(mu, var) (Cunningham, Hennig and Lacoste-Julien, 2011).  Entropy search represents its
belief about the minimiser by it.

Every EP problem (one per point) and the renormalisation run in libgpk.so (gpk_ep_joint_min, gpk_es.cuh); there is
no host fallback.  2 <= Nb <= 64.
"""
import numpy as np

from .. import _lib


def joint_min(mu, var, with_derivatives=False, **kwargs):
    """log p_min of N(mu, var) (epmgp.joint_min).

    mu: np.ndarray(N,), var: np.ndarray(N, N).  Returns logP (mu's shape); with_derivatives=True returns
    (logP, dlogPdMu (N, N), dlogPdSigma (N, N (N + 1) / 2), dlogPdMudMu (N, N, N)).  Raises the reference's
    ``Exception`` when an EP update yields a NaN variance, numpy.linalg.LinAlgError when the final IRSR system is
    not positive definite, ValueError for N outside 2 .. 64."""
    mu = np.asarray(mu, dtype=np.float64)
    r = _lib.moments_handle().ep_joint_min(mu.ravel(), np.asarray(var, dtype=np.float64), derivatives=with_derivatives)
    logP = r["logP"].reshape(mu.shape)
    if not with_derivatives:
        return logP
    return logP, r["dlogPdMu"], r["dlogPdSigma"], r["dlogPdMudMu"]
