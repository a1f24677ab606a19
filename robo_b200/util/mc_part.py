"""joint_pmin — robo/util/mc_part.py:7-68 on the GPU (gpk_mc_pmin): the probability of each of Nb points to be the
minimum of N(m, V), estimated by counting which point is smallest over Nf correlated function draws (and, for m of
shape (Nb, Np), over each of its Np mean columns).

The factorisation of V + noise I climbs the reference's jitter ladder float for float (0, 1e-9, ..., 10000.0) and
raises numpy.linalg.LinAlgError past its last rung.  The reference draws F with np.random.multivariate_normal; here F
comes from the device's Philox stream keyed by a 64-bit seed drawn from ``rng`` (np.random when rng is None, so a run
is reproducible under np.random.seed), with Box-Muller: the same law, not the same numbers.
"""
import logging

import numpy as np

logger = logging.getLogger(__name__)


def draw_seed(rng=None):
    """A 64-bit seed of the device's draws from ``rng`` (np.random's global stream when None)."""
    r = np.random if rng is None else rng
    return int(r.randint(0, 2 ** 63, dtype=np.int64))


def joint_pmin(m, V, Nf, rng=None):
    """m (Nb,) or (Nb, Np) means, V (Nb, Nb) covariance, Nf draws -> pmin (Nb,), clamped below at 1e-70."""
    from robo_b200 import _lib
    m = np.asarray(m, dtype=np.float64)
    if m.ndim == 1:
        m = m[:, None]
    pmin, n_jitter = _lib.moments_handle().mc_pmin(m, np.asarray(V, dtype=np.float64), int(Nf), draw_seed(rng))
    if n_jitter:
        logger.error("Added noise on the diagonal of the covariance to factorise it.")
    return pmin
