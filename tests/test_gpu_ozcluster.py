"""Option "ozcluster": the int8 variance contraction in clusters of 1, 2 or 4 CTAs that share the L^-1 digit slices by
TMA multicast.  The level sums are exact int32 sums and every tile writes its own partial-sum slot, so the posterior
moments and EI must be bit-identical to ozcluster = 1 for every cluster size, with and without the persistent walk,
and with the walk capped at one or two clusters ("ozgrid"), so that each cluster walks many tiles of different lengths."""
import numpy as np
import pytest

from robo_b200 import kernels as K

pytestmark = pytest.mark.gpu

# the ragged shapes of test_int8_scoring_edge_shapes (one, two, three and five row blocks, candidate counts off the
# tile sizes) and the benchmark's training-set size
SHAPES = [(100, 3, 2048), (129, 2, 2049), (256, 16, 2177), (640, 5, 4099), (384, 8, 2500), (4096, 16, 20000)]


def _score(N, D, M, cluster, persist, grid=0):
    from robo_b200 import _lib
    rng = np.random.RandomState(N * 7 + D)
    X, Xs = rng.rand(N, D), rng.rand(M, D)
    y = np.sin(X.sum(axis=1)) + 0.5
    theta = np.concatenate(([0.2], rng.uniform(-0.5, 0.5, D)))
    h = _lib.Handle(0)
    h.set_option("ozaki", 1)
    h.set_option("ozcluster", cluster)
    h.set_option("ozpersist", persist)
    h.set_option("ozgrid", grid)
    h.set_data(X, y)
    f = K.Product(K.ConstantKernel(theta[0], ndim=D), K.Matern52Kernel(np.exp(theta[1:]), ndim=D)).flatten()
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    h.fit(1e-3, float(np.mean(y)))
    r = h.acq(Xs, _lib.ACQ_EI, float(np.min(y)), 0.0, want_values=True, want_moments=True)
    t = h.timings()
    h.close()
    return r, t


@pytest.mark.parametrize("N,D,M", SHAPES)
def test_cluster_sizes_are_bit_identical(N, D, M):
    ref, t = _score(N, D, M, 1, 0)
    assert t["launches_ozaki"] >= 1 and int(t["ozaki_kernel_variant"]) == 1, t
    for cluster in (1, 2, 4):
        for persist in (0, 1):
            r, t = _score(N, D, M, cluster, persist)
            assert int(t["ozaki_kernel_variant"]) == 1 + 8 * persist + {1: 0, 2: 16, 4: 32}[cluster], t
            for k in ("values", "mu", "var"):
                np.testing.assert_array_equal(r[k], ref[k])
            assert r["best_idx"] == ref["best_idx"]
        # the persistent walk on one or two clusters: each cluster walks many tiles of different lengths
        for grid in (1, 2):
            r, t = _score(N, D, M, cluster, 1, grid)
            assert int(t["ozaki_kernel_variant"]) == 1 + 8 + {1: 0, 2: 16, 4: 32}[cluster], t
            for k in ("values", "mu", "var"):
                np.testing.assert_array_equal(r[k], ref[k])


def test_cluster_size_is_validated():
    from robo_b200 import _lib
    h = _lib.Handle(0)
    for bad in (0, 3, 8):
        with pytest.raises(ValueError):
            h.set_option("ozcluster", bad)
    for bad in (-1, -5):
        with pytest.raises(ValueError):
            h.set_option("ozgrid", bad)
    for good in (0, 1, 2, 1000):
        h.set_option("ozgrid", good)
    h.close()
