"""The entropy change of a candidate (InformationGain._dh_fun) restated twice in tests/es_model.py: in the
reference's matrix order and in the folded order gpk_es_dh_kernel uses.  Folding the quadratic form of dlogPdMudMu
to its lower triangle is exact algebra (only the symmetric part counts), so the two agree to rounding: 1e-10 of
max(|dH|, 1e-3) where |v - sn2| >= 1e-3 v."""
import numpy as np
import pytest

from tests import es_model as M
from tests.conftest import GOLDEN


def _state(name, rng):
    G = np.load(GOLDEN + "/es_ep.npz")
    mu, V = G[name + "_mu"], G[name + "_V"]
    ep = M.joint_min(mu, V)
    nb = mu.size
    W = np.linspace(-2.5, 2.5, 40)
    return dict(logP=ep["logP"], lmb=rng.randn(nb), dlogPdMu=ep["dlogPdMu"], dlogPdSigma=ep["dlogPdSigma"],
                dlogPdMudMu=ep["dlogPdMudMu"], W=W, sn2=1e-3), V


@pytest.mark.parametrize("name", ["rand17", "mixed", "rand2"])
def test_folded_equals_matrix_order(name):
    rng = np.random.RandomState(5)
    st, V = _state(name, rng)
    nb = V.shape[0]
    for _ in range(30):
        v = float(rng.choice([5e-4, 1e-2, 0.3, 1.5]))
        sigma = np.abs(rng.randn(nb)) * 0.1
        a, b = M.dh_matrix(st, v, sigma), M.dh_folded(st, v, sigma)
        assert abs(a - b) <= 1e-10 * max(abs(a), 1e-3), (a, b)


def test_compute_replacements():
    lo, up = np.zeros(2), np.ones(2)
    assert M.compute_value(0.3, np.array([1.5, 0.5]), lo, up) == np.spacing(1)
    assert M.compute_value(np.nan, np.array([0.5, 0.5]), lo, up) == -np.finfo(float).max
    assert M.compute_value(np.inf, np.array([0.5, 0.5]), lo, up) == -np.finfo(float).max
    assert M.compute_value(-np.inf, np.array([0.5, 0.5]), lo, up) == -np.inf
