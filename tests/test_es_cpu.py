"""EPMGP p_min (entropy search's belief about the minimiser): the numpy restatement tests/es_model.py against the
reference's own joint_min outputs (tests/golden/es_ep.npz, written by tools/make_es_golden.py), and the reference
test's known answers.

Tolerances.  The restatement runs the sweeps in the reference's scalar order, so the EP step counts must be equal.
Its closed form sums in a different order than numpy's dense products (R has two entries per column), so the
outputs agree to rounding, measured against the scale of each array: logP to 1e-12 of max |logP|, the derivatives
to 1e-10 of their max |entry|.  Observed on these cases: at most 9e-14 for logP and 4e-13 for the derivatives (both
on the Branin posterior); on a rougher posterior than these the derivatives were seen 2e-11 apart, hence the margin.
"""
import numpy as np
import pytest

from tests import es_model as M
from tests.conftest import GOLDEN

_G = np.load(GOLDEN + "/es_ep.npz")
NAMES = [str(n) for n in _G["names"]]
_MODEL = {}


def _model(name):
    if name not in _MODEL:
        _MODEL[name] = M.joint_min(_G[name + "_mu"], _G[name + "_V"])
    return _MODEL[name]


def _close(a, b, rel):
    scale = np.max(np.abs(b)) if b.size else 0.0
    assert np.all(np.abs(a - b) <= rel * scale), (np.max(np.abs(a - b)), scale)


@pytest.mark.parametrize("name", NAMES)
def test_model_matches_reference(name):
    m = _model(name)
    assert np.array_equal(m["lt_calls"], _G[name + "_lt_calls"])
    _close(m["logP"], _G[name + "_logP"], 1e-12)
    keep = _G[name + "_dlogPdMu"].shape[0]
    for key in ("dlogPdMu", "dlogPdSigma", "dlogPdMudMu"):
        _close(m[key][:keep], _G[name + "_" + key], 1e-10)


def test_known_answers():
    """test/test_acquisition_functions/test_information_gain.py:33-56 of the reference."""
    p = np.exp(_model("uniform")["logP"])
    assert np.all(p < 1 / 50 + 0.03) and np.all(p > 1 / 50 - 0.01)
    p = np.exp(_model("dirac")["logP"])
    assert p[0] == 1.0
    assert np.all(_G["dirac_logP"][1:] < -400)          # the z < -6 exit: logZ = -inf, replaced by -500


def test_model_sweeps_bounded():
    for name in NAMES:
        m = _model(name)
        nb = _G[name + "_mu"].shape[0]
        assert np.all((m["sweeps"] >= 1) & (m["sweeps"] <= 50))
        assert np.all(m["lt_calls"] <= m["sweeps"] * (nb - 1))


def test_nan_variance_raises():
    V = np.eye(4)
    V[2, 3] = V[3, 2] = np.nan
    with pytest.raises(M.EPFailed, match="Resulting variance contains NaN"):
        M.joint_min(np.zeros(4), V)


def test_binding_declares_ep():
    from robo_b200 import _lib
    assert "gpk_ep_joint_min" in _lib.exported_symbols()
    assert _lib.GPK_EP_FAILED == 6
