"""``_lib.maximize_lbfgs`` on the oracle-backed FakeHandle (tests/fake_gpk.py) — TEST INFRASTRUCTURE ONLY.

The iteration is tests/lbfgs_model.py, the exact restatement of gpk_maximize_lbfgs; the scores come from the fake
handles (the oracle): acquisition values averaged over the models like gpk_acq_multi mode 0, or the mixture moments of
mode 1 for the posterior objectives.  Argument checks mirror the C side's GPK_BAD_ARG cases as ValueError.  ``calls``
records every call (kind, starts) for the dispatch tests."""
import numpy as np

from tests import fake_de, lbfgs_model

calls = []


def maximize_lbfgs(handles, kind, eta, par, x0, lower, upper, **options):
    from robo_b200 import _lib
    lower, upper = np.asarray(lower, dtype=np.float64).ravel(), np.asarray(upper, dtype=np.float64).ravel()
    x0 = np.atleast_2d(np.asarray(x0, dtype=np.float64))
    o = dict(_lib.LB_DEFAULTS, **options)
    if lower.size > _lib.LB_MAX_D or not 1 <= o["maxcor"] <= 32 or not np.all(lower < upper) \
            or x0.shape[1] != lower.size or not np.all(np.isfinite(x0)) or kind not in (1, 2, 3, 4, 5, 6):
        raise ValueError("gpk_maximize_lbfgs: bad arguments")
    calls.append(dict(kind=kind, x0=x0.copy(), n_models=len(handles)))
    n_negative = [0]

    def energy_fn(X):
        if kind in (_lib.OBJ_MEAN, _lib.OBJ_MEAN_STD):
            r = _lib.acq_multi(handles, X, 1)
            return r["mean"] if kind == _lib.OBJ_MEAN else r["mean"] + np.sqrt(r["var"])
        etas = np.broadcast_to(np.asarray(eta, dtype=np.float64), (len(handles),))
        rs = [h.acq(X, kind, float(e), par) for h, e in zip(handles, etas)]
        n_negative[0] += sum(r["n_negative"] for r in rs)
        return -np.mean([r["values"] for r in rs], axis=0)

    r = lbfgs_model.minimize(energy_fn, x0, lower, upper, **options)
    r["n_negative"] = n_negative[0]
    return r


def install(monkeypatch):
    """fake_de.install plus the L-BFGS entry point."""
    from robo_b200 import _lib
    cls = fake_de.install(monkeypatch)
    del calls[:]
    monkeypatch.setattr(_lib, "maximize_lbfgs", maximize_lbfgs)
    return cls
