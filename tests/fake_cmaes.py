"""``_lib.maximize_cmaes`` on the oracle-backed FakeHandle (tests/fake_gpk.py) — TEST INFRASTRUCTURE ONLY.

The strategy is tests/cmaes_model.py, the exact restatement of gpk_maximize_cmaes, on its numpy normals; the
acquisition values come from the fake handles (the oracle), averaged over the models like gpk_acq_multi mode 0.
Argument checks mirror the C side's GPK_BAD_ARG cases as ValueError."""
import numpy as np

from robo_b200 import _lib
from tests import cmaes_model, fake_gpk


def maximize_cmaes(handles, kind, eta, par, seed, x0, lower, upper, n_func_evals=1000, restarts=0, sigma0=0.6):
    lower, upper = np.asarray(lower, dtype=np.float64).ravel(), np.asarray(upper, dtype=np.float64).ravel()
    x0 = np.asarray(x0, dtype=np.float64).ravel()
    d = lower.size
    if not 2 <= d <= _lib.CMA_MAX_D or not np.all(lower < upper) or not np.all(np.isfinite(x0)) \
            or not np.all((lower <= x0) & (x0 <= upper)) or not sigma0 > 0 or n_func_evals < 1 or restarts < 0 \
            or _lib.cmaes_lambda(d, restarts) > _lib.CMA_MAX_LAMBDA or kind not in (1, 2, 3, 4) \
            or len(set(map(id, handles))) != len(handles):
        raise ValueError("gpk_maximize_cmaes: bad arguments")
    etas = np.broadcast_to(np.asarray(eta, dtype=np.float64), (len(handles),))
    n_negative = [0]

    def acq_fn(X):
        rs = [h.acq(X, kind, float(e), par) for h, e in zip(handles, etas)]
        n_negative[0] += sum(r["n_negative"] for r in rs)
        return np.mean([r["values"] for r in rs], axis=0)

    r = cmaes_model.run(acq_fn, cmaes_model.numpy_normals(seed), x0, lower, upper, int(n_func_evals), int(restarts),
                        float(sigma0))
    r["n_negative"] = n_negative[0]
    return r


def install(monkeypatch):
    """fake_gpk.install plus the CMA-ES entry point."""
    cls = fake_gpk.install(monkeypatch)
    monkeypatch.setattr(_lib, "maximize_cmaes", maximize_cmaes)
    return cls
