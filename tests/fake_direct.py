"""``_lib.maximize_direct`` on the oracle-backed FakeHandle (tests/fake_gpk.py) — TEST INFRASTRUCTURE ONLY.

The search is tests/direct_model.py, the exact restatement of gpk_maximize_direct; the acquisition values come from
the fake handles (the oracle), averaged over the models like gpk_acq_multi mode 0.  Argument checks mirror the C
side's GPK_BAD_ARG cases as ValueError."""
import numpy as np

from robo_b200 import _lib
from tests import direct_model, fake_gpk


def maximize_direct(handles, kind, eta, par, lower, upper, n_func_evals=400, n_iters=200):
    lower, upper = np.asarray(lower, dtype=np.float64).ravel(), np.asarray(upper, dtype=np.float64).ravel()
    d = lower.size
    if not 1 <= d <= _lib.DIRECT_MAX_D or lower.size != upper.size or not np.all(lower < upper) \
            or not np.all(np.isfinite(lower)) or not np.all(np.isfinite(upper)) or n_func_evals < 1 or n_iters < 1 \
            or (2 * d + 1) * max(n_func_evals, 2 * d + 1) > _lib.DIRECT_MAX_RECTS or kind not in (1, 2, 3, 4) \
            or len(set(map(id, handles))) != len(handles):
        raise ValueError("gpk_maximize_direct: bad arguments")
    etas = np.broadcast_to(np.asarray(eta, dtype=np.float64), (len(handles),))
    n_negative = [0]

    def energies(X):
        rs = [h.acq(X, kind, float(e), par) for h, e in zip(handles, etas)]
        n_negative[0] += sum(r["n_negative"] for r in rs)
        return -np.mean([r["values"] for r in rs], axis=0)

    r = direct_model.run(energies, lower, upper, int(n_func_evals), int(n_iters))
    return dict(x=r["x"], energy=r["fun"], nit=r["nit"], nfev=r["nfev"], stop=r["stop"],
                rows=np.asarray(r["rows"], dtype=np.int64), n_negative=n_negative[0])


def install(monkeypatch):
    """fake_gpk.install plus the DIRECT entry point."""
    cls = fake_gpk.install(monkeypatch)
    monkeypatch.setattr(_lib, "maximize_direct", maximize_direct)
    return cls
