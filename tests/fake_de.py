"""``_lib.maximize_de`` on the oracle-backed FakeHandle (tests/fake_gpk.py) — TEST INFRASTRUCTURE ONLY.

The evolution is tests/de_model.py, the exact restatement of gpk_maximize_de; the acquisition values come from the
fake handles (the oracle), averaged over the models like gpk_acq_multi mode 0.  Argument checks mirror the C side's
GPK_BAD_ARG cases as ValueError."""
import numpy as np

from tests import de_model, fake_gpk


def maximize_de(handles, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper, kind, eta, par=0.0,
                want_population=False):
    lower, upper = np.asarray(lower, dtype=np.float64).ravel(), np.asarray(upper, dtype=np.float64).ravel()
    if not 5 <= pop <= 1 << 24 or not 0 <= mutation[0] <= mutation[1] < 2 or not 0 <= recombination <= 1 \
            or maxiter < 0 or not np.all(lower < upper) or kind not in (1, 2, 3, 4) or len(set(map(id, handles))) != len(handles):
        raise ValueError("gpk_maximize_de: bad arguments")
    etas = np.broadcast_to(np.asarray(eta, dtype=np.float64), (len(handles),))
    n_negative = [0]

    def acq_fn(X):
        rs = [h.acq(X, kind, float(e), par) for h, e in zip(handles, etas)]
        n_negative[0] += sum(r["n_negative"] for r in rs)
        return np.mean([r["values"] for r in rs], axis=0)

    r = de_model.maximize_de(acq_fn, seed, int(pop), lower, upper, int(maxiter), tuple(map(float, mutation)),
                             float(recombination), float(tol), float(atol))
    out = dict(x=r["x"], energy=r["energy"], nit=r["nit"], nfev=r["nfev"], n_negative=n_negative[0])
    if want_population:
        out.update(population=r["population"], energies=r["energies"])
    return out


def install(monkeypatch):
    """fake_gpk.install plus the differential-evolution entry point."""
    from robo_b200 import _lib
    cls = fake_gpk.install(monkeypatch)
    monkeypatch.setattr(_lib, "maximize_de", maximize_de)
    return cls
