"""The information-gain entry points of ``_lib`` on the oracle-backed FakeHandle (tests/fake_gpk.py, tests/fake_de.py) —
TEST INFRASTRUCTURE ONLY.

The fake handle gains gpk_es_update / gpk_es_compute with a stand-in for the entropy change: the oracle's predictive
variance of the candidate (DBL_EPSILON outside gpk_es_update's [lower, upper]), which keeps the host logic's contract
(ValueError before gpk_es_update or after a refit, "lmb should not be infinite.") without restating EP.  gpk_es_multi,
gpk_es_cost_multi and the two evolutions are built on it as the library builds them: the mean over the handles, the
Fabolas transform and ratio, and tests/de_model.py for the evolution.  Argument checks mirror the C side's GPK_BAD_ARG
cases as ValueError."""
import numpy as np

from tests import de_model, fake_de, fabolas_acq_model as F


def es_update(self, zb, lmb, sn2, W, lower, upper):
    if not np.all(np.isfinite(lmb)):
        raise ValueError("lmb should not be infinite.")
    nb = np.asarray(zb).shape[0]
    self.es_state = (np.asarray(lower, float).ravel(), np.asarray(upper, float).ravel(), self.L)
    return dict(logP=np.full(nb, -np.log(nb)), dlogPdMu=np.zeros((nb, nb)),
                dlogPdSigma=np.zeros((nb, nb * (nb + 1) // 2)), dlogPdMudMu=np.zeros((nb, nb, nb)))


def _dh(self, Xm, Xb):
    state = getattr(self, "es_state", None)
    if state is None:
        raise ValueError("gpk_es_compute: call gpk_es_update first")
    lower, upper, L = state
    if L is not self.L:
        raise ValueError("gpk_es_compute: the model changed since gpk_es_update")
    _, var = self.predict(Xm)
    inside = np.all((Xb >= lower) & (Xb <= upper), axis=1)
    return np.where(inside, var, F.EPS)


def es_compute(self, Xs):
    Xs = np.asarray(Xs, dtype=np.float64)
    return _dh(self, Xs, Xs)


def _distinct(handles):
    if len(handles) == 0 or len(set(map(id, handles))) != len(handles):
        raise ValueError("need distinct handles")


def es_multi(objective, Xs, want_values=True):
    _distinct(objective)
    vals = np.mean([h.es_compute(Xs) for h in objective], axis=0)
    return dict(values=vals if want_values else None, best_val=float(np.max(vals)), best_idx=int(np.argmax(vals)))


def _transform(X, lower, upper, basis):
    T = np.array(X, dtype=np.float64)
    T[:, :-1] = (T[:, :-1] - lower) / (upper - lower)
    s = T[:, -1]
    T[:, -1] = s if basis == 0 else (1 - s) ** 2
    return T


def es_cost_multi(objective, cost, Xs, lower, upper, basis_objective, basis_cost, overhead, want_values=True):
    _distinct(list(objective) + list(cost))
    lower, upper = np.asarray(lower, float).ravel(), np.asarray(upper, float).ravel()
    Xs = np.asarray(Xs, dtype=np.float64)
    if len(objective) != len(cost) or basis_objective not in (0, 1) or basis_cost not in (0, 1) \
            or lower.size != Xs.shape[1] - 1 or not np.all(lower < upper):
        raise ValueError("gpk_es_cost_multi: bad arguments")
    Xo, Xc = _transform(Xs, lower, upper, basis_objective), _transform(Xs, lower, upper, basis_cost)
    vals = np.mean([F.per_unit_cost(_dh(o, Xo, Xs), c.predict(Xc)[0], overhead) for o, c in zip(objective, cost)],
                   axis=0)
    return dict(values=vals if want_values else None, best_val=float(np.max(vals)), best_idx=int(np.argmax(vals)))


def _evolve(acq_fn, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper, want_population):
    lower, upper = np.asarray(lower, dtype=np.float64).ravel(), np.asarray(upper, dtype=np.float64).ravel()
    if not 5 <= pop <= 1 << 24 or not 0 <= mutation[0] <= mutation[1] < 2 or not 0 <= recombination <= 1 \
            or maxiter < 0 or not np.all(lower < upper):
        raise ValueError("gpk_maximize_de_es: bad arguments")
    r = de_model.maximize_de(acq_fn, seed, int(pop), lower, upper, int(maxiter), tuple(map(float, mutation)),
                             float(recombination), float(tol), float(atol))
    out = dict(x=r["x"], energy=r["energy"], nit=r["nit"], nfev=r["nfev"])
    if want_population:
        out.update(population=r["population"], energies=r["energies"])
    return out


def maximize_de_es(objective, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper,
                   want_population=False):
    _distinct(objective)
    acq_fn = objective[0].es_compute if len(objective) == 1 else (lambda X: es_multi(objective, X)["values"])
    return _evolve(acq_fn, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper, want_population)


def maximize_de_es_cost(objective, cost, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper,
                        cfg_lower, cfg_upper, basis_objective, basis_cost, overhead, want_population=False):
    def acq_fn(X):
        return es_cost_multi(objective, cost, X, cfg_lower, cfg_upper, basis_objective, basis_cost, overhead)["values"]
    return _evolve(acq_fn, seed, pop, maxiter, mutation, recombination, tol, atol, lower, upper, want_population)


def install(monkeypatch):
    """fake_de.install plus the information-gain entry points."""
    from robo_b200 import _lib
    cls = fake_de.install(monkeypatch)
    monkeypatch.setattr(cls, "es_update", es_update, raising=False)
    monkeypatch.setattr(cls, "es_compute", es_compute, raising=False)
    for name, fn in (("es_multi", es_multi), ("es_cost_multi", es_cost_multi), ("maximize_de_es", maximize_de_es),
                     ("maximize_de_es_cost", maximize_de_es_cost)):
        monkeypatch.setattr(_lib, name, fn)
    return cls
