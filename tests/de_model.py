"""Exact numpy restatement of gpk_maximize_de (robo_b200/csrc/gpk_de.cuh) — TEST INFRASTRUCTURE ONLY.

scipy.optimize.differential_evolution with strategy 'best1bin', updating='deferred' and Latin-hypercube
initialisation, driven by the library's counter-based Philox stream.  Every rounding step follows the kernels: numpy's
elementwise float64 operations round each product and sum once, like the kernels' __dmul_rn / __dadd_rn, and mean /
std use the kernels' fixed summation order.  Given the same acquisition values the population, the energies, nit and
nfev are the device's bit for bit.  The acquisition is pluggable: ``acq_fn(X)`` maps a (pop, d) batch of scaled,
clipped parameters to acquisition values (the energy is -acq, infinities replaced by DBL_MAX)."""
import numpy as np

from oracle.robo_oracle import philox4x32_10

TAG_INIT, TAG_GEN = 0x44450001, 0x44450002
RED = 1024                                   # threads of gpk_de_finish_kernel: fixes the summation order
DBL_MAX = np.finfo(np.float64).max
_U32 = np.uint64(0xFFFFFFFF)


def _philox(seed, c0, c1, c2, c3):
    c0, c1, c2, c3 = np.broadcast_arrays(*[np.asarray(c, dtype=np.uint64) for c in (c0, c1, c2, c3)])
    return philox4x32_10(c0, c1, c2, c3, int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF)


def _u01(lo, hi):
    return ((hi << np.uint64(32) | lo) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def _mulshift(w, n):
    return ((w * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def limits(lower, upper):
    """(lower, upper, arg1, arg2) of scipy's _scale_parameters."""
    lower, upper = np.asarray(lower, dtype=np.float64), np.asarray(upper, dtype=np.float64)
    return lower, upper, 0.5 * (lower + upper), np.fabs(lower - upper)


def scale(U, lim):
    """clip(arg1 + (u - 0.5) arg2, lower, upper): the parameters scoring sees."""
    lower, upper, arg1, arg2 = lim
    return np.fmin(np.fmax(arg1 + (U - 0.5) * arg2, lower), upper)


def energy(acq_values):
    e = -np.asarray(acq_values, dtype=np.float64)
    return np.where(np.isinf(e), DBL_MAX, e)


def init_population(seed, pop, d):
    """Latin hypercube: member i's stratum in column j is the rank of its Philox key among the column's keys (ties by
    member index); its coordinate is fl(fl(seg u) + fl(rank seg)), seg = 1 / pop."""
    i = np.arange(pop, dtype=np.uint64)[None, :]
    j = np.arange(d, dtype=np.uint64)[:, None]
    r0, _, r2, r3 = _philox(seed, i, 0, j, TAG_INIT)                  # (d, pop)
    order = np.argsort((r0 << np.uint64(24)) | i, axis=1, kind="stable")
    rank = np.empty((d, pop), dtype=np.int64)
    np.put_along_axis(rank, order, np.arange(pop, dtype=np.int64)[None, :], axis=1)
    seg = 1.0 / pop
    return (seg * _u01(r2, r3) + rank.astype(np.float64) * seg).T.copy()


def promote(P, E):
    """numpy.argmin (first minimum, NaN first) swapped into slot 0 with its row."""
    b = int(np.argmin(E))
    if b > 0:
        P[[0, b]] = P[[b, 0]]
        E[[0, b]] = E[[b, 0]]
    return b


def _tree_sum(terms):
    pop = terms.size
    acc = np.zeros(RED)
    padded = np.zeros(-(-pop // RED) * RED)
    padded[:pop] = terms
    for row in padded.reshape(-1, RED):
        acc = acc + row
    s = RED // 2
    while s > 0:
        acc[:s] = acc[:s] + acc[s:2 * s]
        s //= 2
    return acc[0]


def stats(E):
    """mean and std of E in gpk_de_finish_kernel's order."""
    pop = E.size
    with np.errstate(over="ignore", invalid="ignore"):          # DBL_MAX energies overflow the squares, as on the device
        mean = _tree_sum(E) / pop
        q = E - mean
        return mean, np.sqrt(_tree_sum(q * q) / pop)


def trial(seed, g, P, mutation, recombination, details=False):
    """Generation g >= 1: best1bin trials of every member (unit cube)."""
    pop, d = P.shape
    f0, f1, _, _ = _philox(seed, 0, g, 0xFFFFFFFF, TAG_GEN)
    F = mutation[0] + (mutation[1] - mutation[0]) * float(_u01(f0, f1))
    i = np.arange(pop, dtype=np.int64)
    w0, w1, w2, _ = _philox(seed, i.astype(np.uint64), g, 0, TAG_GEN)
    r0 = _mulshift(w0, pop - 1)
    r0 += r0 >= i
    r1 = _mulshift(w1, pop - 2)
    a, b = np.minimum(i, r0), np.maximum(i, r0)
    r1 += r1 >= a
    r1 += r1 >= b
    fill = _mulshift(w2, d)
    c0, c1, c2, c3 = _philox(seed, i.astype(np.uint64)[:, None], g, 1 + np.arange(d, dtype=np.uint64)[None, :], TAG_GEN)
    bprime = P[0][None, :] + F * (P[r0] - P[r1])
    cross = (_u01(c0, c1) < recombination) | (np.arange(d)[None, :] == fill[:, None])
    T = np.where(cross, bprime, P)
    crossed = T.copy()
    out = (T > 1.0) | (T < 0.0)
    T[out] = _u01(c2, c3)[out]
    if details:
        return T, dict(F=F, r0=r0, r1=r1, fill=fill, bprime=bprime, cross=cross, crossed=crossed)
    return T


def maximize_de(acq_fn, seed, pop, lower, upper, maxiter, mutation=(0.5, 1.0), recombination=0.7, tol=0.01, atol=0.0,
                trace=None):
    """The whole run.  -> dict(x, energy, nit, nfev, population, energies).  ``trace`` (a list) receives the best
    energy after the initial population and after every generation."""
    lim = limits(lower, upper)
    d = lim[0].size
    P = init_population(seed, pop, d)
    E = energy(acq_fn(scale(P, lim)))
    promote(P, E)
    nfev, nit = pop, 0
    if trace is not None:
        trace.append(E[0])
    for g in range(1, maxiter + 1):
        T = trial(seed, g, P, mutation, recombination)
        e = energy(acq_fn(scale(T, lim)))
        acc = e <= E
        P[acc] = T[acc]
        E[acc] = e[acc]
        promote(P, E)
        nfev += pop
        nit = g
        if trace is not None:
            trace.append(E[0])
        mean, std = stats(E)
        if std <= atol + tol * np.abs(mean):
            break
    return dict(x=scale(P[0], lim), energy=float(E[0]), nit=nit, nfev=nfev, population=P, energies=E)
