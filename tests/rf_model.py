"""Exact numpy restatement of the device random forest (robo_b200/csrc/gpk_rf.cuh) — TEST INFRASTRUCTURE ONLY.

pyrfr, the library robo/models/random_forest.py wraps, is not available, so the forest is stated here and in gpk_rf.cuh:

* Sample per tree.  Tree t draws n_t rows (n_t = n_points_per_tree, or N when 0).  Draw j is Philox4x32-10 with key
  (seed low, seed high) and counter (j, t, train counter, tag); its first word w becomes an index below m as
  floor(w m / 2^32), exact in integers, so it never rounds up to m.  Bootstrap (TAG_BOOT): row floor(w N / 2^32), with
  replacement.  Otherwise (TAG_PERM): the first n_t steps of a Fisher-Yates shuffle, step j swapping p[j] and
  p[j + floor(w (N - j) / 2^32)]; rows p[:n_t] once each.
* Growth (CART, residual sum of squares, every feature at every node).  A node is a leaf when it holds fewer than 2
  samples (with multiplicity), when fl(max y - min y) <= 1e-8, or when no feature takes two values in it.  Otherwise for
  each feature f the samples are ordered by (x_f, row index) and W_l, S, Q are the running count, sum of y and sum of
  fl(y y) (running sums from 0.0, left to right); S_t, Q_t are the same sums over the node's samples in ascending row order.  A
  candidate after position k where x_f[k] < x_f[k+1] has loss fl(Q - fl(S S) / W_l) + fl(fl(Q_t - Q) - fl(S_r S_r) / W_r),
  S_r = S_t - S, W_r = W - W_l.  The least loss wins under strict < over features ascending, then positions.  The
  threshold is fl(fl(x_k + x_{k+1}) / 2), x_k where that equals x_{k+1}; a row goes left iff x_f <= threshold.
* Leaves: W, mean = S_t / W, var = (sum of fl((y - mean)^2), rows ascending with multiplicity, sequential) / W.
* Nodes are numbered breadth first; the children of a level's split nodes follow in the level's order, left first.
* Moments: mean = (sum of m_t in ascending t) / T; var = (sum of (m_t - mean)^2) / T, plus (sum of v_t) / T when the
  total variance is asked for; every sum sequential.
"""
import numpy as np

from tests.de_model import _philox

TAG_BOOT, TAG_PERM = 0x52460001, 0x52460002
PURITY = 1e-8
FIELDS = ("feat", "thr", "left", "W", "mean", "var")


def index(w, m):
    """floor(w m / 2^32) for 32-bit draws w: an index below m."""
    return ((np.asarray(w, dtype=np.uint64) * np.uint64(m)) >> np.uint64(32)).astype(np.int64)


def multiplicities(seed, counter, t, N, nt, bootstrap):
    """How often each of the N rows is in tree t's sample."""
    if bootstrap:
        j = np.arange(nt, dtype=np.uint64)
        w = _philox(seed, j, t, counter, TAG_BOOT)[0]
        return np.bincount(index(w, N), minlength=N)
    if nt > N:
        raise ValueError("n_points_per_tree > N without bootstrapping")
    w = _philox(seed, np.arange(nt, dtype=np.uint64), t, counter, TAG_PERM)[0]
    p = np.arange(N)
    cnt = np.zeros(N, dtype=np.int64)
    for j in range(nt):
        k = j + int(index(w[j], N - j))
        p[j], p[k] = p[k], p[j]
        cnt[p[j]] = 1
    return cnt


def _cumsum(v):
    """Running sums from 0.0, as the device accumulates them (np.cumsum alone starts at v[0], which keeps a -0.0)."""
    return np.cumsum(np.concatenate(([0.0], v)))[1:]


def _seqsum(v):
    return _cumsum(v)[-1] if len(v) else 0.0


def _best_split(X, y, rows, cnt, St, Qt, W):
    """(loss, feature, threshold) of the winning split, or None."""
    best = None
    for f in range(X.shape[1]):
        o = rows[np.lexsort((rows, X[rows, f]))]
        rep = np.repeat(o, cnt[o])
        ys, xs = y[rep], X[rep, f]
        cS = _cumsum(ys)
        cQ = _cumsum(ys * ys)
        Wl = np.arange(1, W + 1, dtype=np.float64)
        k = np.flatnonzero(xs[:-1] < xs[1:])
        if k.size == 0:
            continue
        Sr = St - cS[k]
        loss = (cQ[k] - cS[k] * cS[k] / Wl[k]) + ((Qt - cQ[k]) - Sr * Sr / (W - Wl[k]))
        ok = ~np.isnan(loss)
        if not ok.any():
            continue
        mn = loss[ok].min()
        if best is None and mn < np.inf or best is not None and mn < best[0]:
            i = k[np.flatnonzero(loss == mn)[0]]
            a, b = xs[i], xs[i + 1]
            th = (a + b) / 2.0
            if th == b:
                th = a
            best = (mn, f, th)
    return best


def grow(X, y, cnt):
    """One tree on the rows with multiplicities cnt: dict of node arrays (FIELDS) in breadth-first order."""
    X, y = np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64)
    nodes = [np.flatnonzero(cnt > 0)]
    out = {k: [] for k in FIELDS}
    lo = 0
    while lo < len(nodes):
        hi = len(nodes)
        for v in range(lo, hi):
            rows = nodes[v]
            rep = np.repeat(rows, cnt[rows])
            ys = y[rep]
            W = len(rep)
            St, Qt = _seqsum(ys), _seqsum(ys * ys)
            split = None
            if W >= 2 and not (ys.max() - ys.min() <= PURITY):
                split = _best_split(X, y, rows, cnt, St, Qt, W)
            if split is None:
                mu = St / float(W)
                var = _seqsum((ys - mu) ** 2) / float(W)
                for k, val in zip(FIELDS, (-1, 0.0, -1, float(W), mu, var)):
                    out[k].append(val)
            else:
                _, f, th = split
                for k, val in zip(FIELDS, (f, th, len(nodes), 0.0, 0.0, 0.0)):
                    out[k].append(val)
                go = X[rows, f] <= th
                nodes.append(rows[go])
                nodes.append(rows[~go])
        lo = hi
    return {k: np.array(v, dtype=np.int32 if k in ("feat", "left") else np.float64) for k, v in out.items()}


def fit(X, y, seed, counter, num_trees, n_per_tree=0, bootstrap=True):
    """The forest gpk_rf_fit grows: a list of trees (grow's dicts)."""
    N = len(y)
    nt = n_per_tree if n_per_tree > 0 else N
    return [grow(X, y, multiplicities(seed, counter, t, N, nt, bootstrap)) for t in range(num_trees)]


def leaves(tree, X):
    """The leaf index of every row of X in one tree."""
    X = np.atleast_2d(np.asarray(X, dtype=np.float64))
    v = np.zeros(len(X), dtype=np.int64)
    while True:
        f = tree["feat"][v]
        inner = f >= 0
        if not inner.any():
            return v
        i = np.flatnonzero(inner)
        right = X[i, f[i]] > tree["thr"][v[i]]
        v[i] = tree["left"][v[i]] + right


def each_tree(forest, X):
    """(m (T, M), v (T, M)): every tree's leaf mean and variance at the rows of X."""
    L = [leaves(t, X) for t in forest]
    return (np.array([t["mean"][l] for t, l in zip(forest, L)]), np.array([t["var"][l] for t, l in zip(forest, L)]))


def predict(forest, X, total_variance=True):
    """The forest's (mean, var) at the rows of X, sums in ascending tree order."""
    m, v = each_tree(forest, X)
    T = float(len(forest))
    sm = np.zeros(m.shape[1])
    sv = np.zeros(m.shape[1])
    for t in range(len(forest)):
        sm = sm + m[t]
        sv = sv + v[t]
    mean = sm / T
    sq = np.zeros(m.shape[1])
    for t in range(len(forest)):
        e = m[t] - mean
        sq = sq + e * e
    var = sq / T
    if total_variance:
        var = var + sv / T
    return mean, var


def pack(forest, slots):
    """The forest as gpk_rf_get_trees returns it: n_nodes (T,) and (T, slots) arrays, zero past n_nodes."""
    T = len(forest)
    out = {k: np.zeros((T, slots), dtype=np.int32 if k in ("feat", "left") else np.float64) for k in FIELDS}
    for t, tree in enumerate(forest):
        for k in FIELDS:
            out[k][t, :len(tree[k])] = tree[k]
    out["n_nodes"] = np.array([len(t["feat"]) for t in forest], dtype=np.int32)
    return out


def unpack(trees):
    """pack's inverse: the list of per-tree dicts."""
    return [{k: trees[k][t, :trees["n_nodes"][t]].copy() for k in FIELDS} for t in range(len(trees["n_nodes"]))]
