"""Exact restatement of gpk_maximize_direct (robo_b200/csrc/gpk_direct.cuh) — TEST INFRASTRUCTURE ONLY.

Jones' original DIRECT as Gablonsky's DIRECT 2.0.4 runs it with the `DIRECT` package's defaults (algmethod = 0,
eps = 1e-4, fglobal = -1e100, fglper = 0.01, volume and length stops off), in the kernels' operation order: the same
rectangle store (unit-cube centres, trisection counts, energies), the same level lists kept sorted by energy, the same
selection (the head of every level on the lower-right hull that passes Jones' test, then every rectangle within 1e-13
of a selected head at its level), the same batch of sample points per iteration, and the same division and
insertion.  Python floats are IEEE doubles rounded to nearest, so every sum and product below is the device's
__dadd_rn / __dmul_rn / __ddiv_rn.

``run(score, lower, upper, maxf, maxT)`` calls ``score(rows)`` once per batch (the centre first, then the 2d initial
points, then one batch per iteration) with rows already mapped to the box, and expects the energies e = -acq(rows).
Non-finite energies follow the device's rule: NaN is stored as +inf; +inf and -inf are kept.
"""
import math

import numpy as np

EPS = 1e-4                 # Jones' epsilon (epsrel; epsabs = 0)
TIE = 1e-13                # DIRDoubleInsert: f(pos) - f(head) <= 1e-13 joins the head
MAXDEEP = 600              # levels 0 .. MAXDEEP - 1; dividing a rectangle at level >= MAXDEEP - 1 ends the run
MAXDIV = 5000              # most rectangles one iteration selects; more (exact ties) end the run before it samples
FGLOBAL, FGLPER = -1e100, 0.01

RUNNING, MAXF, MAXT, FGLOBAL_HIT, DEPTH, MAXDIV_HIT = range(6)
STOP_NAMES = ("running", "maxf", "maxT", "fglobal", "maxdeep", "maxdiv")


def tables(n):
    """(levels, thirds): levels[n k + j] = 0.5 sqrt(n - j + j / 9) / 3^k, the centre-to-vertex distance of a
    rectangle with j sides trisected k + 1 times and n - j sides k times; thirds[k] = 1 / 3^k."""
    w = [0.5 * math.sqrt(n - j + j / 9.0) for j in range(n)]
    levels = [0.0] * (MAXDEEP + n)
    help2 = 1.0
    for i in range((MAXDEEP + n) // n + 1):
        for j in range(n):
            if i * n + j < len(levels):
                levels[i * n + j] = w[j] / help2
        help2 = help2 * 3.0
    thirds = [1.0] * (MAXDEEP + 2)
    help2 = 3.0
    for i in range(1, MAXDEEP + 2):
        thirds[i] = 1.0 / help2
        help2 = help2 * 3.0
    return levels, thirds


def level_of(ln):
    """DIRGetlevel for jones = 0: n k + (number of sides at k + 1), written as Gablonsky counts it."""
    n = len(ln)
    help_ = ln[0]
    k = help_
    p = 1
    for i in range(1, n):
        if ln[i] < k:
            k = ln[i]
        if ln[i] == help_:
            p += 1
    return n * k + n - p if k == help_ else n * k + p


def clean(e):
    e = float(e)
    return math.inf if e != e else e


class _Store:
    def __init__(self, n, lower, upper):
        self.n = n
        self.c, self.ln, self.f, self.nxt = [], [], [], []
        self.anchor = {}
        self.span = [float(u) - float(l) for l, u in zip(lower, upper)]          # c2 = u - l
        self.shift = [float(l) / s for l, s in zip(lower, self.span)]            # c1 = l / (u - l)

    def box(self, c):
        return [(ci + a) * b for ci, a, b in zip(c, self.shift, self.span)]      # (c + c1) c2

    def result_x(self, c):
        return [ci * b + a * b for ci, a, b in zip(c, self.shift, self.span)]    # c c2 + c1 c2

    def add(self, c, ln):
        self.c.append(c)
        self.ln.append(ln)
        self.f.append(math.inf)
        self.nxt.append(-1)
        return len(self.c) - 1

    def insert_after(self, start, ins):
        """DIRInsert: behind start, before the first successor with a strictly larger energy."""
        f = self.f
        while True:
            nx = self.nxt[start]
            if nx < 0:
                self.nxt[start] = ins
                self.nxt[ins] = -1
                return
            if f[ins] < f[nx]:
                self.nxt[start] = ins
                self.nxt[ins] = nx
                return
            start = nx

    def insert_pair(self, pos1, pos2):
        """DIRInsertList for one (+, -) pair of children, as Gablonsky orders them."""
        f, anchor, nxt = self.f, self.anchor, self.nxt
        deep = level_of(self.ln[pos1])
        head = anchor.get(deep, -1)
        if head < 0:
            if f[pos2] < f[pos1]:
                anchor[deep] = pos2
                nxt[pos2] = pos1
                nxt[pos1] = -1
            else:
                anchor[deep] = pos1
                nxt[pos1] = pos2
                nxt[pos2] = -1
            return
        pos = head
        if f[pos2] < f[pos1]:
            if f[pos2] < f[pos]:
                anchor[deep] = pos2
                if f[pos1] < f[pos]:
                    nxt[pos2] = pos1
                    nxt[pos1] = pos
                else:
                    nxt[pos2] = pos
                    self.insert_after(pos, pos1)
            else:
                self.insert_after(pos, pos2)
                self.insert_after(pos, pos1)
        else:
            if f[pos1] < f[pos]:
                anchor[deep] = pos1
                if f[pos] < f[pos2]:
                    nxt[pos1] = pos
                    self.insert_after(pos, pos2)
                else:
                    nxt[pos1] = pos2
                    nxt[pos2] = pos
            else:
                self.insert_after(pos, pos1)
                self.insert_after(pos, pos2)

    def insert_one(self, samp):
        deep = level_of(self.ln[samp])
        pos = self.anchor.get(deep, -1)
        if pos < 0:
            self.anchor[deep] = samp
            self.nxt[samp] = -1
        elif self.f[samp] < self.f[pos]:
            self.anchor[deep] = samp
            self.nxt[samp] = pos
        else:
            self.insert_after(pos, samp)

    def remove(self, deep, r):
        if self.anchor[deep] == r:
            self.anchor[deep] = self.nxt[r]
            if self.anchor[deep] < 0:
                del self.anchor[deep]
        else:
            p = self.anchor[deep]
            while self.nxt[p] != r:
                p = self.nxt[p]
            self.nxt[p] = self.nxt[r]


def choose(st, levels, minf):
    """DIRChoose + DIRDoubleInsert: [(rectangle, level)] in processing order.  S holds the head of every non-empty
    level in ascending level (descending size); j runs from the smallest rectangle up.  Against the larger heads
    (all of them) j needs every slope h = (f_i - f_j) / (d_i - d_j) > 0 and takes K = their minimum (+inf when there
    are none); against the smaller heads still kept it needs every h > 0 and takes G = their maximum.  Then
    G > K keeps j without the epsilon test (as scipy's translation runs, see gpk_direct.cuh), otherwise j is kept
    when f_j - K d_j <= min(minf - eps |minf|, minf) or that difference is NaN.  NaN slopes are skipped."""
    f = st.f
    S = [[st.anchor[lv], lv] for lv in sorted(st.anchor)]
    thresh = min(minf - EPS * abs(minf), minf - 0.0)
    for j in range(len(S) - 1, -1, -1):
        fj, dj = f[S[j][0]], levels[S[j][1]]
        lower, greater, keep = math.inf, 0.0, True
        for i in range(j):
            h = (f[S[i][0]] - fj) / (levels[S[i][1]] - dj)
            if h <= 0.0:
                keep = False
                break
            if h < lower:
                lower = h
        if keep:
            for i in range(j + 1, len(S)):
                if S[i][0] >= 0:
                    h = (f[S[i][0]] - fj) / (levels[S[i][1]] - dj)
                    if h <= 0.0:
                        keep = False
                        break
                    if h > greater:
                        greater = h
        if keep and lower >= greater:
            keep = not (fj - lower * dj > thresh)
        if not keep:
            S[j][0] = -1
    out = [(r, lv) for r, lv in S if r >= 0]
    for r, lv in list(out):
        pos = st.nxt[r]
        while pos >= 0 and f[pos] - f[r] <= TIE:
            out.append((pos, lv))
            pos = st.nxt[pos]
    return out


def run(score, lower, upper, maxf, maxT):
    """One whole run -> dict(x, fun, nfev, nit, stop, rows (per iteration, the first two batches excluded),
    points (every scored row in order))."""
    lower = [float(v) for v in np.asarray(lower, dtype=np.float64).ravel()]
    upper = [float(v) for v in np.asarray(upper, dtype=np.float64).ravel()]
    n = len(lower)
    levels, thirds = tables(n)
    st = _Store(n, lower, upper)
    points, rows_per_iter = [], []

    def evaluate(rects):
        X = np.array([st.box(st.c[r]) for r in rects], dtype=np.float64).reshape(len(rects), n)
        e = np.asarray(score(X), dtype=np.float64).ravel()
        points.append(X)
        for r, v in zip(rects, e):
            st.f[r] = clean(v)

    root = st.add([0.5] * n, [0] * n)
    evaluate([root])
    minf, minpos = st.f[root], root
    nfev = 1

    def sample(parent):
        """DIRSamplepoints: 2 maxI children of ``parent`` over its longest sides, + before -."""
        ln = st.ln[parent]
        k = min(ln)
        dims = [i for i in range(n) if ln[i] == k]
        delta = thirds[k + 1]
        kids = []
        for i in dims:
            for sgn in (1.0, -1.0):
                c = list(st.c[parent])
                c[i] = c[i] + delta if sgn > 0 else c[i] - delta
                kids.append(st.add(c, list(ln)))
        return dims, k, kids

    def divide(parent, dims, k, kids):
        """DIRDivide + DIRInsertList: trisect in ascending w = min(f+, f-), ties by dimension."""
        f = st.f
        w = [f[kids[2 * a + 1]] if f[kids[2 * a + 1]] <= f[kids[2 * a]] else f[kids[2 * a]] for a in range(len(dims))]
        order = []
        for a in range(len(dims)):                       # DIRInsertList_2: stable insertion by strict <
            p = 0
            while p < len(order) and not (w[a] < w[order[p]]):
                p += 1
            order.insert(p, a)
        for t, a in enumerate(order):
            i = dims[a]
            st.ln[parent][i] = k + 1
            for b in order[t:]:
                st.ln[kids[2 * b]][i] = k + 1
                st.ln[kids[2 * b + 1]][i] = k + 1
        for a in range(len(dims)):
            st.insert_pair(kids[2 * a], kids[2 * a + 1])
        st.insert_one(parent)

    def incumbent(rects):
        nonlocal minf, minpos
        for r in rects:
            if st.f[r] < minf:
                minf, minpos = st.f[r], r

    dims, k, kids = sample(root)
    evaluate(kids)
    incumbent(kids)
    divide(root, dims, k, kids)
    nfev += len(kids)

    t, stop = 2, RUNNING
    while True:
        if t >= maxT:                    # iterations 2 .. maxT - 1 sample; nit = maxT (at least 2)
            stop = MAXT
            break
        S = choose(st, levels, minf)
        if len(S) > MAXDIV:
            rows_per_iter.append(0)
            stop = MAXDIV_HIT
            break
        work, depth = [], False
        for r, lv in S:
            if lv + 1 >= MAXDEEP:
                depth = True
                break
            work.append((r, lv) + sample(r))
        batch = [c for w_ in work for c in w_[4]]
        rows_per_iter.append(len(batch))
        if batch:
            evaluate(batch)
        for r, lv, dims, k, kids in work:
            st.remove(lv, r)
            incumbent(kids)
            divide(r, dims, k, kids)
        nfev += len(batch)
        if depth:
            stop = DEPTH
        elif (minf - FGLOBAL) * 100.0 / abs(FGLOBAL) <= FGLPER:
            stop = FGLOBAL_HIT
        elif nfev >= maxf:
            stop = MAXF
        if stop != RUNNING:
            break
        t += 1
    x = np.array(st.result_x(st.c[minpos]), dtype=np.float64)
    return dict(x=x, c=np.array(st.c[minpos]), fun=minf, nfev=nfev, nit=t, stop=stop, rows=rows_per_iter,
                points=np.concatenate(points, axis=0))
