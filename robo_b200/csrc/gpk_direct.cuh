// gpk_direct.cuh — device-resident DIRECT for gpk_maximize_direct*: Jones' original DIRECT (algmethod = 0) as
// Gablonsky's DIRECT 2.0.4 runs it for robo/maximizers/direct.py:56-85 (DIRECT.solve with maxT = n_iters,
// maxf = n_func_evals, eps = 1e-4, fglobal = -1e100, fglper = 0.01, volume and length stops off), minimising the
// energy e = -acq of the reference's _direct_acquisition_fkt_wrapper.
//
// Every point an iteration samples is known once its potentially optimal rectangles are chosen, so an iteration is
// one selection CTA, one batched scoring pass over every row it samples, and one division CTA.  The bookkeeping is
// Gablonsky's, restated in his order: the rectangle store (unit-cube centre, trisection count per dimension,
// energy), one list per level sorted by energy (DIRInsertList / DIRInsert, whose tie order decides which rectangle
// heads a level), DIRChoose over the level heads, DIRDoubleInsert for the rectangles within 1e-13 of a chosen head,
// DIRSamplepoints (c +- delta e_i over the longest sides, + before -, ascending i), DIRDivide (ascending
// w_i = min(e(c + delta e_i), e(c - delta e_i)), ties by dimension) and the incumbent update (strictly lower wins).
// The selection follows scipy.optimize.direct's C translation of that code, the executable restatement of the
// package: a rectangle whose lower slope bound K exceeds its upper bound G is kept without the epsilon test there.
//
// Every sum, product and quotient is rounded explicitly (__dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn /
// __dsqrt_rn: nothing is contracted) and every loop runs in Gablonsky's order, so tests/direct_model.py restates a
// whole run bit for bit.  The list work is sequential by nature and runs on one thread; the rows of a batch are
// written by the whole CTA.
//
// Non-finite energies: NaN is stored as +inf (it never becomes the incumbent, and it sorts last in its level);
// +inf and -inf are kept.  -inf as the incumbent ends the run on the fglobal test.
#pragma once
#include "gpk_internal.cuh"

#define GPK_DIRECT_LEVELS (GPK_DIRECT_MAXDEEP + GPK_DIRECT_MAX_D)   // level indices a rectangle can reach
#define GPK_DIRECT_THREADS 256
#define GPK_DIRECT_EPS 1e-4
#define GPK_DIRECT_TIE 1e-13
#define GPK_DIRECT_FGLOBAL (-1e100)
#define GPK_DIRECT_FGLPER 0.01

// the persistent state of a run
struct DirState {
    double levels[GPK_DIRECT_LEVELS];        // centre-to-vertex distance of level n k + j
    double thirds[GPK_DIRECT_MAXDEEP + 2];   // 1 / 3^k
    double shift[GPK_DIRECT_MAX_D];          // c1 = l / (u - l)
    double span[GPK_DIRECT_MAX_D];           // c2 = u - l
    int anchor[GPK_DIRECT_LEVELS];           // head of each level's list, -1: empty
    double minf;                             // incumbent energy
    int minpos;                              // incumbent rectangle
    int nrect;                               // rectangles in the store
    long long nfev;
    int t;                                   // iteration (1 after the initial division)
    int stop;                                // gpk_direct_stop
    int pending;                             // stop the selection found (maxdeep / maxdiv), taken after the division
    int nsel;                                // rectangles this iteration divides
    int nrows;                               // rows this iteration samples
};

// the record read back once per iteration (24 bytes)
struct DirStatus {
    long long nfev;
    int nrows;
    int stop;
    int t;
    int pad;
};
#define GPK_DIRECT_OVERFLOW (-1)   // the store bound of direct_drive was wrong: an internal error, never a result

// the per-run arrays, all in one device allocation (see direct_drive)
struct DirArrays {
    double* c;       // R x d unit-cube centres
    int* ln;         // R x d trisection counts
    double* f;       // R energies
    int* nxt;        // R list successors, -1: end
    int* sel_r;      // GPK_DIRECT_MAXDIV chosen rectangles, in processing order
    int* sel_lv;     // their levels
    int* sel_k;      // their smallest trisection count
    int* sel_off;    // their first row
    int* rowpar;     // per row: the chosen entry it samples around
    int* rowdim;     // per row: the dimension it moves along (even rows +, odd rows -)
    double* rows;    // rows x d, mapped to the box
};

// DIRGetlevel for jones = 0, counted as Gablonsky counts it
__device__ __forceinline__ int gpk_direct_level(const int* ln, int n) {
    const int help = ln[0];
    int k = help, p = 1;
    for (int i = 1; i < n; ++i) {
        if (ln[i] < k) k = ln[i];
        if (ln[i] == help) ++p;
    }
    return k == help ? n * k + n - p : n * k + p;
}

// DIRInsert: behind start, before the first successor with a strictly larger energy
__device__ void gpk_direct_insert_after(int start, int ins, const double* f, int* nxt) {
    for (;;) {
        const int nx = nxt[start];
        if (nx < 0) { nxt[start] = ins; nxt[ins] = -1; return; }
        if (f[ins] < f[nx]) { nxt[start] = ins; nxt[ins] = nx; return; }
        start = nx;
    }
}

// DIRInsertList for one (+, -) pair of children
__device__ void gpk_direct_insert_pair(DirState* s, const DirArrays& a, int n, int pos1, int pos2) {
    const double* f = a.f;
    int* nxt = a.nxt;
    const int deep = gpk_direct_level(a.ln + (size_t)pos1 * n, n);
    const int pos = s->anchor[deep];
    if (pos < 0) {
        if (f[pos2] < f[pos1]) { s->anchor[deep] = pos2; nxt[pos2] = pos1; nxt[pos1] = -1; }
        else { s->anchor[deep] = pos1; nxt[pos1] = pos2; nxt[pos2] = -1; }
        return;
    }
    if (f[pos2] < f[pos1]) {
        if (f[pos2] < f[pos]) {
            s->anchor[deep] = pos2;
            if (f[pos1] < f[pos]) { nxt[pos2] = pos1; nxt[pos1] = pos; }
            else { nxt[pos2] = pos; gpk_direct_insert_after(pos, pos1, f, nxt); }
        } else {
            gpk_direct_insert_after(pos, pos2, f, nxt);
            gpk_direct_insert_after(pos, pos1, f, nxt);
        }
    } else {
        if (f[pos1] < f[pos]) {
            s->anchor[deep] = pos1;
            if (f[pos] < f[pos2]) { nxt[pos1] = pos; gpk_direct_insert_after(pos, pos2, f, nxt); }
            else { nxt[pos1] = pos2; nxt[pos2] = pos; }
        } else {
            gpk_direct_insert_after(pos, pos1, f, nxt);
            gpk_direct_insert_after(pos, pos2, f, nxt);
        }
    }
}

// the divided parent goes back into the list of its new level
__device__ void gpk_direct_insert_one(DirState* s, const DirArrays& a, int n, int samp) {
    const int deep = gpk_direct_level(a.ln + (size_t)samp * n, n);
    const int pos = s->anchor[deep];
    if (pos < 0) { s->anchor[deep] = samp; a.nxt[samp] = -1; }
    else if (a.f[samp] < a.f[pos]) { s->anchor[deep] = samp; a.nxt[samp] = pos; }
    else gpk_direct_insert_after(pos, samp, a.f, a.nxt);
}

__device__ __forceinline__ double gpk_direct_box(double c, double shift, double span) {
    return __dmul_rn(__dadd_rn(c, shift), span);                          // (c + c1) c2: DIRInfcn
}

// The tables, the box map and the root (the centre of the unit cube) as row 0.  One CTA of GPK_DIRECT_MAX_D threads.
__global__ void gpk_direct_init_kernel(int n, const double* lower, const double* upper, DirState* s, DirArrays a) {
    const int j = threadIdx.x;
    if (j < n) {
        const double span = __dsub_rn(upper[j], lower[j]);
        const double shift = __ddiv_rn(lower[j], span);
        s->span[j] = span;
        s->shift[j] = shift;
        a.c[j] = 0.5;
        a.ln[j] = 0;
        a.rows[j] = gpk_direct_box(0.5, shift, span);
    }
    for (int l = j; l < GPK_DIRECT_LEVELS; l += blockDim.x) s->anchor[l] = -1;
    if (j == 0) {
        double w[GPK_DIRECT_MAX_D];
        for (int q = 0; q < n; ++q)                                       // 0.5 sqrt(n - q + q / 9)
            w[q] = __dmul_rn(0.5, __dsqrt_rn(__dadd_rn((double)(n - q), __ddiv_rn((double)q, 9.0))));
        double help2 = 1.0;
        for (int i = 0; i * n < GPK_DIRECT_LEVELS; ++i) {
            for (int q = 0; q < n && i * n + q < GPK_DIRECT_LEVELS; ++q) s->levels[i * n + q] = __ddiv_rn(w[q], help2);
            help2 = __dmul_rn(help2, 3.0);
        }
        s->thirds[0] = 1.0;
        help2 = 3.0;
        for (int i = 1; i < GPK_DIRECT_MAXDEEP + 2; ++i) {
            s->thirds[i] = __ddiv_rn(1.0, help2);
            help2 = __dmul_rn(help2, 3.0);
        }
        a.f[0] = INFINITY;
        a.nxt[0] = -1;
        s->minf = INFINITY;
        s->minpos = 0;
        s->nrect = 1;
        s->nfev = 0;
        s->t = 0;
        s->stop = GPK_DIRECT_RUNNING;
        s->pending = GPK_DIRECT_RUNNING;
        s->nsel = 0;
        s->nrows = 1;
    }
}

// Selection (DIRChoose + DIRDoubleInsert) and the rows of the iteration.  first: the initial division of the root.
// One CTA of GPK_DIRECT_THREADS threads; thread 0 chooses, then the CTA writes the children and their rows.
__global__ void __launch_bounds__(GPK_DIRECT_THREADS)
gpk_direct_select_kernel(int n, int first, int maxT, long long cap, DirState* s, DirArrays a, DirStatus* status) {
    __shared__ int sh_go;
    if (threadIdx.x == 0) {
        int nsel = 0, nrows = 0;
        if (s->stop == GPK_DIRECT_RUNNING) {
            const double* f = a.f;
            if (first) {
                a.sel_r[0] = 0;
                a.sel_lv[0] = 0;
                nsel = 1;
            } else if ((s->t += 1) >= maxT) {                   // iterations 2 .. maxT - 1 sample
                s->stop = GPK_DIRECT_MAXT;
            } else {
                // S: the head of every non-empty level, largest rectangles first
                int m = 0;
                for (int l = 0; l < GPK_DIRECT_LEVELS; ++l)
                    if (s->anchor[l] >= 0) { a.sel_r[m] = s->anchor[l]; a.sel_lv[m] = l; ++m; }
                const double minf = s->minf;
                const double t1 = __dsub_rn(minf, __dmul_rn(GPK_DIRECT_EPS, fabs(minf)));
                const double t2 = __dsub_rn(minf, 0.0);
                const double thresh = t1 < t2 ? t1 : t2;
                for (int j = m - 1; j >= 0; --j) {
                    const double fj = f[a.sel_r[j]], dj = s->levels[a.sel_lv[j]];
                    double lower = INFINITY, greater = 0.0;
                    bool keep = true;
                    for (int i = 0; i < j && keep; ++i) {          // larger heads: every slope > 0, K = the least
                        const double h = __ddiv_rn(__dsub_rn(f[a.sel_r[i]], fj), __dsub_rn(s->levels[a.sel_lv[i]], dj));
                        if (h <= 0.0) keep = false;
                        else if (h < lower) lower = h;
                    }
                    for (int i = j + 1; i < m && keep; ++i) {      // smaller heads still kept: every slope > 0, G = the largest
                        if (a.sel_r[i] < 0) continue;
                        const double h = __ddiv_rn(__dsub_rn(f[a.sel_r[i]], fj), __dsub_rn(s->levels[a.sel_lv[i]], dj));
                        if (h <= 0.0) keep = false;
                        else if (h > greater) greater = h;
                    }
                    if (keep && lower >= greater) keep = !(__dsub_rn(fj, __dmul_rn(lower, dj)) > thresh);
                    if (!keep) a.sel_r[j] = -1;
                }
                for (int j = 0; j < m; ++j)
                    if (a.sel_r[j] >= 0) { a.sel_r[nsel] = a.sel_r[j]; a.sel_lv[nsel] = a.sel_lv[j]; ++nsel; }
                // DIRDoubleInsert: every rectangle within 1e-13 of a chosen head, behind all heads
                const int heads = nsel;
                for (int q = 0; q < heads && s->pending == GPK_DIRECT_RUNNING; ++q) {
                    const int head = a.sel_r[q];
                    for (int pos = a.nxt[head]; pos >= 0 && __dsub_rn(f[pos], f[head]) <= GPK_DIRECT_TIE; pos = a.nxt[pos]) {
                        if (nsel == GPK_DIRECT_MAXDIV) { s->pending = GPK_DIRECT_MAXDIV_HIT; nsel = 0; break; }
                        a.sel_r[nsel] = pos;
                        a.sel_lv[nsel] = a.sel_lv[q];
                        ++nsel;
                    }
                }
                if (s->pending != GPK_DIRECT_RUNNING) nsel = 0;
            }
            // the children: 2 per longest side, + before -, ascending dimension; a rectangle whose division would
            // pass the last level ends the run after the ones before it
            int kept = 0;
            for (int q = 0; q < nsel; ++q) {
                if (a.sel_lv[q] + 1 >= GPK_DIRECT_MAXDEEP) { s->pending = GPK_DIRECT_MAXDEEP_HIT; break; }
                const int* lp = a.ln + (size_t)a.sel_r[q] * n;
                int k = lp[0];
                for (int i = 1; i < n; ++i) k = lp[i] < k ? lp[i] : k;
                int add = 0;
                for (int i = 0; i < n; ++i) add += lp[i] == k ? 2 : 0;
                if ((long long)s->nrect + nrows + add > cap) { s->stop = GPK_DIRECT_OVERFLOW; kept = 0; nrows = 0; break; }
                a.sel_k[q] = k;
                a.sel_off[q] = nrows;
                for (int i = 0; i < n; ++i)
                    if (lp[i] == k) {
                        a.rowpar[nrows] = q; a.rowdim[nrows] = i;
                        a.rowpar[nrows + 1] = q; a.rowdim[nrows + 1] = i;
                        nrows += 2;
                    }
                ++kept;
            }
            nsel = s->stop == GPK_DIRECT_RUNNING ? kept : 0;
        }
        s->nsel = nsel;
        s->nrows = nrows;
        status->nfev = s->nfev;
        status->nrows = nrows;
        status->stop = s->stop;
        status->t = s->t;
        sh_go = nrows;
    }
    __syncthreads();
    const int nrows = sh_go;
    const size_t base = (size_t)s->nrect;
    for (long long e = threadIdx.x; e < (long long)nrows * n; e += blockDim.x) {
        const int r = (int)(e / n), j = (int)(e % n);
        const int q = a.rowpar[r];
        const int p = a.sel_r[q];
        double v = a.c[(size_t)p * n + j];
        if (j == a.rowdim[r]) {
            const double delta = s->thirds[a.sel_k[q] + 1];
            v = (r & 1) ? __dsub_rn(v, delta) : __dadd_rn(v, delta);
        }
        a.c[(base + r) * n + j] = v;
        a.ln[(base + r) * n + j] = a.ln[(size_t)p * n + j];
        a.rows[(size_t)r * n + j] = gpk_direct_box(v, s->shift[j], s->span[j]);
    }
}

// Division of every chosen rectangle in processing order (DIRSamplef's incumbent update, DIRDivide, DIRInsertList),
// then the stop tests.  phase 0: the root's energy; 1: the initial division; 2: an iteration.  One thread.
__global__ void gpk_direct_divide_kernel(int n, int phase, long long maxf, const double* val, DirState* s,
                                         DirArrays a) {
    if (threadIdx.x != 0) return;
    if (phase == 0) {
        const double e = -val[0];
        a.f[0] = isnan(e) ? INFINITY : e;
        s->minf = a.f[0];
        s->minpos = 0;
        s->nfev = 1;
        s->t = 1;
        return;
    }
    if (s->stop != GPK_DIRECT_RUNNING) return;
    const int base = s->nrect;
    const int nsel = s->nsel;
    for (int q = 0; q < nsel; ++q) {
        const int r = a.sel_r[q], k = a.sel_k[q], off = a.sel_off[q];
        if (phase == 2) {                                            // out of its level's list
            const int lv = a.sel_lv[q];
            if (s->anchor[lv] == r) s->anchor[lv] = a.nxt[r];
            else {
                int p = s->anchor[lv];
                while (a.nxt[p] != r) p = a.nxt[p];
                a.nxt[p] = a.nxt[r];
            }
        }
        int* lp = a.ln + (size_t)r * n;
        int dims[GPK_DIRECT_MAX_D], ord[GPK_DIRECT_MAX_D];
        double w[GPK_DIRECT_MAX_D];
        int m = 0;
        for (int i = 0; i < n; ++i)
            if (lp[i] == k) dims[m++] = i;
        for (int b = 0; b < 2 * m; ++b) {
            const int kid = base + off + b;
            const double e = -val[off + b];
            a.f[kid] = isnan(e) ? INFINITY : e;
            a.nxt[kid] = -1;
            if (a.f[kid] < s->minf) { s->minf = a.f[kid]; s->minpos = kid; }
        }
        for (int b = 0; b < m; ++b) {                                // w = MIN(f-, f+); stable insertion by strict <
            const double fp = a.f[base + off + 2 * b], fm = a.f[base + off + 2 * b + 1];
            w[b] = fm <= fp ? fm : fp;
            int p = b;
            while (p > 0 && w[b] < w[ord[p - 1]]) { ord[p] = ord[p - 1]; --p; }
            ord[p] = b;
        }
        for (int t = 0; t < m; ++t) {
            const int i = dims[ord[t]];
            lp[i] = k + 1;
            for (int u = t; u < m; ++u) {
                const int kid = base + off + 2 * ord[u];
                a.ln[(size_t)kid * n + i] = k + 1;
                a.ln[(size_t)(kid + 1) * n + i] = k + 1;
            }
        }
        for (int b = 0; b < m; ++b) gpk_direct_insert_pair(s, a, n, base + off + 2 * b, base + off + 2 * b + 1);
        gpk_direct_insert_one(s, a, n, r);
    }
    s->nrect = base + s->nrows;
    s->nfev += s->nrows;
    if (phase == 1) return;
    const double g = __ddiv_rn(__dmul_rn(__dsub_rn(s->minf, GPK_DIRECT_FGLOBAL), 100.0), fabs(GPK_DIRECT_FGLOBAL));
    if (s->pending != GPK_DIRECT_RUNNING) s->stop = s->pending;
    else if (g <= GPK_DIRECT_FGLPER) s->stop = GPK_DIRECT_FGLOBAL_HIT;
    else if (s->nfev >= maxf) s->stop = GPK_DIRECT_MAXF;
}

// The result point as the package returns it: c c2 + c1 c2 (not the evaluated (c + c1) c2).
__global__ void gpk_direct_result_kernel(int n, const DirState* s, DirArrays a, double* x) {
    const int j = threadIdx.x;
    if (j < n) {
        const double c = a.c[(size_t)s->minpos * n + j];
        x[j] = __dadd_rn(__dmul_rn(c, s->span[j]), __dmul_rn(s->shift[j], s->span[j]));
    }
}
