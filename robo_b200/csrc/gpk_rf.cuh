// gpk_rf.cuh — the random forest of robo/models/random_forest.py on the device: bagged regression trees grown by CART
// with the residual-sum-of-squares loss, and the forest's predictive moments scoring candidates for every device
// maximizer.  pyrfr (the reference's C++ library) is not available, so this file restates the algorithm RoBO's wrapper
// configures (random_forest.py:52-57 sets the forest options; the tree options are pyrfr's defaults).  tests/rf_model.py
// restates every step below in the same order; the device equals it bit for bit.
//
// Sample per tree.  Tree t (0 <= t < T) sees n_t draws from the N training rows (n_t = n_points_per_tree, or N when
// that is 0, random_forest.py:75-76).  Every draw is Philox4x32-10 with key (seed low, seed high) and counter
// (j, t, train counter, tag); its first word w becomes an index below m as floor(w m / 2^32), computed exactly in 64-bit
// integers, so it never rounds up to m.
//   bootstrap (GPK_RF_TAG_BOOT): draw j of tree t is row floor(w N / 2^32), j < n_t, with replacement; a row's
//     multiplicity is how often it was drawn.
//   no bootstrap (GPK_RF_TAG_PERM): the first n_t steps of a Fisher-Yates shuffle of the identity permutation p: step
//     j swaps p[j] and p[j + floor(w (N - j) / 2^32)]; the rows p[0..n_t) have multiplicity 1 (n_t <= N).
//
// Growth, level by level (breadth first; nodes are numbered in that order, the children of a level's split nodes in
// the level's node order, left before right, so the right child of v is left[v] + 1).  A node holds a multiset of rows.
//   Leaf when: fewer than 2 samples (with multiplicity), or fl(max y - min y) <= 1e-8, or no split candidate.
//   Totals: W = the sample count; S_t and Q_t accumulate y and fl(y * y) once per copy, rows in ascending index.
//   Split search, feature f = 0 .. D-1 (max_features = D): the node's samples ordered by (x_f, row index), copies of a row
//   adjacent.  W_l, S and Q accumulate 1, y and fl(y * y) once per copy, left to right.  After the last copy of entry k
//   whose x_f is < the next entry's, a candidate: loss = fl(Q - fl(S S) / W_l) + fl(fl(Q_t - Q) - fl(S_r S_r) / W_r),
//   S_r = fl(S_t - S), W_r = W - W_l.  The smallest loss wins under strict < in scan order (features ascending, then
//   positions), so ties go to the lowest feature and the leftmost position; a NaN loss never wins.
//   Threshold: fl(fl(x_k + x_{k+1}) / 2), replaced by x_k where it equals x_{k+1}.  A row goes left iff x_f <= threshold.
//   Leaf statistics: W, mean = fl(S_t / W), var = fl(V / W) with V accumulating fl(d d), d = fl(y - mean), once per copy,
//   rows ascending (two passes, so identical responses give exactly 0).
// Moments at x (gpk_rf_score_kernel): tree t gives the (m_t, v_t) of the leaf x falls into;
//   mean = fl(M / T), M = m_0 + m_1 + ... in ascending t, sequentially;
//   var = fl(B / T), B accumulating fl(e e), e = fl(m_t - mean), ascending t; plus fl(V / T) (V = sum of v_t, ascending t)
//   when the total variance is asked for (compute_law_of_total_variance, random_forest.py:57).  No clip.
//
// Device layout.  gpk_rf_set_data keeps X (N x D), y and, for each feature, the N rows sorted by (x_f, row index), once:
// a tree's multiset only changes multiplicities, so its per-feature lists are the shared order with the undrawn rows
// removed.  gpk_rf_grow_kernel grows one tree per CTA without a host round trip: per level, one warp per node finds the
// totals (lanes over the rows) and scans the features (lanes over features, each scan sequential); thread 0 numbers the
// children; then one thread per (split node, list) partitions the node's D + 1 lists (D features and the rows ascending)
// stably into the other buffer, where each child is a contiguous segment.  Nodes (split feature, threshold, left child,
// leaf W, mean, var) stay in device memory, T x 2N slots.
#pragma once
#include "gpk_kernels.cuh"

#define GPK_RF_TAG_BOOT 0x52460001u
#define GPK_RF_TAG_PERM 0x52460002u
#define GPK_RF_GROW_THREADS 256
#define GPK_RF_SCORE_WARPS 4
#define GPK_RF_PURITY 1e-8

// floor(w m / 2^32): an index below m from one 32-bit draw
__device__ __forceinline__ int gpk_rf_index(uint32_t w, uint32_t m)
{
    return (int)(((unsigned long long)w * m) >> 32);
}

struct RfGrowArgs {
    const double* X; const double* y; const int* order;   // X (n x d), y (n), order (d x n)
    int n, d, nt, bootstrap, t0;                         // t0: tree index of blockIdx.x == 0
    unsigned long long seed; unsigned counter;
    int* cnt; int* lists; int* seg;                      // per CTA: n; 2 (d + 1) n; 3 (2 n)
    int* feat; int* left; double* thr; double* W; double* mean; double* var;   // per tree: 2 n slots
    int* n_nodes;                                        // per tree
};

__global__ void __launch_bounds__(GPK_RF_GROW_THREADS) gpk_rf_grow_kernel(const RfGrowArgs a)
{
    constexpr int NT = GPK_RF_GROW_THREADS, NW = NT / 32;
    const unsigned FULL = 0xffffffffu;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int t = a.t0 + blockIdx.x, n = a.n, d = a.d, L = d + 1;
    const long S = 2L * n, ts = (long)t * S;
    const double* X = a.X;
    const double* y = a.y;
    int* cnt = a.cnt + (long)blockIdx.x * n;
    int* cur = a.lists + (long)blockIdx.x * 2 * L * n;
    int* nxt = cur + (long)L * n;
    int* sstart = a.seg + (long)blockIdx.x * 3 * S;
    int* slen = sstart + S;
    int* snl = slen + S;
    int* feat = a.feat + ts;
    int* left = a.left + ts;
    double* thr = a.thr + ts;
    double* Wn = a.W + ts;
    double* mean = a.mean + ts;
    double* var = a.var + ts;
    const uint32_t k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32);
    __shared__ int s_nu, s_lo, s_hi;

    // the tree's multiplicities
    for (int i = tid; i < n; i += NT) cnt[i] = 0;
    __syncthreads();
    if (a.bootstrap) {
        for (int j = tid; j < a.nt; j += NT) {
            uint32_t w[4];
            gpk_philox4x32_10((uint32_t)j, (uint32_t)t, a.counter, GPK_RF_TAG_BOOT, k0, k1, w);
            atomicAdd(cnt + gpk_rf_index(w[0], (uint32_t)n), 1);
        }
    } else {
        int* perm = nxt;                                  // scratch until the lists are built
        for (int i = tid; i < n; i += NT) perm[i] = i;
        __syncthreads();
        if (tid == 0)
            for (int j = 0; j < a.nt; ++j) {
                uint32_t w[4];
                gpk_philox4x32_10((uint32_t)j, (uint32_t)t, a.counter, GPK_RF_TAG_PERM, k0, k1, w);
                const int k = j + gpk_rf_index(w[0], (uint32_t)(n - j));
                const int r = perm[k];
                perm[k] = perm[j];
                perm[j] = r;
                cnt[r] = 1;
            }
    }
    __syncthreads();

    // the root's lists: feature f's shared order without the undrawn rows (stable compaction, one warp per list), and
    // list d the drawn rows ascending
    for (int l = warp; l < L; l += NW) {
        const int* src = l < d ? a.order + (long)l * n : nullptr;
        int* dst = cur + (long)l * n;
        int base = 0;
        for (int i0 = 0; i0 < n; i0 += 32) {
            const int i = i0 + lane;
            const int r = i < n ? (src ? src[i] : i) : 0;
            const bool keep = i < n && cnt[r] > 0;
            const unsigned bal = __ballot_sync(FULL, keep);
            if (keep) dst[base + __popc(bal & ((1u << lane) - 1u))] = r;
            base += __popc(bal);
        }
        if (l == d && lane == 0) s_nu = base;
    }
    if (tid == 0) { s_lo = 0; s_hi = 1; }
    __syncthreads();
    if (tid == 0) { sstart[0] = 0; slen[0] = s_nu; }
    __syncthreads();

    while (true) {
        const int lo = s_lo, hi = s_hi;
        if (lo >= hi) break;
        // one warp per node of the level: leaf or split
        for (int v = lo + warp; v < hi; v += NW) {
            const int st = sstart[v], len = slen[v];
            const int* ids = cur + (long)d * n + st;
            long long wc = 0;
            double ymin = INFINITY, ymax = -INFINITY;
            for (int i = lane; i < len; i += 32) {
                const int r = ids[i];
                wc += cnt[r];
                ymin = fmin(ymin, y[r]);
                ymax = fmax(ymax, y[r]);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                wc += __shfl_xor_sync(FULL, wc, o);
                ymin = fmin(ymin, __shfl_xor_sync(FULL, ymin, o));
                ymax = fmax(ymax, __shfl_xor_sync(FULL, ymax, o));
            }
            double St = 0.0, Qt = 0.0;
            if (lane == 0)
                for (int i = 0; i < len; ++i) {
                    const int r = ids[i], c = cnt[r];
                    const double yv = y[r], yy = __dmul_rn(yv, yv);
                    for (int k = 0; k < c; ++k) { St = __dadd_rn(St, yv); Qt = __dadd_rn(Qt, yy); }
                }
            St = __shfl_sync(FULL, St, 0);
            Qt = __shfl_sync(FULL, Qt, 0);
            const double Wt = (double)wc;
            bool leaf = wc < 2 || __dsub_rn(ymax, ymin) <= GPK_RF_PURITY;
            double best = INFINITY;
            int bf = 0x7fffffff, bpos = -1;
            if (!leaf) {
                for (int f = lane; f < d; f += 32) {
                    const int* lf = cur + (long)f * n + st;
                    double Wl = 0.0, Sl = 0.0, Ql = 0.0;
                    int r = lf[0];
                    double xr = X[(long)r * d + f];
                    for (int i = 0; i + 1 < len; ++i) {
                        const int c = cnt[r];
                        const double yv = y[r], yy = __dmul_rn(yv, yv);
                        for (int k = 0; k < c; ++k) { Sl = __dadd_rn(Sl, yv); Ql = __dadd_rn(Ql, yy); }
                        Wl = __dadd_rn(Wl, (double)c);
                        const int rn = lf[i + 1];
                        const double xn = X[(long)rn * d + f];
                        if (xr < xn) {
                            const double Sr = __dsub_rn(St, Sl), Wr = __dsub_rn(Wt, Wl);
                            const double lossl = __dsub_rn(Ql, __ddiv_rn(__dmul_rn(Sl, Sl), Wl));
                            const double lossr = __dsub_rn(__dsub_rn(Qt, Ql), __ddiv_rn(__dmul_rn(Sr, Sr), Wr));
                            const double loss = __dadd_rn(lossl, lossr);
                            if (loss < best) { best = loss; bf = f; bpos = i; }
                        }
                        r = rn;
                        xr = xn;
                    }
                }
                // the lowest (loss, feature) over the lanes: a total order, so every lane ends with the same winner
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const double ob = __shfl_xor_sync(FULL, best, o);
                    const int of = __shfl_xor_sync(FULL, bf, o), op = __shfl_xor_sync(FULL, bpos, o);
                    if (ob < best || (ob == best && of < bf)) { best = ob; bf = of; bpos = op; }
                }
                if (bpos < 0) leaf = true;
            }
            if (lane == 0) {
                if (leaf) {
                    const double mu = __ddiv_rn(St, Wt);
                    double V = 0.0;
                    for (int i = 0; i < len; ++i) {
                        const int r = ids[i], c = cnt[r];
                        const double e = __dsub_rn(y[r], mu), ee = __dmul_rn(e, e);
                        for (int k = 0; k < c; ++k) V = __dadd_rn(V, ee);
                    }
                    feat[v] = -1; left[v] = -1; thr[v] = 0.0;
                    Wn[v] = Wt; mean[v] = mu; var[v] = __ddiv_rn(V, Wt);
                } else {
                    const int* lf = cur + (long)bf * n + st;
                    const double xa = X[(long)lf[bpos] * d + bf], xb = X[(long)lf[bpos + 1] * d + bf];
                    double th = __ddiv_rn(__dadd_rn(xa, xb), 2.0);
                    if (th == xb) th = xa;
                    feat[v] = bf; thr[v] = th;
                    Wn[v] = 0.0; mean[v] = 0.0; var[v] = 0.0;
                    snl[v] = bpos + 1;                    // entries of the segment that go left
                }
            }
        }
        __syncthreads();
        // the children of the level's split nodes, in node order
        if (tid == 0) {
            int nx = hi;
            for (int v = lo; v < hi; ++v)
                if (feat[v] >= 0) {
                    left[v] = nx;
                    sstart[nx] = sstart[v];
                    slen[nx] = snl[v];
                    sstart[nx + 1] = sstart[v] + snl[v];
                    slen[nx + 1] = slen[v] - snl[v];
                    nx += 2;
                }
            s_lo = hi;
            s_hi = nx;
        }
        __syncthreads();
        // every list of every split node, stably partitioned into the other buffer
        const long tasks = (long)(hi - lo) * L;
        for (long q = tid; q < tasks; q += NT) {
            const int v = lo + (int)(q / L), l = (int)(q - (q / L) * L);
            const int f = feat[v];
            if (f < 0) continue;
            const double th = thr[v];
            const int st = sstart[v], len = slen[v];
            const int* src = cur + (long)l * n + st;
            int* dl = nxt + (long)l * n + st;
            int* dr = dl + snl[v];
            int il = 0, ir = 0;
            for (int i = 0; i < len; ++i) {
                const int r = src[i];
                if (X[(long)r * d + f] <= th) dl[il++] = r;
                else dr[ir++] = r;
            }
        }
        __syncthreads();
        int* sw = cur;
        cur = nxt;
        nxt = sw;
    }
    if (tid == 0) a.n_nodes[t] = s_hi;
}

struct RfScoreArgs {
    const double* X; long m; int D, T; long S;           // S: node slots per tree
    const int* feat; const int* left; const double* thr; const double* mean; const double* var;
    int total_var;
    ScoreOut o;
};

// doubles of dynamic shared memory of gpk_rf_score_kernel for T trees
__host__ __device__ inline long gpk_rf_score_smem_doubles(int T) { return 2L * GPK_RF_SCORE_WARPS * T; }

// one warp per candidate, lanes over trees: the leaf of every tree, the moments in ascending t (lane 0), the
// acquisition and the block arg-max (gpk_finish_kernel's)
__global__ void __launch_bounds__(GPK_RF_SCORE_WARPS * 32) gpk_rf_score_kernel(const RfScoreArgs a)
{
    extern __shared__ double rs[];                      // [warp][m_t (T), v_t (T)]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, T = a.T;
    const long c = (long)blockIdx.x * GPK_RF_SCORE_WARPS + warp;
    double* mt = rs + (long)warp * 2 * T;
    double* vt = mt + T;
    double val = 0.0;
    long long idx = -1;
    if (c < a.m) {
        const double* x = a.X + c * a.D;
        for (int t = lane; t < T; t += 32) {
            const long o = (long)t * a.S;
            int v = 0, f;
            while ((f = __ldg(a.feat + o + v)) >= 0) v = __ldg(a.left + o + v) + (x[f] <= __ldg(a.thr + o + v) ? 0 : 1);
            mt[t] = __ldg(a.mean + o + v);
            vt[t] = __ldg(a.var + o + v);
        }
        __syncwarp();
        if (lane == 0) {
            const double Td = (double)T;
            double sm = 0.0, sv = 0.0;
            for (int t = 0; t < T; ++t) { sm = __dadd_rn(sm, mt[t]); sv = __dadd_rn(sv, vt[t]); }
            const double mu = __ddiv_rn(sm, Td);
            double sq = 0.0;
            for (int t = 0; t < T; ++t) {
                const double e = __dsub_rn(mt[t], mu);
                sq = __dadd_rn(sq, __dmul_rn(e, e));
            }
            double vr = __ddiv_rn(sq, Td);
            if (a.total_var) vr = __dadd_rn(vr, __ddiv_rn(sv, Td));
            // a zero std gives EI 0 (ei.py:72-74), not s (z Phi(z) + phi(z)) = 0 * inf
            gpk_score_emit(a.o, c, mu, vr, val, idx, true);
        }
    }
    if (a.o.acq_kind == GPK_ACQ_NONE) return;
    gpk_block_best<GPK_RF_SCORE_WARPS>(val, idx);
    if (threadIdx.x == 0) a.o.block_best[blockIdx.x] = {val, idx};
}
