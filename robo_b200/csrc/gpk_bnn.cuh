// gpk_bnn.cuh — the Bayesian neural network of robo/models/wrapper_bohamiann.py on the device: the network sampled by
// adaptive SGHMC (Springenberg, Klein, Falkner, Hutter, "Bayesian Optimization with Robust Bayesian Neural Networks",
// NIPS 2016) in one launch, and its predictive moments scoring candidates for every device maximizer.  pybnn (the
// library the wrapper calls) is not available, so the model is restated here, in tests/bnn_model.py and in DESIGN §1
// row a28; the pybnn details below are this project's statement, not checked against pybnn.
//
// Network (wrapper_bohamiann.py:10-34): Linear(D, 50) . tanh . Linear(50, 50) . tanh . Linear(50, 1), and a scalar lv
// (homoscedastic log-variance) as the second output.  theta, P = 50 D + 2652 doubles, in this order: W1 (50 x D, row j
// = hidden unit j), b1 (50), W2 (50 x 50), b2 (50), W3 (50), b3, lv.  Initialisation: W_l = xi / sqrt(fan_in) with xi the
// step -1 normals (below), biases 0, lv = log(1e-2).
//
// Data: gpk_bnn_set_data scales X per column and y to zero mean and unit population std on the host (sums in ascending
// row order, std = sqrt(sum of (x - mean)^2 / N)); N = 1, a constant column or a constant y is GPK_BAD_ARG.
//
// Batches: B rows; epoch e visits the rows in the ranks of (Philox word 0 of (row, e, counter, GPK_BNN_TAG_ORDER), row),
// B at a time, the last batch of an epoch partial (B_t = N - B floor(N / B) rows); then epoch e + 1.  Step s takes
// batch s mod ceil(N / B) of epoch floor(s / ceil(N / B)).
//
// Gradient G = N dL/dtheta of L = nll - lvp / N - wp / N on a batch of B_t rows (every product, sum and quotient rounded
// once, __dmul_rn / __dadd_rn / __ddiv_rn, never contracted; a "sum" starts at the bias, or at +0.0, and adds the terms
// in ascending index):
//   a1 = b1_j + sum_d W1_jd x_d; h1 = tanh(a1); a2 = b2_j + sum_k W2_jk h1_k; h2 = tanh(a2); f = b3 + sum_j W3_j h2_j
//   ev = exp(lv), s2 = ev + 1e-16, c = N / B_t; per row r = y - f, q = r / s2, df = -(c q), u = 0.5 - 0.5 ((q q) ev)
//   G_b3 = sum_i df_i, G_W3_j = sum_i df_i h2_ij, G_lv = (c sum_i u_i) + (lv - ln 1e-6) / 0.01
//   d2_ij = (df_i W3_j) (1 - h2_ij h2_ij);  G_b2_j = sum_i d2_ij, G_W2_jk = sum_i d2_ij h1_ik
//   d1_ik = (sum_j d2_ij W2_jk) (1 - h1_ik h1_ik);  G_b1_k = sum_i d1_ik, G_W1_kd = sum_i d1_ik x_id
//   then every entry, lv included: G_p = G_p + theta_p / P (the weight prior)
// exp is gpk_cmaes_exp; tanh is gpk_bnn_tanh below.
//
// Adaptive SGHMC, per parameter, step s = 0 .. num_steps - 1 (t = s + 1), state tau = g = vhat = 1, p = 0:
//   while t <= burn_in: r = 1 / (tau + 1); tau = (tau - (tau (g g)) / (vhat + eps)) + 1; g = (g - g r) + r G;
//                       vhat = (vhat - vhat r) + r (G G)      [tau from the old g and vhat, g before vhat]
//   minv = 1 / (sqrt(vhat) + eps); lr2 = lr lr; s2 = ((2 lr2) mdecay) minv - lr2 lr2
//   p = ((p - (lr2 minv) G) - mdecay p) + sqrt(max(s2, 1e-16)) xi;  theta = theta + p
// and theta is kept (written to sample k, k = 0, 1, ...) after step s when s > burn_in and (s - burn_in) % keep_every
// == 0.  xi of parameters 2q and 2q + 1 at step s: Box-Muller (gpk_cmaes_normals' arithmetic) of Philox4x32-10 keyed by
// the 64-bit seed with counter (q, s, counter, GPK_BNN_TAG_NOISE); step -1 (0xFFFFFFFF) gives the initial weights.
//
// gpk_bnn_chain_kernel runs the whole chain in one CTA: theta, its gradient, the batch and every activation stay in
// shared memory for the whole run; one thread owns a parameter pair in the update, and its optimizer state (p, tau, g,
// vhat) lives in device memory, in the handle's state buffer, read and written by that thread alone (registers cannot
// hold 4 x 23 doubles per thread at D = 64 without spilling).  Every phase of a step ends in one __syncthreads.
//
// Predict (gpk_bnn_score_kernel), over the S kept networks k in ascending order: m = mean_k f_k, v = mean_k (f_k - m)^2
// + mean_k exp(lv_k) (Welford's running mean and M2 in network order), then m y_std + y_mean and v y_std^2.  Scoring
// uses fma and libdevice tanh / exp; it is pinned by tolerance, not bit for bit.
#pragma once
#include "gpk_internal.cuh"
#include "gpk_kernels.cuh"
#include "gpk_gemm.cuh"
#include "gpk_cmaes.cuh"

#define GPK_BNN_H 50                      // hidden units per layer
#define GPK_BNN_THREADS 256               // threads of the chain kernel
#define GPK_BNN_SCORE_THREADS 128         // threads of the scoring kernel ...
#define GPK_BNN_SCORE_C 2                 // ... candidates per thread
#define GPK_BNN_TAG_NOISE 0x424E0001u
#define GPK_BNN_TAG_ORDER 0x424E0002u
#define GPK_BNN_LOG_LV0 -4.605170185988091       // log(1e-2)
#define GPK_BNN_LOG_1EM6 -13.815510557964274     // log(1e-6)

__host__ __device__ inline int gpk_bnn_params(int d) { return GPK_BNN_H * d + 2652; }

// tanh(x) as a fixed operation sequence: |x| < 2^-8: x + x (x^2 (-1/3 + x^2 (2/15 - 17/315 x^2))); otherwise
// t = exp(-2 |x|) (gpk_cmaes_exp) and sign(x) (1 - t) / (1 + t).  NaN stays NaN.
__device__ __forceinline__ double gpk_bnn_tanh(double x) {
    const double ax = fabs(x);
    if (ax < 0.00390625) {
        const double x2 = __dmul_rn(x, x);
        const double p = __dadd_rn(-0.3333333333333333,
                                   __dmul_rn(x2, __dsub_rn(0.13333333333333333, __dmul_rn(0.05396825396825397, x2))));
        return __dadd_rn(x, __dmul_rn(x, __dmul_rn(x2, p)));
    }
    const double t = gpk_cmaes_exp(__dmul_rn(-2.0, ax));
    const double r = __ddiv_rn(__dsub_rn(1.0, t), __dadd_rn(1.0, t));
    return x < 0.0 ? -r : (x > 0.0 ? r : x);
}

// the normals of parameters 2q and 2q + 1 at chain step `step` (0xFFFFFFFF: the initial weights)
__device__ __forceinline__ void gpk_bnn_normals(unsigned long long seed, unsigned counter, uint32_t step, int q,
                                                double* z0, double* z1) {
    uint32_t w[4];
    gpk_philox4x32_10((uint32_t)q, step, counter, GPK_BNN_TAG_NOISE, (uint32_t)seed, (uint32_t)(seed >> 32), w);
    const double u1 = (double)(((((unsigned long long)w[1] << 32) | w[0]) >> 11) + 1ull) * 1.1102230246251565e-16;
    const double u2 = gpk_u01(w[2], w[3]);
    const double rr = __dsqrt_rn(__dmul_rn(-2.0, log(u1)));
    double s, c;
    sincospi(__dmul_rn(2.0, u2), &s, &c);
    *z0 = __dmul_rn(rr, c);
    *z1 = __dmul_rn(rr, s);
}

// gpk_bnn_draws: Z (ns x P) of steps step0 .. step0 + ns - 1 (uint32 arithmetic, so step0 = -1 is the initialisation)
__global__ void gpk_bnn_draws_kernel(unsigned long long seed, unsigned counter, int step0, int ns, int P,
                                     double* __restrict__ Z) {
    const int nq = P / 2;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)ns * nq) return;
    const int q = (int)(t % nq), si = (int)(t / nq);
    double z0, z1;
    gpk_bnn_normals(seed, counter, (uint32_t)step0 + (uint32_t)si, q, &z0, &z1);
    Z[(size_t)si * P + 2 * q] = z0;
    Z[(size_t)si * P + 2 * q + 1] = z1;
}

struct BnnChainArgs {
    const double* X; const double* y;      // scaled training set, N x D and N
    int n, d, P, B;
    unsigned long long seed; unsigned counter;
    double lr, mdecay, eps;
    long long burn_in, num_steps, keep_every;
    double* samples;                       // S x P kept networks
    double* state;                         // theta, p, tau, g, vhat (P each)
};

// doubles of dynamic shared memory of gpk_bnn_chain_kernel before the epoch order (8 + 4 bytes per row)
__host__ __device__ inline long gpk_bnn_chain_doubles(int d, int B) {
    return 2L * gpk_bnn_params(d) + (long)B * (d + 1) + 4L * B * GPK_BNN_H + 2L * B;
}
__host__ __device__ inline long gpk_bnn_chain_smem(int n, int d, int B) {
    return gpk_bnn_chain_doubles(d, B) * 8 + 12L * n;
}

__global__ void __launch_bounds__(GPK_BNN_THREADS) gpk_bnn_chain_kernel(const BnnChainArgs a)
{
    constexpr int NT = GPK_BNN_THREADS, H = GPK_BNN_H;
    extern __shared__ double bsm[];
    const int tid = threadIdx.x, N = a.n, D = a.d, P = a.P, B = a.B;
    double* th = bsm;                       // theta
    double* gr = th + P;                    // gradient (backprop part)
    double* xb = gr + P;                    // batch inputs, B x D
    double* yb = xb + (long)B * D;          // batch targets
    double* h1 = yb + B;                    // B x 50
    double* h2 = h1 + B * H;
    double* d2 = h2 + B * H;
    double* d1 = d2 + B * H;
    double* df = d1 + B * H;                // B
    double* ub = df + B;                    // B
    unsigned long long* keys = (unsigned long long*)(ub + B);
    int* order = (int*)(keys + N);
    const int oW1 = 0, oB1 = H * D, oW2 = oB1 + H, oB2 = oW2 + H * H, oW3 = oB2 + H, oB3 = oW3 + H, oLV = oB3 + 1;
    double* sp = a.state + P;
    double* stau = sp + P;
    double* sg = stau + P;
    double* sv = sg + P;
    const double Pd = (double)P, Nd = (double)N;
    const double lr2 = __dmul_rn(a.lr, a.lr), lr4 = __dmul_rn(lr2, lr2);
    const double sc1 = __ddiv_rn(1.0, __dsqrt_rn((double)D)), sc2 = __ddiv_rn(1.0, __dsqrt_rn((double)H));

    // initial weights and optimizer state
    for (int q = tid; q < P / 2; q += NT) {
        double z[2];
        gpk_bnn_normals(a.seed, a.counter, 0xFFFFFFFFu, q, z, z + 1);
        for (int e = 0; e < 2; ++e) {
            const int j = 2 * q + e;
            double v = 0.0;
            if (j < oB1) v = __dmul_rn(z[e], sc1);
            else if ((j >= oW2 && j < oB2) || (j >= oW3 && j < oB3)) v = __dmul_rn(z[e], sc2);
            else if (j == oLV) v = GPK_BNN_LOG_LV0;
            th[j] = v;
            sp[j] = 0.0; stau[j] = 1.0; sg[j] = 1.0; sv[j] = 1.0;
        }
    }
    __syncthreads();

    const int nb = (N + B - 1) / B;
    long long kept = 0;
    for (long long s = 0; s < a.num_steps; ++s) {
        const long long e = s / nb;
        const int bi = (int)(s - e * nb), pos0 = bi * B, Bt = min(B, N - pos0);
        if (bi == 0) {                      // the epoch's order: ranks of (key, row)
            for (int i = tid; i < N; i += NT) {
                uint32_t w[4];
                gpk_philox4x32_10((uint32_t)i, (uint32_t)e, a.counter, GPK_BNN_TAG_ORDER, (uint32_t)a.seed,
                                  (uint32_t)(a.seed >> 32), w);
                keys[i] = ((unsigned long long)w[0] << 32) | (unsigned)i;
            }
            __syncthreads();
            for (int i = tid; i < N; i += NT) {
                const unsigned long long ki = keys[i];
                int r = 0;
                for (int j = 0; j < N; ++j) r += keys[j] < ki;
                order[r] = i;
            }
            __syncthreads();
        }
        for (int q = tid; q < Bt * D; q += NT) {
            const int i = q / D;
            xb[q] = a.X[(long)order[pos0 + i] * D + (q - i * D)];
        }
        for (int i = tid; i < Bt; i += NT) yb[i] = a.y[order[pos0 + i]];
        __syncthreads();
        // forward
        for (int q = tid; q < Bt * H; q += NT) {
            const int i = q / H, j = q - i * H;
            double acc = th[oB1 + j];
            for (int k = 0; k < D; ++k) acc = __dadd_rn(acc, __dmul_rn(th[oW1 + j * D + k], xb[i * D + k]));
            h1[q] = gpk_bnn_tanh(acc);
        }
        __syncthreads();
        for (int q = tid; q < Bt * H; q += NT) {
            const int i = q / H, j = q - i * H;
            double acc = th[oB2 + j];
            for (int k = 0; k < H; ++k) acc = __dadd_rn(acc, __dmul_rn(th[oW2 + j * H + k], h1[i * H + k]));
            h2[q] = gpk_bnn_tanh(acc);
        }
        __syncthreads();
        const double lv = th[oLV];
        const double ev = gpk_cmaes_exp(lv), s2 = __dadd_rn(ev, 1e-16), c = __ddiv_rn(Nd, (double)Bt);
        for (int i = tid; i < Bt; i += NT) {
            double f = th[oB3];
            for (int j = 0; j < H; ++j) f = __dadd_rn(f, __dmul_rn(th[oW3 + j], h2[i * H + j]));
            const double q = __ddiv_rn(__dsub_rn(yb[i], f), s2);
            df[i] = -__dmul_rn(c, q);
            ub[i] = __dsub_rn(0.5, __dmul_rn(0.5, __dmul_rn(__dmul_rn(q, q), ev)));
        }
        __syncthreads();
        // backward: output layer and the second layer's deltas
        for (int q = tid; q < Bt * H + H + 2; q += NT) {
            if (q < Bt * H) {
                const int i = q / H, j = q - i * H;
                d2[q] = __dmul_rn(__dmul_rn(df[i], th[oW3 + j]), __dsub_rn(1.0, __dmul_rn(h2[q], h2[q])));
            } else if (q < Bt * H + H) {
                const int j = q - Bt * H;
                double acc = 0.0;
                for (int i = 0; i < Bt; ++i) acc = __dadd_rn(acc, __dmul_rn(df[i], h2[i * H + j]));
                gr[oW3 + j] = acc;
            } else if (q == Bt * H + H) {
                double acc = 0.0;
                for (int i = 0; i < Bt; ++i) acc = __dadd_rn(acc, df[i]);
                gr[oB3] = acc;
            } else {
                double acc = 0.0;
                for (int i = 0; i < Bt; ++i) acc = __dadd_rn(acc, ub[i]);
                gr[oLV] = __dadd_rn(__dmul_rn(c, acc), __ddiv_rn(__dsub_rn(lv, GPK_BNN_LOG_1EM6), 0.01));
            }
        }
        __syncthreads();
        // the first layer's deltas, the second layer's gradient
        for (int q = tid; q < Bt * H + H * H + H; q += NT) {
            if (q < Bt * H) {
                const int i = q / H, k = q - i * H;
                double acc = 0.0;
                for (int j = 0; j < H; ++j) acc = __dadd_rn(acc, __dmul_rn(d2[i * H + j], th[oW2 + j * H + k]));
                d1[q] = __dmul_rn(acc, __dsub_rn(1.0, __dmul_rn(h1[q], h1[q])));
            } else if (q < Bt * H + H * H) {
                const int jk = q - Bt * H, j = jk / H, k = jk - j * H;
                double acc = 0.0;
                for (int i = 0; i < Bt; ++i) acc = __dadd_rn(acc, __dmul_rn(d2[i * H + j], h1[i * H + k]));
                gr[oW2 + jk] = acc;
            } else {
                const int j = q - Bt * H - H * H;
                double acc = 0.0;
                for (int i = 0; i < Bt; ++i) acc = __dadd_rn(acc, d2[i * H + j]);
                gr[oB2 + j] = acc;
            }
        }
        __syncthreads();
        // the first layer's gradient
        for (int q = tid; q < H * D + H; q += NT) {
            double acc = 0.0;
            if (q < H * D) {
                const int j = q / D, k = q - j * D;
                for (int i = 0; i < Bt; ++i) acc = __dadd_rn(acc, __dmul_rn(d1[i * H + j], xb[i * D + k]));
                gr[oW1 + q] = acc;
            } else {
                const int j = q - H * D;
                for (int i = 0; i < Bt; ++i) acc = __dadd_rn(acc, d1[i * H + j]);
                gr[oB1 + j] = acc;
            }
        }
        __syncthreads();
        // adaptive SGHMC, one parameter pair per thread
        const bool adapt = s + 1 <= a.burn_in;
        for (int q = tid; q < P / 2; q += NT) {
            double z[2];
            gpk_bnn_normals(a.seed, a.counter, (uint32_t)s, q, z, z + 1);
            for (int e2 = 0; e2 < 2; ++e2) {
                const int j = 2 * q + e2;
                const double G = __dadd_rn(gr[j], __ddiv_rn(th[j], Pd));
                double tau = stau[j], g = sg[j], v = sv[j];
                if (adapt) {
                    const double r = __ddiv_rn(1.0, __dadd_rn(tau, 1.0));
                    tau = __dadd_rn(__dsub_rn(tau, __ddiv_rn(__dmul_rn(tau, __dmul_rn(g, g)), __dadd_rn(v, a.eps))), 1.0);
                    g = __dadd_rn(__dsub_rn(g, __dmul_rn(g, r)), __dmul_rn(r, G));
                    v = __dadd_rn(__dsub_rn(v, __dmul_rn(v, r)), __dmul_rn(r, __dmul_rn(G, G)));
                    stau[j] = tau; sg[j] = g; sv[j] = v;
                }
                const double minv = __ddiv_rn(1.0, __dadd_rn(__dsqrt_rn(v), a.eps));
                const double ns2 = __dsub_rn(__dmul_rn(__dmul_rn(__dmul_rn(2.0, lr2), a.mdecay), minv), lr4);
                const double p = __dadd_rn(__dsub_rn(__dsub_rn(sp[j], __dmul_rn(__dmul_rn(lr2, minv), G)),
                                                     __dmul_rn(a.mdecay, sp[j])),
                                           __dmul_rn(__dsqrt_rn(fmax(ns2, 1e-16)), z[e2]));
                sp[j] = p;
                th[j] = __dadd_rn(th[j], p);
            }
        }
        __syncthreads();
        if (s > a.burn_in && (s - a.burn_in) % a.keep_every == 0) {
            double* out = a.samples + (size_t)kept * P;
            for (int j = tid; j < P; j += NT) out[j] = th[j];
            ++kept;
        }
    }
    for (int j = tid; j < P; j += NT) a.state[j] = th[j];
}

struct BnnScoreArgs {
    const double* X; long m; int D, P, S;
    const double* samples;                 // S x P (16-byte aligned rows: P is even)
    const double* xm; const double* xs;    // input mean and std (D each)
    double y_mean, y_std;
    ScoreOut o;
};

// dynamic shared memory of gpk_bnn_score_kernel: the two-stage ring of networks, the scaled candidate tile, 2 mbarriers
__host__ __device__ inline long gpk_bnn_score_smem(int d) {
    return 2L * gpk_bnn_params(d) * 8 + (long)d * GPK_BNN_SCORE_THREADS * GPK_BNN_SCORE_C * 8 + 16;
}

__device__ __forceinline__ void gpk_bnn_bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    mbar_arrive_expect_tx(bar, bytes);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// A CTA scores a tile of GPK_BNN_SCORE_THREADS x GPK_BNN_SCORE_C candidates (thread t: candidates t and t + 128 of the
// tile) and walks the S networks in order.  Network k + 1 is brought into the other stage of a two-stage ring by one 1-D
// TMA bulk copy while network k computes.  Every weight is read from shared memory by a warp-uniform (broadcast) load
// and feeds GPK_BNN_SCORE_C FMAs per thread; the second layer reads W2 two entries at a time (16-byte loads), so one
// load feeds four FMAs.  Layer-1 activations stay in registers; layer 2 streams into the output unit.
__global__ void __launch_bounds__(GPK_BNN_SCORE_THREADS) gpk_bnn_score_kernel(const BnnScoreArgs a)
{
    constexpr int NT = GPK_BNN_SCORE_THREADS, C = GPK_BNN_SCORE_C, H = GPK_BNN_H, TILE = NT * C;
    extern __shared__ __align__(16) double ssm[];
    const int tid = threadIdx.x, D = a.D, P = a.P;
    double* ring = ssm;                                   // 2 x P
    double* xt = ring + 2L * P;                           // [d][TILE] scaled candidates
    const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(xt + (long)D * TILE);
    const uint32_t ring_s = (uint32_t)__cvta_generic_to_shared(ring);
    const uint32_t bytes = (uint32_t)P * 8u;
    const long c0 = (long)blockIdx.x * TILE;
    if (tid == 0) {
        mbar_init(bar0, 1);
        mbar_init(bar0 + 8, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (tid == 0) {
        gpk_bnn_bulk_load(ring_s, a.samples, bytes, bar0);
        if (a.S > 1) gpk_bnn_bulk_load(ring_s + bytes, a.samples + P, bytes, bar0 + 8);
    }
    for (int q = tid; q < D * TILE; q += NT) {
        const int d = q / TILE, r = q - d * TILE;
        const long c = c0 + r;
        xt[q] = c < a.m ? __ddiv_rn(__dsub_rn(a.X[c * D + d], a.xm[d]), a.xs[d]) : 0.0;
    }
    __syncthreads();

    const int oB1 = H * D, oW2 = oB1 + H, oB2 = oW2 + H * H, oW3 = oB2 + H, oB3 = oW3 + H, oLV = oB3 + 1;
    double mean[C], m2[C];
#pragma unroll
    for (int c = 0; c < C; ++c) { mean[c] = 0.0; m2[c] = 0.0; }
    double sum_ev = 0.0;
    for (int k = 0; k < a.S; ++k) {
        const int st = k & 1;
        while (!mbar_try_wait(bar0 + 8 * st, (uint32_t)((k >> 1) & 1))) {}
        const double* W = ring + (long)st * P;
        double h[C][H];
#pragma unroll
        for (int j = 0; j < H; ++j) {
            const double b = W[oB1 + j];
#pragma unroll
            for (int c = 0; c < C; ++c) h[c][j] = b;
        }
#pragma unroll 1
        for (int dd = 0; dd < D; ++dd) {
            double xv[C];
#pragma unroll
            for (int c = 0; c < C; ++c) xv[c] = xt[dd * TILE + c * NT + tid];
#pragma unroll
            for (int j = 0; j < H; ++j) {
                const double w = W[j * D + dd];
#pragma unroll
                for (int c = 0; c < C; ++c) h[c][j] = fma(w, xv[c], h[c][j]);
            }
        }
#pragma unroll
        for (int j = 0; j < H; ++j)
#pragma unroll
            for (int c = 0; c < C; ++c) h[c][j] = tanh(h[c][j]);
        double f[C];
        const double b3 = W[oB3];
#pragma unroll
        for (int c = 0; c < C; ++c) f[c] = b3;
#pragma unroll 1
        for (int j = 0; j < H; ++j) {
            const double2* w2 = reinterpret_cast<const double2*>(W + oW2 + j * H);
            double acc[C];
            const double b2 = W[oB2 + j];
#pragma unroll
            for (int c = 0; c < C; ++c) acc[c] = b2;
#pragma unroll
            for (int k2 = 0; k2 < H / 2; ++k2) {
                const double2 w = w2[k2];
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    acc[c] = fma(w.x, h[c][2 * k2], acc[c]);
                    acc[c] = fma(w.y, h[c][2 * k2 + 1], acc[c]);
                }
            }
            const double w3 = W[oW3 + j];
#pragma unroll
            for (int c = 0; c < C; ++c) f[c] = fma(w3, tanh(acc[c]), f[c]);
        }
        sum_ev += exp(W[oLV]);
        const double inv = 1.0 / (double)(k + 1);
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const double dl = f[c] - mean[c];
            mean[c] = fma(dl, inv, mean[c]);
            m2[c] = fma(dl, f[c] - mean[c], m2[c]);
        }
        __syncthreads();                                  // every thread is done with stage st
        if (tid == 0 && k + 2 < a.S) {
            fence_proxy_async();
            gpk_bnn_bulk_load(ring_s + st * bytes, a.samples + (size_t)(k + 2) * P, bytes, bar0 + 8 * st);
        }
    }

    double val = 0.0;
    long long idx = -1;
    const double Sd = (double)a.S, ys2 = a.y_std * a.y_std, vev = sum_ev / Sd;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const long ci = c0 + c * NT + tid;
        if (ci >= a.m) continue;
        const double mu = fma(mean[c], a.y_std, a.y_mean);
        const double var = (m2[c] / Sd + vev) * ys2;
        double v = 0.0;
        long long vi = -1;
        gpk_score_emit(a.o, ci, mu, var, v, vi);
        if (gpk_better(v, vi, val, idx)) { val = v; idx = vi; }
    }
    if (a.o.acq_kind == GPK_ACQ_NONE) return;
    gpk_block_best<NT / 32>(val, idx);
    if (tid == 0) a.o.block_best[blockIdx.x] = {val, idx};
}
