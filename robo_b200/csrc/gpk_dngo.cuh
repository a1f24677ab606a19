// gpk_dngo.cuh — DNGO on the device (Snoek et al., "Scalable Bayesian Optimization Using Deep Neural Networks", ICML
// 2015; pybnn's DNGO, which robo/fmin/bayesian_optimization.py:105-109 takes as model_type="dngo"): a tanh feature
// network trained by Adam in one launch, Bayesian linear regression over its last hidden layer (gpk_blr.cuh, reused as it
// stands), and the collapsed predictive scoring candidates for every device maximizer.  pybnn's dngo.py is not available,
// so the model is restated here, in tests/dngo_model.py and in DESIGN §1 row a29; the pybnn details below are this
// project's statement, not checked against pybnn.
//
// Network: Linear(D, 50) . tanh . Linear(50, 50) . tanh . Linear(50, 50) . tanh . Linear(50, 1), in fp64 (pybnn trains
// in float32).  theta, P = 50 D + 5201 doubles, in this order: W1 (50 x D, row j = unit j), b1 (50), W2 (50 x 50), b2,
// W3 (50 x 50), b3, W4 (50), b4.  Initialisation (torch's nn.Linear default): every weight and bias of a layer with
// fan_in inputs is (2 u - 1) / sqrt(fan_in), u = gpk_u01 of words 0, 1 of Philox4x32-10 keyed by the 64-bit seed with
// counter (p, 0, counter, GPK_DNGO_TAG_INIT), p the parameter's index in theta.
//
// Data: gpk_dngo_set_data scales X per column and y to zero mean and unit population std on the host, with
// gpk_bnn_set_data's code; with a flag off that side keeps mean 0 and std 1 (used as given).
//
// Batches: B = min(batch, N) rows; epoch e visits the rows in the ranks of (Philox word 0 of (row, e, counter,
// GPK_DNGO_TAG_ORDER), row) in floor(N / B) full batches and drops the remaining N mod B rows of that epoch (pybnn's
// iterate_minibatches).  num_epochs epochs: t = 1 .. num_epochs floor(N / B) Adam steps.
//
// Gradient of the batch loss L = mean_i (f_i - y_i)^2 (every product, sum, quotient and square root rounded once,
// __dmul_rn / __dadd_rn / __ddiv_rn / __dsqrt_rn, never contracted; a "sum" starts at the bias, or at +0.0, and adds
// the terms in ascending index):
//   h1 = tanh(b1_j + sum_d W1_jd x_d); h2 = tanh(b2_j + sum_k W2_jk h1_k); h3 = tanh(b3_j + sum_k W3_jk h2_k)
//   f = b4 + sum_j W4_j h3_j;  df_i = (2 (f_i - y_i)) / B
//   G_b4 = sum_i df_i, G_W4_j = sum_i df_i h3_ij;  d3_ij = (df_i W4_j) (1 - h3_ij h3_ij)
//   G_b3_j = sum_i d3_ij, G_W3_jk = sum_i d3_ij h2_ik;  d2_ik = (sum_j d3_ij W3_jk) (1 - h2_ik h2_ik)
//   G_b2_j = sum_i d2_ij, G_W2_jk = sum_i d2_ij h1_ik;  d1_ik = (sum_j d2_ij W2_jk) (1 - h1_ik h1_ik)
//   G_b1_k = sum_i d1_ik, G_W1_kd = sum_i d1_ik x_id
// tanh is gpk_bnn_tanh.
//
// Adam (torch.optim.Adam's single-tensor update, beta1 = 0.9, beta2 = 0.999, eps = 1e-8, no weight decay), per parameter
// at step t, with m = v = 0 and running products p1 = p2 = 1 at the start:
//   p1 = p1 beta1; p2 = p2 beta2; m = m + (1 - beta1) (G - m); v = v beta2 + ((1 - beta2) G) G
//   theta = theta - (lr / (1 - p1)) (m / (sqrt(v) / sqrt(1 - p2) + eps))
// 1 - beta1 and 1 - beta2 are the rounded doubles.  torch takes beta^t by pow and may fuse its lerp / addcmul.
//
// gpk_dngo_train_kernel runs every epoch in one CTA: theta, its gradient, the batch and its activations stay in shared
// memory; one thread owns a parameter in the update, and its m and v live in the handle's state buffer.  The kernel
// ends by writing the features Theta (N x 50, the third tanh layer over the scaled training rows in row order), which
// gpk_blr_gram_kernel turns into the Bayesian linear regression's G = Theta^T Theta and b = Theta^T y.
//
// Predict: with the BLR fit's (m_i, S_i, beta_i), i < k, gpk_dngo_collapse_kernel forms m_bar = mean m_i, Q = mean S_i +
// (1 / k) sum (m_i - m_bar)(m_i - m_bar)^T, its Cholesky factor R (gpk_blr_factor) and c_bar = mean 1 / beta_i, so that
// the mixture's mean and full variance at features phi are m = phi^T m_bar and v = c_bar + ||R^T phi||^2 (the mixture
// mean over i of mu_i^2 + var_i minus m^2, with mu_i = phi^T m_i and var_i = 1 / beta_i + phi^T S_i phi).  v is clipped
// to DBL_EPSILON, then m y_std + y_mean and v y_std^2.  Scoring (gpk_dngo_score_kernel) uses fma and libdevice tanh; it is
// pinned by tolerance, not bit for bit.
#pragma once
#include "gpk_internal.cuh"
#include "gpk_kernels.cuh"
#include "gpk_blr.cuh"
#include "gpk_bnn.cuh"

#define GPK_DNGO_H 50                     // units per hidden layer: the BLR's F
#define GPK_DNGO_THREADS 256              // threads of the training kernel
#define GPK_DNGO_SCORE_THREADS 256        // threads (one candidate each) of the scoring kernel
#define GPK_DNGO_TAG_INIT 0x444E0001u
#define GPK_DNGO_TAG_ORDER 0x444E0002u
#define GPK_DNGO_BETA1 0.9
#define GPK_DNGO_BETA2 0.999
#define GPK_DNGO_ADAM_EPS 1e-8

__host__ __device__ inline int gpk_dngo_params(int d) { return GPK_DNGO_H * d + 5201; }

// offsets of the layers in theta
struct DngoLayout {
    int W1, b1, W2, b2, W3, b3, W4, b4;
    __host__ __device__ explicit DngoLayout(int d) {
        constexpr int H = GPK_DNGO_H;
        W1 = 0; b1 = H * d; W2 = b1 + H; b2 = W2 + H * H; W3 = b2 + H; b3 = W3 + H * H; W4 = b3 + H; b4 = W4 + H;
    }
};

struct DngoTrainArgs {
    const double* X; const double* y;      // scaled training set, N x D and N
    int n, d, P, B, epochs;
    unsigned long long seed; unsigned counter;
    double lr;
    double* state;                         // Adam's m and v (P each)
    double* net;                           // theta after the last step (P)
    double* Theta;                         // N x 50 features
};

// dynamic shared memory of gpk_dngo_train_kernel: theta, gradient, batch inputs and targets, three activations and two
// delta buffers (B x 50 each), df, then the epoch order (8 + 4 bytes per row)
__host__ __device__ inline long gpk_dngo_train_doubles(int d, int B) {
    return 2L * gpk_dngo_params(d) + (long)B * (d + 2) + 5L * B * GPK_DNGO_H;
}
__host__ __device__ inline long gpk_dngo_train_smem(int n, int d, int B) {
    return gpk_dngo_train_doubles(d, B) * 8 + 12L * n;
}

// the three tanh layers over Bt rows xb (Bt x D) into h1, h2, h3 (Bt x 50 each), on the whole CTA
__device__ __forceinline__ void gpk_dngo_forward(const double* th, const DngoLayout& L, int D, int Bt, const double* xb, double* h1,
                                 double* h2, double* h3)
{
    constexpr int NT = GPK_DNGO_THREADS, H = GPK_DNGO_H;
    const int tid = threadIdx.x;
    for (int q = tid; q < Bt * H; q += NT) {
        const int i = q / H, j = q - i * H;
        double acc = th[L.b1 + j];
        for (int k = 0; k < D; ++k) acc = __dadd_rn(acc, __dmul_rn(th[L.W1 + j * D + k], xb[i * D + k]));
        h1[q] = gpk_bnn_tanh(acc);
    }
    __syncthreads();
    for (int q = tid; q < Bt * H; q += NT) {
        const int i = q / H, j = q - i * H;
        double acc = th[L.b2 + j];
        for (int k = 0; k < H; ++k) acc = __dadd_rn(acc, __dmul_rn(th[L.W2 + j * H + k], h1[i * H + k]));
        h2[q] = gpk_bnn_tanh(acc);
    }
    __syncthreads();
    for (int q = tid; q < Bt * H; q += NT) {
        const int i = q / H, j = q - i * H;
        double acc = th[L.b3 + j];
        for (int k = 0; k < H; ++k) acc = __dadd_rn(acc, __dmul_rn(th[L.W3 + j * H + k], h2[i * H + k]));
        h3[q] = gpk_bnn_tanh(acc);
    }
    __syncthreads();
}

__global__ void __launch_bounds__(GPK_DNGO_THREADS) gpk_dngo_train_kernel(const DngoTrainArgs a)
{
    constexpr int NT = GPK_DNGO_THREADS, H = GPK_DNGO_H;
    extern __shared__ double dsm[];
    const int tid = threadIdx.x, N = a.n, D = a.d, P = a.P, B = a.B;
    const DngoLayout L(D);
    double* th = dsm;                       // theta
    double* gr = th + P;                    // gradient
    double* xb = gr + P;                    // batch inputs, B x D
    double* yb = xb + (long)B * D;          // batch targets
    double* h1 = yb + B;                    // B x 50 each
    double* h2 = h1 + B * H;
    double* h3 = h2 + B * H;
    double* da = h3 + B * H;                // d3, then d1
    double* db = da + B * H;                // d2
    double* df = db + B * H;                // B
    unsigned long long* keys = (unsigned long long*)(df + B);
    int* order = (int*)(keys + N);
    double* sm = a.state;
    double* sv = sm + P;
    const double w1 = __dsub_rn(1.0, GPK_DNGO_BETA1), w2 = __dsub_rn(1.0, GPK_DNGO_BETA2), Bd = (double)B;

    // initial weights and Adam state
    {
        const double bd = __ddiv_rn(1.0, __dsqrt_rn((double)D)), bh = __ddiv_rn(1.0, __dsqrt_rn((double)H));
        for (int j = tid; j < P; j += NT) {
            uint32_t w[4];
            gpk_philox4x32_10((uint32_t)j, 0u, a.counter, GPK_DNGO_TAG_INIT, (uint32_t)a.seed, (uint32_t)(a.seed >> 32), w);
            const double u = gpk_u01(w[0], w[1]);
            th[j] = __dmul_rn(__dsub_rn(__dmul_rn(2.0, u), 1.0), j < L.W2 ? bd : bh);
            sm[j] = 0.0; sv[j] = 0.0;
        }
    }
    __syncthreads();

    const int nb = N / B;
    double p1 = 1.0, p2 = 1.0;
    for (int e = 0; e < a.epochs; ++e) {
        // the epoch's order: ranks of (key, row)
        for (int i = tid; i < N; i += NT) {
            uint32_t w[4];
            gpk_philox4x32_10((uint32_t)i, (uint32_t)e, a.counter, GPK_DNGO_TAG_ORDER, (uint32_t)a.seed,
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
        for (int bi = 0; bi < nb; ++bi) {
            const int pos0 = bi * B;
            for (int q = tid; q < B * D; q += NT) {
                const int i = q / D;
                xb[q] = a.X[(long)order[pos0 + i] * D + (q - i * D)];
            }
            for (int i = tid; i < B; i += NT) yb[i] = a.y[order[pos0 + i]];
            __syncthreads();
            gpk_dngo_forward(th, L, D, B, xb, h1, h2, h3);
            for (int i = tid; i < B; i += NT) {
                double f = th[L.b4];
                for (int j = 0; j < H; ++j) f = __dadd_rn(f, __dmul_rn(th[L.W4 + j], h3[i * H + j]));
                df[i] = __ddiv_rn(__dmul_rn(2.0, __dsub_rn(f, yb[i])), Bd);
            }
            __syncthreads();
            // the output layer's gradient and d3
            for (int q = tid; q < B * H + H + 1; q += NT) {
                if (q < B * H) {
                    const int i = q / H, j = q - i * H;
                    da[q] = __dmul_rn(__dmul_rn(df[i], th[L.W4 + j]), __dsub_rn(1.0, __dmul_rn(h3[q], h3[q])));
                } else if (q < B * H + H) {
                    const int j = q - B * H;
                    double acc = 0.0;
                    for (int i = 0; i < B; ++i) acc = __dadd_rn(acc, __dmul_rn(df[i], h3[i * H + j]));
                    gr[L.W4 + j] = acc;
                } else {
                    double acc = 0.0;
                    for (int i = 0; i < B; ++i) acc = __dadd_rn(acc, df[i]);
                    gr[L.b4] = acc;
                }
            }
            __syncthreads();
            // hidden layers 3 and 2: the layer's gradient from the deltas `din` over inputs `hin`, and the deltas below
            for (int layer = 3; layer >= 2; --layer) {
                const double* din = layer == 3 ? da : db;
                double* dout = layer == 3 ? db : da;
                const double* hin = layer == 3 ? h2 : h1;
                const int oW = layer == 3 ? L.W3 : L.W2, ob = layer == 3 ? L.b3 : L.b2;
                for (int q = tid; q < B * H + H * H + H; q += NT) {
                    if (q < B * H) {
                        const int i = q / H, k = q - i * H;
                        double acc = 0.0;
                        for (int j = 0; j < H; ++j) acc = __dadd_rn(acc, __dmul_rn(din[i * H + j], th[oW + j * H + k]));
                        dout[q] = __dmul_rn(acc, __dsub_rn(1.0, __dmul_rn(hin[q], hin[q])));
                    } else if (q < B * H + H * H) {
                        const int jk = q - B * H, j = jk / H, k = jk - j * H;
                        double acc = 0.0;
                        for (int i = 0; i < B; ++i) acc = __dadd_rn(acc, __dmul_rn(din[i * H + j], hin[i * H + k]));
                        gr[oW + jk] = acc;
                    } else {
                        const int j = q - B * H - H * H;
                        double acc = 0.0;
                        for (int i = 0; i < B; ++i) acc = __dadd_rn(acc, din[i * H + j]);
                        gr[ob + j] = acc;
                    }
                }
                __syncthreads();
            }
            // the first layer's gradient (d1 in da)
            for (int q = tid; q < H * D + H; q += NT) {
                double acc = 0.0;
                if (q < H * D) {
                    const int j = q / D, k = q - j * D;
                    for (int i = 0; i < B; ++i) acc = __dadd_rn(acc, __dmul_rn(da[i * H + j], xb[i * D + k]));
                    gr[L.W1 + q] = acc;
                } else {
                    const int j = q - H * D;
                    for (int i = 0; i < B; ++i) acc = __dadd_rn(acc, da[i * H + j]);
                    gr[L.b1 + j] = acc;
                }
            }
            __syncthreads();
            // Adam, one parameter per thread
            p1 = __dmul_rn(p1, GPK_DNGO_BETA1);
            p2 = __dmul_rn(p2, GPK_DNGO_BETA2);
            const double ss = __ddiv_rn(a.lr, __dsub_rn(1.0, p1)), c2 = __dsqrt_rn(__dsub_rn(1.0, p2));
            for (int j = tid; j < P; j += NT) {
                const double G = gr[j];
                const double m = __dadd_rn(sm[j], __dmul_rn(w1, __dsub_rn(G, sm[j])));
                const double v = __dadd_rn(__dmul_rn(sv[j], GPK_DNGO_BETA2), __dmul_rn(__dmul_rn(w2, G), G));
                sm[j] = m; sv[j] = v;
                const double den = __dadd_rn(__ddiv_rn(__dsqrt_rn(v), c2), GPK_DNGO_ADAM_EPS);
                th[j] = __dsub_rn(th[j], __dmul_rn(ss, __ddiv_rn(m, den)));
            }
            __syncthreads();
        }
    }
    for (int j = tid; j < P; j += NT) a.net[j] = th[j];
    // Theta over the training rows, B at a time in row order
    for (int r0 = 0; r0 < N; r0 += B) {
        const int Bt = min(B, N - r0);
        for (int q = tid; q < Bt * D; q += NT) xb[q] = a.X[(long)r0 * D + q];
        __syncthreads();
        gpk_dngo_forward(th, L, D, Bt, xb, h1, h2, h3);
        for (int q = tid; q < Bt * H; q += NT) a.Theta[(long)r0 * H + q] = h3[q];
        __syncthreads();
    }
}

// Theta (m x 50) of the rows X (m x D): one CTA of 64 threads per row, the training kernel's arithmetic.  xm / xs: the
// input scaling ((x - xm) / xs), or NULL for rows already scaled
__global__ void __launch_bounds__(64) gpk_dngo_features_kernel(const double* __restrict__ X, long m, int D,
                                                               const double* __restrict__ xm,
                                                               const double* __restrict__ xs,
                                                               const double* __restrict__ th, double* __restrict__ out)
{
    constexpr int H = GPK_DNGO_H;
    __shared__ double x[GPK_DNGO_MAX_D], a1[H], a2[H];
    const long r = blockIdx.x;
    const int j = threadIdx.x;
    const DngoLayout L(D);
    if (j < D) {
        const double v = X[r * D + j];
        x[j] = xm ? __ddiv_rn(__dsub_rn(v, xm[j]), xs[j]) : v;
    }
    __syncthreads();
    if (j < H) {
        double acc = th[L.b1 + j];
        for (int k = 0; k < D; ++k) acc = __dadd_rn(acc, __dmul_rn(th[L.W1 + j * D + k], x[k]));
        a1[j] = gpk_bnn_tanh(acc);
    }
    __syncthreads();
    if (j < H) {
        double acc = th[L.b2 + j];
        for (int k = 0; k < H; ++k) acc = __dadd_rn(acc, __dmul_rn(th[L.W2 + j * H + k], a1[k]));
        a2[j] = gpk_bnn_tanh(acc);
    }
    __syncthreads();
    if (j < H) {
        double acc = th[L.b3 + j];
        for (int k = 0; k < H; ++k) acc = __dadd_rn(acc, __dmul_rn(th[L.W3 + j * H + k], a2[k]));
        out[r * H + j] = gpk_bnn_tanh(acc);
    }
}

// the offset of R's row j in the scoring pack's R section: the rows before it, each padded to an even length
__host__ __device__ constexpr int gpk_dngo_rrow(int j) { return (j % 2 == 0) ? j * (j + 2) / 2 : (j + 1) * (j + 1) / 2; }

// The scoring pack (doubles) gpk_dngo_collapse_kernel writes and gpk_dngo_score_kernel copies to shared memory: the
// first three layers transposed (W^T: row k holds the 50 weights of input k), their biases, m_bar, c_bar (and a pad),
// then R's rows, row j padded to an even length (every section and row starts 16-byte aligned)
struct DngoPack {
    int W1, b1, W2, b2, W3, b3, mb, cb, R, total;
    __host__ __device__ explicit DngoPack(int d) {
        constexpr int H = GPK_DNGO_H;
        W1 = 0; b1 = H * d; W2 = b1 + H; b2 = W2 + H * H; W3 = b2 + H; b3 = W3 + H * H; mb = b3 + H; cb = mb + H;
        R = cb + 2; total = R + gpk_dngo_rrow(H);
    }
};

// doubles of dynamic shared memory of gpk_dngo_collapse_kernel: Q, gpk_blr_factor's A, m and col, then b = 0
__host__ __device__ inline long gpk_dngo_collapse_doubles() {
    return 2L * GPK_DNGO_H * GPK_DNGO_H + 3L * (GPK_DNGO_H + 1);
}

// One CTA: from the BLR fit's M (k x 50), S (k x 50 x 50) and ib (k) and the net, the scoring pack; *fail = 1 where Q's
// factorisation meets a pivot that is not > 0.  Sums over i in ascending order.
__global__ void __launch_bounds__(GPK_BLR_THREADS) gpk_dngo_collapse_kernel(const double* __restrict__ M,
                                                                            const double* __restrict__ S,
                                                                            const double* __restrict__ ib, int k,
                                                                            const double* __restrict__ th, int D,
                                                                            double* __restrict__ pack,
                                                                            int* __restrict__ fail)
{
    constexpr int H = GPK_DNGO_H, NT = GPK_BLR_THREADS;
    extern __shared__ double csm[];
    double* Q = csm;
    double* A = Q + H * H;                    // Q's factor
    double* m = A + H * H;                    // gpk_blr_factor's m (H + 1)
    double* col = m + (H + 1);                // its column (H + 1)
    double* zb = col + (H + 1);               // b = 0
    const int tid = threadIdx.x;
    const DngoLayout L(D);
    const DngoPack K(D);
    const double kd = (double)k;
    // the net's layers, transposed
    for (int q = tid; q < H * D; q += NT) {
        const int dd = q / H, j = q - dd * H;
        pack[K.W1 + q] = th[L.W1 + j * D + dd];
    }
    for (int q = tid; q < H * H; q += NT) {
        const int kk = q / H, j = q - kk * H;
        pack[K.W2 + q] = th[L.W2 + j * H + kk];
        pack[K.W3 + q] = th[L.W3 + j * H + kk];
    }
    for (int j = tid; j < H; j += NT) {
        pack[K.b1 + j] = th[L.b1 + j]; pack[K.b2 + j] = th[L.b2 + j]; pack[K.b3 + j] = th[L.b3 + j];
        double s = 0.0;
        for (int i = 0; i < k; ++i) s += M[(long)i * H + j];
        m[j] = s / kd;
        zb[j] = 0.0;
    }
    __syncthreads();
    for (int e = tid; e < H * H; e += NT) {
        const int r = e / H, c = e - r * H;
        double s = 0.0, o = 0.0;
        for (int i = 0; i < k; ++i) {
            s += S[(long)i * H * H + e];
            o = fma(M[(long)i * H + r] - m[r], M[(long)i * H + c] - m[c], o);
        }
        Q[e] = s / kd + o / kd;
    }
    for (int j = tid; j < H; j += NT) pack[K.mb + j] = m[j];
    if (tid == 0) {
        double s = 0.0;
        for (int i = 0; i < k; ++i) s += ib[i];
        pack[K.cb] = s / kd;
        pack[K.cb + 1] = 0.0;
    }
    __syncthreads();                          // m is gpk_blr_factor's scratch from here on
    const bool ok = gpk_blr_factor(Q, zb, H, 0.0, 1.0, A, col, m);      // A = fl(fl(1 Q) + 0 I) = Q
    if (tid == 0) *fail = ok ? 0 : 1;
    if (!ok) return;
    for (int j = tid; j < H; j += NT) {
        double* row = pack + K.R + gpk_dngo_rrow(j);
        for (int c = 0; c <= j; ++c) row[c] = A[j * H + c];
        if (j % 2 == 0) row[j + 1] = 0.0;
    }
}

struct DngoScoreArgs {
    const double* X; long m; int D, ntiles;
    const double* pack; int pack_doubles;
    const double* xm; const double* xs;    // input mean and std (D each)
    double y_mean, y_std;
    ScoreOut o;
};

// dynamic shared memory of gpk_dngo_score_kernel: the pack and every thread's column of 50 activations
__host__ __device__ inline long gpk_dngo_score_smem(int d) {
    return ((long)DngoPack(d).total + 1) / 2 * 16 + (long)GPK_DNGO_H * GPK_DNGO_SCORE_THREADS * 8;
}

// one layer of 50 units on one candidate: acc_j = b_j + sum_k W_jk in_k with W^T's rows (16-byte loads, each broadcast
// over the warp) and the inputs in the thread's shared-memory column; then the tanh of each back into the column
__device__ __forceinline__ void gpk_dngo_score_layer(const double* __restrict__ Wt, const double* __restrict__ b,
                                                     double* col, double (&acc)[GPK_DNGO_H])
{
    constexpr int H = GPK_DNGO_H, NT = GPK_DNGO_SCORE_THREADS;
#pragma unroll
    for (int j = 0; j < H; ++j) acc[j] = b[j];
#pragma unroll 1
    for (int k = 0; k < H; ++k) {
        const double a = col[k * NT];
        const double2* w = reinterpret_cast<const double2*>(Wt + k * H);
#pragma unroll
        for (int j2 = 0; j2 < H / 2; ++j2) {
            const double2 v = w[j2];
            acc[2 * j2] = fma(v.x, a, acc[2 * j2]);
            acc[2 * j2 + 1] = fma(v.y, a, acc[2 * j2 + 1]);
        }
    }
#pragma unroll
    for (int j = 0; j < H; ++j) col[j * NT] = tanh(acc[j]);
}

// Each CTA copies the pack to shared memory once, then scores tiles blockIdx.x, blockIdx.x + gridDim.x, ... of
// GPK_DNGO_SCORE_THREADS candidates, one per thread: the scaled candidate through the three layers to phi, then
// m = phi^T m_bar and v = c_bar + ||R^T phi||^2 (t_r = sum_{j >= r} R_jr phi_j accumulated in registers over j), the clip,
// the de-normalisation and gpk_score_emit; the CTA's arg-max over all its tiles goes to block_best[blockIdx.x].
__global__ void __launch_bounds__(GPK_DNGO_SCORE_THREADS, 1) gpk_dngo_score_kernel(const DngoScoreArgs a)
{
    constexpr int NT = GPK_DNGO_SCORE_THREADS, H = GPK_DNGO_H;
    extern __shared__ __align__(16) double ssm[];
    const int tid = threadIdx.x, D = a.D;
    const DngoPack K(D);
    double* pk = ssm;
    double* col = ssm + ((long)K.total + 1) / 2 * 2;      // [50][NT]: this thread's column at col + tid
    {
        const double2* src = reinterpret_cast<const double2*>(a.pack);
        double2* dst = reinterpret_cast<double2*>(pk);
        for (int q = tid; q < (K.total + 1) / 2; q += NT) dst[q] = src[q];
    }
    __syncthreads();
    double* mycol = col + tid;
    double val = 0.0;
    long long idx = -1;
    const double ys2 = a.y_std * a.y_std;
    for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
        const long c = (long)tile * NT + tid;
        if (c >= a.m) continue;
        double acc[H];
#pragma unroll
        for (int j = 0; j < H; ++j) acc[j] = pk[K.b1 + j];
#pragma unroll 1
        for (int dd = 0; dd < D; ++dd) {
            const double x = (a.X[c * D + dd] - __ldg(a.xm + dd)) / __ldg(a.xs + dd);
            const double2* w = reinterpret_cast<const double2*>(pk + K.W1 + dd * H);
#pragma unroll
            for (int j2 = 0; j2 < H / 2; ++j2) {
                const double2 v = w[j2];
                acc[2 * j2] = fma(v.x, x, acc[2 * j2]);
                acc[2 * j2 + 1] = fma(v.y, x, acc[2 * j2 + 1]);
            }
        }
#pragma unroll
        for (int j = 0; j < H; ++j) mycol[j * NT] = tanh(acc[j]);
        gpk_dngo_score_layer(pk + K.W2, pk + K.b2, mycol, acc);
        gpk_dngo_score_layer(pk + K.W3, pk + K.b3, mycol, acc);    // the column holds phi
        double mu = 0.0;
#pragma unroll
        for (int r = 0; r < H; ++r) acc[r] = 0.0;
#pragma unroll
        for (int j = 0; j < H; ++j) {
            const double ph = mycol[j * NT];
            mu = fma(pk[K.mb + j], ph, mu);
            const double2* Rj = reinterpret_cast<const double2*>(pk + K.R + gpk_dngo_rrow(j));
#pragma unroll
            for (int r2 = 0; r2 <= j / 2; ++r2) {
                const double2 v = Rj[r2];
                acc[2 * r2] = fma(v.x, ph, acc[2 * r2]);
                if (2 * r2 + 1 <= j) acc[2 * r2 + 1] = fma(v.y, ph, acc[2 * r2 + 1]);
            }
        }
        double q = 0.0;
#pragma unroll
        for (int r = 0; r < H; ++r) q = fma(acc[r], acc[r], q);
        double var = pk[K.cb] + q;
        if (var < GPK_EPS) var = GPK_EPS;                  // NaN stays NaN
        double v = 0.0;
        long long vi = -1;
        gpk_score_emit(a.o, c, fma(mu, a.y_std, a.y_mean), var * ys2, v, vi);
        if (gpk_better(v, vi, val, idx)) { val = v; idx = vi; }
    }
    if (a.o.acq_kind == GPK_ACQ_NONE) return;
    gpk_block_best<NT / 32>(val, idx);
    if (tid == 0) a.o.block_best[blockIdx.x] = {val, idx};
}
