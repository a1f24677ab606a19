// gpk_kernels.cuh — covariance builders, diagonal-block Cholesky/inverse, scoring epilogue.
#pragma once
#include "gpk_internal.cuh"

// ---------------------------------------------------------------------------------------
// Covariance tile builder.  out[c][j] = k(cand_c, train_j)   (row-major, ld = ldo)
//   train side : TERM-major, pre-scaled   Xs[t][j] = x_j[axis_t] * sqrt(c_f / metric_t)   (gpk_termmajor_kernel),
//                one cp.async.bulk.tensor.2d (box n_terms x 128 columns, no swizzle) per CTA into shared memory,
//                completion on an mbarrier; threads read their two train points with one 16-byte LDS per term
//   candidates : row-major raw inputs, scaled (x - lower) / (upper - lower), then by the same per-term factor, while
//                filling shared memory
// so the inner loop is  d = s - x ; q = fma(d, d, q)  : 2 FP64 instructions per (pair, term), and one broadcast LDS per
// CC pairs.  Rows c >= m and columns j >= n are written as exact zeros (padding must not contribute to the contractions
// that follow).  tri != 0: skip tiles entirely above the diagonal (K build).  Used for K (cand = train), K* (scoring),
// K** (full_cov) and kernel.get_value.
// CTA = 128 train points x 4 CC candidates, 256 threads, thread = 2 train points x CC candidates (CC = 8: 128 x 32 tile;
// CC = 4: 128 x 16 tile, <= 64 registers so that a CTA fits next to a resident variance-GEMM CTA).
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cov_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int CC>
__global__ void __launch_bounds__(256, CC == 8 ? 2 : 4)
gpk_cov_tma_kernel(const __grid_constant__ CUtensorMap mapX, const KSpec ks, int n,
                   const double* __restrict__ cand, int dc, long m,
                   const double* __restrict__ lower, const double* __restrict__ upper,
                   double* __restrict__ out, long ldo, int tri)
{
    constexpr int TC = 4 * CC;
    extern __shared__ unsigned char cov_raw[];
    const int tid = threadIdx.x;
    const long c0 = (long)blockIdx.y * TC;
    if (tri && (long)blockIdx.x * 128 > c0 + TC - 1) return;
    const int nt = ks.n_terms;
    const uint32_t base = (cov_smem_u32(cov_raw) + 127u) & ~127u;
    const uint32_t xs = base;                                   // nt x 128 doubles
    const uint32_t scb = xs + (uint32_t)nt * 1024u;             // TC x nt doubles
    const uint32_t bar = scb + (uint32_t)(TC * nt) * 8u;        // 8-byte aligned mbarrier
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"((uint32_t)nt * 1024u) : "memory");
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                     :: "r"(xs), "l"((uint64_t)&mapX), "r"(bar), "r"((int)(blockIdx.x * 128)), "r"(0) : "memory");
    }
    for (int e = tid; e < TC * nt; e += 256) {
        const int c = e / nt, t = e - c * nt;
        const long ci = c0 + c;
        double v = 0.0;
        if (ci < m) {
            const int a = ks.axis[t];
            v = cand[ci * dc + a];
            if (lower != nullptr) v = (v - lower[a]) / (upper[a] - lower[a]);
            v *= ks.scale[t];
        }
        asm volatile("st.shared.f64 [%0], %1;" :: "r"(scb + (uint32_t)e * 8u), "d"(v) : "memory");
    }
    __syncthreads();
    {
        uint32_t ok = 0;
        while (!ok)
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(ok) : "r"(bar) : "memory");
    }
    const int jp = tid & 63, cgp = tid >> 6;
    double q[CC][2], pr[CC][2];
#pragma unroll
    for (int c = 0; c < CC; ++c) { q[c][0] = q[c][1] = 0.0; pr[c][0] = pr[c][1] = 1.0; }
    const uint32_t xrow = xs + (uint32_t)jp * 16u;
    const uint32_t srow = scb + (uint32_t)(cgp * CC * nt) * 8u;
    for (int t = 0; t < nt; ++t) {
        double x0, x1;
        asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(x0), "=d"(x1) : "r"(xrow + (uint32_t)t * 1024u));
#pragma unroll
        for (int c = 0; c < CC; ++c) {
            double sv;
            asm volatile("ld.shared.f64 %0, [%1];" : "=d"(sv) : "r"(srow + (uint32_t)(c * nt + t) * 8u));
            const double d0 = sv - x0, d1 = sv - x1;
            q[c][0] = fma(d0, d0, q[c][0]);
            q[c][1] = fma(d1, d1, q[c][1]);
        }
        if (ks.last[t]) {
#pragma unroll
            for (int c = 0; c < CC; ++c) {
                pr[c][0] *= gpk_radial_q(ks.family, q[c][0]);
                pr[c][1] *= gpk_radial_q(ks.family, q[c][1]);
                q[c][0] = q[c][1] = 0.0;
            }
        }
    }
    const int j0 = blockIdx.x * 128 + 2 * jp;
    const bool v0 = j0 < n, v1 = j0 + 1 < n;
#pragma unroll
    for (int c = 0; c < CC; ++c) {
        const long ci = c0 + cgp * CC + c;
        const bool cv = ci < m;
        double2 o;
        o.x = (cv && v0) ? ks.amp * pr[c][0] : 0.0;
        o.y = (cv && v1) ? ks.amp * pr[c][1] : 0.0;
        *reinterpret_cast<double2*>(out + ci * ldo + j0) = o;
    }
}

// Single-column factor over a tile the builders above wrote: out[c][j] *= gpk_factor_value(z_c, z_j), z the factor's
// coordinate of the candidates (row-major raw inputs cand, bounds lo / up) and of the points (row-major raw inputs
// pts, bounds plo / pup).  Runs only when the kernel has a factor, so the builders, their registers and their bits
// stay those of the kernel without it.  tri != 0: only the tiles the triangular K build wrote (column tile start <= the
// row's 32-row block end).
__global__ void __launch_bounds__(256)
gpk_factor_scale_kernel(const KSpec ks, const double* __restrict__ cand, int dc, long m,
                     const double* __restrict__ lo, const double* __restrict__ up,
                     const double* __restrict__ pts, int dp, int n,
                     const double* __restrict__ plo, const double* __restrict__ pup,
                     double* __restrict__ out, long ldo, int tri)
{
    const int j = blockIdx.x * 128 + (threadIdx.x & 127);
    if (j >= n) return;
    const double zj = gpk_factor_coord(ks.factor, pts + (long)j * dp, plo, pup);
    for (long c = (long)blockIdx.y * 2 + (threadIdx.x >> 7); c < m; c += (long)gridDim.y * 2) {
        if (tri && (long)(j & ~127) > (c | 31)) continue;
        const double zc = gpk_factor_coord(ks.factor, cand + c * dc, lo, up);
        out[c * ldo + j] *= gpk_factor_value(ks.factor, zc, zj);
    }
}

inline size_t cov_tma_smem_bytes(int n_terms, int cc) { return (size_t)n_terms * 1024 + (size_t)4 * cc * n_terms * 8 + 8 + 128; }

// Xs[t][j] = scaled x_j[axis_t] * scale_t  (term-major operand of gpk_cov_tma_kernel), zero padded to ldx columns
__global__ void gpk_termmajor_kernel(const KSpec ks, const double* __restrict__ X, long n, int d,
                                     const double* __restrict__ lower, const double* __restrict__ upper,
                                     double* __restrict__ Xs, long ldx)
{
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    long total = (long)ks.n_terms * ldx;
    if (idx >= total) return;
    int t = (int)(idx / ldx);
    long j = idx - (long)t * ldx;
    double v = 0.0;
    if (j < n) {
        const int a = ks.axis[t];
        v = X[j * d + a];
        if (lower != nullptr) v = (v - lower[a]) / (upper[a] - lower[a]);
        v *= ks.scale[t];
    }
    Xs[idx] = v;
}

// Xt[a][j] = X[j][a] (optionally scaled), zero padded to ldx columns.
__global__ void gpk_transpose_kernel(const double* __restrict__ X, long n, int d,
                                     const double* __restrict__ lower, const double* __restrict__ upper,
                                     double* __restrict__ Xt, long ldx)
{
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    long total = (long)d * ldx;
    if (idx >= total) return;
    int a = (int)(idx / ldx);
    long j = idx - (long)a * ldx;
    double v = 0.0;
    if (j < n) {
        v = X[j * d + a];
        if (lower != nullptr) v = (v - lower[a]) / (upper[a] - lower[a]);
    }
    Xt[idx] = v;
}

// After the K build: diagonal += diag_add (george: yerr^2 + TINY), unit diagonal on padding rows,
// and the augmented right-hand-side row  K[NP][j] = y_j - mean  (so the blocked Cholesky also
// produces z = L^-1 (y - mean) as row NP of the factor; rows NP+1.. stay zero).
__global__ void gpk_kfix_kernel(double* __restrict__ K, long ld, int n, int NP, double diag_add,
                                const double* __restrict__ y, double mean)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= NP) return;
    K[(long)i * ld + i] = (i < n) ? K[(long)i * ld + i] + diag_add : 1.0;
    K[(long)NP * ld + i] = (i < n) ? y[i] - mean : 0.0;
}

// ---------------------------------------------------------------------------------------
// Scoring epilogue: sum the per-row-block partials in fixed order, finish mean / variance,
// apply the output transform + clip (gaussian_process.py:282-294), the acquisition closed form,
// and a per-block arg-max with numpy.argmax tie-breaking.
// ---------------------------------------------------------------------------------------
struct FinishArgs {
    const double* part_mu; const double* part_ssq; long ldpart; int nparts;
    long m;                 // valid candidates in this chunk
    double kss;             // k(x*, x*) = amplitude (stationary kernels)
    // the kernel's factor: k(x*, x*) = kss * gpk_factor_value(z*, z*), z* from the chunk's candidates (row-major raw
    // inputs, cand_dc columns, bounds lo / up)
    KFactor factor;
    const double* cand; int cand_dc; const double* lo; const double* up;
    double mean;            // GP constant mean
    int norm_out; double y_mean, y_std;
    ScoreOut o;             // chunk-local: base is the global index of the chunk's first candidate
};

__global__ void __launch_bounds__(256) gpk_finish_kernel(const FinishArgs f)
{
    const long c = (long)blockIdx.x * 256 + threadIdx.x;
    double val = 0.0;
    long long idx = -1;
    if (c < f.m) {
        double ssq = 0.0, mu = 0.0;
        for (int p = 0; p < f.nparts; ++p) {
            ssq += f.part_ssq[(long)p * f.ldpart + c];
            mu += f.part_mu[(long)p * f.ldpart + c];
        }
        double kss = f.kss;
        if (f.factor.kind != GPK_FACTOR_NONE) {
            const double z = gpk_factor_coord(f.factor, f.cand + c * f.cand_dc, f.lo, f.up);
            kss *= gpk_factor_value(f.factor, z, z);
        }
        double var = kss - ssq;
        mu += f.mean;
        if (f.norm_out) { mu = mu * f.y_std + f.y_mean; var = var * (f.y_std * f.y_std); }
        if (var < GPK_EPS) var = GPK_EPS;                  // np.clip(var, eps, inf); NaN stays NaN
        gpk_score_emit(f.o, c, mu, var, val, idx);
    }
    if (f.o.acq_kind == GPK_ACQ_NONE) return;
    gpk_block_best<8>(val, idx);
    if (threadIdx.x == 0) f.o.block_best[blockIdx.x] = {val, idx};
}

// Mean-only epilogue (gpk_predict_mean): gpk_finish_kernel's mean, with the same fixed-order sum of the per-tile
// partials, constant mean and output transform, and no variance partials.
__global__ void __launch_bounds__(256) gpk_mu_parts_finish_kernel(const double* __restrict__ part_mu, long ldpart,
                                                                  int nparts, long m, double mean, int norm_out,
                                                                  double y_mean, double y_std, double* __restrict__ out)
{
    const long c = (long)blockIdx.x * 256 + threadIdx.x;
    if (c >= m) return;
    double mu = 0.0;
    for (int p = 0; p < nparts; ++p) mu += part_mu[(long)p * ldpart + c];
    mu += mean;
    if (norm_out) mu = mu * y_std + y_mean;
    out[c] = mu;
}

// Final arg-max over block results, merged into *best (which may hold the running best of
// earlier chunks; idx < 0 means empty).
__global__ void __launch_bounds__(256) gpk_argmax_final_kernel(const BestPair* __restrict__ bb, int nblocks,
                                                               BestPair* __restrict__ best)
{
    double val = 0.0;
    long long idx = -1;
    for (int b = threadIdx.x; b < nblocks; b += 256)
        if (gpk_better(bb[b].val, bb[b].idx, val, idx)) { val = bb[b].val; idx = bb[b].idx; }
    gpk_block_best<8>(val, idx);
    if (threadIdx.x == 0 && gpk_better(val, idx, best->val, best->idx)) { best->val = val; best->idx = idx; }
}

// Acquisition closed form on supplied moments (gpk_acq_moments).
__global__ void gpk_acq_moments_kernel(const double* __restrict__ mu, const double* __restrict__ var, long m,
                                       int kind, double eta, double par, double* __restrict__ out,
                                       unsigned long long* n_negative)
{
    long c = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= m) return;
    double v = gpk_acq_value(kind, mu[c], var[c], eta, par);
    out[c] = v;
    if (kind == GPK_ACQ_EI && v < 0.0) atomicAdd(n_negative, 1ULL);
}

// full_cov epilogue: output transform, then (clip != 0) every entry clipped to >= eps
// (gaussian_process.py:282-294 applies the clip to the whole matrix).  clip == 0 keeps the raw posterior
// covariance, negative off-diagonal entries included: what george's sample_conditional draws from
// (gaussian_process.py:324; only predict() clips).
__global__ void gpk_cov_finish_kernel(double* __restrict__ cov, long ld, long m, int norm_out, double y_std, int clip)
{
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= m * m) return;
    long r = idx / m, c = idx - r * m;
    double v = cov[r * ld + c];
    if (norm_out) v *= y_std * y_std;
    if (clip && v < GPK_EPS) v = GPK_EPS;
    cov[r * ld + c] = v;
}


// ---------------------------------------------------------------------------------------
// Marginal-likelihood gradient, trace pass (gaussian_process.py:168-191 with the noise term
// corrected):  d(-ll)/d theta_p = -1/2 sum_ij A_ij dK_ij/d theta_p,  A = alpha alpha^T - K^-1.
// Same tiling as the covariance builder (128 columns j x 32 rows i per CTA, lower tiles only,
// off-diagonal pairs counted twice); dK/d theta is recomputed on the fly and never stored
// (the reference materialises an (N, N, H) array, :181-182).  Per CTA it writes nv = n_terms + 2
// partial sums: [sum w k, sum_t ..., trace A]; a second kernel adds the CTAs in fixed order.
//   dk/d log_amp      = k
//   dk/d log_metric_t = -k * (dlog f / d r2)(r2_g) * (x_t - x'_t)^2 / metric_t      (t in group g)
// With the environment factor k = amp R (c0 + c1 z z'), nv = n_terms + 4: [sum w k, sum_t ..., log_a, log_b, trace A],
//   dk/d log_a = amp R c0,   dk/d log_b = amp R c1 z z'
// With the task factor k = amp R K_t[t_i][t_j] (training tasks are valid indices) the sums above use that k, nv stays
// n_terms + 2; the task entries come from gpk_grad_task_kernel.  FK = the kernel's factor kind (GPK_FACTOR_*): each
// instance compiles the other factors' code out.
// ---------------------------------------------------------------------------------------
template <int FK>
__global__ void __launch_bounds__(256)
gpk_grad_trace_kernel(const KSpec ks, const double* __restrict__ Xt, long ldx, int n,
                      const double* __restrict__ Xrow, int dc,
                      const double* __restrict__ Kinv, long ldk, const double* __restrict__ alpha,
                      double* __restrict__ part)
{
    __shared__ double sc[32][GPK_MAX_TERMS + 1];
    __shared__ double szc[32];
    __shared__ double red[8];
    const int tid = threadIdx.x;
    const int nt = ks.n_terms, nv = nt + (FK == GPK_FACTOR_ENV ? 4 : 2);
    const int fax = ks.factor.axis;
    const long bid = (long)blockIdx.y * gridDim.x + blockIdx.x;
    const int j = blockIdx.x * 128 + (tid & 127);
    const long c0 = (long)blockIdx.y * 32;
    if ((long)blockIdx.x * 128 > c0 + 31) {                  // tile entirely above the diagonal
        if (tid < nv) part[bid * nv + tid] = 0.0;
        return;
    }
    for (int e = tid; e < 32 * nt; e += 256) {
        int c = e / nt, t = e - c * nt;
        long ci = c0 + c;
        sc[c][t] = (ci < n) ? Xrow[ci * dc + ks.axis[t]] : 0.0;
    }
    if (FK != GPK_FACTOR_NONE && tid < 32) szc[tid] = (c0 + tid < n) ? Xrow[(c0 + tid) * dc + fax] : 0.0;
    __syncthreads();

    const int cg = (tid >> 7) * 16;
    const bool jv = j < n;
    double gl[GPK_MAX_TERMS];                                // per-term partial sums (local memory)
    for (int t = 0; t < nt; ++t) gl[t] = 0.0;
    double gamp = 0.0, gtr = 0.0, genva = 0.0, genvb = 0.0;
    const double zj = (FK != GPK_FACTOR_NONE && jv) ? Xt[(long)fax * ldx + j] : 0.0;

    double r2[16], wk[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) { r2[c] = 0.0; wk[c] = 1.0; }
    for (int t = 0; t < nt; ++t) {                           // pass 1: k(x_i, x_j) / amp
        const double xj = jv ? Xt[(long)ks.axis[t] * ldx + j] : 0.0;
        const double im = ks.inv_metric[t];
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            double d = sc[cg + c][t] - xj;
            r2[c] = fma(d * d, im, r2[c]);
        }
        if (ks.last[t]) {
#pragma unroll
            for (int c = 0; c < 16; ++c) { wk[c] *= gpk_radial(ks.family, r2[c]); r2[c] = 0.0; }
        }
    }
#pragma unroll
    for (int c = 0; c < 16; ++c) {                           // weights w_ij * k_ij
        const long i = c0 + cg + c;
        double w = 0.0;
        if (jv && i < n && j <= i) {
            const double a = alpha[i] * alpha[j] - Kinv[i * ldk + j];
            if (i == j) { gtr += a; w = a; } else w = 2.0 * a;
        }
        wk[c] = w * ks.amp * wk[c];
        if constexpr (FK == GPK_FACTOR_ENV) {
            const double zc = szc[cg + c];
            genva = fma(wk[c], ks.factor.c0, genva);
            genvb = fma(wk[c], ks.factor.c1 * zc * zj, genvb);
            wk[c] *= gpk_env(ks.factor.c0, ks.factor.c1, zc, zj);
        } else if constexpr (FK == GPK_FACTOR_TASK) {
            wk[c] *= ks.factor.K[(int)szc[cg + c] * ks.factor.n_tasks + (int)zj];
        }
        gamp += wk[c];
    }
    int t0 = 0;
    while (t0 < nt) {                                        // pass 2: group by group
        int t1 = t0;
        while (!ks.last[t1]) ++t1;
#pragma unroll
        for (int c = 0; c < 16; ++c) r2[c] = 0.0;
        for (int t = t0; t <= t1; ++t) {
            const double xj = jv ? Xt[(long)ks.axis[t] * ldx + j] : 0.0;
            const double im = ks.inv_metric[t];
#pragma unroll
            for (int c = 0; c < 16; ++c) {
                double d = sc[cg + c][t] - xj;
                r2[c] = fma(d * d, im, r2[c]);
            }
        }
        double coef[16];
#pragma unroll
        for (int c = 0; c < 16; ++c) coef[c] = -wk[c] * gpk_radial_dlog(ks.family, r2[c]);
        for (int t = t0; t <= t1; ++t) {
            const double xj = jv ? Xt[(long)ks.axis[t] * ldx + j] : 0.0;
            double sacc = 0.0;
#pragma unroll
            for (int c = 0; c < 16; ++c) {
                double d = sc[cg + c][t] - xj;
                sacc = fma(coef[c], d * d, sacc);
            }
            gl[t] += sacc * ks.inv_metric[t];
        }
        t0 = t1 + 1;
    }
    // block reduction of the nv values (fixed order: lanes, then warps)
    for (int v = 0; v < nv; ++v) {
        double x = (v == 0) ? gamp : (v == nv - 1 ? gtr : (v <= nt ? gl[v - 1] : (v == nt + 1 ? genva : genvb)));
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
        if ((tid & 31) == 0) red[tid >> 5] = x;
        __syncthreads();
        if (tid == 0) {
            double sum = 0.0;
            for (int w = 0; w < 8; ++w) sum += red[w];
            part[bid * nv + v] = sum;
        }
        __syncthreads();
    }
}

// Task entries of the marginal-likelihood gradient: the same tiling and weights w_ij as gpk_grad_trace_kernel, per CTA
// the T x T partial sums G_ab = sum_{i >= j, t_i = a, t_j = b} w_ij amp R_ij (row-major, T = n_tasks), R the radial
// product.  gpk_grad_final_kernel adds the CTAs (with noise_var = 1: no noise entry) and gpk_nll_grad contracts G with
// dK_t[a][b] / dtheta_pq on the host.  A kernel of its own, so the trace kernel's registers stay those of the kernel
// without a task factor.
__global__ void __launch_bounds__(256)
gpk_grad_task_kernel(const KSpec ks, const double* __restrict__ Xt, long ldx, int n,
                     const double* __restrict__ Kinv, long ldk, const double* __restrict__ alpha,
                     double* __restrict__ part)
{
    __shared__ double red[8];
    const int tid = threadIdx.x, nT = ks.factor.n_tasks, nv = nT * nT;
    const long bid = (long)blockIdx.y * gridDim.x + blockIdx.x;
    const int j = blockIdx.x * 128 + (tid & 127);
    const long c0 = (long)blockIdx.y * 32;
    if ((long)blockIdx.x * 128 > c0 + 31) {
        for (int v = tid; v < nv; v += 256) part[bid * nv + v] = 0.0;
        return;
    }
    const bool jv = j < n;
    const double* tx = Xt + (long)ks.factor.axis * ldx;
    const int tj = jv ? (int)tx[j] : 0;
    double g[GPK_MAX_TASKS];                                 // G_{a, t_j}: this thread's column task is t_j
    for (int a = 0; a < nT; ++a) g[a] = 0.0;
    for (int c = 0; c < 16; ++c) {
        const long i = c0 + (tid >> 7) * 16 + c;
        if (!(jv && i < n && j <= i)) continue;
        double r = 1.0, r2 = 0.0;
        for (int t = 0; t < ks.n_terms; ++t) {
            const double* xa = Xt + (long)ks.axis[t] * ldx;
            const double d = xa[i] - xa[j];
            r2 = fma(d * d, ks.inv_metric[t], r2);
            if (ks.last[t]) { r *= gpk_radial(ks.family, r2); r2 = 0.0; }
        }
        const double a = alpha[i] * alpha[j] - Kinv[i * ldk + j];
        g[(int)tx[i]] += (i == j ? a : 2.0 * a) * ks.amp * r;
    }
    for (int v = 0; v < nv; ++v) {                           // fixed order: lanes, then warps
        double x = (v % nT == tj) ? g[v / nT] : 0.0;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
        if ((tid & 31) == 0) red[tid >> 5] = x;
        __syncthreads();
        if (tid == 0) {
            double sum = 0.0;
            for (int w = 0; w < 8; ++w) sum += red[w];
            part[bid * nv + v] = sum;
        }
        __syncthreads();
    }
}

// out[v] = -1/2 * sum over CTAs (fixed order); the noise entry is scaled by sigma^2.
__global__ void gpk_grad_final_kernel(const double* __restrict__ part, long nblocks, int nv, double noise_var,
                                      double* __restrict__ out)
{
    const int v = blockIdx.x;
    __shared__ double sh[256];
    double s = 0.0;
    for (long b = threadIdx.x; b < nblocks; b += 256) s += part[b * nv + v];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[v] = -0.5 * sh[0] * (v == nv - 1 ? noise_var : 1.0);
}

// ---------------------------------------------------------------------------------------
// Reductions over the hyper-parameter samples of a GP-MCMC model (A, B are [n_models][m]):
//   mode 0: out1 = mean_i A_i                       (MarginalizationGPMCMC.compute, marginalization.py:121)
//   mode 1: out1 = mean_i A_i ; out2 = var_i(A_i) + mean_i B_i, clipped at eps
//           (GaussianProcessMCMC.predict, gaussian_process_mcmc.py:235-247; np.var is the
//            two-pass population variance)
// ---------------------------------------------------------------------------------------
__global__ void gpk_reduce_models_kernel(const double* __restrict__ A, const double* __restrict__ B, int n_models,
                                         long m, int mode, double* __restrict__ out1, double* __restrict__ out2)
{
    long c = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= m) return;
    double s = 0.0;
    for (int i = 0; i < n_models; ++i) s += A[(long)i * m + c];
    const double mean = s / (double)n_models;
    out1[c] = mean;
    if (mode == 1) {
        double v = 0.0, sb = 0.0;
        for (int i = 0; i < n_models; ++i) {
            double d = A[(long)i * m + c] - mean;
            v += d * d;
            sb += B[(long)i * m + c];
        }
        double r = v / (double)n_models + sb / (double)n_models;
        if (r < GPK_EPS) r = GPK_EPS;
        out2[c] = r;
    }
}

// ---------------------------------------------------------------------------------------
// On-device candidate generation for RandomSampling.maximize (random_sampling.py:38-47):
//   candidate i < n_uniform : lower + (upper - lower) * U[0,1)^d          (init_random_uniform)
//   otherwise               : clip(incumbent + scale * N(0,1)^d, lower, upper)
// Philox4x32-10 counter-based generator keyed by (seed, global candidate index, coordinate pair):
// the stream depends on nothing else, so results are identical for any chunking or GPU count.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void gpk_philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                  uint32_t k0, uint32_t k1, uint32_t (&out)[4])
{
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

__device__ __forceinline__ double gpk_u01(uint32_t lo, uint32_t hi) {      // 53-bit uniform in [0, 1)
    const unsigned long long v = ((unsigned long long)hi << 32) | lo;
    return (double)(v >> 11) * 1.1102230246251565e-16;
}

__global__ void gpk_candidates_kernel(unsigned long long seed, long first, long count, long n_uniform, int d,
                                      const double* __restrict__ lower, const double* __restrict__ upper,
                                      const double* __restrict__ incumbent, double scale,
                                      double* __restrict__ out)
{
    const int npair = (d + 1) / 2;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count * npair) return;
    const long li = t / npair;
    const int pb = (int)(t - li * npair);
    const unsigned long long gi = (unsigned long long)(first + li);
    uint32_t r[4];
    gpk_philox4x32_10((uint32_t)gi, (uint32_t)(gi >> 32), (uint32_t)pb, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    const double u0 = gpk_u01(r[0], r[1]), u1 = gpk_u01(r[2], r[3]);
    double v0, v1;
    const int a0 = 2 * pb, a1 = 2 * pb + 1;
    if ((long)gi < n_uniform) {
        // explicit rounding steps (no fma contraction): bit-identical to numpy's lower + (upper-lower)*u
        v0 = __dadd_rn(lower[a0], __dmul_rn(upper[a0] - lower[a0], u0));
        if (a1 < d) v1 = __dadd_rn(lower[a1], __dmul_rn(upper[a1] - lower[a1], u1));
    } else {                                              // Box-Muller, u in (0, 1]
        const double rad = sqrt(-2.0 * log(1.0 - u0));
        double sn, cs;
        sincospi(2.0 * u1, &sn, &cs);
        v0 = fmin(fmax(incumbent[a0] + scale * rad * cs, lower[a0]), upper[a0]);
        if (a1 < d) v1 = fmin(fmax(incumbent[a1] + scale * rad * sn, lower[a1]), upper[a1]);
    }
    out[li * d + a0] = v0;
    if (a1 < d) out[li * d + a1] = v1;
}

// ---------------------------------------------------------------------------------------
// Predictive gradients (SURVEY.md section 8f rank 3; the API robo/acquisition_functions/ei.py:80-85,
// pi.py:65-71, lcb.py:66-69 expect from a model but no reference model implements):
//   d mu / d x*_a   =  sum_j alpha_j        d k(x*, x_j) / d x*_a
//   d var / d x*_a  = -2 sum_j (K^-1 k*)_j  d k(x*, x_j) / d x*_a          (k** is constant: stationary kernels)
//   d k / d x*_t    =  k * (dlog f / d r2)(r2_g) * 2 (x*_t - x_jt) / metric_t    per kernel term t (axis a = axis[t])
// One CTA per candidate, threads stride over the training points, block reduction per term, chain
// rule of the input scaling (1 / (upper - lower)) and of the output transform applied at the end.
// With the environment factor k = amp R (c0 + c1 z* z_j): the terms above use that k, the environment axis gains
//   d k / d z* = amp R c1 z_j,   and  d var / d z* gains d k(x*, x*) / d z* = 2 amp c1 z*.
// With the task factor k = amp R K_t[t*][t_j]: the terms above use that k; the task axis and k(x*, x*) = amp K_t[t*][t*]
// have zero derivative (the task index is piecewise constant).  FK = GPK_FACTOR_TASK or GPK_FACTOR_ENV: each instance
// compiles the other factor's code out.  A kernel without a factor runs the ENV instance, which tests the kind at run
// time: an instance of its own compiles to 8 / 8 bytes of spills where this one has none (sm_90a, CUDA 12.9).
// ---------------------------------------------------------------------------------------
template <int FK>
__global__ void __launch_bounds__(256)
gpk_predict_grad_kernel(const KSpec ks, const double* __restrict__ Xt, long ldx, int n,
                        const double* __restrict__ cand, int dc,
                        const double* __restrict__ lower, const double* __restrict__ upper,
                        const double* __restrict__ alpha, const double* __restrict__ Wt, long ldw,
                        int norm_out, double y_std, double* __restrict__ dmu, double* __restrict__ dvar)
{
    __shared__ double xs[GPK_MAX_TERMS];
    __shared__ double red[16];
    const int tid = threadIdx.x, nt = ks.n_terms;
    const long c = blockIdx.x;
    const bool fac = FK == GPK_FACTOR_TASK || ks.factor.kind == GPK_FACTOR_ENV;
    const double zs = fac ? gpk_factor_coord<FK>(ks.factor, cand + c * dc, lower, upper) : 0.0;
    double gem = 0.0, gev = 0.0;                                        // environment-axis sums
    for (int t = tid; t < nt; t += 256) {
        const int a = ks.axis[t];
        double v = cand[c * dc + a];
        if (lower != nullptr) v = (v - lower[a]) / (upper[a] - lower[a]);
        xs[t] = v;
    }
    for (int a = tid; a < dc; a += 256) { dmu[c * dc + a] = 0.0; dvar[c * dc + a] = 0.0; }
    __syncthreads();
    double gm[GPK_MAX_TERMS], gv[GPK_MAX_TERMS];
    for (int t = 0; t < nt; ++t) { gm[t] = 0.0; gv[t] = 0.0; }
    for (int j = tid; j < n; j += 256) {
        double k = ks.amp, r2 = 0.0;
        for (int t = 0; t < nt; ++t) {                                  // kernel value
            const double d = xs[t] - Xt[(long)ks.axis[t] * ldx + j];
            r2 = fma(d * d, ks.inv_metric[t], r2);
            if (ks.last[t]) { k *= gpk_radial(ks.family, r2); r2 = 0.0; }
        }
        if (fac) {
            const double zj = Xt[(long)ks.factor.axis * ldx + j];
            if constexpr (FK == GPK_FACTOR_ENV) {
                const double dkz = k * gpk_env_dz(ks.factor.c1, zj);
                gem = fma(alpha[j], dkz, gem);
                gev = fma(-2.0 * Wt[c * ldw + j], dkz, gev);
            }
            k *= gpk_factor_value<FK>(ks.factor, zs, zj);
        }
        const double ka = k * alpha[j], kw = -2.0 * k * Wt[c * ldw + j];
        int t0 = 0;
        while (t0 < nt) {                                               // group by group
            int t1 = t0;
            while (!ks.last[t1]) ++t1;
            r2 = 0.0;
            for (int t = t0; t <= t1; ++t) {
                const double d = xs[t] - Xt[(long)ks.axis[t] * ldx + j];
                r2 = fma(d * d, ks.inv_metric[t], r2);
            }
            const double ratio = 2.0 * gpk_radial_dlog(ks.family, r2);
            for (int t = t0; t <= t1; ++t) {
                const double d = xs[t] - Xt[(long)ks.axis[t] * ldx + j];
                const double f = ratio * d * ks.inv_metric[t];
                gm[t] = fma(ka, f, gm[t]);
                gv[t] = fma(kw, f, gv[t]);
            }
            t0 = t1 + 1;
        }
    }
    for (int t = 0; t < nt; ++t) {
#pragma unroll
        for (int pass = 0; pass < 2; ++pass) {
            double x = pass == 0 ? gm[t] : gv[t];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
            if ((tid & 31) == 0) red[pass * 8 + (tid >> 5)] = x;
        }
        __syncthreads();
        if (tid == 0) {
            double sm = 0.0, sv = 0.0;
            for (int w = 0; w < 8; ++w) { sm += red[w]; sv += red[8 + w]; }
            const int a = ks.axis[t];
            double scale = 1.0;
            if (lower != nullptr) scale = 1.0 / (upper[a] - lower[a]);
            if (norm_out) { sm *= y_std; sv *= y_std * y_std; }
            dmu[c * dc + a] += sm * scale;
            dvar[c * dc + a] += sv * scale;
        }
        __syncthreads();
    }
    if (FK == GPK_FACTOR_ENV && fac) {
#pragma unroll
        for (int pass = 0; pass < 2; ++pass) {
            double x = pass == 0 ? gem : gev;
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
            if ((tid & 31) == 0) red[pass * 8 + (tid >> 5)] = x;
        }
        __syncthreads();
        if (tid == 0) {
            double sm = 0.0, sv = 0.0;
            for (int w = 0; w < 8; ++w) { sm += red[w]; sv += red[8 + w]; }
            sv += 2.0 * ks.amp * ks.factor.c1 * zs;                    // d k(x*, x*) / d z*
            const int a = ks.factor.axis;
            double scale = 1.0;
            if (lower != nullptr) scale = 1.0 / (upper[a] - lower[a]);
            if (norm_out) { sm *= y_std; sv *= y_std * y_std; }
            dmu[c * dc + a] += sm * scale;
            dvar[c * dc + a] += sv * scale;
        }
    }
}

// Acquisition value and gradient from moments and their gradients (ei.py:76-85, pi.py:61-71, lcb.py:65-69).
__global__ void gpk_acq_grad_kernel(const double* __restrict__ mu, const double* __restrict__ var,
                                    const double* __restrict__ dmu, const double* __restrict__ dvar, long m, int d,
                                    int kind, double eta, double par, double* __restrict__ f, double* __restrict__ df)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= m * d) return;
    const long c = idx / d;
    const double s = sqrt(var[c]);
    const double dm = dmu[idx], ds = dvar[idx] / (2.0 * s);
    double g;
    if (kind == GPK_ACQ_EI) {
        const double z = (eta - mu[c] - par) / s;
        g = -dm * gpk_ndtr(z) + ds * gpk_norm_pdf(z);
    } else if (kind == GPK_ACQ_PI) {
        const double z = (eta - mu[c] - par) / s;
        g = -(gpk_norm_pdf(z) / s) * (dm + ds * z);
    } else {
        g = -(dm - par * ds);
    }
    df[idx] = g;
    if (idx == c * d) f[c] = gpk_acq_value(kind, mu[c], var[c], eta, par);
}

// ---------------------------------------------------------------------------------------
// fp64 issue-rate peaks of the GPU we run on (register-resident operands, no memory traffic): the
// denominators of the roofline reported by bench.py.  DMMA m8n8k4 = the tensor pipe every GEMM of this
// library uses; DFMA = the vector pipe of the covariance builder.
// ---------------------------------------------------------------------------------------
__global__ void gpk_peak_dmma_kernel(double* out, int iters)
{
    double c[16][2], a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-6;
#pragma unroll
    for (int i = 0; i < 16; ++i) { c[i][0] = 0.0; c[i][1] = 0.0; }
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += c[i][0] + c[i][1];
    if (s == 12345.678) out[0] = s;
}

__global__ void gpk_peak_dfma_kernel(double* out, int iters)
{
    double a[8];
    const double b = 1.0000001, c = 0.9999999;
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = threadIdx.x * 1e-3 + i;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) a[i] = fma(a[i], b, c);
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += a[i];
    if (s == 12345.678) out[0] = s;
}
