// gpk_chain.cuh — step X(k) of the split Cholesky chain (option "chainsplit" = 1, see gpk_fit_begin).
//
// diag(k+1) needs only A[k+1,k+1] -= L[k+1,k] L[k+1,k]^T with L[k+1,k] = A[k+1,k] inv(L_kk)^T.  As two GEMM launches
// the panel solve and this update contract over K = 128 only: ~11 us each of which 4 us is arithmetic, plus a dependent
// launch gap.  Here ONE launch of four CTAs does both for the four 32-row tiles of block row k+1: CTA b solves its tile
// of the panel, publishes it (store, __threadfence, bump a counter), waits until all four tiles have arrived and then
// applies
//   A[rows, k+1] -= L[rows, k] L[k+1, k]^T
// to its own rows of block column k+1.  Each CTA needs one SM and waits only for the other three, which get SMs as
// other work drains, so the spin cannot deadlock.  All operands of both passes come in through cp.async (generic proxy,
// L2): the second pass reads what other CTAs of the same launch stored moments ago.
#pragma once
#include "gpk_gemm.cuh"

constexpr int CH_TM = 32;                                          // tile rows
constexpr int CH_ROWB = PAD_STRIDE * 8;                            // bytes per staged row (16 k + padding)
constexpr int CH_A_BYTES = CH_TM * CH_ROWB;                        // 5120
constexpr int CH_STAGE_BYTES = (CH_TM + BN) * CH_ROWB;             // 25600
constexpr int CH_STAGES = 8;                                       // the whole K = 128 contraction is staged at once
constexpr int CH_SMEM = CH_STAGES * CH_STAGE_BYTES + 256;          // 205056

struct ChainArgs {
    double* K; long ld;              // factor buffer (in place)
    const double* P; long ldp;       // inverse diagonal blocks
    const GemmJob* solve_jobs;       // 32-row panel-solve jobs of block row k+1, one per CTA
    const GemmJob* update_jobs;      // 32-row update jobs of tile (k+1, k+1), same order
    int* counter;                    // arrivals of the four tiles of block row k+1 (zeroed before the factorisation)
    const int* status;
};

// C(32 x 128) = beta C + alpha A(32 x 128) B(128 x 128)^T over the job's 128-long contraction range.
__device__ __forceinline__ void chain_tile(const uint32_t smem, const double* __restrict__ A, const long lda,
                                           const double* __restrict__ B, const long ldb, double* __restrict__ C,
                                           const long ldc, const GemmJob job, const double alpha, const int beta,
                                           const int tid)
{
    const int lane = tid & 31, warp = tid >> 5;
    const int gq = lane >> 2, tq = lane & 3;
    const int wm = warp >> 2, wn = warp & 3;
    // ---- stage everything: 8 groups of (32 + 128) rows x 16 k
#pragma unroll
    for (int s = 0; s < CH_STAGES; ++s) {
        const uint32_t st = smem + s * CH_STAGE_BYTES;
        const int kcol = job.k0 + s * BK;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int c = tid + i * GEMM_THREADS;        // 16-byte chunks, 8 per row
            const int row = c >> 3, kc = c & 7;
            if (row < CH_TM)
                cp_async16(st + (uint32_t)((row * PAD_STRIDE + kc * 2) * 8), A + (long)(job.a_row + row) * lda + kcol + kc * 2);
            cp_async16(st + (uint32_t)(CH_A_BYTES + (row * PAD_STRIDE + kc * 2) * 8),
                       B + (long)(job.b_row + row) * ldb + kcol + kc * 2);
        }
        cp_async_commit();
    }
    double acc[2][4][2];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
        const long r = job.c_row + wm * 16 + mi * 8 + gq;
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
#pragma unroll
            for (int j = 0; j < 2; ++j)
                acc[mi][ni][j] = beta ? alpha * C[r * ldc + job.c_col + wn * 32 + ni * 8 + 2 * tq + j] : 0.0;
    }
    const int offA = ((wm * 16 + gq) * PAD_STRIDE + tq) * 8;
    const int offB = CH_A_BYTES + ((wn * 32 + gq) * PAD_STRIDE + tq) * 8;
    constexpr int BLK = 8 * CH_ROWB;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        if (half == 0) cp_async_wait<4>(); else cp_async_wait<0>();
        __syncthreads();
#pragma unroll
        for (int s4 = 0; s4 < 4; ++s4) {
            const uint32_t st = smem + (half * 4 + s4) * CH_STAGE_BYTES;
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                double a[2], b[4];
#pragma unroll
                for (int mi = 0; mi < 2; ++mi) a[mi] = lds64(st + offA + ks * 32 + mi * BLK);
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) b[ni] = lds64(st + offB + ks * 32 + ni * BLK);
#pragma unroll
                for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                    for (int ni = 0; ni < 4; ++ni) dmma884(acc[mi][ni][0], acc[mi][ni][1], a[mi], b[ni]);
            }
        }
    }
    // ---- epilogue through shared memory (coalesced stores); the operand ring is free
    __syncthreads();
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
        const int r = wm * 16 + mi * 8 + gq;
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
#pragma unroll
            for (int j = 0; j < 2; ++j)
                sts64(smem + 8 * (r * CT_STRIDE + wn * 32 + ni * 8 + 2 * tq + j), alpha * acc[mi][ni][j]);
    }
    __syncthreads();
    for (int e = tid; e < CH_TM * BN; e += GEMM_THREADS) {
        const int r = e >> 7, c = e & 127;
        C[(long)(job.c_row + r) * ldc + job.c_col + c] = lds64(smem + 8 * (r * CT_STRIDE + c));
    }
}

__global__ void __launch_bounds__(GEMM_THREADS, 1)
gpk_chain_step_kernel(const ChainArgs g)
{
    cudaGridDependencySynchronize();
    if (g.status != nullptr && *g.status != 0) return;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t smem = (smem_u32(smem_raw) + 127u) & ~127u;
    const int tid = threadIdx.x;

    // pass 1: L[rows, k] = A[rows, k] inv(L_kk)^T   (in place: the whole tile is staged before anything is stored)
    chain_tile(smem, g.K, g.ld, g.P, g.ldp, g.K, g.ld, g.solve_jobs[blockIdx.x], 1.0, 0, tid);

    // publish; the four tiles of block row k+1 are the B operand of everybody's pass 2
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        atomicAdd(g.counter, 1);
        while (atomicAdd(g.counter, 0) < 4) __nanosleep(64);
        __threadfence();
    }
    __syncthreads();

    // pass 2: A[rows, k+1] -= L[rows, k] L[k+1, k]^T
    chain_tile(smem, g.K, g.ld, g.K, g.ld, g.K, g.ld, g.update_jobs[blockIdx.x], -1.0, 1, tid);
}
