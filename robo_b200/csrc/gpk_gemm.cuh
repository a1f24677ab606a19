// gpk_gemm.cuh — fp64 tensor-core (DMMA) tile engine:  C(128x128) (+)= alpha * A(128xK) * B(128xK)^T
//
// Every dense contraction of the hot path is an "NT" product of two K-contiguous operands:
//   Cholesky panel solve    L_ik  =  A_ik * inv(L_kk)^T                     (store)
//   Cholesky trailing update A_ij -=  L_ik * L_jk^T                          (store, beta = 1)
//   triangular inverse       T'   =  Q * L^T ;  R = -P * T'^T               (store C and C^T)
//   predictive variance      V    =  L^-1 * K*^T  ->  sum_i V_ic^2 , sum_i V_ic z_i   (column reduce)
// One CTA = one output tile described by a GemmJob; 8 DMMA warps, each a (TM/2)x32 sub-tile of m8n8k4 fragments.
// Limitation on H100: m8n8k4 is Hopper's legacy fp64 MMA shape and issues at about half of the fp64 tensor-core rate
// (measured with gpk_measure_fp64_peaks against cuBLAS DGEMM, DESIGN.md section 5); the m16n8k{4,8,16} shapes are the way
// to the full rate.  Operand tiles (rows x 16 k) are staged by cp.async.bulk.tensor.2d + mbarrier complete_tx,
// 128B-swizzled (sm_90a), which gives bank-conflict-free 8-byte fragment loads (see rowmap()).  Two kernels:
//   gpk_gemm_ws_kernel   128 x 128 tiles (throughput): a dedicated producer warp issues the loads into a 4-stage ring
//   gpk_gemm_nt_kernel   32 x 128 tiles (the latency-critical panel solve / next-panel update of the Cholesky chain,
//                        launched with programmatic dependent launch): thread 0 issues every load up front
#pragma once
#include "gpk_internal.cuh"

enum { EPI_STORE = 0, EPI_COLREDUCE = 1 };
enum { JOBS_TABLE = 0, JOBS_VARIANCE = 1 };

constexpr int BM = 128, BN = 128, BK = 16, NSTAGE = 4, GEMM_THREADS = 256;
constexpr int VAR_GROUP = 16;                                    // candidate blocks per L2-resident group
constexpr int STAGE_BYTES_TMA = (BM + BN) * BK * 8;              // 32768
constexpr int CT_STRIDE = 129;                                   // doubles per row of the epilogue staging tile
constexpr int CT_BYTES = BM * CT_STRIDE * 8;                     // 132096
constexpr int RING_TMA = NSTAGE * STAGE_BYTES_TMA > CT_BYTES ? NSTAGE * STAGE_BYTES_TMA : ((CT_BYTES + 1023) / 1024) * 1024;
constexpr int GEMM_SMEM_TMA = RING_TMA + 1024 /*align*/ + 64 /*barriers*/ + 2048 /*reduce*/;
// The 32-row chain tiles contract over K = 128 only (8 k-steps): their ring holds all 8 steps, so every operand load is
// in flight before the first DMMA instead of trickling through a 4-deep ring (latency, not bandwidth).
constexpr int CHAIN_TM = 32, CHAIN_NSTAGE = 8;
constexpr int CHAIN_RING = CHAIN_NSTAGE * (CHAIN_TM + BN) * BK * 8;
constexpr int GEMM_SMEM_CHAIN = CHAIN_RING + 1024 /*align*/ + 64 /*barriers*/;

struct GemmJob {
    int a_row;      // first row of the A tile
    int b_row;      // first row of the B tile
    int k0, k1;     // contraction range [k0, k1), multiples of BK
    int c_row;      // output tile origin (row follows A rows, col follows B rows)
    int c_col;
    int aux;        // EPI_COLREDUCE: partial-sum slot
    int pad;
};

struct GemmArgs {
    const double* A; long lda;         // not read on the device: the kernels load through mapA / mapB
    const double* B; long ldb;
    double* C; long ldc;               // may be NULL
    double* Ct; long ldct;             // transposed copy of the output tile, may be NULL
    double alpha;                      // +1 / -1
    int beta;                          // 0: overwrite, 1: accumulate into C
    const GemmJob* jobs;
    int job_mode;                      // JOBS_TABLE / JOBS_VARIANCE
    int nb, mcb;                       // JOBS_VARIANCE generator: nb row-blocks x mcb candidate blocks
    const double* z;                   // EPI_COLREDUCE: row weights (z = L^-1 (y - mean))
    double* part_mu; double* part_ssq; long ldpart;
    const int* status;                 // non-zero -> factorisation failed, skip work
};

// ---------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ double lds64(uint32_t addr) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts64(uint32_t addr, double v) {
    asm volatile("st.shared.f64 [%0], %1;" :: "r"(addr), "d"(v) : "memory");
}
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
    asm ("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, int c_inner, int c_outer,
                                            uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
                 " [%0], [%1, {%3, %4}], [%2];"
                 :: "r"(smem_dst), "l"((uint64_t)map), "r"(bar), "r"(c_inner), "r"(c_outer)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// Which tile row feeds fragment row g (0..7) of an 8-row block.  With the 128B TMA swizzle the
// 16-byte chunk index is XORed with (row & 7); mapping fragment rows {0,1,2,3 | 4,5,6,7} to tile
// rows {0,2,4,6 | 1,3,5,7} makes the 16 lanes of each half-warp (4 rows x 4 k) hit 16 distinct
// 8-byte banks.
__device__ __forceinline__ int rowmap(int g) { return ((g & 3) << 1) | (g >> 2); }

// Byte offset inside an operand stage of element (row, k).
__device__ __forceinline__ int tile_off(int row, int k) {
    return row * 128 + ((((k >> 1) ^ (row & 7))) << 4) + ((k & 1) << 3);
}

// ---------------------------------------------------------------------------------------
// 32 x 128 chain tile (EPI_STORE, job table)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gpk_gemm_nt_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                   const GemmArgs g)
{
    // Programmatic dependent launch: when launched with the stream-serialization attribute this CTA may
    // start while the producing kernel drains; nothing is read before the dependency is resolved.
    cudaGridDependencySynchronize();
    if (g.status != nullptr && *g.status != 0) return;
    constexpr int MI = CHAIN_TM / 16;                                   // 8-row fragment blocks per warp
    constexpr int TM = CHAIN_TM;                                        // tile rows (A rows)
    constexpr int NS = CHAIN_NSTAGE;                                    // ring depth
    constexpr int HM = TM / 2;                                          // rows per warp row-group

    extern __shared__ unsigned char smem_raw[];
    // all shared-memory traffic goes through 32-bit shared-window addresses (LDS/STS, not generic LD/ST)
    const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;        // 1024B alignment for the 128B swizzle
    constexpr int ROWB = BK * 8;                                        // bytes per staged row
    constexpr int A_BYTES = TM * ROWB;
    constexpr int STAGE_BYTES = (TM + BN) * ROWB;
    constexpr int RING = CHAIN_RING;
    static_assert(RING == NS * STAGE_BYTES, "ring = NS stages");
    static_assert(RING >= ((TM * CT_STRIDE * 8 + 1023) / 1024) * 1024, "epilogue staging tile must fit the operand ring");
    const uint32_t full_bar = smem + RING;                              // NS x 8 bytes

    const GemmJob job = g.jobs[blockIdx.x];
    const int KT = (job.k1 - job.k0) / BK;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gq = lane >> 2, tq = lane & 3;
    const int wm = warp >> 2, wn = warp & 3;

    // per-thread fragment offsets (bytes) inside a stage
    constexpr int BLK = 8 * ROWB;                                        // 8 tile rows
    const int rA = wm * HM + rowmap(gq);
    const int rB = wn * 32 + rowmap(gq);
    int kxA[4], kxB[4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        kxA[ks] = tile_off(rA, ks * 4 + tq);
        kxB[ks] = A_BYTES + tile_off(rB, ks * 4 + tq);
    }

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < NS; ++s) mbar_init(full_bar + 8 * s, 1);
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();

    auto issue_load = [&](int kt) {
        const int s = kt % NS;
        const uint32_t st = smem + s * STAGE_BYTES;
        const int kcol = job.k0 + kt * BK;
        if (tid == 0) {
            fence_proxy_async();
            mbar_arrive_expect_tx(full_bar + 8 * s, STAGE_BYTES);
            tma_load_2d(st, &mapA, kcol, job.a_row, full_bar + 8 * s);            // box TM rows x 16
            tma_load_2d(st + A_BYTES, &mapB, kcol, job.b_row, full_bar + 8 * s);  // box 128 rows x 16
        }
    };

    double acc[MI][4][2];
#pragma unroll
    for (int mi = 0; mi < MI; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) { acc[mi][ni][0] = 0.0; acc[mi][ni][1] = 0.0; }

    // ---- prologue ----
#pragma unroll
    for (int s = 0; s < NS - 1; ++s)
        if (s < KT) issue_load(s);
    if (g.beta) {
        // C_new = C_old + alpha * A B^T with alpha = +-1: start the accumulators at alpha * C_old; the
        // loads overlap the pipeline fill instead of sitting in the epilogue.
#pragma unroll
        for (int mi = 0; mi < MI; ++mi) {
            const long r = job.c_row + wm * HM + mi * 8 + rowmap(gq);
#pragma unroll
            for (int ni = 0; ni < 4; ++ni)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const long c = job.c_col + wn * 32 + ni * 8 + rowmap(2 * tq + j);
                    acc[mi][ni][j] = g.alpha * g.C[r * g.ldc + c];
                }
        }
    }

    // ---- main loop ----
    for (int kt = 0; kt < KT; ++kt) {
        const int s = kt % NS;
        const uint32_t parity = (uint32_t)((kt / NS) & 1);
        while (!mbar_try_wait(full_bar + 8 * s, parity)) { }
        __syncthreads();          // stage s visible to all; everyone is done with stage (kt-1)%NS
        if (kt + NS - 1 < KT) issue_load(kt + NS - 1);

        const uint32_t st = smem + s * STAGE_BYTES;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            double a[MI], b[4];
#pragma unroll
            for (int mi = 0; mi < MI; ++mi) a[mi] = lds64(st + kxA[ks] + mi * BLK);
#pragma unroll
            for (int ni = 0; ni < 4; ++ni) b[ni] = lds64(st + kxB[ks] + ni * BLK);
#pragma unroll
            for (int mi = 0; mi < MI; ++mi)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) dmma884(acc[mi][ni][0], acc[mi][ni][1], a[mi], b[ni]);
        }
    }

    // ---- epilogue ----
    // acc[mi][ni][j]  <->  tile row  wm*HM + mi*8 + rowmap(gq),  tile col  wn*32 + ni*8 + rowmap(2*tq + j)
    // stage the tile through shared memory (the operand ring is free now) so that the global
    // stores of C and of its transpose are fully coalesced
    __syncthreads();
#pragma unroll
    for (int mi = 0; mi < MI; ++mi) {
        const int r = wm * HM + mi * 8 + rowmap(gq);
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int c = wn * 32 + ni * 8 + rowmap(2 * tq + j);
                sts64(smem + 8 * (r * CT_STRIDE + c), g.alpha * acc[mi][ni][j]);
            }
    }
    __syncthreads();
    if (g.C) {
        for (int e = tid; e < TM * BN; e += GEMM_THREADS) {
            const int r = e >> 7, c = e & 127;
            g.C[(long)(job.c_row + r) * g.ldc + job.c_col + c] = lds64(smem + 8 * (r * CT_STRIDE + c));
        }
    }
    if (g.Ct) {
        for (int e = tid; e < TM * BN; e += GEMM_THREADS) {
            const int c = e / TM, r = e - c * TM;
            g.Ct[(long)(job.c_col + c) * g.ldct + job.c_row + r] = lds64(smem + 8 * (r * CT_STRIDE + c));
        }
    }
}

// ---------------------------------------------------------------------------------------
// 128 x 128 tile, warp-specialised: warp 8 is a dedicated producer (one elected lane issues the TMA
// loads), warps 0-7 are DMMA consumers.  Stage hand-over uses a full/empty mbarrier pair per stage
// instead of a block-wide __syncthreads per k-step, so consumer warps never rendezvous with each
// other inside the main loop and may drift by up to NSTAGE-1 stages.
// ---------------------------------------------------------------------------------------
constexpr int WS_THREADS = GEMM_THREADS + 32;

template <int EPI>
__global__ void __launch_bounds__(WS_THREADS, 1)
gpk_gemm_ws_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                   const GemmArgs g)
{
    if (g.status != nullptr && *g.status != 0) return;
    constexpr int MI = 8, TM = 128, HM = 64;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;
    constexpr int ROWB = BK * 8;
    constexpr int A_BYTES = TM * ROWB;
    constexpr int STAGE_BYTES = (TM + BN) * ROWB;
    constexpr int RING = RING_TMA;
    const uint32_t full_bar = smem + RING;               // NSTAGE x 8 bytes
    const uint32_t empty_bar = smem + RING + 32;         // NSTAGE x 8 bytes
    const uint32_t red = smem + RING + 64;

    GemmJob job;
    if (g.job_mode == JOBS_TABLE) {
        job = g.jobs[blockIdx.x];
    } else {
        const int full = g.mcb / VAR_GROUP;
        int id = (int)blockIdx.x, grp = id / (g.nb * VAR_GROUP), gsz = VAR_GROUP;
        if (grp >= full) { grp = full; gsz = g.mcb - full * VAR_GROUP; }
        id -= grp * g.nb * VAR_GROUP;
        int ib = g.nb - 1 - id / gsz;
        int cb = grp * VAR_GROUP + id % gsz;
        job.a_row = ib * BM; job.b_row = cb * BN; job.k0 = 0; job.k1 = (ib + 1) * BM;
        job.c_row = ib * BM; job.c_col = cb * BN; job.aux = ib; job.pad = 0;
    }
    const int KT = (job.k1 - job.k0) / BK;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, 8); }
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();

    if (warp == 8) {
        // ---------------- producer ----------------
        if (lane == 0) {
            for (int kt = 0; kt < KT; ++kt) {
                const int s = kt % NSTAGE;
                if (kt >= NSTAGE) {                      // wait until all 8 consumer warps released use (kt/NSTAGE - 1)
                    const uint32_t parity = (uint32_t)(((kt / NSTAGE) - 1) & 1);
                    while (!mbar_try_wait(empty_bar + 8 * s, parity)) { }
                }
                const uint32_t st = smem + s * STAGE_BYTES;
                const int kcol = job.k0 + kt * BK;
                fence_proxy_async();
                mbar_arrive_expect_tx(full_bar + 8 * s, STAGE_BYTES);
                tma_load_2d(st, &mapA, kcol, job.a_row, full_bar + 8 * s);
                tma_load_2d(st + A_BYTES, &mapB, kcol, job.b_row, full_bar + 8 * s);
            }
        }
        return;
    }

    // ---------------- consumers (warps 0-7) ----------------
    const int gq = lane >> 2, tq = lane & 3;
    const int wm = warp >> 2, wn = warp & 3;
    constexpr int BLK = 8 * ROWB;
    const int rA = wm * HM + rowmap(gq);
    const int rB = wn * 32 + rowmap(gq);
    int kxA[4], kxB[4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        kxA[ks] = tile_off(rA, ks * 4 + tq);
        kxB[ks] = A_BYTES + tile_off(rB, ks * 4 + tq);
    }
    double acc[MI][4][2];
#pragma unroll
    for (int mi = 0; mi < MI; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) { acc[mi][ni][0] = 0.0; acc[mi][ni][1] = 0.0; }
    if (EPI == EPI_STORE && g.beta) {
#pragma unroll
        for (int mi = 0; mi < MI; ++mi) {
            const long r = job.c_row + wm * HM + mi * 8 + rowmap(gq);
#pragma unroll
            for (int ni = 0; ni < 4; ++ni)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const long c = job.c_col + wn * 32 + ni * 8 + rowmap(2 * tq + j);
                    acc[mi][ni][j] = g.alpha * g.C[r * g.ldc + c];
                }
        }
    }
    for (int kt = 0; kt < KT; ++kt) {
        const int s = kt % NSTAGE;
        const uint32_t parity = (uint32_t)((kt / NSTAGE) & 1);
        while (!mbar_try_wait(full_bar + 8 * s, parity)) { }
        const uint32_t st = smem + s * STAGE_BYTES;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            double a[MI], b[4];
#pragma unroll
            for (int mi = 0; mi < MI; ++mi) a[mi] = lds64(st + kxA[ks] + mi * BLK);
#pragma unroll
            for (int ni = 0; ni < 4; ++ni) b[ni] = lds64(st + kxB[ks] + ni * BLK);
#pragma unroll
            for (int mi = 0; mi < MI; ++mi)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) dmma884(acc[mi][ni][0], acc[mi][ni][1], a[mi], b[ni]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar + 8 * s);   // this warp is done reading stage s
    }

    if (EPI == EPI_STORE) {
        named_bar_sync(1, GEMM_THREADS);                 // all consumers finished the ring
#pragma unroll
        for (int mi = 0; mi < MI; ++mi) {
            const int r = wm * HM + mi * 8 + rowmap(gq);
#pragma unroll
            for (int ni = 0; ni < 4; ++ni)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int c = wn * 32 + ni * 8 + rowmap(2 * tq + j);
                    sts64(smem + 8 * (r * CT_STRIDE + c), g.alpha * acc[mi][ni][j]);
                }
        }
        named_bar_sync(1, GEMM_THREADS);
        if (g.C) {
            for (int e = tid; e < TM * BN; e += GEMM_THREADS) {
                const int r = e >> 7, c = e & 127;
                g.C[(long)(job.c_row + r) * g.ldc + job.c_col + c] = lds64(smem + 8 * (r * CT_STRIDE + c));
            }
        }
        if (g.Ct) {
            for (int e = tid; e < TM * BN; e += GEMM_THREADS) {
                const int c = e / TM, r = e - c * TM;
                g.Ct[(long)(job.c_col + c) * g.ldct + job.c_row + r] = lds64(smem + 8 * (r * CT_STRIDE + c));
            }
        }
    } else {
        double zr[MI];
#pragma unroll
        for (int mi = 0; mi < MI; ++mi) zr[mi] = g.z[job.c_row + wm * HM + mi * 8 + rowmap(gq)];
        double ssq[4][2], smu[4][2];
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                double s2 = 0.0, sm = 0.0;
#pragma unroll
                for (int mi = 0; mi < MI; ++mi) {
                    double v = acc[mi][ni][j];
                    s2 = fma(v, v, s2);
                    sm = fma(v, zr[mi], sm);
                }
#pragma unroll
                for (int off = 4; off < 32; off <<= 1) {
                    s2 += __shfl_xor_sync(0xffffffffu, s2, off);
                    sm += __shfl_xor_sync(0xffffffffu, sm, off);
                }
                ssq[ni][j] = s2; smu[ni][j] = sm;
            }
        if (gq == 0) {
#pragma unroll
            for (int ni = 0; ni < 4; ++ni)
#pragma unroll
                for (int j = 0; j < 2; ++j)
                    sts64(red + 8 * (wm * 128 + wn * 32 + ni * 8 + rowmap(2 * tq + j)), ssq[ni][j]);
        }
        named_bar_sync(1, GEMM_THREADS);
        if (tid < 128)
            g.part_ssq[(long)job.aux * g.ldpart + job.c_col + tid] = lds64(red + 8 * tid) + lds64(red + 8 * (128 + tid));
        named_bar_sync(1, GEMM_THREADS);
        if (gq == 0) {
#pragma unroll
            for (int ni = 0; ni < 4; ++ni)
#pragma unroll
                for (int j = 0; j < 2; ++j)
                    sts64(red + 8 * (wm * 128 + wn * 32 + ni * 8 + rowmap(2 * tq + j)), smu[ni][j]);
        }
        named_bar_sync(1, GEMM_THREADS);
        if (tid < 128)
            g.part_mu[(long)job.aux * g.ldpart + job.c_col + tid] = lds64(red + 8 * tid) + lds64(red + 8 * (128 + tid));
    }
}
