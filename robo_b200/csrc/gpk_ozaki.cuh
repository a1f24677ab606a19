// gpk_ozaki.cuh — the variance contraction on the int8 tensor pipe (option "ozaki" = 1).
//
// An error-free (Ozaki) split turns the fp64 product V = L^-1 K*^T into exact integer products that Hopper's int8
// warpgroup MMA (wgmma s8 x s8 -> s32, accumulators in registers) computes:
//   P  = L^-1 :  P[i][k]  ~ 2^eP[i] sum_s Pq[s][i][k] 2^(-8 (s+1))     per-row exponent, S = 7 balanced base-256 digits
//   K*        :  K*[c][k] ~ 2^eK    sum_t Kq[t][c][k] 2^(-8 (t+1))     one exponent (0 < k <= amp)
//   V[i][c] = 2^(eP[i] + eK) sum_lvl 2^(-8 (lvl + 2)) sum_{s + t = lvl} <Pq[s][i][:], Kq[t][c][:]>      (lvl < S)
// Digits are BALANCED (-128 .. 127, oz_digits below), so every int8 carries 8 bits: 7 slices hold 56 bits of each
// operand relative to its row maximum and the triangle s + t < 7 has 28 slice pairs (tools/ozaki_study.py prints the
// error of this split against 7-bit truncated digits).  The pairs of one level share one int32 accumulator
// ((lvl + 1) K 128^2 < 2^31 for K <= 16384), so a tile keeps 7 accumulators.  Per 64-byte k-block the CTA stages all
// 7 + 7 slice tiles (TMA, 64B swizzle) once and issues 56 MMAs per warpgroup on them; the CTAs of a cluster share the
// L^-1 slices by TMA multicast (option "ozcluster").  The L^-1 slice is the A operand
// and comes from registers (ldmatrix once per slice and k-block, reused by its 7 - s levels); only the K* slice is read
// from shared memory by every MMA.  With both operands in shared memory the 56 MMAs read 168 KB per warpgroup and
// k-block, more than the SM's shared-memory bandwidth delivers at the tensor pipe's issue rate; in registers, 84 KB
// (tools/microbench/int8_operand_rates.cu measures both forms).
// Accuracy (tools/ozaki_study.py): the split is exact to 2^-57 of the row maximum per operand; the handle falls back to
// the fp64 DMMA kernel when the factor is worse conditioned than max |L^-1| < 64 (eP > OZ_MAX_EXP) or N > 16384.
//
// Output: the per-row-block partial sums part_ssq [nb][ld] the DMMA kernel writes too.  The posterior MEAN does not go
// through the slices: mu - mean = K* alpha is one fp64 dot product of length N per candidate (gpk_rowdot_kernel on the
// fp64 K* that is built anyway, alpha = L^-T z once per fit), like george's own K* alpha; sum_i V_i z_i would put the
// slices' error in front of |z| ~ 1e2 and cost the 1e-10 tolerance on the mean.
#pragma once
#include "gpk_gemm.cuh"

constexpr int OZ_S = 7;                       // slices (balanced base-256 digits) per operand
constexpr int OZ_PAIRS = OZ_S * (OZ_S + 1) / 2;   // slice pairs with s + t < OZ_S
// Tile: 128 rows of L^-1 x 32 candidates.  Each of the two consumer warpgroups owns 64 rows and keeps the 7 level
// accumulators of its 64 x 32 share in registers (7 x 16 = 112 int32 per thread), next to two 8-register A fragments.
constexpr int OZ_TM = 128, OZ_TN = 32;
constexpr int OZ_KB = 64;                     // k-block: 64 int8 = one 64-byte swizzle row
constexpr int OZ_UK = 32;                     // K of one wgmma m64n32k32 s8
constexpr int OZ_NSTG = 3;
constexpr int OZ_A_SLICE = OZ_TM * OZ_KB, OZ_B_SLICE = OZ_TN * OZ_KB;
constexpr int OZ_STAGE = OZ_S * (OZ_A_SLICE + OZ_B_SLICE);               // 71680 bytes
constexpr int OZ_THREADS = 384;               // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + epilogue
constexpr int OZ_SMEM = OZ_NSTG * OZ_STAGE + 1024 + 256 + 2 * 8 * OZ_TN * 8;
constexpr int OZ_MAX_EXP = 7;                 // row exponents above this (|L^-1| >= 64): use the fp64 kernel

// Exponent e with |x| 2^-e inside the balanced digit interval [-128/255, 127/255) for every |x| <= amax: normally
// frexp's exponent + 1 (|x| 2^-e in [1/4, 1/2)), one more when the largest mantissa is within 0.004 of 1.
__host__ __device__ inline int oz_exponent(double amax) {
    if (!(amax > 0.0)) return 0;
    int ex;
    const double m = frexp(amax, &ex);
    return ex + 1 + (m * 128.0 >= 127.49 ? 1 : 0);
}
// The OZ_S balanced base-256 digits of v (|v| < 127.49 / 256, i.e. already scaled by 2^-e), most significant first in
// the bytes 6 .. 0 of the result, each digit d as the int8 bit pattern: v ~ sum_s d_s 256^-(s+1), |error| <= 2^-57.
// Integer arithmetic: X = rint(v 2^56) (exact power-of-two scaling, one F2I), then with B = 0x80 in every byte the
// bytes b of X + B are the digits + 128 (sum (b_j - 128) 256^j = X, and 0 <= X + B < 2^56 because |X| < 0.997 2^55), so
// XOR 0x80 turns each byte into the two's-complement digit.  One conversion and three integer instructions replace
// seven rounds of scale / floor / clamp / subtract in fp64.
__device__ __forceinline__ unsigned long long oz_digits(double v) {
    const long long X = __double2ll_rn(v * 72057594037927936.0);             // 2^56
    return (unsigned long long)(X + 0x0080808080808080LL) ^ 0x0080808080808080ULL;
}
__device__ __forceinline__ int oz_digit_of(unsigned long long y, int s) { return (int)((y >> (8 * (OZ_S - 1 - s))) & 0xFFull); }

__device__ __forceinline__ void oz_mbar_wait(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) { }
}
// ---- CTA clusters -------------------------------------------------------------------------------------------------
// A launch without a cluster attribute is a cluster of one CTA: rank 0 of 1.
__device__ __forceinline__ uint32_t oz_cluster_size() {
    uint32_t n;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(n));
    return n;
}
__device__ __forceinline__ uint32_t oz_cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// every thread of every CTA of the cluster; orders shared-memory and mbarrier operations across the cluster
__device__ __forceinline__ void oz_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// TMA 2D load whose box lands at the same shared-memory offset in every CTA of cta_mask, and completes bytes on the
// mbarrier at the same offset in each of them
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t smem_dst, const CUtensorMap* map, int c_inner, int c_outer,
                                                      uint32_t bar, uint16_t cta_mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
                 " [%0], [%1, {%3, %4}], [%2], %5;"
                 :: "r"(smem_dst), "l"((uint64_t)map), "r"(bar), "r"(c_inner), "r"(c_outer), "h"(cta_mask)
                 : "memory");
}
// Hands a ring stage back to the producers: one arrival on the empty barrier at offset `bar` of every CTA of the
// cluster, since each of their producers multicasts into this CTA's copy of the stage.  Called by threads 0 .. cs - 1
// of a consumer warpgroup, thread r arriving for CTA r: the cs arrivals go out as one warp instruction.  The reads they
// release are complete (ldmatrix into registers, wgmma retired by wait_group), so the default .cta release suffices.
__device__ __forceinline__ void oz_release_stage(uint32_t bar, uint32_t cs, uint32_t r) {
    if (cs == 1) { mbar_arrive(bar); return; }
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(bar), "r"(r));
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" :: "r"(remote) : "memory");
}
// K-major SWIZZLE_64B shared-memory matrix descriptor of wgmma: start address >> 4, leading byte offset (unused for
// swizzled K-major layouts) 1, stride byte offset 512 (8 rows x 64 bytes), layout type 2 = SWIZZLE_64B in bits [62,64)
__device__ __forceinline__ uint64_t oz_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(512 >> 4) << 32;
    d |= (uint64_t)2 << 62;
    return d;
}
#define OZ_ACC16(d) "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), \
                    "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
// d (64 x 32 s32, wgmma accumulator layout) += A (64 x 32 s8, from registers: one fragment of oz_lda_frag) *
// B (32 x 32 s8, K-major in shared memory)^T
__device__ __forceinline__ void oz_wgmma_rs(uint32_t (&d)[16], const uint32_t (&a)[4], uint64_t b_desc) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, 1;"
                 : OZ_ACC16(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));
}
// A fragments of one 64-byte k-block (two k32 halves) of a 64-row, 64B-swizzled K-major slice tile at `tile`, for the
// warp's 16 rows starting at row0.  The wgmma register layout of an s8 A fragment (reg 0: row lane/4, k 4 (lane%4) ..
// + 3; reg 1: row + 8; regs 2, 3: the same at k + 16) is what ldmatrix.x4 of four 8-row x 16-byte matrices delivers.
// Lane L addresses row L % 8 + 8 ((L / 8) & 1), 16-byte chunk L / 16 of the half; SWIZZLE_64B XORs the chunk index
// (address bits 4-5) with bits 7-8, i.e. with (row / 2) % 4 for 64-byte rows.
__device__ __forceinline__ void oz_lda_frag(uint32_t (&a)[2][4], uint32_t tile, int row0, int lane) {
    const int r = row0 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
    for (int k = 0; k < OZ_KB / OZ_UK; ++k) {
        const int chunk = 2 * k + (lane >> 4);
        const uint32_t addr = tile + (uint32_t)(r * OZ_KB + ((chunk ^ ((r >> 1) & 3)) << 4));
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                     : "=r"(a[k][0]), "=r"(a[k][1]), "=r"(a[k][2]), "=r"(a[k][3]) : "r"(addr) : "memory");
    }
}
__device__ __forceinline__ void oz_wgmma_fence(uint32_t (&d)[16]) { asm volatile("" : OZ_ACC16(d) :: "memory"); }
__device__ __forceinline__ void wgmma_arrive() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_one() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// exact int32 -> fp64 without the quarter-rate I2F.F64: 2^52 + 2^31 + d as bit pattern, minus the constant
__device__ __forceinline__ double oz_i2d(uint32_t d) {
    return __hiloint2double(0x43300000, (int)(d ^ 0x80000000u)) - 4503601774854144.0;
}

// ---- operand split ------------------------------------------------------------------------------------------------
// per-row exponent e[r] = oz_exponent(max |A[r][:]|); emax receives the maximum over the rows (atomicMax)
__global__ void gpk_oz_rowexp_kernel(const double* __restrict__ A, long ld, int cols, int* __restrict__ e, int* __restrict__ emax) {
    const long r = blockIdx.x;
    double m = 0.0;
    for (int c = threadIdx.x; c < cols; c += 256) m = fmax(m, fabs(A[r * ld + c]));
    __shared__ double sh[256];
    sh[threadIdx.x] = m;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] = fmax(sh[threadIdx.x], sh[threadIdx.x + o]); __syncthreads(); }
    if (threadIdx.x == 0) {
        const int ex = oz_exponent(sh[0]);
        e[r] = ex;
        atomicMax(emax, ex);
    }
}
// q[s][row][col] (slices slice_stride bytes apart) = the s-th balanced base-256 digit of A[row][col] / 2^e; e = erow[row]
// or (erow == NULL) e0.  One thread per element.
__global__ void gpk_oz_split_kernel(const double* __restrict__ A, long rows, long ld, const int* __restrict__ erow, int e0,
                                    int8_t* __restrict__ q, long slice_stride) {
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * ld) return;
    const long r = idx / ld;
    double v = ldexp(A[idx], -(erow ? erow[r] : e0));
    const unsigned long long y = oz_digits(v);
#pragma unroll
    for (int s = 0; s < OZ_S; ++s) q[(long)s * slice_stride + idx] = (int8_t)oz_digit_of(y, s);
}

// ---- the contraction ----------------------------------------------------------------------------------------------
// Tile order: candidate blocks are taken in groups of `group` blocks whose K* slices (group x TN x NP x 7 bytes, about
// half of the 50 MB L2, see score_dev) stay L2-resident while the group walks all row blocks of L^-1, longest
// contraction first; without the grouping every row block re-reads the whole chunk's slices from HBM.  The kernel
// calls it in units of cluster tiles (CS adjacent candidate blocks of one row block): ncb and group divided by CS.
__device__ __forceinline__ void oz_tile_of(int id, int nb, int ncb, int group, int& ib, int& cb) {
    const int full = ncb / group;
    int grp = id / (nb * group), gsz = group;
    if (grp >= full) { grp = full; gsz = ncb - full * group; }
    id -= grp * nb * group;
    ib = nb - 1 - id / gsz;
    cb = grp * group + id % gsz;
}

struct OzArgs {
    int nb, ncb;                        // row blocks of L^-1 (128 rows), candidate blocks of the chunk (32 candidates)
    int group;                          // candidate blocks per L2-resident group (a multiple of the cluster size)
    int NP, rows;                       // L^-1 is NP x NP; the K* slices have `rows` rows each
    const int* eP; int eK;
    double* part_ssq; long ldpart;
};

// ---------------------------------------------------------------------------------------
// The contraction: tile t of the L2-grouped, longest-first order (oz_tile_of) for t = blockIdx.x, + gridDim.x, ...
// A grid of one CTA per tile does one tile each; a grid of as many clusters as fit at once ("ozpersist" = 1) walks the list, so
// barriers and the pipeline fill are paid once and the producer runs ahead into the next tile during the epilogue.
// Warpgroup 0 (one thread, 40 registers after setmaxnreg) streams the 7 + 7 slice tiles of each 64-byte k-block into a
// 3-stage ring with TMA; warpgroups 1 and 2 (232 registers) each issue the 56 wgmma m64n32k32 of their 64 rows per
// stage with the L^-1 slice in registers, then fold the 7 level accumulators to fp64 (least significant level first),
// scale by the row exponent, square and reduce over the tile's 128 rows.
// Launched in clusters of CS = 1, 2 or 4 CTAs (cluster size = the launch's cluster dimension): the CTAs of a cluster
// take the same row block ib and the adjacent candidate blocks cb = CS p + rank, so they stage the same L^-1 slices.
// Each producer loads 128 / CS rows of every L^-1 slice (mapP has a box of 128 / CS rows) and multicasts them into
// the same stage of all CTAs of the cluster, and loads its own K* slices alone.  A stage is refilled only when the
// consumers of every CTA of the cluster have released it: the empty barriers count 2 CS arrivals.  The persistent
// walk goes by cluster tiles, so the CTAs of a cluster run the same k-block sequence.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(OZ_THREADS, 1)
gpk_oz_vargemm_kernel(const __grid_constant__ CUtensorMap mapP, const __grid_constant__ CUtensorMap mapK, const OzArgs g)
{
    extern __shared__ unsigned char oz_raw[];
    const uint32_t base = (smem_u32(oz_raw) + 1023u) & ~1023u;
    const uint32_t bar_full = base + OZ_NSTG * OZ_STAGE, bar_empty = bar_full + 8 * OZ_NSTG;
    const uint32_t red = base + OZ_NSTG * OZ_STAGE + 256;            // 2 x [8 consumer warps][32 columns] partial sums of V^2
    const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
    const uint32_t cs = oz_cluster_size(), rank = oz_cluster_rank();
    const int ncl = (int)(gridDim.x / cs), cid = (int)(blockIdx.x / cs);     // clusters of the grid, this CTA's cluster
    const int ncbc = g.ncb / (int)cs, gc = g.group / (int)cs;                // ... and the tile list in cluster tiles
    const int total = g.nb * ncbc;

    if (tid == 0) {
        for (int s = 0; s < OZ_NSTG; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 2 * cs); }
        fence_barrier_init();
        fence_proxy_async();
    }
    // peers multicast into this CTA's stages and arrive on its empty barriers only after they are initialised
    if (cs > 1) oz_cluster_sync(); else __syncthreads();

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (tid == 0) {
            const int prow = OZ_TM / (int)cs;                                         // L^-1 rows this CTA loads
            const uint16_t mask = (uint16_t)((1u << cs) - 1u);
            int it = 0;
            for (int t = cid; t < total; t += ncl) {
                int ib, cbc;
                oz_tile_of(t, g.nb, ncbc, gc, ib, cbc);
                const int cb = cbc * (int)cs + (int)rank;
                const int nkb = (ib + 1) * OZ_TM / OZ_KB;                                 // lower triangle only
                for (int kb = 0; kb < nkb; ++kb, ++it) {
                    const int s = it % OZ_NSTG;
                    if (it >= OZ_NSTG) oz_mbar_wait(bar_empty + 8 * s, (uint32_t)((it / OZ_NSTG - 1) & 1));
                    const uint32_t st = base + s * OZ_STAGE;
                    mbar_arrive_expect_tx(bar_full + 8 * s, OZ_STAGE);               // every byte of the stage lands here
#pragma unroll
                    for (int q = 0; q < OZ_S; ++q) {
                        const uint32_t pdst = st + q * OZ_A_SLICE + rank * prow * OZ_KB;
                        const int prow0 = q * g.NP + ib * OZ_TM + (int)rank * prow;
                        if (cs == 1) tma_load_2d(pdst, &mapP, kb * OZ_KB, prow0, bar_full + 8 * s);
                        else tma_load_2d_multicast(pdst, &mapP, kb * OZ_KB, prow0, bar_full + 8 * s, mask);
                        tma_load_2d(st + OZ_S * OZ_A_SLICE + q * OZ_B_SLICE, &mapK, kb * OZ_KB, q * g.rows + cb * OZ_TN,
                                    bar_full + 8 * s);
                    }
                }
            }
        }
        if (cs > 1) oz_cluster_sync();              // pairs with the consumers' cluster barrier at the end
        return;
    }
    // consumers: warpgroup c = wg - 1 owns tile rows 64 c .. 64 c + 63; accumulator element e of a thread sits at row
    // 16 w + lane / 4 + 8 ((e >> 1) & 1), column 8 (e >> 2) + 2 (lane % 4) + (e & 1)   (w = warp within the warpgroup)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int c = wg - 1, cw = (tid - 128) >> 5;                     // cw: consumer warp 0..7
    const int r0 = c * 64 + (cw & 3) * 16 + (lane >> 2);
    int it = 0, tl = 0;
    for (int t = cid; t < total; t += ncl, ++tl) {
        int ib, cbc;
        oz_tile_of(t, g.nb, ncbc, gc, ib, cbc);
        const int cb = cbc * (int)cs + (int)rank;
        const int nkb = (ib + 1) * OZ_TM / OZ_KB;                    // even: the k-loop takes two stages per pass
        uint32_t acc[OZ_S][16];
#pragma unroll
        for (int l = 0; l < OZ_S; ++l)
#pragma unroll
            for (int e = 0; e < 16; ++e) acc[l][e] = 0u;
        // Slice s of L^-1 is loaded into registers once per k-block and multiplies the K* slices t = 0 .. 6 - s into
        // acc[s + t]: one commit group per slice.  The fragment is double-buffered over the global slice sequence (two
        // stages = 14 slices per pass keep the buffer index static); wait_group 1 after each commit retires the group
        // two slices back, so its buffer can be reloaded, and after slice 0 of a stage, the previous stage's last group,
        // so that stage is handed back to the producer while this one runs.
        uint32_t fa[2][2][4];
        for (int kb = 0; kb < nkb; kb += 2) {
#pragma unroll
            for (int h = 0; h < 2; ++h, ++it) {
                const int s = it % OZ_NSTG;
                oz_mbar_wait(bar_full + 8 * s, (uint32_t)((it / OZ_NSTG) & 1));
                const uint32_t st = base + s * OZ_STAGE;
#pragma unroll
                for (int a = 0; a < OZ_S; ++a) {
                    uint32_t (&f)[2][4] = fa[(h * OZ_S + a) & 1];
                    oz_lda_frag(f, st + a * OZ_A_SLICE, c * 64 + (cw & 3) * 16, lane);
                    wgmma_arrive();
#pragma unroll
                    for (int tk = 0; tk < OZ_S - a; ++tk)
#pragma unroll
                        for (int k = 0; k < OZ_KB / OZ_UK; ++k)
                            oz_wgmma_rs(acc[a + tk], f[k], oz_desc(st + OZ_S * OZ_A_SLICE + tk * OZ_B_SLICE + k * OZ_UK));
                    wgmma_commit();
                    wgmma_wait_one();
                    if (a == 0 && (h == 1 || kb > 0) && (uint32_t)(tid & 127) < cs)       // previous stage fully read
                        oz_release_stage(bar_empty + 8 * ((it + OZ_NSTG - 1) % OZ_NSTG), cs, (uint32_t)(tid & 127));
                }
            }
        }
        wgmma_wait_all();
#pragma unroll
        for (int l = 0; l < OZ_S; ++l) oz_wgmma_fence(acc[l]);
        if ((uint32_t)(tid & 127) < cs) oz_release_stage(bar_empty + 8 * ((it + OZ_NSTG - 1) % OZ_NSTG), cs, (uint32_t)(tid & 127));
        const double rs0 = ldexp(1.0, g.eP[ib * OZ_TM + r0] + g.eK), rs1 = ldexp(1.0, g.eP[ib * OZ_TM + r0 + 8] + g.eK);
        // per thread 8 columns x 2 rows; column sums over the warp's 16 rows (lanes with equal lane % 4), then over warps.
        // The rounding sequence is a contract that tests/ozaki_model.py restates bit for bit (change both together):
        //   v = 0, v = fma(acc[lvl], 2^(-8 (lvl + 2)), v) for lvl = 6 .. 0;  x = v 2^(eP[row] + eK);
        //   warp w (rows 16 w .. 16 w + 15), row pair g: c_g = fma(x(16 w + g + 8), x(16 w + g + 8), x(16 w + g)^2)
        //   (nvcc contracts col += x * x);  butterfly ((c0 + c1) + (c2 + c3)) + ((c4 + c5) + (c6 + c7));
        //   tile column sum = (((0 + w0) + w1) + ...) + w7;  gpk_finish_kernel then adds part_ssq over ib = 0 .. nb - 1.
        double col[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) col[j] = 0.0;
#pragma unroll
        for (int e = 0; e < 16; ++e) {
            double v = 0.0;
#pragma unroll
            for (int lvl = OZ_S - 1; lvl >= 0; --lvl) v = fma(oz_i2d(acc[lvl][e]), ldexp(1.0, -8 * (lvl + 2)), v);
            const double x = v * (((e >> 1) & 1) ? rs1 : rs0);
            col[2 * (e >> 2) + (e & 1)] += x * x;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) col[j] += __shfl_xor_sync(0xffffffffu, col[j], o);
        const uint32_t redt = red + (uint32_t)((tl & 1) * 8 * OZ_TN * 8);
        if (lane < 4) {
#pragma unroll
            for (int j = 0; j < 8; ++j) sts64(redt + (uint32_t)((cw * OZ_TN + 8 * (j >> 1) + 2 * lane + (j & 1)) * 8), col[j]);
        }
        named_bar_sync(1, 256);
        const int et = tid - 128;
        if (et < OZ_TN) {
            double s2 = 0.0;
#pragma unroll
            for (int w8 = 0; w8 < 8; ++w8) s2 += lds64(redt + (uint32_t)((w8 * OZ_TN + et) * 8));
            g.part_ssq[(long)ib * g.ldpart + cb * OZ_TN + et] = s2;
        }
    }
    // no CTA leaves while a peer may still arrive on its empty barriers
    if (cs > 1) oz_cluster_sync();
}

// ---------------------------------------------------------------------------------------
// Covariance builder for the int8 path: gpk_cov_tma_kernel's tile loop (TMA-staged pre-scaled train operand, thread =
// 2 train points x CC candidates), but the fp64 K* never reaches HBM: every value k = amp * prod f(q) leaves as its
// OZ_S balanced base-256 digits (Kq[s][cand][j], two adjacent int8 per thread and slice), and the posterior mean's share
// sum_j k(c, j) alpha_j of this 128-column tile is reduced over the 64 threads of a candidate group and written to
// part_mu[tile][cand] (summed in fixed order by gpk_finish_kernel: deterministic).  Replaces K* store (8 B / element)
// + split kernel (8 B read, 8 B written) + mean dot (8 B read) by 8 B written per element.
// DIGITS = false compiles the digit stores out (Kq unused): the mean-only prediction (gpk_predict_mean) writes nothing
// but part_mu, with the same arithmetic and reduction order, so its mean is bit-identical to the int8 scoring pass's.
// Only that instance applies the kernel's factor (gpk_factor_value; z_j from the row-major training inputs Xenv): the digit split assumes 0 < k <= amp, so scoring with a factor takes the fp64 contraction.
// ---------------------------------------------------------------------------------------
template <int CC, bool DIGITS = true>
__global__ void __launch_bounds__(256, CC == 8 ? 2 : 4)
gpk_cov_oz_kernel(const __grid_constant__ CUtensorMap mapX, const KSpec ks, int n,
                  const double* __restrict__ cand, int dc, long m,
                  const double* __restrict__ lower, const double* __restrict__ upper,
                  const double* __restrict__ alpha, int eK, int8_t* __restrict__ Kq, long ldq, long slice_stride,
                  double* __restrict__ part_mu, long ldpart, int gx, const double* __restrict__ Xenv)
{
    // one CTA per (train tile bx of 128 columns, candidate group of 4 CC rows): a 1-D grid of gx x (candidate groups)
    constexpr int TC = 4 * CC;
    extern __shared__ unsigned char cov_raw[];
    const int tid = threadIdx.x;
    const long w = blockIdx.x;
    const int bx = (int)(w % gx);
    const long c0 = (w / gx) * TC;
    const int nt = ks.n_terms;
    const uint32_t base = (cov_smem_u32(cov_raw) + 127u) & ~127u;
    const uint32_t xs = base;                                   // nt x 128 doubles
    const uint32_t scb = xs + (uint32_t)nt * 1024u;             // TC x nt doubles
    const uint32_t bar = scb + (uint32_t)(TC * nt) * 8u;
    const uint32_t mred = bar + 8u;                             // 8 warps x CC doubles: cross-warp mean reduction
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"((uint32_t)nt * 1024u) : "memory");
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                     :: "r"(xs), "l"((uint64_t)&mapX), "r"(bar), "r"(bx * 128), "r"(0) : "memory");
    }
    const int jp = tid & 63, cgp = tid >> 6, lane = tid & 31;
    const double sc = ldexp(1.0, -eK);
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
    const int j0 = bx * 128 + 2 * jp;
    const bool v0 = j0 < n, v1 = j0 + 1 < n;
    const double a0 = v0 ? alpha[j0] : 0.0, a1 = v1 ? alpha[j0 + 1] : 0.0;
#pragma unroll
    for (int c = 0; c < CC; ++c) {
        const long ci = c0 + cgp * CC + c;
        const bool cv = ci < m;
        double k0 = (cv && v0) ? ks.amp * pr[c][0] : 0.0;
        double k1 = (cv && v1) ? ks.amp * pr[c][1] : 0.0;
        if (!DIGITS && ks.factor.kind != GPK_FACTOR_NONE && cv) {
            const double zc = gpk_factor_coord(ks.factor, cand + ci * dc, lower, upper);
            if (v0) k0 *= gpk_factor_value(ks.factor, zc, Xenv[(long)j0 * dc + ks.factor.axis]);
            if (v1) k1 *= gpk_factor_value(ks.factor, zc, Xenv[(long)(j0 + 1) * dc + ks.factor.axis]);
        }
        if (DIGITS) {
            // digits: two adjacent int8 per slice
            const unsigned long long y0 = oz_digits(k0 * sc), y1 = oz_digits(k1 * sc);
            int8_t* dst = Kq + ci * ldq + j0;
#pragma unroll
            for (int s2 = 0; s2 < OZ_S; ++s2)
                *reinterpret_cast<uint16_t*>(dst + (long)s2 * slice_stride) = (uint16_t)(oz_digit_of(y0, s2) | (oz_digit_of(y1, s2) << 8));
        }
        // mean share of this tile: reduce over the 64 threads (2 warps) of the candidate group, fixed order
        double pm = fma(k0, a0, k1 * a1);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) pm += __shfl_xor_sync(0xffffffffu, pm, off);
        if (lane == 0) asm volatile("st.shared.f64 [%0], %1;" :: "r"(mred + (uint32_t)(((tid >> 5) * CC + c) * 8)), "d"(pm) : "memory");
    }
    __syncthreads();
    if (tid < TC) {
        const int g = tid / CC, c = tid - g * CC;               // candidate group g = warps 2g, 2g + 1
        double lo2, hi2;
        asm volatile("ld.shared.f64 %0, [%1];" : "=d"(lo2) : "r"(mred + (uint32_t)(((2 * g) * CC + c) * 8)));
        asm volatile("ld.shared.f64 %0, [%1];" : "=d"(hi2) : "r"(mred + (uint32_t)(((2 * g + 1) * CC + c) * 8)));
        part_mu[(long)bx * ldpart + c0 + tid] = lo2 + hi2;
    }
}
inline size_t cov_oz_smem_bytes(int n_terms, int cc) { return (size_t)n_terms * 1024 + (size_t)4 * cc * n_terms * 8 + 8 + 8 * cc * 8 + 128; }

// ---------------------------------------------------------------------------------------
// int8 tensor-pipe issue-rate peak of this GPU (roofline denominator of the int8 contraction in bench.py): on every SM
// two warpgroups issue `iters` x 2 wgmma m64n128k32 s8 on one shared-memory operand pair (contents irrelevant) into a
// register accumulator; no loads in the loop.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void oz_wgmma_n128(uint32_t (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
                   "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
                   "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
                   "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
                   "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
                   "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
                   "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
                   "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void oz_wgmma_fence64(uint32_t (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; i += 16) oz_wgmma_fence(*reinterpret_cast<uint32_t(*)[16]>(d + i));
}
__global__ void __launch_bounds__(256, 1) gpk_peak_i8_kernel(int iters, int random_operands, unsigned* sink)
{
    extern __shared__ unsigned char pk_raw[];
    const uint32_t base = (smem_u32(pk_raw) + 1023u) & ~1023u;            // A: 128 x 64 B, B: 128 x 64 B (64B swizzle atoms)
    const int tid = threadIdx.x, wg = tid >> 7;
    // operands: a constant pattern (no switching activity in the datapath) or pseudo-random bytes (the statistics of real
    // digit slices: this is what decides how far the power limit lets the pipe run in a long measurement)
    for (int e = tid; e < 4096; e += 256) {
        uint32_t w = 0x01010101u * (e & 3);
        if (random_operands) { w = (uint32_t)e * 2654435761u + blockIdx.x * 40503u; w ^= w >> 15; w *= 2246822519u; w ^= w >> 13; }
        asm volatile("st.shared.u32 [%0], %1;" :: "r"(base + 4u * e), "r"(w) : "memory");
    }
    fence_proxy_async();
    __syncthreads();
    uint32_t d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0u;
    const uint32_t a0 = base + wg * 64 * 64;
    const uint64_t da0 = oz_desc(a0), da1 = oz_desc(a0 + 32), db0 = oz_desc(base + 8192), db1 = oz_desc(base + 8192 + 32);
    // batches of 8 iterations (16 MMAs) with one batch in flight while the next is issued; iters is a multiple of 8
    for (int i = 0; i < iters; i += 8) {
        oz_wgmma_fence64(d);
        wgmma_arrive();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            oz_wgmma_n128(d, da0, db0, 1u);
            oz_wgmma_n128(d, da1, db1, 1u);
        }
        wgmma_commit();
        asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
        oz_wgmma_fence64(d);
    }
    wgmma_wait_all();
    oz_wgmma_fence64(d);
    // The accumulator must be read, or the compiler drops every MMA of the loop. A store that almost never happens is
    // enough: it depends on all 64 registers.
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < 64; ++i) x ^= d[i];
    if (x == 0x9e3779b9u) sink[0] = x;
}
