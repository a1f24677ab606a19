// Operand-delivery rates of the int8 variance contraction (gpk_oz_vargemm_kernel) on the GPU it runs on.  One JSON line:
//   ss_m64n32_pops   wgmma m64n32k32 s8, both operands from shared memory (SS), descriptors cycling over one 70 KB stage
//                    laid out like the kernel's (7 A slices of 128 x 64 B, 7 B slices of 32 x 64 B, 64B swizzle): the
//                    28 slice pairs of a k-block, 56 MMAs per warpgroup
//   rs_m64n32_pops   the same products with A in registers (RS): each A slice is loaded once per k-block with ldmatrix and
//                    multiplies its 7 - s K* slices
//   ss_m64n128_pops  wgmma m64n128k32 SS on one operand pair, the int8 issue-rate peak bench.py uses as its denominator
//   tma_l2_tbps      TMA read rate into shared memory from an L2-resident 24 MB buffer, 64-byte x 128-row boxes
// Every SM runs one CTA; the MMA tests use two warpgroups and pseudo-random operand bytes.  ops = 2 x MACs.
// nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a int8_operand_rates.cu -o int8_operand_rates -ldl
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <dlfcn.h>
#include <cuda.h>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

constexpr int S = 7, KB = 64, A_SLICE = 128 * KB, B_SLICE = 32 * KB, STAGE = S * (A_SLICE + B_SLICE);

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint64_t desc64b(uint32_t a) {      // K-major SWIZZLE_64B descriptor, as in gpk_ozaki.cuh
    return (uint64_t)((a & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(512 >> 4) << 32) | ((uint64_t)2 << 62);
}
#define ACC16(d) "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), \
                 "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
__device__ __forceinline__ void mma_ss(uint32_t (&d)[16], uint64_t a, uint64_t b) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1;"
                 : ACC16(d) : "l"(a), "l"(b));
}
__device__ __forceinline__ void mma_rs(uint32_t (&d)[16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, 1;"
                 : ACC16(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
__device__ __forceinline__ void mma_ss128(uint32_t (&d)[64], uint64_t a, uint64_t b) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
                 "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, "
                 "%45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1;"
                 : ACC16(d), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]),
                   "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]),
                   "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]),
                   "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]),
                   "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]),
                   "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]),
                   "+r"(d[63])
                 : "l"(a), "l"(b));
}
__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void keep(uint32_t (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+r"(d[i]) :: "memory");
}

__device__ uint32_t base_of(unsigned char* raw) { return (smem_u32(raw) + 1023u) & ~1023u; }
__device__ void fill_random(uint32_t base, int bytes) {
    for (int e = threadIdx.x; e < bytes / 4; e += blockDim.x) {
        uint32_t w = (uint32_t)e * 2654435761u + blockIdx.x * 40503u;
        w ^= w >> 15; w *= 2246822519u; w ^= w >> 13;
        asm volatile("st.shared.u32 [%0], %1;" :: "r"(base + 4u * e), "r"(w) : "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
}
template <int N> __device__ void sink_acc(uint32_t (&d)[N], unsigned* sink) {
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) x ^= d[i];
    if (x == 0x9e3779b9u) sink[0] = x;
}

// (a) SS: per k-block and warpgroup the kernel's 56 MMAs (level-major, as the SS mainloop issued them)
__global__ void __launch_bounds__(256, 1) ss_kernel(int iters, unsigned* sink) {
    extern __shared__ unsigned char raw[];
    const uint32_t st = base_of(raw);
    fill_random(st, STAGE);
    const int wg = threadIdx.x >> 7;
    uint32_t acc[S][16];
#pragma unroll
    for (int l = 0; l < S; ++l)
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[l][e] = 0u;
    for (int i = 0; i < iters; ++i) {
        fence();
#pragma unroll
        for (int lvl = 0; lvl < S; ++lvl)
#pragma unroll
            for (int a = 0; a <= lvl; ++a)
#pragma unroll
                for (int k = 0; k < 2; ++k)
                    mma_ss(acc[lvl], desc64b(st + a * A_SLICE + wg * 64 * KB + 32 * k), desc64b(st + S * A_SLICE + (lvl - a) * B_SLICE + 32 * k));
        commit();
        wait<1>();
    }
    wait<0>();
#pragma unroll
    for (int l = 0; l < S; ++l) { keep(acc[l]); sink_acc(acc[l], sink); }
}

// (b) RS: the same products, slice-major, A fragment from ldmatrix, double-buffered, one commit group per slice
__global__ void __launch_bounds__(256, 1) rs_kernel(int iters, unsigned* sink) {
    extern __shared__ unsigned char raw[];
    const uint32_t st = base_of(raw);
    fill_random(st, STAGE);
    const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const int r = wg * 64 + w * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
    uint32_t acc[S][16], fa[2][2][4];
#pragma unroll
    for (int l = 0; l < S; ++l)
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[l][e] = 0u;
    for (int i = 0; i < iters; i += 2) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int a = 0; a < S; ++a) {
                uint32_t (&f)[2][4] = fa[(h * S + a) & 1];
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    const int chunk = 2 * k + (lane >> 4);
                    const uint32_t addr = st + a * A_SLICE + r * KB + ((chunk ^ ((r >> 1) & 3)) << 4);
                    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                                 : "=r"(f[k][0]), "=r"(f[k][1]), "=r"(f[k][2]), "=r"(f[k][3]) : "r"(addr) : "memory");
                }
                fence();
#pragma unroll
                for (int t = 0; t < S - a; ++t)
#pragma unroll
                    for (int k = 0; k < 2; ++k) mma_rs(acc[a + t], f[k], desc64b(st + S * A_SLICE + t * B_SLICE + 32 * k));
                commit();
                wait<1>();
            }
    }
    wait<0>();
#pragma unroll
    for (int l = 0; l < S; ++l) { keep(acc[l]); sink_acc(acc[l], sink); }
}

// (c) m64n128k32 SS on one operand pair, 16 MMAs per commit group
__global__ void __launch_bounds__(256, 1) n128_kernel(int iters, unsigned* sink) {
    extern __shared__ unsigned char raw[];
    const uint32_t st = base_of(raw);
    fill_random(st, 16384);
    const int wg = threadIdx.x >> 7;
    uint32_t d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0u;
    const uint64_t a0 = desc64b(st + wg * 64 * 64), a1 = desc64b(st + wg * 64 * 64 + 32);
    const uint64_t b0 = desc64b(st + 8192), b1 = desc64b(st + 8192 + 32);
    for (int i = 0; i < iters; i += 8) {
        keep(d);
        fence();
#pragma unroll
        for (int j = 0; j < 8; ++j) { mma_ss128(d, a0, b0); mma_ss128(d, a1, b1); }
        commit();
        wait<1>();
        keep(d);
    }
    wait<0>();
    keep(d);
    sink_acc(d, sink);
}

// (d) one thread per CTA streams boxes of 128 rows x 64 B through a ring of NR shared-memory slots
constexpr int NR = 16, BOX = 128 * 64;
__global__ void tma_kernel(const __grid_constant__ CUtensorMap map, int rowblocks, int colblocks, int boxes_per_cta) {
    extern __shared__ unsigned char raw[];
    const uint32_t buf = base_of(raw), bar = buf + NR * BOX;
    if (threadIdx.x != 0) return;
    for (int s = 0; s < NR; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar + 8 * s) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const int nboxes = rowblocks * colblocks;
    for (int i = 0; i < boxes_per_cta + NR; ++i) {
        const int s = i % NR;
        if (i >= NR) {
            uint32_t ok = 0, par = (uint32_t)((i / NR - 1) & 1);
            while (!ok)
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                             : "=r"(ok) : "r"(bar + 8 * s), "r"(par) : "memory");
        }
        if (i >= boxes_per_cta) continue;
        const int b = (int)(((long)blockIdx.x * 7919 + i) % nboxes);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar + 8 * s), "r"(BOX) : "memory");
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                     :: "r"(buf + s * BOX), "l"((uint64_t)&map), "r"(bar + 8 * s), "r"((b % colblocks) * 64), "r"((b / colblocks) * 128)
                     : "memory");
    }
}

template <typename F> float time_ms(F launch, int reps) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    launch();
    cudaDeviceSynchronize();
    float best = 1e30f;
    for (int r = 0; r < reps; ++r) {
        cudaEventRecord(e0);
        launch();
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return best;
}

// card name and power limit through NVML (read only), "unknown" / -1 when it is not available
static void card_info(char* name, int len, double* watts) {
    snprintf(name, len, "unknown");
    *watts = -1.0;
    void* h = dlopen("libnvidia-ml.so.1", RTLD_NOW);
    if (!h) return;
    typedef int (*InitFn)();
    typedef int (*HandleFn)(unsigned, void**);
    typedef int (*NameFn)(void*, char*, unsigned);
    typedef int (*LimitFn)(void*, unsigned*);
    InitFn init = (InitFn)dlsym(h, "nvmlInit_v2");
    HandleFn handle = (HandleFn)dlsym(h, "nvmlDeviceGetHandleByIndex_v2");
    NameFn nm = (NameFn)dlsym(h, "nvmlDeviceGetName");
    LimitFn lim = (LimitFn)dlsym(h, "nvmlDeviceGetEnforcedPowerLimit");
    void* dev = nullptr;
    if (!init || !handle || init() != 0) return;
    int ord = 0;
    cudaGetDevice(&ord);
    if (handle((unsigned)ord, &dev) != 0) return;
    if (nm) nm(dev, name, (unsigned)len);
    unsigned mw = 0;
    if (lim && lim(dev, &mw) == 0) *watts = mw / 1000.0;
}

int main() {
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, 0));
    const int sms = p.multiProcessorCount;
    unsigned* sink;
    CK(cudaMalloc(&sink, 4));
    const int smem_mma = STAGE + 1024;
    CK(cudaFuncSetAttribute(ss_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_mma));
    CK(cudaFuncSetAttribute(rs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_mma));
    CK(cudaFuncSetAttribute(n128_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 + 1024));
    const int smem_tma = NR * BOX + 1024 + 8 * NR;
    CK(cudaFuncSetAttribute(tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_tma));

    // MACs per CTA: two warpgroups x (56 per k-block of m64n32k32 | 16 per pass of m64n128k32) x 64 n k
    const int it32 = 4000, it128 = 16000;
    const double ops32 = 2.0 * sms * 2 * 56 * it32 * (64.0 * 32 * 32), ops128 = 2.0 * sms * 2 * 2 * it128 * (64.0 * 128 * 32);
    const float ms_ss = time_ms([&] { ss_kernel<<<sms, 256, smem_mma>>>(it32, sink); }, 5);
    const float ms_rs = time_ms([&] { rs_kernel<<<sms, 256, smem_mma>>>(it32, sink); }, 5);
    const float ms_128 = time_ms([&] { n128_kernel<<<sms, 256, 16384 + 1024>>>(it128, sink); }, 5);
    CK(cudaGetLastError());

    // 24 MB int8 buffer, 6144 rows x 4096 bytes, 64-byte x 128-row boxes with the kernel's 64B swizzle
    const int rows = 6144, cols = 4096;
    void* buf;
    CK(cudaMalloc(&buf, (size_t)rows * cols));
    CK(cudaMemset(buf, 0x5a, (size_t)rows * cols));
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q));
    CUtensorMap map;
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)cols};
    cuuint32_t box[2] = {64u, 128u}, estr[2] = {1, 1};
    if (((EncodeFn)fp)(&map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, buf, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
        fprintf(stderr, "cuTensorMapEncodeTiled failed\n");
        return 1;
    }
    const int per_cta = 8192;
    const float ms_tma = time_ms([&] { tma_kernel<<<sms, 32, smem_tma>>>(map, rows / 128, cols / 64, per_cta); }, 5);
    CK(cudaGetLastError());
    const double tbps = (double)sms * per_cta * BOX / (ms_tma * 1e-3) / 1e12;

    char name[96];
    double watts;
    card_info(name, sizeof(name), &watts);
    printf("{\"gpu\": \"%s\", \"power_limit_w\": %.0f, \"sms\": %d, \"ss_m64n32_pops\": %.3f, \"rs_m64n32_pops\": %.3f, "
           "\"ss_m64n128_pops\": %.3f, \"tma_l2_tbps\": %.2f}\n",
           name, watts, sms, ops32 / (ms_ss * 1e-3) / 1e15, ops32 / (ms_rs * 1e-3) / 1e15, ops128 / (ms_128 * 1e-3) / 1e15, tbps);
    return 0;
}
