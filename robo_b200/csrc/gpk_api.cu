// gpk_api.cu — C ABI (include/gpk.h) and host orchestration of the sm_90a kernels.
//
// Data layout in HBM (all fp64, row-major, NP = n rounded up to 128, nb = NP / 128):
//   Xt    [d][NP]        training inputs, transposed (coalesced reads in the covariance builder)
//   Kbuf  [NP+128][NP]   K, overwritten in place by its lower Cholesky factor L; block row nb is
//                        the augmented right-hand side: after the factorisation row NP holds
//                        z = L^-1 (y - mean), so the log-likelihood needs no separate solve
//   P     [NP][NP]       L^-1   (lower; diagonal blocks come out of the Cholesky diag kernel)
//   Q     [NP][NP]       L^-T   (upper) — only needed while building P, and for alpha
//   W     [NP][NP]       scratch of the recursive triangular inverse
//   Kstar [chunk][NP]    K(X*, X) of the current candidate chunk
//   part_mu/part_ssq [nb][chunk]  per-row-block partial sums of the variance contraction
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <dlfcn.h>
#include <string>
#include <vector>

#include "gpk_gemm.cuh"
#include "gpk_kernels.cuh"
#include "gpk_diag16.cuh"
#include "gpk_ozaki.cuh"
#include "gpk_de.cuh"
#include "gpk_lbfgs.cuh"
#include "gpk_cmaes.cuh"
#include "gpk_direct.cuh"
#include "gpk_es.cuh"
#include "gpk_esmc.cuh"
#include "gpk_rs.cuh"
#include "gpk_hyper.cuh"
#include "gpk_hyperopt.cuh"
#include "gpk_hyper_blocked.cuh"
#include "gpk_blr.cuh"
#include "gpk_rf.cuh"
#include "gpk_bnn.cuh"
#include "gpk_dngo.cuh"

namespace {

constexpr int APP_KC = 512;          // split-K chunk of gpk_fit_append's long contractions

struct Range { int off = 0, cnt = 0; };

// a device allocation of cap bytes, freed with its owner
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
};

// the model a handle holds: a Gaussian process unless a gpk_*_set_data made it a surrogate, which it stays for life
enum ModelKind { MODEL_GP, MODEL_BLR, MODEL_RF, MODEL_BNN, MODEL_DNGO };

}  // namespace

// Every CUDA resource of a handle is released with it: the buffers by their DevBuf members, the streams, events and
// pinned host memory by the destructor.
struct gpk_handle {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t own_stream = nullptr;
    cudaStream_t side_stream = nullptr;     // trailing updates of the look-ahead Cholesky
    std::vector<cudaEvent_t> ev_panel, ev_rest;
    // variance contraction on the int8 tensor pipe (gpk_ozaki.cuh)
    struct {
        int enabled = 1;            // 0 = fp64 DMMA kernels
        DevBuf Pq, Kq, Kq2, eP, emax, pmu2;
        int last_variant = 0;       // contraction of the last int8 launch: 1 = gpk_oz_vargemm_kernel, + 8 when it walked the tile
                                    // list persistently, + 16 / + 32 in clusters of 2 / 4 CTAs
        int cluster = 4;            // CTAs per cluster of the int8 contraction (1, 2 or 4): they share the L^-1 slices by TMA
                                    // multicast [default 4: tools/persist_threshold.py and bench.py on an H100, DESIGN 9.5]
        int map_cs = 0;             // cluster size mapP's box was encoded for (0: not encoded)
        int max_clusters[5] = {0, 0, 0, 0, 0};  // co-resident clusters of the contraction per cluster size (0: not queried)
        int persist = 3;            // 1: one CTA per SM walks the tile list; 0: one CTA per tile; 3 = automatic [default]: persistent
                                    // for N <= 4096 (tools/persist_threshold.py and bench.py on an H100 with 4-CTA clusters: the
                                    // walk is as fast or faster up to N = 4096, one CTA per tile is faster at 6144)
        int grid = 0;               // most clusters the persistent walk launches (0: as many as fit at once [default])
        DevBuf probe;               // scratch of gpk_oz_contract (operands, slices, exponents, partial sums)
        long linv_serial = -1;      // linv_serial the slices of L^-1 were made for
        int emax_host = 0;
        CUtensorMap mapP, mapK, mapK2;
        double launches = 0;
    } oz;
    long linv_serial = 0;           // bumped whenever L^-1 is (re)built
    int n_sm = 0;
    char err[1024] = {0};
    long chunk = 16384;
    bool chunk_user = false;        // false: candidates per scoring pass chosen from N (chunk_rows)
    int diag_prof = 0;            // 1: the blocked diagonal kernel records clock64() stamps per phase (diagnostics)
    DevBuf dprof;

    // model
    int n = 0, d = 0, NP = 0, nb = 0;
    bool has_data = false, has_spec = false, fitted = false, linv_ready = false, alpha_ready = false;
    KSpec spec;
    bool has_bounds = false;
    std::vector<double> task_theta; // gpk_set_task_factor's packed log-entries (the gradient's contraction)
    std::vector<int> col_tasks;     // per input column: 1 + the largest value when every value is an integer >= 0 (the
                                    // fewest tasks that make the column valid task indices), INT_MAX otherwise
    int norm_out = 0;
    double y_mean = 0.0, y_std = 1.0, mean = 0.0, diag_add = 0.0;

    // device buffers
    DevBuf Xrow, Xt, y, Kbuf, P, Q, W, lower, upper, logdet_part, scal, status;
    DevBuf Kstar2;
    DevBuf Xts;                     // training inputs, term-major and pre-scaled (operand of gpk_cov_tma_kernel)
    cudaStream_t copy_stream = nullptr;
    std::vector<cudaEvent_t> ev_copied;
    DevBuf cand, Kstar, part_mu, part_ssq, out_mu, out_var, out_acq, block_best, best, nneg;
    DevBuf Vt, cov, XsT, tmpjobs, alpha, tmp1, tmp2, tmp3;
    int layout_NP = -1;           // NP the P/Q/W buffers were zeroed for

    // job tables: the GEMM jobs of the fit, L^-1, K^-1 and gpk_fit_append, and their ranges, built for nb row blocks
    DevBuf jobs;
    struct {
        int nb = -1;
        std::vector<Range> syrk, tri1, tri2, trsm32, pu32;
        std::vector<Range> syrk2;       // depth-2 trailing update: columns >= k+2 with panels k-1 and k in one contraction (K = 256)
        Range kinv;
        Range app_syrk, app_p;          // gpk_fit_append (last block row only)
        Range app_row2, app_t2;         // its two long contractions, split-K
    } ranges;
    int depth2 = 2;                 // 0 / 1, or 2 = automatic: on for nb >= 48 (trailing updates gate the fit only there)

    // tensor maps
    CUtensorMap mapK, mapP, mapQ, mapW, mapKs, mapVt;
    CUtensorMap mapK32, mapKs2;     // mapK32: Kbuf with a 32-row box, A operand of the 32-row chain GEMMs
    long mapKs2_rows = 0;
    std::vector<cudaEvent_t> ev_cov, ev_gemm;
    int overlap = 1;                // build K* of chunk i+1 on the side stream while chunk i contracts
    int mean_only = 1;              // gpk_predict_mean: 1 = mean-only builder pass [default]; 0 = the full scoring pass
    bool maps_ok = false;
    long mapKs_rows = 0, mapVt_rows = 0;

    // timing
    struct {
        cudaEvent_t ev[16] = {};
        std::vector<cudaEvent_t> ev_g0, ev_g1;    // timed pairs around every variance-GEMM launch of the last scoring call
        int last_nchunks = 0;
        bool fit_timed = false, score_timed = false;
        double launches_total = 0, launches_var = 0;
    } timing;
    cudaEvent_t ev_order = nullptr;
    double* pin = nullptr;        // pinned host: [0..1] z^T z, logdet ; [2] status (as int) for async fits
    double* stage[2] = {nullptr, nullptr};    // pinned staging of pageable candidate batches (gpk_acq)
    size_t stage_cap = 0;
    bool fit_pending = false;

    // scratch of the entry points over several handles, owned by the first handle of the call
    struct {
        // several models, one batch (gpk_acq_multi)
        DevBuf cand, A, B, out, bb;
        cudaEvent_t ev = nullptr;       // fork_join's start of the sub-handles' work
        // differential evolution (gpk_maximize_de): population, trials, scaled batch, energies, {status, limits, winner},
        // radix-sort scratch of the LHS initialisation
        DevBuf de_pop, de_trial, de_param, de_E, de_small, de_sort;
        // multi-start L-BFGS (gpk_maximize_lbfgs): per-start state, pair memory, scored batch, active lists, status record
        DevBuf lb_buf;
        // CMA-ES (gpk_maximize_cmaes*): state, status record, constant table, bounds and x0, the Z / Y / G / P rows of a
        // generation (gpk_cmaes_draws uses it as scratch)
        DevBuf cma_buf;
        // DIRECT (gpk_maximize_direct*): state, status record, box, rectangle store, row buffer, selection
        DevBuf dir_buf;
        DevBuf ep_buf;                  // scratch of gpk_ep_joint_min (operands, raw and renormalised outputs, status)
        // information gain per unit cost (gpk_es_cost_multi): the batch under the objective's and the cost's Fabolas
        // transform and the configuration bounds; owned by the first objective handle of the call
        DevBuf fab_in;
        // representer sampling (gpk_sample_representers): walkers, log-probabilities, proposals, scored batches, bounds,
        // accept counts, seeds, slots
        DevBuf rs_buf;
    } multi;
    // entropy search (gpk_es_update / gpk_es_compute): EP state, W, bounds, scaled zb, U = K^-1 K(X, zb), per-chunk v, sigma
    struct {
        DevBuf state, U, work, in;
        int nb = 0, np = 0;
        double sn2 = 0.0, H = 0.0;
        long linv_serial = -1;          // linv_serial U was built for (-1: no update yet)
        int kind = 0;                   // which update is current: ES_KIND_EP (gpk_es_update) or ES_KIND_MC (gpk_esmc_update)
    } es;
    // sampling-based entropy search (gpk_esmc_update / gpk_esmc_compute): Mb, Vb, W, lmb, scaled zb and the draws F;
    // the scratch of gpk_mc_pmin / gpk_mc_draws; the two status words of the last pass (gpk_esmc.cuh)
    struct {
        DevBuf state, buf, stat;
        int nf = 0;
        long last_jitter = 0;
    } mc;
    // hyper-parameter sampling (gpk_sample_hypers): theta -> kernel map and prior, walkers / log-posteriors / accepts;
    // the byte budget of a chunk of the blocked path (gpk_hyper_blocked.cuh, "hyper_batch_bytes")
    struct {
        bool has_model = false;
        HyperModel model;
        DevBuf buf;
        long batch_bytes = GPK_HYPER_BATCH_BYTES;
    } hyper;
    // a surrogate handle serves its own entry points and the scoring ones only; its scoring pass uses block_best, best
    // and nneg as the GP's does
    ModelKind model = MODEL_GP;
    // Bayesian linear regression (gpk_blr.cuh, gpk_blr_set_data).  data: Phi (n x F), y, G = Phi^T Phi, b = Phi^T y;
    // post: the fit's M (k x F), L^-1 and S (k x F x F each), 1 / beta (k), failure flags; work: thetas / walkers and
    // their values
    struct {
        bool fitted = false;
        int basis = 0, F = 0, k = 0;
        BlrPrior prior;
        DevBuf data, post, work;
    } blr;
    // random forest (gpk_rf.cuh, gpk_rf_set_data).  data: X (n x d), y (n), the per-feature row order (d x n ints);
    // work: the growth's per-tree multiplicities, lists and segments; nodes: the trees (RfNodes)
    struct {
        bool fitted = false;
        int T = 0, total = 0;
        DevBuf data, work, nodes;
    } rf;
    // Bayesian neural network (gpk_bnn.cuh, gpk_bnn_set_data).  data: the scaled X (n x d), y (n), the input mean and
    // std (d each), with the y statistics in ymean / ystd (a DNGO handle keeps its training set here too); samples: the
    // kept networks (S x P); state: the chain's final theta, p, tau, g, vhat (P each)
    struct {
        int P = 0, S = 0;
        double ymean = 0.0, ystd = 1.0;
        DevBuf data, samples, state;
    } bnn;
    // DNGO (gpk_dngo.cuh, gpk_dngo_set_data): the training set in bnn.data, the trained net (P), Adam's m and v (P each,
    // after t steps; -1: the net was set, not trained), the scoring pack and the collapse's failure flag.  The Bayesian
    // linear regression over the features lives in blr (F = 50, no basis).
    struct {
        bool trained = false, fitted = false;
        int P = 0;
        long long t = -1;
        DevBuf net, state, pack;
    } dngo;
    // multi-GPU (gpk_comm_*): NCCL communicator bound at run time, one 16-byte pair per rank
    struct {
        void* comm = nullptr;
        int rank = 0, world = 1;
        DevBuf gather, best_global;
    } dist;

    // the caller makes the handle's device current; the communicator goes first (gpk_comm_destroy)
    ~gpk_handle() {
        for (cudaEvent_t e : timing.ev)
            if (e) cudaEventDestroy(e);
        for (cudaEvent_t e : {ev_order, multi.ev})
            if (e) cudaEventDestroy(e);
        for (const auto* evs : {&ev_panel, &ev_rest, &ev_cov, &ev_gemm, &ev_copied, &timing.ev_g0, &timing.ev_g1})
            for (cudaEvent_t e : *evs) cudaEventDestroy(e);
        for (cudaStream_t s : {copy_stream, side_stream, own_stream})
            if (s) cudaStreamDestroy(s);
        for (double* p : {pin, stage[0], stage[1]})
            if (p) cudaFreeHost(p);
    }
};

namespace {

void set_err(gpk_handle* h, const char* fmt, ...) {
    if (!h) return;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(h->err, sizeof(h->err), fmt, ap);
    va_end(ap);
}

#define CK(call)                                                                                 \
    do {                                                                                         \
        cudaError_t e_ = (call);                                                                 \
        if (e_ != cudaSuccess) {                                                                 \
            set_err(h, "%s -> %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__);   \
            return GPK_CUDA_ERROR;                                                               \
        }                                                                                        \
    } while (0)

#define CKL()                                                                                    \
    do {                                                                                         \
        cudaError_t e_ = cudaGetLastError();                                                     \
        if (e_ != cudaSuccess) {                                                                 \
            set_err(h, "kernel launch -> %s (%s:%d)", cudaGetErrorString(e_), __FILE__, __LINE__); \
            return GPK_CUDA_ERROR;                                                               \
        }                                                                                        \
        h->timing.launches_total += 1;                                                           \
    } while (0)

#define BAD(...)                           \
    do {                                   \
        set_err(h, __VA_ARGS__);           \
        return GPK_BAD_ARG;                \
    } while (0)

int ensure(gpk_handle* h, DevBuf& b, size_t bytes, bool* grew = nullptr) {
    if (grew) *grew = false;
    if (bytes <= b.cap && b.p) return GPK_OK;
    if (b.p) CK(cudaFree(b.p));
    b.p = nullptr;
    b.cap = 0;
    size_t want = std::max<size_t>(bytes, 256);
    CK(cudaMalloc(&b.p, want));
    b.cap = want;
    if (grew) *grew = true;
    return GPK_OK;
}

template <typename T> T* ptr(const DevBuf& b) { return reinterpret_cast<T*>(b.p); }

// grows evs to n events created with flags; the handle's destructor releases them
int grow_events(gpk_handle* h, std::vector<cudaEvent_t>& evs, size_t n, unsigned flags) {
    while (evs.size() < n) {
        cudaEvent_t e;
        CK(cudaEventCreateWithFlags(&e, flags));
        evs.push_back(e);
    }
    return GPK_OK;
}

// the two timing events of a gpk_measure_* call, released on every return
struct TimerEvents {
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    ~TimerEvents() {
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
    }
};

inline long round_up(long x, long m) { return (x + m - 1) / m * m; }

// ---- tensor maps ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// fp64 row-major matrix [rows][ld]; box = 128 rows x 16 doubles (128 B), 128B swizzle.
int make_map(gpk_handle* h, CUtensorMap* map, void* base, long rows, long cols, long ld, int box_rows = BM) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) {
        set_err(h, "cuTensorMapEncodeTiled entry point not available");
        return GPK_CUDA_ERROR;
    }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 8};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, base, dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_err(h, "cuTensorMapEncodeTiled failed with CUresult %d (rows=%ld cols=%ld ld=%ld)", (int)r, rows, cols, ld);
        return GPK_CUDA_ERROR;
    }
    return GPK_OK;
}

// term-major operand [n_terms][ld] of the covariance builder: box = n_terms rows x 128 columns, no swizzle
int make_cov_map(gpk_handle* h, CUtensorMap* map, void* base, int n_terms, long ld) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) {
        set_err(h, "cuTensorMapEncodeTiled entry point not available");
        return GPK_CUDA_ERROR;
    }
    cuuint64_t dims[2] = {(cuuint64_t)ld, (cuuint64_t)n_terms};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 8};
    cuuint32_t box[2] = {128u, (cuuint32_t)n_terms};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_err(h, "cuTensorMapEncodeTiled (covariance operand) failed with CUresult %d (terms=%d ld=%ld)", (int)r, n_terms, ld);
        return GPK_CUDA_ERROR;
    }
    return GPK_OK;
}

// "Transposed" operand of the covariance builder for n points X (row-major, n x d) into dst with ld columns:
// term-major and pre-scaled (dst needs n_terms x ld doubles).  lo / up: input bounds to apply first (NULL: none).
int build_cov_operand(gpk_handle* h, cudaStream_t st, const double* X, long n, int d, const double* lo, const double* up,
                      double* dst, long ld) {
    const long total = (long)h->spec.n_terms * ld;
    gpk_termmajor_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(h->spec, X, n, d, lo, up, dst, ld);
    CKL();
    return GPK_OK;
}
inline size_t cov_operand_rows(const gpk_handle* h, int d) { return (size_t)std::max(d, h->spec.n_terms); }

// out[c][j] = k(cand_c, point_j) for m candidates (row-major raw inputs, bounds lo / up applied on the fly) against
// the n points of `operand` (built by build_cov_operand, ld = ldx columns); out has ldo columns and at least
// round_up(m, tile) rows.  small: the 128 x 16 tile variant that fits next to a resident variance-GEMM CTA.
// pts (row-major raw inputs, dc columns, bounds plo / pup) are the operand's n points before build_cov_operand: the
// kernel's factor reads its coordinate there, since the term-major operand carries the radial terms only.
int launch_cov_tiles(gpk_handle* h, cudaStream_t st, const double* operand, long ldx, int n, const double* cand, int dc,
                     long m, long m_padded, const double* lo, const double* up, double* out, long ldo, int tri, bool small,
                     const double* pts, const double* plo, const double* pup) {
    const unsigned gx = (unsigned)(ldx / 128);
    CUtensorMap map;
    int rc = make_cov_map(h, &map, (void*)operand, h->spec.n_terms, ldx);
    if (rc) return rc;
    if (small)
        gpk_cov_tma_kernel<4><<<dim3(gx, (unsigned)(m_padded / 16)), 256, cov_tma_smem_bytes(h->spec.n_terms, 4), st>>>(
            map, h->spec, n, cand, dc, m, lo, up, out, ldo, tri);
    else
        gpk_cov_tma_kernel<8><<<dim3(gx, (unsigned)(m_padded / 32)), 256, cov_tma_smem_bytes(h->spec.n_terms, 8), st>>>(
            map, h->spec, n, cand, dc, m, lo, up, out, ldo, tri);
    CKL();
    if (h->spec.factor.kind != GPK_FACTOR_NONE && m > 0) {
        gpk_factor_scale_kernel<<<dim3(gx, (unsigned)std::min<long>((m + 1) / 2, 1024)), 256, 0, st>>>(
            h->spec, cand, dc, m, lo, up, pts, dc, n, plo, pup, out, ldo, tri);
        CKL();
    }
    return GPK_OK;
}

// ---- GEMM launch ---------------------------------------------------------------------------
// Launch with the programmatic-stream-serialization attribute (PDL): the kernel's launch latency and prologue
// overlap the tail of the previous kernel on the stream; the kernels call cudaGridDependencySynchronize().
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// int8 contraction launch in clusters of cs CTAs (grid a multiple of cs)
template <typename... KArgs, typename... Args>
cudaError_t launch_oz(void (*kernel)(KArgs...), unsigned grid, int cs, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(OZ_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = cs > 1 ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// How many clusters of cs contraction CTAs fit on the device at once (the grid of the persistent walk), once per handle
int oz_max_clusters(gpk_handle* h, int cs, int* out) {
    if (h->oz.max_clusters[cs] == 0) {
        if (cs == 1) {
            h->oz.max_clusters[cs] = std::max(h->n_sm, 1);
        } else {
            cudaLaunchConfig_t cfg;
            memset(&cfg, 0, sizeof(cfg));
            cfg.gridDim = dim3((unsigned)cs);
            cfg.blockDim = dim3(OZ_THREADS);
            cfg.dynamicSmemBytes = OZ_SMEM;
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = (unsigned)cs;
            attr[0].val.clusterDim.y = 1;
            attr[0].val.clusterDim.z = 1;
            cfg.attrs = attr;
            cfg.numAttrs = 1;
            int n = 0;
            CK(cudaOccupancyMaxActiveClusters(&n, gpk_oz_vargemm_kernel, &cfg));
            if (n < 1) { set_err(h, "no cluster of %d int8 contraction CTAs fits on this device", cs); return GPK_CUDA_ERROR; }
            h->oz.max_clusters[cs] = n;
        }
    }
    *out = h->oz.max_clusters[cs];
    return GPK_OK;
}

// One launch of the int8 contraction over nb row blocks of L^-1 and the ncb = rows_padded / 32 candidate blocks whose
// slices mapK covers (stacked [7][rows][NP]), with the handle's "ozcluster", "ozpersist" and "ozgrid": L2 group,
// persistent grid and the variant code timings() reports.  Shared by score_dev and gpk_oz_contract.
int launch_oz_contraction(gpk_handle* h, const CUtensorMap& mapP, const CUtensorMap& mapK, int nb, long rows_padded,
                          long NP, long rows, const int* eP, int eK, double* part_ssq, long ldpart) {
    OzArgs o;
    o.nb = nb; o.ncb = (int)(rows_padded / OZ_TN); o.NP = (int)NP; o.rows = (int)rows;
    // a group's K* slices take about 24 MB, half of the L2; whole clusters of candidate blocks (ncb = rows_padded / 32 is
    // a multiple of 4, so of every cluster size)
    const int cs = h->oz.cluster;
    o.group = (int)std::min<long>(512, std::max<long>(4, ((long)24 << 20) / ((long)OZ_TN * NP * OZ_S))) / cs * cs;
    o.eP = eP; o.eK = eK;
    o.part_ssq = part_ssq; o.ldpart = ldpart;
    const int persist = h->oz.persist == 3 ? (nb <= 32 ? 1 : 0) : h->oz.persist;
    const int tiles = o.nb * o.ncb;
    int grid = tiles;
    if (persist == 1) {
        int nclusters = 0, rc;
        if ((rc = oz_max_clusters(h, cs, &nclusters))) return rc;
        if (h->oz.grid > 0) nclusters = std::min(nclusters, h->oz.grid);
        grid = cs * std::min(tiles / cs, nclusters);
    }
    h->oz.last_variant = 1 + (persist == 1 ? 8 : 0) + (cs == 2 ? 16 : cs == 4 ? 32 : 0);
    CK(launch_oz(gpk_oz_vargemm_kernel, (unsigned)grid, cs, (size_t)OZ_SMEM, h->stream, mapP, mapK, o));
    CKL();
    return GPK_OK;
}

// MI = 8: 128-row tiles on gpk_gemm_ws_kernel; MI = 2: the 32-row chain tiles (store only), through PDL
template <int EPI, int MI = 8>
int launch_gemm(gpk_handle* h, const CUtensorMap& mA, const CUtensorMap& mB, const GemmArgs& a, int njobs,
                cudaStream_t stream = nullptr) {
    static_assert(MI == 8 || (MI == 2 && EPI == EPI_STORE), "128-row tiles, or 32-row chain tiles that store");
    if (njobs <= 0) return GPK_OK;
    if (stream == nullptr) stream = h->stream;
    if constexpr (MI == 2) {
        CK(launch_pdl(gpk_gemm_nt_kernel, dim3(njobs), dim3(GEMM_THREADS), (size_t)GEMM_SMEM_CHAIN, stream, mA, mB, a));
        h->timing.launches_total += 1;
        return GPK_OK;
    }
    gpk_gemm_ws_kernel<EPI><<<njobs, WS_THREADS, GEMM_SMEM_TMA, stream>>>(mA, mB, a);
    CKL();
    return GPK_OK;
}

int set_kernel_attrs(gpk_handle* h) {
    CK(cudaFuncSetAttribute(gpk_gemm_ws_kernel<EPI_STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM_TMA));
    CK(cudaFuncSetAttribute(gpk_gemm_ws_kernel<EPI_COLREDUCE>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM_TMA));
    CK(cudaFuncSetAttribute(gpk_gemm_nt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM_CHAIN));
    CK(cudaFuncSetAttribute(gpk_oz_vargemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, OZ_SMEM));
    CK(cudaFuncSetAttribute(gpk_cov_oz_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cov_oz_smem_bytes(GPK_MAX_TERMS, 8)));
    CK(cudaFuncSetAttribute(gpk_cov_oz_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cov_oz_smem_bytes(GPK_MAX_TERMS, 4)));
    CK(cudaFuncSetAttribute(gpk_cov_oz_kernel<8, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cov_oz_smem_bytes(GPK_MAX_TERMS, 8)));
    {
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, h->device));
        h->n_sm = prop.multiProcessorCount;
    }
    CK(cudaFuncSetAttribute(gpk_cov_tma_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cov_tma_smem_bytes(GPK_MAX_TERMS, 8)));
    CK(cudaFuncSetAttribute(gpk_cov_tma_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cov_tma_smem_bytes(GPK_MAX_TERMS, 4)));
    CK(cudaFuncSetAttribute(gpk_potrf_diag_dmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DIAG_SMEM));
    return GPK_OK;
}

// ---- job tables ----------------------------------------------------------------------------
struct Node { int lo, mid, hi, height; };

int build_nodes(int lo, int hi, std::vector<Node>& nodes) {
    if (hi - lo <= 1) return 0;
    int mid = lo + (hi - lo + 1) / 2;
    int hl = build_nodes(lo, mid, nodes);
    int hr = build_nodes(mid, hi, nodes);
    int ht = 1 + std::max(hl, hr);
    nodes.push_back({lo, mid, hi, ht});
    return ht;
}

int build_job_tables(gpk_handle* h) {
    const int nb = h->nb;
    if (h->ranges.nb == nb) return GPK_OK;
    std::vector<GemmJob> jobs;
    h->ranges.syrk.assign(nb, Range());
    for (int k = 0; k < nb; ++k) {
        h->ranges.syrk[k].off = (int)jobs.size();
        for (int j = k + 1; j < nb; ++j)
            for (int i = j; i <= nb; ++i)
                jobs.push_back({i * BM, j * BM, k * BM, (k + 1) * BM, i * BM, j * BM, 0, 0});
        h->ranges.syrk[k].cnt = (int)jobs.size() - h->ranges.syrk[k].off;
    }
    // depth-2 trailing update (odd steps k >= 1): tile (i, j), j >= k+2, receives panels k-1 and k in ONE contraction
    // over the 256 columns [(k-1)*128, (k+1)*128): same arithmetic, in the same order, as the two separate updates
    h->ranges.syrk2.assign(nb, Range());
    for (int k = 1; k < nb; k += 2) {
        h->ranges.syrk2[k].off = (int)jobs.size();
        for (int j = k + 2; j < nb; ++j)
            for (int i = j; i <= nb; ++i)
                jobs.push_back({i * BM, j * BM, (k - 1) * BM, (k + 1) * BM, i * BM, j * BM, 0, 0});
        h->ranges.syrk2[k].cnt = (int)jobs.size() - h->ranges.syrk2[k].off;
    }
    // 32-row versions of the two GEMMs on the critical chain (row split only: the in-place panel solve
    // stays race-free because every CTA reads and writes its own rows)
    h->ranges.trsm32.assign(nb, Range());
    h->ranges.pu32.assign(nb, Range());
    for (int k = 0; k < nb; ++k) {
        h->ranges.trsm32[k].off = (int)jobs.size();
        for (int i = k + 1; i <= nb; ++i)
            for (int q = 0; q < 4; ++q) {
                if (i == nb && q > 0) break;         // augmented block: only its first rows are non-zero
                jobs.push_back({i * BM + 32 * q, k * BM, k * BM, (k + 1) * BM, i * BM + 32 * q, k * BM, 0, 0});
            }
        h->ranges.trsm32[k].cnt = (int)jobs.size() - h->ranges.trsm32[k].off;
        h->ranges.pu32[k].off = (int)jobs.size();
        if (k + 1 < nb)
            for (int i = k + 1; i <= nb; ++i)
                for (int q = 0; q < 4; ++q) {
                    if (i == nb && q > 0) break;
                    jobs.push_back({i * BM + 32 * q, (k + 1) * BM, k * BM, (k + 1) * BM, i * BM + 32 * q, (k + 1) * BM, 0, 0});
                }
        h->ranges.pu32[k].cnt = (int)jobs.size() - h->ranges.pu32[k].off;
    }
    std::vector<Node> nodes;
    int hmax = build_nodes(0, nb, nodes);
    h->ranges.tri1.assign(hmax + 1, Range());
    h->ranges.tri2.assign(hmax + 1, Range());
    auto by_len = [](const GemmJob& a, const GemmJob& b) { return (a.k1 - a.k0) > (b.k1 - b.k0); };
    for (int ht = 1; ht <= hmax; ++ht) {
        size_t s1 = jobs.size();
        for (const Node& nd : nodes) {
            if (nd.height != ht) continue;
            for (int c = nd.lo; c < nd.mid; ++c)
                for (int i = nd.mid; i < nd.hi; ++i)   // T'[c][i] = sum_{k=c..mid} Q[c][k] L[i][k]
                    jobs.push_back({c * BM, i * BM, c * BM, nd.mid * BM, c * BM, i * BM, 0, 0});
        }
        std::stable_sort(jobs.begin() + s1, jobs.end(), by_len);
        h->ranges.tri1[ht].off = (int)s1;
        h->ranges.tri1[ht].cnt = (int)(jobs.size() - s1);
        size_t s2 = jobs.size();
        for (const Node& nd : nodes) {
            if (nd.height != ht) continue;
            for (int i = nd.mid; i < nd.hi; ++i)
                for (int c = nd.lo; c < nd.mid; ++c)   // R[i][c] = -sum_{k=mid..i} P[i][k] T'[c][k]
                    jobs.push_back({i * BM, c * BM, nd.mid * BM, (i + 1) * BM, i * BM, c * BM, 0, 0});
        }
        std::stable_sort(jobs.begin() + s2, jobs.end(), by_len);
        h->ranges.tri2[ht].off = (int)s2;
        h->ranges.tri2[ht].cnt = (int)(jobs.size() - s2);
    }
    // K^-1 = Q Q^T (lower tiles), Q = L^-T upper: K^-1[i][j] = sum_{k >= i} Q[i][k] Q[j][k], i >= j
    h->ranges.kinv.off = (int)jobs.size();
    for (int j = 0; j < nb; ++j)
        for (int i = j; i < nb; ++i)
            jobs.push_back({i * BM, j * BM, i * BM, nb * BM, i * BM, j * BM, 0, 0});
    std::stable_sort(jobs.begin() + h->ranges.kinv.off, jobs.end(), by_len);
    h->ranges.kinv.cnt = (int)jobs.size() - h->ranges.kinv.off;
    // gpk_fit_append: only block row b = nb-1 changes.  N1 = b*128 leading rows keep their factor L11 and inverse P11.
    {
        const int b = nb - 1, N1 = b * BM;
        // partial Gram tiles  T_s = L_row[:, s] L_row[:, s]^T  into the free tiles (s, b) of W; summed in fixed order
        h->ranges.app_syrk.off = (int)jobs.size();
        for (int sblk = 0; sblk < b; ++sblk)
            jobs.push_back({N1, N1, sblk * BM, (sblk + 1) * BM, sblk * BM, N1, 0, 0});
        h->ranges.app_syrk.cnt = (int)jobs.size() - h->ranges.app_syrk.off;
        // L_row = K[b, 0:N1] P11^T and T = L_row P11 (= L_row Q11^T in NT form), split-K: 128-row tiles, the contraction
        // cut into chunks of APP_KC columns, partial tile (chunk c, column block j) -> scratch tile W(c, j); summed in
        // fixed order by gpk_append_reduce_kernel
        h->ranges.app_row2.off = (int)jobs.size();
        for (int j = b - 1; j >= 0; --j)
            for (int c = 0, k0 = 0; k0 < (j + 1) * BM; ++c, k0 += APP_KC)
                jobs.push_back({N1, j * BM, k0, std::min(k0 + APP_KC, (j + 1) * BM), c * BM, j * BM, 0, 0});
        h->ranges.app_row2.cnt = (int)jobs.size() - h->ranges.app_row2.off;
        h->ranges.app_t2.off = (int)jobs.size();
        for (int j = 0; j < b; ++j)
            for (int c = 0, k0 = j * BM; k0 < N1; ++c, k0 += APP_KC)
                jobs.push_back({N1, j * BM, k0, std::min(k0 + APP_KC, N1), c * BM, j * BM, 0, 0});
        h->ranges.app_t2.cnt = (int)jobs.size() - h->ranges.app_t2.off;
        // P[b, j] = -P_bb T[:, j]
        h->ranges.app_p.off = (int)jobs.size();
        for (int j = 0; j < b; ++j)
            jobs.push_back({N1, j * BM, N1, nb * BM, N1, j * BM, 0, 0});
        h->ranges.app_p.cnt = (int)jobs.size() - h->ranges.app_p.off;
    }
    if (jobs.empty()) jobs.push_back({0, 0, 0, 0, 0, 0, 0, 0});
    int rc = ensure(h, h->jobs, jobs.size() * sizeof(GemmJob));
    if (rc) return rc;
    CK(cudaMemcpyAsync(h->jobs.p, jobs.data(), jobs.size() * sizeof(GemmJob), cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->ranges.nb = nb;
    return GPK_OK;
}

int rebuild_maps(gpk_handle* h) {
    const long NP = h->NP;
    int rc;
    if ((rc = make_map(h, &h->mapK, h->Kbuf.p, NP + BM, NP, NP))) return rc;
    if ((rc = make_map(h, &h->mapK32, h->Kbuf.p, NP + BM, NP, NP, 32))) return rc;
    if ((rc = make_map(h, &h->mapP, h->P.p, NP, NP, NP))) return rc;
    if ((rc = make_map(h, &h->mapQ, h->Q.p, NP, NP, NP))) return rc;
    if ((rc = make_map(h, &h->mapW, h->W.p, NP, NP, NP))) return rc;
    h->mapKs_rows = 0;
    h->mapKs2_rows = 0;
    h->mapVt_rows = 0;
    h->maps_ok = true;
    return GPK_OK;
}

// scratch for scoring `rows` (multiple of 128) candidates at once
int ensure_score_scratch(gpk_handle* h, long rows) {
    const long NP = h->NP;
    bool grew = false;
    int rc;
    if ((rc = ensure(h, h->Kstar, (size_t)rows * NP * 8, &grew))) return rc;
    if (grew || h->mapKs_rows != rows) {
        if ((rc = make_map(h, &h->mapKs, h->Kstar.p, rows, NP, NP))) return rc;
        h->mapKs_rows = rows;
    }
    if (h->overlap) {
        if ((rc = ensure(h, h->Kstar2, (size_t)rows * NP * 8, &grew))) return rc;
        if (grew || h->mapKs2_rows != rows) {
            if ((rc = make_map(h, &h->mapKs2, h->Kstar2.p, rows, NP, NP))) return rc;
            h->mapKs2_rows = rows;
        }
    }
    if ((rc = ensure(h, h->part_mu, (size_t)h->nb * rows * 8))) return rc;
    if ((rc = ensure(h, h->part_ssq, (size_t)h->nb * rows * 8))) return rc;
    if ((rc = ensure(h, h->block_best, (size_t)(rows / 256 + 1) * sizeof(BestPair)))) return rc;
    if ((rc = ensure(h, h->best, sizeof(BestPair)))) return rc;
    if ((rc = ensure(h, h->nneg, 8))) return rc;
    return GPK_OK;
}

__global__ void gpk_fit_reduce_kernel(const double* __restrict__ z, int n, const double* __restrict__ logdet_part,
                                      int nb, double* __restrict__ out2) {
    // single block, fixed summation order: out2[0] = z^T z, out2[1] = 2 * sum log diag
    __shared__ double sh[256];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) s = fma(z[i], z[i], s);
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        out2[0] = sh[0];
        double l = 0.0;
        for (int k = 0; k < nb; ++k) l += logdet_part[k];
        out2[1] = 2.0 * l;
    }
}

// mu_c = sum_k M[c][k] * z[k] over k in [k_lo(c), NP): one warp per row (tri: k >= c)
__global__ void gpk_rowdot_kernel(const double* __restrict__ M, long ld, long rows, int NP, int tri,
                                  const double* __restrict__ z, double* __restrict__ out) {
    long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= rows) return;
    double s = 0.0;
    int kstart = tri ? (int)(row & ~31L) : 0;
    for (int k = kstart + lane; k < NP; k += 32)
        if (!tri || k >= row) s = fma(M[row * ld + k], z[k], s);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) out[row] = s;
}

__global__ void gpk_mu_finish_kernel(double* __restrict__ mu, long m, double mean, int norm_out, double y_mean,
                                     double y_std) {
    long c = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= m) return;
    double v = mu[c] + mean;
    if (norm_out) v = v * y_std + y_mean;
    mu[c] = v;
}

// gpk_fit_append helpers -------------------------------------------------------------------
// diagonal of the rows [i0, NP): += diag_add for training rows, unit diagonal on padding rows
__global__ void gpk_kfix_rows_kernel(double* __restrict__ K, long ld, int n, int NP, double diag_add, int i0) {
    int i = i0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= NP) return;
    K[(long)i * ld + i] = (i < n) ? K[(long)i * ld + i] + diag_add : 1.0;
}

// dst[:, j-block] = sum_c W(c, j) over the nc(j) partial tiles of column block j (c ascending: deterministic);
// mode 0: nc = ceil((j + 1) * 128 / APP_KC) (L_row), mode 1: nc = ceil((b - j) * 128 / APP_KC) (L_row P11).
// dstT (may be NULL) receives the transpose: dstT[j*128 + c][r].  grid = (b, 64), 256 threads, one element each.
__global__ void gpk_append_reduce_kernel(const double* __restrict__ W, long ld, int b, int mode, double* __restrict__ dst,
                                         long ldd, double* __restrict__ dstT, long lddT, int tcol0) {
    const int j = blockIdx.x;
    const int e = blockIdx.y * 256 + threadIdx.x;              // 0 .. 128*128-1
    const int r = e >> 7, c = e & 127;
    const int len = mode == 0 ? (j + 1) * 128 : (b - j) * 128;
    const int nc = (len + APP_KC - 1) / APP_KC;
    double acc = 0.0;
    for (int q = 0; q < nc; ++q) acc += W[(long)(q * 128 + r) * ld + j * 128 + c];
    dst[(long)r * ldd + j * 128 + c] = acc;
    if (dstT != nullptr) dstT[(long)(j * 128 + c) * lddT + tcol0 + r] = acc;
}

// K[b,b] -= sum_s T_s with T_s = W tile (s, b), s ascending (deterministic); one thread per element
__global__ void gpk_append_schur_kernel(double* __restrict__ K, const double* __restrict__ W, long ld, int N1, int nparts) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;         // 0 .. 128*128-1
    const int i = e >> 7, c = e & 127;
    double acc = 0.0;
    for (int sblk = 0; sblk < nparts; ++sblk) acc += W[(long)(sblk * 128 + i) * ld + N1 + c];
    K[(long)(N1 + i) * ld + N1 + c] -= acc;
}

__global__ void gpk_resid_kernel(const double* __restrict__ y, double mean, int n, int NP, double* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < NP) out[i] = (i < n) ? y[i] - mean : 0.0;
}

// What the refusals between model kinds say about each kind, indexed by ModelKind
struct ModelInfo {
    const char* holds;          // "the handle holds <holds>"
    const char* set_data;       // the entry point that gives a handle this kind
    const char* use_for;        // "use a new handle for <use_for>"
    const char* not_fitted;     // the scoring entry points' refusal before the model is trained
    const char* gp_refusal;     // the Gaussian-process entry points' refusal
};
#define SURROGATE(what, set_data, use_for, not_fitted)                                                               \
    {what " (" set_data ")", set_data, use_for, not_fitted,                                                         \
     "the handle holds " what " (" set_data "); this entry point serves Gaussian-process handles only"}
const ModelInfo MODELS[] = {
    {"a Gaussian-process model", nullptr, nullptr, nullptr, nullptr},
    SURROGATE("a Bayesian linear regression model", "gpk_blr_set_data", "Bayesian linear regression",
              "model is not fitted (gpk_blr_fit)"),
    SURROGATE("a random forest", "gpk_rf_set_data", "a random forest", "model is not fitted (gpk_rf_fit)"),
    SURROGATE("a Bayesian neural network", "gpk_bnn_set_data", "a Bayesian neural network",
              "model is not trained (gpk_bnn_train)"),
    SURROGATE("a DNGO model", "gpk_dngo_set_data", "DNGO", "model is not fitted (gpk_dngo_fit)"),
};
#undef SURROGATE

// the refusal of a Gaussian-process entry point for the handle's model kind, or nullptr for a Gaussian-process handle
const char* gp_refusal(const gpk_handle* h) { return MODELS[h->model].gp_refusal; }

// the refusal of the `kind` entry point `who` on a handle that holds another model
int refuse_model(gpk_handle* h, ModelKind kind, const char* who) {
    BAD("%s: the handle holds %s; use a new handle for %s", who, MODELS[h->model].holds, MODELS[kind].use_for);
}

// gpk_*_set_data's check before the handle takes the surrogate `kind`: it holds no other surrogate, and no GP data or
// kernel
int claim_model(gpk_handle* h, ModelKind kind, const char* who) {
    if (h->model == MODEL_GP ? h->has_data || h->has_spec : h->model != kind) return refuse_model(h, kind, who);
    return GPK_OK;
}

// the check of every other `kind` entry point: the handle holds that surrogate; then its device is made current
int model_ready(gpk_handle* h, ModelKind kind, const char* who) {
    if (!h) return GPK_BAD_ARG;
    if (h->model != MODEL_GP && h->model != kind) return refuse_model(h, kind, who);
    if (h->model != kind) BAD("%s: %s has not been called", who, MODELS[kind].set_data);
    CK(cudaSetDevice(h->device));
    return GPK_OK;
}

int require(gpk_handle* h, bool data, bool spec, bool fitted) {
    if (!h) return GPK_BAD_ARG;
    if (gp_refusal(h)) { set_err(h, "%s", gp_refusal(h)); return GPK_BAD_ARG; }
    if (data && !h->has_data) { set_err(h, "gpk_set_data has not been called"); return GPK_BAD_ARG; }
    if (spec && !h->has_spec) { set_err(h, "gpk_set_kernel has not been called"); return GPK_BAD_ARG; }
    if (fitted && !h->fitted) { set_err(h, "model is not fitted (gpk_fit)"); return GPK_NOT_FITTED; }
    return GPK_OK;
}

// the preconditions of the entry points that score any model kind: a fitted GP, or a trained surrogate
int require_model(gpk_handle* h) {
    if (!h || h->model == MODEL_GP) return require(h, true, true, true);
    const bool trained = h->model == MODEL_BLR ? h->blr.fitted : h->model == MODEL_RF ? h->rf.fitted
                       : h->model == MODEL_BNN ? h->bnn.S >= 1 : h->dngo.fitted;
    if (!trained) { set_err(h, "%s", MODELS[h->model].not_fitted); return GPK_NOT_FITTED; }
    return GPK_OK;
}

// L^-1 by recursive block inversion (P lower, Q = P^T upper), after a successful fit.
int build_linv(gpk_handle* h) {
    if (h->linv_ready) return GPK_OK;
    CK(cudaEventRecord(h->timing.ev[4], h->stream));
    const long NP = h->NP;
    const int hmax = (int)h->ranges.tri1.size() - 1;
    for (int ht = 1; ht <= hmax; ++ht) {
        GemmArgs a;
        memset(&a, 0, sizeof(a));
        a.A = ptr<double>(h->Q); a.lda = NP;
        a.B = ptr<double>(h->Kbuf); a.ldb = NP;
        a.C = ptr<double>(h->W); a.ldc = NP;
        a.alpha = 1.0; a.beta = 0;
        a.jobs = ptr<GemmJob>(h->jobs) + h->ranges.tri1[ht].off;
        a.job_mode = JOBS_TABLE;
        int rc = launch_gemm<EPI_STORE>(h, h->mapQ, h->mapK, a, h->ranges.tri1[ht].cnt);
        if (rc) return rc;
        GemmArgs b;
        memset(&b, 0, sizeof(b));
        b.A = ptr<double>(h->P); b.lda = NP;
        b.B = ptr<double>(h->W); b.ldb = NP;
        b.C = ptr<double>(h->P); b.ldc = NP;
        b.Ct = ptr<double>(h->Q); b.ldct = NP;
        b.alpha = -1.0; b.beta = 0;
        b.jobs = ptr<GemmJob>(h->jobs) + h->ranges.tri2[ht].off;
        b.job_mode = JOBS_TABLE;
        rc = launch_gemm<EPI_STORE>(h, h->mapP, h->mapW, b, h->ranges.tri2[ht].cnt);
        if (rc) return rc;
    }
    CK(cudaEventRecord(h->timing.ev[5], h->stream));
    h->linv_ready = true;
    h->linv_serial += 1;
    h->alpha_ready = false;
    return GPK_OK;
}

// alpha = L^-T z (Q = L^-T is upper triangular), once per factorisation: the posterior mean is mu - mean = K* alpha.
// Needs L^-1 (build_linv).
int ensure_alpha(gpk_handle* h) {
    if (h->alpha_ready) return GPK_OK;
    const long NP = h->NP;
    int rc;
    if ((rc = ensure(h, h->alpha, (size_t)NP * 8))) return rc;
    gpk_rowdot_kernel<<<(unsigned)((NP + 7) / 8), 256, 0, h->stream>>>(ptr<double>(h->Q), NP, NP, (int)NP, 1,
                                                                       ptr<double>(h->Kbuf) + NP * NP, ptr<double>(h->alpha));
    CKL();
    h->alpha_ready = true;
    return GPK_OK;
}

// int8 tensor map over S stacked slice matrices [S * rows][cols] (int8, K contiguous): box = 64 bytes x box_rows, 64B swizzle
int make_oz_map(gpk_handle* h, CUtensorMap* map, void* base, long rows_total, long cols, int box_rows, int box_bytes = OZ_KB) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) { set_err(h, "cuTensorMapEncodeTiled entry point not available"); return GPK_CUDA_ERROR; }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows_total};
    cuuint64_t strides[1] = {(cuuint64_t)cols};
    cuuint32_t box[2] = {(cuuint32_t)box_bytes, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    box_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_err(h, "cuTensorMapEncodeTiled (int8 slices) failed with CUresult %d", (int)r); return GPK_CUDA_ERROR; }
    return GPK_OK;
}

// Slices of L^-1 for the int8 contraction, once per factorisation.  Returns true in *usable when the factor is
// conditioned well enough for S = 8 slices (row exponents <= OZ_MAX_EXP) and the sizes fit the int32 accumulators.
// A kernel with a factor is never eligible: the digit split of K* assumes 0 < k <= amp.
int prepare_ozaki(gpk_handle* h, bool* usable) {
    *usable = false;
    if (!h->oz.enabled || h->NP > 16384 || h->spec.factor.kind != GPK_FACTOR_NONE)
        return GPK_OK;
    const long NP = h->NP;
    if (h->oz.linv_serial != h->linv_serial) {
        int rc;
        if ((rc = ensure(h, h->oz.Pq, (size_t)OZ_S * NP * NP))) return rc;
        if ((rc = ensure(h, h->oz.eP, (size_t)NP * 4))) return rc;
        if ((rc = ensure(h, h->oz.emax, 4))) return rc;
        const int lowest = -100000;
        CK(cudaMemcpyAsync(h->oz.emax.p, &lowest, 4, cudaMemcpyHostToDevice, h->stream));
        gpk_oz_rowexp_kernel<<<(unsigned)NP, 256, 0, h->stream>>>(ptr<double>(h->P), NP, (int)NP, ptr<int>(h->oz.eP), ptr<int>(h->oz.emax));
        CKL();
        gpk_oz_split_kernel<<<(unsigned)((NP * NP + 255) / 256), 256, 0, h->stream>>>(ptr<double>(h->P), NP, NP, ptr<int>(h->oz.eP), 0,
                                                                                   ptr<int8_t>(h->oz.Pq), NP * NP);
        CKL();
        // the mean goes through fp64, mu - mean = K* alpha
        if ((rc = ensure_alpha(h))) return rc;
        CK(cudaMemcpyAsync(&h->oz.emax_host, h->oz.emax.p, 4, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        h->oz.map_cs = 0;
        h->oz.linv_serial = h->linv_serial;
    }
    // each CTA of a cluster loads 128 / CS rows of every L^-1 slice; 64-row (CS = 2) and 32-row (CS = 4) offsets are
    // multiples of the 512-byte SWIZZLE_64B atom, so the multicast pieces form the same swizzled 128-row tile
    if (h->oz.map_cs != h->oz.cluster) {
        int rc;
        if ((rc = make_oz_map(h, &h->oz.mapP, h->oz.Pq.p, (long)OZ_S * NP, NP, OZ_TM / h->oz.cluster))) return rc;
        h->oz.map_cs = h->oz.cluster;
    }
    *usable = h->oz.emax_host <= OZ_MAX_EXP;
    return GPK_OK;
}

// Candidates per scoring pass.  Unless the caller fixed it ("chunk" option) the K* buffer is kept at about 512 MB:
// 16384 candidates at N = 4096, 65536 at N <= 1024 (fewer, longer launches where a candidate costs only N^2 = 1 MFLOP).
long chunk_rows(const gpk_handle* h) {
    if (h->chunk_user) return h->chunk;
    long c = ((1L << 26) / std::max(h->NP, 128)) / BM * BM;
    return std::min<long>(65536, std::max<long>(4096, c));
}

// Host batches are fed to score_dev chunk by chunk: ready(lo, hi, st) makes sure the candidate rows [lo, hi) are on
// their way to the device buffer and lets stream `st` wait for them (gpk_acq: H2D of chunk i+1, and for pageable memory
// the host staging copy, overlap the scoring of chunk i inside ONE scoring pass with full K* look-ahead).
struct Feeder {
    virtual int ready(long lo, long hi, cudaStream_t st) = 0;
    virtual ~Feeder() {}
};

int surrogate_score(gpk_handle* h, const double* dX, long m, int kind, double eta, double par, double* d_out,
                    double* d_mu, double* d_var, BestPair* d_best, unsigned long long* d_nneg, long index_offset,
                    bool reset, long global_base, Feeder* feeder);

// the outputs of a scoring launch whose first candidate is row `offset` of the caller's batch (score_dev's arguments)
ScoreOut score_out(gpk_handle* h, int kind, double eta, double par, double* d_out, double* d_mu, double* d_var,
                   unsigned long long* d_nneg, long offset, long global_base) {
    ScoreOut o;
    o.base = global_base + offset;
    o.acq_kind = kind; o.eta = eta; o.par = par;
    o.out_mu = d_mu ? d_mu + offset : nullptr;
    o.out_var = d_var ? d_var + offset : nullptr;
    o.out_acq = d_out ? d_out + offset : nullptr;
    o.block_best = ptr<BestPair>(h->block_best);
    o.n_negative = d_nneg;
    return o;
}

// Score m candidates resident on the device.  All output pointers are device pointers or NULL.
// index_offset: position of dX[0] in the caller's batch (offset into the output arrays and into the arg-max index);
// global_base: added to the arg-max index only (first index of this rank's shard in a sharded batch); reset: start a
// new running arg-max / negative-EI count (false when a host batch is fed in several pieces)
int score_dev(gpk_handle* h, const double* dX, long m, int kind, double eta, double par, double* d_out,
              double* d_mu, double* d_var, BestPair* d_best, unsigned long long* d_nneg,
              long index_offset = 0, bool reset = true, long global_base = 0, Feeder* feeder = nullptr) {
    if (h->model != MODEL_GP)
        return surrogate_score(h, dX, m, kind, eta, par, d_out, d_mu, d_var, d_best, d_nneg, index_offset, reset,
                               global_base, feeder);
    int rc = build_linv(h);
    if (rc) return rc;
    const long NP = h->NP;
    const long cap = std::min<long>(chunk_rows(h), round_up(std::max<long>(m, 1), BM));
    if ((rc = ensure_score_scratch(h, cap))) return rc;
    // int8 path only for batches that amortise slicing L^-1 (once per fit)
    bool use_oz = false;
    if (m >= 2048 && (rc = prepare_ozaki(h, &use_oz))) return rc;
    int oz_eK = 0;
    if (use_oz) {
        // slices of K* per chunk buffer: [S][cap][NP] int8; one exponent for the whole matrix (0 < k <= amp)
        // (the tensor maps are re-encoded per call: a few microseconds, and they depend on the buffer, cap and NP)
        if ((rc = ensure(h, h->oz.Kq, (size_t)OZ_S * cap * NP))) return rc;
        if (h->overlap && (rc = ensure(h, h->oz.Kq2, (size_t)OZ_S * cap * NP))) return rc;
        if ((rc = make_oz_map(h, &h->oz.mapK, h->oz.Kq.p, (long)OZ_S * cap, NP, OZ_TN))) return rc;
        if (h->overlap && (rc = make_oz_map(h, &h->oz.mapK2, h->oz.Kq2.p, (long)OZ_S * cap, NP, OZ_TN))) return rc;
        if (h->overlap && (rc = ensure(h, h->oz.pmu2, (size_t)h->nb * cap * 8))) return rc;
        oz_eK = oz_exponent(h->spec.amp);
    }
    if (d_best == nullptr) d_best = ptr<BestPair>(h->best);
    if (d_nneg == nullptr) d_nneg = ptr<unsigned long long>(h->nneg);
    if (reset) {
        CK(cudaMemsetAsync(d_best, 0xFF, sizeof(BestPair), h->stream));
        CK(cudaMemsetAsync(d_nneg, 0, 8, h->stream));
    }
    CK(cudaEventRecord(h->timing.ev[6], h->stream));
    const int nchunks = (int)((m + cap - 1) / cap);
    // With more than one chunk, K* of chunk i+1 is built on the low-priority side stream (8 candidates
    // per thread, ~60 registers: its CTAs fit next to the resident GEMM CTAs and use the FP64 ALUs while
    // the GEMM keeps the DMMA pipe busy); two K* buffers alternate.
    const bool pipelined = h->overlap && nchunks > 1;
    if (pipelined && ((rc = grow_events(h, h->ev_cov, nchunks, cudaEventDisableTiming)) ||
                      (rc = grow_events(h, h->ev_gemm, nchunks, cudaEventDisableTiming))))
        return rc;
    if ((rc = grow_events(h, h->timing.ev_g0, nchunks, cudaEventDefault)) ||
        (rc = grow_events(h, h->timing.ev_g1, nchunks, cudaEventDefault)))
        return rc;
    h->timing.last_nchunks = nchunks;
    auto launch_cov = [&](int ci, cudaStream_t st, bool small) -> int {
        const long base = (long)ci * cap;
        const long mc = std::min(cap, m - base);
        const long mcp = round_up(mc, BM);
        const bool second = pipelined && (ci & 1);
        if (feeder) {
            int frc = feeder->ready(base, base + mc, st);
            if (frc) return frc;
        }
        const double* lo = h->has_bounds ? ptr<double>(h->lower) : nullptr;
        const double* up = h->has_bounds ? ptr<double>(h->upper) : nullptr;
        if (!use_oz)
            return launch_cov_tiles(h, st, ptr<double>(h->Xts), NP, h->n, dX + base * h->d, h->d, mc, mcp, lo, up,
                                    second ? ptr<double>(h->Kstar2) : ptr<double>(h->Kstar), NP, 0, small,
                                    ptr<double>(h->Xrow), nullptr, nullptr);
        // K* never reaches HBM in fp64: digits + this tile's share of the mean straight out of the builder
        CUtensorMap map;
        int mrc = make_cov_map(h, &map, h->Xts.p, h->spec.n_terms, NP);
        if (mrc) return mrc;
        int8_t* qdst = second ? ptr<int8_t>(h->oz.Kq2) : ptr<int8_t>(h->oz.Kq);
        double* pmu = second ? ptr<double>(h->oz.pmu2) : ptr<double>(h->part_mu);
        const int gx = (int)(NP / 128);
        if (small)
            gpk_cov_oz_kernel<4><<<(unsigned)(gx * (mcp / 16)), 256, cov_oz_smem_bytes(h->spec.n_terms, 4), st>>>(
                map, h->spec, h->n, dX + base * h->d, h->d, mc, lo, up, ptr<double>(h->alpha), oz_eK, qdst, NP, cap * NP, pmu, cap, gx,
                nullptr);
        else
            gpk_cov_oz_kernel<8><<<(unsigned)(gx * (mcp / 32)), 256, cov_oz_smem_bytes(h->spec.n_terms, 8), st>>>(
                map, h->spec, h->n, dX + base * h->d, h->d, mc, lo, up, ptr<double>(h->alpha), oz_eK, qdst, NP, cap * NP, pmu, cap, gx,
                nullptr);
        CKL();
        return GPK_OK;
    };
    if (pipelined) {
        CK(cudaEventRecord(h->ev_order, h->stream));          // side stream starts after all prior work
        CK(cudaStreamWaitEvent(h->side_stream, h->ev_order, 0));
        if ((rc = launch_cov(0, h->side_stream, false))) return rc;
        CK(cudaEventRecord(h->ev_cov[0], h->side_stream));
    }
    for (int ci = 0; ci < nchunks; ++ci) {
        const long base = (long)ci * cap;
        const long mc = std::min(cap, m - base);
        const long mcp = round_up(mc, BM);
        const bool last = ci == nchunks - 1;
        if (last) CK(cudaEventRecord(h->timing.ev[8], h->stream));
        if (pipelined) {
            CK(cudaStreamWaitEvent(h->stream, h->ev_cov[ci], 0));
            if (ci + 1 < nchunks) {
                if (ci >= 1) CK(cudaStreamWaitEvent(h->side_stream, h->ev_gemm[ci - 1], 0));   // buffer (ci+1)&1 is free
                if ((rc = launch_cov(ci + 1, h->side_stream, true))) return rc;
                CK(cudaEventRecord(h->ev_cov[ci + 1], h->side_stream));
            }
        } else {
            if ((rc = launch_cov(ci, h->stream, false))) return rc;
        }
        const bool second = pipelined && (ci & 1);
        GemmArgs a;
        memset(&a, 0, sizeof(a));
        a.A = ptr<double>(h->P); a.lda = NP;
        a.B = second ? ptr<double>(h->Kstar2) : ptr<double>(h->Kstar); a.ldb = NP;
        a.alpha = 1.0;
        a.job_mode = JOBS_VARIANCE;
        a.nb = h->nb; a.mcb = (int)(mcp / BN);
        a.z = ptr<double>(h->Kbuf) + NP * NP;
        a.part_mu = ptr<double>(h->part_mu);
        a.part_ssq = ptr<double>(h->part_ssq);
        a.ldpart = cap;
        if (last) CK(cudaEventRecord(h->timing.ev[10], h->stream));
        CK(cudaEventRecord(h->timing.ev_g0[ci], h->stream));
        if (use_oz) {
            if ((rc = launch_oz_contraction(h, h->oz.mapP, second ? h->oz.mapK2 : h->oz.mapK, h->nb, mcp, NP, cap,
                                            ptr<int>(h->oz.eP), oz_eK, a.part_ssq, a.ldpart)))
                return rc;
            h->oz.launches += 1;
        } else if ((rc = launch_gemm<EPI_COLREDUCE>(h, h->mapP, second ? h->mapKs2 : h->mapKs, a, h->nb * a.mcb))) return rc;
        CK(cudaEventRecord(h->timing.ev_g1[ci], h->stream));
        if (last) CK(cudaEventRecord(h->timing.ev[11], h->stream));
        // fp64 path: this parity's K* buffer is free once the contraction has read it
        if (pipelined && !use_oz) CK(cudaEventRecord(h->ev_gemm[ci], h->stream));
        h->timing.launches_var += 1;
        FinishArgs f;
        memset(&f, 0, sizeof(f));
        f.part_mu = ptr<double>(h->part_mu); f.part_ssq = ptr<double>(h->part_ssq);
        f.ldpart = cap; f.nparts = h->nb; f.m = mc;
        f.kss = h->spec.amp; f.mean = h->mean;
        f.factor = h->spec.factor;
        f.cand = dX + base * h->d; f.cand_dc = h->d;
        f.lo = h->has_bounds ? ptr<double>(h->lower) : nullptr;
        f.up = h->has_bounds ? ptr<double>(h->upper) : nullptr;
        f.norm_out = h->norm_out; f.y_mean = h->y_mean; f.y_std = h->y_std;
        f.o = score_out(h, kind, eta, par, d_out, d_mu, d_var, d_nneg, index_offset + base, global_base);
        if (use_oz && second) f.part_mu = ptr<double>(h->oz.pmu2);
        const int fb = (int)((mc + 255) / 256);
        gpk_finish_kernel<<<fb, 256, 0, h->stream>>>(f);
        CKL();
        if (kind != GPK_ACQ_NONE) {
            gpk_argmax_final_kernel<<<1, 256, 0, h->stream>>>(ptr<BestPair>(h->block_best), fb, d_best);
            CKL();
        }
        // int8 path: the builder also writes this parity's mean partials, which the finish kernel above still reads
        if (pipelined && use_oz) CK(cudaEventRecord(h->ev_gemm[ci], h->stream));
        if (last) CK(cudaEventRecord(h->timing.ev[12], h->stream));
    }
    CK(cudaEventRecord(h->timing.ev[7], h->stream));
    h->timing.score_timed = true;
    return GPK_OK;
}

// layout of h->es.state (doubles): logP (nb), lmb (nb), dMu (nb x nb), dSig (nb x T), Hs (nb x T), W (np), lower (d),
// upper (d), scaled zb (nb x d)
struct EsLayout {
    size_t logP, lmb, dMu, dSig, Hs, W, lo, up, zb, total;
    EsLayout(int nb, int np_, int d) {
        const size_t T = (size_t)nb * (nb + 1) / 2;
        logP = 0; lmb = logP + nb; dMu = lmb + nb; dSig = dMu + (size_t)nb * nb; Hs = dSig + nb * T; W = Hs + nb * T;
        lo = W + np_; up = lo + d; zb = up + d; total = zb + (size_t)nb * d;
    }
};

// layout of h->mc.state (doubles): Mb (nb), Vb (nb x nb), W (np), lmb (nb), scaled zb (nb x d), F (nb x nf)
struct McLayout {
    size_t Mb, Vb, W, lmb, zb, F, total;
    McLayout(int nb, int np_, int d, int nf) {
        Mb = 0; Vb = Mb + nb; W = Vb + (size_t)nb * nb; lmb = W + np_; zb = lmb + nb; F = zb + (size_t)nb * d;
        total = F + (size_t)nb * nf;
    }
};

enum { ES_KIND_NONE = 0, ES_KIND_EP = 1, ES_KIND_MC = 2 };

// Posterior mean alone of m candidates resident on the device (d_mu: m doubles), asynchronous on the handle's stream.
// The int8 path's covariance builder with its digit stores compiled out writes each 128-column tile's share of K* alpha,
// and gpk_mu_parts_finish_kernel sums the shares in tile order: no K* in HBM, no L^-1 slices, no contraction.  Every
// candidate is independent, so the values depend neither on "chunk" nor on how a batch is split, and equal the mean of
// score_dev's int8 path bit for bit.
int predict_mean_dev(gpk_handle* h, const double* dX, long m, double* d_mu) {
    if (!h->mean_only)                      // option "meanonly" = 0: the mean of the full scoring pass (comparisons)
        return score_dev(h, dX, m, GPK_ACQ_NONE, 0.0, 0.0, nullptr, d_mu, nullptr, nullptr, nullptr);
    int rc;
    if ((rc = build_linv(h))) return rc;
    if ((rc = ensure_alpha(h))) return rc;
    const long NP = h->NP;
    const long cap = std::min<long>(chunk_rows(h), round_up(m, BM));
    if ((rc = ensure(h, h->part_mu, (size_t)h->nb * cap * 8))) return rc;
    CUtensorMap map;
    if ((rc = make_cov_map(h, &map, h->Xts.p, h->spec.n_terms, NP))) return rc;
    const double* lo = h->has_bounds ? ptr<double>(h->lower) : nullptr;
    const double* up = h->has_bounds ? ptr<double>(h->upper) : nullptr;
    const int gx = (int)(NP / 128);
    for (long base = 0; base < m; base += cap) {
        const long mc = std::min(cap, m - base);
        const long mcp = round_up(mc, BM);
        gpk_cov_oz_kernel<8, false><<<(unsigned)(gx * (mcp / 32)), 256, cov_oz_smem_bytes(h->spec.n_terms, 8), h->stream>>>(
            map, h->spec, h->n, dX + base * h->d, h->d, mc, lo, up, ptr<double>(h->alpha), 0, nullptr, NP, 0,
            ptr<double>(h->part_mu), cap, gx, ptr<double>(h->Xrow));
        CKL();
        gpk_mu_parts_finish_kernel<<<(unsigned)((mc + 255) / 256), 256, 0, h->stream>>>(
            ptr<double>(h->part_mu), cap, h->nb, mc, h->mean, h->norm_out, h->y_mean, h->y_std, d_mu + base);
        CKL();
    }
    return GPK_OK;
}

const long ES_CH = 16384;                   // candidates per pass of es_dh_dev; every candidate is independent of the others

// es_dh_dev's scratch (variance and sigma of one pass), sized for the handle's current gpk_es_update
int es_reserve(gpk_handle* h) {
    return ensure(h, h->es.work, (size_t)ES_CH * (h->es.nb + 1) * 8);
}

// One pass of es_dh_dev's first half: the predictive variance of rows <= ES_CH candidates X (the scoring pass) into
// es.work's var (rows) and their clipped covariance to zb into its sig (rows x nb), the two buffers gpk_es_dh_kernel
// reads.  Asynchronous on the handle's stream; needs es_reserve and a current gpk_es_update.
int es_moments_pass(gpk_handle* h, const double* X, long rows) {
    const int nb = h->es.nb, d = h->d;
    const double* zs = h->es.kind == ES_KIND_MC ? ptr<double>(h->mc.state) + McLayout(nb, h->es.np, d, h->mc.nf).zb
                                                : ptr<double>(h->es.state) + EsLayout(nb, h->es.np, d).zb;
    double* var = ptr<double>(h->es.work);
    double* sig = var + ES_CH;
    const double* lo = h->has_bounds ? ptr<double>(h->lower) : nullptr;
    const double* up = h->has_bounds ? ptr<double>(h->upper) : nullptr;
    const double out_scale = h->norm_out ? h->y_std * h->y_std : 1.0;
    int rc;
    if ((rc = score_dev(h, X, rows, GPK_ACQ_NONE, 0.0, 0.0, nullptr, nullptr, var, nullptr, nullptr))) return rc;
    gpk_es_sigma_kernel<<<(unsigned)rows, GPK_ES_THREADS, 0, h->stream>>>(h->spec, X, rows, d, lo, up,
                                                                          ptr<double>(h->Xrow), h->n,
                                                                          ptr<double>(h->es.U), zs, nb,
                                                                          out_scale, sig);
    CKL();
    return GPK_OK;
}

// Entropy change of m candidates on the device (InformationGain.compute): Xm are the inputs the model's scoring pass and
// covariance to zb take, Xb the ones the bounds test of gpk_es_update's [lower, upper] sees (the same array unless the
// model's inputs were transformed).  Asynchronous on the handle's stream; needs a current gpk_es_update.
int es_dh_dev(gpk_handle* h, const double* Xm, const double* Xb, long m, double* d_out) {
    const int nb = h->es.nb, d = h->d;
    EsLayout L(nb, h->es.np, d);
    const double* st = ptr<double>(h->es.state);
    const long CH = ES_CH;
    int rc;
    if ((rc = es_reserve(h))) return rc;
    const double* var = ptr<double>(h->es.work);
    const double* sig = var + CH;
    for (long c0 = 0; c0 < m; c0 += CH) {
        const long rows = std::min(CH, m - c0);
        if ((rc = es_moments_pass(h, Xm + c0 * d, rows))) return rc;
        gpk_es_dh_kernel<<<(unsigned)rows, GPK_ES_THREADS, 0, h->stream>>>(
            Xb + c0 * d, rows, d, st + L.lo, st + L.up, var, sig, nb, h->es.np, h->es.sn2, h->es.H, st + L.logP,
            st + L.lmb, st + L.dMu, st + L.dSig, st + L.Hs, st + L.W, d_out + c0);
        CKL();
    }
    return GPK_OK;
}

// the checks gpk_es_compute makes before it runs: a current gpk_es_update on an unchanged model.  kind: the update the
// caller needs (ES_KIND_EP: gpk_es_update, ES_KIND_MC: gpk_esmc_update, ES_KIND_NONE: either).
int es_ready(gpk_handle* h, gpk_handle* report, const char* who, int kind = ES_KIND_EP) {
    gpk_handle* r = report ? report : h;
    const char* upd = kind == ES_KIND_MC ? "gpk_esmc_update" : "gpk_es_update";
    if (gp_refusal(h)) { set_err(r, "%s: %s", who, gp_refusal(h)); return GPK_BAD_ARG; }
    if (h->es.linv_serial < 0) { set_err(r, "%s: call %s first", who, upd); return GPK_BAD_ARG; }
    if (!h->linv_ready || h->es.linv_serial != h->linv_serial) {
        set_err(r, "%s: the model changed since %s", who, upd);
        return GPK_BAD_ARG;
    }
    if (kind != ES_KIND_NONE && h->es.kind != kind) {
        set_err(r, "%s: the current update is %s, not %s", who,
                h->es.kind == ES_KIND_MC ? "gpk_esmc_update" : "gpk_es_update", upd);
        return GPK_BAD_ARG;
    }
    return GPK_OK;
}

// The zb half of an entropy-search update, shared by gpk_es_update and gpk_esmc_update: the raw representer points zb
// (nb x d, host) scaled like the model's inputs into zs (device), and U = L^-T (L^-1 K(X, zb)) in fp64 from the handle's
// L^-1 into h->es.U.  Asynchronous on the handle's stream.
int es_build_u(gpk_handle* h, const double* zb, int nb, double* zs) {
    const int d = h->d, n = h->n, NP = h->NP;
    const size_t D = (size_t)nb;
    cudaStream_t s = h->stream;
    int rc;
    if ((rc = ensure(h, h->tmp1, D * d * 8))) return rc;
    CK(cudaMemcpyAsync(h->tmp1.p, zb, D * d * 8, cudaMemcpyHostToDevice, s));
    const double* lo = h->has_bounds ? ptr<double>(h->lower) : nullptr;
    const double* up = h->has_bounds ? ptr<double>(h->upper) : nullptr;
    gpk_es_scale_kernel<<<(unsigned)((D * d + 255) / 256), 256, 0, s>>>(ptr<double>(h->tmp1), nb, d, lo, up, zs);
    CKL();
    if (!h->linv_ready && (rc = build_linv(h))) return rc;
    if ((rc = ensure(h, h->es.U, (size_t)NP * D * 8 * 2))) return rc;
    double* U = ptr<double>(h->es.U);
    double* tmp = U + (size_t)NP * D;
    CK(cudaMemsetAsync(tmp, 0, (size_t)NP * D * 8, s));
    gpk_es_kxz_kernel<<<(unsigned)(((long)n * nb + 255) / 256), 256, 0, s>>>(h->spec, ptr<double>(h->Xrow), n, d, zs, nb,
                                                                              tmp);
    CKL();
    gpk_es_trmm_kernel<<<(unsigned)(((long)NP * nb + 255) / 256), 256, 0, s>>>(ptr<double>(h->P), NP, tmp, nb, 0, U);
    CKL();
    gpk_es_trmm_kernel<<<(unsigned)(((long)NP * nb + 255) / 256), 256, 0, s>>>(ptr<double>(h->P), NP, U, nb, 1, tmp);
    CKL();
    CK(cudaMemcpyAsync(U, tmp, (size_t)NP * D * 8, cudaMemcpyDeviceToDevice, s));
    return GPK_OK;
}

// gpk_mc_pmin_kernel's ~100 KB of shared memory, with the carveout that lets two CTAs share an SM
int mc_kernel_attrs(gpk_handle* h) {
    CK(cudaFuncSetAttribute(gpk_mc_pmin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GPK_MC_SMEM));
    CK(cudaFuncSetAttribute(gpk_mc_pmin_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                            cudaSharedmemCarveoutMaxShared));
    return GPK_OK;
}

// the 2 status words of gpk_mc_pmin_kernel on h (device), zeroed on h's stream
int mc_stat_reset(gpk_handle* h) {
    int rc;
    if ((rc = ensure(h, h->mc.stat, 2 * sizeof(int)))) return rc;
    CK(cudaMemsetAsync(h->mc.stat.p, 0, 2 * sizeof(int), h->stream));
    return GPK_OK;
}

// Waits for h's stream and reads the status words at d_stat: GPK_NOT_PD (numpy.linalg.LinAlgError, mc_part.py:40-41)
// when a factorisation failed at every rung of the jitter ladder; the jittered count goes to h->mc.last_jitter.
int mc_stat_check(gpk_handle* h, const int* d_stat, const char* who) {
    int st[2] = {0, 0};
    CK(cudaMemcpyAsync(st, d_stat, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->mc.last_jitter = st[GPK_MC_STAT_JITTER];
    if (st[GPK_MC_STAT_NOT_PD] > 0) {
        set_err(h, "%s: Cholesky decomposition failed. (%d factorisation(s) not positive definite at noise 10000)", who,
                st[GPK_MC_STAT_NOT_PD]);
        return GPK_NOT_PD;
    }
    return GPK_OK;
}

// The sampling-based entropy change of m candidates on the device (InformationGainMC.compute): v and sigma by
// es_moments_pass, then gpk_mc_pmin_kernel, in passes of ES_CH.  The status words go to d_stat (2 ints, device), which
// the caller zeroes and reads.  Asynchronous on the handle's stream; needs a current gpk_esmc_update.
int esmc_dev(gpk_handle* h, const double* X, long m, double* d_out, int* d_stat) {
    const int nb = h->es.nb, d = h->d;
    McLayout L(nb, h->es.np, d, h->mc.nf);
    const double* st = ptr<double>(h->mc.state);
    int rc;
    if ((rc = es_reserve(h))) return rc;
    const double* var = ptr<double>(h->es.work);
    const double* sig = var + ES_CH;
    if ((rc = mc_kernel_attrs(h))) return rc;
    for (long c0 = 0; c0 < m; c0 += ES_CH) {
        const long rows = std::min(ES_CH, m - c0);
        if ((rc = es_moments_pass(h, X + c0 * d, rows))) return rc;
        gpk_mc_pmin_kernel<<<(unsigned)rows, GPK_MC_THREADS, GPK_MC_SMEM, h->stream>>>(
            nullptr, st + L.Mb, st + L.W, h->es.np, st + L.Vb, nb, st + L.F, h->mc.nf, var, sig, h->es.sn2, st + L.lmb,
            h->es.H, d_out + c0, nullptr, nullptr, d_stat);
        CKL();
    }
    return GPK_OK;
}

// the layout of h->blr.data (doubles): Phi (n x F), y (n), G (F x F), b (F)
inline double* blr_phi(gpk_handle* h) { return ptr<double>(h->blr.data); }
inline double* blr_y(gpk_handle* h) { return blr_phi(h) + (size_t)h->n * h->blr.F; }
inline double* blr_G(gpk_handle* h) { return blr_y(h) + h->n; }
inline double* blr_b(gpk_handle* h) { return blr_G(h) + (size_t)h->blr.F * h->blr.F; }

// the layout of h->blr.post (doubles) for k posteriors: M (k x F), L^-1 (k x F x F), S (k x F x F), 1 / beta (k), then
// k int failure flags
struct BlrPost {
    size_t M, Li, S, ib, fail, total;
    BlrPost(int k, int F) {
        const size_t FF = (size_t)F * F;
        M = 0; Li = M + (size_t)k * F; S = Li + k * FF; ib = S + k * FF; fail = ib + k;
        total = fail * 8 + (size_t)k * 4;
    }
};

// the check of the BLR entry points, which also serve the Bayesian linear regression of a trained DNGO handle
int blr_ready(gpk_handle* h, const char* who) {
    int rc;
    if (h && h->model == MODEL_DNGO) {
        if ((rc = model_ready(h, MODEL_DNGO, who))) return rc;
        if (!h->dngo.trained) { set_err(h, "%s: model is not trained (gpk_dngo_train)", who); return GPK_NOT_FITTED; }
    } else if ((rc = model_ready(h, MODEL_BLR, who))) {
        return rc;
    }
    const int sm_eval = (int)(gpk_blr_smem_doubles(h->blr.F) * 8);
    CK(cudaFuncSetAttribute(gpk_blr_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sm_eval));
    CK(cudaFuncSetAttribute(gpk_blr_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sm_eval));
    CK(cudaFuncSetAttribute(gpk_blr_fit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            sm_eval + h->blr.F * h->blr.F * 8));
    CK(cudaFuncSetAttribute(gpk_blr_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            h->blr.F * GPK_BLR_SCORE_THREADS * 8));
    return GPK_OK;
}

// the layout of h->rf.data: X (n x d doubles), y (n doubles), the per-feature row order (d x n ints)
inline double* rf_X(gpk_handle* h) { return ptr<double>(h->rf.data); }
inline double* rf_y(gpk_handle* h) { return rf_X(h) + (size_t)h->n * h->d; }
inline int* rf_order(gpk_handle* h) { return (int*)(rf_y(h) + h->n); }

// the layout of h->rf.nodes (bytes) for T trees of S = 2 n node slots: feat, left (T x S ints), n_nodes (T ints, padded
// to 8 bytes), thr, W, mean, var (T x S doubles each)
struct RfNodes {
    size_t feat, left, nn, thr, W, mean, var, total;
    RfNodes(int T, long S) {
        const size_t TS = (size_t)T * S;
        feat = 0; left = feat + TS * 4; nn = left + TS * 4;
        thr = nn + ((size_t)T * 4 + 7) / 8 * 8;
        W = thr + TS * 8; mean = W + TS * 8; var = mean + TS * 8; total = var + TS * 8;
    }
};

// the layout of h->bnn.data: the scaled X (n x d), the scaled y (n), the input mean and std (d each)
inline double* bnn_X(gpk_handle* h) { return ptr<double>(h->bnn.data); }
inline double* bnn_y(gpk_handle* h) { return bnn_X(h) + (size_t)h->n * h->d; }
inline double* bnn_xm(gpk_handle* h) { return bnn_y(h) + h->n; }
inline double* bnn_xs(gpk_handle* h) { return bnn_xm(h) + h->d; }

// score_dev for a surrogate handle: its scoring kernel over the m rows dX in one launch, with score_dev's outputs,
// offsets and running arg-max
int surrogate_score(gpk_handle* h, const double* dX, long m, int kind, double eta, double par, double* d_out,
                    double* d_mu, double* d_var, BestPair* d_best, unsigned long long* d_nneg, long index_offset,
                    bool reset, long global_base, Feeder* feeder) {
    int rc = h->model == MODEL_BLR ? blr_ready(h, "scoring") : model_ready(h, h->model, "scoring");
    if (rc) return rc;
    // candidates per CTA (DNGO: per tile; one resident CTA per SM walks the tiles)
    const long tile = h->model == MODEL_BLR ? GPK_BLR_SCORE_THREADS
                    : h->model == MODEL_RF  ? GPK_RF_SCORE_WARPS
                    : h->model == MODEL_BNN ? GPK_BNN_SCORE_THREADS * GPK_BNN_SCORE_C
                                            : GPK_DNGO_SCORE_THREADS;
    const long ntiles = (m + tile - 1) / tile;
    const long nblk = h->model == MODEL_DNGO ? std::min(ntiles, (long)h->n_sm) : ntiles;
    if ((rc = ensure(h, h->block_best, (size_t)std::max(nblk, 1L) * sizeof(BestPair)))) return rc;
    if ((rc = ensure(h, h->best, sizeof(BestPair)))) return rc;
    if ((rc = ensure(h, h->nneg, 8))) return rc;
    if (d_best == nullptr) d_best = ptr<BestPair>(h->best);
    if (d_nneg == nullptr) d_nneg = ptr<unsigned long long>(h->nneg);
    if (reset) {
        CK(cudaMemsetAsync(d_best, 0xFF, sizeof(BestPair), h->stream));
        CK(cudaMemsetAsync(d_nneg, 0, 8, h->stream));
    }
    if (feeder && (rc = feeder->ready(0, m, h->stream))) return rc;
    if (m == 0) return GPK_OK;
    const ScoreOut o = score_out(h, kind, eta, par, d_out, d_mu, d_var, d_nneg, index_offset, global_base);
    switch (h->model) {
    case MODEL_BLR: {
        const int F = h->blr.F, k = h->blr.k;
        const BlrPost L(k, F);
        const double* post = ptr<double>(h->blr.post);
        BlrScoreArgs a;
        memset(&a, 0, sizeof(a));
        a.X = dX; a.m = m; a.D = h->d; a.F = F; a.basis = h->blr.basis; a.k = k;
        a.M = post + L.M; a.Li = post + L.Li; a.ib = post + L.ib;
        a.o = o;
        gpk_blr_score_kernel<<<(unsigned)nblk, GPK_BLR_SCORE_THREADS, (size_t)F * GPK_BLR_SCORE_THREADS * 8, h->stream>>>(a);
        break;
    }
    case MODEL_RF: {
        const long S = 2L * h->n;
        const RfNodes L(h->rf.T, S);
        const char* nodes = ptr<char>(h->rf.nodes);
        RfScoreArgs a;
        memset(&a, 0, sizeof(a));
        a.X = dX; a.m = m; a.D = h->d; a.T = h->rf.T; a.S = S;
        a.feat = (const int*)(nodes + L.feat); a.left = (const int*)(nodes + L.left);
        a.thr = (const double*)(nodes + L.thr); a.mean = (const double*)(nodes + L.mean);
        a.var = (const double*)(nodes + L.var);
        a.total_var = h->rf.total;
        a.o = o;
        gpk_rf_score_kernel<<<(unsigned)nblk, GPK_RF_SCORE_WARPS * 32, gpk_rf_score_smem_doubles(h->rf.T) * 8,
                              h->stream>>>(a);
        break;
    }
    case MODEL_BNN: {
        BnnScoreArgs a;
        memset(&a, 0, sizeof(a));
        a.X = dX; a.m = m; a.D = h->d; a.P = h->bnn.P; a.S = h->bnn.S;
        a.samples = ptr<double>(h->bnn.samples);
        a.xm = bnn_xm(h); a.xs = bnn_xs(h);
        a.y_mean = h->bnn.ymean; a.y_std = h->bnn.ystd;
        a.o = o;
        const size_t smem = (size_t)gpk_bnn_score_smem(h->d);
        CK(cudaFuncSetAttribute(gpk_bnn_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        gpk_bnn_score_kernel<<<(unsigned)nblk, GPK_BNN_SCORE_THREADS, smem, h->stream>>>(a);
        break;
    }
    case MODEL_DNGO: {
        DngoScoreArgs a;
        memset(&a, 0, sizeof(a));
        a.X = dX; a.m = m; a.D = h->d; a.ntiles = (int)ntiles;
        a.pack = ptr<double>(h->dngo.pack);
        a.xm = bnn_xm(h); a.xs = bnn_xs(h);
        a.y_mean = h->bnn.ymean; a.y_std = h->bnn.ystd;
        a.o = o;
        const size_t smem = (size_t)gpk_dngo_score_smem(h->d);
        CK(cudaFuncSetAttribute(gpk_dngo_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        gpk_dngo_score_kernel<<<(unsigned)nblk, GPK_DNGO_SCORE_THREADS, smem, h->stream>>>(a);
        break;
    }
    default:
        BAD("scoring: unknown model kind %d", (int)h->model);
    }
    CKL();
    if (kind != GPK_ACQ_NONE) {
        gpk_argmax_final_kernel<<<1, 256, 0, h->stream>>>(ptr<BestPair>(h->block_best), (int)nblk, d_best);
        CKL();
    }
    return GPK_OK;
}

}  // namespace

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

int gpk_comm_destroy(gpk_handle* h);

const char* gpk_version(void) { return "gpk 0.2 (sm_90a, fp64 DMMA + TMA)"; }

const char* gpk_last_error(gpk_handle* h) { return h ? h->err : "null handle"; }

int gpk_create(gpk_handle** out, int device) {
    if (!out) return GPK_BAD_ARG;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) return GPK_CUDA_ERROR;
    gpk_handle* h = new gpk_handle();
    h->device = device;
    memset(&h->spec, 0, sizeof(h->spec));
    if (cudaSetDevice(device) != cudaSuccess) { delete h; return GPK_CUDA_ERROR; }
    {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);      // hi = numerically smallest = highest priority
        if (cudaStreamCreateWithPriority(&h->own_stream, cudaStreamNonBlocking, hi) != cudaSuccess) { delete h; return GPK_CUDA_ERROR; }
        if (cudaStreamCreateWithPriority(&h->side_stream, cudaStreamNonBlocking, lo) != cudaSuccess) { delete h; return GPK_CUDA_ERROR; }
        if (cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking) != cudaSuccess) { delete h; return GPK_CUDA_ERROR; }
    }
    h->stream = h->own_stream;
    for (int i = 0; i < 16; ++i)
        if (cudaEventCreate(&h->timing.ev[i]) != cudaSuccess) { delete h; return GPK_CUDA_ERROR; }
    if (cudaEventCreateWithFlags(&h->ev_order, cudaEventDisableTiming) != cudaSuccess) { delete h; return GPK_CUDA_ERROR; }
    int rc = set_kernel_attrs(h);
    if (rc) { fprintf(stderr, "gpk_create: %s\n", h->err); delete h; return rc; }
    if (get_encode_fn() == nullptr) {
        fprintf(stderr, "gpk_create: the driver has no cuTensorMapEncodeTiled (TMA descriptors)\n");
        delete h;
        return GPK_CUDA_ERROR;
    }
    rc = ensure(h, h->status, 4);
    if (!rc) rc = ensure(h, h->scal, 64);
    if (rc) { delete h; return rc; }
    if (cudaMallocHost((void**)&h->pin, 64) != cudaSuccess) { delete h; return GPK_CUDA_ERROR; }
    *out = h;
    return GPK_OK;
}

int gpk_destroy(gpk_handle* h) {
    if (!h) return GPK_OK;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    gpk_comm_destroy(h);
    delete h;
    return GPK_OK;
}

int gpk_set_option(gpk_handle* h, const char* key, long value) {
    if (!h || !key) return GPK_BAD_ARG;
    if (!strcmp(key, "ozpersist")) {
        if (value != 0 && value != 1 && value != 3) BAD("ozpersist must be 0, 1 or 3");
        h->oz.persist = (int)value;
        return GPK_OK;
    }
    if (!strcmp(key, "ozcluster")) {
        if (value != 1 && value != 2 && value != 4) BAD("ozcluster must be 1, 2 or 4");
        h->oz.cluster = (int)value;
        return GPK_OK;
    }
    if (!strcmp(key, "ozgrid")) {
        if (value < 0 || value > (1L << 20)) BAD("ozgrid must be >= 0 (0: as many clusters as fit)");
        h->oz.grid = (int)value;
        return GPK_OK;
    }
    if (!strcmp(key, "ozaki")) {
        if (value != 0 && value != 1)
            BAD("ozaki must be 0 (fp64 DMMA) or 1 (int8 tensor pipe, error-free split; kernels with the environment "
                "factor always take fp64)");
        h->oz.enabled = (int)value;
        return GPK_OK;
    }
    if (!strcmp(key, "depth2")) {
        if (value < 0 || value > 2) BAD("depth2 must be 0, 1 or 2 (automatic)");
        h->depth2 = (int)value;
        return GPK_OK;
    }
    if (!strcmp(key, "meanonly")) {
        if (value != 0 && value != 1) BAD("meanonly must be 0 or 1");
        h->mean_only = (int)value;
        return GPK_OK;
    }
    if (!strcmp(key, "overlap")) {
        if (value != 0 && value != 1) BAD("overlap must be 0 or 1");
        h->overlap = (int)value;
        return GPK_OK;
    }
    if (!strcmp(key, "diagprof")) {                 // 1: stamps; 2: stamps + skip the kernel's global stores (timing only)
        h->diag_prof = value != 0;
        if (h->diag_prof) {
            int rc = ensure(h, h->dprof, 64 * 8);
            if (rc) return rc;
            CK(cudaMemset(h->dprof.p, 0, 64 * 8));
            if (value == 2) {
                const long long one = 1;
                CK(cudaMemcpy((char*)h->dprof.p + 63 * 8, &one, 8, cudaMemcpyHostToDevice));
            }
        }
        return GPK_OK;
    }
    if (!strcmp(key, "hyper_batch_bytes")) {
        if (value < 1) BAD("hyper_batch_bytes must be >= 1 (default %ld)", (long)GPK_HYPER_BATCH_BYTES);
        h->hyper.batch_bytes = value;
        return GPK_OK;
    }
    if (!strcmp(key, "chunk")) {
        if (value == 0) { h->chunk_user = false; return GPK_OK; }          // back to the automatic choice
        if (value < BM || value % BM) BAD("chunk must be a positive multiple of 128 (0 = automatic)");
        h->chunk = value;
        h->chunk_user = true;
        return GPK_OK;
    }
    BAD("unknown option '%s'", key);
}

int gpk_set_stream(gpk_handle* h, void* s) {
    if (!h) return GPK_BAD_ARG;
    cudaStreamSynchronize(h->stream);
    h->stream = s ? (cudaStream_t)s : h->own_stream;
    return GPK_OK;
}

int gpk_synchronize(gpk_handle* h) {
    if (!h) return GPK_BAD_ARG;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

namespace {
// col_tasks (gpk_handle) of n rows of row-major inputs X (d columns)
std::vector<int> scan_task_columns(const double* X, int n, int d) {
    std::vector<int> cols(d, 0);
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < d; ++j) {
            const double v = X[(long)i * d + j];
            int& c = cols[j];
            if (c == INT_MAX) continue;
            c = (v >= 0.0 && v < 1e9 && v == floor(v)) ? std::max(c, (int)v + 1) : INT_MAX;
        }
    return cols;
}

// The kernel's factor against inputs of d columns: its axis inside them.  With cols, the column summary of a training
// set (scan_task_columns), the task factor also needs unscaled inputs (no input bounds) and valid task indices.
int factor_data_check(gpk_handle* h, int d, const std::vector<int>* cols, const char* who) {
    const KFactor& f = h->spec.factor;
    if (f.kind == GPK_FACTOR_NONE) return GPK_OK;
    if (f.axis >= d)
        BAD("%s: %s axis %d >= d = %d", who, f.kind == GPK_FACTOR_ENV ? "environment" : "task", f.axis, d);
    if (f.kind != GPK_FACTOR_TASK || !cols) return GPK_OK;
    if (h->has_bounds) BAD("%s: the task factor needs unscaled inputs (no input bounds)", who);
    if ((int)cols->size() != d || (*cols)[f.axis] > f.n_tasks)
        BAD("%s: training column %d holds a value that is not a task index in [0, %d)", who, f.axis, f.n_tasks);
    return GPK_OK;
}

// gpk_set_env_factor / gpk_set_task_factor after their checks: f (kind NONE: clear) replaces the kernel's factor,
// except that clearing one kind leaves a factor of the other kind in place
int set_factor(gpk_handle* h, int kind, const KFactor& f) {
    if (f.kind != GPK_FACTOR_NONE || h->spec.factor.kind == kind) h->spec.factor = f;
    h->fitted = false;
    h->linv_ready = false;
    h->alpha_ready = false;
    return GPK_OK;
}
}  // namespace

int gpk_set_data(gpk_handle* h, const double* X, const double* y, int n, int d) {
    if (!h) return GPK_BAD_ARG;
    if (gp_refusal(h)) BAD("gpk_set_data: %s", gp_refusal(h));
    if (!X || !y || n <= 0 || d <= 0) BAD("gpk_set_data: need X, y, n > 0, d > 0");
    if (d > GPK_MAX_TERMS) BAD("gpk_set_data: d = %d exceeds GPK_MAX_TERMS = %d", d, GPK_MAX_TERMS);
    CK(cudaSetDevice(h->device));
    const long NP = round_up(n, BM);
    int rc;
    bool g1, g2, g3, g4;
    if ((rc = ensure(h, h->Xrow, (size_t)NP * d * 8))) return rc;      // room for the rows gpk_fit_append may add
    if ((rc = ensure(h, h->Xt, (size_t)d * NP * 8))) return rc;
    if ((rc = ensure(h, h->y, (size_t)NP * 8))) return rc;
    if ((rc = ensure(h, h->Kbuf, (size_t)(NP + BM) * NP * 8, &g1))) return rc;
    if ((rc = ensure(h, h->P, (size_t)NP * NP * 8, &g2))) return rc;
    if ((rc = ensure(h, h->Q, (size_t)NP * NP * 8, &g3))) return rc;
    if ((rc = ensure(h, h->W, (size_t)NP * NP * 8, &g4))) return rc;
    if ((rc = ensure(h, h->logdet_part, (size_t)(NP / BM) * 8))) return rc;
    const bool relayout = (h->layout_NP != NP) || g1 || g2 || g3 || g4;
    h->n = n; h->d = d; h->NP = (int)NP; h->nb = (int)(NP / BM);
    if (relayout) {
        CK(cudaMemsetAsync(h->Kbuf.p, 0, (size_t)(NP + BM) * NP * 8, h->stream));
        CK(cudaMemsetAsync(h->P.p, 0, (size_t)NP * NP * 8, h->stream));
        CK(cudaMemsetAsync(h->Q.p, 0, (size_t)NP * NP * 8, h->stream));
        CK(cudaMemsetAsync(h->W.p, 0, (size_t)NP * NP * 8, h->stream));
        h->layout_NP = (int)NP;
        h->maps_ok = false;
    }
    CK(cudaMemcpyAsync(h->Xrow.p, X, (size_t)n * d * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemsetAsync(h->y.p, 0, (size_t)NP * 8, h->stream));
    CK(cudaMemcpyAsync(h->y.p, y, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
    {
        long total = (long)d * NP;
        gpk_transpose_kernel<<<(unsigned)((total + 255) / 256), 256, 0, h->stream>>>(ptr<double>(h->Xrow), n, d, nullptr,
                                                                                    nullptr, ptr<double>(h->Xt), NP);
        CKL();
    }
    CK(cudaStreamSynchronize(h->stream));     // host buffers are caller-owned: done with them
    h->col_tasks = scan_task_columns(X, n, d);
    if ((rc = build_job_tables(h))) return rc;
    if (!h->maps_ok && (rc = rebuild_maps(h))) return rc;
    h->has_data = true;
    h->fitted = false;
    h->linv_ready = false;
    h->alpha_ready = false;
    return GPK_OK;
}

int gpk_set_input_bounds(gpk_handle* h, const double* lower, const double* upper, int d) {
    if (!h) return GPK_BAD_ARG;
    if (gp_refusal(h)) BAD("gpk_set_input_bounds: %s", gp_refusal(h));
    CK(cudaSetDevice(h->device));
    if (!lower || !upper) { h->has_bounds = false; return GPK_OK; }
    if (d <= 0 || d > GPK_MAX_TERMS) BAD("gpk_set_input_bounds: bad d");
    int rc;
    if ((rc = ensure(h, h->lower, (size_t)d * 8))) return rc;
    if ((rc = ensure(h, h->upper, (size_t)d * 8))) return rc;
    CK(cudaMemcpyAsync(h->lower.p, lower, (size_t)d * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->upper.p, upper, (size_t)d * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->has_bounds = true;
    return GPK_OK;
}

int gpk_set_output_transform(gpk_handle* h, int enabled, double y_mean, double y_std) {
    if (!h) return GPK_BAD_ARG;
    if (gp_refusal(h)) BAD("gpk_set_output_transform: %s", gp_refusal(h));
    h->norm_out = enabled ? 1 : 0;
    h->y_mean = y_mean;
    h->y_std = y_std;
    return GPK_OK;
}

int gpk_set_kernel(gpk_handle* h, int family, double log_amp, int n_terms, const int* axis, const int* group,
                   const double* log_metric) {
    if (!h) return GPK_BAD_ARG;
    if (gp_refusal(h)) BAD("gpk_set_kernel: %s", gp_refusal(h));
    if (family < GPK_MATERN52 || family > GPK_MATERN32) BAD("gpk_set_kernel: unknown family %d", family);
    if (n_terms <= 0 || n_terms > GPK_MAX_TERMS || !axis || !group || !log_metric)
        BAD("gpk_set_kernel: need 1..%d terms", GPK_MAX_TERMS);
    KSpec s;
    memset(&s, 0, sizeof(s));
    s.family = family;
    s.n_terms = n_terms;
    s.amp = exp(log_amp);
    for (int t = 0; t < n_terms; ++t) {
        if (axis[t] < 0 || axis[t] >= GPK_MAX_TERMS) BAD("gpk_set_kernel: axis out of range");
        if (t > 0 && (group[t] < group[t - 1] || group[t] > group[t - 1] + 1)) BAD("gpk_set_kernel: groups must be contiguous");
        s.axis[t] = axis[t];
        s.inv_metric[t] = 1.0 / exp(log_metric[t]);
        s.scale[t] = sqrt((family == GPK_MATERN52 ? 5.0 : family == GPK_MATERN32 ? 3.0 : 0.5) * s.inv_metric[t]);
        s.last[t] = (t == n_terms - 1) || (group[t + 1] != group[t]);
    }
    if (group[0] != 0) BAD("gpk_set_kernel: groups must start at 0");
    h->spec = s;
    h->has_spec = true;
    h->fitted = false;
    h->linv_ready = false;
    h->alpha_ready = false;
    return GPK_OK;
}

int gpk_set_env_factor(gpk_handle* h, int axis, double log_a, double log_b) {
    if (!h) return GPK_BAD_ARG;
    if (gp_refusal(h)) BAD("gpk_set_env_factor: %s", gp_refusal(h));
    if (axis < -1 || axis >= GPK_MAX_TERMS) BAD("gpk_set_env_factor: axis %d out of range", axis);
    if (!std::isfinite(log_a) || !std::isfinite(log_b)) BAD("gpk_set_env_factor: log_a and log_b must be finite");
    if (axis >= 0 && h->spec.factor.kind == GPK_FACTOR_TASK) BAD("gpk_set_env_factor: the kernel has a task factor");
    KFactor f{};
    if (axis >= 0) {
        const double p[2] = {log_a, log_b};
        f = KFactor{GPK_FACTOR_ENV, axis};
        gpk_factor_build(f, p);
    }
    return set_factor(h, GPK_FACTOR_ENV, f);
}

int gpk_set_task_factor(gpk_handle* h, int axis, int n_tasks, const double* theta) {
    if (!h) return GPK_BAD_ARG;
    if (gp_refusal(h)) BAD("gpk_set_task_factor: %s", gp_refusal(h));
    if (axis < -1 || axis >= GPK_MAX_TERMS) BAD("gpk_set_task_factor: axis %d out of range", axis);
    KFactor f{};
    if (axis >= 0) {
        if (n_tasks < 1 || n_tasks > GPK_MAX_TASKS)
            BAD("gpk_set_task_factor: n_tasks = %d outside 1..%d (GPK_MAX_TASKS)", n_tasks, GPK_MAX_TASKS);
        if (!theta) BAD("gpk_set_task_factor: need theta");
        for (int k = 0; k < n_tasks * (n_tasks + 1) / 2; ++k)
            if (!std::isfinite(theta[k])) BAD("gpk_set_task_factor: theta[%d] is not finite", k);
        if (h->spec.factor.kind == GPK_FACTOR_ENV) BAD("gpk_set_task_factor: the kernel has an environment factor");
        f = KFactor{GPK_FACTOR_TASK, axis, n_tasks};
        gpk_factor_build(f, theta);
        h->task_theta.assign(theta, theta + n_tasks * (n_tasks + 1) / 2);
    }
    return set_factor(h, GPK_FACTOR_TASK, f);
}


int gpk_fit_begin(gpk_handle* h, double diag_add, double mean) {
    int rc = require(h, true, true, false);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    for (int t = 0; t < h->spec.n_terms; ++t)
        if (h->spec.axis[t] >= h->d) BAD("gpk_fit: kernel axis %d >= d = %d", h->spec.axis[t], h->d);
    if ((rc = factor_data_check(h, h->d, &h->col_tasks, "gpk_fit"))) return rc;
    const long NP = h->NP;
    const int nb = h->nb;
    if (!h->maps_ok && (rc = rebuild_maps(h))) return rc;        // staging mode changed after gpk_set_data
    h->fitted = false;
    h->linv_ready = false;
    h->alpha_ready = false;
    h->mean = mean;
    h->diag_add = diag_add;
    double* K = ptr<double>(h->Kbuf);

    CK(cudaEventRecord(h->timing.ev[0], h->stream));
    {
        // the pre-scaled operand depends on the hyper-parameters: rebuilt per fit (n_terms x NP)
        if ((rc = ensure(h, h->Xts, (size_t)GPK_MAX_TERMS * NP * 8))) return rc;
        if ((rc = build_cov_operand(h, h->stream, ptr<double>(h->Xrow), h->n, h->d, nullptr, nullptr, ptr<double>(h->Xts), NP)))
            return rc;
        if ((rc = launch_cov_tiles(h, h->stream, ptr<double>(h->Xts), NP, h->n, ptr<double>(h->Xrow), h->d, (long)h->n, NP,
                                   nullptr, nullptr, K, NP, 1, false, ptr<double>(h->Xrow), nullptr, nullptr)))
            return rc;
        gpk_kfix_kernel<<<(unsigned)((NP + 255) / 256), 256, 0, h->stream>>>(K, NP, h->n, (int)NP, diag_add,
                                                                            ptr<double>(h->y), mean);
        CKL();
    }
    CK(cudaMemsetAsync(h->status.p, 0, 4, h->stream));
    CK(cudaEventRecord(h->timing.ev[1], h->stream));
    if ((rc = grow_events(h, h->ev_panel, nb, cudaEventDisableTiming)) ||
        (rc = grow_events(h, h->ev_rest, nb, cudaEventDisableTiming)))
        return rc;
    std::vector<char> rest_recorded(nb, 0);
    // ---- look-ahead schedule: diag(k), then the panel solve and the update of block column k+1 in 32-row tiles on the
    // critical stream; the rest of the trailing update on the side stream
    gpk_diag_prezero_kernel<<<nb, 256, 0, h->stream>>>(K, (long)NP, ptr<double>(h->P), (long)NP);
    CKL();
    for (int k = 0; k < nb; ++k) {
        long long* dprof = h->diag_prof ? ptr<long long>(h->dprof) : nullptr;
        if (k > 0)
            CK(launch_pdl(gpk_potrf_diag_dmma_kernel, dim3(1), dim3(256), (size_t)DIAG_SMEM, h->stream, K, (long)NP, k,
                          ptr<double>(h->P), ptr<double>(h->Q), (long)NP, ptr<int>(h->status), ptr<double>(h->logdet_part), dprof));
        else
            gpk_potrf_diag_dmma_kernel<<<1, 256, DIAG_SMEM, h->stream>>>(K, NP, k, ptr<double>(h->P), ptr<double>(h->Q), NP,
                                                                         ptr<int>(h->status), ptr<double>(h->logdet_part), dprof);
        CKL();
        GemmArgs a;
        memset(&a, 0, sizeof(a));
        a.A = K; a.lda = NP;
        a.B = ptr<double>(h->P); a.ldb = NP;
        a.C = K; a.ldc = NP;
        a.alpha = 1.0; a.beta = 0;
        a.job_mode = JOBS_TABLE;
        a.status = ptr<int>(h->status);
        a.jobs = ptr<GemmJob>(h->jobs) + h->ranges.trsm32[k].off;
        if ((rc = launch_gemm<EPI_STORE, 2>(h, h->mapK32, h->mapP, a, h->ranges.trsm32[k].cnt))) return rc;
        GemmArgs s;
        memset(&s, 0, sizeof(s));
        s.A = K; s.lda = NP;
        s.B = K; s.ldb = NP;
        s.C = K; s.ldc = NP;
        s.alpha = -1.0; s.beta = 1;
        s.job_mode = JOBS_TABLE;
        s.status = ptr<int>(h->status);
        const int off = h->ranges.syrk[k].off, cnt = h->ranges.syrk[k].cnt;
        if (cnt > 0) {
            // Look-ahead: the first nb-k jobs update column block k+1 (what the next diagonal block
            // and panel solve need) and stay on the critical stream; the rest of the trailing update
            // runs on the low-priority side stream, overlapped with diag(k+1) / panel(k+1).
            const int npu = nb - k;
            CK(cudaEventRecord(h->ev_panel[k], h->stream));                       // panel k solved
            if (k >= 1 && rest_recorded[k - 1]) CK(cudaStreamWaitEvent(h->stream, h->ev_rest[k - 1], 0));
            s.jobs = ptr<GemmJob>(h->jobs) + h->ranges.pu32[k].off;
            if ((rc = launch_gemm<EPI_STORE, 2>(h, h->mapK32, h->mapK, s, h->ranges.pu32[k].cnt))) return rc;
            const bool d2 = h->depth2 == 1 || (h->depth2 == 2 && nb >= 48);
            if (cnt > npu && !d2) {
                CK(cudaStreamWaitEvent(h->side_stream, h->ev_panel[k], 0));
                s.jobs = ptr<GemmJob>(h->jobs) + off + npu;
                if ((rc = launch_gemm<EPI_STORE>(h, h->mapK, h->mapK, s, cnt - npu, h->side_stream))) return rc;
                CK(cudaEventRecord(h->ev_rest[k], h->side_stream));
                rest_recorded[k] = 1;
            } else if (cnt > npu) {
                // depth 2: even steps update block column k+2 only (what step k+1 needs) and defer the columns behind it;
                // odd steps apply panels k-1 and k together to every column >= k+2 in one K = 256 contraction (twice the
                // work per tile: a 128-long update is mostly pipeline fill and tile I/O)
                CK(cudaStreamWaitEvent(h->side_stream, h->ev_panel[k], 0));
                if ((k & 1) == 0) {
                    s.jobs = ptr<GemmJob>(h->jobs) + off + npu;
                    if ((rc = launch_gemm<EPI_STORE>(h, h->mapK, h->mapK, s, std::min(nb - k - 1, cnt - npu), h->side_stream))) return rc;
                } else {
                    s.jobs = ptr<GemmJob>(h->jobs) + h->ranges.syrk2[k].off;
                    if ((rc = launch_gemm<EPI_STORE>(h, h->mapK, h->mapK, s, h->ranges.syrk2[k].cnt, h->side_stream))) return rc;
                }
                CK(cudaEventRecord(h->ev_rest[k], h->side_stream));
                rest_recorded[k] = 1;
            }
        }
    }
    gpk_diag_qfill_kernel<<<nb, 256, 0, h->stream>>>(ptr<double>(h->P), ptr<double>(h->Q), (long)NP, ptr<int>(h->status));
    CKL();
    CK(cudaEventRecord(h->timing.ev[2], h->stream));
    gpk_fit_reduce_kernel<<<1, 256, 0, h->stream>>>(K + NP * NP, h->n, ptr<double>(h->logdet_part), nb,
                                                    ptr<double>(h->scal));
    CKL();
    CK(cudaEventRecord(h->timing.ev[3], h->stream));
    CK(cudaMemcpyAsync(h->pin, h->scal.p, 16, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(h->pin + 2, h->status.p, 4, cudaMemcpyDeviceToHost, h->stream));
    h->fit_pending = true;
    return GPK_OK;
}

int gpk_fit_end(gpk_handle* h, double* logdet, double* loglik) {
    if (!h) return GPK_BAD_ARG;
    if (!h->fit_pending) BAD("gpk_fit_end without gpk_fit_begin");
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    h->fit_pending = false;
    const double* sc = h->pin;
    int st = 0;
    memcpy(&st, h->pin + 2, 4);
    h->timing.fit_timed = true;
    if (st != 0) {
        set_err(h, "matrix is not positive definite: pivot %d <= 0", st - 1);
        return GPK_NOT_PD;
    }
    const double ld = sc[1];
    const double ll = -0.5 * sc[0] - 0.5 * ld - 0.5 * (double)h->n * log(2.0 * M_PI);
    if (logdet) *logdet = ld;
    if (loglik) *loglik = ll;
    h->fitted = true;
    return GPK_OK;
}

int gpk_fit(gpk_handle* h, double diag_add, double mean, double* logdet, double* loglik) {
    int rc = gpk_fit_begin(h, diag_add, mean);
    if (rc) return rc;
    return gpk_fit_end(h, logdet, loglik);
}

// ---------------------------------------------------------------------------------------
// Incremental refit (SURVEY.md 8f-4: BaseModel.update / train(do_optimize=False) with frozen hyper-parameters).
// The rows appended since the last fit live in the last 128-row block b of the padded layout, so the leading factor
// L11 (N1 = 128 b rows), its inverse P11 and every earlier block of K are unchanged.  With L11^-1 explicit:
//   L_row = K[b, 0:N1] P11^T                      (one launch, 32-row tiles)
//   S     = K[b, b] - L_row L_row^T               (b partial Gram tiles + fixed-order sum)
//   L_bb, P_bb = chol / inverse of S              (the diagonal-block kernel)
//   P[b, 0:N1] = -P_bb (L_row P11)                (two launches; transposes kept in Q)
//   z = P (y - mean),  log|K| = 2 sum log diag    (y and the mean change with every new observation)
// O(N^2) work instead of the O(N^3) factorisation + inversion.  Returns GPK_NOT_APPLICABLE (nothing touched) when
// the preconditions do not hold; the caller then runs gpk_set_data + gpk_fit.
// ---------------------------------------------------------------------------------------
int gpk_fit_append(gpk_handle* h, const double* X, const double* y, int n, int d, double diag_add, double mean,
                   double* logdet, double* loglik) {
    if (!h) return GPK_BAD_ARG;
    if (gp_refusal(h)) BAD("gpk_fit_append: %s", gp_refusal(h));
    if (!X || !y || n <= 0 || d <= 0) BAD("gpk_fit_append: need X, y, n > 0, d > 0");
    const long NP = h->NP;
    const int nb = h->nb, b = nb - 1, N1 = b * BM;
    if (!h->has_data || !h->has_spec || !h->fitted || !h->linv_ready || h->fit_pending || d != h->d || nb < 2 ||
        round_up(n, BM) != NP || n <= h->n || h->n <= N1 || diag_add != h->diag_add) {
        set_err(h, "gpk_fit_append: not applicable (needs a fitted model with L^-1 built, the same kernel / "
                   "diagonal term, new rows inside the last 128-row block)");
        return GPK_NOT_APPLICABLE;
    }
    CK(cudaSetDevice(h->device));
    int rc;
    if (!h->maps_ok && (rc = rebuild_maps(h))) return rc;
    // checked before anything is uploaded; committed once the device holds the new rows
    std::vector<int> cols = scan_task_columns(X, n, d);
    if ((rc = factor_data_check(h, d, &cols, "gpk_fit_append"))) return rc;
    double* K = ptr<double>(h->Kbuf);
    double* P = ptr<double>(h->P);
    double* Q = ptr<double>(h->Q);
    double* W = ptr<double>(h->W);
    if ((rc = ensure(h, h->tmp1, (size_t)NP * 8))) return rc;
    CK(cudaEventRecord(h->timing.ev[0], h->stream));
    // inputs (everything is re-uploaded: 8 n (d + 1) bytes; the first h->n rows of X must be the ones already fitted)
    if ((rc = ensure(h, h->Xrow, (size_t)NP * d * 8))) return rc;      // no-op: gpk_set_data sized it for NP rows
    CK(cudaMemcpyAsync(h->Xrow.p, X, (size_t)n * d * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemsetAsync(h->y.p, 0, (size_t)NP * 8, h->stream));
    CK(cudaMemcpyAsync(h->y.p, y, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
    {
        long total = (long)d * NP;
        gpk_transpose_kernel<<<(unsigned)((total + 255) / 256), 256, 0, h->stream>>>(ptr<double>(h->Xrow), n, d, nullptr,
                                                                                    nullptr, ptr<double>(h->Xt), NP);
        CKL();
    }
    // block row b of K (all columns), diagonal term, padding rows
    {
        if ((rc = ensure(h, h->Xts, (size_t)GPK_MAX_TERMS * NP * 8))) return rc;
        if ((rc = build_cov_operand(h, h->stream, ptr<double>(h->Xrow), n, d, nullptr, nullptr, ptr<double>(h->Xts), NP)))
            return rc;
        if ((rc = launch_cov_tiles(h, h->stream, ptr<double>(h->Xts), NP, n, ptr<double>(h->Xrow) + (long)N1 * d, d,
                                   (long)(n - N1), BM, nullptr, nullptr, K + (long)N1 * NP, NP, 0, false,
                                   ptr<double>(h->Xrow), nullptr, nullptr)))
            return rc;
        gpk_kfix_rows_kernel<<<1, 128, 0, h->stream>>>(K, NP, n, (int)NP, diag_add, N1);
        CKL();
    }
    CK(cudaMemsetAsync(h->status.p, 0, 4, h->stream));
    CK(cudaEventRecord(h->timing.ev[1], h->stream));
    GemmArgs a;
    // L_row = K[b, 0:N1] P11^T -> W[b, 0:N1]: split-K partial tiles into the free tiles W(c, j), then a fixed-order sum
    memset(&a, 0, sizeof(a));
    a.A = K; a.lda = NP; a.B = P; a.ldb = NP; a.C = W; a.ldc = NP;
    a.alpha = 1.0; a.beta = 0; a.job_mode = JOBS_TABLE;
    a.jobs = ptr<GemmJob>(h->jobs) + h->ranges.app_row2.off;
    if ((rc = launch_gemm<EPI_STORE>(h, h->mapK, h->mapP, a, h->ranges.app_row2.cnt))) return rc;
    gpk_append_reduce_kernel<<<dim3(b, 64), 256, 0, h->stream>>>(W, NP, b, 0, W + (long)N1 * NP, NP, nullptr, 0, 0);
    CKL();
    // partial Gram tiles, then the Schur complement of the last block
    memset(&a, 0, sizeof(a));
    a.A = W; a.lda = NP; a.B = W; a.ldb = NP; a.C = W; a.ldc = NP;
    a.alpha = 1.0; a.beta = 0; a.job_mode = JOBS_TABLE;
    a.jobs = ptr<GemmJob>(h->jobs) + h->ranges.app_syrk.off;
    if ((rc = launch_gemm<EPI_STORE>(h, h->mapW, h->mapW, a, h->ranges.app_syrk.cnt))) return rc;
    gpk_append_schur_kernel<<<64, 256, 0, h->stream>>>(K, W, NP, N1, b);
    CKL();
    // L_row to its final place (rows N1.. of K, columns 0..N1)
    CK(cudaMemcpy2DAsync(K + (long)N1 * NP, (size_t)NP * 8, W + (long)N1 * NP, (size_t)NP * 8, (size_t)N1 * 8, BM,
                         cudaMemcpyDeviceToDevice, h->stream));
    // factor + invert the last diagonal block
    gpk_diag_prezero_kernel<<<1, 256, 0, h->stream>>>(K + (long)N1 * NP + N1, (long)NP, P + (long)N1 * NP + N1, (long)NP);
    CKL();
    gpk_potrf_diag_dmma_kernel<<<1, 256, DIAG_SMEM, h->stream>>>(K, NP, b, P, Q, NP, ptr<int>(h->status),
                                                                 ptr<double>(h->logdet_part), nullptr);
    CKL();
    gpk_diag_qfill_kernel<<<1, 256, 0, h->stream>>>(P + (long)N1 * NP + N1, Q + (long)N1 * NP + N1, (long)NP,
                                                     ptr<int>(h->status));
    CKL();
    // T = L_row P11 -> P[b, 0:N1], T^T -> Q[0:N1, b]   (split-K like L_row; the Gram partials in W(s, b) are consumed)
    memset(&a, 0, sizeof(a));
    a.A = K; a.lda = NP; a.B = Q; a.ldb = NP; a.C = W; a.ldc = NP;
    a.alpha = 1.0; a.beta = 0; a.job_mode = JOBS_TABLE; a.status = ptr<int>(h->status);
    a.jobs = ptr<GemmJob>(h->jobs) + h->ranges.app_t2.off;
    if ((rc = launch_gemm<EPI_STORE>(h, h->mapK, h->mapQ, a, h->ranges.app_t2.cnt))) return rc;
    gpk_append_reduce_kernel<<<dim3(b, 64), 256, 0, h->stream>>>(W, NP, b, 1, P + (long)N1 * NP, NP, Q, NP, N1);
    CKL();
    // P[b, 0:N1] = -P_bb T (and its transpose into Q)
    memset(&a, 0, sizeof(a));
    a.A = P; a.lda = NP; a.B = Q; a.ldb = NP; a.C = P; a.ldc = NP; a.Ct = Q; a.ldct = NP;
    a.alpha = -1.0; a.beta = 0; a.job_mode = JOBS_TABLE; a.status = ptr<int>(h->status);
    a.jobs = ptr<GemmJob>(h->jobs) + h->ranges.app_p.off;
    if ((rc = launch_gemm<EPI_STORE>(h, h->mapP, h->mapQ, a, h->ranges.app_p.cnt))) return rc;
    // z = P (y - mean) into row NP of K, then z^T z and the log-determinant
    gpk_resid_kernel<<<(unsigned)((NP + 255) / 256), 256, 0, h->stream>>>(ptr<double>(h->y), mean, n, (int)NP,
                                                                          ptr<double>(h->tmp1));
    CKL();
    gpk_rowdot_kernel<<<(unsigned)((NP + 7) / 8), 256, 0, h->stream>>>(P, NP, NP, (int)NP, 0, ptr<double>(h->tmp1),
                                                                       K + NP * NP);
    CKL();
    CK(cudaEventRecord(h->timing.ev[2], h->stream));
    gpk_fit_reduce_kernel<<<1, 256, 0, h->stream>>>(K + NP * NP, n, ptr<double>(h->logdet_part), nb, ptr<double>(h->scal));
    CKL();
    CK(cudaEventRecord(h->timing.ev[3], h->stream));
    CK(cudaMemcpyAsync(h->pin, h->scal.p, 16, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(h->pin + 2, h->status.p, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->timing.launches_total += 12;
    h->timing.fit_timed = true;
    int st = 0;
    memcpy(&st, h->pin + 2, 4);
    if (st != 0) {                      // the block row of K / P is half updated: the model has to be refitted
        h->fitted = false;
        h->linv_ready = false;
        h->alpha_ready = false;
        h->n = n;
        h->col_tasks = std::move(cols);
        set_err(h, "matrix is not positive definite: pivot %d <= 0", st - 1);
        return GPK_NOT_PD;
    }
    h->n = n;
    h->col_tasks = std::move(cols);
    h->mean = mean;
    h->alpha_ready = false;
    h->linv_serial += 1;                 // L^-1 changed in place: slices / alpha derived from it are stale
    const double ld2 = h->pin[1];
    const double ll = -0.5 * h->pin[0] - 0.5 * ld2 - 0.5 * (double)n * log(2.0 * M_PI);
    if (logdet) *logdet = ld2;
    if (loglik) *loglik = ll;
    return GPK_OK;
}

int gpk_acq_dev(gpk_handle* h, const void* d_Xs, long m, int kind, double eta, double par, void* d_out, void* d_mu,
                void* d_var, void* d_best) {
    int rc = require_model(h);
    if (rc) return rc;
    if (!d_Xs || m <= 0) BAD("gpk_acq_dev: need candidates");
    if (kind < GPK_ACQ_NONE || kind > GPK_ACQ_LCB) BAD("gpk_acq_dev: unknown acquisition %d", kind);
    CK(cudaSetDevice(h->device));
    return score_dev(h, (const double*)d_Xs, m, kind, eta, par, (double*)d_out, (double*)d_mu, (double*)d_var,
                     (BestPair*)d_best, nullptr);
}

// Pageable host memory reaches the device slowly through cudaMemcpyAsync (the driver stages it synchronously in small
// pieces): for a 2^20 x 8 candidate batch (67 MB, config C3) the copy takes longer than the scoring.  Large pageable
// batches are therefore copied by the host into two pinned staging buffers and go out by DMA while the next piece is
// being staged.  Pinned / registered caller buffers are used in place.
static bool host_is_pinned(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost;
}

static int ensure_stage(gpk_handle* h, size_t bytes) {
    if (bytes <= h->stage_cap) return GPK_OK;
    for (int i = 0; i < 2; ++i) {
        if (h->stage[i]) CK(cudaFreeHost(h->stage[i]));
        h->stage[i] = nullptr;
    }
    h->stage_cap = 0;
    for (int i = 0; i < 2; ++i) CK(cudaHostAlloc((void**)&h->stage[i], bytes, cudaHostAllocDefault));
    h->stage_cap = bytes;
    return GPK_OK;
}

namespace {
// rows of a host batch -> h->cand, piece by piece on the copy stream; pageable memory goes through two pinned staging
// buffers filled by the host while the previous piece is in flight
struct HostFeeder : Feeder {
    gpk_handle* h;
    const double* Xs;          // first row of the (super-)batch being scored
    long rows, piece;
    bool staged;
    long next = 0;             // rows already enqueued
    int npieces = 0;
    int ready(long lo, long hi, cudaStream_t st) override {
        (void)lo;
        const long d = h->d;
        while (next < hi && next < rows) {
            const int i = npieces;
            const long mc = std::min(piece, rows - next);
            if (int rc = grow_events(h, h->ev_copied, i + 1, cudaEventDisableTiming)) return rc;
            const double* src = Xs + next * d;
            if (staged) {
                if (i >= 2) CK(cudaEventSynchronize(h->ev_copied[i - 2]));   // the DMA out of this staging buffer is done
                memcpy(h->stage[i & 1], src, (size_t)mc * d * 8);
                src = h->stage[i & 1];
            }
            CK(cudaMemcpyAsync(ptr<double>(h->cand) + next * d, src, (size_t)mc * d * 8, cudaMemcpyHostToDevice, h->copy_stream));
            CK(cudaEventRecord(h->ev_copied[i], h->copy_stream));
            next += mc;
            ++npieces;
        }
        if (npieces > 0) CK(cudaStreamWaitEvent(st, h->ev_copied[npieces - 1], 0));
        return GPK_OK;
    }
};
}  // namespace

int gpk_acq(gpk_handle* h, const double* Xs, long m, int kind, double eta, double par, double* out, double* mu,
            double* var, double* best_val, long* best_idx, long* n_negative) {
    int rc = require_model(h);
    if (rc) return rc;
    if (!Xs || m <= 0) BAD("gpk_acq: need candidates");
    if (kind < GPK_ACQ_NONE || kind > GPK_ACQ_LCB) BAD("gpk_acq: unknown acquisition %d", kind);
    CK(cudaSetDevice(h->device));
    const long d = h->d;
    // the device copy of the batch: whole batches up to 1 GiB, larger ones in super-batches of that size
    const long super = std::max<long>(BM, (((long)1 << 30) / (d * 8)) / BM * BM);
    if ((rc = ensure(h, h->cand, (size_t)std::min<long>(m, super) * d * 8))) return rc;
    if (out && (rc = ensure(h, h->out_acq, (size_t)m * 8))) return rc;
    if (mu && (rc = ensure(h, h->out_mu, (size_t)m * 8))) return rc;
    if (var && (rc = ensure(h, h->out_var, (size_t)m * 8))) return rc;
    CK(cudaEventRecord(h->timing.ev[14], h->stream));
    const long piece = std::min<long>(chunk_rows(h), round_up(m, BM));       // one H2D piece per scoring chunk
    const bool small = (size_t)m * d * 8 <= ((size_t)1 << 20);
    const bool staged = !small && !host_is_pinned(Xs);
    if (staged && (rc = ensure_stage(h, (size_t)piece * d * 8))) return rc;
    if (small) {
        CK(cudaMemcpyAsync(h->cand.p, Xs, (size_t)m * d * 8, cudaMemcpyHostToDevice, h->stream));
        rc = score_dev(h, ptr<double>(h->cand), m, kind, eta, par, out ? ptr<double>(h->out_acq) : nullptr,
                       mu ? ptr<double>(h->out_mu) : nullptr, var ? ptr<double>(h->out_var) : nullptr, nullptr, nullptr);
        if (rc) return rc;
    } else {
        for (long base = 0; base < m; base += super) {
            const long rows = std::min(super, m - base);
            // the copy stream starts after everything already queued on the scoring stream (earlier users of h->cand)
            CK(cudaEventRecord(h->ev_order, h->stream));
            CK(cudaStreamWaitEvent(h->copy_stream, h->ev_order, 0));
            if (base > 0) CK(cudaStreamSynchronize(h->copy_stream));     // staging buffers and h->cand are reused
            HostFeeder feeder;
            feeder.h = h; feeder.Xs = Xs + base * d; feeder.rows = rows; feeder.piece = piece; feeder.staged = staged;
            rc = score_dev(h, ptr<double>(h->cand), rows, kind, eta, par, out ? ptr<double>(h->out_acq) : nullptr,
                           mu ? ptr<double>(h->out_mu) : nullptr, var ? ptr<double>(h->out_var) : nullptr, nullptr, nullptr,
                           base, base == 0, 0, &feeder);
            if (rc) return rc;
        }
    }
    if (out) CK(cudaMemcpyAsync(out, h->out_acq.p, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    if (mu) CK(cudaMemcpyAsync(mu, h->out_mu.p, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    if (var) CK(cudaMemcpyAsync(var, h->out_var.p, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    BestPair bp;
    unsigned long long nn = 0;
    CK(cudaMemcpyAsync(&bp, h->best.p, sizeof(bp), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(&nn, h->nneg.p, 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaEventRecord(h->timing.ev[15], h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (best_val) *best_val = bp.val;
    if (best_idx) *best_idx = (long)bp.idx;
    if (n_negative) *n_negative = (long)nn;
    return GPK_OK;
}

// candidates [first, first+count) of the device generator into h->cand (device, count x d)
static int generate_candidates(gpk_handle* h, unsigned long long seed, long first, long count, long n_uniform, int d,
                               const double* lower, const double* upper, const double* incumbent, double scale) {
    int rc;
    if ((rc = ensure(h, h->cand, (size_t)count * d * 8))) return rc;
    if ((rc = ensure(h, h->tmp1, (size_t)3 * d * 8))) return rc;
    double* dl = ptr<double>(h->tmp1);
    CK(cudaMemcpyAsync(dl, lower, (size_t)d * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(dl + d, upper, (size_t)d * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(dl + 2 * d, incumbent, (size_t)d * 8, cudaMemcpyHostToDevice, h->stream));
    const long total = count * ((d + 1) / 2);
    gpk_candidates_kernel<<<(unsigned)((total + 255) / 256), 256, 0, h->stream>>>(seed, first, count, n_uniform, d, dl, dl + d,
                                                                              dl + 2 * d, scale, ptr<double>(h->cand));
    CKL();
    return GPK_OK;
}

int gpk_generate_candidates(gpk_handle* h, unsigned long long seed, long first, long count, long n_uniform, int d,
                            const double* lower, const double* upper, const double* incumbent, double scale,
                            double* out) {
    if (!h) return GPK_BAD_ARG;
    if (!lower || !upper || !incumbent || !out || count <= 0 || d <= 0 || d > GPK_MAX_TERMS || first < 0)
        BAD("gpk_generate_candidates: bad arguments");
    CK(cudaSetDevice(h->device));
    int rc = generate_candidates(h, seed, first, count, n_uniform, d, lower, upper, incumbent, scale);
    if (rc) return rc;
    CK(cudaMemcpyAsync(out, h->cand.p, (size_t)count * d * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_maximize_random(gpk_handle* h, unsigned long long seed, long first, long count, long n_uniform,
                        const double* lower, const double* upper, const double* incumbent, double scale, int kind,
                        double eta, double par, double* best_x, double* best_val, long* best_idx) {
    int rc = require_model(h);
    if (rc) return rc;
    if (!lower || !upper || !incumbent || count <= 0 || first < 0) BAD("gpk_maximize_random: bad arguments");
    if (kind < GPK_ACQ_EI || kind > GPK_ACQ_LCB) BAD("gpk_maximize_random: unknown acquisition %d", kind);
    CK(cudaSetDevice(h->device));
    if ((rc = generate_candidates(h, seed, first, count, n_uniform, h->d, lower, upper, incumbent, scale))) return rc;
    if ((rc = score_dev(h, ptr<double>(h->cand), count, kind, eta, par, nullptr, nullptr, nullptr, nullptr, nullptr)))
        return rc;
    BestPair bp;
    CK(cudaMemcpyAsync(&bp, h->best.p, sizeof(bp), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (bp.idx >= 0 && best_x)
        CK(cudaMemcpy(best_x, ptr<double>(h->cand) + bp.idx * h->d, (size_t)h->d * 8, cudaMemcpyDeviceToHost));
    if (best_val) *best_val = bp.val;
    if (best_idx) *best_idx = bp.idx >= 0 ? (long)(first + bp.idx) : -1;
    return GPK_OK;
}

int gpk_predict(gpk_handle* h, const double* Xs, long m, double* mu, double* var) {
    return gpk_acq(h, Xs, m, GPK_ACQ_NONE, 0.0, 0.0, nullptr, mu, var, nullptr, nullptr, nullptr);
}

int gpk_predict_mean_dev(gpk_handle* h, const void* d_Xs, long m, void* d_mu) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!d_Xs || !d_mu || m <= 0) BAD("gpk_predict_mean_dev: need candidates and mu");
    CK(cudaSetDevice(h->device));
    return predict_mean_dev(h, (const double*)d_Xs, m, (double*)d_mu);
}

int gpk_predict_mean(gpk_handle* h, const double* Xs, long m, double* mu) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!Xs || !mu || m <= 0) BAD("gpk_predict_mean: need candidates and mu");
    CK(cudaSetDevice(h->device));
    if ((rc = ensure(h, h->cand, (size_t)m * h->d * 8))) return rc;
    if ((rc = ensure(h, h->out_mu, (size_t)m * 8))) return rc;
    CK(cudaMemcpyAsync(h->cand.p, Xs, (size_t)m * h->d * 8, cudaMemcpyHostToDevice, h->stream));
    if ((rc = predict_mean_dev(h, ptr<double>(h->cand), m, ptr<double>(h->out_mu)))) return rc;
    CK(cudaMemcpyAsync(mu, h->out_mu.p, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

static int predict_cov_impl(gpk_handle* h, const double* Xs, long m, double* mu, double* cov, int clip) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!Xs || m <= 0 || !mu || !cov) BAD("gpk_predict_cov: need Xs, mu, cov");
    if (m > 16384) BAD("gpk_predict_cov: m = %ld too large for a dense m x m covariance", m);
    CK(cudaSetDevice(h->device));
    if ((rc = build_linv(h))) return rc;
    const long NP = h->NP, mp = round_up(m, BM);
    const int nb = h->nb, mb = (int)(mp / BM);
    if ((rc = ensure(h, h->cand, (size_t)m * h->d * 8))) return rc;
    if ((rc = ensure_score_scratch(h, mp))) return rc;
    bool grew = false;
    if ((rc = ensure(h, h->Vt, (size_t)mp * NP * 8, &grew))) return rc;
    if (grew || h->mapVt_rows != mp) {
        if ((rc = make_map(h, &h->mapVt, h->Vt.p, mp, NP, NP))) return rc;
        h->mapVt_rows = mp;
    }
    if ((rc = ensure(h, h->cov, (size_t)mp * mp * 8))) return rc;
    if ((rc = ensure(h, h->XsT, cov_operand_rows(h, h->d) * mp * 8))) return rc;
    if ((rc = ensure(h, h->out_mu, (size_t)mp * 8))) return rc;
    CK(cudaMemcpyAsync(h->cand.p, Xs, (size_t)m * h->d * 8, cudaMemcpyHostToDevice, h->stream));
    const double* lo = h->has_bounds ? ptr<double>(h->lower) : nullptr;
    const double* up = h->has_bounds ? ptr<double>(h->upper) : nullptr;
    // K* (mp x NP)
    if ((rc = launch_cov_tiles(h, h->stream, ptr<double>(h->Xts), NP, h->n, ptr<double>(h->cand), h->d, m, mp, lo, up,
                               ptr<double>(h->Kstar), NP, 0, false, ptr<double>(h->Xrow), nullptr, nullptr)))
        return rc;
    // K** (mp x mp): candidates against the (scaled, transposed) candidates
    if ((rc = build_cov_operand(h, h->stream, ptr<double>(h->cand), m, h->d, lo, up, ptr<double>(h->XsT), mp))) return rc;
    if ((rc = launch_cov_tiles(h, h->stream, ptr<double>(h->XsT), mp, (int)m, ptr<double>(h->cand), h->d, m, mp, lo, up,
                               ptr<double>(h->cov), mp, 0, false, ptr<double>(h->cand), lo, up)))
        return rc;
    // V^T = (L^-1 K*^T)^T  ->  Vt[cand][i]
    std::vector<GemmJob> jobs;
    for (int ib = nb - 1; ib >= 0; --ib)
        for (int cb = 0; cb < mb; ++cb) jobs.push_back({ib * BM, cb * BM, 0, (ib + 1) * BM, ib * BM, cb * BM, 0, 0});
    const size_t n1 = jobs.size();
    for (int a = 0; a < mb; ++a)
        for (int b = 0; b < mb; ++b) jobs.push_back({a * BM, b * BM, 0, (int)NP, a * BM, b * BM, 0, 0});
    if ((rc = ensure(h, h->tmpjobs, jobs.size() * sizeof(GemmJob)))) return rc;
    CK(cudaMemcpyAsync(h->tmpjobs.p, jobs.data(), jobs.size() * sizeof(GemmJob), cudaMemcpyHostToDevice, h->stream));
    {
        GemmArgs a;
        memset(&a, 0, sizeof(a));
        a.A = ptr<double>(h->P); a.lda = NP;
        a.B = ptr<double>(h->Kstar); a.ldb = NP;
        a.Ct = ptr<double>(h->Vt); a.ldct = NP;
        a.alpha = 1.0;
        a.jobs = ptr<GemmJob>(h->tmpjobs);
        a.job_mode = JOBS_TABLE;
        if ((rc = launch_gemm<EPI_STORE>(h, h->mapP, h->mapKs, a, (int)n1))) return rc;
    }
    // mu = Vt z ; cov = K** - Vt Vt^T
    gpk_rowdot_kernel<<<(unsigned)((mp + 7) / 8), 256, 0, h->stream>>>(ptr<double>(h->Vt), NP, m, (int)NP, 0,
                                                                        ptr<double>(h->Kbuf) + NP * NP,
                                                                        ptr<double>(h->out_mu));
    CKL();
    gpk_mu_finish_kernel<<<(unsigned)((m + 255) / 256), 256, 0, h->stream>>>(ptr<double>(h->out_mu), m, h->mean,
                                                                            h->norm_out, h->y_mean, h->y_std);
    CKL();
    {
        GemmArgs a;
        memset(&a, 0, sizeof(a));
        a.A = ptr<double>(h->Vt); a.lda = NP;
        a.B = ptr<double>(h->Vt); a.ldb = NP;
        a.C = ptr<double>(h->cov); a.ldc = mp;
        a.alpha = -1.0; a.beta = 1;
        a.jobs = ptr<GemmJob>(h->tmpjobs) + n1;
        a.job_mode = JOBS_TABLE;
        if ((rc = launch_gemm<EPI_STORE>(h, h->mapVt, h->mapVt, a, (int)(jobs.size() - n1)))) return rc;
    }
    gpk_cov_finish_kernel<<<(unsigned)((m * m + 255) / 256), 256, 0, h->stream>>>(ptr<double>(h->cov), mp, m,
                                                                                 h->norm_out, h->y_std, clip);
    CKL();
    CK(cudaMemcpyAsync(mu, h->out_mu.p, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpy2DAsync(cov, (size_t)m * 8, h->cov.p, (size_t)mp * 8, (size_t)m * 8, (size_t)m, cudaMemcpyDeviceToHost,
                         h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_predict_cov(gpk_handle* h, const double* Xs, long m, double* mu, double* cov) {
    return predict_cov_impl(h, Xs, m, mu, cov, 1);
}

int gpk_posterior_cov(gpk_handle* h, const double* Xs, long m, double* mu, double* cov) {
    return predict_cov_impl(h, Xs, m, mu, cov, 0);
}

int gpk_predict_grad(gpk_handle* h, const double* Xs, long m, int kind, double eta, double par, double* mu, double* var,
                     double* dmu, double* dvar, double* f, double* df) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!Xs || m <= 0 || !mu || !var || !dmu || !dvar) BAD("gpk_predict_grad: need Xs, mu, var, dmu, dvar");
    if (m > 16384) BAD("gpk_predict_grad: m = %ld too large", m);
    if (kind != GPK_ACQ_NONE && (kind == GPK_ACQ_LOG_EI || kind < GPK_ACQ_NONE || kind > GPK_ACQ_LCB || !f || !df))
        BAD("gpk_predict_grad: acquisition gradients exist for EI, PI, LCB and need f, df");
    CK(cudaSetDevice(h->device));
    if ((rc = build_linv(h))) return rc;
    const long NP = h->NP, mp = round_up(m, BM);
    const int nb = h->nb, mb = (int)(mp / BM), d = h->d;
    if ((rc = ensure(h, h->cand, (size_t)m * d * 8))) return rc;
    if ((rc = ensure_score_scratch(h, mp))) return rc;
    bool grew = false;
    if ((rc = ensure(h, h->Vt, (size_t)mp * NP * 8, &grew))) return rc;
    if (grew || h->mapVt_rows != mp) {
        if ((rc = make_map(h, &h->mapVt, h->Vt.p, mp, NP, NP))) return rc;
        h->mapVt_rows = mp;
    }
    if ((rc = ensure(h, h->cov, (size_t)mp * NP * 8))) return rc;            // Wt = (K^-1 K*^T)^T
    if ((rc = ensure(h, h->alpha, (size_t)NP * 8))) return rc;
    if ((rc = ensure(h, h->out_mu, (size_t)mp * 8))) return rc;
    if ((rc = ensure(h, h->out_var, (size_t)mp * 8))) return rc;
    if ((rc = ensure(h, h->tmp1, (size_t)m * d * 8 * 2))) return rc;
    if ((rc = ensure(h, h->tmp2, (size_t)m * (d + 1) * 8))) return rc;
    CK(cudaMemcpyAsync(h->cand.p, Xs, (size_t)m * d * 8, cudaMemcpyHostToDevice, h->stream));
    // moments through the regular scoring path (same numbers as gpk_predict)
    if ((rc = score_dev(h, ptr<double>(h->cand), m, GPK_ACQ_NONE, 0.0, 0.0, nullptr, ptr<double>(h->out_mu),
                        ptr<double>(h->out_var), nullptr, nullptr)))
        return rc;
    const double* lo = h->has_bounds ? ptr<double>(h->lower) : nullptr;
    const double* up = h->has_bounds ? ptr<double>(h->upper) : nullptr;
    if ((rc = ensure_score_scratch(h, mp))) return rc;       // score_dev may have sized the K* map for a smaller chunk
    // K* again into the first buffer (score_dev may have used either), then Vt = (L^-1 K*^T)^T, Wt = (L^-T V)^T
    if ((rc = launch_cov_tiles(h, h->stream, ptr<double>(h->Xts), NP, h->n, ptr<double>(h->cand), d, m, mp, lo, up,
                               ptr<double>(h->Kstar), NP, 0, false, ptr<double>(h->Xrow), nullptr, nullptr)))
        return rc;
    std::vector<GemmJob> jobs;
    for (int ib = nb - 1; ib >= 0; --ib)
        for (int cb = 0; cb < mb; ++cb) jobs.push_back({ib * BM, cb * BM, 0, (ib + 1) * BM, ib * BM, cb * BM, 0, 0});
    const size_t n1 = jobs.size();
    for (int jb = 0; jb < nb; ++jb)
        for (int cb = 0; cb < mb; ++cb) jobs.push_back({cb * BM, jb * BM, jb * BM, (int)NP, cb * BM, jb * BM, 0, 0});
    if ((rc = ensure(h, h->tmpjobs, jobs.size() * sizeof(GemmJob)))) return rc;
    CK(cudaMemcpyAsync(h->tmpjobs.p, jobs.data(), jobs.size() * sizeof(GemmJob), cudaMemcpyHostToDevice, h->stream));
    {
        GemmArgs a;
        memset(&a, 0, sizeof(a));
        a.A = ptr<double>(h->P); a.lda = NP;
        a.B = ptr<double>(h->Kstar); a.ldb = NP;
        a.Ct = ptr<double>(h->Vt); a.ldct = NP;
        a.alpha = 1.0;
        a.jobs = ptr<GemmJob>(h->tmpjobs);
        a.job_mode = JOBS_TABLE;
        if ((rc = launch_gemm<EPI_STORE>(h, h->mapP, h->mapKs, a, (int)n1))) return rc;
        GemmArgs b;
        memset(&b, 0, sizeof(b));
        b.A = ptr<double>(h->Vt); b.lda = NP;                // Wt[c][j] = sum_{i >= j} Vt[c][i] Q[j][i]
        b.B = ptr<double>(h->Q); b.ldb = NP;
        b.C = ptr<double>(h->cov); b.ldc = NP;
        b.alpha = 1.0;
        b.jobs = ptr<GemmJob>(h->tmpjobs) + n1;
        b.job_mode = JOBS_TABLE;
        if ((rc = launch_gemm<EPI_STORE>(h, h->mapVt, h->mapQ, b, (int)(jobs.size() - n1)))) return rc;
    }
    gpk_rowdot_kernel<<<(unsigned)((NP + 7) / 8), 256, 0, h->stream>>>(ptr<double>(h->Q), NP, NP, (int)NP, 1,
                                                                       ptr<double>(h->Kbuf) + NP * NP,
                                                                       ptr<double>(h->alpha));
    CKL();
    double* d_dmu = ptr<double>(h->tmp1);
    double* d_dvar = d_dmu + m * d;
    {
        auto kern = h->spec.factor.kind == GPK_FACTOR_TASK ? gpk_predict_grad_kernel<GPK_FACTOR_TASK>
                                                           : gpk_predict_grad_kernel<GPK_FACTOR_ENV>;
        kern<<<(unsigned)m, 256, 0, h->stream>>>(h->spec, ptr<double>(h->Xt), NP, h->n, ptr<double>(h->cand), d, lo, up,
                                                 ptr<double>(h->alpha), ptr<double>(h->cov), NP, h->norm_out, h->y_std,
                                                 d_dmu, d_dvar);
    }
    CKL();
    CK(cudaMemcpyAsync(mu, h->out_mu.p, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(var, h->out_var.p, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(dmu, d_dmu, (size_t)m * d * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(dvar, d_dvar, (size_t)m * d * 8, cudaMemcpyDeviceToHost, h->stream));
    if (kind != GPK_ACQ_NONE) {
        double* d_f = ptr<double>(h->tmp2);
        double* d_df = d_f + m;
        gpk_acq_grad_kernel<<<(unsigned)((m * d + 255) / 256), 256, 0, h->stream>>>(
            ptr<double>(h->out_mu), ptr<double>(h->out_var), d_dmu, d_dvar, m, d, kind, eta, par, d_f, d_df);
        CKL();
        CK(cudaMemcpyAsync(f, d_f, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaMemcpyAsync(df, d_df, (size_t)m * d * 8, cudaMemcpyDeviceToHost, h->stream));
    }
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_acq_moments(gpk_handle* h, const double* mu, const double* var, long m, int kind, double eta, double par,
                    double* out, long* n_negative) {
    if (!h) return GPK_BAD_ARG;
    if (!mu || !var || !out || m <= 0) BAD("gpk_acq_moments: need mu, var, out");
    if (kind < GPK_ACQ_EI || kind > GPK_ACQ_LCB) BAD("gpk_acq_moments: unknown acquisition %d", kind);
    CK(cudaSetDevice(h->device));
    int rc;
    if ((rc = ensure(h, h->tmp1, (size_t)m * 8))) return rc;
    if ((rc = ensure(h, h->tmp2, (size_t)m * 8))) return rc;
    if ((rc = ensure(h, h->tmp3, (size_t)m * 8))) return rc;
    if ((rc = ensure(h, h->nneg, 8))) return rc;
    CK(cudaMemcpyAsync(h->tmp1.p, mu, (size_t)m * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->tmp2.p, var, (size_t)m * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemsetAsync(h->nneg.p, 0, 8, h->stream));
    gpk_acq_moments_kernel<<<(unsigned)((m + 255) / 256), 256, 0, h->stream>>>(
        ptr<double>(h->tmp1), ptr<double>(h->tmp2), m, kind, eta, par, ptr<double>(h->tmp3),
        ptr<unsigned long long>(h->nneg));
    CKL();
    unsigned long long nn = 0;
    CK(cudaMemcpyAsync(out, h->tmp3.p, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(&nn, h->nneg.p, 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (n_negative) *n_negative = (long)nn;
    return GPK_OK;
}

int gpk_reduce_models(gpk_handle* h, const double* A, const double* B, int n_models, long m, int mode, double* out1,
                      double* out2) {
    if (!h) return GPK_BAD_ARG;
    if (!A || !out1 || n_models <= 0 || m <= 0 || (mode != 0 && mode != 1)) BAD("gpk_reduce_models: bad arguments");
    if (mode == 1 && (!B || !out2)) BAD("gpk_reduce_models: mode 1 needs B and out2");
    CK(cudaSetDevice(h->device));
    int rc;
    const size_t bytes = (size_t)n_models * m * 8;
    if ((rc = ensure(h, h->tmp1, bytes))) return rc;
    if ((rc = ensure(h, h->tmp2, mode == 1 ? bytes : 8))) return rc;
    if ((rc = ensure(h, h->tmp3, (size_t)m * 16))) return rc;
    CK(cudaMemcpyAsync(h->tmp1.p, A, bytes, cudaMemcpyHostToDevice, h->stream));
    if (mode == 1) CK(cudaMemcpyAsync(h->tmp2.p, B, bytes, cudaMemcpyHostToDevice, h->stream));
    double* o1 = ptr<double>(h->tmp3);
    double* o2 = o1 + m;
    gpk_reduce_models_kernel<<<(unsigned)((m + 255) / 256), 256, 0, h->stream>>>(
        ptr<double>(h->tmp1), mode == 1 ? ptr<double>(h->tmp2) : nullptr, n_models, m, mode, o1, o2);
    CKL();
    CK(cudaMemcpyAsync(out1, o1, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    if (mode == 1) CK(cudaMemcpyAsync(out2, o2, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

// ---------------------------------------------------------------------------------------
// GP-MCMC hyper-parameters on the device (gpk_hyper.cuh; GaussianProcessMCMC.train, gaussian_process_mcmc.py:114-142)
// ---------------------------------------------------------------------------------------
int gpk_set_hyper_model(gpk_handle* h, int n_params, const int* amp_slot, const int* term_param, int n_terms,
                        double mean, double tiny, int prior_kind, const double* prior_par, int n_ls, int n_lr) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_set_hyper_model";
    if (gp_refusal(h)) BAD("%s: %s", who, gp_refusal(h));
    h->hyper.has_model = false;
    if (!h->has_spec) BAD("%s: gpk_set_kernel has not been called", who);
    if (n_params < 1 || n_params + 1 > GPK_HYPER_MAX_DIM || !amp_slot || !term_param)
        BAD("%s: need 1 <= n_params <= %d and the slot table", who, GPK_HYPER_MAX_DIM - 1);
    if (n_terms != h->spec.n_terms) BAD("%s: %d terms in the slot table, the kernel has %d", who, n_terms, h->spec.n_terms);
    if (prior_kind < GPK_PRIOR_NONE || prior_kind > GPK_PRIOR_MTBO) BAD("%s: unknown prior kind %d", who, prior_kind);
    if (prior_kind != GPK_PRIOR_NONE && !prior_par) BAD("%s: the prior needs its constants", who);
    if ((prior_kind == GPK_PRIOR_ENV || prior_kind == GPK_PRIOR_MTBO) && (n_ls < 0 || n_lr < 0))
        BAD("%s: need n_ls >= 0 and n_lr >= 0", who);
    HyperModel m;
    memset(&m, 0, sizeof(m));
    m.family = h->spec.family;
    m.n_terms = n_terms;
    m.n_params = n_params;
    std::vector<int> used(n_params, 0);
    int pa = -1, pb = -1;                     // the log_a and log_b slots; the task slots go straight into m.fp
    for (int p = 0; p < n_params; ++p) {
        if (amp_slot[p] < 0 || amp_slot[p] > 4) BAD("%s: slot kind %d of parameter %d is not 0..4", who, amp_slot[p], p);
        if (amp_slot[p] == 4) {
            if (m.n_fp == GPK_MAX_TASKS * (GPK_MAX_TASKS + 1) / 2) BAD("%s: too many task slots", who);
            m.fp[m.n_fp++] = (unsigned char)p;
        }
        m.amp[p] = amp_slot[p] == 1 ? 1 : 0;
        int* env_p = amp_slot[p] == 2 ? &pa : amp_slot[p] == 3 ? &pb : nullptr;
        if (env_p) {
            if (*env_p >= 0) BAD("%s: more than one log_%c slot", who, amp_slot[p] == 2 ? 'a' : 'b');
            *env_p = p;
        }
    }
    const KFactor& f = h->spec.factor;
    if ((pa >= 0) != (pb >= 0) || (pa >= 0) != (f.kind == GPK_FACTOR_ENV))
        BAD("%s: the log_a / log_b slots must match the kernel's environment factor", who);
    const int n_kt = f.kind == GPK_FACTOR_TASK ? f.n_tasks * (f.n_tasks + 1) / 2 : 0;
    if (m.n_fp != n_kt) BAD("%s: %d task slots, the kernel's task factor has %d entries", who, m.n_fp, n_kt);
    if (pa >= 0) { m.fp[0] = (unsigned char)pa; m.fp[1] = (unsigned char)pb; m.n_fp = 2; }
    m.f_kind = f.kind;
    m.f_axis = f.axis;
    m.f_n_tasks = f.n_tasks;
    for (int t = 0; t < n_terms; ++t) {
        const int p = term_param[t];
        if (p < 0 || p >= n_params || amp_slot[p] != 0) BAD("%s: term %d is not set by a metric slot", who, t);
        m.axis[t] = h->spec.axis[t];
        m.last[t] = h->spec.last[t];
        m.term_param[t] = p;
        used[p] = 1;
    }
    for (int p = 0; p < n_params; ++p)
        if (amp_slot[p] == 0 && !used[p]) BAD("%s: metric slot %d sets no term", who, p);
    m.mean = mean;
    m.tiny = tiny;
    m.prior = prior_kind;
    m.n_ls = n_ls;
    m.n_lr = n_lr;
    if (prior_kind != GPK_PRIOR_NONE) {
        m.ln_sigma = prior_par[0]; m.ln_loc = prior_par[1]; m.th_lo = prior_par[2]; m.th_hi = prior_par[3];
        m.hs_scale = prior_par[4]; m.nrm_sigma = prior_par[5]; m.nrm_mean = prior_par[6];
    }
    h->hyper.model = m;
    h->hyper.has_model = true;
    return GPK_OK;
}

namespace {
// the preconditions of the hyper-parameter entry points; blocked: the gpk_*_blocked ones (n up to
// GPK_HYPER_BLOCKED_MAX_N)
int hyper_check(gpk_handle* h, int dim, const char* who, bool blocked) {
    int rc = require(h, true, true, false);
    if (rc) return rc;
    if (!h->hyper.has_model) BAD("%s: gpk_set_hyper_model has not been called", who);
    const HyperModel& m = h->hyper.model;
    const KFactor& f = h->spec.factor;
    if (m.f_kind != f.kind || m.f_axis != f.axis || m.f_n_tasks != f.n_tasks)
        BAD("%s: the kernel structure changed since gpk_set_hyper_model", who);
    if ((rc = factor_data_check(h, h->d, &h->col_tasks, who))) return rc;
    if (m.n_terms != h->spec.n_terms || m.family != h->spec.family)
        BAD("%s: the kernel structure changed since gpk_set_hyper_model", who);
    for (int t = 0; t < m.n_terms; ++t) {
        if (m.axis[t] != h->spec.axis[t] || m.last[t] != h->spec.last[t])
            BAD("%s: the kernel structure changed since gpk_set_hyper_model", who);
        if (m.axis[t] >= h->d) BAD("%s: kernel axis %d >= d = %d", who, m.axis[t], h->d);
    }
    if (!blocked && h->n > GPK_HYPER_MAX_N)
        BAD("%s: n = %d exceeds GPK_HYPER_MAX_N = %d", who, h->n, GPK_HYPER_MAX_N);
    if (blocked && (h->n < 2 || h->n > GPK_HYPER_BLOCKED_MAX_N))
        BAD("%s: need 2 <= n <= GPK_HYPER_BLOCKED_MAX_N = %d (n = %d)", who, GPK_HYPER_BLOCKED_MAX_N, h->n);
    if (dim != m.n_params + 1) BAD("%s: dim = %d, the slot table needs %d", who, dim, m.n_params + 1);
    CK(cudaSetDevice(h->device));
    return GPK_OK;
}

// the preconditions of gpk_hyper_lnpost / gpk_sample_hypers, and the kernels' shared-memory opt-in
int hyper_ready(gpk_handle* h, int dim, const char* who) {
    int rc = hyper_check(h, dim, who, false);
    if (rc) return rc;
    const int smem = (int)(gpk_hy_smem_doubles(h->n) * 8);
    CK(cudaFuncSetAttribute(gpk_hy_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(gpk_hy_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    return GPK_OK;
}
}  // namespace

int gpk_hyper_lnpost(gpk_handle* h, const double* theta, int count, int dim, double* ll, double* lp) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_hyper_lnpost";
    if (count < 1 || !theta || !ll || !lp) BAD("%s: need count >= 1, theta, ll and lp", who);
    int rc = hyper_ready(h, dim, who);
    if (rc) return rc;
    const size_t nT = (size_t)count * dim;
    if ((rc = ensure(h, h->hyper.buf, (nT + 2 * (size_t)count) * 8))) return rc;
    double* dT = ptr<double>(h->hyper.buf);
    double* dll = dT + nT;
    double* dlp = dll + count;
    CK(cudaMemcpyAsync(dT, theta, nT * 8, cudaMemcpyHostToDevice, h->stream));
    gpk_hy_eval_kernel<<<count, GPK_HY_THREADS, gpk_hy_smem_doubles(h->n) * 8, h->stream>>>(
        h->hyper.model, ptr<double>(h->Xt), h->NP, ptr<double>(h->y), h->n, dT, dll, dlp, nullptr);
    CKL();
    CK(cudaMemcpyAsync(ll, dll, (size_t)count * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(lp, dlp, (size_t)count * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

extern "C++" {                     // the shared drivers are templates over the launches they enqueue
namespace {
// the argument checks gpk_sample_hypers and gpk_sample_hypers_blocked share (before their hyper-model checks)
int hy_args(gpk_handle* h, const char* who, const double* p0, int nwalkers, int dim, int steps, const double* pos,
            const double* lnpost) {
    if (!p0 || !pos || !lnpost) BAD("%s: need p0, pos and lnpost", who);
    if (nwalkers % 2 != 0 || nwalkers < 2 * dim || nwalkers < 2)
        BAD("%s: need an even number of walkers >= 2 dim (nwalkers = %d, dim = %d)", who, nwalkers, dim);
    if (steps < 0) BAD("%s: need steps >= 0", who);
    return GPK_OK;
}

// One EnsembleSampler.run_mcmc on the device, shared by both samplers: P (nwalkers x dim), L (nwalkers) and the accept
// counts (nwalkers) contiguous in h->hyper.buf, so that one copy brings the run back, then `extra` doubles for the caller.
// score(P, L, extra) enqueues the initial log-posteriors, half(s, half, P, L, acc, extra) one half-step; no host
// synchronisation until the final copy.
template <class Score, class Half>
int hy_run(gpk_handle* h, const double* p0, int nwalkers, int dim, int steps, size_t extra, Score score, Half half,
           double* pos, double* lnpost, long* n_accepted) {
    static_assert(sizeof(long) == sizeof(long long) && sizeof(long long) == sizeof(double),
                  "the accept counts travel in the walkers' transfer");
    const size_t nP = (size_t)nwalkers * dim, total = nP + 2 * (size_t)nwalkers;
    int rc = ensure(h, h->hyper.buf, (total + extra) * 8);
    if (rc) return rc;
    double* P = ptr<double>(h->hyper.buf);
    double* L = P + nP;
    long long* acc = (long long*)(L + nwalkers);
    double* ex = P + total;
    CK(cudaMemcpyAsync(P, p0, nP * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemsetAsync(acc, 0, (size_t)nwalkers * 8, h->stream));
    if ((rc = score(P, L, ex))) return rc;
    for (int s = 0; s < steps; ++s)
        for (int hf = 0; hf < 2; ++hf)
            if ((rc = half(s, hf, P, L, acc, ex))) return rc;
    std::vector<double> out(total);
    CK(cudaMemcpyAsync(out.data(), P, total * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    memcpy(pos, out.data(), nP * 8);
    memcpy(lnpost, out.data() + nP, (size_t)nwalkers * 8);
    if (n_accepted) memcpy(n_accepted, out.data() + nP + nwalkers, (size_t)nwalkers * 8);
    return GPK_OK;
}

// the argument checks gpk_optimize_hypers and gpk_optimize_hypers_blocked share (before their hyper-model checks)
int ho_args(gpk_handle* h, const char* who, const double* p0, const double* theta, int dim, int maxcor, int maxiter,
            long maxfun, double eps, int maxls) {
    if (!p0 || !theta) BAD("%s: need p0 and theta", who);
    if (dim < 1 || dim > GPK_HYPER_MAX_DIM) BAD("%s: need 1 <= dim <= %d (dim = %d)", who, GPK_HYPER_MAX_DIM, dim);
    for (int j = 0; j < dim; ++j)
        if (!std::isfinite(p0[j])) BAD("%s: p0[%d] = %g is not finite", who, j, p0[j]);
    if (maxcor < 1 || maxcor > GPK_LB_MAX_COR) BAD("%s: need 1 <= maxcor <= %d (maxcor = %d)", who, GPK_LB_MAX_COR, maxcor);
    if (maxls < 1) BAD("%s: need maxls >= 1 (maxls = %d)", who, maxls);
    if (!(eps > 0.0)) BAD("%s: need eps > 0 (eps = %g)", who, eps);
    if (maxiter < 1 || maxfun < 1) BAD("%s: need maxiter >= 1 and maxfun >= 1 (%d, %ld)", who, maxiter, maxfun);
    return GPK_OK;
}

// One L-BFGS-B run on the device, shared by both optimisers: the state record, the work buffer and `extra` doubles for
// the caller in h->hyper.buf; round(dst, work, q, extra) enqueues one round; the host reads the status once per
// GPK_HO_CHUNK rounds.
template <class Round>
int ho_run(gpk_handle* h, const double* p0, int dim, int maxcor, int maxiter, long maxfun, double ftol, double pgtol,
           double eps, int maxls, size_t extra, Round round, double* theta, double* f, int* nit, long* nfev,
           int* status) {
    // the state record, then the work buffer
    const size_t nst = (sizeof(HOState) + 7) / 8, nw = (size_t)gpk_ho_work_doubles(dim, maxcor);
    int rc = ensure(h, h->hyper.buf, (nst + nw + extra) * 8);
    if (rc) return rc;
    HOState* dst = ptr<HOState>(h->hyper.buf);
    double* work = ptr<double>(h->hyper.buf) + nst;
    const HOWork w = gpk_ho_work(work, dim, maxcor);
    HOState s0;
    memset(&s0, 0, sizeof(s0));
    s0.status = GPK_LB_RUNNING;
    s0.phase = GPK_HO_START;
    HOParams q;
    q.maxcor = maxcor; q.maxiter = maxiter; q.maxls = maxls; q.maxfun = maxfun;
    q.tol = (ftol / GPK_LB_DBL_EPS) * GPK_LB_DBL_EPS;      // scipy's factr = ftol / eps, L-BFGS-B's tol = factr eps
    q.pgtol = pgtol; q.eps = eps;
    CK(cudaMemcpyAsync(dst, &s0, sizeof(s0), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(w.xt, p0, (size_t)dim * 8, cudaMemcpyHostToDevice, h->stream));
    int* pst = reinterpret_cast<int*>(h->pin);
    for (;;) {
        for (int r = 0; r < GPK_HO_CHUNK; ++r)
            if ((rc = round(dst, work, q, work + nw))) return rc;
        CK(cudaMemcpyAsync(pst, &dst->status, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        if (*pst != GPK_LB_RUNNING) break;
    }
    HOState s;
    CK(cudaMemcpyAsync(&s, dst, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(theta, w.x, (size_t)dim * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (f) *f = s.f;
    if (nit) *nit = s.nit;
    if (nfev) *nfev = (long)s.nfev;
    if (status) *status = s.status;
    return GPK_OK;
}
}  // namespace
}  // extern "C++"

int gpk_sample_hypers(gpk_handle* h, const double* p0, int nwalkers, int dim, int steps, unsigned long long seed,
                      double* pos, double* lnpost, long* n_accepted) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_sample_hypers";
    int rc = hy_args(h, who, p0, nwalkers, dim, steps, pos, lnpost);
    if (rc) return rc;
    if ((rc = hyper_ready(h, dim, who))) return rc;
    const size_t smem = gpk_hy_smem_doubles(h->n) * 8;
    const double* Xt = ptr<double>(h->Xt);
    const double* y = ptr<double>(h->y);
    auto score = [&](double* P, double* L, double*) -> int {
        gpk_hy_eval_kernel<<<nwalkers, GPK_HY_THREADS, smem, h->stream>>>(h->hyper.model, Xt, h->NP, y, h->n, P, nullptr,
                                                                          nullptr, L);
        CKL();
        return GPK_OK;
    };
    auto half = [&](int s, int hf, double* P, double* L, long long* acc, double*) -> int {
        gpk_hy_step_kernel<<<nwalkers / 2, GPK_HY_THREADS, smem, h->stream>>>(h->hyper.model, Xt, h->NP, y, h->n, nwalkers,
                                                                            s, hf, seed, P, L, acc);
        CKL();
        return GPK_OK;
    };
    return hy_run(h, p0, nwalkers, dim, steps, 0, score, half, pos, lnpost, n_accepted);
}

// GaussianProcess.optimize on the device (gpk_hyperopt.cuh; gaussian_process.py:193-219)
int gpk_optimize_hypers(gpk_handle* h, const double* p0, int dim, int maxcor, int maxiter, long maxfun, double ftol,
                        double pgtol, double eps, int maxls, double* theta, double* f, int* nit, long* nfev,
                        int* status) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_optimize_hypers";
    int rc = ho_args(h, who, p0, theta, dim, maxcor, maxiter, maxfun, eps, maxls);
    if (rc) return rc;
    if ((rc = hyper_ready(h, dim, who))) return rc;
    const size_t smem = gpk_hy_smem_doubles(h->n) * 8;
    CK(cudaFuncSetAttribute(gpk_ho_round_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const double* Xt = ptr<double>(h->Xt);
    const double* y = ptr<double>(h->y);
    auto round = [&](HOState* dst, double* work, const HOParams& q, double*) -> int {
        gpk_ho_round_kernel<<<dim + 1, GPK_HY_THREADS, smem, h->stream>>>(h->hyper.model, Xt, h->NP, y, h->n, q, work, dst);
        CKL();
        return GPK_OK;
    };
    return ho_run(h, p0, dim, maxcor, maxiter, maxfun, ftol, pgtol, eps, maxls, 0, round, theta, f, nit, nfev, status);
}

// ---------------------------------------------------------------------------------------
// The same three at large N (gpk_hyper_blocked.cuh): every theta's matrix in HBM, factored by the fit's diagonal-block
// kernel and tile engine with job tables that span the chunk
// ---------------------------------------------------------------------------------------
namespace {
// One chunk of B thetas, in HBM in buf: B matrices (one stacked array, tensor map mapA), B P strips (mapP), B HBPar,
// B x nb block log-sums, B status words, the chunk's skip word and the job tables.  Each blocked call holds its own, so
// the buffer (it can take most of the budget) is released before the call returns, whatever its outcome.
struct HBChunk {
    DevBuf buf;
    GemmJob* jobs = nullptr;
    int B = 0;
    double* A = nullptr;
    double* P = nullptr;
    HBPar* par = nullptr;
    double* logpart = nullptr;
    int* st = nullptr;
    int* skip = nullptr;
    CUtensorMap mapA, mapP;
    std::vector<Range> panel_r, update_r;       // per step k: the jobs of matrix 0; matrix b follows at + b cnt
};

// The chunk size under the handle's byte budget for `count` thetas, its buffer, tensor maps and job tables.  The jobs of
// step k are matrix-major (matrix b's jobs are rows b R of the stacked array), so a chunk of B' <= B matrices launches
// the first B' cnt of them.
int hb_reserve(gpk_handle* h, int count, const char* who, HBChunk* c) {
    const int n = h->n, nb = gpk_hb_nb(n);
    const long NP = (long)nb * HB_T, R = NP + HB_T;
    const long per = gpk_hb_theta_bytes(n);
    const long fit = h->hyper.batch_bytes / per;
    if (fit < 1)
        BAD("%s: one theta needs %ld bytes at n = %d, more than hyper_batch_bytes = %ld", who, per, n,
            h->hyper.batch_bytes);
    c->B = (int)std::min<long>(std::min<long>(fit, count), 32768);
    const int B = c->B;
    const size_t nA = (size_t)B * R * NP, nPs = (size_t)B * HB_T * NP, npar = (size_t)B * ((sizeof(HBPar) + 7) / 8);
    const size_t nlog = (size_t)B * nb, nst = ((size_t)B + 2) / 2;
    if ((size_t)B * R > (size_t)INT_MAX) BAD("%s: the chunk's rows exceed the job table's range", who);
    // the job tables
    std::vector<GemmJob> jobs;
    c->panel_r.assign(nb, Range());
    c->update_r.assign(nb, Range());
    for (int k = 0; k < nb; ++k) {
        c->panel_r[k].off = (int)jobs.size();
        for (int b = 0; b < B; ++b) {
            const int r0 = (int)(b * R), p0 = b * HB_T;
            for (int i = k + 1; i <= nb; ++i)
                jobs.push_back({r0 + i * HB_T, p0, k * HB_T, (k + 1) * HB_T, r0 + i * HB_T, k * HB_T, 0, 0});
            if (b == 0) c->panel_r[k].cnt = (int)jobs.size() - c->panel_r[k].off;
        }
        c->update_r[k].off = (int)jobs.size();
        for (int b = 0; b < B; ++b) {
            const int r0 = (int)(b * R);
            for (int j = k + 1; j < nb; ++j)
                for (int i = j; i <= nb; ++i)
                    jobs.push_back({r0 + i * HB_T, r0 + j * HB_T, k * HB_T, (k + 1) * HB_T, r0 + i * HB_T, j * HB_T, 0, 0});
            if (b == 0) c->update_r[k].cnt = (int)jobs.size() - c->update_r[k].off;
        }
    }
    const size_t njob = (jobs.size() * sizeof(GemmJob) + 7) / 8;
    int rc = ensure(h, c->buf, (nA + nPs + npar + nlog + nst + njob) * 8);
    if (rc) return rc;
    c->A = ptr<double>(c->buf);
    c->P = c->A + nA;
    c->par = reinterpret_cast<HBPar*>(c->P + nPs);
    c->logpart = c->P + nPs + npar;
    c->st = reinterpret_cast<int*>(c->logpart + nlog);
    c->skip = c->st + B;
    c->jobs = reinterpret_cast<GemmJob*>(c->logpart + nlog + nst);
    if (!jobs.empty())
        CK(cudaMemcpyAsync(c->jobs, jobs.data(), jobs.size() * sizeof(GemmJob), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemsetAsync(c->skip, 0, sizeof(int), h->stream));
    CK(cudaStreamSynchronize(h->stream));         // the host job vector goes out of scope
    if ((rc = make_map(h, &c->mapA, c->A, (long)B * R, NP, NP))) return rc;
    if ((rc = make_map(h, &c->mapP, c->P, (long)B * HB_T, NP, NP))) return rc;
    return GPK_OK;
}

// The log-posterior parts of the count thetas T (device, count x dim) in chunks of c.B, enqueued on the handle's stream
// without a host synchronisation; ll / lp / post / fobj (device, count each) may be NULL.  skip (device, may be NULL:
// the chunk's own zero word): non-zero makes every launch return at once.
int hb_score(gpk_handle* h, const HBChunk& c, const double* T, int count, const int* skip, double* ll, double* lp,
             double* post, double* fobj) {
    const int n = h->n, nb = gpk_hb_nb(n), D = h->hyper.model.n_params + 1;
    const long NP = (long)nb * HB_T, R = NP + HB_T;
    if (!skip) skip = c.skip;
    auto at = [](double* p, int off) { return p ? p + off : nullptr; };
    int rc;
    for (int c0 = 0; c0 < count; c0 += c.B) {
        const int B = std::min(c.B, count - c0);
        // the P strips: zero right of the diagonal 16-blocks, where the diagonal kernel never stores
        CK(cudaMemsetAsync(c.P, 0, (size_t)B * HB_T * NP * 8, h->stream));
        gpk_hb_prep_kernel<<<B, 32, 0, h->stream>>>(h->hyper.model, T + (size_t)c0 * D, skip, c.par, c.st);
        CKL();
        gpk_hb_build_kernel<<<dim3(nb, nb + 1, B), 256, 0, h->stream>>>(h->hyper.model, ptr<double>(h->Xt), h->NP,
                                                                        ptr<double>(h->y), n, c.par, c.A);
        CKL();
        for (int k = 0; k < nb; ++k) {
            for (int b = 0; b < B; ++b) {
                // the fit's diagonal kernel on matrix b; it stores inv(L_kk) at P + k 128 ldp + k 128, which the
                // offset base puts at row 0, column k 128 of matrix b's strip
                double* Pb = reinterpret_cast<double*>(reinterpret_cast<uintptr_t>(c.P + (size_t)b * HB_T * NP) -
                                                       (uintptr_t)k * HB_T * NP * 8);
                gpk_potrf_diag_dmma_kernel<<<1, 256, DIAG_SMEM, h->stream>>>(c.A + (size_t)b * R * NP, NP, k, Pb,
                                                                             nullptr, NP, c.st + b,
                                                                             c.logpart + (size_t)b * nb, nullptr);
                CKL();
            }
            GemmArgs a;
            memset(&a, 0, sizeof(a));
            a.A = c.A; a.lda = NP;
            a.B = c.P; a.ldb = NP;
            a.C = c.A; a.ldc = NP;
            a.alpha = 1.0; a.beta = 0;
            a.job_mode = JOBS_TABLE;
            a.status = skip;
            a.jobs = c.jobs + c.panel_r[k].off;
            if ((rc = launch_gemm<EPI_STORE>(h, c.mapA, c.mapP, a, B * c.panel_r[k].cnt))) return rc;
            if (c.update_r[k].cnt > 0) {
                a.B = c.A;
                a.alpha = -1.0; a.beta = 1;
                a.jobs = c.jobs + c.update_r[k].off;
                if ((rc = launch_gemm<EPI_STORE>(h, c.mapA, c.mapA, a, B * c.update_r[k].cnt))) return rc;
            }
        }
        gpk_hb_finish_kernel<<<B, GPK_HY_THREADS, 0, h->stream>>>(h->hyper.model, n, c.par, c.A, c.logpart, c.st, at(ll, c0),
                                                                  at(lp, c0), at(post, c0), at(fobj, c0));
        CKL();
    }
    return GPK_OK;
}
}  // namespace

int gpk_hyper_lnpost_blocked(gpk_handle* h, const double* theta, int count, int dim, double* ll, double* lp) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_hyper_lnpost_blocked";
    if (count < 1 || !theta || !ll || !lp) BAD("%s: need count >= 1, theta, ll and lp", who);
    int rc = hyper_check(h, dim, who, true);
    if (rc) return rc;
    HBChunk c;
    if ((rc = hb_reserve(h, count, who, &c))) return rc;
    const size_t nT = (size_t)count * dim;
    if ((rc = ensure(h, h->hyper.buf, (nT + 2 * (size_t)count) * 8))) return rc;
    double* dT = ptr<double>(h->hyper.buf);
    double* dll = dT + nT;
    double* dlp = dll + count;
    CK(cudaMemcpyAsync(dT, theta, nT * 8, cudaMemcpyHostToDevice, h->stream));
    if ((rc = hb_score(h, c, dT, count, nullptr, dll, dlp, nullptr, nullptr))) return rc;
    CK(cudaMemcpyAsync(ll, dll, (size_t)count * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(lp, dlp, (size_t)count * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_sample_hypers_blocked(gpk_handle* h, const double* p0, int nwalkers, int dim, int steps, unsigned long long seed,
                              double* pos, double* lnpost, long* n_accepted) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_sample_hypers_blocked";
    int rc = hy_args(h, who, p0, nwalkers, dim, steps, pos, lnpost);
    if (rc) return rc;
    if ((rc = hyper_check(h, dim, who, true))) return rc;
    HBChunk c;
    if ((rc = hb_reserve(h, nwalkers, who, &c))) return rc;
    // after the walkers: the proposals Q (nwalkers / 2 x dim) and their log-posteriors V
    const int hb = nwalkers / 2;
    auto score = [&](double* P, double* L, double*) {
        return hb_score(h, c, P, nwalkers, nullptr, nullptr, nullptr, L, nullptr);
    };
    auto half = [&](int s, int hf, double* P, double* L, long long* acc, double* Q) -> int {
        double* V = Q + (size_t)hb * dim;
        gpk_hb_propose_kernel<<<hb, 32, 0, h->stream>>>(dim, nwalkers, s, hf, seed, P, Q);
        CKL();
        int r = hb_score(h, c, Q, hb, nullptr, nullptr, nullptr, V, nullptr);
        if (r) return r;
        gpk_hb_accept_kernel<<<hb, 32, 0, h->stream>>>(dim, nwalkers, s, hf, seed, Q, V, P, L, acc);
        CKL();
        return GPK_OK;
    };
    return hy_run(h, p0, nwalkers, dim, steps, (size_t)hb * dim + hb, score, half, pos, lnpost, n_accepted);
}

int gpk_optimize_hypers_blocked(gpk_handle* h, const double* p0, int dim, int maxcor, int maxiter, long maxfun,
                                double ftol, double pgtol, double eps, int maxls, double* theta, double* f, int* nit,
                                long* nfev, int* status) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_optimize_hypers_blocked";
    int rc = ho_args(h, who, p0, theta, dim, maxcor, maxiter, maxfun, eps, maxls);
    if (rc) return rc;
    if ((rc = hyper_check(h, dim, who, true))) return rc;
    HBChunk c;
    if ((rc = hb_reserve(h, dim + 1, who, &c))) return rc;
    // after the work buffer: the stencil's thetas ((dim + 1) x dim); the chunk's skip word rises with the final status
    auto round = [&](HOState* dst, double* work, const HOParams& q, double* T) -> int {
        gpk_hb_stencil_kernel<<<dim + 1, 32, 0, h->stream>>>(dim, q, work, dst, T);
        CKL();
        const HOWork w = gpk_ho_work(work, dim, q.maxcor);
        int r = hb_score(h, c, T, dim + 1, c.skip, nullptr, nullptr, nullptr, w.fv);
        if (r) return r;
        gpk_hb_update_ho_kernel<<<1, 32, 0, h->stream>>>(dim, q, work, dst, c.skip);
        CKL();
        return GPK_OK;
    };
    return ho_run(h, p0, dim, maxcor, maxiter, maxfun, ftol, pgtol, eps, maxls, (size_t)(dim + 1) * dim, round, theta,
                  f, nit, nfev, status);
}

// ---------------------------------------------------------------------------------------
// Bayesian linear regression (gpk_blr.cuh; robo/models/bayesian_linear_regression.py)
// ---------------------------------------------------------------------------------------
int gpk_blr_set_data(gpk_handle* h, const double* X, const double* y, int n, int d, int basis, const double* prior_par) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_blr_set_data";
    int rc = claim_model(h, MODEL_BLR, who);
    if (rc) return rc;
    if (!X || !y || !prior_par || n <= 0 || d <= 0) BAD("%s: need X, y, prior_par, n > 0, d > 0", who);
    if (basis < GPK_BLR_LINEAR || basis > GPK_BLR_NONE) BAD("%s: unknown basis %d", who, basis);
    const long F = basis == GPK_BLR_LINEAR ? (long)d + 1 : basis == GPK_BLR_QUADRATIC ? 2L * d + 1 : d;
    if (F > GPK_BLR_MAX_F)
        BAD("%s: %ld features (d = %d) exceed GPK_BLR_MAX_F = %d", who, F, d, GPK_BLR_MAX_F);
    CK(cudaSetDevice(h->device));
    h->model = MODEL_BLR;
    h->blr.fitted = false;
    h->n = n; h->d = d; h->blr.F = (int)F; h->blr.basis = basis;
    h->blr.prior.ln_sigma = prior_par[0]; h->blr.prior.ln_loc = prior_par[1]; h->blr.prior.hs_scale = prior_par[2];
    if ((rc = ensure(h, h->blr.data, ((size_t)n * F + n + F * F + F) * 8))) return rc;
    if ((rc = ensure(h, h->cand, (size_t)n * d * 8))) return rc;
    CK(cudaMemcpyAsync(h->cand.p, X, (size_t)n * d * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(blr_y(h), y, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
    gpk_blr_phi_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(ptr<double>(h->cand), n, d, (int)F, basis, blr_phi(h));
    CKL();
    gpk_blr_gram_kernel<<<(unsigned)(F * F + F), 256, 0, h->stream>>>(blr_phi(h), blr_y(h), n, (int)F, blr_G(h), blr_b(h));
    CKL();
    CK(cudaStreamSynchronize(h->stream));     // host buffers are caller-owned: done with them
    h->has_data = true;
    return GPK_OK;
}

int gpk_blr_lnpost(gpk_handle* h, const double* thetas, int count, double* out) {
    const char* who = "gpk_blr_lnpost";
    int rc = blr_ready(h, who);
    if (rc) return rc;
    if (count < 1 || !thetas || !out) BAD("%s: need count >= 1, thetas and out", who);
    if ((rc = ensure(h, h->blr.work, (size_t)count * 3 * 8))) return rc;
    double* dT = ptr<double>(h->blr.work);
    double* dv = dT + 2 * (size_t)count;
    CK(cudaMemcpyAsync(dT, thetas, (size_t)count * 2 * 8, cudaMemcpyHostToDevice, h->stream));
    gpk_blr_eval_kernel<<<count, GPK_BLR_THREADS, gpk_blr_smem_doubles(h->blr.F) * 8, h->stream>>>(
        blr_phi(h), blr_y(h), blr_G(h), blr_b(h), h->n, h->blr.F, h->blr.prior, dT, dv);
    CKL();
    CK(cudaMemcpyAsync(out, dv, (size_t)count * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_blr_sample(gpk_handle* h, unsigned long long seed, int nwalkers, const double* p0, int steps, double* pos,
                   double* lnpost, long* n_accepted) {
    static_assert(sizeof(long) == sizeof(long long) && sizeof(long long) == sizeof(double),
                  "the accept counts travel in the walkers' transfer");
    const char* who = "gpk_blr_sample";
    int rc = blr_ready(h, who);
    if (rc) return rc;
    if (!p0 || !pos || !lnpost) BAD("%s: need p0, pos and lnpost", who);
    if (nwalkers % 2 != 0 || nwalkers < 4)
        BAD("%s: need an even number of walkers >= 4 (twice the dimension 2; nwalkers = %d)", who, nwalkers);
    if (steps < 0) BAD("%s: need steps >= 0", who);
    // P (nwalkers x 2), L (nwalkers), accept counts (nwalkers): contiguous, so that one copy brings the run back
    const size_t nP = 2 * (size_t)nwalkers, total = nP + 2 * (size_t)nwalkers;
    if ((rc = ensure(h, h->blr.work, total * 8))) return rc;
    double* P = ptr<double>(h->blr.work);
    double* L = P + nP;
    long long* acc = (long long*)(L + nwalkers);
    const size_t smem = gpk_blr_smem_doubles(h->blr.F) * 8;
    CK(cudaMemcpyAsync(P, p0, nP * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemsetAsync(acc, 0, (size_t)nwalkers * 8, h->stream));
    gpk_blr_eval_kernel<<<nwalkers, GPK_BLR_THREADS, smem, h->stream>>>(blr_phi(h), blr_y(h), blr_G(h), blr_b(h), h->n,
                                                                       h->blr.F, h->blr.prior, P, L);
    CKL();
    for (int s = 0; s < steps; ++s)
        for (int half = 0; half < 2; ++half) {
            gpk_blr_step_kernel<<<nwalkers / 2, GPK_BLR_THREADS, smem, h->stream>>>(
                blr_phi(h), blr_y(h), blr_G(h), blr_b(h), h->n, h->blr.F, h->blr.prior, nwalkers, s, half, seed, P, L, acc);
            CKL();
        }
    std::vector<double> out(total);
    CK(cudaMemcpyAsync(out.data(), P, total * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    memcpy(pos, out.data(), nP * 8);
    memcpy(lnpost, out.data() + nP, (size_t)nwalkers * 8);
    if (n_accepted) memcpy(n_accepted, out.data() + nP + nwalkers, (size_t)nwalkers * 8);
    return GPK_OK;
}

}  // extern "C"

namespace {
// gpk_blr_fit's work, shared with gpk_dngo_fit: the k weight posteriors of hypers on a handle past blr_ready
int blr_fit(gpk_handle* h, const double* hypers, int k, const char* who) {
    int rc;
    if (!hypers || k < 1) BAD("%s: need hypers and k >= 1", who);
    h->blr.fitted = false;
    const int F = h->blr.F;
    const BlrPost L(k, F);
    if ((rc = ensure(h, h->blr.post, L.total))) return rc;
    if ((rc = ensure(h, h->blr.work, (size_t)k * 2 * 8))) return rc;
    double* post = ptr<double>(h->blr.post);
    double* dH = ptr<double>(h->blr.work);
    CK(cudaMemcpyAsync(dH, hypers, (size_t)k * 2 * 8, cudaMemcpyHostToDevice, h->stream));
    gpk_blr_fit_kernel<<<k, GPK_BLR_THREADS, (gpk_blr_smem_doubles(F) + (size_t)F * F) * 8, h->stream>>>(
        blr_G(h), blr_b(h), F, dH, post + L.M, post + L.Li, post + L.S, post + L.ib, (int*)(post + L.fail));
    CKL();
    std::vector<int> fail(k);
    CK(cudaMemcpyAsync(fail.data(), post + L.fail, (size_t)k * 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < k; ++i)
        if (fail[i]) {
            set_err(h, "%s: A = beta Phi^T Phi + alpha I of hypers %d (alpha = %g, beta = %g) is not positive definite",
                    who, i, hypers[2 * i], hypers[2 * i + 1]);
            return GPK_NOT_PD;
        }
    h->blr.k = k;
    h->blr.fitted = true;
    return GPK_OK;
}
}  // namespace

extern "C" {

int gpk_blr_fit(gpk_handle* h, const double* hypers, int k) {
    const char* who = "gpk_blr_fit";
    if (h && h->model == MODEL_DNGO) BAD("%s: the handle holds %s; its fit is gpk_dngo_fit", who, MODELS[MODEL_DNGO].holds);
    int rc = blr_ready(h, who);
    if (rc) return rc;
    return blr_fit(h, hypers, k, who);
}

int gpk_blr_get_models(gpk_handle* h, double* m, double* S) {
    const char* who = "gpk_blr_get_models";
    int rc = blr_ready(h, who);
    if (rc) return rc;
    if (!h->blr.fitted) { set_err(h, "%s: %s", who, MODELS[MODEL_BLR].not_fitted); return GPK_NOT_FITTED; }
    const BlrPost L(h->blr.k, h->blr.F);
    const double* post = ptr<double>(h->blr.post);
    if (m) CK(cudaMemcpyAsync(m, post + L.M, (size_t)h->blr.k * h->blr.F * 8, cudaMemcpyDeviceToHost, h->stream));
    if (S)
        CK(cudaMemcpyAsync(S, post + L.S, (size_t)h->blr.k * h->blr.F * h->blr.F * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_blr_dims(gpk_handle* h, int* n, int* F, int* k) {
    int rc = blr_ready(h, "gpk_blr_dims");
    if (rc) return rc;
    if (n) *n = h->n;
    if (F) *F = h->blr.F;
    if (k) *k = h->blr.fitted ? h->blr.k : 0;
    return GPK_OK;
}

// ---------------------------------------------------------------------------------------
// Random forest (gpk_rf.cuh; robo/models/random_forest.py)
// ---------------------------------------------------------------------------------------
int gpk_rf_set_data(gpk_handle* h, const double* X, const double* y, int n, int d) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_rf_set_data";
    int rc = claim_model(h, MODEL_RF, who);
    if (rc) return rc;
    if (!X || !y || n <= 0 || d <= 0) BAD("%s: need X, y, n > 0, d > 0", who);
    if (n > GPK_RF_MAX_N) BAD("%s: n = %d training points exceed GPK_RF_MAX_N = %d", who, n, GPK_RF_MAX_N);
    if (d > GPK_RF_MAX_D) BAD("%s: d = %d exceeds GPK_RF_MAX_D = %d", who, d, GPK_RF_MAX_D);
    for (long i = 0; i < (long)n * d; ++i)
        if (!std::isfinite(X[i])) BAD("%s: X must be finite", who);
    for (int i = 0; i < n; ++i)
        if (!std::isfinite(y[i])) BAD("%s: y must be finite", who);
    CK(cudaSetDevice(h->device));
    // each feature's rows ordered by (x_f, row index), once per training set
    std::vector<int> order((size_t)d * n);
    for (int f = 0; f < d; ++f) {
        int* o = order.data() + (size_t)f * n;
        for (int i = 0; i < n; ++i) o[i] = i;
        std::sort(o, o + n, [&](int a, int b) {
            const double xa = X[(size_t)a * d + f], xb = X[(size_t)b * d + f];
            return xa < xb || (xa == xb && a < b);
        });
    }
    h->model = MODEL_RF;
    h->rf.fitted = false;
    h->n = n; h->d = d;
    if ((rc = ensure(h, h->rf.data, ((size_t)n * d + n) * 8 + (size_t)d * n * 4))) return rc;
    CK(cudaMemcpyAsync(rf_X(h), X, (size_t)n * d * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(rf_y(h), y, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(rf_order(h), order.data(), (size_t)d * n * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));     // host buffers are caller-owned: done with them
    return GPK_OK;
}

int gpk_rf_fit(gpk_handle* h, unsigned long long seed, unsigned counter, int T, int n_per_tree, int bootstrap,
               int total_variance) {
    const char* who = "gpk_rf_fit";
    int rc = model_ready(h, MODEL_RF, who);
    if (rc) return rc;
    const int n = h->n, d = h->d;
    if (T < 1 || T > GPK_RF_MAX_T) BAD("%s: need 1 <= num_trees <= GPK_RF_MAX_T = %d (num_trees = %d)", who, GPK_RF_MAX_T, T);
    if (n_per_tree < 0) BAD("%s: need n_points_per_tree >= 0", who);
    const int nt = n_per_tree > 0 ? n_per_tree : n;
    if (!bootstrap && nt > n)
        BAD("%s: without bootstrapping a tree cannot take %d of %d points (n_points_per_tree <= n)", who, nt, n);
    h->rf.fitted = false;
    const long S = 2L * n;
    const RfNodes L(T, S);
    if ((rc = ensure(h, h->rf.nodes, L.total))) return rc;
    // growth scratch per CTA: multiplicities (n), two list buffers (2 (d + 1) n) and the segments (3 x 2 n), ints;
    // trees are grown in batches that keep it near 512 MB
    const size_t per_tree = (size_t)n * (1 + 2 * (size_t)(d + 1) + 6) * 4;
    const int batch = (int)std::max<size_t>(1, std::min<size_t>((size_t)T, ((size_t)512 << 20) / per_tree));
    if ((rc = ensure(h, h->rf.work, per_tree * batch))) return rc;
    char* nodes = ptr<char>(h->rf.nodes);
    int* work = ptr<int>(h->rf.work);
    RfGrowArgs a;
    memset(&a, 0, sizeof(a));
    a.X = rf_X(h); a.y = rf_y(h); a.order = rf_order(h);
    a.n = n; a.d = d; a.nt = nt; a.bootstrap = bootstrap ? 1 : 0;
    a.seed = seed; a.counter = counter;
    a.cnt = work;
    a.lists = work + (size_t)batch * n;
    a.seg = a.lists + (size_t)batch * 2 * (d + 1) * n;
    a.feat = (int*)(nodes + L.feat); a.left = (int*)(nodes + L.left); a.n_nodes = (int*)(nodes + L.nn);
    a.thr = (double*)(nodes + L.thr); a.W = (double*)(nodes + L.W); a.mean = (double*)(nodes + L.mean);
    a.var = (double*)(nodes + L.var);
    for (int t0 = 0; t0 < T; t0 += batch) {
        a.t0 = t0;
        gpk_rf_grow_kernel<<<std::min(batch, T - t0), GPK_RF_GROW_THREADS, 0, h->stream>>>(a);
        CKL();
    }
    CK(cudaStreamSynchronize(h->stream));
    h->rf.T = T;
    h->rf.total = total_variance ? 1 : 0;
    h->rf.fitted = true;
    return GPK_OK;
}

int gpk_rf_dims(gpk_handle* h, int* n, int* d, int* T, int* slots) {
    int rc = model_ready(h, MODEL_RF, "gpk_rf_dims");
    if (rc) return rc;
    if (n) *n = h->n;
    if (d) *d = h->d;
    if (T) *T = h->rf.fitted ? h->rf.T : 0;
    if (slots) *slots = 2 * h->n;
    return GPK_OK;
}

int gpk_rf_get_trees(gpk_handle* h, int* n_nodes, int* feat, double* thr, int* left, double* W, double* mean,
                     double* var) {
    const char* who = "gpk_rf_get_trees";
    int rc = model_ready(h, MODEL_RF, who);
    if (rc) return rc;
    if (!h->rf.fitted) { set_err(h, "%s: %s", who, MODELS[MODEL_RF].not_fitted); return GPK_NOT_FITTED; }
    const long S = 2L * h->n;
    const size_t TS = (size_t)h->rf.T * S;
    const RfNodes L(h->rf.T, S);
    const char* nodes = ptr<char>(h->rf.nodes);
    const struct { void* dst; size_t off, bytes; } parts[] = {
        {n_nodes, L.nn, (size_t)h->rf.T * 4}, {feat, L.feat, TS * 4}, {thr, L.thr, TS * 8}, {left, L.left, TS * 4},
        {W, L.W, TS * 8}, {mean, L.mean, TS * 8}, {var, L.var, TS * 8}};
    for (const auto& p : parts)
        if (p.dst) CK(cudaMemcpyAsync(p.dst, nodes + p.off, p.bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_rf_set_trees(gpk_handle* h, int T, int total_variance, const int* n_nodes, const int* feat, const double* thr,
                     const int* left, const double* W, const double* mean, const double* var) {
    const char* who = "gpk_rf_set_trees";
    int rc = model_ready(h, MODEL_RF, who);
    if (rc) return rc;
    if (T < 1 || T > GPK_RF_MAX_T) BAD("%s: need 1 <= T <= GPK_RF_MAX_T = %d", who, GPK_RF_MAX_T);
    if (!n_nodes || !feat || !thr || !left || !W || !mean || !var) BAD("%s: need every node array", who);
    const long S = 2L * h->n;
    // every walk must end in a leaf: a split node's children come after it and exist
    for (int t = 0; t < T; ++t) {
        const int nn = n_nodes[t];
        if (nn < 1 || nn >= S) BAD("%s: tree %d has %d nodes (1 .. %ld allowed)", who, t, nn, S - 1);
        for (int v = 0; v < nn; ++v) {
            const int f = feat[(size_t)t * S + v], c = left[(size_t)t * S + v];
            if (f >= h->d || (f >= 0 && (c <= v || c + 1 >= nn)))
                BAD("%s: node %d of tree %d is not a valid split or leaf", who, v, t);
        }
    }
    h->rf.fitted = false;
    const size_t TS = (size_t)T * S;
    const RfNodes L(T, S);
    if ((rc = ensure(h, h->rf.nodes, L.total))) return rc;
    char* nodes = ptr<char>(h->rf.nodes);
    const struct { const void* src; size_t off, bytes; } parts[] = {
        {n_nodes, L.nn, (size_t)T * 4}, {feat, L.feat, TS * 4}, {thr, L.thr, TS * 8}, {left, L.left, TS * 4},
        {W, L.W, TS * 8}, {mean, L.mean, TS * 8}, {var, L.var, TS * 8}};
    for (const auto& p : parts) CK(cudaMemcpyAsync(nodes + p.off, p.src, p.bytes, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->rf.T = T;
    h->rf.total = total_variance ? 1 : 0;
    h->rf.fitted = true;
    return GPK_OK;
}

}  // extern "C"

namespace {
// The host scaling of gpk_bnn_set_data and gpk_dngo_set_data: X and y must be finite; then buf = the scaled X (n x d),
// the scaled y (n), the input mean and std (d each), and *ym / *ysd the y statistics.  Each column of X (norm_x) and y
// (norm_y) goes to zero mean and unit population std (sums in ascending row order); a constant one is GPK_BAD_ARG.  A
// side whose flag is off is copied as given, with mean 0 and std 1.
int scale_set(gpk_handle* h, const char* who, const double* X, const double* y, int n, int d, bool norm_x, bool norm_y,
              std::vector<double>& buf, double* ym, double* ysd) {
    for (long i = 0; i < (long)n * d; ++i)
        if (!std::isfinite(X[i])) BAD("%s: X must be finite", who);
    for (int i = 0; i < n; ++i)
        if (!std::isfinite(y[i])) BAD("%s: y must be finite", who);
    // column statistics: sums in ascending row order, population std
    const size_t nd = (size_t)n * d;
    buf.assign(nd + n + 2 * (size_t)d, 0.0);
    double* xs = buf.data();
    double* ys = xs + nd;
    double* xm = ys + n;
    double* xsd = xm + d;
    auto stats = [n](const double* v, long stride, double* mean, double* sd) {
        double s = 0.0;
        for (int i = 0; i < n; ++i) s += v[(long)i * stride];
        const double m = s / (double)n;
        double q = 0.0;
        for (int i = 0; i < n; ++i) {
            const double e = v[(long)i * stride] - m;
            q += e * e;
        }
        *mean = m;
        *sd = std::sqrt(q / (double)n);
    };
    for (int c = 0; c < d; ++c) {
        if (!norm_x) {
            xm[c] = 0.0; xsd[c] = 1.0;
            for (int i = 0; i < n; ++i) xs[(size_t)i * d + c] = X[(size_t)i * d + c];
            continue;
        }
        stats(X + c, d, xm + c, xsd + c);
        if (!(xsd[c] > 0.0)) BAD("%s: input column %d is constant; it cannot be normalised", who, c);
        for (int i = 0; i < n; ++i) xs[(size_t)i * d + c] = (X[(size_t)i * d + c] - xm[c]) / xsd[c];
    }
    if (!norm_y) {
        *ym = 0.0; *ysd = 1.0;
        for (int i = 0; i < n; ++i) ys[i] = y[i];
        return GPK_OK;
    }
    stats(y, 1, ym, ysd);
    if (!(*ysd > 0.0)) BAD("%s: y is constant; it cannot be normalised", who);
    for (int i = 0; i < n; ++i) ys[i] = (y[i] - *ym) / *ysd;
    return GPK_OK;
}
}  // namespace

extern "C" {

// ---------------------------------------------------------------------------------------
// Bayesian neural network (gpk_bnn.cuh; robo/models/wrapper_bohamiann.py)
// ---------------------------------------------------------------------------------------
int gpk_bnn_set_data(gpk_handle* h, const double* X, const double* y, int n, int d) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_bnn_set_data";
    int rc = claim_model(h, MODEL_BNN, who);
    if (rc) return rc;
    if (!X || !y || n <= 0 || d <= 0) BAD("%s: need X, y, n > 0, d > 0", who);
    if (n < 2) BAD("%s: need n >= 2 training points to normalise the data (n = %d)", who, n);
    if (n > GPK_BNN_MAX_N) BAD("%s: n = %d training points exceed GPK_BNN_MAX_N = %d", who, n, GPK_BNN_MAX_N);
    if (d > GPK_BNN_MAX_D) BAD("%s: d = %d exceeds GPK_BNN_MAX_D = %d", who, d, GPK_BNN_MAX_D);
    std::vector<double> buf;
    double ym, ysd;
    if ((rc = scale_set(h, who, X, y, n, d, true, true, buf, &ym, &ysd))) return rc;
    CK(cudaSetDevice(h->device));
    h->model = MODEL_BNN;
    h->bnn.S = 0;
    h->n = n; h->d = d;
    h->bnn.P = gpk_bnn_params(d);
    h->bnn.ymean = ym; h->bnn.ystd = ysd;
    if ((rc = ensure(h, h->bnn.data, buf.size() * 8))) return rc;
    CK(cudaMemcpyAsync(bnn_X(h), buf.data(), buf.size() * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));     // the staging vector dies here
    return GPK_OK;
}

int gpk_bnn_train(gpk_handle* h, unsigned long long seed, unsigned counter, double lr, double mdecay, double eps,
                  long burn_in, long num_steps, long keep_every, int batch) {
    const char* who = "gpk_bnn_train";
    int rc = model_ready(h, MODEL_BNN, who);
    if (rc) return rc;
    if (!(std::isfinite(lr) && lr > 0.0) || !(std::isfinite(mdecay) && mdecay > 0.0) || !(std::isfinite(eps) && eps >= 0.0))
        BAD("%s: need finite lr > 0, mdecay > 0 and eps >= 0", who);
    if (batch < 1 || batch > GPK_BNN_MAX_BATCH) BAD("%s: need 1 <= batch <= GPK_BNN_MAX_BATCH = %d", who, GPK_BNN_MAX_BATCH);
    if (keep_every < 1 || burn_in < 0) BAD("%s: need keep_every >= 1 and burn_in >= 0", who);
    if (num_steps < 1 || num_steps > INT_MAX) BAD("%s: need 1 <= num_steps <= 2^31 - 1", who);
    const long S = num_steps - 1 > burn_in ? (num_steps - 1 - burn_in) / keep_every : 0;
    if (S < 1) BAD("%s: the chain keeps no network (num_steps = %ld, burn_in = %ld, keep_every = %ld)", who, num_steps,
                   burn_in, keep_every);
    const int P = h->bnn.P;
    h->bnn.S = 0;
    if ((rc = ensure(h, h->bnn.samples, (size_t)S * P * 8))) return rc;
    if ((rc = ensure(h, h->bnn.state, (size_t)5 * P * 8))) return rc;
    const size_t smem = (size_t)gpk_bnn_chain_smem(h->n, h->d, batch);
    CK(cudaFuncSetAttribute(gpk_bnn_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    BnnChainArgs a;
    memset(&a, 0, sizeof(a));
    a.X = bnn_X(h); a.y = bnn_y(h);
    a.n = h->n; a.d = h->d; a.P = P; a.B = batch;
    a.seed = seed; a.counter = counter;
    a.lr = lr; a.mdecay = mdecay; a.eps = eps;
    a.burn_in = burn_in; a.num_steps = num_steps; a.keep_every = keep_every;
    a.samples = ptr<double>(h->bnn.samples);
    a.state = ptr<double>(h->bnn.state);
    gpk_bnn_chain_kernel<<<1, GPK_BNN_THREADS, smem, h->stream>>>(a);
    CKL();
    CK(cudaStreamSynchronize(h->stream));
    h->bnn.S = (int)S;
    return GPK_OK;
}

int gpk_bnn_dims(gpk_handle* h, int* n, int* d, int* P, int* S) {
    int rc = model_ready(h, MODEL_BNN, "gpk_bnn_dims");
    if (rc) return rc;
    if (n) *n = h->n;
    if (d) *d = h->d;
    if (P) *P = h->bnn.P;
    if (S) *S = h->bnn.S;
    return GPK_OK;
}

int gpk_bnn_get_samples(gpk_handle* h, double* samples) {
    const char* who = "gpk_bnn_get_samples";
    int rc = model_ready(h, MODEL_BNN, who);
    if (rc) return rc;
    if (h->bnn.S < 1) { set_err(h, "%s: %s", who, MODELS[MODEL_BNN].not_fitted); return GPK_NOT_FITTED; }
    if (!samples) BAD("%s: need the output array", who);
    CK(cudaMemcpyAsync(samples, h->bnn.samples.p, (size_t)h->bnn.S * h->bnn.P * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_bnn_set_samples(gpk_handle* h, int S, const double* samples) {
    const char* who = "gpk_bnn_set_samples";
    int rc = model_ready(h, MODEL_BNN, who);
    if (rc) return rc;
    if (S < 1 || !samples) BAD("%s: need S >= 1 networks", who);
    h->bnn.S = 0;
    if ((rc = ensure(h, h->bnn.samples, (size_t)S * h->bnn.P * 8))) return rc;
    CK(cudaMemcpyAsync(h->bnn.samples.p, samples, (size_t)S * h->bnn.P * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->bnn.S = S;
    return GPK_OK;
}

int gpk_bnn_get_state(gpk_handle* h, double* theta, double* p, double* tau, double* g, double* vhat) {
    const char* who = "gpk_bnn_get_state";
    int rc = model_ready(h, MODEL_BNN, who);
    if (rc) return rc;
    if (h->bnn.S < 1 || !h->bnn.state.p) { set_err(h, "%s: no chain has run (gpk_bnn_train)", who); return GPK_NOT_FITTED; }
    double* out[5] = {theta, p, tau, g, vhat};
    const size_t P = h->bnn.P;
    for (int i = 0; i < 5; ++i)
        if (out[i]) CK(cudaMemcpyAsync(out[i], ptr<double>(h->bnn.state) + i * P, P * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_bnn_draws(gpk_handle* h, unsigned long long seed, unsigned counter, int step0, int ns, double* Z) {
    const char* who = "gpk_bnn_draws";
    int rc = model_ready(h, MODEL_BNN, who);
    if (rc) return rc;
    if (ns < 1 || !Z) BAD("%s: need ns >= 1 and an output array", who);
    const int P = h->bnn.P;
    const size_t bytes = (size_t)ns * P * 8;
    if ((rc = ensure(h, h->tmp1, bytes))) return rc;
    const long threads = (long)ns * (P / 2);
    gpk_bnn_draws_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, h->stream>>>(seed, counter, step0, ns, P,
                                                                                  ptr<double>(h->tmp1));
    CKL();
    CK(cudaMemcpyAsync(Z, h->tmp1.p, bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

// ---------------------------------------------------------------------------------------
// DNGO (gpk_dngo.cuh; pybnn's DNGO, robo/fmin/bayesian_optimization.py:105-109)
// ---------------------------------------------------------------------------------------
}  // extern "C"

namespace {
// G = Theta^T Theta and b = Theta^T y of the Bayesian linear regression over the features in blr_phi(h); then the handle
// holds a trained net and no fit
int dngo_gram(gpk_handle* h) {
    gpk_blr_gram_kernel<<<(unsigned)(GPK_DNGO_H * GPK_DNGO_H + GPK_DNGO_H), 256, 0, h->stream>>>(
        blr_phi(h), blr_y(h), h->n, GPK_DNGO_H, blr_G(h), blr_b(h));
    CKL();
    CK(cudaStreamSynchronize(h->stream));
    h->dngo.trained = true;
    return GPK_OK;
}

int dngo_trained(gpk_handle* h, const char* who) {
    int rc = model_ready(h, MODEL_DNGO, who);
    if (rc) return rc;
    if (!h->dngo.trained) { set_err(h, "%s: model is not trained (gpk_dngo_train)", who); return GPK_NOT_FITTED; }
    return GPK_OK;
}
}  // namespace

extern "C" {

int gpk_dngo_set_data(gpk_handle* h, const double* X, const double* y, int n, int d, int normalize_input,
                      int normalize_output, const double* prior_par) {
    if (!h) return GPK_BAD_ARG;
    const char* who = "gpk_dngo_set_data";
    int rc = claim_model(h, MODEL_DNGO, who);
    if (rc) return rc;
    if (!X || !y || !prior_par || n <= 0 || d <= 0) BAD("%s: need X, y, prior_par, n > 0, d > 0", who);
    if ((normalize_input || normalize_output) && n < 2)
        BAD("%s: need n >= 2 training points to normalise the data (n = %d)", who, n);
    if (n > GPK_DNGO_MAX_N) BAD("%s: n = %d training points exceed GPK_DNGO_MAX_N = %d", who, n, GPK_DNGO_MAX_N);
    if (d > GPK_DNGO_MAX_D) BAD("%s: d = %d exceeds GPK_DNGO_MAX_D = %d", who, d, GPK_DNGO_MAX_D);
    std::vector<double> buf;
    double ym, ysd;
    if ((rc = scale_set(h, who, X, y, n, d, normalize_input != 0, normalize_output != 0, buf, &ym, &ysd))) return rc;
    CK(cudaSetDevice(h->device));
    h->model = MODEL_DNGO;
    h->dngo.trained = h->dngo.fitted = h->blr.fitted = false;
    h->dngo.t = -1;
    h->n = n; h->d = d;
    h->dngo.P = gpk_dngo_params(d);
    h->bnn.ymean = ym; h->bnn.ystd = ysd;
    h->blr.F = GPK_DNGO_H; h->blr.basis = GPK_BLR_NONE;
    h->blr.prior.ln_sigma = prior_par[0]; h->blr.prior.ln_loc = prior_par[1]; h->blr.prior.hs_scale = prior_par[2];
    if ((rc = ensure(h, h->bnn.data, buf.size() * 8))) return rc;
    if ((rc = ensure(h, h->blr.data, ((size_t)n * GPK_DNGO_H + n + GPK_DNGO_H * GPK_DNGO_H + GPK_DNGO_H) * 8))) return rc;
    CK(cudaMemcpyAsync(bnn_X(h), buf.data(), buf.size() * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(blr_y(h), buf.data() + (size_t)n * d, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));     // the staging vector dies here
    return GPK_OK;
}

int gpk_dngo_train(gpk_handle* h, unsigned long long seed, unsigned counter, double lr, int batch, int epochs) {
    const char* who = "gpk_dngo_train";
    int rc = model_ready(h, MODEL_DNGO, who);
    if (rc) return rc;
    if (!(std::isfinite(lr) && lr > 0.0)) BAD("%s: need a finite lr > 0", who);
    if (batch < 1 || epochs < 1) BAD("%s: need batch >= 1 and epochs >= 1", who);
    const int B = std::min(batch, h->n);
    if (B > GPK_DNGO_MAX_BATCH)
        BAD("%s: a batch of min(batch, n) = %d rows exceeds GPK_DNGO_MAX_BATCH = %d", who, B, GPK_DNGO_MAX_BATCH);
    const int P = h->dngo.P;
    h->dngo.trained = h->dngo.fitted = h->blr.fitted = false;
    h->dngo.t = -1;
    if ((rc = ensure(h, h->dngo.net, (size_t)P * 8))) return rc;
    if ((rc = ensure(h, h->dngo.state, (size_t)2 * P * 8))) return rc;
    const size_t smem = (size_t)gpk_dngo_train_smem(h->n, h->d, B);
    CK(cudaFuncSetAttribute(gpk_dngo_train_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DngoTrainArgs a;
    memset(&a, 0, sizeof(a));
    a.X = bnn_X(h); a.y = bnn_y(h);
    a.n = h->n; a.d = h->d; a.P = P; a.B = B; a.epochs = epochs;
    a.seed = seed; a.counter = counter;
    a.lr = lr;
    a.state = ptr<double>(h->dngo.state);
    a.net = ptr<double>(h->dngo.net);
    a.Theta = blr_phi(h);
    gpk_dngo_train_kernel<<<1, GPK_DNGO_THREADS, smem, h->stream>>>(a);
    CKL();
    if ((rc = dngo_gram(h))) return rc;
    h->dngo.t = (long long)epochs * (h->n / B);
    return GPK_OK;
}

int gpk_dngo_fit(gpk_handle* h, const double* hypers, int k) {
    const char* who = "gpk_dngo_fit";
    int rc = dngo_trained(h, who);
    if (!rc) rc = blr_ready(h, who);
    if (!rc) rc = blr_fit(h, hypers, k, who);
    if (rc) return rc;
    h->dngo.fitted = false;
    const DngoPack K(h->d);
    if ((rc = ensure(h, h->dngo.pack, (size_t)K.total * 8 + 8))) return rc;
    double* pack = ptr<double>(h->dngo.pack);
    int* fail = (int*)(pack + K.total);
    const BlrPost L(k, GPK_DNGO_H);
    const double* post = ptr<double>(h->blr.post);
    gpk_dngo_collapse_kernel<<<1, GPK_BLR_THREADS, gpk_dngo_collapse_doubles() * 8, h->stream>>>(
        post + L.M, post + L.S, post + L.ib, k, ptr<double>(h->dngo.net), h->d, pack, fail);
    CKL();
    int f = 0;
    CK(cudaMemcpyAsync(&f, fail, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (f) {
        set_err(h, "%s: the mixture covariance mean S_i + cov(m_i) of the %d hypers is not positive definite", who, k);
        return GPK_NOT_PD;
    }
    h->dngo.fitted = true;
    return GPK_OK;
}

int gpk_dngo_dims(gpk_handle* h, int* n, int* d, int* P, int* k) {
    int rc = model_ready(h, MODEL_DNGO, "gpk_dngo_dims");
    if (rc) return rc;
    if (n) *n = h->n;
    if (d) *d = h->d;
    if (P) *P = h->dngo.P;
    if (k) *k = h->dngo.fitted ? h->blr.k : 0;
    return GPK_OK;
}

int gpk_dngo_get_net(gpk_handle* h, double* net) {
    const char* who = "gpk_dngo_get_net";
    int rc = dngo_trained(h, who);
    if (rc) return rc;
    if (!net) BAD("%s: need the output array", who);
    CK(cudaMemcpyAsync(net, h->dngo.net.p, (size_t)h->dngo.P * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_dngo_set_net(gpk_handle* h, const double* net) {
    const char* who = "gpk_dngo_set_net";
    int rc = model_ready(h, MODEL_DNGO, who);
    if (rc) return rc;
    if (!net) BAD("%s: need the net", who);
    const int P = h->dngo.P;
    for (int i = 0; i < P; ++i)
        if (!std::isfinite(net[i])) BAD("%s: the net must be finite", who);
    h->dngo.trained = h->dngo.fitted = h->blr.fitted = false;
    h->dngo.t = -1;
    if ((rc = ensure(h, h->dngo.net, (size_t)P * 8))) return rc;
    CK(cudaMemcpyAsync(h->dngo.net.p, net, (size_t)P * 8, cudaMemcpyHostToDevice, h->stream));
    gpk_dngo_features_kernel<<<(unsigned)h->n, 64, 0, h->stream>>>(bnn_X(h), h->n, h->d, nullptr, nullptr,
                                                                   ptr<double>(h->dngo.net), blr_phi(h));
    CKL();
    return dngo_gram(h);
}

int gpk_dngo_features(gpk_handle* h, const double* X, long m, double* out) {
    const char* who = "gpk_dngo_features";
    int rc = dngo_trained(h, who);
    if (rc) return rc;
    if (!X || !out || m < 1 || m > INT_MAX) BAD("%s: need X, out and 1 <= m <= 2^31 - 1", who);
    const size_t xb = (size_t)m * h->d * 8, ob = (size_t)m * GPK_DNGO_H * 8;
    if ((rc = ensure(h, h->tmp1, xb + ob))) return rc;
    double* dX = ptr<double>(h->tmp1);
    double* dO = dX + (size_t)m * h->d;
    CK(cudaMemcpyAsync(dX, X, xb, cudaMemcpyHostToDevice, h->stream));
    gpk_dngo_features_kernel<<<(unsigned)m, 64, 0, h->stream>>>(dX, m, h->d, bnn_xm(h), bnn_xs(h),
                                                               ptr<double>(h->dngo.net), dO);
    CKL();
    CK(cudaMemcpyAsync(out, dO, ob, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_dngo_get_state(gpk_handle* h, double* m, double* v, long long* t) {
    const char* who = "gpk_dngo_get_state";
    int rc = model_ready(h, MODEL_DNGO, who);
    if (rc) return rc;
    if (h->dngo.t < 0) { set_err(h, "%s: no training has run (gpk_dngo_train)", who); return GPK_NOT_FITTED; }
    const size_t P = h->dngo.P;
    if (m) CK(cudaMemcpyAsync(m, ptr<double>(h->dngo.state), P * 8, cudaMemcpyDeviceToHost, h->stream));
    if (v) CK(cudaMemcpyAsync(v, ptr<double>(h->dngo.state) + P, P * 8, cudaMemcpyDeviceToHost, h->stream));
    if (t) *t = h->dngo.t;
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_kernel_matrix(gpk_handle* h, const double* X1, long n1, const double* X2, long n2, int d, double* out) {
    int rc = require(h, false, true, false);
    if (rc) return rc;
    if (!X1 || !X2 || !out || n1 <= 0 || n2 <= 0 || d <= 0 || d > GPK_MAX_TERMS) BAD("gpk_kernel_matrix: bad arguments");
    for (int t = 0; t < h->spec.n_terms; ++t)
        if (h->spec.axis[t] >= d) BAD("gpk_kernel_matrix: kernel axis %d >= d = %d", h->spec.axis[t], d);
    if ((rc = factor_data_check(h, d, nullptr, "gpk_kernel_matrix"))) return rc;
    CK(cudaSetDevice(h->device));
    const long n1p = round_up(n1, 32), n2p = round_up(n2, 128);
    if ((rc = ensure(h, h->tmp1, (size_t)n1 * d * 8))) return rc;
    const long x2off = round_up(n2 * d, 16);                 // keeps the operand 128-byte aligned (TMA source)
    if ((rc = ensure(h, h->tmp2, (size_t)(x2off + (long)cov_operand_rows(h, d) * n2p) * 8))) return rc;
    if ((rc = ensure(h, h->tmp3, (size_t)n1p * n2p * 8))) return rc;
    double* X2row = ptr<double>(h->tmp2);
    double* X2t = X2row + x2off;
    CK(cudaMemcpyAsync(h->tmp1.p, X1, (size_t)n1 * d * 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(X2row, X2, (size_t)n2 * d * 8, cudaMemcpyHostToDevice, h->stream));
    if ((rc = build_cov_operand(h, h->stream, X2row, n2, d, nullptr, nullptr, X2t, n2p))) return rc;
    if ((rc = launch_cov_tiles(h, h->stream, X2t, n2p, (int)n2, ptr<double>(h->tmp1), d, n1, n1p, nullptr, nullptr,
                               ptr<double>(h->tmp3), n2p, 0, false, X2row, nullptr, nullptr)))
        return rc;
    CK(cudaMemcpy2DAsync(out, (size_t)n2 * 8, h->tmp3.p, (size_t)n2p * 8, (size_t)n2 * 8, (size_t)n1,
                         cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_nll_grad(gpk_handle* h, double noise_var, double* grad) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!grad) BAD("gpk_nll_grad: null output");
    CK(cudaSetDevice(h->device));
    if ((rc = build_linv(h))) return rc;
    const long NP = h->NP;
    // [amp, metric..., factor parameters..., noise]: environment entries from the trace kernel, task entries below
    const int fk = h->spec.factor.kind;
    const int nT = fk == GPK_FACTOR_TASK ? h->spec.factor.n_tasks : 0;
    const int nv = h->spec.n_terms + (fk == GPK_FACTOR_ENV ? 4 : 2);
    // alpha = L^-T z
    if ((rc = ensure(h, h->alpha, (size_t)NP * 8))) return rc;
    gpk_rowdot_kernel<<<(unsigned)((NP + 7) / 8), 256, 0, h->stream>>>(ptr<double>(h->Q), NP, NP, (int)NP, 1,
                                                                       ptr<double>(h->Kbuf) + NP * NP,
                                                                       ptr<double>(h->alpha));
    CKL();
    // K^-1 (lower tiles) into W
    {
        GemmArgs a;
        memset(&a, 0, sizeof(a));
        a.A = ptr<double>(h->Q); a.lda = NP;
        a.B = ptr<double>(h->Q); a.ldb = NP;
        a.C = ptr<double>(h->W); a.ldc = NP;
        a.alpha = 1.0; a.beta = 0;
        a.jobs = ptr<GemmJob>(h->jobs) + h->ranges.kinv.off;
        a.job_mode = JOBS_TABLE;
        if ((rc = launch_gemm<EPI_STORE>(h, h->mapQ, h->mapQ, a, h->ranges.kinv.cnt))) return rc;
    }
    dim3 tg((unsigned)(NP / 128), (unsigned)(NP / 32));
    const long nblocks = (long)tg.x * tg.y;
    if ((rc = ensure(h, h->tmp1, (size_t)nblocks * (nv + nT * nT) * 8))) return rc;
    if ((rc = ensure(h, h->tmp2, (size_t)(nv + nT * nT) * 8))) return rc;
    {
        auto kern = fk == GPK_FACTOR_ENV ? gpk_grad_trace_kernel<GPK_FACTOR_ENV>
                  : fk == GPK_FACTOR_TASK ? gpk_grad_trace_kernel<GPK_FACTOR_TASK> : gpk_grad_trace_kernel<GPK_FACTOR_NONE>;
        kern<<<tg, 256, 0, h->stream>>>(h->spec, ptr<double>(h->Xt), NP, h->n, ptr<double>(h->Xrow), h->d,
                                        ptr<double>(h->W), NP, ptr<double>(h->alpha), ptr<double>(h->tmp1));
    }
    CKL();
    gpk_grad_final_kernel<<<nv, 256, 0, h->stream>>>(ptr<double>(h->tmp1), nblocks, nv, noise_var, ptr<double>(h->tmp2));
    CKL();
    if (nT == 0) {
        CK(cudaMemcpyAsync(grad, h->tmp2.p, (size_t)nv * 8, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        return GPK_OK;
    }
    // task factor: the T x T sums G_ab (gpk_grad_task_kernel, times -1/2) contracted with
    // dK_t[a][b] / dtheta_pq = L_pq (delta_ap L_bq + delta_bp L_aq), L_pq = exp(theta[p (p + 1) / 2 + q])
    double* tpart = ptr<double>(h->tmp1) + (size_t)nblocks * nv;
    gpk_grad_task_kernel<<<tg, 256, 0, h->stream>>>(h->spec, ptr<double>(h->Xt), NP, h->n, ptr<double>(h->W), NP,
                                                    ptr<double>(h->alpha), tpart);
    CKL();
    gpk_grad_final_kernel<<<nT * nT, 256, 0, h->stream>>>(tpart, nblocks, nT * nT, 1.0, ptr<double>(h->tmp2) + nv);
    CKL();
    std::vector<double> g(nv + nT * nT);
    CK(cudaMemcpyAsync(g.data(), h->tmp2.p, g.size() * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    const int nt = h->spec.n_terms, nkt = nT * (nT + 1) / 2;
    const double* G = g.data() + nv;
    std::vector<double> L(nT * nT, 0.0);
    for (int p = 0; p < nT; ++p)
        for (int q = 0; q <= p; ++q) L[p * nT + q] = std::exp(h->task_theta[p * (p + 1) / 2 + q]);
    for (int v = 0; v <= nt; ++v) grad[v] = g[v];
    for (int p = 0; p < nT; ++p)
        for (int q = 0; q <= p; ++q) {
            double acc = 0.0;
            for (int b = q; b < nT; ++b) acc += G[p * nT + b] * L[b * nT + q];   // a = p, q <= b
            for (int a = q; a < nT; ++a) acc += G[a * nT + p] * L[a * nT + q];   // b = p, q <= a
            grad[nt + 1 + p * (p + 1) / 2 + q] = L[p * nT + q] * acc;
        }
    grad[nt + 1 + nkt] = g[nv - 1];
    return GPK_OK;
}

int gpk_measure_fp64_peaks(gpk_handle* h, double* dmma_tflops, double* dfma_tflops) {
    if (!h) return GPK_BAD_ARG;
    CK(cudaSetDevice(h->device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, h->device));
    const int blocks = prop.multiProcessorCount, warps = 16, threads = warps * 32, iters = 8000;
    int rc;
    if ((rc = ensure(h, h->tmp1, 64))) return rc;
    TimerEvents t;
    CK(cudaEventCreate(&t.e0));
    CK(cudaEventCreate(&t.e1));
    const cudaEvent_t e0 = t.e0, e1 = t.e1;
    double best_mma = 0.0, best_fma = 0.0;
    for (int rep = 0; rep < 3; ++rep) {
        float ms = 0.f;
        CK(cudaEventRecord(e0, h->stream));
        gpk_peak_dmma_kernel<<<blocks, threads, 0, h->stream>>>(ptr<double>(h->tmp1), iters);
        CKL();
        CK(cudaEventRecord(e1, h->stream));
        CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&ms, e0, e1));
        best_mma = std::max(best_mma, 2.0 * 256 * 16 * (double)iters * warps * blocks / (ms * 1e-3) / 1e12);
        CK(cudaEventRecord(e0, h->stream));
        gpk_peak_dfma_kernel<<<blocks, threads, 0, h->stream>>>(ptr<double>(h->tmp1), iters);
        CKL();
        CK(cudaEventRecord(e1, h->stream));
        CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&ms, e0, e1));
        best_fma = std::max(best_fma, 2.0 * 8 * (double)iters * threads * blocks / (ms * 1e-3) / 1e12);
    }
    if (dmma_tflops) *dmma_tflops = best_mma;
    if (dfma_tflops) *dfma_tflops = best_fma;
    return GPK_OK;
}

int gpk_measure_int8_peak(gpk_handle* h, double* tops) {
    if (!h || !tops) return GPK_BAD_ARG;
    CK(cudaSetDevice(h->device));
    const int blocks = std::max(h->n_sm, 1), iters = 4000, smem = 2 * 8192 + 1024 + 64;
    int rc;
    if ((rc = ensure(h, h->tmp1, 64))) return rc;
    TimerEvents t;
    CK(cudaEventCreate(&t.e0));
    CK(cudaEventCreate(&t.e1));
    const cudaEvent_t e0 = t.e0, e1 = t.e1;
    double best = 0.0;
    for (int rep = 0; rep < 3; ++rep) {
        float ms = 0.f;
        CK(cudaEventRecord(e0, h->stream));
        gpk_peak_i8_kernel<<<blocks, 256, smem, h->stream>>>(iters, 0, ptr<unsigned>(h->tmp1));
        CKL();
        CK(cudaEventRecord(e1, h->stream));
        CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&ms, e0, e1));
        best = std::max(best, 2.0 * 128 * 128 * 32 * 2.0 * iters * blocks / (ms * 1e-3) / 1e12);
    }
    *tops = best;
    return GPK_OK;
}

int gpk_measure_int8_peak_sustained(gpk_handle* h, double seconds, int random_operands, double* tops) {
    if (!h || !tops || !(seconds > 0.0) || seconds > 10.0) return GPK_BAD_ARG;
    CK(cudaSetDevice(h->device));
    // back-to-back launches of the issue-rate kernel for `seconds`; the rate of the SECOND half is reported: by then the
    // SM clock has settled where the board's power limit puts it (the int8 pipe at full rate runs into sw_power_cap)
    const int blocks = std::max(h->n_sm, 1), iters = 8000, smem = 2 * 8192 + 1024 + 64;
    const double ops = 2.0 * 128 * 128 * 32 * 2.0 * iters * blocks;
    int rc;
    if ((rc = ensure(h, h->tmp1, 64))) return rc;
    TimerEvents t;
    CK(cudaEventCreate(&t.e0));
    CK(cudaEventCreate(&t.e1));
    const cudaEvent_t e0 = t.e0, e1 = t.e1;
    float ms1 = 0.f;
    CK(cudaEventRecord(e0, h->stream));
    gpk_peak_i8_kernel<<<blocks, 256, smem, h->stream>>>(iters, random_operands, ptr<unsigned>(h->tmp1));
    CKL();
    CK(cudaEventRecord(e1, h->stream));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&ms1, e0, e1));
    const int n_half = std::max(1, (int)(0.5 * seconds * 1e3 / std::max(ms1, 1e-3f)));
    for (int i = 0; i < n_half; ++i) gpk_peak_i8_kernel<<<blocks, 256, smem, h->stream>>>(iters, random_operands, ptr<unsigned>(h->tmp1));
    CK(cudaEventRecord(e0, h->stream));
    for (int i = 0; i < n_half; ++i) gpk_peak_i8_kernel<<<blocks, 256, smem, h->stream>>>(iters, random_operands, ptr<unsigned>(h->tmp1));
    CKL();
    CK(cudaEventRecord(e1, h->stream));
    CK(cudaEventSynchronize(e1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    *tops = ops * n_half / (ms * 1e-3) / 1e12;
    return GPK_OK;
}

int gpk_get_factor(gpk_handle* h, double* L) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!L) BAD("gpk_get_factor: null output");
    CK(cudaSetDevice(h->device));
    const long n = h->n, NP = h->NP;
    CK(cudaMemcpy2DAsync(L, (size_t)n * 8, h->Kbuf.p, (size_t)NP * 8, (size_t)n * 8, (size_t)n, cudaMemcpyDeviceToHost,
                         h->stream));
    CK(cudaStreamSynchronize(h->stream));
    for (long i = 0; i < n; ++i)
        for (long j = i + 1; j < n; ++j) L[i * n + j] = 0.0;
    return GPK_OK;
}

int gpk_get_linv(gpk_handle* h, double* Linv) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!Linv) BAD("gpk_get_linv: null output");
    CK(cudaSetDevice(h->device));
    if ((rc = build_linv(h))) return rc;
    const long n = h->n, NP = h->NP;
    CK(cudaMemcpy2DAsync(Linv, (size_t)n * 8, h->P.p, (size_t)NP * 8, (size_t)n * 8, (size_t)n, cudaMemcpyDeviceToHost,
                         h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_get_z(gpk_handle* h, double* z) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!z) BAD("gpk_get_z: null output");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(z, ptr<double>(h->Kbuf) + (long)h->NP * h->NP, (size_t)h->n * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_oz_contract(gpk_handle* h, const double* P, int n, const double* Ks, long m, double amp, double* part_ssq,
                    int* eP, int* eK) {
    if (!h) return GPK_BAD_ARG;
    if (!P || !Ks || !part_ssq || !eP || !eK || n <= 0 || m <= 0 || !(amp > 0.0) || !std::isfinite(amp))
        BAD("gpk_oz_contract: bad arguments");
    const long NP = round_up(n, OZ_TM), MP = round_up(m, OZ_TM), nb = NP / OZ_TM;
    if (NP > 16384) BAD("gpk_oz_contract: n = %d pads to %ld > 16384 (the int32 level sums hold K <= 16384)", n, NP);
    for (long i = 0; i < m * (long)n; ++i)
        if (!(std::fabs(Ks[i]) <= amp)) BAD("gpk_oz_contract: |Ks| exceeds amp at entry %ld", i);
    CK(cudaSetDevice(h->device));
    // scratch, every piece a multiple of 512 bytes: P, Ks (zero-padded to NP x NP and MP x NP), their slices, the
    // partial sums, the row exponents and the exponent maximum the row-exponent kernel also writes
    const size_t oK = (size_t)NP * NP * 8, oPq = oK + (size_t)MP * NP * 8, oKq = oPq + (size_t)OZ_S * NP * NP;
    const size_t opart = oKq + (size_t)OZ_S * MP * NP, oe = opart + (size_t)nb * MP * 8, oemax = oe + (size_t)NP * 4;
    int rc;
    if ((rc = ensure(h, h->oz.probe, oemax + 4))) return rc;
    char* b = (char*)h->oz.probe.p;
    double* dP = (double*)b;
    double* dK = (double*)(b + oK);
    int8_t* dPq = (int8_t*)(b + oPq);
    int8_t* dKq = (int8_t*)(b + oKq);
    double* dpart = (double*)(b + opart);
    int* de = (int*)(b + oe);
    cudaStream_t st = h->stream;
    CK(cudaMemsetAsync(dP, 0, (size_t)NP * NP * 8, st));
    CK(cudaMemcpy2DAsync(dP, (size_t)NP * 8, P, (size_t)n * 8, (size_t)n * 8, (size_t)n, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(dK, 0, (size_t)MP * NP * 8, st));
    CK(cudaMemcpy2DAsync(dK, (size_t)NP * 8, Ks, (size_t)n * 8, (size_t)n * 8, (size_t)m, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(b + oemax, 0, 4, st));
    CK(cudaMemsetAsync(dpart, 0xFF, (size_t)nb * MP * 8, st));      // NaN: a tile that is never written shows
    gpk_oz_rowexp_kernel<<<(unsigned)NP, 256, 0, st>>>(dP, NP, (int)NP, de, (int*)(b + oemax));
    CKL();
    gpk_oz_split_kernel<<<(unsigned)((NP * NP + 255) / 256), 256, 0, st>>>(dP, NP, NP, de, 0, dPq, NP * NP);
    CKL();
    const int ek = oz_exponent(amp);
    gpk_oz_split_kernel<<<(unsigned)((MP * NP + 255) / 256), 256, 0, st>>>(dK, MP, NP, nullptr, ek, dKq, MP * NP);
    CKL();
    CUtensorMap mapP, mapK;
    if ((rc = make_oz_map(h, &mapP, dPq, (long)OZ_S * NP, NP, OZ_TM / h->oz.cluster))) return rc;
    if ((rc = make_oz_map(h, &mapK, dKq, (long)OZ_S * MP, NP, OZ_TN))) return rc;
    if ((rc = launch_oz_contraction(h, mapP, mapK, (int)nb, MP, NP, MP, de, ek, dpart, MP))) return rc;
    CK(cudaMemcpy2DAsync(part_ssq, (size_t)m * 8, dpart, (size_t)MP * 8, (size_t)m * 8, (size_t)nb, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(eP, de, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    *eK = ek;
    return GPK_OK;
}

int gpk_ep_joint_min(gpk_handle* h, const double* mu, const double* V, int nb, double* logP, double* dlogPdMu,
                     double* dlogPdSigma, double* dlogPdMudMu, int* sweeps) {
    if (!h) return GPK_BAD_ARG;
    if (!mu || !V || !logP) BAD("gpk_ep_joint_min: need mu, V and logP");
    if (nb < 2 || nb > GPK_EP_MAX_NB) BAD("gpk_ep_joint_min: nb = %d outside 2 .. %d", nb, GPK_EP_MAX_NB);
    CK(cudaSetDevice(h->device));
    const size_t D = (size_t)nb, T = D * (D + 1) / 2;
    // scratch in doubles: mu, V, logP, dMu, dMuMu, dSigma, Zm, Zs, adds, then 2 nb ints (sweeps, status)
    const size_t omu = 0, oV = omu + D, oP = oV + D * D, odM = oP + D, odMM = odM + D * D, odS = odMM + D * D * D;
    const size_t oZm = odS + D * T, oZs = oZm + D, oad = oZs + T, oint = oad + D * D;
    int rc;
    if ((rc = ensure(h, h->multi.ep_buf, oint * 8 + 2 * D * 4))) return rc;
    double* b = ptr<double>(h->multi.ep_buf);
    int* dsw = (int*)(b + oint);
    int* dst = dsw + D;
    cudaStream_t st = h->stream;
    CK(cudaMemcpyAsync(b + omu, mu, D * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b + oV, V, D * D * 8, cudaMemcpyHostToDevice, st));
    CK(cudaFuncSetAttribute(gpk_ep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GPK_EP_SMEM));
    gpk_ep_kernel<<<nb, GPK_EP_THREADS, GPK_EP_SMEM, st>>>(b + omu, b + oV, nb, b + oP, b + odM, b + odMM, b + odS, dsw, dst);
    CKL();
    std::vector<int> status(D);
    CK(cudaMemcpyAsync(status.data(), dst, D * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    // the reference solves the problems in order k = 0, 1, ...: the first failing one decides the error
    for (size_t k = 0; k < D; ++k) {
        if (status[k] == GPK_EP_NAN_VARIANCE) {
            set_err(h, "an error occurs while running expectation propagation in entropy search. "
                       "Resulting variance contains NaN");
            return GPK_EP_FAILED;
        }
        if (status[k] == GPK_EP_IRSR_NOT_PD) {
            set_err(h, "gpk_ep_joint_min: IRSR of problem %zu is not positive definite", k);
            return GPK_NOT_PD;
        }
    }
    gpk_ep_norm_kernel<<<1, GPK_EP_THREADS, 0, st>>>(nb, b + oP, b + odM, b + odMM, b + odS, b + oZm, b + oZs, b + oad);
    CKL();
    gpk_ep_apply_kernel<<<nb, GPK_EP_THREADS, 0, st>>>(nb, b + odM, b + odMM, b + odS, b + oZm, b + oZs, b + oad);
    CKL();
    CK(cudaMemcpyAsync(logP, b + oP, D * 8, cudaMemcpyDeviceToHost, st));
    if (dlogPdMu) CK(cudaMemcpyAsync(dlogPdMu, b + odM, D * D * 8, cudaMemcpyDeviceToHost, st));
    if (dlogPdSigma) CK(cudaMemcpyAsync(dlogPdSigma, b + odS, D * T * 8, cudaMemcpyDeviceToHost, st));
    if (dlogPdMudMu) CK(cudaMemcpyAsync(dlogPdMudMu, b + odMM, D * D * D * 8, cudaMemcpyDeviceToHost, st));
    if (sweeps) CK(cudaMemcpyAsync(sweeps, dsw, D * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return GPK_OK;
}

int gpk_es_update(gpk_handle* h, const double* zb, int nb, const double* lmb, double sn2, const double* W, int np_,
                  const double* lower, const double* upper, double* logP, double* dlogPdMu, double* dlogPdSigma,
                  double* dlogPdMudMu) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!zb || !lmb || !W || !lower || !upper) BAD("gpk_es_update: need zb, lmb, W, lower and upper");
    if (nb < 2 || nb > GPK_EP_MAX_NB) BAD("gpk_es_update: Nb = %d outside 2 .. %d", nb, GPK_EP_MAX_NB);
    if (np_ < 1) BAD("gpk_es_update: Np = %d < 1", np_);
    for (int i = 0; i < nb; ++i)
        if (!std::isfinite(lmb[i])) BAD("lmb should not be infinite.");
    const int d = h->d;
    const size_t D = (size_t)nb, T = D * (D + 1) / 2;
    std::vector<double> mu(D), V(D * D), lp(D), dMu(D * D), dSig(D * T), dMuMu(D * D * D);
    if ((rc = gpk_predict_cov(h, zb, nb, mu.data(), V.data()))) return rc;          // predict(zb, full_cov=True)
    if ((rc = gpk_ep_joint_min(h, mu.data(), V.data(), nb, lp.data(), dMu.data(), dSig.data(), dMuMu.data(), nullptr)))
        return rc;
    // H of the loss (information_gain.py:82) and dlogPdMudMu folded to its lower triangle
    double H = 0.0;
    for (size_t i = 0; i < D; ++i) H += std::exp(lp[i]) * (lp[i] + lmb[i]);
    H = -H;
    std::vector<double> Hs(D * T);
    for (size_t i = 0; i < D; ++i)
        for (size_t a = 0; a < D; ++a)
            for (size_t b = 0; b <= a; ++b)
                Hs[i * T + a * (a + 1) / 2 + b] = a == b ? dMuMu[(i * D + a) * D + a]
                                                         : dMuMu[(i * D + a) * D + b] + dMuMu[(i * D + b) * D + a];
    EsLayout L(nb, np_, d);
    if ((rc = ensure(h, h->es.state, L.total * 8))) return rc;
    double* st = ptr<double>(h->es.state);
    cudaStream_t s = h->stream;
    CK(cudaMemcpyAsync(st + L.logP, lp.data(), D * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(st + L.lmb, lmb, D * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(st + L.dMu, dMu.data(), D * D * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(st + L.dSig, dSig.data(), D * T * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(st + L.Hs, Hs.data(), D * T * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(st + L.W, W, (size_t)np_ * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(st + L.lo, lower, (size_t)d * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(st + L.up, upper, (size_t)d * 8, cudaMemcpyHostToDevice, s));
    // scaled zb, then U = L^-T (L^-1 K(X, zb)) in fp64 from the handle's L^-1
    if ((rc = es_build_u(h, zb, nb, st + L.zb))) return rc;
    CK(cudaStreamSynchronize(s));
    h->es.nb = nb;
    h->es.np = np_;
    h->es.sn2 = sn2;
    h->es.H = H;
    h->es.linv_serial = h->linv_serial;
    h->es.kind = ES_KIND_EP;
    if (logP) std::copy(lp.begin(), lp.end(), logP);
    if (dlogPdMu) std::copy(dMu.begin(), dMu.end(), dlogPdMu);
    if (dlogPdSigma) std::copy(dSig.begin(), dSig.end(), dlogPdSigma);
    if (dlogPdMudMu) std::copy(dMuMu.begin(), dMuMu.end(), dlogPdMudMu);
    return GPK_OK;
}

int gpk_es_compute_dev(gpk_handle* h, const void* d_Xs, long m, void* d_out) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!d_Xs || !d_out || m <= 0) BAD("gpk_es_compute_dev: need candidates and out");
    if ((rc = es_ready(h, nullptr, "gpk_es_compute"))) return rc;
    CK(cudaSetDevice(h->device));
    return es_dh_dev(h, (const double*)d_Xs, (const double*)d_Xs, m, (double*)d_out);
}

int gpk_es_compute(gpk_handle* h, const double* Xs, long m, double* out) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!Xs || !out || m <= 0) BAD("gpk_es_compute: need candidates and out");
    CK(cudaSetDevice(h->device));
    if ((rc = ensure(h, h->es.in, (size_t)m * (h->d + 1) * 8))) return rc;
    double* dX = ptr<double>(h->es.in);
    double* dout = dX + (size_t)m * h->d;
    CK(cudaMemcpyAsync(dX, Xs, (size_t)m * h->d * 8, cudaMemcpyHostToDevice, h->stream));
    if ((rc = gpk_es_compute_dev(h, dX, m, dout))) return rc;
    CK(cudaMemcpyAsync(out, dout, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_es_moments(gpk_handle* h, const double* Xs, long m, double* var, double* sigma) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!Xs || !var || !sigma || m <= 0) BAD("gpk_es_moments: need candidates, var and sigma");
    if ((rc = es_ready(h, nullptr, "gpk_es_moments", ES_KIND_NONE))) return rc;
    CK(cudaSetDevice(h->device));
    const int nb = h->es.nb, d = h->d;
    if ((rc = es_reserve(h))) return rc;
    if ((rc = ensure(h, h->es.in, (size_t)m * d * 8))) return rc;
    double* dX = ptr<double>(h->es.in);
    const double* dvar = ptr<double>(h->es.work);
    const double* dsig = dvar + ES_CH;
    CK(cudaMemcpyAsync(dX, Xs, (size_t)m * d * 8, cudaMemcpyHostToDevice, h->stream));
    for (long c0 = 0; c0 < m; c0 += ES_CH) {          // the passes of es_dh_dev, each read back before the next
        const long rows = std::min(ES_CH, m - c0);
        if ((rc = es_moments_pass(h, dX + c0 * d, rows))) return rc;
        CK(cudaMemcpyAsync(var + c0, dvar, (size_t)rows * 8, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaMemcpyAsync(sigma + c0 * nb, dsig, (size_t)rows * nb * 8, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
    }
    return GPK_OK;
}

int gpk_es_dims(gpk_handle* h, int* n, int* nb) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!n || !nb) BAD("gpk_es_dims: null output");
    if ((rc = es_ready(h, nullptr, "gpk_es_dims", ES_KIND_NONE))) return rc;
    *n = h->n;
    *nb = h->es.nb;
    return GPK_OK;
}

int gpk_es_get_u(gpk_handle* h, double* U) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!U) BAD("gpk_es_get_u: null output");
    if ((rc = es_ready(h, nullptr, "gpk_es_get_u", ES_KIND_NONE))) return rc;
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(U, h->es.U.p, (size_t)h->n * h->es.nb * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

// ---- sampling-based entropy search (gpk_esmc.cuh) ----------------------------------------------------------------
int gpk_mc_draws(gpk_handle* h, unsigned long long seed, int nb, int nf, double* F) {
    if (!h) return GPK_BAD_ARG;
    if (!F || nb < 1 || nf < 1 || (long)nb * nf > (1L << 28)) BAD("gpk_mc_draws: need F, nb >= 1, nf >= 1");
    CK(cudaSetDevice(h->device));
    const size_t bytes = (size_t)nb * nf * 8;
    int rc;
    if ((rc = ensure(h, h->mc.buf, bytes))) return rc;
    const long work = (long)nb * ((nf + 1) / 2);
    gpk_mc_draws_kernel<<<(unsigned)((work + 255) / 256), 256, 0, h->stream>>>(seed, nb, nf, ptr<double>(h->mc.buf));
    CKL();
    CK(cudaMemcpyAsync(F, h->mc.buf.p, bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

// the shape checks of joint_pmin's operands: 1 <= nb <= 64, np >= 1, nf >= 1, nf * np columns counted in an int
static int mc_check_shape(gpk_handle* h, int nb, int np_, int nf, int nb_min, const char* who) {
    if (nb < nb_min || nb > GPK_MC_MAX_NB) BAD("%s: Nb = %d outside %d .. %d", who, nb, nb_min, GPK_MC_MAX_NB);
    if (np_ < 1 || nf < 1) BAD("%s: need Np >= 1 and Nf >= 1 (Np = %d, Nf = %d)", who, np_, nf);
    if ((long)nf * np_ > 0x7FFFFFFFL) BAD("%s: Nf Np = %ld columns exceed the int counts", who, (long)nf * np_);
    return GPK_OK;
}

int gpk_mc_pmin(gpk_handle* h, const double* m, int np_, const double* V, int nb, int nf, unsigned long long seed,
                double* pmin, int* n_jitter) {
    if (!h) return GPK_BAD_ARG;
    int rc;
    if (!m || !V || !pmin) BAD("gpk_mc_pmin: need m, V and pmin");
    if ((rc = mc_check_shape(h, nb, np_, nf, 1, "gpk_mc_pmin"))) return rc;
    CK(cudaSetDevice(h->device));
    // scratch in doubles: m (nb x np), V (nb x nb), F (nb x nf), pmin (nb), then the status words
    const size_t om = 0, oV = om + (size_t)nb * np_, oF = oV + (size_t)nb * nb, oP = oF + (size_t)nb * nf, oS = oP + nb;
    if ((rc = ensure(h, h->mc.buf, oS * 8 + 2 * sizeof(int)))) return rc;
    double* b = ptr<double>(h->mc.buf);
    int* dst = (int*)(b + oS);
    cudaStream_t st = h->stream;
    CK(cudaMemcpyAsync(b + om, m, (size_t)nb * np_ * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b + oV, V, (size_t)nb * nb * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(dst, 0, 2 * sizeof(int), st));
    const long work = (long)nb * ((nf + 1) / 2);
    gpk_mc_draws_kernel<<<(unsigned)((work + 255) / 256), 256, 0, st>>>(seed, nb, nf, b + oF);
    CKL();
    if ((rc = mc_kernel_attrs(h))) return rc;
    gpk_mc_pmin_kernel<<<1, GPK_MC_THREADS, GPK_MC_SMEM, st>>>(b + om, nullptr, nullptr, np_, b + oV, nb, b + oF, nf,
                                                                 nullptr, nullptr, 0.0, nullptr, 0.0, nullptr, b + oP,
                                                                 nullptr, dst);
    CKL();
    CK(cudaMemcpyAsync(pmin, b + oP, (size_t)nb * 8, cudaMemcpyDeviceToHost, st));
    if ((rc = mc_stat_check(h, dst, "gpk_mc_pmin"))) return rc;
    if (n_jitter) *n_jitter = (int)h->mc.last_jitter;
    return GPK_OK;
}

int gpk_esmc_update(gpk_handle* h, const double* zb, int nb, const double* lmb, double sn2, const double* W, int np_,
                    int nf, unsigned long long seed, double* logP, double* pmin) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!zb || !lmb || !W) BAD("gpk_esmc_update: need zb, lmb and W");
    if ((rc = mc_check_shape(h, nb, np_, nf, 2, "gpk_esmc_update"))) return rc;
    for (int i = 0; i < nb; ++i)
        if (!std::isfinite(lmb[i])) BAD("lmb should not be infinite.");
    const int d = h->d;
    const size_t D = (size_t)nb;
    h->es.linv_serial = -1;                     // no update is current until this one completes
    std::vector<double> mu(D), V(D * D), pm(D);
    if ((rc = gpk_predict_cov(h, zb, nb, mu.data(), V.data()))) return rc;          // predict(zb, full_cov=True)
    McLayout L(nb, np_, d, nf);
    if ((rc = ensure(h, h->mc.state, L.total * 8))) return rc;
    double* st = ptr<double>(h->mc.state);
    cudaStream_t s = h->stream;
    CK(cudaMemcpyAsync(st + L.Mb, mu.data(), D * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(st + L.Vb, V.data(), D * D * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(st + L.W, W, (size_t)np_ * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(st + L.lmb, lmb, D * 8, cudaMemcpyHostToDevice, s));
    const long work = (long)nb * ((nf + 1) / 2);
    gpk_mc_draws_kernel<<<(unsigned)((work + 255) / 256), 256, 0, s>>>(seed, nb, nf, st + L.F);
    CKL();
    // pmin = joint_pmin(Mb, Vb, Nf) with Mb as (Nb, 1): one column of innovations
    if ((rc = ensure(h, h->mc.buf, D * 8))) return rc;
    if ((rc = mc_stat_reset(h))) return rc;
    if ((rc = mc_kernel_attrs(h))) return rc;
    gpk_mc_pmin_kernel<<<1, GPK_MC_THREADS, GPK_MC_SMEM, s>>>(st + L.Mb, nullptr, nullptr, 1, st + L.Vb, nb, st + L.F, nf,
                                                                nullptr, nullptr, 0.0, nullptr, 0.0, nullptr,
                                                                ptr<double>(h->mc.buf), nullptr, ptr<int>(h->mc.stat));
    CKL();
    CK(cudaMemcpyAsync(pm.data(), h->mc.buf.p, D * 8, cudaMemcpyDeviceToHost, s));
    if ((rc = mc_stat_check(h, ptr<int>(h->mc.stat), "gpk_esmc_update"))) return rc;
    // logP = log(pmin); H of the loss (information_gain.py:82), summed in index order
    std::vector<double> lp(D);
    double H = 0.0;
    for (size_t i = 0; i < D; ++i) {
        lp[i] = std::log(pm[i]);
        H += std::exp(lp[i]) * (lp[i] + lmb[i]);
    }
    H = -H;
    if ((rc = es_build_u(h, zb, nb, st + L.zb))) return rc;
    CK(cudaStreamSynchronize(s));
    h->es.nb = nb;
    h->es.np = np_;
    h->mc.nf = nf;
    h->es.sn2 = sn2;
    h->es.H = H;
    h->es.linv_serial = h->linv_serial;
    h->es.kind = ES_KIND_MC;
    if (logP) std::copy(lp.begin(), lp.end(), logP);
    if (pmin) std::copy(pm.begin(), pm.end(), pmin);
    return GPK_OK;
}

int gpk_esmc_compute_dev(gpk_handle* h, const void* d_Xs, long m, void* d_out) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!d_Xs || !d_out || m <= 0) BAD("gpk_esmc_compute_dev: need candidates and out");
    if ((rc = es_ready(h, nullptr, "gpk_esmc_compute", ES_KIND_MC))) return rc;
    CK(cudaSetDevice(h->device));
    if ((rc = mc_stat_reset(h))) return rc;
    return esmc_dev(h, (const double*)d_Xs, m, (double*)d_out, ptr<int>(h->mc.stat));
}

int gpk_esmc_compute(gpk_handle* h, const double* Xs, long m, double* out) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!Xs || !out || m <= 0) BAD("gpk_esmc_compute: need candidates and out");
    CK(cudaSetDevice(h->device));
    if ((rc = es_ready(h, nullptr, "gpk_esmc_compute", ES_KIND_MC))) return rc;
    if ((rc = ensure(h, h->es.in, (size_t)m * (h->d + 1) * 8))) return rc;
    double* dX = ptr<double>(h->es.in);
    double* dout = dX + (size_t)m * h->d;
    CK(cudaMemcpyAsync(dX, Xs, (size_t)m * h->d * 8, cudaMemcpyHostToDevice, h->stream));
    if ((rc = gpk_esmc_compute_dev(h, dX, m, dout))) return rc;
    CK(cudaMemcpyAsync(out, dout, (size_t)m * 8, cudaMemcpyDeviceToHost, h->stream));
    return mc_stat_check(h, ptr<int>(h->mc.stat), "gpk_esmc_compute");
}

int gpk_esmc_get_draws(gpk_handle* h, double* F) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!F) BAD("gpk_esmc_get_draws: null output");
    if ((rc = es_ready(h, nullptr, "gpk_esmc_get_draws", ES_KIND_MC))) return rc;
    CK(cudaSetDevice(h->device));
    const McLayout L(h->es.nb, h->es.np, h->d, h->mc.nf);
    CK(cudaMemcpyAsync(F, ptr<double>(h->mc.state) + L.F, (size_t)h->es.nb * h->mc.nf * 8, cudaMemcpyDeviceToHost,
                       h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_esmc_get_state(gpk_handle* h, double* Mb, double* Vb) {
    int rc = require(h, true, true, true);
    if (rc) return rc;
    if (!Mb || !Vb) BAD("gpk_esmc_get_state: null output");
    if ((rc = es_ready(h, nullptr, "gpk_esmc_get_state", ES_KIND_MC))) return rc;
    CK(cudaSetDevice(h->device));
    const int nb = h->es.nb;
    const McLayout L(nb, h->es.np, h->d, h->mc.nf);
    const double* st = ptr<double>(h->mc.state);
    CK(cudaMemcpyAsync(Mb, st + L.Mb, (size_t)nb * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(Vb, st + L.Vb, (size_t)nb * nb * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return GPK_OK;
}

int gpk_esmc_last_jitter(gpk_handle* h, long* n_jitter) {
    if (!h) return GPK_BAD_ARG;
    if (!n_jitter) BAD("gpk_esmc_last_jitter: null output");
    *n_jitter = h->mc.last_jitter;
    return GPK_OK;
}

int gpk_get_diag_profile(gpk_handle* h, long long* out34) {      // 64 entries
    if (!h || !out34) return GPK_BAD_ARG;
    if (!h->diag_prof || !h->dprof.p) BAD("gpk_get_diag_profile: set option diagprof = 1 first");
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaMemcpy(out34, h->dprof.p, 64 * 8, cudaMemcpyDeviceToHost));
    return GPK_OK;
}

int gpk_get_timings(gpk_handle* h, double* out /* 16 */) {
    if (!h || !out) return GPK_BAD_ARG;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < 16; ++i) out[i] = 0.0;
    float ms = 0.f;
    if (h->timing.fit_timed) {
        if (cudaEventElapsedTime(&ms, h->timing.ev[0], h->timing.ev[3]) == cudaSuccess) out[0] = ms;
        if (cudaEventElapsedTime(&ms, h->timing.ev[0], h->timing.ev[1]) == cudaSuccess) out[1] = ms;
        if (cudaEventElapsedTime(&ms, h->timing.ev[1], h->timing.ev[2]) == cudaSuccess) out[2] = ms;
    }
    if (h->linv_ready && cudaEventElapsedTime(&ms, h->timing.ev[4], h->timing.ev[5]) == cudaSuccess) out[3] = ms;
    if (h->timing.score_timed) {
        if (cudaEventElapsedTime(&ms, h->timing.ev[6], h->timing.ev[7]) == cudaSuccess) out[4] = ms;
        if (cudaEventElapsedTime(&ms, h->timing.ev[8], h->timing.ev[10]) == cudaSuccess) out[5] = ms;    // K* of the last chunk
        // variance GEMM: mean over the FULL-SIZE chunk launches of the last scoring call (the last chunk
        // is included only when it is the only one)
        double sum = 0.0;
        int cnt = 0;
        const int nfull = h->timing.last_nchunks > 1 ? h->timing.last_nchunks - 1 : h->timing.last_nchunks;
        for (int i = 0; i < nfull && i < (int)h->timing.ev_g0.size(); ++i)
            if (cudaEventElapsedTime(&ms, h->timing.ev_g0[i], h->timing.ev_g1[i]) == cudaSuccess) { sum += ms; ++cnt; }
        if (cnt > 0) out[6] = sum / cnt;
        if (cudaEventElapsedTime(&ms, h->timing.ev[11], h->timing.ev[12]) == cudaSuccess) out[7] = ms;   // epilogue, last chunk
    }
    cudaGetLastError();
    out[8] = h->timing.launches_var;
    out[9] = h->timing.launches_total;
    out[10] = h->oz.launches;
    out[11] = (double)h->oz.emax_host;
    out[13] = (double)OZ_PAIRS;
    out[14] = (double)h->oz.last_variant;
    return GPK_OK;
}

}  // extern "C"

#include "gpk_multi.inl"
