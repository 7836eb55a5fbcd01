// capi.cu -- the C ABI of libnufhe_b200.so (see include/nufhe_b200.h).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <nvtx3/nvToolsExt.h>
#include "../../include/nufhe_b200.h"
#include "kernels.cuh"
#include "index_lookup.cuh"
#include "compact.cuh"
#include "reencrypt.cuh"
#include "tables.h"

using namespace nb;

// smallest batch whose key switch runs on keyswitch_mma_kernel when the key is prepared (NUFHE_B200_KS_MMA_MIN
// overrides it)
constexpr size_t KS_MMA_MIN_DEFAULT = 256;

struct nb_ctx {
    int device;
    cudaStream_t stream;
    u64 *d_ph_fwd, *d_ph_inv;            // middle-twiddle tables [row][j2] of the transform passes
    u64 *d_ones512;                      // 512 * NTT(all-ones), natural order (bk_prepare)
    cplx *d_fft_tab;                     // tables of the FP64 step (tables.h: FftTables)
    // engine keys prepared on this context whose coefficients are centred 32-bit integers: they carry the spectra of
    // the FP64 step, which the throughput shape runs on them (begin, end of the key's rows)
    std::vector<std::pair<const u64 *, const u64 *>> spectral_keys;
    // multi-bit keys prepared on this context (nb_bk_prepare_multibit): 3 rows of spectra per group of two key bits,
    // which every launch with them runs on the FP64 step (begin, end of the key's rows)
    std::vector<std::pair<const u64 *, const u64 *>> multibit_keys;
    // slots of the multi-key machine filled by nb_mk_bk_expand: engine key rows whose FP64 part only is written (their
    // NTT planes are garbage), so only the nb_mk_* bootstraps accept them (begin, end of the slot's rows)
    std::vector<std::pair<const u64 *, const u64 *>> mk_slots;
    int fft;                             // developer knob: 0 keeps the NTT step for every key
    int sm_count;
    size_t wide_max;                     // largest batch launched in the wide (1 ciphertext / 256 threads) shape
    size_t wide2_max;                    // largest batch launched in the wide2 (1 ciphertext / 512 threads / SM) shape
    size_t pair_max;                     // largest batch launched in the pair shape (1 ciphertext / cluster of 2 CTAs on 2 SMs)
    int pair_async;                      // pair shape: exchange by st.async + mbarrier (1) or plain stores + barrier.cluster (0)
    int max_chunks;                      // upper bound on the chunks a chain is cut into (1 = no time slicing)
    unsigned *d_sched;                   // work-queue state of the fused bootstrap (kernels.cuh: BlindRotateArgs)
    size_t sched_words;
    int32_t *d_state;                    // parked accumulators of time-sliced launches
    size_t state_words;
    float *d_cv_blocks;                  // block sums of the key-switch variances (split launches)
    // key-switch keys prepared on this context for keyswitch_mma_kernel (nb_ks_prepare): (ks_a, ks_b) -> planes
    struct KsKey { const int32_t *ks_a, *ks_b; const uint8_t *planes; };
    std::vector<KsKey> ks_keys;
    size_t ks_mma_min;                   // smallest batch whose key switch runs as the tensor-core GEMM
    u64 *d_index_tmp;                    // nb_index_prepare: field elements of one chunk of selector rows
    size_t index_tmp_words;
    size_t cv_words;
    int force_chunks;                    // developer knob: chunk count of every multi-wave launch (0 = automatic)
    int stagger_cycles;                  // start-up offset of the second CTA per SM in single-wave launches
    void *d_mk;                          // multi-key calls: the uploaded tenant tables (nb_mk_*)
    size_t mk_bytes;
    std::string err;
};

static int fail(nb_ctx *ctx, int code, const std::string &msg)
{
    if (ctx) ctx->err = msg;
    return code;
}

static int check(nb_ctx *ctx, cudaError_t e, const char *what)
{
    if (e == cudaSuccess) return NB_OK;
    return fail(ctx, NB_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

#define NB_TRY(expr)                         \
    do {                                     \
        int _rc = (expr);                    \
        if (_rc != NB_OK) return _rc;        \
    } while (0)

static int launch_check(nb_ctx *ctx, const char *what) { return check(ctx, cudaGetLastError(), what); }

// Every entry point works on ctx->device and leaves the caller's current device as it found it (one process may
// hold several engines, one per GPU, like the reference's one-Context-per-device model, api_high_level.py:153-181).
struct DeviceGuard {
    int prev = -1;
    bool switched = false;
    cudaError_t err;
    explicit DeviceGuard(int dev)
    {
        err = cudaGetDevice(&prev);
        if (err == cudaSuccess && prev != dev) {
            err = cudaSetDevice(dev);
            switched = err == cudaSuccess;
        }
    }
    ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
};
// NVTX range around the launches of one entry point (prologue + blind rotation, key switch, transforms, ...): shows up
// in Nsight Systems / `ncu --nvtx`; a no-op costing two library calls when no tool is attached (nvtx3 is header-only).
struct NvtxRange {
    explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

#define NB_ON_DEVICE(ctx)                   \
    DeviceGuard _guard((ctx)->device);      \
    NB_TRY(check(ctx, _guard.err, "cudaSetDevice"))

// A CTA of the fused bootstrap's work queue may wait for work that another resident CTA produces, so all the
// sm_count x CTAS_PER_SM CTAs a launch is sized for must be co-resident: fail at context creation instead of hanging.
// (the gate kernel and the programmable-bootstrap kernel of each shape)
template <class Cfg, bool MB = false> static int check_resident(nb_ctx *ctx)
{
    for (auto kernel : {blind_rotate_kernel<Cfg, false, MB>, blind_rotate_kernel<Cfg, true, MB>}) {
        int n = 0;
        NB_TRY(check(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)br_smem_bytes<Cfg>()),
                     "cudaFuncSetAttribute(blind_rotate)"));
        NB_TRY(check(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, Cfg::THREADS, br_smem_bytes<Cfg>()),
                     "cudaOccupancyMaxActiveBlocksPerMultiprocessor"));
        if (n < Cfg::CTAS_PER_SM)
            return fail(ctx, NB_EUNSUPPORTED, "blind_rotate_kernel: " + std::to_string(n) + " resident CTAs per SM, the work "
                                              "queue needs " + std::to_string(Cfg::CTAS_PER_SM));
    }
    return NB_OK;
}

extern "C" {

int nb_ctx_create(int device, void *stream, nb_ctx **out)
{
    if (!out) return NB_EINVAL;
    *out = nullptr;
    nb_ctx *ctx = new nb_ctx();
    ctx->device = device;
    ctx->stream = (cudaStream_t)stream;
    ctx->d_ph_fwd = ctx->d_ph_inv = ctx->d_ones512 = nullptr;
    ctx->d_fft_tab = nullptr;
    ctx->d_sched = nullptr; ctx->d_state = nullptr; ctx->sched_words = ctx->state_words = 0;
    ctx->d_cv_blocks = nullptr; ctx->cv_words = 0;
    ctx->d_index_tmp = nullptr; ctx->index_tmp_words = 0;
    ctx->d_mk = nullptr; ctx->mk_bytes = 0;
    *out = ctx;   // returned even on failure so that nb_last_error() can be read; caller destroys it
    NB_ON_DEVICE(ctx);
    cudaDeviceProp prop;
    NB_TRY(check(ctx, cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties"));
    ctx->sm_count = prop.multiProcessorCount;
    {
        const char *e = getenv("NUFHE_B200_MAX_CHUNKS");  // developer knob: 1 disables the time slicing of chains
        ctx->max_chunks = e ? atoi(e) : 50;
        if (ctx->max_chunks < 1) ctx->max_chunks = 1;
        e = getenv("NUFHE_B200_FORCE_CHUNKS");
        ctx->force_chunks = e ? atoi(e) : 0;
        e = getenv("NUFHE_B200_STAGGER");
        ctx->stagger_cycles = e ? atoi(e) : 12000;        // about a quarter of a CMux step (measured best of 0 / 12k / 24k / 36k)
        e = getenv("NUFHE_B200_FFT");
        ctx->fft = e ? atoi(e) : 1;
    }
    if (const char *e = getenv("NUFHE_B200_FORCE_RARE_PATH")) {
        // test knob: run the canonicalisation fix-up of the deferred-canonicalisation phases on every task
        if (atoi(e)) {
            const u32 zero = 0;
            NB_TRY(check(ctx, cudaMemcpyToSymbol(nb_c_canon_trigger, &zero, sizeof(zero)), "cudaMemcpyToSymbol"));
        }
    }
    if (prop.major != 9 || prop.minor != 0)     // sm_90a code loads on compute capability 9.0 only
        return fail(ctx, NB_EUNSUPPORTED, "libnufhe_b200 is built for sm_90a only; device is sm_" +
                                              std::to_string(prop.major) + std::to_string(prop.minor));
    PhaseTables pt;
    NB_TRY(check(ctx, cudaMalloc(&ctx->d_ph_fwd, NTT_N * sizeof(u64)), "cudaMalloc"));
    NB_TRY(check(ctx, cudaMalloc(&ctx->d_ph_inv, NTT_N * sizeof(u64)), "cudaMalloc"));
    NB_TRY(check(ctx, cudaMemcpy(ctx->d_ph_fwd, pt.fwd.data(), NTT_N * sizeof(u64), cudaMemcpyHostToDevice), "memcpy"));
    NB_TRY(check(ctx, cudaMemcpy(ctx->d_ph_inv, pt.inv.data(), NTT_N * sizeof(u64), cudaMemcpyHostToDevice), "memcpy"));
    NB_TRY(check(ctx, cudaMalloc(&ctx->d_ones512, NTT_N * sizeof(u64)), "cudaMalloc"));
    NB_TRY(check(ctx, cudaMemcpy(ctx->d_ones512, pt.ones512.data(), NTT_N * sizeof(u64), cudaMemcpyHostToDevice), "memcpy"));
    {
        FftTables ft;
        NB_TRY(check(ctx, cudaMalloc(&ctx->d_fft_tab, (FFT_TAB_CPLX + FFT_ROOTS) * sizeof(cplx)), "cudaMalloc"));
        NB_TRY(check(ctx, cudaMemcpy(ctx->d_fft_tab, ft.tab.data(), FFT_TAB_CPLX * sizeof(cplx), cudaMemcpyHostToDevice), "memcpy"));
        NB_TRY(check(ctx, cudaMemcpy(ctx->d_fft_tab + FFT_TAB_ROOTS, ft.roots.data(), FFT_ROOTS * sizeof(cplx), cudaMemcpyHostToDevice), "memcpy"));
    }
    // (check_resident sets the shared-memory limit of the single-CTA shapes)
    for (auto kernel : {blind_rotate_pair_kernel<true>, blind_rotate_pair_kernel<false>, blind_rotate_pair_kernel<true, true>,
                        blind_rotate_pair_kernel<false, true>})
        NB_TRY(check(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BR_PAIR_SMEM_BYTES),
                     "cudaFuncSetAttribute(blind_rotate pair)"));
    NB_TRY(check(ctx, cudaFuncSetAttribute(keyswitch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)KS_SMEM_BYTES), "cudaFuncSetAttribute(keyswitch)"));
    NB_TRY(check(ctx, cudaFuncSetAttribute(keyswitch_grouped_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)KS_SMEM_BYTES), "cudaFuncSetAttribute(keyswitch_grouped)"));
    NB_TRY(check(ctx, cudaFuncSetAttribute(keyswitch_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)KM_SMEM_BYTES), "cudaFuncSetAttribute(keyswitch_mma)"));
    {
        // below this batch the split launch of keyswitch_kernel is faster than the GEMM
        const char *e = getenv("NUFHE_B200_KS_MMA_MIN");
        ctx->ks_mma_min = e ? (size_t)atoll(e) : KS_MMA_MIN_DEFAULT;
    }
    NB_TRY(check_resident<BrDefault>(ctx));
    NB_TRY(check_resident<BrWide>(ctx));
    NB_TRY(check_resident<BrWide2>(ctx));
    NB_TRY(check_resident<BrFft>(ctx));
    NB_TRY((check_resident<BrFft, true>(ctx)));
    NB_TRY(check_resident<BrFftMk>(ctx));
    for (auto kernel : {index_lookup_kernel<false>, index_lookup_kernel<true>, index_lookup_kernel<false, true>,
                        index_lookup_kernel<true, true>})
        NB_TRY(check(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)br_smem_bytes<BrFft>()),
                     "cudaFuncSetAttribute(index_lookup)"));
    for (auto kernel : {index_write_kernel<false>, index_write_kernel<true>})
        NB_TRY(check(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)br_smem_bytes<BrFft>()),
                     "cudaFuncSetAttribute(index_write)"));
    {   // batches that fit one wave of wide CTAs (one ciphertext on 256 threads) take the low-latency shape
        const char *e = getenv("NUFHE_B200_WIDE_MAX");
        // up to one wave the wide shape has the shortest step; between one and ~1.7 waves it still wins, time-sliced
        // over all SMs, against a throughput-shape launch that leaves half of the SMs with one CTA (H100 SXM: 11.8
        // against 13.0 ms at 448 ciphertexts, 14.4 against 12.8 at 528)
        ctx->wide_max = e ? (size_t)atoll(e) : (size_t)ctx->sm_count * BrWide::CTAS_PER_SM * 17 / 10;
        // up to 1.5 ciphertexts per SM: 512 threads per ciphertext, forward phases split as well (lowest latency;
        // whole gate_nand on an H100 SXM, median of 7 runs in one process, shapes alternated: 512 threads 6.3 / 7.3 /
        // 8.6 ms at 198 / 231 / 264 ciphertexts against 8.0 / 8.1 / 7.3 for 256 threads, spread within 3 %; the
        // 256-thread shape is slower in partial waves than in the full one with or without the start-up stagger)
        e = getenv("NUFHE_B200_WIDE2_MAX");
        ctx->wide2_max = e ? (size_t)atoll(e) : (size_t)ctx->sm_count * 3 / 2;
        // up to one cluster of two SMs per ciphertext: the pair shape, while all clusters are resident at once (the
        // driver knows how many pairs of SMs it can form)
        e = getenv("NUFHE_B200_PAIR_ASYNC");
        ctx->pair_async = e ? atoi(e) : 1;
        e = getenv("NUFHE_B200_PAIR_MAX");
        if (e) {
            ctx->pair_max = (size_t)atoll(e);
        } else {
            cudaLaunchConfig_t cfg = {};
            cudaLaunchAttribute attr;
            attr.id = cudaLaunchAttributeClusterDimension;
            attr.val.clusterDim.x = 2; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
            cfg.gridDim = dim3(2 * (unsigned)ctx->sm_count); cfg.blockDim = dim3(PAIR_THREADS);
            cfg.dynamicSmemBytes = BR_PAIR_SMEM_BYTES; cfg.attrs = &attr; cfg.numAttrs = 1;
            int clusters = 0;
            if (cudaOccupancyMaxActiveClusters(&clusters, blind_rotate_pair_kernel<true>, &cfg) != cudaSuccess) {
                cudaGetLastError();
                clusters = 0;
            }
            // on an H100 SXM the pair shape beats the 512-thread shape whenever all clusters are resident: 2.8 / 3.1 /
            // 3.7 / 3.7 ms at batch 1 / 16 / 48 / 64 against 4.2 - 4.3 ms
            ctx->pair_max = clusters > 0 ? (size_t)clusters : 0;
        }
        if (getenv("NUFHE_B200_VERBOSE"))
            fprintf(stderr, "nufhe_b200: device %d, %d SMs; fused-kernel shapes by batch: pair <= %zu, wide2 <= %zu, wide <= %zu\n",
                    ctx->device, ctx->sm_count, ctx->pair_max, ctx->wide2_max, ctx->wide_max);
    }
    NB_TRY(check(ctx, cudaFuncSetAttribute(ntt_forward_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ntt_smem_bytes(NTT_RAW_I32_BYTES)), "attr"));
    NB_TRY(check(ctx, cudaFuncSetAttribute(ntt_forward_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ntt_smem_bytes(NTT_RAW_U64_BYTES)), "attr"));
    NB_TRY(check(ctx, cudaFuncSetAttribute(ntt_inverse_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ntt_smem_bytes(NTT_RAW_U64_BYTES)), "attr"));
    NB_TRY(check(ctx, cudaFuncSetAttribute(ntt_inverse_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ntt_smem_bytes(NTT_RAW_U64_BYTES)), "attr"));
    NB_TRY(check(ctx, cudaFuncSetAttribute(reencrypt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)reenc_smem_bytes()), "attr"));
    return NB_OK;
}

void nb_ctx_destroy(nb_ctx *ctx)
{
    if (!ctx) return;
    DeviceGuard guard(ctx->device);
    if (ctx->d_ph_fwd) cudaFree(ctx->d_ph_fwd);
    if (ctx->d_ph_inv) cudaFree(ctx->d_ph_inv);
    if (ctx->d_ones512) cudaFree(ctx->d_ones512);
    if (ctx->d_fft_tab) cudaFree(ctx->d_fft_tab);
    if (ctx->d_sched) cudaFree(ctx->d_sched);
    if (ctx->d_state) cudaFree(ctx->d_state);
    if (ctx->d_cv_blocks) cudaFree(ctx->d_cv_blocks);
    if (ctx->d_index_tmp) cudaFree(ctx->d_index_tmp);
    if (ctx->d_mk) cudaFree(ctx->d_mk);
    delete ctx;
}

const char *nb_last_error(const nb_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int nb_ctx_set_stream(nb_ctx *ctx, void *stream)
{
    if (!ctx) return NB_EINVAL;
    ctx->stream = (cudaStream_t)stream;
    return NB_OK;
}

int nb_ctx_synchronize(nb_ctx *ctx)
{
    if (!ctx) return NB_EINVAL;
    NB_ON_DEVICE(ctx);
    return check(ctx, cudaStreamSynchronize(ctx->stream), "cudaStreamSynchronize");
}

const char *nb_build_info(void)
{
    static std::string info;
    if (info.empty()) {
        char buf[512];
        cudaFuncAttributes a{}, b{}, c{};
        cudaFuncGetAttributes(&a, blind_rotate_kernel<BrDefault>);
        cudaFuncGetAttributes(&b, ntt_forward_kernel<true>);
        cudaFuncGetAttributes(&c, keyswitch_kernel);
        snprintf(buf, sizeof(buf),
                 "nufhe_b200 sm_90a; blind_rotate: %d regs, %zu B dyn smem, %d thr/CTA, %d ct/CTA; "
                 "ntt_forward: %d regs; keyswitch: %d regs, tile %d",
                 a.numRegs, BR2_SMEM_BYTES, BR2_THREADS, BR2_CT, b.numRegs, c.numRegs, KS_TILE);
        info = buf;
    }
    return info.c_str();
}

static int ntt_grid(nb_ctx *ctx, size_t batch)
{
    size_t blocks = (batch + NTT_SWEEP_POLYS - 1) / NTT_SWEEP_POLYS;
    size_t cap = (size_t)ctx->sm_count * NTT_CTAS;   // persistent: NTT_CTAS CTAs per SM, grid-stride over the batch
    return (int)(blocks < cap ? blocks : cap);
}

int nb_ntt_forward_i32(nb_ctx *ctx, const int32_t *in, uint64_t *out, size_t batch)
{
    if (!ctx) return NB_EINVAL;
    if (batch == 0) return NB_OK;
    if (!in || !out) return fail(ctx, NB_EINVAL, "nb_ntt_forward_i32: null argument");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:ntt_forward");
    ntt_forward_kernel<true><<<ntt_grid(ctx, batch), NTT_SWEEP_THREADS, ntt_smem_bytes(NTT_RAW_I32_BYTES), ctx->stream>>>(in, (u64 *)out, ctx->d_ph_fwd, batch);
    return launch_check(ctx, "ntt_forward_kernel<i32>");
}

int nb_ntt_forward_u64(nb_ctx *ctx, const uint64_t *in, uint64_t *out, size_t batch)
{
    if (!ctx) return NB_EINVAL;
    if (batch == 0) return NB_OK;
    if (!in || !out) return fail(ctx, NB_EINVAL, "nb_ntt_forward_u64: null argument");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:ntt_forward");
    ntt_forward_kernel<false><<<ntt_grid(ctx, batch), NTT_SWEEP_THREADS, ntt_smem_bytes(NTT_RAW_U64_BYTES), ctx->stream>>>(in, (u64 *)out, ctx->d_ph_fwd, batch);
    return launch_check(ctx, "ntt_forward_kernel<u64>");
}

int nb_ntt_inverse_i32(nb_ctx *ctx, const uint64_t *in, int32_t *out, size_t batch)
{
    if (!ctx) return NB_EINVAL;
    if (batch == 0) return NB_OK;
    if (!in || !out) return fail(ctx, NB_EINVAL, "nb_ntt_inverse_i32: null argument");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:ntt_inverse");
    ntt_inverse_kernel<true><<<ntt_grid(ctx, batch), NTT_SWEEP_THREADS, ntt_smem_bytes(NTT_RAW_U64_BYTES), ctx->stream>>>((const u64 *)in, out, ctx->d_ph_inv, batch);
    return launch_check(ctx, "ntt_inverse_kernel<i32>");
}

int nb_ntt_inverse_u64(nb_ctx *ctx, const uint64_t *in, uint64_t *out, size_t batch)
{
    if (!ctx) return NB_EINVAL;
    if (batch == 0) return NB_OK;
    if (!in || !out) return fail(ctx, NB_EINVAL, "nb_ntt_inverse_u64: null argument");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:ntt_inverse");
    ntt_inverse_kernel<false><<<ntt_grid(ctx, batch), NTT_SWEEP_THREADS, ntt_smem_bytes(NTT_RAW_U64_BYTES), ctx->stream>>>((const u64 *)in, out, ctx->d_ph_inv, batch);
    return launch_check(ctx, "ntt_inverse_kernel<u64>");
}

int nb_ff_elementwise(nb_ctx *ctx, int op, const uint64_t *a, const uint64_t *b, uint64_t *out, size_t n,
                      size_t b_period)
{
    if (!ctx || !a || !out) return fail(ctx, NB_EINVAL, "nb_ff_elementwise: null argument");
    if (op < 0 || op > NB_FF_LSH_CONST) return fail(ctx, NB_EINVAL, "nb_ff_elementwise: unknown op");
    if (op != NB_FF_PREPARE && !b) return fail(ctx, NB_EINVAL, "nb_ff_elementwise: binary op needs b");
    if (n == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    size_t blocks = (n + 255) / 256, cap = (size_t)ctx->sm_count * 16;
    ff_elementwise_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>(
        op, (const u64 *)a, (const u64 *)b, (u64 *)out, n, b_period);
    return launch_check(ctx, "ff_elementwise_kernel");
}

size_t nb_bk_row_u64(void) { return BK_ROW_U64; }
size_t nb_bk_multibit_row_u64(void) { return BK_FFT_U64; }

}  // extern "C"

// forget the registrations of keys that [begin, end) overwrites
static void forget_keys(nb_ctx *ctx, const u64 *begin, const u64 *end)
{
    for (auto *keys : {&ctx->spectral_keys, &ctx->multibit_keys, &ctx->mk_slots})
        for (size_t i = 0; i < keys->size();) {
            if ((*keys)[i].first < end && begin < (*keys)[i].second) keys->erase(keys->begin() + i);
            else i++;
        }
}

extern "C" {

int nb_bk_prepare(nb_ctx *ctx, const uint64_t *bk_ref, uint64_t *bk_int, size_t rows)
{
    if (!ctx || !bk_ref || !bk_int) return fail(ctx, NB_EINVAL, "nb_bk_prepare: null argument");
    if (rows == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:bk_prepare");
    size_t total = rows * NTT_N, blocks = (total + 255) / 256, cap = (size_t)ctx->sm_count * 16;
    bk_prepare_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>((const u64 *)bk_ref, (u64 *)bk_int,
                                                                                  ctx->d_ones512, rows);
    NB_TRY(launch_check(ctx, "bk_prepare_kernel"));
    // the FP64 part of every row: key polynomials back to coefficients (plain form, inverse transform), integrality
    // check, 16-bit split, spectra (kernels.cuh: bk_spectra_kernel)
    const u64 *key_begin = (const u64 *)bk_int, *key_end = key_begin + rows * BK_ROW_U64;
    forget_keys(ctx, key_begin, key_end);
    const size_t polys = rows * 8, words = polys * NTT_N;
    u64 *tmp = nullptr;
    NB_TRY(check(ctx, cudaMalloc(&tmp, 2 * words * sizeof(u64) + sizeof(int)), "cudaMalloc(bk_prepare)"));
    int *d_flag = (int *)(tmp + 2 * words), not_integral = 0;
    int rc = check(ctx, cudaMemsetAsync(d_flag, 0, sizeof(int), ctx->stream), "cudaMemsetAsync");
    if (rc == NB_OK) {
        blocks = (words + 255) / 256;
        bk_plain_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>((const u64 *)bk_ref, tmp, words);
        ntt_inverse_kernel<false><<<ntt_grid(ctx, polys), NTT_SWEEP_THREADS, ntt_smem_bytes(NTT_RAW_U64_BYTES), ctx->stream>>>(tmp, tmp + words, ctx->d_ph_inv, polys);
        bk_spectra_kernel<<<(unsigned)polys, 64, 0, ctx->stream>>>(tmp + words, (u64 *)bk_int, ctx->d_fft_tab, d_flag, BK_ROW_U64, BK_NTT_U64);
        rc = launch_check(ctx, "bk_spectra_kernel");
    }
    if (rc == NB_OK) rc = check(ctx, cudaMemcpyAsync(&not_integral, d_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream), "cudaMemcpyAsync");
    if (rc == NB_OK) rc = check(ctx, cudaStreamSynchronize(ctx->stream), "cudaStreamSynchronize");
    cudaFree(tmp);
    NB_TRY(rc);
    if (!not_integral) ctx->spectral_keys.emplace_back(key_begin, key_end);
    return NB_OK;
}

int nb_bk_prepare_multibit(nb_ctx *ctx, const uint64_t *bk_ref, uint64_t *bk_mb, size_t groups)
{
    if (!ctx || !bk_ref || !bk_mb) return fail(ctx, NB_EINVAL, "nb_bk_prepare_multibit: null argument");
    if (groups == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:bk_prepare_multibit");
    const u64 *key_begin = (const u64 *)bk_mb, *key_end = key_begin + 3 * groups * BK_FFT_U64;
    forget_keys(ctx, key_begin, key_end);
    // as the FP64 part of nb_bk_prepare: coefficients (plain form, inverse transform), integrality check, 16-bit split,
    // spectra; only the spectra are stored
    const size_t polys = 3 * groups * 8, words = polys * NTT_N;
    const size_t blocks = (words + 255) / 256, cap = (size_t)ctx->sm_count * 16;
    u64 *tmp = nullptr;
    NB_TRY(check(ctx, cudaMalloc(&tmp, 2 * words * sizeof(u64) + sizeof(int)), "cudaMalloc(bk_prepare_multibit)"));
    int *d_flag = (int *)(tmp + 2 * words), not_integral = 0;
    int rc = check(ctx, cudaMemsetAsync(d_flag, 0, sizeof(int), ctx->stream), "cudaMemsetAsync");
    if (rc == NB_OK) {
        bk_plain_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>((const u64 *)bk_ref, tmp, words);
        ntt_inverse_kernel<false><<<ntt_grid(ctx, polys), NTT_SWEEP_THREADS, ntt_smem_bytes(NTT_RAW_U64_BYTES), ctx->stream>>>(tmp, tmp + words, ctx->d_ph_inv, polys);
        bk_spectra_kernel<<<(unsigned)polys, 64, 0, ctx->stream>>>(tmp + words, (u64 *)bk_mb, ctx->d_fft_tab, d_flag, BK_FFT_U64, 0);
        rc = launch_check(ctx, "bk_spectra_kernel(multi-bit)");
    }
    if (rc == NB_OK) rc = check(ctx, cudaMemcpyAsync(&not_integral, d_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream), "cudaMemcpyAsync");
    if (rc == NB_OK) rc = check(ctx, cudaStreamSynchronize(ctx->stream), "cudaStreamSynchronize");
    cudaFree(tmp);
    NB_TRY(rc);
    // a multi-bit key has no NTT form to fall back on
    if (not_integral) return fail(ctx, NB_EINVAL, "nb_bk_prepare_multibit: key coefficients are not centred 32-bit integers");
    ctx->multibit_keys.emplace_back(key_begin, key_end);
    return NB_OK;
}

}  // extern "C"

// Chunks per chain for `chains` chains on `slots` resident CTAs (kernels.cuh: blind_rotate_kernel).  One wave or
// less needs no slicing.  Otherwise the launch takes ceil(chains * C / slots) rounds of ceil(n / C) steps; each chunk
// also pays for parking / fetching the accumulators (modelled as 0.1 step here).
static int pick_chunks(size_t chains, size_t slots, int n, int max_chunks)
{
    if (chains <= slots || n <= 1 || max_chunks <= 1) return 1;
    int best = 1;
    double best_cost = 0;
    for (int c = 1; c <= max_chunks && c <= n / 8; c++) {
        const int steps = (n + c - 1) / c;
        const int chunks = (n + steps - 1) / steps;
        const double rounds = (double)((chains * (size_t)chunks + slots - 1) / slots);
        const double cost = rounds * (steps + 0.1);
        if (c == 1 || cost < best_cost * 0.995) { best = chunks; best_cost = cost; }
    }
    return best;
}

static int reserve_words(nb_ctx *ctx, void **buf, size_t *have, size_t want, size_t elem)
{
    if (*have >= want) return NB_OK;
    if (*buf) NB_TRY(check(ctx, cudaFree(*buf), "cudaFree"));
    *buf = nullptr; *have = 0;
    const size_t grow = want + want / 4;
    NB_TRY(check(ctx, cudaMalloc(buf, grow * elem), "cudaMalloc(work queue)"));
    *have = grow;
    return NB_OK;
}

// MB: a multi-bit key, whose chains are p.n / 2 groups long
template <class Cfg, bool MB = false> static int launch_br_cfg(nb_ctx *ctx, BlindRotateArgs &p)
{
    const size_t slots = (size_t)ctx->sm_count * Cfg::CTAS_PER_SM;
    const size_t chains = (p.batch + Cfg::CT - 1) / Cfg::CT;
    const int nsteps = MB ? p.n / 2 : p.n;
    int chunks = p.plain ? 1 : pick_chunks(chains, slots, nsteps, ctx->max_chunks);
    if (!p.plain && ctx->force_chunks > 0 && chains > slots) chunks = ctx->force_chunks < nsteps ? ctx->force_chunks : nsteps;
    p.chains = (unsigned)chains;
    p.steps_per_chunk = p.plain ? 1 : (nsteps + chunks - 1) / chunks;
    chunks = p.plain ? 1 : (nsteps + p.steps_per_chunk - 1) / p.steps_per_chunk;
    p.chunks = (unsigned)chunks;
    p.sched = nullptr; p.state = nullptr;
    p.sm_count = ctx->sm_count; p.stagger_cycles = ctx->stagger_cycles;
    p.fft_tab = ctx->d_fft_tab;
    size_t grid = chains;
    if (chains > slots) {
        // more than one wave: persistent CTAs pull (chain, chunk) tickets
        // ready queue: head, tail, then one entry per (chain, chunk); entries of first chunks stay 0 (implicit)
        const size_t entries = chunks > 1 ? chains * (size_t)chunks : 0;
        NB_TRY(reserve_words(ctx, (void **)&ctx->d_sched, &ctx->sched_words, BR_SCHED_HEADER + entries, sizeof(unsigned)));
        if (chunks > 1)
            NB_TRY(reserve_words(ctx, (void **)&ctx->d_state, &ctx->state_words, chains * Cfg::CT * 2 * NTT_N, sizeof(int32_t)));
        NB_TRY(check(ctx, cudaMemsetAsync(ctx->d_sched, 0, (BR_SCHED_HEADER + entries) * sizeof(unsigned), ctx->stream), "cudaMemsetAsync"));
        p.sched = ctx->d_sched; p.state = ctx->d_state;
        grid = slots;
    }
    if (p.tv) blind_rotate_kernel<Cfg, true, MB><<<(int)grid, Cfg::THREADS, br_smem_bytes<Cfg>(), ctx->stream>>>(p, ctx->d_ph_fwd, ctx->d_ph_inv);
    else blind_rotate_kernel<Cfg, false, MB><<<(int)grid, Cfg::THREADS, br_smem_bytes<Cfg>(), ctx->stream>>>(p, ctx->d_ph_fwd, ctx->d_ph_inv);
    return NB_OK;
}

// One launch of the fused kernel in the shape that suits the batch: "wide" CTAs (1 ciphertext on 256 threads,
// shortest step) while the batch fits one wave of them, else 2 ciphertexts per CTA (highest throughput), with the FP64
// step when the key has spectra.
static int launch_br(nb_ctx *ctx, BlindRotateArgs &p)
{
    for (const auto &k : ctx->multibit_keys) {
        if (p.bk < k.first || k.second <= p.bk) continue;
        // a multi-bit key: the FP64 throughput shape at every batch size.  The explicit-accumulator calls
        // (nb_blind_rotate, nb_external_product) have the per-bit semantics of the reference's key, which this key lacks.
        if (p.plain || p.accum || p.bara)
            return fail(ctx, NB_EUNSUPPORTED, "a multi-bit bootstrap key serves the fused bootstrap entry points only");
        if (p.n % 2 || p.bk + (size_t)(p.n / 2) * 3 * BK_FFT_U64 > k.second)
            return fail(ctx, NB_EINVAL, "the multi-bit key has fewer groups than n / 2, or n is odd");
        return launch_br_cfg<BrFft, true>(ctx, p);
    }
    if (!p.plain && p.n > 0 && p.batch <= ctx->pair_max) {
        p.sched = nullptr; p.state = nullptr; p.chains = (unsigned)p.batch; p.chunks = 1; p.steps_per_chunk = p.n;
        p.sm_count = ctx->sm_count; p.stagger_cycles = 0;
        auto kernel = p.tv ? (ctx->pair_async ? blind_rotate_pair_kernel<true, true> : blind_rotate_pair_kernel<false, true>)
                           : (ctx->pair_async ? blind_rotate_pair_kernel<true> : blind_rotate_pair_kernel<false>);
        kernel<<<(unsigned)(2 * p.batch), PAIR_THREADS, BR_PAIR_SMEM_BYTES, ctx->stream>>>(p, ctx->d_ph_fwd, ctx->d_ph_inv);
        return NB_OK;
    }
    if (p.batch <= ctx->wide2_max) return launch_br_cfg<BrWide2>(ctx, p);
    if (p.batch <= ctx->wide_max) return launch_br_cfg<BrWide>(ctx, p);
    if (ctx->fft) {
        // the FP64 step needs the spectra of every row the launch reads: all of them must come from one nb_bk_prepare
        // call on this context whose key had integral coefficients (rows prepared by other calls may have none)
        const u64 *end = p.bk + (size_t)(p.plain ? 1 : p.n) * BK_ROW_U64;
        for (const auto &k : ctx->spectral_keys)
            if (k.first <= p.bk && end <= k.second) return launch_br_cfg<BrFft>(ctx, p);
    }
    return launch_br_cfg<BrDefault>(ctx, p);
}

extern "C" {

int nb_ctx_reserve(nb_ctx *ctx, size_t batch)
{
    if (!ctx) return NB_EINVAL;
    NB_ON_DEVICE(ctx);
    // everything launch_br_cfg / nb_keyswitch could ask for with up to `batch` ciphertexts (2 * batch for gate_mux's
    // double launch, B * 2^L for the key switch of nb_bootstrap_lut_extract's samples, is the caller's business): after
    // this, those calls never allocate, so they can be captured
    NB_TRY(reserve_words(ctx, (void **)&ctx->d_sched, &ctx->sched_words, BR_SCHED_HEADER + (batch + 1) * (size_t)ctx->max_chunks, sizeof(unsigned)));
    NB_TRY(reserve_words(ctx, (void **)&ctx->d_state, &ctx->state_words, (batch + 2) * 2 * NTT_N, sizeof(int32_t)));
    NB_TRY(reserve_words(ctx, (void **)&ctx->d_cv_blocks, &ctx->cv_words, batch * KS_CV_BLOCKS, sizeof(float)));
    return NB_OK;
}

int nb_external_product(nb_ctx *ctx, int32_t *accum, const uint64_t *bk_int, size_t bk_row, size_t batch)
{
    if (ctx && batch == 0) return NB_OK;     // nothing to do: empty arrays have no storage to check
    if (!ctx || !accum || !bk_int) return fail(ctx, NB_EINVAL, "nb_external_product: null argument");
    if (batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:external_product");
    BlindRotateArgs p{};
    p.accum = accum; p.accum_out = accum; p.bk = (const u64 *)bk_int + bk_row * BK_ROW_U64;
    p.plain = 1; p.batch = batch;
    NB_TRY(launch_br(ctx, p));
    return launch_check(ctx, "blind_rotate_kernel(plain external product)");
}

}  // extern "C"

static int launch_blind_rotate(nb_ctx *ctx, BlindRotateArgs &p)
{
    if (p.n <= 0 || p.n > LWE_N_MAX) return fail(ctx, NB_EUNSUPPORTED, "LWE dimension out of range");
    // the LUT kernels have one job and read no explicit accumulator
    if (p.tv && (p.job_batch || p.accum || p.bara)) return fail(ctx, NB_EINVAL, "a test vector takes a single gate-style job");
    if (p.batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:gate_prologue+blind_rotate+extract");
    NB_TRY(launch_br(ctx, p));
    return launch_check(ctx, "blind_rotate_kernel");
}

// copy `bytes` of host data into the context's multi-key scratch (stream-ordered after every earlier launch that reads it)
static int mk_upload(nb_ctx *ctx, const void *host, size_t bytes)
{
    NB_TRY(reserve_words(ctx, &ctx->d_mk, &ctx->mk_bytes, bytes, 1));
    return check(ctx, cudaMemcpyAsync(ctx->d_mk, host, bytes, cudaMemcpyHostToDevice, ctx->stream), "cudaMemcpyAsync(multi-key tables)");
}

// the two parts `names` of an optional operand are both given or both null
static int check_pair(nb_ctx *ctx, const char *what, const void *a, const void *b, const char *names)
{
    if ((a == nullptr) != (b == nullptr)) return fail(ctx, NB_EINVAL, std::string(what) + ": " + names + " must come together");
    return NB_OK;
}

// entry t of each of the host tables `tables` is non-null for every tenant t
template <class... T> static int mk_check_tenants(nb_ctx *ctx, const char *what, const char *kind, size_t tenants, T... tables)
{
    for (size_t t = 0; t < tenants; t++)
        if (((tables[t] == nullptr) || ...))
            return fail(ctx, NB_EINVAL, std::string(what) + ": null " + kind + " of tenant " + std::to_string(t));
    return NB_OK;
}

// The first checks of a multi-key call over `batch` rows, tenant t owning counts[t] of them: the host tables (counts
// and `tables`) are given while there are tenants, the counts add up to the batch, the operands are given unless the
// batch is empty (`operands`), and so is every tenant's entry of `tables`.  All of it holds for an empty batch too.
template <class... T>
static int mk_preamble(nb_ctx *ctx, const char *what, const size_t *counts, size_t tenants, size_t batch, bool operands,
                       const char *kind, T... tables)
{
    if (!ctx) return NB_EINVAL;
    if (tenants && (!counts || ((tables == nullptr) || ...))) return fail(ctx, NB_EINVAL, std::string(what) + ": null argument");
    size_t sum = 0;
    for (size_t t = 0; t < tenants; t++) sum += counts[t];
    if (sum != batch)
        return fail(ctx, NB_EINVAL, std::string(what) + ": the counts add up to " + std::to_string(sum) + ", not the batch " +
                                        std::to_string(batch));
    if (batch && !operands) return fail(ctx, NB_EINVAL, std::string(what) + ": null argument");
    return mk_check_tenants(ctx, what, kind, tenants, tables...);
}

// The common part of the multi-key bootstraps: p carries everything but the keys, for a batch of jobs x sum(counts)
// ciphertexts whose job j covers rows [j B, (j + 1) B), split into tenants by the same counts.  Every tenant's key must lie
// inside an engine key with FP64 spectra prepared on this context, or inside a slot nb_mk_bk_expand filled, since the
// multi-key kernel runs the FP64 step.  The keys are checked before an empty batch returns.
static int mk_blind_rotate(nb_ctx *ctx, const char *what, BlindRotateArgs &p, const uint64_t *const *bk,
                           const size_t *counts, size_t tenants, size_t job_batch, int jobs)
{
    if (p.n <= 0 || p.n > LWE_N_MAX) return fail(ctx, NB_EUNSUPPORTED, std::string(what) + ": LWE dimension out of range");
    if (!ctx->fft) return fail(ctx, NB_EUNSUPPORTED, std::string(what) + ": multi-key launches run the FP64 step, which NUFHE_B200_FFT=0 disables");
    for (size_t t = 0; t < tenants; t++) {
        const u64 *key = (const u64 *)bk[t];
        for (const auto &k : ctx->multibit_keys)
            if (k.first <= key && key < k.second)
                return fail(ctx, NB_EUNSUPPORTED, std::string(what) + ": tenant " + std::to_string(t) + " has a multi-bit key");
        bool spectral = false;
        for (auto *keys : {&ctx->spectral_keys, &ctx->mk_slots})
            for (const auto &k : *keys) spectral |= k.first <= key && key + (size_t)p.n * BK_ROW_U64 <= k.second;
        if (!spectral)
            return fail(ctx, NB_EINVAL, std::string(what) + ": the key of tenant " + std::to_string(t) +
                                            " is not inside an engine key with FP64 spectra prepared on this context "
                                            "or a slot filled by nb_mk_bk_expand");
    }
    if (p.batch == 0) return NB_OK;
    // [tenant key pointers][tenant of each ciphertext]
    std::vector<unsigned char> host(tenants * sizeof(const u64 *) + p.batch * sizeof(unsigned));
    memcpy(host.data(), bk, tenants * sizeof(const u64 *));
    unsigned *tenant_of = reinterpret_cast<unsigned *>(host.data() + tenants * sizeof(const u64 *));
    for (int j = 0; j < jobs; j++) {
        size_t c = (size_t)j * job_batch;
        for (size_t t = 0; t < tenants; t++)
            for (size_t i = 0; i < counts[t]; i++) tenant_of[c++] = (unsigned)t;
    }
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:multikey_blind_rotate");
    NB_TRY(mk_upload(ctx, host.data(), host.size()));
    p.bk = nullptr;
    p.mk_bk = reinterpret_cast<const u64 *const *>(ctx->d_mk);
    p.mk_tenant = reinterpret_cast<const unsigned *>(reinterpret_cast<unsigned char *>(ctx->d_mk) + tenants * sizeof(const u64 *));
    NB_TRY(launch_br_cfg<BrFftMk>(ctx, p));
    return launch_check(ctx, "blind_rotate_kernel(multi-key)");
}

// The keys of a bootstrap: one engine key, or per-tenant keys (bk_host[t] serves counts[t] ciphertexts of every job)
struct BrKeys {
    bool multi = false;
    const uint64_t *bk = nullptr;
    const uint64_t *const *bk_host = nullptr;
    const size_t *counts = nullptr;
    size_t tenants = 0;

    explicit BrKeys(const uint64_t *bk) : bk(bk) {}
    BrKeys(const uint64_t *const *bk_host, const size_t *counts, size_t tenants) : multi(true), bk_host(bk_host), counts(counts), tenants(tenants) {}
    // One key: an empty batch needs no check (empty arrays have no storage to check).  Per-tenant keys are checked
    // even then, so that an empty launch validates them (MultiKeyVirtualMachine does).
    bool nothing_to_do(const nb_ctx *ctx, size_t batch) const { return ctx && !multi && batch == 0; }
    // the key tables and counts, and the operands, which `operands` says are all given
    int check(nb_ctx *ctx, const char *what, bool operands, size_t batch) const
    {
        if (multi) return mk_preamble(ctx, what, counts, tenants, batch, operands, "key", bk_host);
        if (!ctx || !operands || !bk) return fail(ctx, NB_EINVAL, std::string(what) + ": null argument");
        return NB_OK;
    }
    // p's `jobs` jobs of `batch` ciphertexts each, extracted into out_a, out_b
    int run(nb_ctx *ctx, const char *what, BlindRotateArgs &p, size_t n, int32_t *out_a, int32_t *out_b, size_t batch, int jobs) const
    {
        p.n = (int)n; p.out_a = out_a; p.out_b = out_b; p.extract = 1; p.batch = jobs * batch;
        if (multi) return mk_blind_rotate(ctx, what, p, bk_host, counts, tenants, batch, jobs);
        p.bk = (const u64 *)bk;
        return launch_blind_rotate(ctx, p);
    }
};

// the operands of a gate-style job: x = (0, c) + s1 * in1 + s2 * in2, in2 optional
struct GateJob { const int32_t *in1_a, *in1_b, *in2_a, *in2_b; int32_t c, s1, s2; };

static void set_job(BlindRotateArgs &p, const GateJob &x)
{
    p.in1_a = x.in1_a; p.in1_b = x.in1_b; p.in2_a = x.in2_a; p.in2_b = x.in2_b; p.c = x.c; p.s1 = x.s1; p.s2 = x.s2;
}

static int bootstrap_extract(nb_ctx *ctx, const char *what, const BrKeys &keys, const GateJob &x, int32_t mu, size_t n,
                             int32_t *out_a, int32_t *out_b, size_t batch)
{
    if (keys.nothing_to_do(ctx, batch)) return NB_OK;
    NB_TRY(keys.check(ctx, what, x.in1_a && x.in1_b && out_a && out_b, batch));
    NB_TRY(check_pair(ctx, what, x.in2_a, x.in2_b, "in2_a/in2_b"));
    BlindRotateArgs p{};
    set_job(p, x);
    p.mu = mu;
    return keys.run(ctx, what, p, n, out_a, out_b, batch, 1);
}

// tv_stride 0: one test vector for the batch, 1024: one per ciphertext; 2^log2_outputs extracted samples per ciphertext
static int bootstrap_lut_extract(nb_ctx *ctx, const char *what, const BrKeys &keys, const GateJob &x, const int32_t *tv,
                                 size_t tv_stride, int log2_outputs, size_t n, int32_t *out_a, int32_t *out_b, size_t batch)
{
    if (keys.nothing_to_do(ctx, batch)) return NB_OK;
    NB_TRY(keys.check(ctx, what, x.in1_a && x.in1_b && tv && out_a && out_b, batch));
    NB_TRY(check_pair(ctx, what, x.in2_a, x.in2_b, "in2_a/in2_b"));
    if (tv_stride != 0 && tv_stride != (size_t)NTT_N) return fail(ctx, NB_EINVAL, std::string(what) + ": tv_stride must be 0 or 1024");
    if (log2_outputs < 0 || log2_outputs > 2) return fail(ctx, NB_EINVAL, std::string(what) + ": log2_outputs must be 0, 1 or 2");
    BlindRotateArgs p{};
    set_job(p, x);
    p.tv = tv; p.tv_stride = tv_stride; p.log2_outputs = log2_outputs;
    return keys.run(ctx, what, p, n, out_a, out_b, batch, 1);
}

static int bootstrap_glwe_lut_extract(nb_ctx *ctx, const char *what, const BrKeys &keys, const int32_t *in_a,
                                      const int32_t *in_b, const int32_t *tv, size_t n, int32_t *out_a, int32_t *out_b,
                                      size_t batch)
{
    if (keys.nothing_to_do(ctx, batch)) return NB_OK;
    NB_TRY(keys.check(ctx, what, in_a && in_b && tv && out_a && out_b, batch));
    BlindRotateArgs p{};
    set_job(p, {in_a, in_b, nullptr, nullptr, 0, 1, 0});
    p.tv = tv; p.tv_stride = 2 * (size_t)NTT_N; p.log2_outputs = 0;
    return keys.run(ctx, what, p, n, out_a, out_b, batch, 1);
}

// two gate bootstraps in one launch: rows [0, batch) of the outputs are job a's, rows [batch, 2 batch) job b's
static int bootstrap_extract2(nb_ctx *ctx, const char *what, const BrKeys &keys, const GateJob &a, const GateJob &b,
                              int32_t mu, size_t n, int32_t *out_a, int32_t *out_b, size_t batch)
{
    if (keys.nothing_to_do(ctx, batch)) return NB_OK;
    NB_TRY(keys.check(ctx, what, a.in1_a && a.in1_b && b.in1_a && b.in1_b && out_a && out_b, batch));
    NB_TRY(check_pair(ctx, what, a.in2_a, a.in2_b, "a/b parts"));
    NB_TRY(check_pair(ctx, what, b.in2_a, b.in2_b, "a/b parts"));
    BlindRotateArgs p{};
    set_job(p, a);
    p.j2_in1_a = b.in1_a; p.j2_in1_b = b.in1_b; p.j2_in2_a = b.in2_a; p.j2_in2_b = b.in2_b; p.j2_c = b.c; p.j2_s1 = b.s1; p.j2_s2 = b.s2;
    p.mu = mu; p.job_batch = batch;
    return keys.run(ctx, what, p, n, out_a, out_b, batch, 2);
}

extern "C" {

int nb_blind_rotate(nb_ctx *ctx, const int32_t *accum, const int32_t *bara, const uint64_t *bk_int, size_t n,
                    int32_t *out_a, int32_t *out_b, int32_t *accum_out, size_t batch)
{
    if (ctx && batch == 0) return NB_OK;     // nothing to do: empty arrays have no storage to check
    if (!ctx || !accum || !bara || !bk_int) return fail(ctx, NB_EINVAL, "nb_blind_rotate: null argument");
    NB_TRY(check_pair(ctx, "nb_blind_rotate", out_a, out_b, "out_a/out_b"));
    BlindRotateArgs p{};
    p.accum = accum; p.bara = bara; p.bk = (const u64 *)bk_int; p.n = (int)n;
    p.out_a = out_a; p.out_b = out_b; p.accum_out = accum_out; p.extract = out_a != nullptr; p.batch = batch;
    return launch_blind_rotate(ctx, p);
}

int nb_bootstrap_extract(nb_ctx *ctx, const int32_t *in1_a, const int32_t *in1_b, const int32_t *in2_a,
                         const int32_t *in2_b, int32_t c, int32_t s1, int32_t s2, int32_t mu,
                         const uint64_t *bk_int, size_t n, int32_t *out_a, int32_t *out_b, size_t batch)
{
    return bootstrap_extract(ctx, "nb_bootstrap_extract", BrKeys(bk_int), {in1_a, in1_b, in2_a, in2_b, c, s1, s2}, mu,
                             n, out_a, out_b, batch);
}

int nb_bootstrap_lut_extract(nb_ctx *ctx, const int32_t *in1_a, const int32_t *in1_b, const int32_t *in2_a,
                             const int32_t *in2_b, int32_t c, int32_t s1, int32_t s2, const int32_t *tv, size_t tv_stride,
                             int log2_outputs, const uint64_t *bk_int, size_t n, int32_t *out_a, int32_t *out_b,
                             size_t batch)
{
    return bootstrap_lut_extract(ctx, "nb_bootstrap_lut_extract", BrKeys(bk_int), {in1_a, in1_b, in2_a, in2_b, c, s1, s2},
                                 tv, tv_stride, log2_outputs, n, out_a, out_b, batch);
}

int nb_bootstrap_glwe_lut_extract(nb_ctx *ctx, const int32_t *in_a, const int32_t *in_b, const int32_t *tv,
                                  const uint64_t *bk_int, size_t n, int32_t *out_a, int32_t *out_b, size_t batch)
{
    return bootstrap_glwe_lut_extract(ctx, "nb_bootstrap_glwe_lut_extract", BrKeys(bk_int), in_a, in_b, tv, n, out_a, out_b, batch);
}

int nb_bootstrap_extract2(nb_ctx *ctx, const int32_t *a1_a, const int32_t *a1_b, const int32_t *a2_a,
                          const int32_t *a2_b, int32_t a_c, int32_t a_s1, int32_t a_s2, const int32_t *b1_a,
                          const int32_t *b1_b, const int32_t *b2_a, const int32_t *b2_b, int32_t b_c, int32_t b_s1,
                          int32_t b_s2, int32_t mu, const uint64_t *bk_int, size_t n, int32_t *out_a, int32_t *out_b,
                          size_t batch)
{
    return bootstrap_extract2(ctx, "nb_bootstrap_extract2", BrKeys(bk_int), {a1_a, a1_b, a2_a, a2_b, a_c, a_s1, a_s2},
                              {b1_a, b1_b, b2_a, b2_b, b_c, b_s1, b_s2}, mu, n, out_a, out_b, batch);
}

// ---- multi-key bootstraps (DESIGN.md section 17) ----

int nb_mk_bootstrap_extract(nb_ctx *ctx, const int32_t *in1_a, const int32_t *in1_b, const int32_t *in2_a,
                            const int32_t *in2_b, int32_t c, int32_t s1, int32_t s2, int32_t mu,
                            const uint64_t *const *bk_int_host, const size_t *counts_host, size_t tenants, size_t n,
                            int32_t *out_a, int32_t *out_b, size_t batch)
{
    return bootstrap_extract(ctx, "nb_mk_bootstrap_extract", BrKeys(bk_int_host, counts_host, tenants),
                             {in1_a, in1_b, in2_a, in2_b, c, s1, s2}, mu, n, out_a, out_b, batch);
}

int nb_mk_bootstrap_extract2(nb_ctx *ctx, const int32_t *a1_a, const int32_t *a1_b, const int32_t *a2_a,
                             const int32_t *a2_b, int32_t a_c, int32_t a_s1, int32_t a_s2, const int32_t *b1_a,
                             const int32_t *b1_b, const int32_t *b2_a, const int32_t *b2_b, int32_t b_c, int32_t b_s1,
                             int32_t b_s2, int32_t mu, const uint64_t *const *bk_int_host, const size_t *counts_host,
                             size_t tenants, size_t n, int32_t *out_a, int32_t *out_b, size_t batch)
{
    return bootstrap_extract2(ctx, "nb_mk_bootstrap_extract2", BrKeys(bk_int_host, counts_host, tenants),
                              {a1_a, a1_b, a2_a, a2_b, a_c, a_s1, a_s2}, {b1_a, b1_b, b2_a, b2_b, b_c, b_s1, b_s2}, mu, n, out_a, out_b, batch);
}

int nb_mk_bootstrap_lut_extract(nb_ctx *ctx, const int32_t *in1_a, const int32_t *in1_b, const int32_t *in2_a,
                                const int32_t *in2_b, int32_t c, int32_t s1, int32_t s2, const int32_t *tv,
                                size_t tv_stride, int log2_outputs, const uint64_t *const *bk_int_host,
                                const size_t *counts_host, size_t tenants, size_t n, int32_t *out_a, int32_t *out_b,
                                size_t batch)
{
    return bootstrap_lut_extract(ctx, "nb_mk_bootstrap_lut_extract", BrKeys(bk_int_host, counts_host, tenants),
                                 {in1_a, in1_b, in2_a, in2_b, c, s1, s2}, tv, tv_stride, log2_outputs, n, out_a, out_b, batch);
}

int nb_mk_bootstrap_glwe_lut_extract(nb_ctx *ctx, const int32_t *in_a, const int32_t *in_b, const int32_t *tv,
                                     const uint64_t *const *bk_int_host, const size_t *counts_host, size_t tenants,
                                     size_t n, int32_t *out_a, int32_t *out_b, size_t batch)
{
    return bootstrap_glwe_lut_extract(ctx, "nb_mk_bootstrap_glwe_lut_extract", BrKeys(bk_int_host, counts_host, tenants),
                                      in_a, in_b, tv, n, out_a, out_b, batch);
}

}  // extern "C"

// The prepared planes of the fast-shape key switch p when it runs as the tensor-core GEMM (registered key, batch from
// ks_mma_min, rows aligned for its loads and stores), else null
static const uint8_t *ks_gemm_planes(nb_ctx *ctx, const KeyswitchArgs &p)
{
    const uint8_t *planes = nullptr;
    if (p.batch >= ctx->ks_mma_min &&
        (((uintptr_t)p.src1_a | (uintptr_t)(p.src2_a ? p.src2_a : p.src1_a)) & 15) == 0 && ((uintptr_t)p.res_a & 7) == 0)
        for (const auto &k : ctx->ks_keys)
            if (k.ks_a == p.ks_a && k.ks_b == p.ks_b) planes = k.planes;
    return planes;
}

// The key switch p as the tensor-core GEMM: tiles of 256 ciphertexts x 32 output columns; K is split over blockIdx.z
// (partial sums meet in integer atomics) while a launch would leave half of the SMs idle
static int ks_gemm(nb_ctx *ctx, const KeyswitchArgs &p, const uint8_t *planes)
{
    KeyswitchMmaArgs m{};
    m.src1_a = p.src1_a; m.src1_b = p.src1_b; m.src2_a = p.src2_a; m.src2_b = p.src2_b; m.c = p.c;
    m.planes = planes; m.res_a = p.res_a; m.res_b = p.res_b; m.batch = p.batch;
    const size_t tiles = (p.batch + KM_M - 1) / KM_M * KM_NTILES;
    int splits = 1;
    while (splits < 16 && tiles * (size_t)splits * 2 <= (size_t)ctx->sm_count) splits *= 2;
    m.splits = splits;
    if (splits > 1) {
        NB_TRY(check(ctx, cudaMemsetAsync(p.res_a, 0, p.batch * p.n * sizeof(int32_t), ctx->stream), "cudaMemsetAsync"));
        NB_TRY(check(ctx, cudaMemsetAsync(p.res_b, 0, p.batch * sizeof(int32_t), ctx->stream), "cudaMemsetAsync"));
    }
    keyswitch_mma_kernel<<<dim3((unsigned)((p.batch + KM_M - 1) / KM_M), KM_NTILES, splits), KM_THREADS, KM_SMEM_BYTES,
                           ctx->stream>>>(m);
    if (p.res_cv) {
        NB_TRY(launch_check(ctx, "keyswitch_mma_kernel"));
        ks_cv_kernel<<<(unsigned)((p.batch + 31) / 32), 256, 0, ctx->stream>>>(p.src1_a, p.src2_a, p.ks_cv, p.res_cv, p.batch);
    }
    return launch_check(ctx, "keyswitch_mma_kernel");
}

// The key switch p on the gather kernel over `ctas` tiles: launch(grid) enqueues the kernel `what`.  The consumer loop
// always walks KS_TILE ciphertext slots, so a CTA costs the same whatever its tile: the 1024 input coefficients are
// split over blockIdx.y until the SMs are covered (partial sums meet in integer atomics).  One ciphertext: 128 CTAs x 8
// coefficients.  Every output row is exact integer arithmetic and its variance the fixed-shape sum, so the split
// changes no bit.
template <class Launch> static int ks_gather(nb_ctx *ctx, KeyswitchArgs &p, size_t ctas, const char *what, Launch launch)
{
    const int splits = (int)std::min<size_t>(128, std::max<size_t>(1, (size_t)ctx->sm_count / ctas));
    p.splits = splits;
    if (splits > 1) {
        NB_TRY(check(ctx, cudaMemsetAsync(p.res_a, 0, p.batch * p.n * sizeof(int32_t), ctx->stream), "cudaMemsetAsync"));
        NB_TRY(check(ctx, cudaMemsetAsync(p.res_b, 0, p.batch * sizeof(int32_t), ctx->stream), "cudaMemsetAsync"));
        if (p.res_cv) {
            NB_TRY(reserve_words(ctx, (void **)&ctx->d_cv_blocks, &ctx->cv_words, p.batch * KS_CV_BLOCKS, sizeof(float)));
            p.cv_blocks = ctx->d_cv_blocks;
        }
    }
    NB_TRY(launch(dim3((unsigned)ctas, splits)));
    NB_TRY(launch_check(ctx, what));
    if (!p.cv_blocks) return NB_OK;
    ks_cv_finalize_kernel<<<(int)((p.batch + 127) / 128), 128, 0, ctx->stream>>>(p.res_cv, p.cv_blocks, p.batch);
    return launch_check(ctx, "ks_cv_finalize_kernel");
}

extern "C" {

int nb_keyswitch(nb_ctx *ctx, const int32_t *src1_a, const int32_t *src1_b, const int32_t *src2_a,
                 const int32_t *src2_b, int32_t c, const int32_t *ks_a, const int32_t *ks_b, const float *ks_cv,
                 size_t in_size, size_t n, int t, int log2_base, int32_t *res_a, int32_t *res_b, float *res_cv,
                 size_t batch)
{
    if (ctx && batch == 0) return NB_OK;     // nothing to do: empty arrays have no storage to check
    if (!ctx || !src1_a || !src1_b || !ks_a || !ks_b || !ks_cv || !res_a || !res_b)
        return fail(ctx, NB_EINVAL, "nb_keyswitch: null argument");
    NB_TRY(check_pair(ctx, "nb_keyswitch", src2_a, src2_b, "src2_a/src2_b"));
    if (n + 1 > 512) return fail(ctx, NB_EUNSUPPORTED, "nb_keyswitch: output LWE dimension above 511");
    if (t < 1 || log2_base < 1 || t * log2_base > 31) return fail(ctx, NB_EINVAL, "nb_keyswitch: bad decomposition");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:keyswitch");
    KeyswitchArgs p{};
    p.src1_a = src1_a; p.src1_b = src1_b; p.src2_a = src2_a; p.src2_b = src2_b; p.c = c;
    p.ks_a = ks_a; p.ks_b = ks_b; p.ks_cv = ks_cv; p.res_a = res_a; p.res_b = res_b; p.res_cv = res_cv;
    p.in_size = (int)in_size; p.n = (int)n; p.t = t; p.log2_base = log2_base; p.batch = batch;
    if (!(t == 8 && log2_base == 2 && in_size == (size_t)KS_IN && n == (size_t)KS_N)) {
        keyswitch_generic_kernel<<<(int)batch, 512, 0, ctx->stream>>>(p);
        return launch_check(ctx, "keyswitch_kernel");
    }
    if (const uint8_t *planes = ks_gemm_planes(ctx, p)) return ks_gemm(ctx, p, planes);
    const size_t tile = batch < (size_t)KS_TILE ? batch : (size_t)KS_TILE;
    p.tile = (int)tile;
    return ks_gather(ctx, p, (batch + tile - 1) / tile, "keyswitch_kernel", [&](dim3 grid) {
        keyswitch_kernel<<<grid, KS_THREADS, KS_SMEM_BYTES, ctx->stream>>>(p);
        return NB_OK;
    });
}

size_t nb_ks_prepared_bytes(void) { return KM_PLANES_BYTES; }

int nb_ks_prepare(nb_ctx *ctx, const int32_t *ks_a, const int32_t *ks_b, uint8_t *out, size_t in_size, size_t n, int t,
                  int log2_base, int *registered)
{
    if (!ctx || !ks_a || !ks_b || !out) return fail(ctx, NB_EINVAL, "nb_ks_prepare: null argument");
    if (registered) *registered = 0;
    if (!(t == 8 && log2_base == 2 && in_size == (size_t)KS_IN && n == (size_t)KS_N))
        return fail(ctx, NB_EUNSUPPORTED, "nb_ks_prepare: the GEMM layout is for in = 1024, n = 500, t = 8, base 4 only");
    if ((uintptr_t)out & 15) return fail(ctx, NB_EINVAL, "nb_ks_prepare: out must be 16-byte aligned");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:ks_prepare");
    nb_ks_forget(ctx, ks_a);
    for (size_t i = 0; i < ctx->ks_keys.size();) {      // registrations whose planes `out` overwrites
        const uint8_t *p = ctx->ks_keys[i].planes;
        if (p < out + KM_PLANES_BYTES && out < p + KM_PLANES_BYTES) ctx->ks_keys.erase(ctx->ks_keys.begin() + i);
        else i++;
    }
    int *d_flag = nullptr, pad_nonzero = 0;
    NB_TRY(check(ctx, cudaMalloc(&d_flag, sizeof(int)), "cudaMalloc(ks_prepare)"));
    int rc = check(ctx, cudaMemsetAsync(d_flag, 0, sizeof(int), ctx->stream), "cudaMemsetAsync");
    if (rc == NB_OK) {
        ks_prepare_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(ks_a, ks_b, out, d_flag);
        rc = launch_check(ctx, "ks_prepare_kernel");
    }
    if (rc == NB_OK) rc = check(ctx, cudaMemcpyAsync(&pad_nonzero, d_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream), "cudaMemcpyAsync");
    if (rc == NB_OK) rc = check(ctx, cudaStreamSynchronize(ctx->stream), "cudaStreamSynchronize");
    cudaFree(d_flag);
    NB_TRY(rc);
    // a key with non-zero d = 0 rows keeps keyswitch_kernel, which adds them
    if (!pad_nonzero) ctx->ks_keys.push_back({ks_a, ks_b, out});
    if (registered) *registered = !pad_nonzero;
    return NB_OK;
}

int nb_ks_forget(nb_ctx *ctx, const int32_t *ks_a)
{
    if (!ctx) return NB_EINVAL;
    for (size_t i = 0; i < ctx->ks_keys.size();) {
        if (ctx->ks_keys[i].ks_a == ks_a) ctx->ks_keys.erase(ctx->ks_keys.begin() + i);
        else i++;
    }
    return NB_OK;
}

static int ew_grid(nb_ctx *ctx, size_t n)
{
    size_t blocks = (n + 255) / 256, cap = (size_t)ctx->sm_count * 16;
    return (int)(blocks < cap ? blocks : cap);
}

int nb_shift_torus_polynomial(nb_ctx *ctx, int32_t *result, const int32_t *source, const int32_t *powers,
                              size_t powers_stride, size_t power_idx, int polys_per_power, int mode, int n_log2,
                              size_t polys)
{
    if (!ctx) return NB_EINVAL;
    if (!result || !source || !powers) return fail(ctx, NB_EINVAL, "nb_shift_torus_polynomial: null argument");
    if (mode < NB_SHIFT_INVERT || mode > NB_SHIFT_PLAIN) return fail(ctx, NB_EINVAL, "nb_shift_torus_polynomial: unknown mode");
    if (n_log2 < 1 || n_log2 > 20 || polys_per_power < 1) return fail(ctx, NB_EINVAL, "nb_shift_torus_polynomial: bad size");
    if (result == source) return fail(ctx, NB_EINVAL, "nb_shift_torus_polynomial: result must not alias source");
    if (polys == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    shift_torus_polynomial_kernel<<<ew_grid(ctx, polys << n_log2), 256, 0, ctx->stream>>>(
        result, source, powers, powers_stride, power_idx, polys_per_power, mode, n_log2, polys);
    return launch_check(ctx, "shift_torus_polynomial_kernel");
}

int nb_tlwe_noiseless_trivial(nb_ctx *ctx, int32_t *acc, float *cv, const int32_t *mu, int mask_size, int n_log2,
                              size_t batch)
{
    if (!ctx) return NB_EINVAL;
    if (!acc || !mu) return fail(ctx, NB_EINVAL, "nb_tlwe_noiseless_trivial: null argument");
    if (mask_size < 1 || n_log2 < 1 || n_log2 > 20) return fail(ctx, NB_EINVAL, "nb_tlwe_noiseless_trivial: bad size");
    if (batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    tlwe_noiseless_trivial_kernel<<<ew_grid(ctx, (batch * (mask_size + 1)) << n_log2), 256, 0, ctx->stream>>>(
        acc, cv, mu, mask_size, n_log2, batch);
    return launch_check(ctx, "tlwe_noiseless_trivial_kernel");
}

int nb_tlwe_extract_lwe_samples(nb_ctx *ctx, int32_t *out_a, int32_t *out_b, const int32_t *acc, int mask_size,
                                int n_log2, size_t batch)
{
    if (!ctx) return NB_EINVAL;
    if (!out_a || !out_b || !acc) return fail(ctx, NB_EINVAL, "nb_tlwe_extract_lwe_samples: null argument");
    if (mask_size < 1 || n_log2 < 1 || n_log2 > 20) return fail(ctx, NB_EINVAL, "nb_tlwe_extract_lwe_samples: bad size");
    if (batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    tlwe_extract_lwe_samples_kernel<<<ew_grid(ctx, (batch * mask_size) << n_log2), 256, 0, ctx->stream>>>(
        out_a, out_b, acc, mask_size, n_log2, batch);
    return launch_check(ctx, "tlwe_extract_lwe_samples_kernel");
}

int nb_t32_to_phase(nb_ctx *ctx, int32_t *out, const int32_t *in, size_t n, uint32_t mspace_size)
{
    if (!ctx) return NB_EINVAL;
    if (!out || !in) return fail(ctx, NB_EINVAL, "nb_t32_to_phase: null argument");
    if (mspace_size == 0 || (mspace_size & (mspace_size - 1))) return fail(ctx, NB_EINVAL, "nb_t32_to_phase: mspace_size must be a power of two");
    if (n == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    t32_to_phase_kernel<<<ew_grid(ctx, n), 256, 0, ctx->stream>>>(out, in, n, mspace_size);
    return launch_check(ctx, "t32_to_phase_kernel");
}

int nb_tgsw_decompose(nb_ctx *ctx, int32_t *out, const int32_t *in, size_t polys, int decomp_length, int bs_log2_base,
                      int32_t offset, int n_log2)
{
    if (!ctx) return NB_EINVAL;
    if (!out || !in) return fail(ctx, NB_EINVAL, "nb_tgsw_decompose: null argument");
    if (decomp_length < 1 || bs_log2_base < 1 || decomp_length * bs_log2_base > 32 || n_log2 < 1 || n_log2 > 20)
        return fail(ctx, NB_EINVAL, "nb_tgsw_decompose: bad decomposition");
    if (polys == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    tgsw_decompose_kernel<<<ew_grid(ctx, (polys * decomp_length) << n_log2), 256, 0, ctx->stream>>>(
        out, in, polys, decomp_length, bs_log2_base, offset, n_log2);
    return launch_check(ctx, "tgsw_decompose_kernel");
}

int nb_tgsw_mac(nb_ctx *ctx, uint64_t *out, const uint64_t *tr, const uint64_t *bk_row, size_t batch, int mask_size,
                int decomp_length)
{
    if (!ctx) return NB_EINVAL;
    if (!out || !tr || !bk_row) return fail(ctx, NB_EINVAL, "nb_tgsw_mac: null argument");
    if (mask_size < 1 || mask_size > 15 || decomp_length < 1 || decomp_length > 32) return fail(ctx, NB_EINVAL, "nb_tgsw_mac: bad size");
    if (batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    tgsw_mac_kernel<<<ew_grid(ctx, batch * (mask_size + 1) * NTT_N), 256, 0, ctx->stream>>>(
        (u64 *)out, (const u64 *)tr, (const u64 *)bk_row, batch, mask_size + 1, decomp_length);
    return launch_check(ctx, "tgsw_mac_kernel");
}

int nb_tlwe_add_to(nb_ctx *ctx, int32_t *res, const int32_t *src, size_t n, float *res_cv, const float *src_cv,
                   size_t n_cv)
{
    if (!ctx) return NB_EINVAL;
    if (!res || !src || ((res_cv == nullptr) != (src_cv == nullptr)))
        return fail(ctx, NB_EINVAL, "nb_tlwe_add_to: null argument");
    if (n_cv > n) return fail(ctx, NB_EINVAL, "nb_tlwe_add_to: more variances than coefficients");
    if (n == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    add_to_kernel<<<ew_grid(ctx, n), 256, 0, ctx->stream>>>(res, src, n, res_cv, src_cv, res_cv ? n_cv : 0);
    return launch_check(ctx, "add_to_kernel");
}

int nb_lwe_affine(nb_ctx *ctx, int32_t *res_a, int32_t *res_b, const int32_t *x1_a, const int32_t *x1_b,
                  const int32_t *x2_a, const int32_t *x2_b, int32_t c, int32_t s1, int32_t s2, size_t batch,
                  size_t n)
{
    if (ctx && batch == 0) return NB_OK;     // nothing to do: empty arrays have no storage to check
    if (!ctx || !res_a || !res_b) return fail(ctx, NB_EINVAL, "nb_lwe_affine: null argument");
    if ((x1_a == nullptr) != (x1_b == nullptr) || (x2_a == nullptr) != (x2_b == nullptr))
        return fail(ctx, NB_EINVAL, "nb_lwe_affine: a/b parts must come together");
    if (batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    size_t total = batch * (n + 1), blocks = (total + 255) / 256, cap = (size_t)ctx->sm_count * 16;
    lwe_affine_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>(
        res_a, res_b, x1_a, x1_b, x2_a, x2_b, c, s1, s2, batch, (int)n);
    return launch_check(ctx, "lwe_affine_kernel");
}

int nb_lwe_dot(nb_ctx *ctx, int32_t *out, const int32_t *a, const int32_t *key, const int32_t *add1,
               const int32_t *add2, int32_t sign, size_t batch, size_t n)
{
    if (!ctx) return NB_EINVAL;
    if (batch == 0) return NB_OK;
    if (!out || !a || !key) return fail(ctx, NB_EINVAL, "nb_lwe_dot: null argument");
    if (n == 0 || n > (1u << 30)) return fail(ctx, NB_EINVAL, "nb_lwe_dot: bad LWE dimension");
    if (batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:lwe_dot");
    size_t blocks = (batch * 32 + 255) / 256, cap = (size_t)ctx->sm_count * 16;
    lwe_dot_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>(out, a, key, add1, add2, sign, batch, (int)n);
    return launch_check(ctx, "lwe_dot_kernel");
}

int nb_make_keyswitch_key(nb_ctx *ctx, int32_t *ks_a, int32_t *ks_b, float *ks_cv, const int32_t *in_key,
                          const int32_t *out_key, const int32_t *noises_a, const int32_t *noises_b, size_t in_size,
                          size_t n, int t, int log2_base, float noise_variance)
{
    if (!ctx) return NB_EINVAL;
    if (!ks_a || !ks_b || !ks_cv || !in_key || !out_key || !noises_a || !noises_b)
        return fail(ctx, NB_EINVAL, "nb_make_keyswitch_key: null argument");
    if (t < 1 || log2_base < 1 || t * log2_base > 31 || n == 0) return fail(ctx, NB_EINVAL, "nb_make_keyswitch_key: bad decomposition");
    if (in_size == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:make_keyswitch_key");
    const size_t rows = in_size * (size_t)t << log2_base;
    size_t blocks = (rows * 32 + 255) / 256, cap = (size_t)ctx->sm_count * 16;
    make_keyswitch_key_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>(
        ks_a, ks_b, ks_cv, in_key, out_key, noises_a, noises_b, in_size, (int)n, t, log2_base, noise_variance);
    return launch_check(ctx, "make_keyswitch_key_kernel");
}

int nb_seeded_uniform_i32(nb_ctx *ctx, const uint32_t *seed_host, uint64_t nonce, uint64_t first, int32_t *out,
                          size_t count)
{
    if (!ctx) return NB_EINVAL;
    if (!seed_host || !out) return fail(ctx, NB_EINVAL, "nb_seeded_uniform_i32: null argument");
    if (count == 0) return NB_OK;
    if ((uint64_t)count - 1 > UINT64_MAX - first)
        return fail(ctx, NB_EINVAL, "nb_seeded_uniform_i32: first + count is past the end of the 2^64-word stream");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:seeded_uniform");
    ChachaSeed seed;
    memcpy(seed.w, seed_host, sizeof(seed.w));
    const u64 blocks = ((first + ((u64)count - 1)) >> 4) - (first >> 4) + 1;
    const u64 ctas = (blocks + SEEDED_THREADS - 1) / SEEDED_THREADS, cap = (u64)ctx->sm_count * 8;
    seeded_uniform_kernel<<<(int)(ctas < cap ? ctas : cap), SEEDED_THREADS, 0, ctx->stream>>>(out, seed, nonce, first,
                                                                                              (u64)count);
    return launch_check(ctx, "seeded_uniform_kernel");
}


size_t nb_pk_planes_bytes(size_t m, size_t n)
{
    if (n == 0 || n > (1u << 30)) return 0;
    return 4 * m * (size_t)pk_cols_padded((u32)n);
}

// m rows of [A | b] for an n-word LWE key: m a multiple of 32 (whole k-steps), and exact sums for 0/1 bytes of R
static int pk_check_shape(nb_ctx *ctx, size_t m, size_t n, const char *what)
{
    if (m == 0 || m % 32 != 0 || !plane_gemm_exact(m, 1))
        return fail(ctx, NB_EINVAL, std::string(what) + ": m must be a positive multiple of 32 with m * 255 < 2^31");
    if (n == 0 || n > (1u << 30)) return fail(ctx, NB_EINVAL, std::string(what) + ": bad LWE dimension");
    return NB_OK;
}

int nb_pk_prepare(nb_ctx *ctx, const int32_t *a, const int32_t *b, size_t m, size_t n, uint8_t *planes)
{
    if (!ctx) return NB_EINVAL;
    if (!a || !b || !planes) return fail(ctx, NB_EINVAL, "nb_pk_prepare: null argument");
    NB_TRY(pk_check_shape(ctx, m, n, "nb_pk_prepare"));
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:pk_prepare");
    const size_t quads = (size_t)pk_cols_padded((u32)n) * (m / 4);
    size_t blocks = (quads + 255) / 256, cap = (size_t)ctx->sm_count * 16;
    plane_prepare_kernel<PkSource, const i32 *__restrict__, const i32 *__restrict__, u32, u32>
        <<<(int)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>(planes, a, b, (u32)m, (u32)n);
    return launch_check(ctx, "plane_prepare_kernel<PkSource>");
}

int nb_pk_encrypt(nb_ctx *ctx, const uint32_t *r_bits, const uint8_t *planes, size_t m, size_t n, const int32_t *mus,
                  float row_variance, int32_t *out_a, int32_t *out_b, float *out_cv, size_t batch)
{
    if (!ctx) return NB_EINVAL;
    if (!r_bits || !planes || !mus || !out_a || !out_b || !out_cv)
        return fail(ctx, NB_EINVAL, "nb_pk_encrypt: null argument");
    NB_TRY(pk_check_shape(ctx, m, n, "nb_pk_encrypt"));
    if (batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:pk_encrypt");
    const size_t rows_per_cta = (size_t)GEMM_WARPS * GEMM_MTILES * 16;
    const size_t ctas = (batch + rows_per_cta - 1) / rows_per_cta;
    if (ctas > 0x7fffffffu) return fail(ctx, NB_EINVAL, "nb_pk_encrypt: batch too large");
    const dim3 grid((unsigned)ctas, pk_cols_padded((u32)n) / (8 * PkGemm::NTILES));
    plane_gemm_kernel<PkGemm, const u32 *__restrict__, u32, u32, const i32 *__restrict__, float, i32 *__restrict__,
                      i32 *__restrict__, float *__restrict__><<<grid, GEMM_WARPS * 32, 0, ctx->stream>>>(
        planes, (u64)batch, r_bits, (u32)m, (u32)n, mus, row_variance, out_a, out_b, out_cv);
    return launch_check(ctx, "plane_gemm_kernel<PkGemm>");
}

int nb_pack_digits(nb_ctx *ctx, const int32_t *a, size_t n, int32_t *digits, size_t batch)
{
    if (!ctx) return NB_EINVAL;
    if (!a || !digits) return fail(ctx, NB_EINVAL, "nb_pack_digits: null argument");
    if (n == 0 || n > (1u << 20)) return fail(ctx, NB_EINVAL, "nb_pack_digits: bad LWE dimension");
    if (batch == 0) return NB_OK;
    const size_t groups = (batch + PACK_N - 1) / PACK_N, tiles = groups * (PACK_N / PACK_TILE);
    if (tiles > 65535) return fail(ctx, NB_EINVAL, "nb_pack_digits: more than 2047 groups in one call");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:pack_digits");
    const dim3 grid((unsigned)((n + PACK_TILE - 1) / PACK_TILE), (unsigned)tiles);
    pack_digits_kernel<<<grid, PACK_DIGITS_THREADS, 0, ctx->stream>>>(a, (u32)n, (u64)batch, digits);
    return launch_check(ctx, "pack_digits_kernel");
}

int nb_ntt_mac(nb_ctx *ctx, const uint64_t *x, const uint64_t *key, uint64_t *out, size_t rows, size_t outs,
               size_t groups)
{
    if (!ctx) return NB_EINVAL;
    if (!x || !key || !out) return fail(ctx, NB_EINVAL, "nb_ntt_mac: null argument");
    if (rows == 0 || outs == 0 || rows > (1u << 24) || outs > (1u << 16))
        return fail(ctx, NB_EINVAL, "nb_ntt_mac: rows must be in [1, 2^24] and outputs in [1, 2^16]");
    if (groups == 0) return NB_OK;
    const size_t ctas = groups * (PACK_N / MAC_POINTS);
    if (ctas > 0x7fffffffu) return fail(ctx, NB_EINVAL, "nb_ntt_mac: too many groups");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:ntt_mac");
    const dim3 grid((unsigned)ctas, (unsigned)((outs + MAC_OUTS - 1) / MAC_OUTS));
    ntt_mac_kernel<<<grid, MAC_WARPS * 32, 0, ctx->stream>>>((const u64 *)x, (const u64 *)key, (u64 *)out, (u32)rows,
                                                            (u32)outs);
    return launch_check(ctx, "ntt_mac_kernel");
}

int nb_pack_finish(nb_ctx *ctx, const int32_t *c, const int32_t *b, int mask_size, uint16_t *out, size_t batch)
{
    if (!ctx) return NB_EINVAL;
    if (!c || !b || !out) return fail(ctx, NB_EINVAL, "nb_pack_finish: null argument");
    if (mask_size < 1 || mask_size > (1 << 16)) return fail(ctx, NB_EINVAL, "nb_pack_finish: bad mask size");
    if (batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:pack_finish");
    const size_t total = (batch + PACK_N - 1) / PACK_N * (size_t)(mask_size + 1) * PACK_N;
    pack_finish_kernel<<<ew_grid(ctx, total), 256, 0, ctx->stream>>>(c, b, (u32)mask_size, (u64)batch, out, (u64)total);
    return launch_check(ctx, "pack_finish_kernel");
}

size_t nb_tree_planes_bytes(size_t n, int mask_size)
{
    if (n == 0 || n > (1u << 20) || mask_size < 1 || mask_size > 16) return 0;
    return 4 * (size_t)tree_k_padded((u32)n) * (size_t)(mask_size + 1) * PACK_N;
}

// n t digit rows padded to kpad, and exact sums for signed digits of magnitude up to 128
static int tree_check_shape(nb_ctx *ctx, size_t n, int mask_size, const char *what)
{
    if (n == 0 || n > (1u << 20) || !plane_gemm_exact(tree_k_padded((u32)n), 128))
        return fail(ctx, NB_EINVAL, std::string(what) + ": n t (padded to 32) * 128 * 255 must be below 2^31");
    if (mask_size < 1 || mask_size > 16) return fail(ctx, NB_EINVAL, std::string(what) + ": bad mask size");
    return NB_OK;
}

int nb_tree_prepare(nb_ctx *ctx, const int32_t *masks, const int32_t *body, size_t n, int mask_size, uint8_t *planes)
{
    if (!ctx) return NB_EINVAL;
    if (!masks || !body || !planes) return fail(ctx, NB_EINVAL, "nb_tree_prepare: null argument");
    NB_TRY(tree_check_shape(ctx, n, mask_size, "nb_tree_prepare"));
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:tree_prepare");
    const size_t quads = (size_t)(mask_size + 1) * PACK_N * (tree_k_padded((u32)n) / 4);
    const size_t blocks = (quads + 255) / 256, cap = (size_t)ctx->sm_count * 16;
    plane_prepare_kernel<TreeSource, const i32 *__restrict__, const i32 *__restrict__, u32, u32>
        <<<(int)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>(planes, masks, body, (u32)n, (u32)mask_size);
    return launch_check(ctx, "plane_prepare_kernel<TreeSource>");
}

int nb_tree_keyswitch(nb_ctx *ctx, const int32_t *a, const uint8_t *planes, size_t n, int mask_size, int32_t *out,
                      size_t rows)
{
    if (!ctx) return NB_EINVAL;
    if (!a || !planes || !out) return fail(ctx, NB_EINVAL, "nb_tree_keyswitch: null argument");
    NB_TRY(tree_check_shape(ctx, n, mask_size, "nb_tree_keyswitch"));
    if (rows == 0) return NB_OK;
    const size_t rows_per_cta = (size_t)GEMM_WARPS * GEMM_MTILES * 16;
    const size_t ctas = (rows + rows_per_cta - 1) / rows_per_cta;
    if (ctas > 0x7fffffffu) return fail(ctx, NB_EINVAL, "nb_tree_keyswitch: too many rows");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:tree_keyswitch");
    const u32 cols = (u32)(mask_size + 1) * PACK_N;
    const dim3 grid((unsigned)ctas, cols / (8 * TreeGemm::NTILES));
    plane_gemm_kernel<TreeGemm, const i32 *__restrict__, u32, u32, i32 *__restrict__>
        <<<grid, GEMM_WARPS * 32, 0, ctx->stream>>>(planes, (u64)rows, a, (u32)n, cols, out);
    return launch_check(ctx, "plane_gemm_kernel<TreeGemm>");
}

int nb_tree_assemble(nb_ctx *ctx, const int32_t *v, const int32_t *b, int bits, int mask_size, int32_t *tv,
                     size_t count)
{
    if (!ctx) return NB_EINVAL;
    if (!v || !b || !tv) return fail(ctx, NB_EINVAL, "nb_tree_assemble: null argument");
    if (bits < 1 || bits > 2) return fail(ctx, NB_EINVAL, "nb_tree_assemble: bits must be 1 or 2");
    if (mask_size < 1 || mask_size > 16) return fail(ctx, NB_EINVAL, "nb_tree_assemble: bad mask size");
    if (count == 0) return NB_OK;
    const size_t ctas = count * (size_t)(mask_size + 1);
    if (ctas > 0x7fffffffu) return fail(ctx, NB_EINVAL, "nb_tree_assemble: too many test vectors");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:tree_assemble");
    tree_assemble_kernel<<<(unsigned)ctas, TREE_ASM_THREADS, 0, ctx->stream>>>(v, b, bits, (u32)mask_size, tv);
    return launch_check(ctx, "tree_assemble_kernel");
}

// ---- encrypted-index lookups (index_lookup.cuh) ----

int nb_index_prepare(nb_ctx *ctx, const int32_t *ggsw, size_t rows, uint64_t *spectra)
{
    if (!ctx) return NB_EINVAL;
    if (!ggsw || !spectra) return fail(ctx, NB_EINVAL, "nb_index_prepare: null argument");
    if (rows == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:index_prepare");
    // field elements of CHUNK rows at a time (64 KB per row) in a scratch buffer the context keeps, so that a call
    // allocates (and synchronises the device) only the first time, then bk_spectra_kernel's split and transforms
    constexpr size_t CHUNK = 1024;
    const size_t chunk = rows < CHUNK ? rows : CHUNK, cap = (size_t)ctx->sm_count * 16;
    NB_TRY(reserve_words(ctx, (void **)&ctx->d_index_tmp, &ctx->index_tmp_words, chunk * 8 * NTT_N + 1, sizeof(u64)));
    u64 *tmp = ctx->d_index_tmp;
    // bk_spectra_kernel's integrality flag: int32 coefficients never set it, so it is neither initialised nor read
    int *d_flag = (int *)(tmp + chunk * 8 * NTT_N);
    for (size_t r0 = 0; r0 < rows; r0 += chunk) {
        const size_t n = (rows - r0 < chunk ? rows - r0 : chunk), words = n * 8 * NTT_N, blocks = (words + 255) / 256;
        index_i32_to_field_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>(ggsw + r0 * 8 * NTT_N, tmp, words);
        bk_spectra_kernel<<<(unsigned)(n * 8), 64, 0, ctx->stream>>>(tmp, (u64 *)spectra + r0 * BK_FFT_U64, ctx->d_fft_tab,
                                                                      d_flag, BK_FFT_U64, 0);
        NB_TRY(launch_check(ctx, "index_prepare"));
    }
    return NB_OK;
}

}  // extern "C"

// the bits of an index and the columns of a table: columns * 2^bits fit one polynomial below 10 bits
static int index_check_bits(nb_ctx *ctx, const char *what, int bits, size_t columns)
{
    if (bits < 1 || bits > 20) return fail(ctx, NB_EINVAL, std::string(what) + ": bits must be 1 to 20");
    if (columns == 0 || (bits < 10 && (columns << bits) > (size_t)NTT_N))
        return fail(ctx, NB_EINVAL, std::string(what) + ": columns * 2^bits must be at most N below 10 bits");
    return NB_OK;
}

// One launch of the index kernel of the entry point `what` over p.queries x p.nodes items, BrFft::CT per CTA, enqueued by
// launch(ctas, smem).  With table_ids_host, query q works on table table_ids_host[q]: each id is checked, then uploaded.
template <class Args, class Launch>
static int index_run(nb_ctx *ctx, const char *what, Args &p, const uint32_t *table_ids_host, size_t tables, Launch launch)
{
    p.items = p.queries * p.nodes;
    const size_t ctas = (p.items + BrFft::CT - 1) / BrFft::CT;
    if (p.nodes > ((size_t)1 << 40) / p.queries || ctas > 0x7fffffffu)
        return fail(ctx, NB_EINVAL, std::string(what) + ": too many items");
    if (table_ids_host)
        for (size_t q = 0; q < p.queries; q++)
            if (table_ids_host[q] >= tables)
                return fail(ctx, NB_EINVAL, std::string(what) + ": query " + std::to_string(q) + " names table " +
                                                std::to_string(table_ids_host[q]) + " of " + std::to_string(tables));
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range(("nufhe_b200:" + std::string(what + 3)).c_str());     // named after the entry point
    p.fft_tab = ctx->d_fft_tab;
    if (table_ids_host) {
        NB_TRY(mk_upload(ctx, table_ids_host, p.queries * sizeof(u32)));
        p.table_id = reinterpret_cast<const u32 *>(ctx->d_mk);
    }
    launch((unsigned)ctas, br_smem_bytes<BrFft>());
    return launch_check(ctx, what);
}

// nb_index_cmux_level, and with `indirect` nb_index_cmux_level_indirect: query q reads table table_ids_host[q] < tables
static int index_cmux_level(nb_ctx *ctx, const char *what, bool indirect, const int32_t *in, size_t in_stride,
                            size_t tables, const uint32_t *table_ids_host, const uint64_t *sel, size_t sel_stride,
                            int32_t *out, size_t nodes, size_t queries)
{
    if (!ctx || !in || !sel || !out || (indirect && !table_ids_host)) return fail(ctx, NB_EINVAL, std::string(what) + ": null argument");
    if (indirect && in_stride < 4 * nodes * (size_t)NTT_N) return fail(ctx, NB_EINVAL, std::string(what) + ": tables overlap");
    if (nodes == 0 || queries == 0) return NB_OK;
    IndexArgs p{};
    p.in = in; p.in_stride = in_stride; p.sel = (const u64 *)sel; p.sel_stride = sel_stride;
    p.out = out; p.nodes = nodes; p.queries = queries;
    return index_run(ctx, what, p, table_ids_host, tables, [&](unsigned ctas, size_t smem) {
        if (indirect) index_lookup_kernel<false, true><<<ctas, BrFft::THREADS, smem, ctx->stream>>>(p);
        else index_lookup_kernel<false><<<ctas, BrFft::THREADS, smem, ctx->stream>>>(p);
    });
}

// nb_index_rotate_extract, and with `indirect` nb_index_rotate_extract_indirect (tables as for index_cmux_level)
static int index_rotate_extract(nb_ctx *ctx, const char *what, bool indirect, const int32_t *in, size_t in_stride,
                                size_t tables, const uint32_t *table_ids_host, const uint64_t *sel, size_t sel_stride,
                                int bits, size_t columns, int32_t *out_a, int32_t *out_b, size_t queries)
{
    if (!ctx || !in || !sel || !out_a || !out_b || (indirect && !table_ids_host)) return fail(ctx, NB_EINVAL, std::string(what) + ": null argument");
    NB_TRY(index_check_bits(ctx, what, bits, columns));
    IndexArgs p{};
    p.nodes = bits >= 10 ? columns : 1;
    if (indirect && in_stride < 2 * p.nodes * (size_t)NTT_N) return fail(ctx, NB_EINVAL, std::string(what) + ": tables overlap");
    if (queries == 0) return NB_OK;
    p.in = in; p.in_stride = in_stride; p.sel = (const u64 *)sel; p.sel_stride = sel_stride;
    p.out_a = out_a; p.out_b = out_b; p.queries = queries;
    p.samples = bits >= 10 ? 1 : (int)columns;
    p.steps = bits < 10 ? bits : 10;
    p.log2_stride = bits;
    return index_run(ctx, what, p, table_ids_host, tables, [&](unsigned ctas, size_t smem) {
        if (indirect) index_lookup_kernel<true, true><<<ctas, BrFft::THREADS, smem, ctx->stream>>>(p);
        else index_lookup_kernel<true><<<ctas, BrFft::THREADS, smem, ctx->stream>>>(p);
    });
}

extern "C" {

int nb_index_cmux_level(nb_ctx *ctx, const int32_t *in, size_t in_query_stride, const uint64_t *sel,
                        size_t sel_query_stride, int32_t *out, size_t nodes, size_t queries)
{
    return index_cmux_level(ctx, "nb_index_cmux_level", false, in, in_query_stride, 0, nullptr, sel, sel_query_stride, out, nodes, queries);
}

int nb_index_rotate_extract(nb_ctx *ctx, const int32_t *acc, size_t acc_query_stride, const uint64_t *sel,
                            size_t sel_query_stride, int bits, size_t columns, int32_t *out_a, int32_t *out_b,
                            size_t queries)
{
    return index_rotate_extract(ctx, "nb_index_rotate_extract", false, acc, acc_query_stride, 0, nullptr, sel,
                                sel_query_stride, bits, columns, out_a, out_b, queries);
}

int nb_index_cmux_level_indirect(nb_ctx *ctx, const int32_t *tables, size_t table_stride, size_t table_count,
                                 const uint32_t *table_ids_host, const uint64_t *sel, size_t sel_query_stride,
                                 int32_t *out, size_t nodes, size_t queries)
{
    return index_cmux_level(ctx, "nb_index_cmux_level_indirect", true, tables, table_stride, table_count, table_ids_host,
                            sel, sel_query_stride, out, nodes, queries);
}

int nb_index_rotate_extract_indirect(nb_ctx *ctx, const int32_t *tables, size_t table_stride, size_t table_count,
                                     const uint32_t *table_ids_host, const uint64_t *sel, size_t sel_query_stride,
                                     int bits, size_t columns, int32_t *out_a, int32_t *out_b, size_t queries)
{
    return index_rotate_extract(ctx, "nb_index_rotate_extract_indirect", true, tables, table_stride, table_count,
                                table_ids_host, sel, sel_query_stride, bits, columns, out_a, out_b, queries);
}

// ---- oblivious writes (index_lookup.cuh, DESIGN.md section 21) ----

int nb_index_write_assemble(nb_ctx *ctx, const int32_t *v, const int32_t *b, int bits, size_t columns, int32_t *out,
                            size_t queries)
{
    const char *what = "nb_index_write_assemble";
    if (!ctx) return NB_EINVAL;
    if (!b || !out) return fail(ctx, NB_EINVAL, std::string(what) + ": null argument");
    NB_TRY(index_check_bits(ctx, what, bits, columns));
    if (queries == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:index_write_assemble");
    const u64 total = (u64)queries * (bits >= 10 ? columns : 1) * 2 * NTT_N;
    index_write_assemble_kernel<<<ew_grid(ctx, total), 256, 0, ctx->stream>>>(v, b, bits, (u32)columns, out, total);
    return launch_check(ctx, "index_write_assemble_kernel");
}

// out or (acc, acc_stride, acc_count, table_ids_host): the last level adds into the tables instead of storing
static int index_write_launch(nb_ctx *ctx, IndexWriteArgs &p, bool rotate, size_t out_nodes, size_t acc_count,
                              const uint32_t *table_ids_host, const char *what)
{
    if (!p.in || !p.sel || (!p.out && !p.acc)) return fail(ctx, NB_EINVAL, std::string(what) + ": null argument");
    if (p.acc && (acc_count == 0 || p.acc_stride < out_nodes * 2 * NTT_N || (!table_ids_host && acc_count != 1)))
        return fail(ctx, NB_EINVAL, std::string(what) + ": the tables overlap or are not named per query");
    if (p.nodes == 0 || p.queries == 0) return NB_OK;
    return index_run(ctx, what, p, p.acc ? table_ids_host : nullptr, acc_count, [&](unsigned ctas, size_t smem) {
        if (rotate) index_write_kernel<true><<<ctas, BrFft::THREADS, smem, ctx->stream>>>(p);
        else index_write_kernel<false><<<ctas, BrFft::THREADS, smem, ctx->stream>>>(p);
    });
}

int nb_index_write_rotate(nb_ctx *ctx, const int32_t *delta, const uint64_t *sel, size_t sel_query_stride, int bits,
                          size_t columns, int32_t *out, int32_t *acc, size_t acc_stride, size_t acc_count,
                          const uint32_t *table_ids_host, size_t queries)
{
    const char *what = "nb_index_write_rotate";
    if (!ctx) return NB_EINVAL;
    NB_TRY(index_check_bits(ctx, what, bits, columns));
    if ((acc != nullptr) != (bits <= 10))
        return fail(ctx, NB_EINVAL, std::string(what) + ": the rotation adds into the tables exactly when bits <= 10");
    IndexWriteArgs p{};
    p.in = delta; p.sel = (const u64 *)sel; p.sel_stride = sel_query_stride;
    p.out = out; p.acc = acc; p.acc_stride = acc_stride; p.queries = queries;
    p.nodes = bits >= 10 ? columns : 1;
    p.steps = bits < 10 ? bits : 10;
    return index_write_launch(ctx, p, true, p.nodes, acc_count, table_ids_host, what);
}

int nb_index_demux_level(nb_ctx *ctx, const int32_t *in, const uint64_t *sel, size_t sel_query_stride, int32_t *out,
                         int32_t *acc, size_t acc_stride, size_t acc_count, const uint32_t *table_ids_host,
                         size_t nodes, size_t queries)
{
    if (!ctx) return NB_EINVAL;
    IndexWriteArgs p{};
    p.in = in; p.sel = (const u64 *)sel; p.sel_stride = sel_query_stride;
    p.out = acc ? nullptr : out; p.acc = acc; p.acc_stride = acc_stride; p.nodes = nodes; p.queries = queries;
    return index_write_launch(ctx, p, false, 2 * nodes, acc_count, table_ids_host, "nb_index_demux_level");
}

// ---- compact public-key encryption (compact.cuh) ----

int nb_compact_finish(nb_ctx *ctx, const int32_t *c, const int32_t *e1, const int32_t *e2, const int32_t *mus,
                      int mask_size, uint16_t *out, size_t batch)
{
    if (!ctx) return NB_EINVAL;
    if (!c || !e1 || !e2 || !mus || !out) return fail(ctx, NB_EINVAL, "nb_compact_finish: null argument");
    if (mask_size < 1 || mask_size > (1 << 16)) return fail(ctx, NB_EINVAL, "nb_compact_finish: bad mask size");
    if (batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:compact_finish");
    const size_t total = (batch + PACK_N - 1) / PACK_N * (size_t)(mask_size + 1) * PACK_N;
    compact_finish_kernel<<<ew_grid(ctx, total), 256, 0, ctx->stream>>>(c, e1, e2, mus, (u32)mask_size, (u64)batch, out,
                                                                        (u64)total);
    return launch_check(ctx, "compact_finish_kernel");
}

int nb_compact_extract(nb_ctx *ctx, const uint16_t *data, int mask_size, int32_t *out_a, int32_t *out_b, size_t rows)
{
    if (!ctx) return NB_EINVAL;
    if (!data || !out_a || !out_b) return fail(ctx, NB_EINVAL, "nb_compact_extract: null argument");
    if (mask_size < 1 || mask_size > 65535) return fail(ctx, NB_EINVAL, "nb_compact_extract: bad mask size");
    if (((uintptr_t)data & 7) || ((uintptr_t)out_a & 15))
        return fail(ctx, NB_EINVAL, "nb_compact_extract: data must be 8-byte and out_a 16-byte aligned");
    if (rows == 0) return NB_OK;
    const size_t groups = (rows + PACK_N - 1) / PACK_N;
    if (groups > 65535) return fail(ctx, NB_EINVAL, "nb_compact_extract: more than 65535 groups in one call");
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:compact_extract");
    const dim3 grid(PACK_N / CX_ROWS, (unsigned)groups, (unsigned)mask_size);
    compact_extract_kernel<<<grid, CX_THREADS, 0, ctx->stream>>>(data, (u32)mask_size, (u64)rows, out_a, out_b);
    return launch_check(ctx, "compact_extract_kernel");
}

}  // extern "C"

// ---- multi-key calls (DESIGN.md section 17) --------------------------------------------------------------------

extern "C" {

int nb_mk_keyswitch(nb_ctx *ctx, const int32_t *src1_a, const int32_t *src1_b, const int32_t *src2_a,
                    const int32_t *src2_b, int32_t c, const int32_t *const *ks_a_host, const int32_t *const *ks_b_host,
                    const float *const *ks_cv_host, const size_t *counts_host, size_t tenants, size_t in_size, size_t n,
                    int t, int log2_base, int32_t *res_a, int32_t *res_b, float *res_cv, size_t batch)
{
    const char *what = "nb_mk_keyswitch";
    NB_TRY(mk_preamble(ctx, what, counts_host, tenants, batch, src1_a && src1_b && res_a && res_b, "key", ks_a_host,
                       ks_b_host, ks_cv_host));
    NB_TRY(check_pair(ctx, what, src2_a, src2_b, "src2_a/src2_b"));
    if (!(t == 8 && log2_base == 2 && in_size == (size_t)KS_IN && n == (size_t)KS_N))
        return fail(ctx, NB_EUNSUPPORTED, std::string(what) + ": the grouped key switch is for in = 1024, n = 500, t = 8, base 4 only");
    if (batch == 0) return NB_OK;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:multikey_keyswitch");
    KeyswitchArgs p{};
    p.src1_a = src1_a; p.src1_b = src1_b; p.src2_a = src2_a; p.src2_b = src2_b; p.c = c;
    p.res_a = res_a; p.res_b = res_b; p.res_cv = res_cv;
    p.in_size = (int)in_size; p.n = (int)n; p.t = t; p.log2_base = log2_base; p.batch = batch; p.tile = KS_TILE;
    // segments that nb_keyswitch would run as the GEMM run so on their own; the others become tiles of the gather kernel
    std::vector<KsTile> tiles;
    std::vector<std::pair<KeyswitchArgs, const uint8_t *>> gemm;      // (segment, planes)
    size_t row = 0;
    for (size_t k = 0; k < tenants; row += counts_host[k], k++) {
        const size_t cnt = counts_host[k];
        KeyswitchArgs s = p;      // rows [row, row + cnt)
        s.src1_a += row * KS_IN; s.src1_b += row; s.src2_a = src2_a ? src2_a + row * KS_IN : nullptr;
        s.src2_b = src2_b ? src2_b + row : nullptr; s.res_a += row * KS_N; s.res_b += row; s.res_cv = res_cv ? res_cv + row : nullptr;
        s.ks_a = ks_a_host[k]; s.ks_b = ks_b_host[k]; s.ks_cv = ks_cv_host[k]; s.batch = cnt;
        if (const uint8_t *planes = cnt ? ks_gemm_planes(ctx, s) : nullptr) {
            gemm.emplace_back(s, planes);
            continue;
        }
        for (size_t q = 0; q < cnt; q += KS_TILE)
            tiles.push_back({ks_a_host[k], ks_b_host[k], ks_cv_host[k], row + q, (int)std::min<size_t>(KS_TILE, cnt - q)});
    }
    // the gather launch zeroes and finalizes the variances of the whole batch: the GEMM segments are written after it
    if (!tiles.empty())
        NB_TRY(ks_gather(ctx, p, tiles.size(), "keyswitch_grouped_kernel", [&](dim3 grid) {
            NB_TRY(mk_upload(ctx, tiles.data(), tiles.size() * sizeof(KsTile)));
            keyswitch_grouped_kernel<<<grid, KS_THREADS, KS_SMEM_BYTES, ctx->stream>>>(p, reinterpret_cast<const KsTile *>(ctx->d_mk));
            return NB_OK;
        }));
    for (const auto &g : gemm) NB_TRY(ks_gemm(ctx, g.first, g.second));
    return NB_OK;
}

int nb_mk_tree_keyswitch(nb_ctx *ctx, const int32_t *a, const uint8_t *const *planes_host, const size_t *counts_host,
                         size_t tenants, size_t n, int mask_size, int32_t *out, size_t rows)
{
    const char *what = "nb_mk_tree_keyswitch";
    NB_TRY(mk_preamble(ctx, what, counts_host, tenants, rows, a && out, "planes", planes_host));
    NB_TRY(tree_check_shape(ctx, n, mask_size, what));
    if (rows == 0) return NB_OK;
    std::vector<TreeTile> tiles(mk_tree_tiles(counts_host, tenants, planes_host, nullptr));
    if (tiles.size() > 0x7fffffffu) return fail(ctx, NB_EINVAL, std::string(what) + ": too many rows");
    mk_tree_tiles(counts_host, tenants, planes_host, tiles.data());
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:multikey_tree_keyswitch");
    NB_TRY(mk_upload(ctx, tiles.data(), tiles.size() * sizeof(TreeTile)));
    const u32 cols = (u32)(mask_size + 1) * PACK_N;
    const dim3 grid((unsigned)tiles.size(), cols / (8 * TreeGemm::NTILES));
    tree_gemm_mk_kernel<<<grid, GEMM_WARPS * 32, 0, ctx->stream>>>(reinterpret_cast<const TreeTile *>(ctx->d_mk), a,
                                                                   (u32)n, cols, out);
    return launch_check(ctx, "tree_gemm_mk_kernel");
}

int nb_mk_ntt_mac(nb_ctx *ctx, const uint64_t *x, const uint64_t *const *key_host, const size_t *group_counts_host,
                  size_t tenants, uint64_t *out, size_t rows, size_t outs, size_t groups)
{
    const char *what = "nb_mk_ntt_mac";
    NB_TRY(mk_preamble(ctx, what, group_counts_host, tenants, groups, x && out, "key", key_host));
    if (rows == 0 || outs == 0 || rows > (1u << 24) || outs > (1u << 16))
        return fail(ctx, NB_EINVAL, std::string(what) + ": rows must be in [1, 2^24] and outputs in [1, 2^16]");
    if (groups == 0) return NB_OK;
    const size_t ctas = groups * (PACK_N / MAC_POINTS);
    if (ctas > 0x7fffffffu) return fail(ctx, NB_EINVAL, std::string(what) + ": too many groups");
    std::vector<const u64 *> group_keys(groups);
    mk_group_keys(group_counts_host, tenants, reinterpret_cast<const u64 *const *>(key_host), group_keys.data());
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:multikey_ntt_mac");
    NB_TRY(mk_upload(ctx, group_keys.data(), groups * sizeof(const u64 *)));
    const dim3 grid((unsigned)ctas, (unsigned)((outs + MAC_OUTS - 1) / MAC_OUTS));
    ntt_mac_mk_kernel<<<grid, MAC_WARPS * 32, 0, ctx->stream>>>((const u64 *)x, reinterpret_cast<const u64 *const *>(ctx->d_mk),
                                                               (u64 *)out, (u32)rows, (u32)outs);
    return launch_check(ctx, "ntt_mac_mk_kernel");
}

// ---- re-encryption (reencrypt.cuh, DESIGN.md section 22) ----

int nb_reencrypt(nb_ctx *ctx, const int32_t *a, const int32_t *b, size_t n, int mask_size,
                 const uint64_t *const *mask_spectra_host, const int32_t *const *bodies_host, const size_t *counts_host,
                 size_t keys, int32_t *out_a, int32_t *out_b, size_t rows)
{
    const char *what = "nb_reencrypt";
    NB_TRY(mk_preamble(ctx, what, counts_host, keys, rows, a && b && out_a && out_b, "key", mask_spectra_host, bodies_host));
    if (n == 0) return fail(ctx, NB_EINVAL, std::string(what) + ": n must be at least 1");
    if (mask_size != 1 || n * REENC_LEVELS > (size_t)PACK_N)
        return fail(ctx, NB_EUNSUPPORTED, std::string(what) + ": re-encryption is for k = 1 and n t <= 1024 only");
    bool aligned = !(((uintptr_t)a | (uintptr_t)b | (uintptr_t)out_b) & 3) && !((uintptr_t)out_a & 15);
    for (size_t q = 0; q < keys; q++)
        aligned = aligned && !((uintptr_t)mask_spectra_host[q] & 15) && !((uintptr_t)bodies_host[q] & 3);
    if (!aligned)
        return fail(ctx, NB_EINVAL, std::string(what) + ": out_a and the mask spectra must be 16-byte aligned, a, b, out_b "
                                                         "and the bodies 4-byte aligned");
    if (rows == 0) return NB_OK;
    const auto *spectra = reinterpret_cast<const u64 *const *>(mask_spectra_host);
    std::vector<ReencTile> tiles(reenc_tiles(counts_host, keys, spectra, bodies_host, nullptr));
    reenc_tiles(counts_host, keys, spectra, bodies_host, tiles.data());
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:reencrypt");
    NB_TRY(mk_upload(ctx, tiles.data(), tiles.size() * sizeof(ReencTile)));
    const size_t cap = (size_t)ctx->sm_count * REENC_CTAS;
    const unsigned grid = (unsigned)(tiles.size() < cap ? tiles.size() : cap);
    reencrypt_kernel<<<grid, NTT_SWEEP_THREADS, reenc_smem_bytes(), ctx->stream>>>(
        reinterpret_cast<const ReencTile *>(ctx->d_mk), (u64)tiles.size(), a, b, (u32)n, out_a, out_b, ctx->d_ph_fwd,
        ctx->d_ph_inv);
    return launch_check(ctx, "reencrypt_kernel");
}

// ---- multi-key expansion of compressed cloud keys (DESIGN.md section 19) ----

int nb_mk_bk_expand(nb_ctx *ctx, const uint32_t *seeds_host, const int32_t *const *bodies_host,
                    uint64_t *const *slots_host, size_t tenants, size_t n, int mask_size, int decomp_length,
                    size_t poly_degree)
{
    const char *what = "nb_mk_bk_expand";
    if (!ctx) return NB_EINVAL;
    if (tenants && (!seeds_host || !bodies_host || !slots_host)) return fail(ctx, NB_EINVAL, std::string(what) + ": null argument");
    if (mask_size != 1 || decomp_length != 2 || poly_degree != (size_t)NTT_N || n == 0 || n > (size_t)LWE_N_MAX)
        return fail(ctx, NB_EUNSUPPORTED, std::string(what) + ": the expansion is for k = 1, l = 2, N = 1024 and 1 <= n <= " +
                                              std::to_string(LWE_N_MAX) + " only");
    NB_TRY(mk_check_tenants(ctx, what, "bodies or slot", tenants, bodies_host, slots_host));
    if (tenants == 0) return NB_OK;
    if (tenants * n * 8 > 0x7fffffffu) return fail(ctx, NB_EINVAL, std::string(what) + ": too many rows in one call");
    std::vector<MkBkTenant> table(tenants);
    for (size_t t = 0; t < tenants; t++) {
        memcpy(table[t].seed, seeds_host + 8 * t, sizeof(table[t].seed));
        table[t].body = bodies_host[t];
        table[t].slot = slots_host[t];
    }
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:multikey_bk_expand");
    NB_TRY(mk_upload(ctx, table.data(), tenants * sizeof(MkBkTenant)));
    mk_bk_expand_kernel<<<(unsigned)(tenants * n * 8), 64, 0, ctx->stream>>>(reinterpret_cast<const MkBkTenant *>(ctx->d_mk),
                                                                          (u32)n, ctx->d_fft_tab);
    NB_TRY(launch_check(ctx, "mk_bk_expand_kernel"));
    // a slot serves the nb_mk_* bootstraps only: its NTT planes are not written
    for (size_t t = 0; t < tenants; t++) {
        const u64 *begin = slots_host[t], *end = begin + n * BK_ROW_U64;
        forget_keys(ctx, begin, end);
        ctx->mk_slots.emplace_back(begin, end);
    }
    return NB_OK;
}

int nb_mk_ks_expand(nb_ctx *ctx, const uint32_t *seeds_host, int32_t *const *ks_a_host, size_t tenants, size_t in_size,
                    int t, int log2_base, size_t n)
{
    const char *what = "nb_mk_ks_expand";
    if (!ctx) return NB_EINVAL;
    if (tenants && (!seeds_host || !ks_a_host)) return fail(ctx, NB_EINVAL, std::string(what) + ": null argument");
    if (!(t == 8 && log2_base == 2 && in_size == (size_t)KS_IN && n == (size_t)KS_N))
        return fail(ctx, NB_EUNSUPPORTED, std::string(what) + ": the expansion is for the multi-key key switch, in = 1024, "
                                                             "n = 500, t = 8, base 4 only");
    NB_TRY(mk_check_tenants(ctx, what, "ks_a", tenants, ks_a_host));
    if (tenants == 0) return NB_OK;
    if (tenants > 65535) return fail(ctx, NB_EINVAL, std::string(what) + ": more than 65535 tenants in one call");
    std::vector<MkKsTenant> table(tenants);
    for (size_t k = 0; k < tenants; k++) {
        memcpy(table[k].seed, seeds_host + 8 * k, sizeof(table[k].seed));
        table[k].ks_a = ks_a_host[k];
        // GEMM planes registered for a key that lived at this address no longer describe it
        for (size_t i = 0; i < ctx->ks_keys.size();) {
            if (ctx->ks_keys[i].ks_a == ks_a_host[k]) ctx->ks_keys.erase(ctx->ks_keys.begin() + i);
            else i++;
        }
    }
    const u32 base = 1u << log2_base;
    const u64 rows = (u64)in_size * t, words = rows * (base - 1) * n;
    const u64 blocks = (words + 15) / 16, per_tenant = (blocks + MK_KS_THREADS - 1) / MK_KS_THREADS;
    u64 ctas = (u64)ctx->sm_count * 8 / tenants;
    if (ctas < 1) ctas = 1;
    if (ctas > per_tenant) ctas = per_tenant;
    NB_ON_DEVICE(ctx);
    NvtxRange nvtx_range("nufhe_b200:multikey_ks_expand");
    NB_TRY(mk_upload(ctx, table.data(), tenants * sizeof(MkKsTenant)));
    mk_ks_expand_kernel<<<dim3((unsigned)ctas, (unsigned)tenants), MK_KS_THREADS, 0, ctx->stream>>>(
        reinterpret_cast<const MkKsTenant *>(ctx->d_mk), words, rows, (u32)n, base);
    return launch_check(ctx, "mk_ks_expand_kernel");
}

int nb_mk_slot_release(nb_ctx *ctx, const uint64_t *slot)
{
    if (!ctx) return NB_EINVAL;
    if (!slot) return fail(ctx, NB_EINVAL, "nb_mk_slot_release: null slot");
    for (size_t i = 0; i < ctx->mk_slots.size();) {
        if (ctx->mk_slots[i].first == (const u64 *)slot) ctx->mk_slots.erase(ctx->mk_slots.begin() + i);
        else i++;
    }
    return NB_OK;
}

}  // extern "C"
