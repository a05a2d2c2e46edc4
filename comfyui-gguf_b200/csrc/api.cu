// api.cu -- the extern "C" boundary declared in include/ggufb200.h.
// Argument validation and route selection live here; kernels live in dequant.cu / rows.cu / gemv.cu / gemv2.cu /
// linear_sm90.cu / repack.cu / scale.cu / lowrank.cu / quantize.cu (declared in internal.h).  Routing is a pure function of the call's arguments (algo | flags):
// no process-wide routing state.
#include <stdlib.h>

#include "blocks.cuh"
#include "fallback.cuh"
#include "internal.h"

using namespace ggufb200;

static bool type_geom(int t, int *bs, int *ts)
{
    int b = 1, s = 2;       // BF16: one 2-byte element per "block"
    const bool known = t == T_BF16 || with_block(t, false, [&](auto blk) {
        b = decltype(blk)::BS;
        s = decltype(blk)::TS;
        return true;
    });
    if (!known) return false;
    if (bs) *bs = b;
    if (ts) *ts = s;
    return true;
}

static bool dtype_ok(int d) { return d >= 0 && d <= 2; }
static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static bool fused_type(int t) { return t != T_BF16 && type_geom(t, nullptr, nullptr); }     // every block format has a fused producer

// the types ggufb200_linear_grad_input dequantises: the table (ggufb200_dequant) and the numpy-fallback types
static bool grad_type(int t, int *bs)
{
    int b = 0;
    const bool known = type_geom(t, &b, nullptr) || with_fallback_block(t, false, [&](auto blk) {
        b = decltype(blk)::BS;
        return true;
    });
    if (known && bs) *bs = b;
    return known;
}

// ------------------------------------------------------------------ device gate
// The library contains sm_90a code only.  Checked once per device, right before the first launch on it (argument
// errors are still reported without a GPU).
static int device_check()
{
    static signed char ok[64] = {};     // 0 = unknown, 1 = sm_90, -1 = something else
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        cudaGetLastError();
        return GGUFB200_E_CUDA;
    }
    if (dev < 0 || dev >= 64) return GGUFB200_OK;
    if (ok[dev] == 0) {
        int major = 0, minor = 0;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) {
            cudaGetLastError();
            return GGUFB200_E_CUDA;
        }
        ok[dev] = (major == 9 && minor == 0) ? 1 : -1;
    }
    return ok[dev] == 1 ? GGUFB200_OK : GGUFB200_E_DEVICE;
}

// ------------------------------------------------------------------ route selection
struct Route {
    int algo;          // GGUFB200_ALGO_* without flags
    size_t ws;         // workspace bytes the route wants (0 = none)
};

// GGUFB200_FLAG_* bits -> the options of the warpgroup-MMA routes (GENERIC wins over EXACT_W, TILE384 over TILE192).
// A straddled weight never cuts K into ranges.
static LinearOptions linear_options(int flags, bool straddled)
{
    LinearOptions o;
    if (flags & GGUFB200_FLAG_GENERIC) o.producers = LinearOptions::GENERIC;
    else if (flags & GGUFB200_FLAG_EXACT_W) o.producers = LinearOptions::EXACT;
    if (flags & GGUFB200_FLAG_TILE384) o.tile = 384;
    else if (flags & GGUFB200_FLAG_TILE192) o.tile = 192;
    o.nosplit = (flags & GGUFB200_FLAG_NOSPLIT) != 0 || straddled;
    return o;
}

// `W` may be NULL (workspace query: assume a 16-byte aligned weight); ws_avail = workspace the caller supplied (SIZE_MAX in a query);
// have_spans: the caller also holds the re-packed span-major copy of the weight (ggufb200_repack), which the FUSED_TMEM
// kernel can read for every block format and every K (for a straddled weight: the block-major copy)
static Route pick_route(int type, const void *W, long long M, long long N, long long K, int act, int math, int algo_flags,
                        const LinearOptions &opt, size_t ws_avail, bool have_spans = false)
{
    const int algo = algo_flags & GGUFB200_ALGO_MASK;
    const int flags = algo_flags & ~GGUFB200_ALGO_MASK;
    const size_t dense = (size_t)N * (size_t)K * 2;
    const bool w_ok = !W || aligned16(W);
    int bs = 1;
    type_geom(type, &bs, nullptr);
    const bool straddled = straddled_rows(bs, N, K);
    const bool fusable = fused_type(type) && math == kF16 && (K % 64) == 0 && (N % 8) == 0 && !straddled;
    Route r{algo, 0};
    if (algo == GGUFB200_ALGO_AUTO) {
        // Measured on an H100 80GB HBM3 (400 W power limit, Q4_K / Q6_K at Flux shapes, tools/bench_linear.py --graph):
        //  * M <= 8: the mma.sync GEMV takes 0.35-0.56 of FUSED_TMEM's time on every weight up to 21504 x 3072, so it serves all
        //    of them (the integer-pattern GEMV when the caller allows the `fast` contract);
        //  * M > 8: the FUSED_TMEM kernel;
        //  * weights that kernel cannot read (no span-major copy at hand): dequant once + the dense GEMM took 0.18-0.89 of the
        //    fused reference-exact kernel's time at every M from 64 to 4608, so FUSED_MMA is only taken when the caller's
        //    workspace cannot hold the dequantised weight.
        //  * a straddled weight (SD1.5 / SDXL K-quants at K % 256 != 0): dequant + dense GEMM at every M.  The GEMVs index whole rows;
        //    above M = 8, tools/bench_sd_linears.py (bf16 and fp16, Q4_K / Q6_K, M = 256 .. 8192, (N, K) = (640, 640), (5120, 640),
        //    (320, 320), (2560, 320)) measured dequant + GEMM at 0.58-1.05 of the reference-exact FUSED_TMEM kernel's time, 0.58-0.93
        //    for Q6_K (which FUSED_TMEM reads from the block-major copy).  FUSED_TMEM serves them when asked for (and the LoRA k-blocks).
        // A math dtype other than fp16 means the reference's own sequence in that dtype: standalone dequant + dense GEMM (or the GEMV).
        const bool tmem_ok = w_ok && fused_type(type) && math == kF16 && (N % 8) == 0 && (have_spans || fused_tmem_supported(type, W, N, K));
        const bool exact = (flags & GGUFB200_FLAG_EXACT_W) != 0 || math != kF16;
        if (!w_ok) r.algo = GGUFB200_ALGO_DEQUANT_MMA;
        else if (straddled) r.algo = GGUFB200_ALGO_DEQUANT_MMA;
        else if (M <= gemv_max_m() && !exact && gemv2_supported(type, W ? W : (const void *)16, N, K, M)) r.algo = GGUFB200_ALGO_GEMV_FAST;
        else if (M <= gemv_max_m()) r.algo = GGUFB200_ALGO_GEMV;
        else if (tmem_ok) r.algo = GGUFB200_ALGO_FUSED_TMEM;
        else if (fusable && ws_avail < dense) r.algo = GGUFB200_ALGO_FUSED_MMA;
        else r.algo = GGUFB200_ALGO_DEQUANT_MMA;
    }
    switch (r.algo) {
    case GGUFB200_ALGO_DEQUANT_MMA: r.ws = dense; break;
    case GGUFB200_ALGO_FUSED_MMA: r.ws = fusable ? fused_mma_workspace(M, N, K, opt) : 0; break;
    case GGUFB200_ALGO_FUSED_TMEM: r.ws = fused_tmem_workspace(M, N, K, opt); break;
    default: r.ws = 0;
    }
    (void)act;
    return r;
}

// ------------------------------------------------------------------ the Linear of the fallback.cuh formats
// block size and alignment (A_BLK) of a fallback format; false for every other code
static bool fallback_geom(int t, int *bs, int *a_blk)
{
    return with_fallback_block(t, false, [&](auto blk) {
        if (bs) *bs = decltype(blk)::BS;
        if (a_blk) *a_blk = decltype(blk)::A_BLK;
        return true;
    });
}

// AUTO: FUSED_SYNC up to this M where the kernel's plan cuts K into ranges (the feature x token tile grid fills at most half the
// SMs), else DEQUANT_MMA.  Measured on an H100 80GB HBM3 (700 W power limit; tools/bench_linear_fallback.py, the seven
// Qwen3-4B / Qwen2.5-VL-7B / Mistral-Small-24B shapes, bf16 and fp16, DESIGN.md section 9): the fused kernel is bound by its
// decoders, not by the packed bytes, so it wins only while it decodes each weight run once (M <= 64, one token tile) and split K
// puts every SM to work.  Median two-step / fused time on the split shapes at M = 64: 1.03 - 1.13 for the i-quants, 1.03 for
// TQ2_0, 0.98 / 0.96 for MXFP4 / NVFP4 (1.12 / 1.08 at M = 32); TQ2_0 stops at 32 too (its weakest point at 64: 0.76).  Over the
// points this rule sends to FUSED_SYNC at 8 < M <= 64 the median is 1.29, the weakest 0.90.  At
// M = 77 and above: 0.17 - 0.75 for every type.  TQ1_0's decoder (one trit per step) loses at every M (0.69 - 0.77): it stays on
// DEQUANT_MMA.  Unsplit grids ([9728, 2560] at 76 feature tiles, [18944, 3584], [32768, 5120]) ran at 0.52 - 0.98: DEQUANT_MMA.
static long long fallback_crossover(int type)
{
    switch (type) {
    case T_TQ1_0: return 0;
    case T_TQ2_0:
    case T_MXFP4:
    case T_NVFP4: return 32;
    }
    return 64;
}

// `W` may be NULL (workspace query: assume an aligned weight)
static Route pick_fallback_route(int type, const void *W, long long M, long long N, long long K, int algo_flags)
{
    int a_blk = 1;
    fallback_geom(type, nullptr, &a_blk);
    const bool w_ok = !W || reinterpret_cast<uintptr_t>(W) % a_blk == 0;
    Route r{algo_flags & GGUFB200_ALGO_MASK, 0};
    if (!w_ok) r.algo = GGUFB200_ALGO_DEQUANT_MMA;
    else if (r.algo == GGUFB200_ALGO_AUTO)
        r.algo = M <= fallback_crossover(type) && fallback_linear_workspace(M, N, K, false) > 0 ? GGUFB200_ALGO_FUSED_SYNC
                                                                                                : GGUFB200_ALGO_DEQUANT_MMA;
    if (r.algo == GGUFB200_ALGO_DEQUANT_MMA) r.ws = (size_t)N * (size_t)K * 2;
    else if (r.algo == GGUFB200_ALGO_FUSED_SYNC) r.ws = fallback_linear_workspace(M, N, K, (algo_flags & GGUFB200_FLAG_NOSPLIT) != 0);
    return r;
}

// the argument checks of ggufb200_linear_fallback that need no pointer (0: fine)
static int fallback_linear_args(int ggml_type, int64_t N, int64_t K, int64_t M, int64_t ldx, int64_t ldy, int act_dtype, int algo)
{
    int bs = 0;
    if (!fallback_geom(ggml_type, &bs, nullptr)) return GGUFB200_E_TYPE;
    if (act_dtype != kF16 && act_dtype != kBF16) return GGUFB200_E_DTYPE;
    const int a = algo & GGUFB200_ALGO_MASK;
    if (a != GGUFB200_ALGO_AUTO && a != GGUFB200_ALGO_FUSED_SYNC && a != GGUFB200_ALGO_DEQUANT_MMA) return GGUFB200_E_UNSUPPORTED;
    if (algo & ~(GGUFB200_ALGO_MASK | GGUFB200_FLAG_EXACT_W | GGUFB200_FLAG_W_STABLE | GGUFB200_FLAG_NOSPLIT)) return GGUFB200_E_UNSUPPORTED;
    if (M < 0 || N <= 0 || K <= 0 || K % 8 != 0 || K % bs != 0 || N % 8 != 0 || ldx < K || ldy < N) return GGUFB200_E_SHAPE;
    return GGUFB200_OK;
}

extern "C" {

int ggufb200_version(void) { return GGUFB200_VERSION; }

const char *ggufb200_strerror(int rc)
{
    switch (rc) {
    case GGUFB200_OK: return "ok";
    case GGUFB200_E_TYPE: return "unsupported ggml quantization type (no CPU fallback is provided)";
    case GGUFB200_E_DTYPE: return "dtype code must be 0 (float16), 1 (bfloat16) or 2 (float32)";
    case GGUFB200_E_ALIGN: return "output / activation pointers must be 16-byte aligned";
    case GGUFB200_E_SHAPE: return "bad shape: sizes must be non-negative, K a multiple of the block size (or of 8 with N*K a multiple of a 256-element block), ld >= row length";
    case GGUFB200_E_NULL: return "required pointer is NULL";
    case GGUFB200_E_CUDA: return "CUDA launch failed";
    case GGUFB200_E_WORKSPACE: return "workspace too small (see ggufb200_linear_workspace)";
    case GGUFB200_E_UNSUPPORTED: return "operation not implemented for this type / dtype / shape combination";
    case GGUFB200_E_DEVICE: return "current CUDA device is not sm_90 (H100)";
    }
    return "unknown error";
}

int ggufb200_type_info(int ggml_type, int *block_size, int *type_size)
{
    return type_geom(ggml_type, block_size, type_size) ? GGUFB200_OK : GGUFB200_E_TYPE;
}

int ggufb200_supported(int ggml_type, int op)
{
    if (op == GGUFB200_OP_DEQUANT_FALLBACK || op == GGUFB200_OP_LINEAR_FALLBACK || op == GGUFB200_OP_ROWS_FALLBACK)
        return fallback_geom(ggml_type, nullptr, nullptr) ? 1 : 0;
    if (op == GGUFB200_OP_QUANTIZE) return quantize_supported(ggml_type) ? 1 : 0;
    if (op == GGUFB200_OP_QUANTIZE_K) return quantize_k_supported(ggml_type) ? 1 : 0;
    if (op == GGUFB200_OP_LINEAR_GRAD) return grad_type(ggml_type, nullptr) ? 1 : 0;
    if (!type_geom(ggml_type, nullptr, nullptr)) return 0;
    switch (op) {
    case GGUFB200_OP_DEQUANT: return 1;
    case GGUFB200_OP_ROWS: return 1;
    case GGUFB200_OP_LINEAR: return 1;
    case GGUFB200_OP_LINEAR_MMA: return 1;   // a fused kernel, or dequant + tensor-core GEMM for types / shapes it does not cover
    }
    return 0;
}

int ggufb200_set_tuning(int key, int value)
{
    static const bool allowed = [] {
        const char *e = getenv("GGUFB200_ALLOW_TUNING");
        return e && e[0] == '1';
    }();
    if (!allowed) return GGUFB200_E_UNSUPPORTED;
    if (key == 1) {
        g_dequant_pdl = value ? 1 : 0;
        return GGUFB200_OK;
    }
    if (key == 2) {
        g_gemv2_ctas = value;
        return GGUFB200_OK;
    }
    return GGUFB200_E_UNSUPPORTED;
}

int ggufb200_dequant(int ggml_type, const void *packed, int64_t n_blocks, void *out, int out_dtype, int math_dtype, void *stream)
{
    if (!type_geom(ggml_type, nullptr, nullptr)) return GGUFB200_E_TYPE;
    const bool stable = (math_dtype & GGUFB200_DEQUANT_SRC_STABLE) != 0;
    math_dtype &= ~GGUFB200_DEQUANT_SRC_STABLE;
    if (!dtype_ok(out_dtype) || !dtype_ok(math_dtype)) return GGUFB200_E_DTYPE;
    if (n_blocks < 0) return GGUFB200_E_SHAPE;
    if (n_blocks == 0) return GGUFB200_OK;
    if (!packed || !out) return GGUFB200_E_NULL;
    if (!aligned16(out)) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return dequant_dispatch(ggml_type, packed, n_blocks, out, out_dtype, math_dtype, (cudaStream_t)stream, stable);
}

int ggufb200_dequant_fallback(int ggml_type, const void *packed, int64_t n_blocks, void *out, int out_dtype, int flags, void *stream)
{
    if (!with_fallback_block(ggml_type, false, [](auto) { return true; })) return GGUFB200_E_TYPE;
    if (flags & ~GGUFB200_DEQUANT_SRC_STABLE) return GGUFB200_E_UNSUPPORTED;
    if (!dtype_ok(out_dtype)) return GGUFB200_E_DTYPE;
    if (n_blocks < 0) return GGUFB200_E_SHAPE;
    if (n_blocks == 0) return GGUFB200_OK;
    if (!packed || !out) return GGUFB200_E_NULL;
    if (!aligned16(out)) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return fallback_dispatch(ggml_type, packed, n_blocks, out, out_dtype, (cudaStream_t)stream, (flags & GGUFB200_DEQUANT_SRC_STABLE) != 0);
}

int ggufb200_quantize(int ggml_type, const void *src, int src_dtype, int64_t n_blocks, void *packed, int flags, void *stream)
{
    if (!quantize_supported(ggml_type)) return GGUFB200_E_TYPE;
    if (flags != 0) return GGUFB200_E_UNSUPPORTED;
    if (!dtype_ok(src_dtype)) return GGUFB200_E_DTYPE;
    if (n_blocks < 0) return GGUFB200_E_SHAPE;
    if (n_blocks == 0) return GGUFB200_OK;
    if (!src || !packed) return GGUFB200_E_NULL;
    if (reinterpret_cast<uintptr_t>(src) % (src_dtype == GGUFB200_F32 ? 4 : 2) != 0) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return quantize_dispatch(ggml_type, src, src_dtype, n_blocks, packed, (cudaStream_t)stream);
}

int ggufb200_quantize_k(int ggml_type, const void *src, int src_dtype, int64_t n_blocks, void *packed, int flags, void *stream)
{
    if (!quantize_k_supported(ggml_type)) return GGUFB200_E_TYPE;
    if (flags != 0) return GGUFB200_E_UNSUPPORTED;
    if (!dtype_ok(src_dtype)) return GGUFB200_E_DTYPE;
    if (n_blocks < 0) return GGUFB200_E_SHAPE;
    if (n_blocks == 0) return GGUFB200_OK;
    if (!src || !packed) return GGUFB200_E_NULL;
    if (reinterpret_cast<uintptr_t>(src) % (src_dtype == GGUFB200_F32 ? 4 : 2) != 0) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return quantize_k_dispatch(ggml_type, src, src_dtype, n_blocks, packed, (cudaStream_t)stream);
}

int ggufb200_dequant_kron(int ggml_type, const void *packed, int64_t N, int64_t K, void *out, int out_dtype, int math_dtype,
                          const ggufb200_kron_patch *patches, int n_patches, void *stream)
{
    int bs;
    if (!type_geom(ggml_type, &bs, nullptr)) return GGUFB200_E_TYPE;
    if (ggml_type == T_BF16) return GGUFB200_E_UNSUPPORTED;
    const bool stable = (math_dtype & GGUFB200_DEQUANT_SRC_STABLE) != 0;
    math_dtype &= ~GGUFB200_DEQUANT_SRC_STABLE;
    if (!dtype_ok(out_dtype) || !dtype_ok(math_dtype)) return GGUFB200_E_DTYPE;
    if (N <= 0 || K <= 0 || K % 8 != 0 || N > 0x7fffffffll || K > 0x7fffffffll || (K % bs != 0 && !straddled_rows(bs, N, K)))
        return GGUFB200_E_SHAPE;
    if (n_patches < 0 || n_patches > kKronMaxPatches) return GGUFB200_E_SHAPE;
    if (n_patches > 0 && !patches) return GGUFB200_E_NULL;
    for (int i = 0; i < n_patches; ++i) {
        const ggufb200_kron_patch &p = patches[i];
        const int64_t dim = p.band_dim;
        if (dim < -1 || dim > 1 || p.a1 <= 0 || p.a2 <= 0 || p.b1 <= 0 || p.b2 <= 0) return GGUFB200_E_SHAPE;
        int64_t rows = N, cols = K;
        if (dim >= 0) {
            const int64_t extent = dim == 0 ? N : K;
            if (p.band_start < 0 || p.band_size <= 0 || p.band_start > extent - p.band_size) return GGUFB200_E_SHAPE;
            (dim == 0 ? rows : cols) = p.band_size;
        }
        if (p.a1 > rows || p.b1 > rows || p.a2 > cols || p.b2 > cols || p.a1 * p.b1 != rows || p.a2 * p.b2 != cols) return GGUFB200_E_SHAPE;
        if (!p.A || !p.B) return GGUFB200_E_NULL;
        if ((reinterpret_cast<uintptr_t>(p.A) & 3) || (reinterpret_cast<uintptr_t>(p.B) & 3)) return GGUFB200_E_ALIGN;
    }
    if (!packed || !out) return GGUFB200_E_NULL;
    if (!aligned16(out)) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return dequant_kron_dispatch(ggml_type, packed, N, K, out, out_dtype, math_dtype, patches, n_patches, (cudaStream_t)stream, stable);
}

int ggufb200_dequant_lowrank(int ggml_type, const void *packed, int64_t N, int64_t K, void *out, int out_dtype, int math_dtype,
                             const ggufb200_lowrank_patch *patches, int n_patches, void *stream)
{
    int bs = 0;
    const bool fallback = with_fallback_block(ggml_type, false, [&](auto blk) {
        bs = decltype(blk)::BS;
        return true;
    });
    if (!fallback && !type_geom(ggml_type, &bs, nullptr)) return GGUFB200_E_TYPE;
    if (ggml_type == T_BF16) return GGUFB200_E_UNSUPPORTED;
    math_dtype &= ~GGUFB200_DEQUANT_SRC_STABLE;
    if (!dtype_ok(out_dtype) || !dtype_ok(math_dtype)) return GGUFB200_E_DTYPE;
    // grid: ceil(K / 128) x ceil(N / 64) CTAs
    if (N <= 0 || K <= 0 || K % 32 != 0 || (N * K) % bs != 0 || N > 64ll * 65535 || K > 0x7fffffffll) return GGUFB200_E_SHAPE;
    if (n_patches < 0 || n_patches > kLowrankMaxPatches) return GGUFB200_E_SHAPE;
    if (n_patches > 0 && !patches) return GGUFB200_E_NULL;
    for (int i = 0; i < n_patches; ++i) {
        const ggufb200_lowrank_patch &p = patches[i];
        const bool loha = p.a2 != nullptr;
        if (p.r1 < 1 || p.r1 > GGUFB200_LOWRANK_MAX_RANK || (loha && (p.r2 < 1 || p.r2 > GGUFB200_LOWRANK_MAX_RANK))) return GGUFB200_E_SHAPE;
        if (!p.a1 || !p.b1 || (loha && !p.b2)) return GGUFB200_E_NULL;
        for (const float *f : {p.a1, p.b1, loha ? p.a2 : nullptr, loha ? p.b2 : nullptr})      // LoRA: b2 is not read
            if (reinterpret_cast<uintptr_t>(f) & 3) return GGUFB200_E_ALIGN;
    }
    if (!packed || !out) return GGUFB200_E_NULL;
    if (!aligned16(out)) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return dequant_lowrank_dispatch(ggml_type, packed, N, K, out, out_dtype, math_dtype, patches, n_patches, (cudaStream_t)stream);
}

// a LOWRANK descriptor as ggufb200_dequant_lowrank checks it (0: fine)
static int lowrank_patch_check(const ggufb200_lowrank_patch &p)
{
    const bool loha = p.a2 != nullptr;
    if (p.r1 < 1 || p.r1 > GGUFB200_LOWRANK_MAX_RANK || (loha && (p.r2 < 1 || p.r2 > GGUFB200_LOWRANK_MAX_RANK))) return GGUFB200_E_SHAPE;
    if (!p.a1 || !p.b1 || (loha && !p.b2)) return GGUFB200_E_NULL;
    for (const float *f : {p.a1, p.b1, loha ? p.a2 : nullptr, loha ? p.b2 : nullptr})      // LoRA: b2 is not read
        if (reinterpret_cast<uintptr_t>(f) & 3) return GGUFB200_E_ALIGN;
    return GGUFB200_OK;
}

// the arguments of ggufb200_dequant_patched as it checks them (0: fine; the device is not checked)
static int patched_args_check(int ggml_type, const void *packed, int64_t N, int64_t K, const void *out, int out_dtype, int math_dtype,
                              const ggufb200_weight_patch *patches, int n_patches)
{
    int bs = 0;
    const bool fallback = with_fallback_block(ggml_type, false, [&](auto blk) {
        bs = decltype(blk)::BS;
        return true;
    });
    if (!fallback && !type_geom(ggml_type, &bs, nullptr)) return GGUFB200_E_TYPE;
    if (ggml_type == T_BF16) return GGUFB200_E_UNSUPPORTED;
    math_dtype &= ~GGUFB200_DEQUANT_SRC_STABLE;
    if (!dtype_ok(out_dtype) || !dtype_ok(math_dtype)) return GGUFB200_E_DTYPE;
    // grid: ceil(K / 128) x ceil(N / 64) CTAs, as ggufb200_dequant_lowrank
    if (N <= 0 || K <= 0 || K % 32 != 0 || (N * K) % bs != 0 || N > 64ll * 65535 || K > 0x7fffffffll) return GGUFB200_E_SHAPE;
    if (n_patches < 0 || n_patches > kLowrankMaxPatches) return GGUFB200_E_SHAPE;
    if (n_patches > 0 && !patches) return GGUFB200_E_NULL;
    for (int i = 0; i < n_patches; ++i) {
        const ggufb200_weight_patch &p = patches[i];
        if (p.kind == GGUFB200_PATCH_LOWRANK) {
            if (int rc = lowrank_patch_check(p.lowrank)) return rc;
        } else if (p.kind == GGUFB200_PATCH_KRON) {
            const ggufb200_kron_patch &k = p.kron;
            if (k.band_dim != -1) return GGUFB200_E_UNSUPPORTED;
            if (k.a1 <= 0 || k.a2 <= 0 || k.b1 <= 0 || k.b2 <= 0 || k.a1 > N || k.b1 > N || k.a2 > K || k.b2 > K || k.a1 * k.b1 != N ||
                k.a2 * k.b2 != K)
                return GGUFB200_E_SHAPE;
            if (!k.A || !k.B) return GGUFB200_E_NULL;
            if ((reinterpret_cast<uintptr_t>(k.A) & 3) || (reinterpret_cast<uintptr_t>(k.B) & 3)) return GGUFB200_E_ALIGN;
        } else {
            return GGUFB200_E_UNSUPPORTED;
        }
    }
    if (!packed || !out) return GGUFB200_E_NULL;
    if (!aligned16(out)) return GGUFB200_E_ALIGN;
    return GGUFB200_OK;
}

int ggufb200_dequant_patched(int ggml_type, const void *packed, int64_t N, int64_t K, void *out, int out_dtype, int math_dtype,
                             const ggufb200_weight_patch *patches, int n_patches, void *stream)
{
    if (int rc = patched_args_check(ggml_type, packed, N, K, out, out_dtype, math_dtype, patches, n_patches)) return rc;
    if (int rc = device_check()) return rc;
    return dequant_patched_dispatch(ggml_type, packed, N, K, out, out_dtype, math_dtype & ~GGUFB200_DEQUANT_SRC_STABLE, patches, n_patches,
                                    (cudaStream_t)stream);
}

int ggufb200_dequant_patched_dora(int ggml_type, const void *packed, int64_t N, int64_t K, void *out, int out_dtype, int math_dtype,
                                  const ggufb200_weight_patch *patches, const ggufb200_dora_patch *dora, int n_patches, void *stream)
{
    if (int rc = patched_args_check(ggml_type, packed, N, K, out, out_dtype, math_dtype, patches, n_patches)) return rc;
    if (n_patches > 0 && !dora) return GGUFB200_E_NULL;
    for (int i = 0; i < n_patches; ++i) {
        const ggufb200_dora_patch &d = dora[i];
        if (!d.factor) continue;
        if (d.axis != GGUFB200_DORA_AXIS_OUT && d.axis != GGUFB200_DORA_AXIS_IN) return GGUFB200_E_SHAPE;
        if (d.axis == GGUFB200_DORA_AXIS_IN && (d.group < 1 || K % d.group != 0)) return GGUFB200_E_SHAPE;
        if (reinterpret_cast<uintptr_t>(d.factor) & 3) return GGUFB200_E_ALIGN;
    }
    if (int rc = device_check()) return rc;
    return dequant_patched_dora_dispatch(ggml_type, packed, N, K, out, out_dtype, math_dtype & ~GGUFB200_DEQUANT_SRC_STABLE, patches, dora,
                                         n_patches, (cudaStream_t)stream);
}

int ggufb200_unpack_int(int ggml_type,const void *packed, int64_t n_blocks, int16_t *q, int16_t *sc, int16_t *mn, void *stream)
{
    if (!type_geom(ggml_type, nullptr, nullptr) || ggml_type == T_BF16) return GGUFB200_E_TYPE;
    if (n_blocks < 0) return GGUFB200_E_SHAPE;
    if (n_blocks == 0) return GGUFB200_OK;
    if (!packed) return GGUFB200_E_NULL;
    if (int rc = device_check()) return rc;
    return unpack_dispatch(ggml_type, packed, n_blocks, q, sc, mn, (cudaStream_t)stream);
}

int ggufb200_dequant_rows(int ggml_type, const void *packed, int64_t n_table_rows, int64_t K, const int64_t *rows, int64_t n_rows,
                          void *out, int out_dtype, int math_dtype, void *stream)
{
    int bs, ts;
    if (!type_geom(ggml_type, &bs, &ts)) return GGUFB200_E_TYPE;
    if (!dtype_ok(out_dtype) || !dtype_ok(math_dtype)) return GGUFB200_E_DTYPE;
    if (n_rows < 0 || n_table_rows < 0 || K <= 0 || K % bs != 0 || K % 8 != 0) return GGUFB200_E_SHAPE;
    if (n_rows == 0) return GGUFB200_OK;
    if (!packed || !rows || !out) return GGUFB200_E_NULL;
    if (!aligned16(out)) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return rows_dispatch(ggml_type, packed, n_table_rows, K, (const long long *)rows, n_rows, out, out_dtype, math_dtype,
                         (cudaStream_t)stream);
}

int ggufb200_dequant_rows_fallback(int ggml_type, const void *packed, int64_t n_table_rows, int64_t K, const int64_t *rows, int64_t n_rows,
                                   void *out, int out_dtype, void *stream)
{
    int bs;
    if (!fallback_geom(ggml_type, &bs, nullptr)) return GGUFB200_E_TYPE;
    if (!dtype_ok(out_dtype)) return GGUFB200_E_DTYPE;
    if (n_rows < 0 || n_table_rows < 0 || K <= 0 || K % bs != 0 || K % 8 != 0) return GGUFB200_E_SHAPE;
    if (n_rows == 0) return GGUFB200_OK;
    if (!packed || !rows || !out) return GGUFB200_E_NULL;
    if (!aligned16(out)) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return rows_fallback_dispatch(ggml_type, packed, n_table_rows, K, (const long long *)rows, n_rows, out, out_dtype, (cudaStream_t)stream);
}

size_t ggufb200_linear_fallback_workspace(int ggml_type, int64_t M, int64_t N, int64_t K, int act_dtype, int algo)
{
    if (fallback_linear_args(ggml_type, N, K, M, K, N, act_dtype, algo) != GGUFB200_OK || M <= 0) return 0;
    return pick_fallback_route(ggml_type, nullptr, M, N, K, algo).ws;
}

int ggufb200_linear_fallback_route(int ggml_type, int64_t M, int64_t N, int64_t K, int act_dtype, int algo)
{
    if (int rc = fallback_linear_args(ggml_type, N, K, M, K, N, act_dtype, algo)) return rc;
    if (M == 0) return GGUFB200_OK;          // the call returns OK without a route: nothing to compute
    return pick_fallback_route(ggml_type, nullptr, M, N, K, algo).algo;
}

int ggufb200_linear_fallback(int ggml_type, const void *W_packed, int64_t N, int64_t K, const void *X, int64_t M, int64_t ldx, int act_dtype,
                             const void *bias, int bias_dtype, void *Y, int64_t ldy, void *workspace, size_t workspace_bytes, int algo,
                             void *stream)
{
    if (int rc = fallback_linear_args(ggml_type, N, K, M, ldx, ldy, act_dtype, algo)) return rc;
    if (bias && !dtype_ok(bias_dtype)) return GGUFB200_E_DTYPE;
    if (M == 0) return GGUFB200_OK;
    if (!W_packed || !X || !Y) return GGUFB200_E_NULL;
    if (!aligned16(X) || (ldx % 8) != 0 || !aligned16(Y) || (ldy % 8) != 0) return GGUFB200_E_ALIGN;
    const size_t ws_avail = (workspace && aligned16(workspace)) ? workspace_bytes : 0;
    const size_t dense = (size_t)N * (size_t)K * 2;
    int bs = 1, a_blk = 1;
    fallback_geom(ggml_type, &bs, &a_blk);
    // a byte-offset view below the type's block alignment: only the standalone dequant reads it (and needs its workspace)
    if (reinterpret_cast<uintptr_t>(W_packed) % a_blk != 0 && ws_avail < dense) return GGUFB200_E_ALIGN;
    const Route r = pick_fallback_route(ggml_type, W_packed, M, N, K, algo);
    if (workspace && !aligned16(workspace) && r.ws) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (r.algo == GGUFB200_ALGO_FUSED_SYNC)
        return fallback_linear(ggml_type, W_packed, N, K, X, M, ldx, act_dtype, bias, bias_dtype, Y, ldy, workspace, ws_avail,
                               (algo & GGUFB200_FLAG_NOSPLIT) != 0, st);
    if (ws_avail < dense) return GGUFB200_E_WORKSPACE;
    const int rc = fallback_dispatch(ggml_type, W_packed, N * K / bs, workspace, act_dtype, st, (algo & GGUFB200_FLAG_W_STABLE) != 0);
    if (rc != GGUFB200_OK) return rc;
    return dense_gemm(workspace, N, K, K, X, M, ldx, act_dtype, bias, bias_dtype, Y, ldy, st);
}

size_t ggufb200_linear_workspace_ex(int ggml_type, int64_t M, int64_t N, int64_t K, int act_dtype, int math_dtype, int algo)
{
    int bs;
    if (!type_geom(ggml_type, &bs, nullptr) || N <= 0 || K <= 0 || M <= 0) return 0;
    return pick_route(ggml_type, nullptr, M, N, K, act_dtype, math_dtype, algo, linear_options(algo, straddled_rows(bs, N, K)), (size_t)-1).ws;
}

size_t ggufb200_linear_workspace(int ggml_type, int64_t M, int64_t N, int64_t K, int act_dtype, int algo)
{
    return ggufb200_linear_workspace_ex(ggml_type, M, N, K, act_dtype, kF16, algo);
}

static int linear_impl(int ggml_type, const void *W_packed, const void *W_spans, int64_t N, int64_t K, const void *X, int64_t M, int64_t ldx,
                       int act_dtype, int math_dtype, const void *bias, int bias_dtype, void *Y, int64_t ldy, void *workspace,
                       size_t workspace_bytes, int algo, void *stream, const LoraOperands *lora = nullptr, const float *scale = nullptr)
{
    int bs, ts;
    if (!type_geom(ggml_type, &bs, &ts)) return GGUFB200_E_TYPE;
    if (act_dtype != kF16 && act_dtype != kBF16) return GGUFB200_E_DTYPE;
    if (!dtype_ok(math_dtype) || (bias && !dtype_ok(bias_dtype))) return GGUFB200_E_DTYPE;
    if (M < 0 || N <= 0 || K <= 0 || K % 8 != 0 || ldx < K || ldy < N) return GGUFB200_E_SHAPE;
    // rows are whole blocks, or a straddled weight: the flat block stream of an [N, K] tensor (internal.h)
    const bool straddled = straddled_rows(bs, N, K);
    if (K % bs != 0 && !straddled) return GGUFB200_E_SHAPE;
    if (M == 0) return GGUFB200_OK;
    if (!W_packed || !X || !Y) return GGUFB200_E_NULL;
    const int flags = algo & ~GGUFB200_ALGO_MASK;
    const LinearOptions opt = linear_options(flags, straddled);
    const bool w_ok = aligned16(W_packed);
    const size_t dense = (size_t)N * (size_t)K * 2;
    const size_t ws_avail = (workspace && aligned16(workspace)) ? workspace_bytes : 0;
    // The fused producers read the packed rows with the per-format natural alignment (up to 16 bytes).  A packed tensor
    // that does not start on a 16-byte boundary (never produced by torch allocations, only by byte-offset views) is
    // always routed through the standalone dequant kernel, which stages any alignment, plus the dense GEMM.
    if (!w_ok) {
        if (ws_avail < dense) return GGUFB200_E_ALIGN;
        algo = GGUFB200_ALGO_DEQUANT_MMA | flags;
    }
    if (W_spans && !aligned16(W_spans)) return GGUFB200_E_ALIGN;
    const Route r = pick_route(ggml_type, W_packed, M, N, K, act_dtype, math_dtype, algo, opt, ws_avail, W_spans != nullptr);
    // the GEMVs and FUSED_MMA index whole rows of blocks: a straddled weight runs on FUSED_TMEM or dequant + GEMM only
    if (straddled && r.algo != GGUFB200_ALGO_FUSED_TMEM && r.algo != GGUFB200_ALGO_DEQUANT_MMA) return GGUFB200_E_UNSUPPORTED;
    // the small-M kernel stores per element: it only needs 2-byte aligned Y rows; every other route moves 16-byte vectors
    const bool vec_y = r.algo != GGUFB200_ALGO_GEMV && r.algo != GGUFB200_ALGO_GEMV_FAST;
    if (!aligned16(X) || (ldx % 8) != 0) return GGUFB200_E_ALIGN;
    if (vec_y && (!aligned16(Y) || (ldy % 8) != 0)) return GGUFB200_E_ALIGN;
    if (workspace && !aligned16(workspace) && r.ws) return GGUFB200_E_ALIGN;
    if (lora) {     // the rank-r update rides as J extra k-blocks of the FUSED_TMEM kernel: no other route can carry it
        if (lora->kblocks < 1 || lora->kblocks > kLoraMaxKblocks) return GGUFB200_E_SHAPE;
        if (r.algo != GGUFB200_ALGO_FUSED_TMEM) return GGUFB200_E_UNSUPPORTED;
        if (!lora->T || !lora->U) return GGUFB200_E_NULL;
        const long long width = 64ll * lora->kblocks;
        if (!aligned16(lora->T) || !aligned16(lora->U) || lora->ldt < width || (lora->ldt % 8) != 0 || lora->ldu < width || (lora->ldu % 8) != 0 ||
            (reinterpret_cast<uintptr_t>(lora->tiles) & 3))
            return GGUFB200_E_ALIGN;
    }
    if (scale && !aligned16(scale)) return GGUFB200_E_ALIGN;     // only the LoRA entry point passes one: FUSED_TMEM
    if (int rc = device_check()) return rc;
    cudaStream_t st = (cudaStream_t)stream;

    switch (r.algo) {
    case GGUFB200_ALGO_GEMV:
        return gemv_dispatch(ggml_type, W_packed, N, K, X, M, ldx, act_dtype, math_dtype, bias, bias_dtype, Y, ldy, st);
    case GGUFB200_ALGO_GEMV_FAST:
        if (math_dtype != kF16 || (flags & GGUFB200_FLAG_EXACT_W)) return GGUFB200_E_UNSUPPORTED;
        return gemv2_dispatch(ggml_type, W_packed, N, K, X, M, ldx, act_dtype, bias, bias_dtype, Y, ldy, st, (flags & GGUFB200_FLAG_W_STABLE) != 0);
    case GGUFB200_ALGO_FUSED_MMA:
        if (!fused_type(ggml_type) || math_dtype != kF16) return GGUFB200_E_UNSUPPORTED;
        return fused_mma_linear(ggml_type, W_packed, N, K, X, M, ldx, act_dtype, bias, bias_dtype, Y, ldy, workspace, ws_avail, opt, st);
    case GGUFB200_ALGO_FUSED_TMEM: {
        if (!fused_type(ggml_type) || math_dtype != kF16) return GGUFB200_E_UNSUPPORTED;
        long long span_stride = 0;
        if (W_spans) repack_bytes(ggml_type, N, K, nullptr, &span_stride);
        return fused_tmem_linear(ggml_type, W_packed, W_spans, span_stride, N, K, X, M, ldx, act_dtype, bias, bias_dtype, Y, ldy, workspace,
                                 ws_avail, opt, lora ? *lora : LoraOperands{}, st, scale);
    }
    case GGUFB200_ALGO_DEQUANT_MMA: {
        if (ws_avail < dense) return GGUFB200_E_WORKSPACE;
        int rc = dequant_dispatch(ggml_type, W_packed, N * K / bs, workspace, act_dtype, math_dtype, st, (flags & GGUFB200_FLAG_W_STABLE) != 0);
        if (rc != GGUFB200_OK) return rc;
        return dense_gemm(workspace, N, K, K, X, M, ldx, act_dtype, bias, bias_dtype, Y, ldy, st);
    }
    }
    return GGUFB200_E_UNSUPPORTED;
}

int ggufb200_linear(int ggml_type, const void *W_packed, int64_t N, int64_t K, const void *X, int64_t M, int64_t ldx, int act_dtype,
                    int math_dtype, const void *bias, int bias_dtype, void *Y, int64_t ldy, void *workspace, size_t workspace_bytes,
                    int algo, void *stream)
{
    return linear_impl(ggml_type, W_packed, nullptr, N, K, X, M, ldx, act_dtype, math_dtype, bias, bias_dtype, Y, ldy, workspace, workspace_bytes,
                       algo, stream);
}

int ggufb200_linear_spans(int ggml_type, const void *W_packed, const void *W_spans, int64_t N, int64_t K, const void *X, int64_t M, int64_t ldx,
                          int act_dtype, int math_dtype, const void *bias, int bias_dtype, void *Y, int64_t ldy, void *workspace,
                          size_t workspace_bytes, int algo, void *stream)
{
    return linear_impl(ggml_type, W_packed, W_spans, N, K, X, M, ldx, act_dtype, math_dtype, bias, bias_dtype, Y, ldy, workspace, workspace_bytes,
                       algo, stream);
}

int ggufb200_linear_lora(int ggml_type, const void *W_packed, const void *W_spans, int64_t N, int64_t K, const void *X, int64_t M, int64_t ldx,
                         int act_dtype, const void *bias, int bias_dtype, const void *T, int64_t ldt, const void *U, void *Y, int64_t ldy,
                         void *workspace, size_t workspace_bytes, int algo, void *stream)
{
    return ggufb200_linear_lora_ex(ggml_type, W_packed, W_spans, N, K, X, M, ldx, act_dtype, bias, bias_dtype, T, ldt, U, 64, 1, nullptr, Y, ldy,
                                   workspace, workspace_bytes, algo, stream);
}

int ggufb200_linear_lora_ex(int ggml_type, const void *W_packed, const void *W_spans, int64_t N, int64_t K, const void *X, int64_t M, int64_t ldx,
                            int act_dtype, const void *bias, int bias_dtype, const void *T, int64_t ldt, const void *U, int64_t ldu,
                            int lora_kblocks, const int32_t *tile_kblocks, void *Y, int64_t ldy, void *workspace, size_t workspace_bytes, int algo,
                            void *stream)
{
    return ggufb200_linear_lora_scaled(ggml_type, W_packed, W_spans, N, K, X, M, ldx, act_dtype, bias, bias_dtype, T, ldt, U, ldu, lora_kblocks,
                                       tile_kblocks, nullptr, Y, ldy, workspace, workspace_bytes, algo, stream);
}

int ggufb200_linear_lora_scaled(int ggml_type, const void *W_packed, const void *W_spans, int64_t N, int64_t K, const void *X, int64_t M,
                                int64_t ldx, int act_dtype, const void *bias, int bias_dtype, const void *T, int64_t ldt, const void *U,
                                int64_t ldu, int lora_kblocks, const int32_t *tile_kblocks, const float *feature_scale, void *Y, int64_t ldy,
                                void *workspace, size_t workspace_bytes, int algo, void *stream)
{
    const LoraOperands lora{T, ldt, U, ldu, lora_kblocks, tile_kblocks};
    return linear_impl(ggml_type, W_packed, W_spans, N, K, X, M, ldx, act_dtype, kF16, bias, bias_dtype, Y, ldy, workspace, workspace_bytes, algo,
                       stream, &lora, feature_scale);
}

size_t ggufb200_repack_bytes(int ggml_type, int64_t N, int64_t K)
{
    int bs;
    if (!type_geom(ggml_type, &bs, nullptr) || N <= 0 || K <= 0 || (K % bs != 0 && !straddled_rows(bs, N, K))) return 0;
    return repack_bytes(ggml_type, N, K, nullptr, nullptr);
}

int ggufb200_repack(int ggml_type, const void *W_packed, int64_t N, int64_t K, void *out, void *stream)
{
    int bs;
    if (!type_geom(ggml_type, &bs, nullptr) || ggml_type == T_BF16) return GGUFB200_E_TYPE;
    if (N <= 0 || K <= 0 || (K % bs != 0 && !straddled_rows(bs, N, K))) return GGUFB200_E_SHAPE;
    if (!W_packed || !out) return GGUFB200_E_NULL;
    if (!aligned16(out) || (reinterpret_cast<uintptr_t>(W_packed) & 1)) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return repack_dispatch(ggml_type, W_packed, N, K, out, (cudaStream_t)stream);
}

int ggufb200_linear_plan(int ggml_type, int64_t M, int64_t N, int64_t K, size_t workspace_bytes, int algo, int *tile_rows, int *k_ranges,
                         int *kblocks_per_range, int *ctas)
{
    int bs;
    if (!type_geom(ggml_type, &bs, nullptr)) return GGUFB200_E_TYPE;
    if (!tile_rows || !k_ranges || !kblocks_per_range || !ctas) return GGUFB200_E_NULL;
    if (M <= 0 || N <= 0 || K <= 0 || K % 64 != 0 || N % 8 != 0) return GGUFB200_E_SHAPE;
    if (!fused_type(ggml_type)) return GGUFB200_E_UNSUPPORTED;
    const LinearOptions opt = linear_options(algo, straddled_rows(bs, N, K));
    if ((algo & GGUFB200_ALGO_MASK) == GGUFB200_ALGO_FUSED_TMEM) {
        int spans = 1;
        fused_tmem_plan(M, N, K, workspace_bytes, opt, tile_rows, k_ranges, &spans, ctas);
        *kblocks_per_range = 4 * spans;
        return GGUFB200_OK;
    }
    if ((algo & GGUFB200_ALGO_MASK) != GGUFB200_ALGO_FUSED_MMA) return GGUFB200_E_UNSUPPORTED;
    fused_mma_plan(M, N, K, workspace_bytes, opt, tile_rows, k_ranges, kblocks_per_range, ctas);
    return GGUFB200_OK;
}

int ggufb200_gemm(const void *W, int64_t N, int64_t K, int64_t ldw, const void *X, int64_t M, int64_t ldx, int act_dtype,
                  const void *bias, int bias_dtype, void *Y, int64_t ldy, void *stream)
{
    return ggufb200_gemm_scaled(W, N, K, ldw, X, M, ldx, act_dtype, bias, bias_dtype, nullptr, Y, ldy, stream);
}

int ggufb200_gemm_scaled(const void *W, int64_t N, int64_t K, int64_t ldw, const void *X, int64_t M, int64_t ldx, int act_dtype,
                         const void *bias, int bias_dtype, const float *feature_scale, void *Y, int64_t ldy, void *stream)
{
    if (act_dtype != kF16 && act_dtype != kBF16) return GGUFB200_E_DTYPE;
    if (bias && !dtype_ok(bias_dtype)) return GGUFB200_E_DTYPE;
    if (M < 0 || N <= 0 || K <= 0 || K % 8 != 0 || ldw < K || ldx < K || ldy < N) return GGUFB200_E_SHAPE;
    if (M == 0) return GGUFB200_OK;
    if (!W || !X || !Y) return GGUFB200_E_NULL;
    if (!aligned16(W) || !aligned16(X) || !aligned16(Y) || (ldw % 8) || (ldx % 8) || (ldy % 8)) return GGUFB200_E_ALIGN;
    if (feature_scale && !aligned16(feature_scale)) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return dense_gemm(W, N, K, ldw, X, M, ldx, act_dtype, bias, bias_dtype, Y, ldy, (cudaStream_t)stream, feature_scale);
}

// BF16 weight, bf16 activations: W's bytes are already the operand
static bool grad_reads_in_place(int ggml_type, int act_dtype) { return ggml_type == T_BF16 && act_dtype == kBF16; }

size_t ggufb200_linear_grad_input_workspace(int ggml_type, int64_t N, int64_t K, int act_dtype)
{
    if (!grad_type(ggml_type, nullptr) || N <= 0 || K <= 0 || grad_reads_in_place(ggml_type, act_dtype)) return 0;
    return (size_t)N * (size_t)K * 2;
}

int ggufb200_linear_grad_input(int ggml_type, const void *W_packed, int64_t N, int64_t K, const void *dY, int64_t M, int64_t ldy, int act_dtype,
                               int math_dtype, void *dX, int64_t ldx, void *workspace, size_t workspace_bytes, int flags, void *stream)
{
    int bs = 0;
    if (!grad_type(ggml_type, &bs)) return GGUFB200_E_TYPE;
    if (act_dtype != kF16 && act_dtype != kBF16) return GGUFB200_E_DTYPE;
    if (!dtype_ok(math_dtype)) return GGUFB200_E_DTYPE;
    if (flags & ~GGUFB200_FLAG_W_STABLE) return GGUFB200_E_UNSUPPORTED;
    const bool fallback = !type_geom(ggml_type, nullptr, nullptr);
    if (M < 0 || N <= 0 || K <= 0 || K % 8 != 0 || ldy < N || ldx < K || (N * K) % bs != 0) return GGUFB200_E_SHAPE;
    if (!fallback && K % bs != 0 && !straddled_rows(bs, N, K)) return GGUFB200_E_SHAPE;
    if (M == 0) return GGUFB200_OK;
    if (!W_packed || !dY || !dX) return GGUFB200_E_NULL;
    if (!aligned16(dY) || !aligned16(dX) || (ldy % 8) || (ldx % 8)) return GGUFB200_E_ALIGN;
    const bool in_place = grad_reads_in_place(ggml_type, act_dtype);
    if (in_place && !aligned16(W_packed)) return GGUFB200_E_ALIGN;
    const size_t dense = in_place ? 0 : (size_t)N * (size_t)K * 2;
    if (dense && (!workspace || workspace_bytes < dense)) return GGUFB200_E_WORKSPACE;
    if (dense && !aligned16(workspace)) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    // An autograd backward runs on a worker thread that may have no current context yet; the first launch of a kernel instance
    // raises its shared-memory limit (cudaFuncSetAttribute), which fails there.  cudaSetDevice binds the primary context.
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaSetDevice(dev) != cudaSuccess) {
        cudaGetLastError();
        return GGUFB200_E_CUDA;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const bool stable = (flags & GGUFB200_FLAG_W_STABLE) != 0;
    const void *W = W_packed;
    if (!in_place) {
        const long long n_blocks = N * K / bs;
        const int rc = fallback ? fallback_dispatch(ggml_type, W_packed, n_blocks, workspace, act_dtype, st, stable)
                                : dequant_dispatch(ggml_type, W_packed, n_blocks, workspace, act_dtype, math_dtype, st, stable);
        if (rc != GGUFB200_OK) return rc;
        W = workspace;
    }
    return dense_gemm_nn(W, N, K, K, dY, M, ldy, act_dtype, dX, ldx, st);
}

int ggufb200_scale_columns(const void *X, int64_t M, int64_t K, int64_t ldx, int act_dtype, const float *col_scale, void *Y, int64_t ldy,
                           void *stream)
{
    if (act_dtype != kF16 && act_dtype != kBF16) return GGUFB200_E_DTYPE;
    if (M < 0 || K <= 0 || K % 8 != 0 || ldx < K || ldy < K) return GGUFB200_E_SHAPE;
    if (M == 0) return GGUFB200_OK;
    if (!X || !col_scale || !Y) return GGUFB200_E_NULL;
    if (!aligned16(X) || !aligned16(Y) || !aligned16(col_scale) || (ldx % 8) || (ldy % 8)) return GGUFB200_E_ALIGN;
    if (int rc = device_check()) return rc;
    return scale_columns_dispatch(X, M, K, ldx, act_dtype, col_scale, Y, ldy, (cudaStream_t)stream);
}

}  // extern "C"
