/*
 * ggufb200.h -- C ABI of libggufb200.so: H100 (sm_90a) GGUF block dequant and the
 * Linear that consumes the dequantised weight.
 *
 * This is the drop-in boundary for the hot path of city96/ComfyUI-GGUF.  The
 * reference has no native code, so each entry point names the PYTHON function it
 * replaces (reference file:line); INTEGRATION.md shows the ctypes binding a
 * maintainer of the reference would add.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer owned by the
 *     caller (PyTorch); the library never allocates, frees or retains device memory
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream)
 *   - all calls are asynchronous on `stream` and re-entrant; routing depends only on the arguments of the call
 *     (the library keeps no mutable routing state; ggufb200_set_tuning() is a benchmark-only switch that is refused
 *     unless the process opted in with GGUFB200_ALLOW_TUNING=1)
 *   - the device code is sm_90a only: calls that would launch a kernel return GGUFB200_E_DEVICE on any other GPU
 *   - return value: 0 = GGUFB200_OK, negative = error (ggufb200_strerror()); no C++
 *     exception crosses the boundary
 *   - ggml_type uses gguf-py's GGMLQuantizationType integer values
 *     (Q4_0=2 Q4_1=3 Q5_0=6 Q5_1=7 Q8_0=8 Q2_K=10 Q3_K=11 Q4_K=12 Q5_K=13 Q6_K=14
 *      IQ4_NL=20 IQ4_XS=23 BF16=30), i.e. the keys of dequant.py:287-301
 *   - dtype codes: 0 = float16, 1 = bfloat16, 2 = float32
 */
#ifndef GGUFB200_H
#define GGUFB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GGUFB200_VERSION 200 /* major*10000 + minor*100 + patch */

/* error codes */
#define GGUFB200_OK 0
#define GGUFB200_E_TYPE (-1)      /* ggml_type not in dequant.py:287-301 */
#define GGUFB200_E_DTYPE (-2)     /* dtype code out of range */
#define GGUFB200_E_ALIGN (-3)     /* output / activation pointer not 16-byte aligned */
#define GGUFB200_E_SHAPE (-4)     /* K not a multiple of the block size (nor a straddled weight), negative size, ld too small ... */
#define GGUFB200_E_NULL (-5)      /* required pointer is NULL */
#define GGUFB200_E_CUDA (-6)      /* a CUDA call failed (cudaGetLastError preserved for the caller) */
#define GGUFB200_E_WORKSPACE (-7) /* workspace smaller than ggufb200_linear_workspace() */
#define GGUFB200_E_UNSUPPORTED (-8) /* op / dtype combination not implemented for this type */
#define GGUFB200_E_DEVICE (-9)    /* current device is not sm_90 */

/* dtype codes */
#define GGUFB200_F16 0
#define GGUFB200_BF16 1
#define GGUFB200_F32 2

/* op codes for ggufb200_supported() */
#define GGUFB200_OP_DEQUANT 0
#define GGUFB200_OP_LINEAR 1
#define GGUFB200_OP_ROWS 2
#define GGUFB200_OP_LINEAR_MMA 3 /* large-M tensor-core path (fused or dequant+GEMM) available for this type */
#define GGUFB200_OP_DEQUANT_FALLBACK 4 /* ggufb200_dequant_fallback() serves this type */
#define GGUFB200_OP_QUANTIZE 5 /* ggufb200_quantize() produces this type */
#define GGUFB200_OP_LINEAR_GRAD 6 /* ggufb200_linear_grad_input() serves this type */
#define GGUFB200_OP_LINEAR_FALLBACK 7 /* ggufb200_linear_fallback() serves this type */
#define GGUFB200_OP_ROWS_FALLBACK 8 /* ggufb200_dequant_rows_fallback() serves this type */
#define GGUFB200_OP_QUANTIZE_K 9 /* ggufb200_quantize_k() produces this type */

/* algorithm selector for ggufb200_linear(): one GGUFB200_ALGO_* value, optionally OR-ed with GGUFB200_FLAG_* bits */
#define GGUFB200_ALGO_AUTO 0
#define GGUFB200_ALGO_GEMV 1        /* M <= 8: fused dequant + mma.sync dot products, W bit-identical to the reference */
#define GGUFB200_ALGO_FUSED_MMA 2   /* fused dequant -> shared memory -> wgmma (W bit-identical to the reference) */
#define GGUFB200_ALGO_DEQUANT_MMA 3 /* dequant into the caller's workspace, then the wgmma GEMM on it (W bit-identical) */
#define GGUFB200_ALGO_FUSED_TMEM 4  /* fused dequant -> shared memory -> wgmma with token tiles sized to M, any M (what AUTO picks for M > 8) */
#define GGUFB200_ALGO_GEMV_FAST 5   /* M <= 8, Q4_K / Q5_K: integer patterns on mma.sync, sub-block scales applied to the partial sums
                                       (W is never formed or rounded: the `fast` contract; AUTO picks it only without EXACT_W) */
#define GGUFB200_ALGO_FUSED_SYNC 6  /* ggufb200_linear_fallback only: the weight decoded in registers, mma.sync over up to 64 tokens */
#define GGUFB200_ALGO_MASK 0xFF

/* Per-call switches (no process-wide state):
 *   EXACT_W    the weight operand must be bit-identical to what the reference hands to F.linear (dequant.py float sequence with
 *              per-op rounding, then the cast to the activation dtype): FUSED_TMEM then runs its reference-sequence
 *              producers (same speed at large M: the kernel is tensor-pipe bound), every other route is exact anyway.
 *              Without it FUSED_TMEM uses the `fast` producers, whose contract is: integer unpack bit-exact; sub-block scale
 *              products as the reference; for Q4_K / Q5_K the per-element float step is ONE fused multiply-add in fp16 (the
 *              correctly rounded value of the step) instead of multiply + subtract; then the reference's cast to the
 *              activation dtype.  Result as close to the exact product as the reference's, within 1e-3 (fp16) / 8e-3
 *              (bf16, = the same bound in bf16 ulps) of the reference's.
 *   GENERIC    FUSED_TMEM: functor producers that follow the reference's rounding sequence op for op (every format; also exact)
 *   TILE384    FUSED_TMEM: force 384-token items (two 192-token CTAs per 128 features)
 *   TILE192    FUSED_TMEM: force 192-token items; default: a cost model picks
 *   NOSPLIT    FUSED_MMA / FUSED_TMEM: never cut K into ranges
 *   UNSTAGED   accepted for compatibility, no effect: FUSED_MMA producers always read the packed rows from global memory */
#define GGUFB200_FLAG_EXACT_W 0x100
#define GGUFB200_FLAG_GENERIC 0x200
#define GGUFB200_FLAG_TILE384 0x400
#define GGUFB200_FLAG_NOSPLIT 0x800
#define GGUFB200_FLAG_UNSTAGED 0x1000
#define GGUFB200_FLAG_TILE192 0x2000 /* FUSED_TMEM: force 192-token items (double-buffered accumulators); default: cost model */
/*   W_STABLE   the caller promises that no kernel still in flight on `stream` writes W_packed (model weights: written once at
 *              load time).  The kernels are launched with programmatic stream serialization; with the promise GEMV_FAST starts
 *              streaming the packed weight into its shared-memory ring while the preceding kernel drains (the activations, the
 *              bias and Y are only touched after that kernel has completed), and DEQUANT_MMA passes
 *              GGUFB200_DEQUANT_SRC_STABLE to its dequant launch.  A kernel that does not signal programmatic completion early
 *              (every torch / cuBLAS kernel) is complete before its successor starts, so the promise only excludes producers
 *              of the packed bytes that execute griddepcontrol.launch_dependents before their last write. */
#define GGUFB200_FLAG_W_STABLE 0x4000

int ggufb200_version(void);
const char *ggufb200_strerror(int rc);

/* Block geometry: replaces gguf.GGML_QUANT_SIZES[qtype] as used at dequant.py:34. */
int ggufb200_type_info(int ggml_type, int *block_size, int *type_size);

/* 1 if (ggml_type, op) is implemented, else 0.  For ops 0-3 mirrors `qtype in dequantize_functions`
 * (dequant.py:21, 287-301).  The types of the reference's numpy fallback (dequant.py:24-28) are served on the GPU by
 * ggufb200_dequant_fallback() instead (op GGUFB200_OP_DEQUANT_FALLBACK); nothing is computed on the CPU. */
int ggufb200_supported(int ggml_type, int op);

/*
 * Standalone dequant.  Replaces dequant.py:30-44 `dequantize()` + the per-type
 * `dequantize_blocks_*` (dequant.py:61-285) + the final `.to(dtype)` (dequant.py:23).
 *   packed     n_blocks * type_size bytes, block b covers out[b*block_size .. +block_size)
 *   out        n_blocks * block_size elements of out_dtype, 16-byte aligned
 *   math_dtype dtype the float ops run in and round to after every op: 0 (fp16) is the
 *              reference default (`dequant_dtype=None`), the activation dtype reproduces
 *              `dequant_dtype="target"`, 2 an explicit float32.  Results are bit-identical
 *              to the reference for every (math_dtype, out_dtype) pair.
 *              Optionally OR-ed with GGUFB200_DEQUANT_SRC_STABLE: the caller promises that no kernel still in flight on
 *              `stream` writes the packed bytes (model weights: written once at load time).  The kernel is launched with
 *              programmatic stream serialization; with the promise it fetches packed tiles and unpacks the first of them
 *              into shared memory while the preceding kernel drains, and only its stores wait for that kernel (whatever
 *              the preceding kernels read or wrote in `out` is complete before the first byte lands).  Same results.
 */
#define GGUFB200_DEQUANT_SRC_STABLE 0x100
int ggufb200_dequant(int ggml_type, const void *packed, int64_t n_blocks, void *out, int out_dtype,
                     int math_dtype, void *stream);

/*
 * Standalone dequant of the types the reference serves only through gguf-py's numpy fallback (dequant.py:24-28,
 * `torch.from_numpy(gguf.quants.dequantize(bytes, qtype)).to(dtype)`): IQ2_XXS=16 IQ2_XS=17 IQ3_XXS=18 IQ1_S=19 IQ3_S=21
 * IQ2_S=22 IQ1_M=29 TQ1_0=34 TQ2_0=35 MXFP4=39 NVFP4=40.  Every element is gguf-py's `dequantize_blocks` value, computed in
 * fp32 with its operation order, then rounded once (to nearest even) to out_dtype: bit-identical to the reference (NaN
 * payloads aside).  There is no math dtype: the reference ignores dequant_dtype on this branch.
 *   packed     n_blocks * type_size bytes, any alignment
 *   out        n_blocks * block_size elements of out_dtype, 16-byte aligned
 *   flags      0 or GGUFB200_DEQUANT_SRC_STABLE (as in ggufb200_dequant); any other bit: GGUFB200_E_UNSUPPORTED
 * Any other ggml_type, including the types of ggufb200_dequant, returns GGUFB200_E_TYPE; ggufb200_supported(t,
 * GGUFB200_OP_DEQUANT_FALLBACK) lists exactly these eleven.  ggufb200_type_info, GGUFB200_OP_DEQUANT, the Linear entry points
 * and ggufb200_dequant_rows keep the reference's table (dequant.py:287-301) only; these types have their own Linear
 * (ggufb200_linear_fallback) and row gather (ggufb200_dequant_rows_fallback).
 */
int ggufb200_dequant_fallback(int ggml_type, const void *packed, int64_t n_blocks, void *out, int out_dtype, int flags,
                              void *stream);

/*
 * Standalone dequant of an [N, K] weight with LoKr (LyCORIS Kronecker) patches applied.  Replaces, for a LoKr-patched weight,
 * the reference's dequantise + comfy.lora.calculate_weight: every element of `out` is the reference's patched weight
 *     W'[n, k] = out( out(W[n, k]) + out( fp32(scale) * fp32(A[i1, i2] * B[j1, j2]) ) )
 * with (i1, j1) = divmod(n - row0, b1) and (i2, j2) = divmod(k - col0, b2) inside the patch's band, out() = rounding to out_dtype
 * and the sum formed in fp32; elements outside a band are left as they are.  Patches are applied in list order, one rounding
 * each, as `weight += ((strength * alpha) * kron(w1, w2)).to(dtype)` does per patch entry.  W is the ggufb200_dequant value
 * in math_dtype cast to out_dtype (math_dtype may carry GGUFB200_DEQUANT_SRC_STABLE).
 *   packed     the rows of W: whole blocks per row, or a straddled weight (see ggufb200_linear); K % 8 == 0; not BF16
 *   out        N*K elements of out_dtype, 16-byte aligned
 *   patches    host array of n_patches (0 .. 8) descriptors; A and B are DEVICE pointers to row-major fp32 matrices
 * Band: band_dim -1 = the whole weight (row0 = col0 = 0), 0 = output rows band_start .. band_start + band_size, 1 = input
 * features band_start .. band_start + band_size (ComfyUI's patch `offset`).  a1*b1 and a2*b2 must equal the band's rows and
 * columns (GGUFB200_E_SHAPE).  A / B must be 4-byte aligned (GGUFB200_E_ALIGN).
 */
typedef struct ggufb200_kron_patch {
    const float *A;        /* [a1, a2]: LoKr w1 (or w1_a @ w1_b) */
    const float *B;        /* [b1, b2]: LoKr w2 (or w2_a @ w2_b) */
    int64_t a1, a2, b1, b2;
    int32_t band_dim;      /* -1, 0 or 1 */
    float scale;           /* strength * alpha */
    int64_t band_start, band_size;
} ggufb200_kron_patch;
int ggufb200_dequant_kron(int ggml_type, const void *packed, int64_t N, int64_t K, void *out, int out_dtype, int math_dtype,
                          const ggufb200_kron_patch *patches, int n_patches, void *stream);

/*
 * Standalone dequant of an [N, K] weight with LoRA / LoCon and LoHa patches applied, in one launch.  Replaces, for a patched
 * Conv2d (N = Cout, K = Cin * kh * kw), the reference's dequantise + comfy.lora.calculate_weight without its fp32 [N, K] delta.
 * Every element of `out` is, patch by patch in list order,
 *     W'[n, k] = out( W[n, k] + out( fp32(scale) * d[n, k] ) )
 *     LoRA  d = sum_j a1[n, j] * b1[j, k]                                   (fp32, j ascending, one fused multiply-add per term)
 *     LoHa  d = fp32( (sum_j a1[n, j] * b1[j, k]) * (sum_j a2[n, j] * b2[j, k]) )
 * with out() = rounding to out_dtype and the sum W + delta formed in fp32: `weight += ((strength * alpha) * diff).type(dtype)` of
 * ComfyUI's LoRA / LoHa adapters; only the order of the rank sums differs from the reference's torch.mm.  W is the
 * ggufb200_dequant value in math_dtype cast to out_dtype; for the types of ggufb200_dequant_fallback it is that function's value
 * (fp32, math_dtype is checked but not used).  math_dtype may carry GGUFB200_DEQUANT_SRC_STABLE (accepted, no effect).
 *   packed     the flat block stream of the [N, K] matrix, any alignment: element n * K + k of the stream is W[n, k], so a
 *              straddled weight (K % 256 != 0 with 256-element blocks) needs nothing special; K % 32 == 0, N * K a multiple of the
 *              block size; not BF16 (GGUFB200_E_UNSUPPORTED)
 *   out        N*K elements of out_dtype, 16-byte aligned
 *   patches    host array of n_patches (0 .. GGUFB200_LOWRANK_MAX_PATCHES) descriptors; a1 / b1 / a2 / b2 are DEVICE pointers to
 *              row-major fp32 matrices, 4-byte aligned (GGUFB200_E_ALIGN); a2 = NULL: LoRA (r2, b2 ignored), else LoHa.
 *              1 <= r1, r2 <= GGUFB200_LOWRANK_MAX_RANK (GGUFB200_E_SHAPE)
 */
#define GGUFB200_LOWRANK_MAX_PATCHES 8
#define GGUFB200_LOWRANK_MAX_RANK 1024
typedef struct ggufb200_lowrank_patch {
    const float *a1;       /* [N, r1]: LoRA up / LoHa w1a */
    const float *b1;       /* [r1, K]: LoRA down / LoHa w1b */
    const float *a2;       /* [N, r2]: LoHa w2a, NULL for LoRA */
    const float *b2;       /* [r2, K]: LoHa w2b */
    int64_t r1, r2;
    float scale;           /* strength * alpha */
} ggufb200_lowrank_patch;
int ggufb200_dequant_lowrank(int ggml_type, const void *packed, int64_t N, int64_t K, void *out, int out_dtype, int math_dtype,
                             const ggufb200_lowrank_patch *patches, int n_patches, void *stream);

/*
 * ggufb200_dequant_lowrank with a third patch kind: LoKr (LyCORIS Kronecker) on the whole weight, in any mix and order with LoRA /
 * LoCon and LoHa.  Replaces, for a Conv2d with LoKr or Tucker-factored LyCORIS patches, the reference's dequantise +
 * comfy.lora.calculate_weight.  Every element of `out` is, patch by patch in list order,
 *     W'[n, k] = out( W[n, k] + out( fp32(scale) * d[n, k] ) )
 *     GGUFB200_PATCH_LOWRANK  d as in ggufb200_dequant_lowrank (`.lowrank`; a2 = NULL: LoRA, else LoHa)
 *     GGUFB200_PATCH_KRON     d = fp32( A[n / b1, k / b2] * B[n % b1, k % b2] )   (`.kron`: A [a1, a2], B [b1, b2])
 * A Kronecker element is the reference's `torch.kron(w1, w2).reshape(weight.shape)` element for element (B = w2 reshaped to
 * [b1, K / a2]), so a list of Kronecker patches only gives the reference's patched weight bit for bit.  packed, out, N, K,
 * out_dtype and math_dtype as in ggufb200_dequant_lowrank; only the descriptor of a patch's kind is read.
 *   patches    host array of n_patches (0 .. GGUFB200_LOWRANK_MAX_PATCHES) descriptors of any mix of kinds.  Checked per patch:
 *              an unknown kind, or a kron band_dim other than -1 (whole weight only): GGUFB200_E_UNSUPPORTED; a LOWRANK rank out of
 *              range, a non-positive a1 / a2 / b1 / b2, a1 * b1 != N or a2 * b2 != K: GGUFB200_E_SHAPE; a NULL factor:
 *              GGUFB200_E_NULL; a factor that is not 4-byte aligned: GGUFB200_E_ALIGN.  A and B are DEVICE pointers to
 *              row-major fp32 matrices.
 */
#define GGUFB200_PATCH_LOWRANK 0   /* .lowrank: LoRA / LoCon (a2 == NULL) or LoHa */
#define GGUFB200_PATCH_KRON 1      /* .kron: LoKr on the whole weight (band_dim must be -1) */
typedef struct ggufb200_weight_patch {
    int32_t kind;
    ggufb200_lowrank_patch lowrank;
    ggufb200_kron_patch kron;
} ggufb200_weight_patch;
int ggufb200_dequant_patched(int ggml_type, const void *packed, int64_t N, int64_t K, void *out, int out_dtype, int math_dtype,
                             const ggufb200_weight_patch *patches, int n_patches, void *stream);

/*
 * ggufb200_dequant_patched with DoRA (weight-decomposed LoRA) steps.  Replaces, for a Conv2d whose patch list carries
 * `dora_scale` entries, the reference's dequantise + comfy.lora.calculate_weight with its weight_decompose.  `dora` is a host
 * array parallel to `patches`; a descriptor with factor == NULL leaves its patch plain (as in ggufb200_dequant_patched).  For a
 * patch with a factor, element by element in list order, with d the patch's delta (any kind) and out() = rounding to out_dtype:
 *     wc = out( W[n, k] + out( fp32(scale) * d[n, k] ) )          scale = alpha, without the strength
 *     wc = out( wc * factor[i] )                                   i = n (axis 0) or k / group (axis 1)
 *     W'[n, k] = wc                                                strength == 1
 *     W'[n, k] = out( W[n, k] + out( strength * out(wc - W[n, k]) ) )   otherwise
 * which is weight_decompose's `Wc = W + (delta * alpha).to(dtype); Wc *= s; W = Wc` or `Wc -= W; W += strength * Wc` once its
 * factor s = (dora_scale / (norm + eps)).to(dtype) is known: the caller forms s (it depends only on the weight and the patch
 * set) and passes it as fp32 holding the dtype values.  The sums and products are formed in fp32.
 *   dora       host array of n_patches descriptors (NULL: GGUFB200_E_NULL when n_patches > 0).  Per descriptor with a factor:
 *              an axis other than 0 / 1, a group < 1 or K % group != 0 on axis 1: GGUFB200_E_SHAPE; a factor that is not 4-byte
 *              aligned: GGUFB200_E_ALIGN.  factor is a DEVICE pointer to N (axis 0) or K / group (axis 1) fp32 values.
 * Everything else as ggufb200_dequant_patched, checked the same way.
 */
#define GGUFB200_DORA_AXIS_OUT 0   /* one factor per output row (weight_decompose's output axis, LyCORIS wd_on_out) */
#define GGUFB200_DORA_AXIS_IN 1    /* one factor per group of `group` input columns (a Conv2d input channel: group = kh * kw) */
typedef struct ggufb200_dora_patch {
    const float *factor;   /* NULL: a plain patch; else s, [N] or [K / group] */
    int32_t axis;          /* GGUFB200_DORA_AXIS_OUT or GGUFB200_DORA_AXIS_IN */
    int32_t group;         /* input columns per factor (axis 1); not read on axis 0 */
    float strength;        /* strength_patch of the entry: 1 -> W' = wc */
} ggufb200_dora_patch;
int ggufb200_dequant_patched_dora(int ggml_type, const void *packed, int64_t N, int64_t K, void *out, int out_dtype, int math_dtype,
                                  const ggufb200_weight_patch *patches, const ggufb200_dora_patch *dora, int n_patches, void *stream);

/*
 * Quantise dense values into packed GGUF blocks: the inverse of ggufb200_dequant, used to write GGUF files.  Replaces
 * gguf-py's `gguf.quants.quantize(values, qtype)` (gguf/quants.py, the Q4_0 ... Q8_0 and BF16 classes) for
 * Q4_0=2 Q4_1=3 Q5_0=6 Q5_1=7 Q8_0=8 BF16=30.  The source values are widened exactly to fp32; for every finite source the output
 * is bit-identical to gguf-py's bytes (BF16: for every source, NaN quieting included).  Any other ggml_type: GGUFB200_E_TYPE;
 * ggufb200_supported(t, GGUFB200_OP_QUANTIZE) lists exactly these six.
 *   src        n_blocks * block_size contiguous values of src_dtype (0 fp16 / 1 bf16 / 2 fp32), aligned to one value
 *              (GGUFB200_E_ALIGN otherwise)
 *   n_blocks   blocks to write (BF16: elements, its block size is 1)
 *   packed     n_blocks * type_size bytes, block b from src[b*block_size .. +block_size), any alignment
 *   flags      0; any other bit: GGUFB200_E_UNSUPPORTED (reserved)
 * The kernels are launched with programmatic stream serialization and execute griddepcontrol.launch_dependents only after
 * their last write of `packed`, so a following ggufb200_dequant with GGUFB200_DEQUANT_SRC_STABLE, or a ggufb200_linear with
 * GGUFB200_FLAG_W_STABLE, on the same stream may consume the packed bytes without any other synchronisation.
 *   stream     a cudaStream_t, as everywhere in this header
 */
int ggufb200_quantize(int ggml_type, const void *src, int src_dtype, int64_t n_blocks, void *packed, int flags, void *stream);

/*
 * Quantise dense values into packed K-quant super-blocks: Q2_K=10 Q3_K=11 Q4_K=12 Q5_K=13 Q6_K=14, 256 values per super-block.
 * The encoders restate llama.cpp's reference quantisers at tag b3962 without an importance matrix (what `llama-quantize` runs
 * without --imatrix): quantize_row_q{2,3,4,5,6}_K_ref with make_qkx2_quants, make_q3_quants, make_qx_quants and nearest_int.
 * Every fp32 operation is rounded on its own in the reference's order, so the bytes are a function of the input: they equal a
 * plain-C restatement compiled with -ffp-contract=off, bit for bit, for every finite source.  Parity with a llama-quantize
 * binary is NOT verified (see DESIGN.md section 8); a build that contracts multiply-adds into FMAs can differ in a scale's last
 * bit.  Any other ggml_type: GGUFB200_E_TYPE; ggufb200_supported(t, GGUFB200_OP_QUANTIZE_K) lists exactly these five.
 *   src        n_blocks * 256 contiguous values of src_dtype (0 fp16 / 1 bf16 / 2 fp32), aligned to one value
 *              (GGUFB200_E_ALIGN otherwise)
 *   n_blocks   super-blocks to write
 *   packed     n_blocks * type_size bytes (84 / 110 / 144 / 176 / 210), any alignment
 *   flags      0; any other bit: GGUFB200_E_UNSUPPORTED (reserved)
 * Launched like ggufb200_quantize: a following stable-source dequant or Linear on the same stream may consume the packed bytes
 * without any other synchronisation.
 *   stream     a cudaStream_t
 */
int ggufb200_quantize_k(int ggml_type, const void *src, int src_dtype, int64_t n_blocks, void *packed, int flags, void *stream);

/*
 * Integer unpack only (test/debug surface for the "bit-exact integer unpack" contract):
 * per element the integer quant value q as it enters the float multiply, the integer
 * sub-block scale sc (1 if the type has none) and min mn (0 if none).  Any of the three
 * int16 output arrays (n_blocks*block_size each) may be NULL.
 */
int ggufb200_unpack_int(int ggml_type, const void *packed, int64_t n_blocks, int16_t *q, int16_t *sc,
                        int16_t *mn, void *stream);

/*
 * Row gather + dequant: out[i, :] = dequant(W[rows[i], :]).  Replaces the
 * "dequantise the whole table, then F.embedding" of ops.py:251-259 for quantised
 * Embedding weights.  rows: n_rows int64 indices on the device; K = logical row length.
 */
int ggufb200_dequant_rows(int ggml_type, const void *packed, int64_t n_table_rows, int64_t K,
                          const int64_t *rows, int64_t n_rows, void *out, int out_dtype, int math_dtype,
                          void *stream);

/*
 * Row gather of the types of ggufb200_dequant_fallback: out[i, :] = dequant(W[rows[i], :]), every element bit-identical to
 * ggufb200_dequant_fallback's value for that row (gguf-py's fp32 value rounded once to out_dtype; no math dtype).  Replaces, for
 * an Embedding table in one of these types, the reference's dequantisation of the whole table on every call.
 *   packed     n_table_rows rows of K / block_size * type_size bytes, any alignment; K % block_size == 0 and K % 8 == 0
 *   rows       n_rows int64 indices on the device; an index outside 0 .. n_table_rows - 1 gives a row of zeros
 *   out        n_rows * K elements of out_dtype (0 / 1 / 2), 16-byte aligned
 * Any other ggml_type: GGUFB200_E_TYPE (ggufb200_supported(t, GGUFB200_OP_ROWS_FALLBACK) lists exactly the eleven types).
 */
int ggufb200_dequant_rows_fallback(int ggml_type, const void *packed, int64_t n_table_rows, int64_t K, const int64_t *rows, int64_t n_rows,
                                   void *out, int out_dtype, void *stream);

/*
 * Fused Linear: Y[M,N] = X[M,K] * dequant(W)[N,K]^T (+ bias[N]).  Replaces
 * ops.py:242-244 `forward_ggml_cast_weights` = cast_bias_weight (ops.py:193-211)
 * -> get_weight/dequantize_tensor (ops.py:166-191) -> F.linear.
 *   W_packed    N rows of K/block_size*type_size bytes (loader.py:118-120 layout), or a STRADDLED weight: 256-element
 *               blocks, K % 256 != 0, N*K % 256 == 0, K % 8 == 0 -- the flat stream of N*K/256 blocks the GGUF converter
 *               writes for SD1.5 / SDXL tensors (reshaped to [N*K/256, 256] before quantising), row n starting at element
 *               n*K, possibly inside a block.  AUTO serves a straddled weight by GGUFB200_ALGO_DEQUANT_MMA (measured the
 *               faster route, DESIGN.md section 9); GGUFB200_ALGO_FUSED_TMEM reads it when K % 64 == 0 (Q4_K / Q5_K from
 *               the canonical bytes, the others with the block-major copy of ggufb200_repack()); GEMV, GEMV_FAST and
 *               FUSED_MMA return GGUFB200_E_UNSUPPORTED.
 *   X, Y        act_dtype (0 fp16 / 1 bf16), row strides ldx / ldy in ELEMENTS, 16-byte aligned
 *   math_dtype  as in ggufb200_dequant().  Routes 1-3: W is first produced in math_dtype with the reference's rounding
 *               sequence and then cast to act_dtype, exactly the weight the reference hands to F.linear.  Route 4
 *               (GGUFB200_ALGO_FUSED_TMEM, fp16 math only) follows the contract under GGUFB200_FLAG_EXACT_W above.
 *               Accumulation is fp32 on every route.
 *   bias        NULL or N values of bias_dtype (0/1/2)
 *   workspace   scratch of at least ggufb200_linear_workspace() bytes (may be NULL if that is 0).  A W_packed that is
 *               not 16-byte aligned is always served by GGUFB200_ALGO_DEQUANT_MMA and needs that algo's workspace.
 *               GGUFB200_ALGO_FUSED_MMA with few output tiles (short M) cuts K into S ranges across SMs and keeps
 *               the fp32 partial results in the workspace (S*M*N*4 bytes, summed in a fixed order: reproducible);
 *               with less room it uses fewer ranges, with none it runs unsplit; GGUFB200_ALGO_FUSED_TMEM likewise.
 *               ggufb200_linear_workspace() assumes math_dtype == fp16 (the reference default);
 *               ggufb200_linear_workspace_ex() takes the math dtype of the call.
 *   algo        GGUFB200_ALGO_* | GGUFB200_FLAG_*
 */
size_t ggufb200_linear_workspace(int ggml_type, int64_t M, int64_t N, int64_t K, int act_dtype, int algo);

/* Same query with the math dtype of the call: GGUFB200_ALGO_AUTO routes a non-fp16 math dtype to
 * GGUFB200_ALGO_DEQUANT_MMA, and this variant reports that route's size (query and call always agree). */
size_t ggufb200_linear_workspace_ex(int ggml_type, int64_t M, int64_t N, int64_t K, int act_dtype, int math_dtype, int algo);

int ggufb200_linear(int ggml_type, const void *W_packed, int64_t N, int64_t K, const void *X, int64_t M,
                    int64_t ldx, int act_dtype, int math_dtype, const void *bias, int bias_dtype, void *Y,
                    int64_t ldy, void *workspace, size_t workspace_bytes, int algo, void *stream);

/*
 * Linear on a weight in one of the types of ggufb200_dequant_fallback: Y[M,N] = X[M,K] * W[N,K]^T (+ bias[N]), W = gguf-py's fp32
 * values rounded once to act_dtype (bit-identical to ggufb200_dequant_fallback's output), fp32 accumulation, the bias rounded to
 * act_dtype first.  Replaces, for these types, the reference's numpy dequantisation + F.linear.  There is one contract, so there
 * is no math dtype and GGUFB200_FLAG_EXACT_W is accepted with no effect.
 *   W_packed   N rows of K / block_size * type_size bytes; K % block_size == 0, K % 8 == 0, N % 8 == 0 (GGUFB200_E_SHAPE)
 *   X, Y       act_dtype (0 fp16 / 1 bf16), row strides ldx >= K and ldy >= N in ELEMENTS, multiples of 8, 16-byte aligned
 *   bias       NULL or N values of bias_dtype (0/1/2)
 *   workspace  at least ggufb200_linear_fallback_workspace() bytes, 16-byte aligned (may be NULL if that is 0)
 *   algo       GGUFB200_ALGO_FUSED_SYNC: the weight decoded in registers from the packed bytes, never written to memory.  With
 *                  few feature x token tiles K is cut into ranges whose fp32 partial results go to the workspace and are summed
 *                  in a fixed order (reproducible); with less workspace it uses fewer ranges, with none it runs unsplit.
 *              GGUFB200_ALGO_DEQUANT_MMA: ggufb200_dequant_fallback into the workspace (N * K * 2 bytes), then the dense GEMM.
 *              GGUFB200_ALGO_AUTO: FUSED_SYNC up to a per-type crossover M where FUSED_SYNC would cut K into ranges,
 *                  DEQUANT_MMA otherwise (DESIGN.md section 9).
 *              GEMV, GEMV_FAST, FUSED_MMA, FUSED_TMEM: GGUFB200_E_UNSUPPORTED.
 *              Flags: GGUFB200_FLAG_W_STABLE (passed on to the dequant of DEQUANT_MMA as GGUFB200_DEQUANT_SRC_STABLE),
 *              GGUFB200_FLAG_EXACT_W (no effect), GGUFB200_FLAG_NOSPLIT (FUSED_SYNC never cuts K); any other bit:
 *              GGUFB200_E_UNSUPPORTED.
 * A W_packed that is not aligned to its type's block alignment (gcd(type_size, 16): a byte-offset view) is always served by
 * GGUFB200_ALGO_DEQUANT_MMA, which reads any alignment, and needs that algo's workspace (GGUFB200_E_ALIGN without it).
 * ggufb200_linear_fallback_workspace() returns the workspace of the route the call takes for an aligned weight (query and call
 * always agree), 0 for arguments the call refuses.  ggufb200_linear_fallback_route() returns that route
 * (GGUFB200_ALGO_FUSED_SYNC or GGUFB200_ALGO_DEQUANT_MMA), GGUFB200_OK for M == 0 (the call computes nothing), or the error
 * code the call would return for these arguments; the packed Linear layer runs the two steps of DEQUANT_MMA itself when AUTO
 * would take them.
 */
size_t ggufb200_linear_fallback_workspace(int ggml_type, int64_t M, int64_t N, int64_t K, int act_dtype, int algo);
int ggufb200_linear_fallback_route(int ggml_type, int64_t M, int64_t N, int64_t K, int act_dtype, int algo);
int ggufb200_linear_fallback(int ggml_type, const void *W_packed, int64_t N, int64_t K, const void *X, int64_t M, int64_t ldx, int act_dtype,
                             const void *bias, int bias_dtype, void *Y, int64_t ldy, void *workspace, size_t workspace_bytes, int algo,
                             void *stream);

/*
 * Span-major shadow layout (SURVEY 8f rank 3, "one-time GPU repack").  The canonical GGUF rows (loader.py:96-120) can be
 * read by the FUSED_TMEM producers only when a row's 256-wide K-span and the row stride are multiples of 16 bytes; Q2_K / Q3_K /
 * Q6_K / IQ4_XS blocks (84 / 110 / 210 / 136 bytes) and e.g. Q8_0 rows of 2432 elements (2584 bytes) are not.
 * ggufb200_repack() writes a copy out[span][row padded to 256][pitch] (pitch = span bytes padded to a multiple of 16, zero
 * filled) that GGUFB200_ALGO_FUSED_TMEM reads with 16-byte loads for EVERY block format and every K.  The
 * canonical bytes are not modified (GGMLTensor / state_dict semantics are the reference's); the copy is a cache owned by
 * the caller: ggufb200_repack_bytes() bytes, 16-byte aligned, valid as long as the caller keeps it.
 * A straddled weight (see ggufb200_linear) gets a BLOCK-major copy instead: out[block][pitch] for the N*K/256 blocks of the
 * stream, zero padded, N*K/256*pitch bytes (pitch 112 / 112 / 240 / 144 for Q2_K / Q3_K / Q6_K / IQ4_XS).
 * ggufb200_linear_spans() = ggufb200_linear() with that copy at hand: AUTO then takes the FUSED_TMEM kernel for every format
 * (W_packed is still required: the reference-exact routes and EXACT_W read the canonical bytes).
 */
size_t ggufb200_repack_bytes(int ggml_type, int64_t N, int64_t K);
int ggufb200_repack(int ggml_type, const void *W_packed, int64_t N, int64_t K, void *out, void *stream);
int ggufb200_linear_spans(int ggml_type, const void *W_packed, const void *W_spans, int64_t N, int64_t K, const void *X,
                          int64_t M, int64_t ldx, int act_dtype, int math_dtype, const void *bias, int bias_dtype, void *Y,
                          int64_t ldy, void *workspace, size_t workspace_bytes, int algo, void *stream);

/*
 * Packed-weight Linear with a low-rank (LoRA) update folded into the SAME kernel (SURVEY 8f rank 1; replaces the
 * per-forward dequant + comfy.lora.calculate_weight + F.linear of ops.py:171-190 / nodes.py:43-47 for plain LoRA patches):
 *     Y = X * dequant(W)^T + T * U^T (+ bias),   T = X * down^T  [M, 64] act_dtype (row stride ldt, zero padded beyond the
 *     total rank R <= 64),   U = scale * up  [N, 64] fp16, contiguous, zero padded.
 * The update is one extra 64-wide k-block of GGUFB200_ALGO_FUSED_TMEM (U rows take the place of a dequantised weight tile,
 * the T tile is TMA-fed like an activation tile): no second pass over Y, no extra GEMM launch for the up-projection.
 * algo must resolve to GGUFB200_ALGO_FUSED_TMEM (AUTO without EXACT_W on a weight that route supports, or explicit),
 * otherwise GGUFB200_E_UNSUPPORTED.  W_spans may be NULL.  fp16 dequant math.
 */
int ggufb200_linear_lora(int ggml_type, const void *W_packed, const void *W_spans, int64_t N, int64_t K, const void *X, int64_t M,
                         int64_t ldx, int act_dtype, const void *bias, int bias_dtype, const void *T, int64_t ldt, const void *U,
                         void *Y, int64_t ldy, void *workspace, size_t workspace_bytes, int algo, void *stream);

/*
 * ggufb200_linear_lora with a total rank up to 512 and per-tile LoRA ranges (row-band patches such as diffusers-format
 * LoRAs on fused qkv weights):
 *     Y = X * dequant(W)^T + T * U^T (+ bias),   T [M, 64*J] act_dtype (row stride ldt),   U [N, 64*J] fp16 (row stride ldu)
 * The update is J = lora_kblocks extra 64-wide k-blocks (1 <= J <= 8, else GGUFB200_E_SHAPE); k-block j reads columns
 * 64*j .. 64*j+63 of T and U.  ldt and ldu must be at least 64*J and multiples of 8 (GGUFB200_E_ALIGN).
 * tile_kblocks (device memory, may be NULL): ceil(N / 128) pairs of int32 (first, count), one pair per 128 output features
 * n = 128*i .. 128*i+127; those features add only k-blocks first .. first+count-1 (count = 0: none; values are clamped to
 * 0 .. J).  Columns of U that are zero on a tile's rows may be skipped this way without changing the result.  NULL: every
 * tile adds all J k-blocks.  ggufb200_linear_lora is this call with ldu = 64, J = 1, tile_kblocks = NULL.
 */
int ggufb200_linear_lora_ex(int ggml_type, const void *W_packed, const void *W_spans, int64_t N, int64_t K, const void *X, int64_t M,
                            int64_t ldx, int act_dtype, const void *bias, int bias_dtype, const void *T, int64_t ldt, const void *U,
                            int64_t ldu, int lora_kblocks, const int32_t *tile_kblocks, void *Y, int64_t ldy, void *workspace,
                            size_t workspace_bytes, int algo, void *stream);

/*
 * ggufb200_linear_lora_ex with a per-output-feature fp32 scale applied to the whole product before the bias:
 *     Y = act(feature_scale[n] * (X * dequant(W)^T + T * U^T)[m, n] + bias[n])
 * feature_scale: NULL (then this is ggufb200_linear_lora_ex, bit for bit) or N floats in device memory, 16-byte aligned
 * (GGUFB200_E_ALIGN).  With split K the scale is applied once, to the summed fp32 partials.  The packed Linear uses it for
 * DoRA patches: feature_scale holds the output-axis norm factors r, U carries rho_j / r so that T * U^T comes out right.
 */
int ggufb200_linear_lora_scaled(int ggml_type, const void *W_packed, const void *W_spans, int64_t N, int64_t K, const void *X, int64_t M,
                                int64_t ldx, int act_dtype, const void *bias, int bias_dtype, const void *T, int64_t ldt, const void *U,
                                int64_t ldu, int lora_kblocks, const int32_t *tile_kblocks, const float *feature_scale, void *Y,
                                int64_t ldy, void *workspace, size_t workspace_bytes, int algo, void *stream);

/*
 * Plain tensor-core GEMM on an already-dense weight: Y = X * W^T (+bias), W[N,K] in
 * act_dtype.  Used for the F16/BF16 (torch-compatible) Linears of a model and as the
 * second half of GGUFB200_ALGO_DEQUANT_MMA.
 */
int ggufb200_gemm(const void *W, int64_t N, int64_t K, int64_t ldw, const void *X, int64_t M, int64_t ldx,
                  int act_dtype, const void *bias, int bias_dtype, void *Y, int64_t ldy, void *stream);

/* ggufb200_gemm with a per-output-feature fp32 scale: Y = act(feature_scale[n] * (X * W^T)[m, n] + bias[n]).
 * feature_scale: NULL (ggufb200_gemm, bit for bit) or N floats in device memory, 16-byte aligned (GGUFB200_E_ALIGN). */
int ggufb200_gemm_scaled(const void *W, int64_t N, int64_t K, int64_t ldw, const void *X, int64_t M, int64_t ldx, int act_dtype,
                         const void *bias, int bias_dtype, const float *feature_scale, void *Y, int64_t ldy, void *stream);

/*
 * Input gradient of the packed-weight Linear: dX[M, K] = dY[M, N] * W[N, K], W = dequant(W_packed) in act_dtype with the
 * reference's rounding sequence in math_dtype (the weight the reference's F.linear saves for its backward; the exact contract
 * whatever the forward ran).  Two steps on `stream`: the standalone dequant (ggufb200_dequant, or ggufb200_dequant_fallback
 * for its eleven types, which ignore math_dtype) writes W into the workspace, then the dense warpgroup-MMA GEMM reads W's rows
 * MN-major (no transposed copy), fp32 accumulation.  A BF16 weight with bf16 activations is read as it is: no dequant, no
 * workspace.
 *   ggml_type   every type of ggufb200_dequant and of ggufb200_dequant_fallback (ggufb200_supported(t, GGUFB200_OP_LINEAR_GRAD))
 *   W_packed    the rows as in ggufb200_linear (straddled weights included); for the types of ggufb200_dequant_fallback the
 *               flat block stream of the [N, K] tensor, N * K a multiple of the block size.  Any alignment, except the BF16 read
 *               in place (16-byte aligned, GGUFB200_E_ALIGN)
 *   dY, dX      act_dtype (0 fp16 / 1 bf16), row strides ldy >= N and ldx >= K in ELEMENTS, multiples of 8, 16-byte aligned
 *               (GGUFB200_E_ALIGN); K % 8 == 0 (GGUFB200_E_SHAPE); any N
 *   workspace   at least ggufb200_linear_grad_input_workspace() bytes (N * K * 2, or 0), 16-byte aligned
 *   flags       0 or GGUFB200_FLAG_W_STABLE (passed on to the dequant as GGUFB200_DEQUANT_SRC_STABLE); any other bit:
 *               GGUFB200_E_UNSUPPORTED
 */
size_t ggufb200_linear_grad_input_workspace(int ggml_type, int64_t N, int64_t K, int act_dtype);
int ggufb200_linear_grad_input(int ggml_type, const void *W_packed, int64_t N, int64_t K, const void *dY, int64_t M, int64_t ldy,
                               int act_dtype, int math_dtype, void *dX, int64_t ldx, void *workspace, size_t workspace_bytes, int flags,
                               void *stream);

/*
 * Column scale: Y[m, k] = act(float(X[m, k]) * col_scale[k]) for m < M, k < K, one fp32 multiply and one round-to-nearest
 * per element (bit-identical to torch's `(x.float() * c).to(x.dtype)`).  X, Y: act_dtype (0 fp16 / 1 bf16), row strides ldx /
 * ldy in elements (>= K, multiples of 8), 16-byte aligned; col_scale: K floats in device memory, 16-byte aligned; K % 8 == 0.
 * Y must not overlap X.  The packed Linear uses it for the input-axis factors of DoRA patches.
 */
int ggufb200_scale_columns(const void *X, int64_t M, int64_t K, int64_t ldx, int act_dtype, const float *col_scale, void *Y, int64_t ldy,
                           void *stream);

/* Diagnostics: the tiling a fused kernel uses for this problem when given `workspace_bytes` of scratch.
 * algo = GGUFB200_ALGO_FUSED_MMA (| flags): activation rows per tile (128), number of K ranges (1 = unsplit),
 *   64-wide k-blocks per range (the last range may be shorter, never empty), CTAs launched (one per 128 x 256 tile and range).
 * algo = GGUFB200_ALGO_FUSED_TMEM (| flags): tokens per item (32 / 128 / 192 / 384), number of K ranges, k-blocks per range,
 *   number of work items (each served by 2 CTAs of 128 features per 192 / 128 / 32 tokens).
 * Pure host arithmetic, no GPU needed. */
int ggufb200_linear_plan(int ggml_type, int64_t M, int64_t N, int64_t K, size_t workspace_bytes, int algo, int *tile_rows, int *k_ranges,
                         int *kblocks_per_range, int *ctas);

/* Benchmark-only launch knobs (they never change routing or results):
 * key 1 = programmatic dependent launch of the standalone dequant kernel (default 1),
 * key 2 = CTAs per SM of the small-M integer-pattern kernel (0 = planner picks).
 * Refused with GGUFB200_E_UNSUPPORTED unless the environment variable GGUFB200_ALLOW_TUNING=1 is set when the
 * library is first used; every other key is refused always (route selection is per call: GGUFB200_ALGO_* | GGUFB200_FLAG_*). */
int ggufb200_set_tuning(int key, int value);

#ifdef __cplusplus
}
#endif
#endif /* GGUFB200_H */
