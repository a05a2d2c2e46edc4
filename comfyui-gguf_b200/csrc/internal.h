// internal.h -- every function api.cu calls in another translation unit, and the two tuning globals.  api.cu and each file
// that defines one of these include this header, so a changed signature fails to compile instead of to link, and default
// arguments are written here only.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/ggufb200.h"

namespace ggufb200 {

// ------------------------------------------------------------------ tuning switches (ggufb200_set_tuning)
extern int g_dequant_pdl;      // dequant.cu: programmatic dependent launch of the dequant kernel (key 1)
extern int g_gemv2_ctas;       // gemv2.cu: CTAs per SM of the integer-pattern GEMV, 0 = pick (key 2)

// ------------------------------------------------------------------ dequant.cu, rows.cu
int dequant_dispatch(int type, const void *packed, long long n_blocks, void *out, int out_dtype, int math_dtype, cudaStream_t st, bool stable = false);
// ggufb200_dequant_fallback: K1 for the formats of fallback.cuh (fp32 math); arguments validated by the caller
int fallback_dispatch(int type, const void *packed, long long n_blocks, void *out, int out_dtype, cudaStream_t st, bool stable);
int unpack_dispatch(int type, const void *packed, long long n_blocks, int16_t *q, int16_t *sc, int16_t *mn, cudaStream_t st);
int rows_dispatch(int type, const void *packed, long long n_table_rows, long long K, const long long *rows, long long n_rows, void *out,
                  int out_dtype, int math_dtype, cudaStream_t st);
// ggufb200_dequant_rows_fallback: the row gather for the formats of fallback.cuh (fp32 math); arguments validated by the caller
int rows_fallback_dispatch(int type, const void *packed, long long n_table_rows, long long K, const long long *rows, long long n_rows, void *out,
                           int out_dtype, cudaStream_t st);
// ggufb200_dequant_kron: the [N, K] weight (whole-block rows or straddled, K % 8 == 0) with LoKr patches applied; `patches` are
// validated by the caller (api.cu), n_patches <= kKronMaxPatches
constexpr int kKronMaxPatches = 8;
int dequant_kron_dispatch(int type, const void *packed, long long N, long long K, void *out, int out_dtype, int math_dtype,
                          const ggufb200_kron_patch *patches, int n_patches, cudaStream_t st, bool stable);
// lowrank.cu, ggufb200_dequant_lowrank: the [N, K] weight (flat block stream, K % 32 == 0) with LoRA / LoHa patches applied;
// block formats and fallback formats; `patches` validated by the caller (api.cu)
constexpr int kLowrankMaxPatches = GGUFB200_LOWRANK_MAX_PATCHES;
int dequant_lowrank_dispatch(int type, const void *packed, long long N, long long K, void *out, int out_dtype, int math_dtype,
                             const ggufb200_lowrank_patch *patches, int n_patches, cudaStream_t st);
// lowrank.cu, ggufb200_dequant_patched: the same with Kronecker (LoKr) patches as well; `patches` validated by the caller (api.cu)
// lowrank.cu, ggufb200_dequant_patched_dora: the same with a DoRA step per patch (`dora`: n_patches descriptors, validated by
// the caller)
int dequant_patched_dora_dispatch(int type, const void *packed, long long N, long long K, void *out, int out_dtype, int math_dtype,
                                  const ggufb200_weight_patch *patches, const ggufb200_dora_patch *dora, int n_patches, cudaStream_t st);
int dequant_patched_dispatch(int type, const void *packed, long long N, long long K, void *out, int out_dtype, int math_dtype,
                             const ggufb200_weight_patch *patches, int n_patches, cudaStream_t st);

// quantize.cu, ggufb200_quantize: dense fp32 / fp16 / bf16 -> packed Q4_0 / Q4_1 / Q5_0 / Q5_1 / Q8_0 / BF16; arguments validated by
// the caller (api.cu)
bool quantize_supported(int type);
int quantize_dispatch(int type, const void *src, int src_dtype, long long n_blocks, void *packed, cudaStream_t st);
// quantize.cu, ggufb200_quantize_k: dense fp32 / fp16 / bf16 -> packed Q2_K / Q3_K / Q4_K / Q5_K / Q6_K (n_blocks super-blocks)
bool quantize_k_supported(int type);
int quantize_k_dispatch(int type, const void *src, int src_dtype, long long n_blocks, void *packed, cudaStream_t st);

// ------------------------------------------------------------------ small-M Linear: gemv.cu (GGUFB200_ALGO_GEMV), gemv2.cu (GEMV_FAST)
int gemv_max_m();
int gemv_dispatch(int type, const void *W, long long N, long long K, const void *X, long long M, long long ldx, int act_dtype, int math_dtype,
                  const void *bias, int bias_dtype, void *Y, long long ldy, cudaStream_t st);
bool gemv2_supported(int type, const void *W, long long N, long long K, long long M);
int gemv2_dispatch(int type, const void *W, long long N, long long K, const void *X, long long M, long long ldx, int act_dtype, const void *bias,
                   int bias_dtype, void *Y, long long ldy, cudaStream_t st, bool w_stable = false);

// A weight whose 256-element super-blocks straddle rows: the flat block stream of an [N, K] tensor with K % 256 != 0,
// as the GGUF converter writes SD1.5 / SDXL K-quant tensors (reshaped to [N * K / 256, 256] before quantising).  Row n
// starts at element n * K of the stream, which may fall inside a block.
inline bool straddled_rows(int block_size, long long N, long long K)
{
    return block_size == 256 && K % 256 != 0 && (N * K) % 256 == 0;
}

// ------------------------------------------------------------------ repack.cu: the span-major copy of a packed weight
// (block-major out[b][pitch] for a straddled weight: span_stride = pitch)
size_t repack_bytes(int type, long long N, long long K, int *pitch, long long *span_stride);
int repack_dispatch(int type, const void *W, long long N, long long K, void *out, cudaStream_t st);

// ------------------------------------------------------------------ linear_sm90.cu: the warpgroup-MMA Linear
// Per-call options of the fused routes, decoded once from the GGUFB200_FLAG_* bits (api.cu).
struct LinearOptions {
    enum Producers { FAST, EXACT, GENERIC };
    Producers producers = FAST;    // FUSED_TMEM weight producers: hand-written with one fused multiply-add per element (FAST),
                                   // hand-written with the reference's rounding sequence (EXACT), functor producers (GENERIC)
    int tile = 0;                  // FUSED_TMEM token items: 0 = the cost model picks, 192 or 384 = forced
    bool nosplit = false;          // never cut K into ranges (always set for a straddled weight)
};

// `ws_bytes` is the usable workspace at `ws`: 0 when the caller passed none or a misaligned one.
// Dense GEMM: ggufb200_gemm and the GEMM half of GGUFB200_ALGO_DEQUANT_MMA.
// scale: nullptr, or fp32 [N] (16-byte aligned) multiplied into each output feature before the bias (ggufb200_gemm_scaled).
int dense_gemm(const void *W, long long N, long long K, long long ldw, const void *X, long long M, long long ldx, int act_dtype,
               const void *bias, int bias_dtype, void *Y, long long ldy, cudaStream_t st, const float *scale = nullptr);
// Y[M, Kout] = X[M, Nred] * B[Nred, Kout] with B row-major (ldb >= Kout), fp32 accumulation, no bias: the GEMM of
// ggufb200_linear_grad_input.  Kout % 8 == 0; the alignment rules of dense_gemm.
int dense_gemm_nn(const void *B, long long Nred, long long Kout, long long ldb, const void *X, long long M, long long ldx, int act_dtype, void *Y,
                  long long ldy, cudaStream_t st);
// GGUFB200_ALGO_FUSED_MMA: reference-exact producers, the weight as the wide operand.
size_t fused_mma_workspace(long long M, long long N, long long K, const LinearOptions &opt);
void fused_mma_plan(long long M, long long N, long long K, size_t ws_bytes, const LinearOptions &opt, int *tile_rows, int *splits,
                    int *kb_per_split, int *ctas);
int fused_mma_linear(int type, const void *W, long long N, long long K, const void *X, long long M, long long ldx, int act_dtype,
                     const void *bias, int bias_dtype, void *Y, long long ldy, void *ws, size_t ws_bytes, const LinearOptions &opt,
                     cudaStream_t st);
// GGUFB200_ALGO_FUSED_TMEM: the transposed product, token tiles sized to the activation, optional LoRA k-blocks.
constexpr int kLoraMaxKblocks = 8;
struct LoraOperands {
    const void *T;         // x * down^T: [M, 64 * kblocks] activation dtype, row stride ldt; nullptr = no LoRA
    long long ldt;
    const void *U;         // scale * up: [N, 64 * kblocks] fp16, row stride ldu
    long long ldu;
    int kblocks;           // J, 1 .. kLoraMaxKblocks
    const int32_t *tiles;  // (first, count) per 128-feature tile, ceil(N / 128) pairs, or nullptr = every tile runs all J
};
bool fused_tmem_supported(int type, const void *W, long long N, long long K);
size_t fused_tmem_workspace(long long M, long long N, long long K, const LinearOptions &opt);
void fused_tmem_plan(long long M, long long N, long long K, size_t ws_bytes, const LinearOptions &opt, int *tile_tokens, int *splits,
                     int *spans_per_split, int *items);
// scale: as for dense_gemm (ggufb200_linear_lora_scaled)
int fused_tmem_linear(int type, const void *W, const void *Wspan, long long span_stride, long long N, long long K, const void *X, long long M,
                      long long ldx, int act_dtype, const void *bias, int bias_dtype, void *Y, long long ldy, void *ws, size_t ws_bytes,
                      const LinearOptions &opt, const LoraOperands &lora, cudaStream_t st, const float *scale = nullptr);

// The split-K finalize of the fused routes: Y = act(sum_s P[s] + bias), P fp32 [splits, M, N], slices added in ascending order;
// N % 8 == 0, Y and ldy as for dense_gemm.
int split_k_finalize(const float *P, int splits, const void *bias, int bias_dtype, void *Y, long long M, long long N, long long ldy, int act_dtype,
                     cudaStream_t st);

// ------------------------------------------------------------------ linear_fallback.cu: GGUFB200_ALGO_FUSED_SYNC, the fused Linear of
// the fallback.cuh formats (arguments validated by the caller: K % 32 == 0, N % 8 == 0, W aligned to the type's A_BLK).
// `ws_bytes` as above; with too little workspace the kernel uses fewer K ranges, with none it runs unsplit.
size_t fallback_linear_workspace(long long M, long long N, long long K, bool nosplit);
int fallback_linear(int type, const void *W, long long N, long long K, const void *X, long long M, long long ldx, int act_dtype, const void *bias,
                    int bias_dtype, void *Y, long long ldy, void *ws, size_t ws_bytes, bool nosplit, cudaStream_t st);

// ------------------------------------------------------------------ scale.cu: Y = act(fp32(X) * c[k]) (ggufb200_scale_columns)
int scale_columns_dispatch(const void *X, long long M, long long K, long long ldx, int act_dtype, const float *col_scale, void *Y,
                           long long ldy, cudaStream_t st);

}  // namespace ggufb200
