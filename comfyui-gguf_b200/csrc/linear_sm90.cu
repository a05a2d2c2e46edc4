// linear_sm90.cu -- host side of the warpgroup-MMA Linear (wg_linear_kernel, linear_sm90.cuh): three launchers, the split-K
// planners of the two fused routes and their finalize.
//
//   Y[M,N] = X[M,K] * W[N,K]^T (+ bias)      X fp16 / bf16, fp32 accumulation
//
//   dense_gemm          W dense: both operands TMA-fed, one CTA per 128-token x BN-feature tile (ggufb200_gemm and the GEMM
//                       half of GGUFB200_ALGO_DEQUANT_MMA).  A ragged last k-block is zero-filled by the TMA engine.
//   dense_gemm_nn       Y[M, Kout] = X[M, Nred] * B[Nred, Kout], B row-major (ggufb200_linear_grad_input: dX = dY * W with the
//                       dequantised W): the same kernel and tiling with B staged MN-major straight from its rows (B_MN).
//   fused_mma_linear    GGUFB200_ALGO_FUSED_MMA: A = 128 activation rows (TMA), B = 256 weight rows that the producer warpgroup
//                       dequantises from the canonical packed rows with the reference's fp16 rounding sequence (Producer<Q>),
//                       so the weight operand is bit-identical to what the reference hands to F.linear.  Every block format,
//                       any row alignment.  One CTA per (K range, 128-token x 256-feature tile).
//   fused_tmem_linear   GGUFB200_ALGO_FUSED_TMEM, AUTO's route: the product is computed TRANSPOSED, D[feature n, token m], so the
//                       token tile is the N dimension of the warpgroup MMA and can be as short as the activation (32 / 128 /
//                       192 tokens): A = 128 weight rows dequantised by the producer warpgroup (produce.cuh: hand-written
//                       producers for the hot formats, the functor producer for the others), B = the TMA-fed activation tile.
//                       The packed rows are read one 256-wide span at a time from the canonical layout (when a row's span and
//                       the row stride are multiples of 16 bytes) or from the span-major copy of repack.cu (every format).
//                       A straddled weight (straddled_rows(): SD1.5 / SDXL K-quants at K % 256 != 0) is read as the flat
//                       stream of 256-element blocks it is, from the canonical bytes (Q4_K / Q5_K) or the block-major copy
//                       of repack.cu (the others): k-block kb of row n is one quarter of block (n K + 64 kb) / 256, the
//                       kernel runs K / 64 k-blocks and K is never split into ranges.
//                       With bf16 activations the weight is cast to bf16 (the reference's cast before F.linear).  Work item =
//                       (K range, 256-feature tile, token tile), served by 2 * ACCS CTAs (128 features x TT tokens each).  An
//                       optional LoRA update rides as J <= 8 extra k-blocks of the K range 0: A = U rows (scale * up), B = T =
//                       x * down^T, k-block j at columns 64 j of both; a per-tile table can narrow each 128-feature tile to the
//                       k-blocks whose U rows are not zero there.  K is processed in whole 256-wide spans: k-blocks past K are
//                       zero on both operands.
//
// Split-K (both fused routes): when the output tiles leave SMs idle, K is cut into ranges of whole 256-wide spans, one CTA
// per (tile, range); each CTA stores its fp32 partial tile into its own slice of the caller's workspace ([S, M, N] fp32) and
// wg_finalize_kernel adds the slices in ascending order.  Every packed byte is still read once per token tile.
//
// Feature scale (ggufb200_gemm_scaled, ggufb200_linear_lora_scaled): the dense GEMM and FUSED_TMEM can multiply each output
// feature by an fp32 factor before the bias, Y = act(scale[n] * acc + bias[n]), in the epilogue or in the split-K finalize.
// Only those two launchers instantiate the SCALED kernels; a NULL scale runs the unscaled instances.
#include "internal.h"
#include "linear_sm90.cuh"

namespace ggufb200 {

// ------------------------------------------------------------------ split-K, shared by both fused routes
constexpr size_t kSplitWsCap = 24u << 20;   // about half of the 50 MB L2 of an H100: the slices stay L2-resident until the finalize
constexpr int kSpan = 256;                  // K elements of one packed span (= 4 k-blocks): K ranges are whole spans

static size_t split_ws(size_t ws_bytes) { return ws_bytes > kSplitWsCap ? kSplitWsCap : ws_bytes; }

// K cut into at most `s` ranges of whole spans: `per` spans each, `count` ranges (the last may be shorter but never empty)
struct KRanges {
    long long per, count;
};
static KRanges k_ranges(long long spans, long long s)
{
    const long long per = (spans + s - 1) / s;
    return {per, (spans + per - 1) / per};
}

static size_t partial_bytes(int splits, long long M, long long N) { return splits > 1 ? (size_t)splits * (size_t)M * (size_t)N * 4 : 0; }

// ------------------------------------------------------------------ dense GEMM
template <int ACT, int BN, bool SCALED>
static int dense_launch(const void *W, long long N, long long K, long long ldw, const void *X, long long M, long long ldx, const void *bias,
                        int bias_dtype, void *Y, long long ldy, cudaStream_t st, const float *scale)
{
    CUtensorMap tmA, tmB;
    if (!make_kblock_map(&tmA, X, M, K, ldx, ACT, 128)) return GGUFB200_E_CUDA;
    if (!make_kblock_map(&tmB, W, N, K, ldw, ACT, BN)) return GGUFB200_E_CUDA;
    WgParams p{};
    p.M = M; p.N = N; p.K = K;
    p.bias = bias; p.bias_dtype = bias_dtype;
    p.Y = reinterpret_cast<uint8_t *>(Y); p.ldy = ldy;
    p.ttiles = (int)((M + 127) / 128);
    p.ftiles = (int)((N + BN - 1) / BN);
    p.kb_total = (int)((K + kBlockK - 1) / kBlockK);
    p.kb_per_split = p.kb_total;
    p.scale = scale;
    return wg_launch<void, void, ACT, BN, false, false, SCALED>(tmA, tmB, tmA, p, 1, st);
}

template <bool SCALED>
static int dense_tiles(const void *W, long long N, long long K, long long ldw, const void *X, long long M, long long ldx, int act_dtype,
                       const void *bias, int bias_dtype, void *Y, long long ldy, cudaStream_t st, const float *scale)
{
    // 256-wide feature tiles; 128 when that leaves most SMs idle (short activations such as a 512-token text stream)
    const long long tiles256 = ((M + 127) / 128) * ((N + 255) / 256);
    const bool narrow = tiles256 < sm_count();
    if (narrow)
        return act_dtype == kBF16 ? dense_launch<kBF16, 128, SCALED>(W, N, K, ldw, X, M, ldx, bias, bias_dtype, Y, ldy, st, scale)
                                  : dense_launch<kF16, 128, SCALED>(W, N, K, ldw, X, M, ldx, bias, bias_dtype, Y, ldy, st, scale);
    return act_dtype == kBF16 ? dense_launch<kBF16, 256, SCALED>(W, N, K, ldw, X, M, ldx, bias, bias_dtype, Y, ldy, st, scale)
                              : dense_launch<kF16, 256, SCALED>(W, N, K, ldw, X, M, ldx, bias, bias_dtype, Y, ldy, st, scale);
}

int dense_gemm(const void *W, long long N, long long K, long long ldw, const void *X, long long M, long long ldx, int act_dtype,
               const void *bias, int bias_dtype, void *Y, long long ldy, cudaStream_t st, const float *scale)
{
    if (K % 8 != 0 || N % 8 != 0) return GGUFB200_E_UNSUPPORTED;
    return scale ? dense_tiles<true>(W, N, K, ldw, X, M, ldx, act_dtype, bias, bias_dtype, Y, ldy, st, scale)
                 : dense_tiles<false>(W, N, K, ldw, X, M, ldx, act_dtype, bias, bias_dtype, Y, ldy, st, nullptr);
}

template <int ACT, int BN>
static int dense_nn_launch(const void *B, long long Nred, long long Kout, long long ldb, const void *X, long long M, long long ldx, void *Y,
                           long long ldy, cudaStream_t st)
{
    CUtensorMap tmA, tmB;
    if (!make_kblock_map(&tmA, X, M, Nred, ldx, ACT, 128)) return GGUFB200_E_CUDA;
    if (!make_kblock_map(&tmB, B, Nred, Kout, ldb, ACT, 64)) return GGUFB200_E_CUDA;      // [64 k rows][64 columns] boxes
    WgParams p{};
    p.M = M; p.N = Kout; p.K = Nred;
    p.Y = reinterpret_cast<uint8_t *>(Y); p.ldy = ldy;
    p.ttiles = (int)((M + 127) / 128);
    p.ftiles = (int)((Kout + BN - 1) / BN);
    p.kb_total = (int)((Nred + kBlockK - 1) / kBlockK);
    p.kb_per_split = p.kb_total;
    return wg_launch<void, void, ACT, BN, false, false, false, true>(tmA, tmB, tmA, p, 1, st);
}

int dense_gemm_nn(const void *B, long long Nred, long long Kout, long long ldb, const void *X, long long M, long long ldx, int act_dtype, void *Y,
                  long long ldy, cudaStream_t st)
{
    if (Kout % 8 != 0) return GGUFB200_E_UNSUPPORTED;
    // output tiles as dense_tiles: 256 columns wide, 128 when that leaves most SMs idle
    const bool narrow = ((M + 127) / 128) * ((Kout + 255) / 256) < sm_count();
    if (narrow)
        return act_dtype == kBF16 ? dense_nn_launch<kBF16, 128>(B, Nred, Kout, ldb, X, M, ldx, Y, ldy, st)
                                  : dense_nn_launch<kF16, 128>(B, Nred, Kout, ldb, X, M, ldx, Y, ldy, st);
    return act_dtype == kBF16 ? dense_nn_launch<kBF16, 256>(B, Nred, Kout, ldb, X, M, ldx, Y, ldy, st)
                              : dense_nn_launch<kF16, 256>(B, Nred, Kout, ldb, X, M, ldx, Y, ldy, st);
}

// ------------------------------------------------------------------ GGUFB200_ALGO_FUSED_MMA
constexpr int kMmaBM = 128;         // token tile
constexpr int kMmaBN = 256;         // feature tile

static long long mma_tiles(long long M, long long N) { return ((M + kMmaBM - 1) / kMmaBM) * ((N + kMmaBN - 1) / kMmaBN); }

// One-wave rule: split only when the tiles fill less than half the SMs, into S ranges with S * tiles <= SMs, at most 16, and
// as many slices as the workspace holds.  (The thresholds follow the one-wave rule; they have not been tuned by measurement
// on the H100.)
static int mma_splits(long long M, long long N, long long K, size_t ws_bytes, bool allow_split)
{
    const size_t slice = (size_t)M * (size_t)N * 4;
    ws_bytes = split_ws(ws_bytes);
    if (slice == 0 || ws_bytes < 2 * slice || !allow_split || K % kSpan != 0) return 1;
    const long long sms = sm_count();
    const long long t = mma_tiles(M, N);
    if (t * 2 > sms) return 1;
    const long long spans = K / kSpan;
    long long s = sms / t;
    if (s > spans) s = spans;
    if (s > 16) s = 16;
    if (s > (long long)(ws_bytes / slice)) s = (long long)(ws_bytes / slice);
    if (s < 2) return 1;
    return (int)k_ranges(spans, s).count;
}

// k-blocks (64 wide) each K range walks: whole spans, the last range may be shorter but never empty
static int mma_kb_per_split(long long K, int splits)
{
    if (splits <= 1) return (int)(K / kBlockK);
    const int spans = (int)(K / kSpan);
    return ((spans + splits - 1) / splits) * 4;
}

size_t fused_mma_workspace(long long M, long long N, long long K, const LinearOptions &opt)
{
    return partial_bytes(mma_splits(M, N, K, kSplitWsCap, !opt.nosplit), M, N);
}

void fused_mma_plan(long long M, long long N, long long K, size_t ws_bytes, const LinearOptions &opt, int *tile_rows, int *splits,
                    int *kb_per_split, int *ctas)
{
    const int s = mma_splits(M, N, K, ws_bytes, !opt.nosplit);
    *tile_rows = kMmaBM;
    *splits = s;
    *kb_per_split = mma_kb_per_split(K, s);
    *ctas = (int)(mma_tiles(M, N) * s);
}

template <class Q, int ACT>
static int fused_mma_run(const void *W, long long N, long long K, const void *X, long long M, long long ldx, const void *bias, int bias_dtype,
                         void *Y, long long ldy, void *ws, size_t ws_bytes, const LinearOptions &opt, cudaStream_t st)
{
    const int splits = mma_splits(M, N, K, ws_bytes, !opt.nosplit);
    float *P = splits > 1 ? reinterpret_cast<float *>(ws) : nullptr;
    CUtensorMap tmA;
    if (!make_kblock_map(&tmA, X, M, K, ldx, ACT, kMmaBM)) return GGUFB200_E_CUDA;
    WgParams p{};
    p.M = M; p.N = N; p.K = K;
    p.bias = P ? nullptr : bias; p.bias_dtype = bias_dtype;
    p.Y = reinterpret_cast<uint8_t *>(Y); p.ldy = ldy;
    p.partial = P;
    p.W = reinterpret_cast<const uint8_t *>(W);
    p.row_bytes = K / Q::BS * Q::TS;
    p.ttiles = (int)((M + kMmaBM - 1) / kMmaBM);
    p.ftiles = (int)((N + kMmaBN - 1) / kMmaBN);
    p.kb_total = (int)(K / kBlockK);
    p.kb_per_split = mma_kb_per_split(K, splits);
    int rc = wg_launch<Q, Producer<Q>, ACT, kMmaBN, false>(tmA, tmA, tmA, p, splits, st);
    if (rc != GGUFB200_OK || !P) return rc;
    return wg_finalize<ACT>(P, splits, bias, bias_dtype, Y, M, N, ldy, st);
}

int fused_mma_linear(int type, const void *W, long long N, long long K, const void *X, long long M, long long ldx, int act_dtype,
                     const void *bias, int bias_dtype, void *Y, long long ldy, void *ws, size_t ws_bytes, const LinearOptions &opt,
                     cudaStream_t st)
{
    if (K % kBlockK != 0 || N % 8 != 0) return GGUFB200_E_UNSUPPORTED;
    return with_block(type, GGUFB200_E_UNSUPPORTED, [&](auto blk) {
        using Q = decltype(blk);
        return act_dtype == kBF16 ? fused_mma_run<Q, kBF16>(W, N, K, X, M, ldx, bias, bias_dtype, Y, ldy, ws, ws_bytes, opt, st)
                                  : fused_mma_run<Q, kF16>(W, N, K, X, M, ldx, bias, bias_dtype, Y, ldy, ws, ws_bytes, opt, st);
    });
}

// ------------------------------------------------------------------ GGUFB200_ALGO_FUSED_TMEM
struct TmemPlan {
    int tt, accs, splits, spans_per_split, ttiles, ftiles, n_items;
};

// Tiling: token tile TT in {32, 128, 192}; ACCS = 2 (384-token items) when asked for; K split into ranges of whole spans
// when the output has fewer CTAs than SMs (short activations; every packed byte is still read once per token tile).
// Cost model (cycles per SM): a CTA of TT tokens x kb k-blocks costs kb * max(4 * TT, 2000) (warpgroup MMA 128 x TT x 64 at
// 2048 FMA per cycle = 4 * TT cycles; ~2000 cycles per k-block is what the producer warpgroup took to dequantise a 128 x 64
// Q4_K weight tile on an H100, read off kernel times at M = 512 and 4608, so the kernel is producer bound at every tile)
// + 3000 (pipeline fill + drain), and the kernel runs ceil(CTAs / SMs) rounds.  Candidates: token tile 32 (M <= 32) / 128 /
// 192 / 384, K cut into 1..32 ranges of whole spans when a workspace for the fp32 partials is available (finalize pass
// charged at 16 bytes / cycle / SM: the slices stay L2 resident).  tile: 0 = let the model decide, 192 / 384 = force
// 192- / 384-token items.
static TmemPlan tmem_plan(long long M, long long N, long long K, size_t ws_bytes, int tile, bool allow_split)
{
    const int sms = sm_count();
    const int ftiles = (int)((N + 255) / 256);
    const int spans = (int)((K + kSpan - 1) / kSpan);
    const size_t slice = (size_t)M * (size_t)N * 4;
    ws_bytes = split_ws(ws_bytes);
    int max_s = 1;
    if (allow_split && slice > 0 && ws_bytes >= 2 * slice) {
        long long cap = (long long)(ws_bytes / slice);
        max_s = (int)(cap < 32 ? cap : 32);
        if (max_s > spans) max_s = spans;
    }
    struct Cand { int tt, accs; };
    Cand cands[4];
    int nc = 0;
    if (M <= 32) cands[nc++] = {32, 1};
    else {
        if (tile == 0 || M <= 192) cands[nc++] = {128, 1};
        if (tile != 384 || M <= 192) cands[nc++] = {192, 1};
        if (tile != 192 && M > 192) cands[nc++] = {192, 2};
    }
    TmemPlan best{};
    double best_cost = 0;
    for (int c = 0; c < nc; ++c) {
        const int item = cands[c].tt * cands[c].accs;
        const int ttiles = (int)((M + item - 1) / item);
        const long long tiles = (long long)ftiles * ttiles;
        for (int s = 1; s <= max_s; ++s) {
            const KRanges r = k_ranges(spans, s);
            if (r.count != s) continue;                                 // same split count as a smaller s: already evaluated
            const int per = (int)r.per, splits = (int)r.count;
            const long long items = tiles * splits;
            const long long ctas = items * 2 * cands[c].accs;
            const long long rounds = (ctas + sms - 1) / sms;
            const double t_kb = 4.0 * cands[c].tt > 2000.0 ? 4.0 * cands[c].tt : 2000.0;
            double cost = (double)rounds * (4.0 * per * t_kb + 3000.0);
            if (splits > 1) cost += (double)(splits + 1) * (double)slice / (16.0 * sms) + 6000.0;   // partial stores + finalize pass (L2 resident) + its launch
            if (best.n_items == 0 || cost < best_cost * 0.98) {         // prefer the earlier (simpler) candidate on near ties
                best_cost = cost;
                best.tt = cands[c].tt; best.accs = cands[c].accs; best.splits = splits; best.spans_per_split = per;
                best.ttiles = ttiles; best.ftiles = ftiles; best.n_items = (int)items;
            }
        }
    }
    return best;
}

size_t fused_tmem_workspace(long long M, long long N, long long K, const LinearOptions &opt)
{
    return partial_bytes(tmem_plan(M, N, K, kSplitWsCap, opt.tile, !opt.nosplit).splits, M, N);
}

void fused_tmem_plan(long long M, long long N, long long K, size_t ws_bytes, const LinearOptions &opt, int *tile_tokens, int *splits,
                     int *spans_per_split, int *items)
{
    const TmemPlan pl = tmem_plan(M, N, K, ws_bytes, opt.tile, !opt.nosplit);
    *tile_tokens = pl.tt * pl.accs;
    *splits = pl.splits;
    *spans_per_split = pl.spans_per_split;
    *items = pl.n_items;
}

struct TmemArgs {
    const void *W;             // canonical packed rows
    const void *Wspan;         // re-packed span-major layout or nullptr
    long long span_stride;
    long long N, K;
    const void *X;
    long long M, ldx;
    const void *bias;
    int bias_dtype;
    void *Y;
    long long ldy;
    void *ws;
    size_t ws_bytes;
    const LinearOptions &opt;
    const LoraOperands &lora;  // lora.T == nullptr: no LoRA k-blocks
    cudaStream_t st;
    bool straddled;            // straddled_rows(): W (or Wspan, the block-major copy) is a flat stream of 256-element blocks
    const float *scale;        // fp32 [N] feature scale (SCALED instances) or nullptr
};

template <class Q, class Prod, int ACT, int TT, bool SCALED>
static int tmem_launch(const TmemArgs &a, const TmemPlan &pl, float *partial)
{
    CUtensorMap tmX, tmT;
    if (!make_kblock_map(&tmX, a.X, a.M, a.K, a.ldx, ACT, TT)) return GGUFB200_E_CUDA;
    tmT = tmX;
    if (a.lora.T && !make_kblock_map(&tmT, a.lora.T, a.M, (long long)kBlockK * a.lora.kblocks, a.lora.ldt, ACT, TT)) return GGUFB200_E_CUDA;
    WgParams p{};
    p.M = a.M; p.N = a.N; p.K = a.K;
    p.bias = partial ? nullptr : a.bias;
    p.bias_dtype = a.bias_dtype;
    p.Y = reinterpret_cast<uint8_t *>(a.Y);
    p.ldy = a.ldy;
    p.partial = partial;
    p.W = reinterpret_cast<const uint8_t *>(a.W);
    if (a.straddled) {                               // the producers address blocks, not rows: base + block * stride
        p.Wspan = reinterpret_cast<const uint8_t *>(a.Wspan ? a.Wspan : a.W);
        p.span_stride = a.Wspan ? a.span_stride : Q::TS;
    } else {
        p.row_bytes = a.K / Q::BS * Q::TS;
        p.Wspan = reinterpret_cast<const uint8_t *>(a.Wspan);
        p.span_stride = a.span_stride;
    }
    p.loraU = a.lora.T ? reinterpret_cast<const uint16_t *>(a.lora.U) : nullptr;
    p.ldu = a.lora.ldu;
    p.lora_kb = a.lora.kblocks;
    p.lora_tiles = a.lora.tiles;
    p.scale = partial ? nullptr : a.scale;           // split K: the finalize applies it
    p.ftiles = 2 * pl.ftiles;                        // 128-feature halves of the 256-feature item
    p.ttiles = pl.ttiles * pl.accs;                  // TT-token parts of the TT * ACCS-token item
    p.kb_per_split = 4 * pl.spans_per_split;
    p.kb_total = a.straddled ? (int)(a.K / kBlockK) : 4 * (int)((a.K + kSpan - 1) / kSpan);
    if constexpr (Q::BS == 256) {
        if (a.straddled) return wg_launch<Q, Prod, ACT, TT, true, true, SCALED>(tmX, tmX, tmT, p, pl.splits, a.st);
    }
    return wg_launch<Q, Prod, ACT, TT, true, false, SCALED>(tmX, tmX, tmT, p, pl.splits, a.st);
}

template <class Q, class Prod, int ACT, bool SCALED> static int tmem_tiles(const TmemArgs &a, const TmemPlan &pl, float *partial)
{
    if (pl.tt == 32) return tmem_launch<Q, Prod, ACT, 32, SCALED>(a, pl, partial);
    if (pl.tt == 128) return tmem_launch<Q, Prod, ACT, 128, SCALED>(a, pl, partial);
    return tmem_launch<Q, Prod, ACT, 192, SCALED>(a, pl, partial);
}

// does the fused-multiply-add flag change the hand-written producer of this format?  (only Q4_K / Q5_K have a two-rounding step)
template <class Q> struct FmaMatters {
    static constexpr bool value = Q::TS == 144 || Q::TS == 176;
};

template <class Q, int ACT, bool SCALED> static int tmem_run(const TmemArgs &a)
{
    const TmemPlan pl = tmem_plan(a.M, a.N, a.K, a.ws_bytes, a.opt.tile, !a.opt.nosplit);
    float *partial = pl.splits > 1 ? reinterpret_cast<float *>(a.ws) : nullptr;
    // the producer is chosen at compile time where the format leaves no choice, so no kernel is built that cannot be launched
    int rc;
    if constexpr (!FastProducer<Q>::fast) {
        rc = tmem_tiles<Q, Producer<Q>, ACT, SCALED>(a, pl, partial);                 // no hand-written producer for this format
    } else if (a.opt.producers == LinearOptions::GENERIC) {
        rc = tmem_tiles<Q, Producer<Q>, ACT, SCALED>(a, pl, partial);
    } else if constexpr (FmaMatters<Q>::value) {
        rc = a.opt.producers == LinearOptions::EXACT ? tmem_tiles<Q, FastProducer<Q, false>, ACT, SCALED>(a, pl, partial)
                                                     : tmem_tiles<Q, FastProducer<Q, true>, ACT, SCALED>(a, pl, partial);
    } else {
        rc = tmem_tiles<Q, FastProducer<Q, true>, ACT, SCALED>(a, pl, partial);       // single-rounding step: FAST and EXACT coincide
    }
    if (rc != GGUFB200_OK || !partial) return rc;
    return wg_finalize<ACT, SCALED>(partial, pl.splits, a.bias, a.bias_dtype, a.Y, a.M, a.N, a.ldy, a.st, a.scale);
}

// The hand-written producers read the canonical packed rows with 16-byte loads when one row's span and the row stride are
// multiples of 16 B, and K is a whole number of k-blocks (a quarter of a span never reaches past the row); every other
// weight needs the re-packed span-major layout of repack.cu.  A straddled weight has no rows to speak of: its blocks
// (Q4_K 144 B, Q5_K 176 B) must be multiples of 16 B, and K a whole number of k-blocks, so that every k-block of every
// row is one quarter of one block; the others need the block-major copy of repack.cu.
template <class Q> static bool canonical_ok(const void *W, long long N, long long K)
{
    const bool aligned = SpanOf<Q>::BYTES % 16 == 0 && K % kBlockK == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0;
    if (straddled_rows(Q::BS, N, K)) return aligned;
    return aligned && (K / Q::BS * Q::TS) % 16 == 0;
}

bool fused_tmem_supported(int type, const void *W, long long N, long long K)
{
    if (N % 8 != 0 || K % 8 != 0) return false;
    return with_block(type, false, [&](auto blk) { return canonical_ok<decltype(blk)>(W, N, K); });
}

int fused_tmem_linear(int type, const void *W, const void *Wspan, long long span_stride, long long N, long long K, const void *X, long long M,
                      long long ldx, int act_dtype, const void *bias, int bias_dtype, void *Y, long long ldy, void *ws, size_t ws_bytes,
                      const LinearOptions &opt, const LoraOperands &lora, cudaStream_t st, const float *scale)
{
    if (N % 8 != 0 || K % 8 != 0) return GGUFB200_E_UNSUPPORTED;
    return with_block(type, GGUFB200_E_UNSUPPORTED, [&](auto blk) {
        using Q = decltype(blk);
        const bool straddled = straddled_rows(Q::BS, N, K);
        if (straddled && K % kBlockK != 0) return GGUFB200_E_UNSUPPORTED;       // a k-block would span two blocks
        if (!Wspan && !canonical_ok<Q>(W, N, K)) return GGUFB200_E_UNSUPPORTED;
        const TmemArgs a{W, Wspan, span_stride, N, K, X, M, ldx, bias, bias_dtype, Y, ldy, ws, ws_bytes, opt, lora, st, straddled, scale};
        if (scale) return act_dtype == kBF16 ? tmem_run<Q, kBF16, true>(a) : tmem_run<Q, kF16, true>(a);
        return act_dtype == kBF16 ? tmem_run<Q, kBF16, false>(a) : tmem_run<Q, kF16, false>(a);
    });
}

int split_k_finalize(const float *P, int splits, const void *bias, int bias_dtype, void *Y, long long M, long long N, long long ldy, int act_dtype,
                     cudaStream_t st)
{
    return act_dtype == kBF16 ? wg_finalize<kBF16>(P, splits, bias, bias_dtype, Y, M, N, ldy, st)
                              : wg_finalize<kF16>(P, splits, bias, bias_dtype, Y, M, N, ldy, st);
}

}  // namespace ggufb200
