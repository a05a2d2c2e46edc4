// gemm4.cu -- K2/K3: fused dequant Linear with token tiles sized to the activation (GGUFB200_ALGO_FUSED_TMEM, AUTO's route).
//
//   Y[M,N] = X[M,K] * dequant(W)[N,K]^T (+ bias)      X fp16 / bf16, W packed GGUF blocks, fp32 accumulation
//
// The product is computed TRANSPOSED:  D[feature n, token m] = sum_k W[n,k] * X[m,k], so the token tile is the N dimension of
// the warpgroup MMA and can be as short as the activation (32 / 128 / 192 tokens): the kernel of linear_sm90.cuh with
// A = 128 weight rows that its producer warpgroup dequantises (produce.cuh: hand-written producers for the hot formats, the
// functor producer for the others) and B = the TMA-fed activation tile.  The packed rows are read one 256-wide span at a
// time from the canonical layout (when a row's span and the row stride are multiples of 16 bytes) or from the span-major
// copy of repack.cu (every format).  With bf16 activations the weight is cast to bf16 (the reference's cast before F.linear).
// Work item = (K range, 256-feature tile, token tile); each item is served by 2 * ACCS CTAs (128 features x TT tokens each).
// An optional LoRA update rides as one extra k-block of the K range 0: A = U rows (scale * up), B = T = x * down^T.
// K is processed in whole 256-wide spans: k-blocks past K are zero on both operands.
#include "linear_sm90.cuh"

namespace ggufb200 {

// ------------------------------------------------------------------ host side
struct G4Plan {
    int tt, accs, splits, spans_per_split, ttiles, ftiles, n_items;
};

// Tiling: token tile TT in {32, 128, 192}; ACCS = 2 (384-token items) when asked for; K split into ranges of whole spans
// when the output has fewer CTAs than SMs (short activations; every packed byte is still read once per token tile).
// Cost model (cycles per SM): a CTA of TT tokens x kb k-blocks costs kb * max(4 * TT, 2000) (warpgroup MMA 128 x TT x 64 at
// 2048 FMA per cycle = 4 * TT cycles; ~2000 cycles per k-block is what the producer warpgroup took to dequantise a 128 x 64
// Q4_K weight tile on an H100, read off kernel times at M = 512 and 4608, so the kernel is producer bound at every tile)
// + 3000 (pipeline fill + drain), and the kernel runs ceil(CTAs / SMs) rounds.  Candidates: token tile 32 (M <= 32) / 128 /
// 192 / 384, K cut into 1..32 ranges of whole spans when a workspace for the fp32 partials is available (finalize pass
// charged at 16 bytes / cycle / SM: the slices stay L2 resident).  want_accs: 0 = let the model decide, 1 = force 192-token
// items, 2 = force 384-token items.
static G4Plan g4_plan(long long M, long long N, long long K, size_t ws_bytes, int want_accs, bool allow_split = true)
{
    const int sms = sm_count();
    const int ftiles = (int)((N + 255) / 256);
    const int spans = (int)((K + 255) / 256);
    const size_t slice = (size_t)M * (size_t)N * 4;
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
        if (want_accs == 0 || M <= 192) cands[nc++] = {128, 1};
        if (want_accs != 2 || M <= 192) cands[nc++] = {192, 1};
        if (want_accs != 1 && M > 192) cands[nc++] = {192, 2};
    }
    G4Plan best{};
    double best_cost = 0;
    for (int c = 0; c < nc; ++c) {
        const int tile = cands[c].tt * cands[c].accs;
        const int ttiles = (int)((M + tile - 1) / tile);
        const long long tiles = (long long)ftiles * ttiles;
        for (int s = 1; s <= max_s; ++s) {
            const int per = (spans + s - 1) / s;
            const int splits = (spans + per - 1) / per;
            if (splits != s) continue;                                  // same split count as a smaller s: already evaluated
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

constexpr size_t kG4SplitWsCap = 24u << 20;   // about half of the 50 MB L2 of an H100

// flags: bit 1 (2) = force 384-token items, bit 5 (32) = force 192-token items, bit 2 (4) = no split-K
static int g4_want_accs(int flags) { return (flags & 2) ? 2 : ((flags & 32) ? 1 : 0); }

size_t gemm4_workspace(long long M, long long N, long long K, int flags)
{
    const G4Plan pl = g4_plan(M, N, K, kG4SplitWsCap, g4_want_accs(flags), !(flags & 4));
    return pl.splits > 1 ? (size_t)pl.splits * (size_t)M * (size_t)N * 4 : 0;
}

void gemm4_plan_info(long long M, long long N, long long K, size_t ws_bytes, int flags, int *tile_tokens, int *splits, int *spans_per_split, int *items)
{
    const G4Plan pl = g4_plan(M, N, K, ws_bytes > kG4SplitWsCap ? kG4SplitWsCap : ws_bytes, g4_want_accs(flags), !(flags & 4));
    *tile_tokens = pl.tt * pl.accs;
    *splits = pl.splits;
    *spans_per_split = pl.spans_per_split;
    *items = pl.n_items;
}

struct G4Args {
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
    int fast, want_accs, nosplit;
    const void *loraT;         // LoRA: T = x * down^T, [M, 64] activation dtype, row stride ldt (nullptr: none)
    long long ldt;
    const void *loraU;         // LoRA: U = scale * up, fp16 [N, 64] contiguous
    cudaStream_t st;
};

template <class Q, int ACT, int TT, int PROD>
static int g4_launch(const G4Args &a, const G4Plan &pl, float *partial)
{
    using Prod = typename std::conditional<PROD == 0, Producer<Q>, FastProducer<Q, PROD == 1>>::type;
    CUtensorMap tmX, tmT;
    if (!g2_make_map(&tmX, a.X, a.M, a.K, a.ldx, ACT, TT)) return GGUFB200_E_CUDA;
    tmT = tmX;
    if (a.loraT && !g2_make_map(&tmT, a.loraT, a.M, 64, a.ldt, ACT, TT)) return GGUFB200_E_CUDA;
    WgParams p{};
    p.M = a.M; p.N = a.N; p.K = a.K;
    p.bias = partial ? nullptr : a.bias;
    p.bias_dtype = a.bias_dtype;
    p.Y = reinterpret_cast<uint8_t *>(a.Y);
    p.ldy = a.ldy;
    p.partial = partial;
    p.W = reinterpret_cast<const uint8_t *>(a.W);
    p.row_bytes = a.K / Q::BS * Q::TS;
    p.Wspan = reinterpret_cast<const uint8_t *>(a.Wspan);
    p.span_stride = a.span_stride;
    p.loraU = a.loraT ? reinterpret_cast<const uint16_t *>(a.loraU) : nullptr;
    p.ftiles = 2 * pl.ftiles;                        // 128-feature halves of the 256-feature item
    p.ttiles = pl.ttiles * pl.accs;                  // TT-token parts of the TT * ACCS-token item
    p.kb_per_split = 4 * pl.spans_per_split;
    p.kb_total = 4 * (int)((a.K + 255) / 256);
    return wg_launch<Q, Prod, ACT, TT, true>(tmX, tmX, tmT, p, pl.splits, a.st);
}

template <class Q, int ACT, int PROD> static int g4_tiles(const G4Args &a, const G4Plan &pl, float *partial)
{
    if (pl.tt == 32) return g4_launch<Q, ACT, 32, PROD>(a, pl, partial);
    if (pl.tt == 128) return g4_launch<Q, ACT, 128, PROD>(a, pl, partial);
    return g4_launch<Q, ACT, 192, PROD>(a, pl, partial);
}

// does the fused-multiply-add flag change the hand-written producer of this format?  (only Q4_K / Q5_K have a two-rounding step)
template <class Q> struct FmaMatters {
    static constexpr bool value = Q::TS == 144 || Q::TS == 176;
};

template <class Q, int ACT> static int g4_run(const G4Args &a)
{
    const bool ws_ok = a.ws && (reinterpret_cast<uintptr_t>(a.ws) & 15) == 0;
    size_t wsb = ws_ok ? a.ws_bytes : 0;
    if (wsb > kG4SplitWsCap) wsb = kG4SplitWsCap;
    const G4Plan pl = g4_plan(a.M, a.N, a.K, wsb, a.want_accs, !a.nosplit);
    float *partial = pl.splits > 1 ? reinterpret_cast<float *>(a.ws) : nullptr;
    // a.fast: 0 = generic producers, 1 = hand-written + fused multiply-add, 2 = hand-written + reference sequence
    int rc;
    if (a.fast == 0 || !FastProducer<Q>::fast) {
        rc = g4_tiles<Q, ACT, 0>(a, pl, partial);
    } else if (a.fast == 2) {
        if constexpr (FmaMatters<Q>::value) rc = g4_tiles<Q, ACT, 2>(a, pl, partial);
        else rc = g4_tiles<Q, ACT, 1>(a, pl, partial);
    } else {
        rc = g4_tiles<Q, ACT, 1>(a, pl, partial);
    }
    if (rc != GGUFB200_OK || !partial) return rc;
    return wg_finalize<ACT>(partial, pl.splits, a.bias, a.bias_dtype, a.Y, a.M, a.N, a.ldy, a.st);
}

// The hand-written producers read the canonical packed rows with 16-byte loads when one row's span and the row stride are
// multiples of 16 B, and K is a whole number of k-blocks (a quarter of a span never reaches past the row); every other
// weight needs the re-packed span-major layout of repack.cu
template <class Q> static bool g4_canonical_ok(const void *W, long long K)
{
    const long long row_bytes = K / Q::BS * Q::TS;
    return SpanOf<Q>::BYTES % 16 == 0 && row_bytes % 16 == 0 && K % kG2BK == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0;
}

// flags: bits 0 / 4 = producers (1: hand-written, fused multiply-add; 17: hand-written, reference sequence; 0: generic),
// bit 1 = force 384-token items (ACCS = 2), bit 5 = force 192-token items, bit 2 = no split-K
int gemm4_fused_dispatch(int type, const void *W, const void *Wspan, long long span_stride, long long N, long long K, const void *X, long long M,
                         long long ldx, int act_dtype, const void *bias, int bias_dtype, void *Y, long long ldy, void *ws, size_t ws_bytes,
                         int flags, const void *loraT, long long ldt, const void *loraU, cudaStream_t st)
{
    if (N % 8 != 0 || K % 8 != 0) return GGUFB200_E_UNSUPPORTED;
    G4Args a{W, Wspan, span_stride, N, K, X, M, ldx, bias, bias_dtype, Y, ldy, ws, ws_bytes, (flags & 1) ? ((flags & 16) ? 2 : 1) : 0, (flags & 2) ? 2 : ((flags & 32) ? 1 : 0), (flags & 4) ? 1 : 0,
             loraT, ldt, loraU, st};
#define GGUFB200_G4_CASE(T)                                                                    \
    case T:                                                                                    \
        if (!Wspan && !g4_canonical_ok<Block<T>>(W, K)) return GGUFB200_E_UNSUPPORTED;         \
        return act_dtype == kBF16 ? g4_run<Block<T>, kBF16>(a) : g4_run<Block<T>, kF16>(a);
    switch (type) {
        GGUFB200_G4_CASE(T_Q4_0)
        GGUFB200_G4_CASE(T_Q4_1)
        GGUFB200_G4_CASE(T_Q5_0)
        GGUFB200_G4_CASE(T_Q5_1)
        GGUFB200_G4_CASE(T_Q8_0)
        GGUFB200_G4_CASE(T_Q2_K)
        GGUFB200_G4_CASE(T_Q3_K)
        GGUFB200_G4_CASE(T_Q4_K)
        GGUFB200_G4_CASE(T_Q5_K)
        GGUFB200_G4_CASE(T_Q6_K)
        GGUFB200_G4_CASE(T_IQ4_NL)
        GGUFB200_G4_CASE(T_IQ4_XS)
    }
#undef GGUFB200_G4_CASE
    return GGUFB200_E_UNSUPPORTED;
}

bool gemm4_supported(int type, const void *W, long long N, long long K)
{
    if (N % 8 != 0 || K % 8 != 0) return false;
    switch (type) {
    case T_Q4_0: return g4_canonical_ok<Block<T_Q4_0>>(W, K);
    case T_Q4_1: return g4_canonical_ok<Block<T_Q4_1>>(W, K);
    case T_Q5_0: return g4_canonical_ok<Block<T_Q5_0>>(W, K);
    case T_Q5_1: return g4_canonical_ok<Block<T_Q5_1>>(W, K);
    case T_Q8_0: return g4_canonical_ok<Block<T_Q8_0>>(W, K);
    case T_Q4_K: return g4_canonical_ok<Block<T_Q4_K>>(W, K);
    case T_Q5_K: return g4_canonical_ok<Block<T_Q5_K>>(W, K);
    case T_IQ4_NL: return g4_canonical_ok<Block<T_IQ4_NL>>(W, K);
    }
    return false;
}

}  // namespace ggufb200
