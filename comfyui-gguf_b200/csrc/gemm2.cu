// gemm2.cu -- K2, fused dequant -> shared memory -> warpgroup MMA (GGUFB200_ALGO_FUSED_MMA, reference-exact weight).
//
//   Y[M,N] = X[M,K] * dequant(W)[N,K]^T (+ bias)      fp16 / bf16 activations, fp32 accumulation
//
// The kernel of linear_sm90.cuh with A = 128 activation rows (TMA) and B = 256 weight rows that its producer warpgroup
// dequantises from the canonical packed rows with the reference's fp16 rounding sequence (Producer<Q>, produce.cuh), so the
// weight operand is bit-identical to what the reference hands to F.linear.  Every block format, any row alignment.
// One CTA per (K range, 128-token x 256-feature tile).
#include "linear_sm90.cuh"

namespace ggufb200 {

constexpr int kG2BM = 128;          // token tile
constexpr int kG2BN = 256;          // feature tile
constexpr int kG2Span = 256;        // K elements of one packed span (= 4 k-blocks): split-K ranges are whole spans

// ------------------------------------------------------------------ host side
// Per-call switch (bit of the `flags` argument; the C ABI passes it inside `algo`, see include/ggufb200.h):
constexpr int kG2NoSplit = 1;     // never cut the K loop into ranges

// Split-K factor of the fused kernel.  Short activations give fewer tiles than half the SMs, so the K loop is cut into S ranges
// of whole 256-wide spans, one CTA per (tile, range), with S * tiles <= SMs (one wave); each CTA stores its fp32 partial tile
// into its own slice of the caller's workspace ([S, M, N] fp32; bounded so the slices stay L2-resident until the finalize
// kernel sums them).  Every packed byte is still read once per token tile.  (The thresholds follow the one-wave rule; they
// have not been tuned by measurement on the H100.)
constexpr size_t kG2SplitWsCap = 24u << 20;   // about half of the 50 MB L2 of an H100

static long long g2_tiles(long long M, long long N) { return ((M + kG2BM - 1) / kG2BM) * ((N + kG2BN - 1) / kG2BN); }

static int g2_fused_splits_ws(long long M, long long N, long long K, size_t ws_bytes, bool allow_split = true)
{
    const size_t slice = (size_t)M * (size_t)N * 4;
    if (ws_bytes > kG2SplitWsCap) ws_bytes = kG2SplitWsCap;
    if (slice == 0 || ws_bytes < 2 * slice || !allow_split || K % kG2Span != 0) return 1;
    const long long sms = sm_count();
    const long long t = g2_tiles(M, N);
    if (t * 2 > sms) return 1;
    const long long spans = K / kG2Span;
    long long s = sms / t;
    if (s > spans) s = spans;
    if (s > 16) s = 16;
    if (s > (long long)(ws_bytes / slice)) s = (long long)(ws_bytes / slice);
    if (s < 2) return 1;
    const long long per = (spans + s - 1) / s;
    return (int)((spans + per - 1) / per);
}

// split-K factor the fused route would use given a workspace (ggufb200_linear_workspace / AUTO routing)
int gemm2_fused_splits(long long M, long long N, long long K) { return g2_fused_splits_ws(M, N, K, kG2SplitWsCap); }

// k-blocks (64 wide) each K range walks: whole 256-wide spans, the last range may be shorter but never empty
static int g2_kb_per_split(long long K, int splits)
{
    if (splits <= 1) return (int)(K / kG2BK);
    const int spans = (int)(K / kG2Span);
    return ((spans + splits - 1) / splits) * 4;
}

// diagnostics (ggufb200_linear_plan): the tiling the fused kernel uses for this problem and workspace size
void gemm2_fused_plan_info(long long M, long long N, long long K, size_t ws_bytes, int flags, int *tile_rows, int *splits, int *kb_per_split, int *ctas)
{
    const int s = g2_fused_splits_ws(M, N, K, ws_bytes, !(flags & kG2NoSplit));
    *tile_rows = kG2BM;
    *splits = s;
    *kb_per_split = g2_kb_per_split(K, s);
    *ctas = (int)(g2_tiles(M, N) * s);
}

template <class Q, int ACT>
static int g2_fused_act(const void *W, long long N, long long K, const void *X, long long M, long long ldx, const void *bias, int bias_dtype,
                        void *Y, long long ldy, void *ws, size_t ws_bytes, int flags, cudaStream_t st)
{
    // split-K needs room for the fp32 [splits, M, N] partial results in the caller's workspace
    const bool ws_ok = ws && (reinterpret_cast<uintptr_t>(ws) & 15) == 0;
    const int splits = g2_fused_splits_ws(M, N, K, ws_ok ? ws_bytes : 0, !(flags & kG2NoSplit));
    float *P = splits > 1 ? reinterpret_cast<float *>(ws) : nullptr;
    CUtensorMap tmA;
    if (!g2_make_map(&tmA, X, M, K, ldx, ACT, kG2BM)) return GGUFB200_E_CUDA;
    WgParams p{};
    p.M = M; p.N = N; p.K = K;
    p.bias = P ? nullptr : bias; p.bias_dtype = bias_dtype;
    p.Y = reinterpret_cast<uint8_t *>(Y); p.ldy = ldy;
    p.partial = P;
    p.W = reinterpret_cast<const uint8_t *>(W);
    p.row_bytes = K / Q::BS * Q::TS;
    p.ttiles = (int)((M + kG2BM - 1) / kG2BM);
    p.ftiles = (int)((N + kG2BN - 1) / kG2BN);
    p.kb_total = (int)(K / kG2BK);
    p.kb_per_split = g2_kb_per_split(K, splits);
    int rc = wg_launch<Q, Producer<Q>, ACT, kG2BN, false>(tmA, tmA, tmA, p, splits, st);
    if (rc != GGUFB200_OK || !P) return rc;
    return wg_finalize<ACT>(P, splits, bias, bias_dtype, Y, M, N, ldy, st);
}

int gemm2_fused_dispatch(int type, const void *W, long long N, long long K, const void *X, long long M, long long ldx, int act_dtype,
                         int math_dtype, const void *bias, int bias_dtype, void *Y, long long ldy, void *ws, size_t ws_bytes, int flags,
                         cudaStream_t st)
{
    if (math_dtype != kF16 || K % kG2BK != 0 || N % 8 != 0) return GGUFB200_E_UNSUPPORTED;
#define GGUFB200_G2_CASE(T)                                                                                               \
    case T:                                                                                                               \
        return act_dtype == kBF16 ? g2_fused_act<Block<T>, kBF16>(W, N, K, X, M, ldx, bias, bias_dtype, Y, ldy, ws, ws_bytes, flags, st)  \
                                  : g2_fused_act<Block<T>, kF16>(W, N, K, X, M, ldx, bias, bias_dtype, Y, ldy, ws, ws_bytes, flags, st);
    switch (type) {
        GGUFB200_G2_CASE(T_Q4_0)
        GGUFB200_G2_CASE(T_Q4_1)
        GGUFB200_G2_CASE(T_Q5_0)
        GGUFB200_G2_CASE(T_Q5_1)
        GGUFB200_G2_CASE(T_Q8_0)
        GGUFB200_G2_CASE(T_Q2_K)
        GGUFB200_G2_CASE(T_Q3_K)
        GGUFB200_G2_CASE(T_Q4_K)
        GGUFB200_G2_CASE(T_Q5_K)
        GGUFB200_G2_CASE(T_Q6_K)
        GGUFB200_G2_CASE(T_IQ4_NL)
        GGUFB200_G2_CASE(T_IQ4_XS)
    }
#undef GGUFB200_G2_CASE
    return GGUFB200_E_UNSUPPORTED;
}

}  // namespace ggufb200
