// gemm3.cu -- K2, tensor-core GEMM for an already dense weight (DENSE mode of the Linear path, ggufb200_gemm).
//
//   Y[M,N] = X[M,K] * W[N,K]^T (+ bias)      fp16 / bf16, fp32 accumulation
//
// The warpgroup-MMA kernel of linear_sm90.cuh with both operands TMA-fed: one CTA per 128-token x BN-feature output tile.
// A ragged last k-block (K % 64 != 0) is zero-filled by the TMA engine on both operands.
#include "linear_sm90.cuh"

namespace ggufb200 {

template <int ACT, int BN>
static int g3_launch(const void *W, long long N, long long K, long long ldw, const void *X, long long M, long long ldx, const void *bias,
                     int bias_dtype, void *Y, long long ldy, cudaStream_t st)
{
    CUtensorMap tmA, tmB;
    if (!g2_make_map(&tmA, X, M, K, ldx, ACT, 128)) return GGUFB200_E_CUDA;
    if (!g2_make_map(&tmB, W, N, K, ldw, ACT, BN)) return GGUFB200_E_CUDA;
    WgParams p{};
    p.M = M; p.N = N; p.K = K;
    p.bias = bias; p.bias_dtype = bias_dtype;
    p.Y = reinterpret_cast<uint8_t *>(Y); p.ldy = ldy;
    p.ttiles = (int)((M + 127) / 128);
    p.ftiles = (int)((N + BN - 1) / BN);
    p.kb_total = (int)((K + kG2BK - 1) / kG2BK);
    p.kb_per_split = p.kb_total;
    return wg_launch<void, void, ACT, BN, false>(tmA, tmB, tmA, p, 1, st);
}

int gemm3_dense_dispatch(const void *W, long long N, long long K, long long ldw, const void *X, long long M, long long ldx, int act_dtype,
                         const void *bias, int bias_dtype, void *Y, long long ldy, cudaStream_t st)
{
    if (K % 8 != 0 || N % 8 != 0) return GGUFB200_E_UNSUPPORTED;
    // 256-wide feature tiles; 128 when that leaves most SMs idle (short activations such as a 512-token text stream)
    const long long tiles256 = ((M + 127) / 128) * ((N + 255) / 256);
    const bool narrow = tiles256 < sm_count();
    if (narrow)
        return act_dtype == kBF16 ? g3_launch<kBF16, 128>(W, N, K, ldw, X, M, ldx, bias, bias_dtype, Y, ldy, st)
                                  : g3_launch<kF16, 128>(W, N, K, ldw, X, M, ldx, bias, bias_dtype, Y, ldy, st);
    return act_dtype == kBF16 ? g3_launch<kBF16, 256>(W, N, K, ldw, X, M, ldx, bias, bias_dtype, Y, ldy, st)
                              : g3_launch<kF16, 256>(W, N, K, ldw, X, M, ldx, bias, bias_dtype, Y, ldy, st);
}

}  // namespace ggufb200
