// scale.cu -- ggufb200_scale_columns: Y[m, k] = act(fp32(X[m, k]) * c[k]), X / Y fp16 or bf16, c fp32.
//
// The input-axis DoRA factor of the packed-weight Linear (ops.py): x * (W diag(c))^T is computed as (x diag(c)) * W^T, so the
// activation is scaled once per forward and the packed weight is read as it is.  One fp32 multiply and one round-to-nearest per element:
// bit-identical to torch's `(x.float() * c).to(act)`.  Each thread moves 16-byte vectors (8 elements); K % 8 == 0.
#include "internal.h"
#include "wgmma.cuh"

namespace ggufb200 {

template <int ACT>
__global__ void __launch_bounds__(256) scale_columns_kernel(const uint8_t *__restrict__ X, long long ldx, const float *__restrict__ c,
                                                            uint8_t *__restrict__ Y, long long ldy, long long M, long long K)
{
    const long long k8 = K / 8;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < M * k8; i += (long long)gridDim.x * 256) {
        const long long m = i / k8, k = (i % k8) * 8;
        const uint4 x = *reinterpret_cast<const uint4 *>(X + (m * ldx + k) * 2);
        const float4 ca = *reinterpret_cast<const float4 *>(c + k), cb = *reinterpret_cast<const float4 *>(c + k + 4);
        const uint32_t w[4] = {x.x, x.y, x.z, x.w};
        const float s[8] = {ca.x, ca.y, ca.z, ca.w, cb.x, cb.y, cb.z, cb.w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float2 f;
            if constexpr (ACT == kBF16) f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&w[j]));
            else f = __half22float2(*reinterpret_cast<const __half2 *>(&w[j]));
            o[j] = wg_pack<ACT>(__fmul_rn(f.x, s[2 * j]), __fmul_rn(f.y, s[2 * j + 1]));
        }
        st_global_v4(Y + (m * ldy + k) * 2, o[0], o[1], o[2], o[3]);
    }
}

int scale_columns_dispatch(const void *X, long long M, long long K, long long ldx, int act_dtype, const float *col_scale, void *Y,
                           long long ldy, cudaStream_t st)
{
    const long long work = M * (K / 8);
    const long long cap = (long long)sm_count() * 8;
    const unsigned grid = (unsigned)((work + 255) / 256 < cap ? (work + 255) / 256 : cap);
    const uint8_t *x = reinterpret_cast<const uint8_t *>(X);
    uint8_t *y = reinterpret_cast<uint8_t *>(Y);
    if (act_dtype == kBF16) scale_columns_kernel<kBF16><<<grid, 256, 0, st>>>(x, ldx, col_scale, y, ldy, M, K);
    else scale_columns_kernel<kF16><<<grid, 256, 0, st>>>(x, ldx, col_scale, y, ldy, M, K);
    return cudaGetLastError() == cudaSuccess ? GGUFB200_OK : GGUFB200_E_CUDA;
}

}  // namespace ggufb200
