// mma_sync.cuh -- the pieces the two mma.sync Linears share: the small-M GEMV (gemv.cu) and the fused Linear of the
// numpy-fallback types (linear_fallback.cu).
#pragma once
#include "blocks.cuh"

namespace ggufb200 {

// bias value rounded to the activation dtype first: the reference casts the bias to x.dtype
// (ops.py:205-207, bias_dtype = dtype) before F.linear adds it
template <int ACT> __device__ __forceinline__ float load_bias(const void *bias, int bias_dtype, long long n)
{
    float b;
    if (bias_dtype == kF32) b = reinterpret_cast<const float *>(bias)[n];
    else if (bias_dtype == kF16) b = __half2float(reinterpret_cast<const __half *>(bias)[n]);
    else b = __bfloat162float(reinterpret_cast<const __nv_bfloat16 *>(bias)[n]);
    if constexpr (ACT == kBF16) return __bfloat162float(__float2bfloat16_rn(b));
    else return __half2float(__float2half_rn(b));
}

// D (fp32 16 x 8) += A (16 x 16) * B (16 x 8), operands in the activation dtype (legacy HMMA path).  Fragments of thread
// (g = lane / 4, c = lane % 4): a0 / a2 = row g, k pairs 2c and 2c + 8; a1 / a3 = row g + 8, the same k; b0 / b1 = column g,
// k pairs 2c and 2c + 8; d[0], d[1] = (row g, columns 2c, 2c + 1), d[2], d[3] = (row g + 8, the same columns).
template <int ACT> __device__ __forceinline__ void mma_16x8x16(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1)
{
    if constexpr (ACT == kBF16) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    } else {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    }
}

}  // namespace ggufb200
