// common.cuh -- shared device helpers for libggufb200 (sm_90a only).
//
//  * PTX wrappers: mbarrier, 1-D bulk async copy (TMA engine, SASS UBLKCP), vector ld/st
//  * "math policies": the reference (dequant.py) runs every float op as its own torch
//    op in a math dtype and therefore rounds after every op.  Each policy reproduces
//    that bit-exactly on the GPU: F16 -> __h*_rn intrinsics (never contracted into FMA),
//    BF16 -> binary32 op then round-to-bf16, F32 -> __f*_rn intrinsics.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <string.h>

#include "../../include/ggufb200.h"

namespace ggufb200 {

constexpr int kF16 = GGUFB200_F16;
constexpr int kBF16 = GGUFB200_BF16;
constexpr int kF32 = GGUFB200_F32;

// The per-format unpack functors (blocks.cuh) and the math policies below are pure functions of their arguments, so they
// are compiled for the host as well: tests/host_functors.cu runs them on the CPU and compares them bit for bit with the
// oracle, which checks the DEVICE arithmetic without a GPU.  Device code generation is unaffected (same SASS).
#define GG_HD __host__ __device__ __forceinline__

// ------------------------------------------------------------------ PTX: smem / mbarrier / bulk copy
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    while (!mbar_try_wait(bar, parity)) {
    }
}

// 1-D bulk async copy global -> shared, completion signalled on an mbarrier (complete_tx).
// src, dst 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

__device__ __forceinline__ void st_global_v4(void *p, uint32_t a, uint32_t b, uint32_t c, uint32_t d)
{
    asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_shared_v4(uint32_t saddr, uint32_t a, uint32_t b, uint32_t c, uint32_t d)
{
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

GG_HD uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel)
{
#ifdef __CUDA_ARCH__
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
#else
    // PTX prmt.b32, default mode: selector nibble i picks byte (n & 7) of {b, a}; bit 3 replicates that byte's sign
    const uint64_t pool = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) {
        const uint32_t n = (sel >> (4 * i)) & 0xFu;
        uint32_t byte = (uint32_t)(pool >> (8 * (n & 7u))) & 0xFFu;
        if (n & 8u) byte = (byte & 0x80u) ? 0xFFu : 0x00u;
        r |= byte << (8 * i);
    }
    return r;
#endif
}

// round-to-nearest binary32 ops that the compiler may not contract into an fma (device: the _rn intrinsics)
GG_HD float f32_mul(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    volatile float r = a * b;
    return r;
#endif
}
GG_HD float f32_add(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    volatile float r = a + b;
    return r;
#endif
}
GG_HD float f32_sub(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    volatile float r = a - b;
    return r;
#endif
}
GG_HD float f32_from_bits(uint32_t u)
{
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}

// ------------------------------------------------------------------ aligned-as-known loads from a byte pointer
// A = compile-time known alignment of p (1, 2, 4, 8, 16); works for shared and global.
template <int A> GG_HD uint32_t ld32(const uint8_t *p)
{
    if constexpr (A >= 4) {
        return *reinterpret_cast<const uint32_t *>(p);
    } else if constexpr (A == 2) {
        const uint16_t *q = reinterpret_cast<const uint16_t *>(p);
        return (uint32_t)q[0] | ((uint32_t)q[1] << 16);
    } else {
        return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
    }
}
template <int A> GG_HD uint32_t ld16(const uint8_t *p)
{
    if constexpr (A >= 2) {
        return *reinterpret_cast<const uint16_t *>(p);
    } else {
        return (uint32_t)p[0] | ((uint32_t)p[1] << 8);
    }
}

// ------------------------------------------------------------------ math policies
// T  : one value in the math dtype;  T2 : two values.
// cvt4(v, bias, lo, hi): v holds four unsigned bytes u0..u3 (element order = byte order);
//   lo = (u0-bias, u1-bias), hi = (u2-bias, u3-bias), exact in every policy.
template <int MATH> struct Math;

template <> struct Math<kF16> {
    using T = __half;
    using T2 = __half2;
    static GG_HD T from_h(uint32_t bits) { return __ushort_as_half((unsigned short)bits); }
    static GG_HD T from_int(int i) { return __int2half_rn(i); }
    static GG_HD T mul(T a, T b) { return __hmul_rn(a, b); }
    static GG_HD T2 bcast(T a) { return __half2half2(a); }
    static GG_HD T2 mul2(T2 a, T2 b) { return __hmul2_rn(a, b); }
    static GG_HD T2 add2(T2 a, T2 b) { return __hadd2_rn(a, b); }
    static GG_HD T2 sub2(T2 a, T2 b) { return __hsub2_rn(a, b); }
    static GG_HD void cvt4(uint32_t v, int bias, T2 &lo, T2 &hi)
    {
        // bytes -> fp16 (1024 + u) by OR-ing the exponent pattern 0x64, then subtract (1024 + bias): exact
        uint32_t l = prmt(v, 0x64646464u, 0x4140u);
        uint32_t h = prmt(v, 0x64646464u, 0x4342u);
        const __half2 off = __half2half2(__ushort_as_half((unsigned short)(0x6400u + (uint32_t)bias)));
        lo = __hsub2_rn(*reinterpret_cast<__half2 *>(&l), off);
        hi = __hsub2_rn(*reinterpret_cast<__half2 *>(&h), off);
    }
    static GG_HD float2 to_f32x2(T2 a) { return __half22float2(a); }
};

template <int MATH> struct MathF {  // binary32 carrier, rounded to MATH after every op
    using T = float;
    using T2 = float2;
    static GG_HD float r(float x)
    {
        if constexpr (MATH == kBF16) return __bfloat162float(__float2bfloat16_rn(x));
        else return x;
    }
    static GG_HD T from_h(uint32_t bits) { return r(__half2float(__ushort_as_half((unsigned short)bits))); }
    static GG_HD T from_int(int i) { return (float)i; }
    static GG_HD T mul(T a, T b) { return r(f32_mul(a, b)); }
    static GG_HD T2 bcast(T a) { return make_float2(a, a); }
    static GG_HD T2 mul2(T2 a, T2 b) { return make_float2(r(f32_mul(a.x, b.x)), r(f32_mul(a.y, b.y))); }
    static GG_HD T2 add2(T2 a, T2 b) { return make_float2(r(f32_add(a.x, b.x)), r(f32_add(a.y, b.y))); }
    static GG_HD T2 sub2(T2 a, T2 b) { return make_float2(r(f32_sub(a.x, b.x)), r(f32_sub(a.y, b.y))); }
    static GG_HD void cvt4(uint32_t v, int bias, T2 &lo, T2 &hi)
    {
        // bytes -> fp32 (2^23 + u) via exponent pattern 0x4B000000, then subtract (2^23 + bias): exact
        const float off = 8388608.0f + (float)bias;
        lo.x = f32_sub(f32_from_bits(prmt(v, 0x4B000000u, 0x7650u)), off);
        lo.y = f32_sub(f32_from_bits(prmt(v, 0x4B000000u, 0x7651u)), off);
        hi.x = f32_sub(f32_from_bits(prmt(v, 0x4B000000u, 0x7652u)), off);
        hi.y = f32_sub(f32_from_bits(prmt(v, 0x4B000000u, 0x7653u)), off);
    }
    static GG_HD float2 to_f32x2(T2 a) { return a; }
};
template <> struct Math<kBF16> : MathF<kBF16> {};
template <> struct Math<kF32> : MathF<kF32> {};

// final `.to(dtype)` (dequant.py:23): pack a pair of math values into the output dtype
template <int OUT> struct OutT;
template <> struct OutT<kF16> {
    using type = __half;
    static constexpr int bytes = 2;
};
template <> struct OutT<kBF16> {
    using type = __nv_bfloat16;
    static constexpr int bytes = 2;
};
template <> struct OutT<kF32> {
    using type = float;
    static constexpr int bytes = 4;
};

template <int OUT, int MATH> GG_HD uint32_t pack16(typename Math<MATH>::T2 v)
{
    static_assert(OUT != kF32, "pack16 is for 16-bit outputs");
    if constexpr (OUT == kF16 && MATH == kF16) {
        return *reinterpret_cast<uint32_t *>(&v);
    } else {
        float2 f = Math<MATH>::to_f32x2(v);
        if constexpr (OUT == kF16) {
            __half2 h = __floats2half2_rn(f.x, f.y);
            return *reinterpret_cast<uint32_t *>(&h);
        } else {
            __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
            return *reinterpret_cast<uint32_t *>(&b);
        }
    }
}

// Index of the CUDA current device for the per-device caches below, -1 when no device is visible.
inline int device_slot()
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
        cudaGetLastError();
        return -1;
    }
    return dev;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE property of a kernel: raise it once on every device the
// process launches on (a process-wide "done" flag would leave the second GPU of a multi-GPU host at the 48 KB default).
template <class Kernel> inline bool ensure_dynamic_smem(Kernel kern, int bytes, unsigned char (&done)[64])
{
    const int dev = device_slot();
    if (dev < 0) return false;
    if (!done[dev]) {
        if (bytes > 48 * 1024 && cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) return false;
        done[dev] = 1;
    }
    return true;
}

// SM count of the current device, queried once per device (the attribute call is a driver round trip that showed up in the
// host cost of short-activation Linears).  132 (an H100 SXM) when no device is visible (plan tests without a GPU).
inline int sm_count()
{
    static int cache[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
        cudaGetLastError();
        return 132;
    }
    if (cache[dev] == 0) {
        int sms = 132;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) {
            cudaGetLastError();
            sms = 132;
        }
        cache[dev] = sms;
    }
    return cache[dev];
}

}  // namespace ggufb200
