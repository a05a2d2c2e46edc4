// fallback.cuh -- decoders of the eleven GGUF types the reference serves only through gguf-py's numpy fallback
// (reference dequant.py:24-28: `gguf.quants.dequantize`, then `.to(dtype)`): IQ2_XXS, IQ2_XS, IQ2_S, IQ3_XXS, IQ3_S, IQ1_S,
// IQ1_M, TQ1_0, TQ2_0, MXFP4 and NVFP4.
//
// Contract: every value is gguf-py's `dequantize_blocks` of the type, computed in fp32 with its operation order (each product
// rounded on its own: f32_mul, never contracted into an fma), then rounded once to the output dtype by the caller.  There is
// no math-dtype variant: the reference ignores dequant_dtype on this branch.
//
// Interface (one struct per type, `__host__ __device__` like blocks.cuh, so tests/host_fallback.cu checks the same lines on
// the CPU against gguf-py):
//   BS, TS       block size (elements) and type size (bytes)                     gguf-py GGML_QUANT_SIZES
//   A_BLK        alignment of a block's first byte in a 16-byte aligned stream: gcd(TS, 16)
//   run32(b, e0, v)   the 32 consecutive values e0 .. e0 + 31 (e0 % 32 == 0) of the block at `b`, as fp32
// These types are not in GGUFB200_BLOCK_TYPES: the GEMVs, the fused producers and repack work on the integer-pattern
// interface of blocks.cuh (q4 / KIND), which these formats do not have (IQ1 values are not integers).
#pragma once
#include <type_traits>

#include "blocks.cuh"
#include "fallback_tables.h"

namespace ggufb200 {

enum : int {
    T_IQ2_XXS = 16, T_IQ2_XS = 17, T_IQ3_XXS = 18, T_IQ1_S = 19, T_IQ3_S = 21, T_IQ2_S = 22, T_IQ1_M = 29, T_TQ1_0 = 34, T_TQ2_0 = 35,
    T_MXFP4 = 39, T_NVFP4 = 40
};

// The 11 formats, X(T) once each.  Dispatch sites go through with_fallback_block() below.
#define GGUFB200_FALLBACK_TYPES(X) \
    X(T_IQ2_XXS) X(T_IQ2_XS) X(T_IQ2_S) X(T_IQ3_XXS) X(T_IQ3_S) X(T_IQ1_S) X(T_IQ1_M) X(T_TQ1_0) X(T_TQ2_0) X(T_MXFP4) X(T_NVFP4)

// ---------------------------------------------------------------- lookup tables (fallback_tables.h, generated from gguf-py)
// Global memory, read through the read-only data path: the row index differs from thread to thread, which the constant
// cache would serialise.  The host copies serve the CPU build of the decoders.
namespace fbtab {
#define GGUFB200_FB_TABLE(name, T, init) \
    static __device__ const T name##_d[] = init; \
    static const T name##_h[] = init;
GGUFB200_FB_TABLE(iq2xxs, unsigned long long, GGUFB200_GRID_IQ2XXS)
GGUFB200_FB_TABLE(iq2xs, unsigned long long, GGUFB200_GRID_IQ2XS)
GGUFB200_FB_TABLE(iq2s, unsigned long long, GGUFB200_GRID_IQ2S)
GGUFB200_FB_TABLE(iq3xxs, unsigned int, GGUFB200_GRID_IQ3XXS)
GGUFB200_FB_TABLE(iq3s, unsigned int, GGUFB200_GRID_IQ3S)
GGUFB200_FB_TABLE(iq1s, unsigned long long, GGUFB200_GRID_IQ1S)
GGUFB200_FB_TABLE(ksigns, unsigned char, GGUFB200_KSIGNS)
#undef GGUFB200_FB_TABLE
struct Fp4 {
    static constexpr signed char kvalues[16] = GGUFB200_FP4_KVALUES;
};
}  // namespace fbtab

#ifdef __CUDA_ARCH__
#define GGUFB200_FB_LOOKUP(name, i) __ldg(&fbtab::name##_d[(i)])
#else
#define GGUFB200_FB_LOOKUP(name, i) (fbtab::name##_h[(i)])
#endif

GG_HD float f16_bits_to_f32(uint32_t bits) { return __half2float(__ushort_as_half((unsigned short)bits)); }

GG_HD uint32_t f32_to_bits(float f)
{
#ifdef __CUDA_ARCH__
    return __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
#endif
}

// x * (bit ? -1 : 1): exact, so a sign flip (only the sign of a NaN can differ, which is not part of the contract)
GG_HD float negate_if(float x, uint32_t bit) { return f32_from_bits(f32_to_bits(x) ^ (bit << 31)); }

// v[j] = (db * grid[j]) * sign[j] for the 8 unsigned grid values packed in `row` (IQ2 types)
GG_HD void grid8_signed(float *v, float db, unsigned long long row, uint32_t signs)
{
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = negate_if(f32_mul(db, (float)(uint32_t)((row >> (8 * j)) & 0xFFu)), (signs >> j) & 1u);
}

// v[j] = dl * (grid[j] + delta) for the 8 int8 grid values (-1, 0, 1) packed in `row` (IQ1 types)
GG_HD void grid8_delta(float *v, float dl, unsigned long long row, float delta)
{
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = f32_mul(dl, f32_add((float)(int)(signed char)((row >> (8 * j)) & 0xFFu), delta));
}

// MXFP4 / NVFP4 kvalues[idx] (idx 0..15), from two 64-bit words folded at compile time
constexpr unsigned long long fp4_word(int half)
{
    unsigned long long w = 0;
    for (int j = 0; j < 8; ++j) w |= (unsigned long long)(unsigned char)fbtab::Fp4::kvalues[8 * half + j] << (8 * j);
    return w;
}
GG_HD int fp4_value(uint32_t idx)
{
    constexpr unsigned long long lo = fp4_word(0), hi = fp4_word(1);
    return (int)(signed char)((((idx & 8u) ? hi : lo) >> (8 * (idx & 7u))) & 0xFFu);
}

template <int QT> struct Fallback;

// ---------------------------------------------------------------- i-quants with a 2-bit grid (values 8, 25, 43) and ksigns
template <> struct Fallback<T_IQ2_XXS> {  // [d][32 x (u32 grid bytes, u32 signs | scale << 28)]
    static constexpr int BS = 256, TS = 66, A_BLK = 2;
    static GG_HD void run32(const uint8_t *b, int e0, float (&v)[32])
    {
        const int ib = e0 >> 5;
        const float d = f16_bits_to_f32(ld16<2>(b));
        const uint32_t aux0 = ld32<2>(b + 2 + 8 * ib), aux1 = ld32<2>(b + 6 + 8 * ib);
        const float db = f32_mul(f32_mul(d, 0.5f + (float)(aux1 >> 28)), 0.25f);
#pragma unroll
        for (int l = 0; l < 4; ++l)
            grid8_signed(v + 8 * l, db, GGUFB200_FB_LOOKUP(iq2xxs, (aux0 >> (8 * l)) & 255u), GGUFB200_FB_LOOKUP(ksigns, (aux1 >> (7 * l)) & 127u));
    }
};
template <> struct Fallback<T_IQ2_XS> {  // [d][qs u16 x 32: grid | ksigns index << 9][scales 8: a nibble per 16]
    static constexpr int BS = 256, TS = 74, A_BLK = 2;
    static GG_HD void run32(const uint8_t *b, int e0, float (&v)[32])
    {
        const int ib = e0 >> 5;
        const float d = f16_bits_to_f32(ld16<2>(b));
        const uint32_t sc = b[66 + ib];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const float db = f32_mul(f32_mul(d, 0.5f + (float)((sc >> (4 * h)) & 15u)), 0.25f);
#pragma unroll
            for (int l = 0; l < 2; ++l) {
                const uint32_t q = ld16<2>(b + 2 + 2 * (4 * ib + 2 * h + l));
                grid8_signed(v + 16 * h + 8 * l, db, GGUFB200_FB_LOOKUP(iq2xs, q & 511u), GGUFB200_FB_LOOKUP(ksigns, q >> 9));
            }
        }
    }
};
template <> struct Fallback<T_IQ2_S> {  // [d][qs 32][signs 32][qh 8][scales 8]: 10-bit grid index, explicit sign bits
    static constexpr int BS = 256, TS = 82, A_BLK = 2;
    static GG_HD void run32(const uint8_t *b, int e0, float (&v)[32])
    {
        const int ib = e0 >> 5;
        const float d = f16_bits_to_f32(ld16<2>(b));
        const uint32_t sc = b[74 + ib], qh = b[66 + ib];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const float db = f32_mul(f32_mul(d, 0.5f + (float)((sc >> (4 * h)) & 15u)), 0.25f);
#pragma unroll
            for (int l = 0; l < 2; ++l) {
                const int g = 4 * ib + 2 * h + l;
                const uint32_t idx = b[2 + g] | (((qh >> (2 * (2 * h + l))) & 3u) << 8);
                grid8_signed(v + 16 * h + 8 * l, db, GGUFB200_FB_LOOKUP(iq2s, idx), b[34 + g]);
            }
        }
    }
};

// ---------------------------------------------------------------- i-quants with a 3-bit, 4-wide grid
template <> struct Fallback<T_IQ3_XXS> {  // [d][qs 64: grid index per 4][8 x u32: ksigns indices | scale << 28]
    static constexpr int BS = 256, TS = 98, A_BLK = 2;
    static GG_HD void run32(const uint8_t *b, int e0, float (&v)[32])
    {
        const int ib = e0 >> 5;
        const float d = f16_bits_to_f32(ld16<2>(b));
        const uint32_t aux = ld32<2>(b + 66 + 4 * ib);
        const float db = f32_mul(f32_mul(d, 0.5f + (float)(aux >> 28)), 0.5f);
#pragma unroll
        for (int l = 0; l < 4; ++l) {
            const uint32_t signs = GGUFB200_FB_LOOKUP(ksigns, (aux >> (7 * l)) & 127u);
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const uint32_t row = GGUFB200_FB_LOOKUP(iq3xxs, b[2 + 8 * ib + 2 * l + k]);
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    v[8 * l + 4 * k + j] = negate_if(f32_mul(db, (float)((row >> (8 * j)) & 0xFFu)), (signs >> (4 * k + j)) & 1u);
            }
        }
    }
};
template <> struct Fallback<T_IQ3_S> {  // [d][qs 64][qh 8][signs 32][scales 4]: 9-bit grid index, db = d * (1 + 2 * nibble)
    static constexpr int BS = 256, TS = 110, A_BLK = 2;
    static GG_HD void run32(const uint8_t *b, int e0, float (&v)[32])
    {
        const int ib = e0 >> 5;
        const float d = f16_bits_to_f32(ld16<2>(b));
        const float db = f32_mul(d, (float)(1u + 2u * ((b[106 + (ib >> 1)] >> (4 * (ib & 1))) & 15u)));
        const uint32_t qh = b[66 + ib];
#pragma unroll
        for (int g = 0; g < 8; ++g) {
            const uint32_t idx = b[2 + 8 * ib + g] | (((qh >> g) & 1u) << 8);
            const uint32_t row = GGUFB200_FB_LOOKUP(iq3s, idx);
            const uint32_t signs = b[74 + 4 * ib + (g >> 1)] >> (4 * (g & 1));
#pragma unroll
            for (int j = 0; j < 4; ++j) v[4 * g + j] = negate_if(f32_mul(db, (float)((row >> (8 * j)) & 0xFFu)), (signs >> j) & 1u);
        }
    }
};

// ---------------------------------------------------------------- i-quants with the ternary 2048 x 8 grid
template <> struct Fallback<T_IQ1_S> {  // [d][qs 32][qh u16 x 8: 3 index bits per 8, scale bits 12-14, delta sign bit 15]
    static constexpr int BS = 256, TS = 50, A_BLK = 2;
    static GG_HD void run32(const uint8_t *b, int e0, float (&v)[32])
    {
        const int ib = e0 >> 5;
        const float d = f16_bits_to_f32(ld16<2>(b));
        const uint32_t qh = ld16<2>(b + 34 + 2 * ib);
        const float dl = f32_mul(d, (float)(2u * ((qh >> 12) & 7u) + 1u));
        const float delta = (qh & 0x8000u) ? -0.125f : 0.125f;
#pragma unroll
        for (int l = 0; l < 4; ++l)
            grid8_delta(v + 8 * l, dl, GGUFB200_FB_LOOKUP(iq1s, b[2 + 4 * ib + l] | (((qh >> (3 * l)) & 7u) << 8)), delta);
    }
};
template <> struct Fallback<T_IQ1_M> {  // [qs 32][qh 16: a nibble per 8][scales u16 x 4: 3 bits per 16, f16 d in the top nibbles]
    static constexpr int BS = 256, TS = 56, A_BLK = 8;
    static GG_HD void run32(const uint8_t *b, int e0, float (&v)[32])
    {
        const int ib = e0 >> 5;
        const uint32_t s0 = ld16<8>(b + 48), s1 = ld16<2>(b + 50), s2 = ld16<4>(b + 52), s3 = ld16<2>(b + 54);
        const float d = f16_bits_to_f32(((s0 & 0xF000u) >> 12) | ((s1 & 0xF000u) >> 8) | ((s2 & 0xF000u) >> 4) | (s3 & 0xF000u));
        const uint32_t sw = ld16<2>(b + 48 + 2 * (ib >> 1));          // scales of 16-element groups 2 ib, 2 ib + 1
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const float dl = f32_mul(d, (float)(2u * ((sw >> (3 * (2 * (ib & 1) + h))) & 7u) + 1u));
#pragma unroll
            for (int l = 0; l < 2; ++l) {
                const int g = 4 * ib + 2 * h + l;
                const uint32_t nib = (b[32 + (g >> 1)] >> (4 * (g & 1))) & 15u;
                grid8_delta(v + 16 * h + 8 * l, dl, GGUFB200_FB_LOOKUP(iq1s, b[g] | ((nib & 7u) << 8)), (nib & 8u) ? -0.125f : 0.125f);
            }
        }
    }
};

// ---------------------------------------------------------------- ternary types
template <> struct Fallback<T_TQ1_0> {  // [qs 48: 5 trits per byte][qh 4: 4 trits per byte][d]
    static constexpr int BS = 256, TS = 54, A_BLK = 2;
    static GG_HD void run32(const uint8_t *b, int e0, float (&v)[32])
    {
        const float d = f16_bits_to_f32(ld16<2>(b + 52));
        constexpr unsigned long long kPow3 = 0x51ull << 32 | 0x1B090301ull;      // 1, 3, 9, 27, 81
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const int e = e0 + j;
            int at, k;
            if (e < 160) {
                at = e & 31;
                k = e >> 5;
            } else if (e < 240) {
                at = 32 + ((e - 160) & 15);
                k = (e - 160) >> 4;
            } else {
                at = 48 + ((e - 240) & 3);
                k = (e - 240) >> 2;
            }
            // gguf-py multiplies in uint8: the product wraps mod 256 before the trit is taken out of it
            const uint32_t q = (b[at] * (uint32_t)((kPow3 >> (8 * k)) & 0xFFu)) & 0xFFu;
            v[j] = f32_mul(d, (float)((int)((q * 3u) >> 8) - 1));
        }
    }
};
template <> struct Fallback<T_TQ2_0> {  // [qs 64: 4 x 2 bits per byte][d]
    static constexpr int BS = 256, TS = 66, A_BLK = 2;
    static GG_HD void run32(const uint8_t *b, int e0, float (&v)[32])
    {
        const float d = f16_bits_to_f32(ld16<2>(b + 64));
        const uint8_t *qs = b + 32 * (e0 >> 7);
        const int sh = 2 * ((e0 >> 5) & 3);
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = f32_mul(d, (float)((int)((qs[j] >> sh) & 3u) - 1));
    }
};

// ---------------------------------------------------------------- FP4 types: e2m1 nibbles (kvalues, doubled) and a block scale
template <> struct Fallback<T_MXFP4> {  // [e8m0 exponent][qs 16: element j low nibble, j + 16 high nibble]
    static constexpr int BS = 32, TS = 17, A_BLK = 1;
    static GG_HD void run32(const uint8_t *b, int, float (&v)[32])
    {
        // ggml_e8m0_to_fp32_half: half of 2^(e - 127), subnormal at e = 0, 1
        const uint32_t e = b[0];
        const float d = f32_from_bits(e < 2 ? 0x00200000u << e : (e - 1u) << 23);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const uint32_t q = b[1 + j];
            v[j] = f32_mul(d, (float)fp4_value(q & 15u));
            v[16 + j] = f32_mul(d, (float)fp4_value(q >> 4));
        }
    }
};
// gguf-py's NVFP4.ue4m3_to_fp32 (with its factor 0.5): exponent bits 3-6 (bit 7 ignored), 0x00 and 0x7F decode to 0
GG_HD float ue4m3_half(uint32_t x)
{
    if (x == 0u || x == 0x7Fu) return 0.0f;
    const uint32_t e = (x >> 3) & 15u, m = x & 7u;
    return e == 0 ? f32_mul((float)m, 0x1p-10f) : f32_mul((float)(8u + m), f32_from_bits((e + 116u) << 23));      // (8 + m) 2^(e - 11)
}
template <> struct Fallback<T_NVFP4> {  // [ue4m3 scale x 4][qs 4 x 8: sub-block s element i low nibble, i + 8 high nibble]
    static constexpr int BS = 64, TS = 36, A_BLK = 4;
    static GG_HD void run32(const uint8_t *b, int e0, float (&v)[32])
    {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int s = (e0 >> 4) + h;
            const float d = ue4m3_half(b[s]);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const uint32_t q = b[4 + 8 * s + i];
                v[16 * h + i] = f32_mul(d, (float)fp4_value(q & 15u));
                v[16 * h + 8 + i] = f32_mul(d, (float)fp4_value(q >> 4));
            }
        }
    }
};

template <class Q> struct IsFallback : std::false_type {};
template <int QT> struct IsFallback<Fallback<QT>> : std::true_type {};

// Host-side dispatch on a ggml type code: f(Fallback<T>{}) for the 11 formats above, `other` for every other code.
template <class R, class F> R with_fallback_block(int type, R other, F &&f)
{
    switch (type) {
#define GGUFB200_FALLBACK_CASE(T) \
    case T: return f(Fallback<T>{});
        GGUFB200_FALLBACK_TYPES(GGUFB200_FALLBACK_CASE)
#undef GGUFB200_FALLBACK_CASE
    }
    return other;
}

}  // namespace ggufb200
