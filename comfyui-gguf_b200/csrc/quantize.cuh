// quantize.cuh -- dense fp32 values -> packed GGUF blocks, one block per call: the legacy block formats Q4_0, Q4_1, Q5_0, Q5_1,
// Q8_0 and the BF16 element format.  Each functor is gguf-py's `quantize_blocks` (gguf/quants.py) op for op in binary32:
//   * every multiply, add, subtract and divide is its own IEEE round-to-nearest operation (f32_* below; nvcc would otherwise
//     contract x * id + 8.5 into one fused multiply-add), and 1 / d is a true division;
//   * ties in the block reductions resolve the way numpy's do: argmax(|x|) takes the FIRST index, min / max take the LAST of
//     equal values (only the sign of a zero can tell them apart);
//   * float -> uint8 / int8 codes follow numpy's cast on x86-64: truncation to int32 (NaN and out-of-range give INT32_MIN,
//     as cvttss2si does), then the low byte; the codes of a block whose 1 / d overflowed to inf come out 0 this way;
//   * d and m are rounded to fp16 to nearest even, overflow giving inf (numpy's astype(np.float16)).
// The functors are __host__ __device__: tests/host_quantize.cu runs the same lines on the CPU against gguf-py.
#pragma once
#include "blocks.cuh"

namespace ggufb200 {

GG_HD float f32_div(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fdiv_rn(a, b);
#else
    volatile float r = a / b;
    return r;
#endif
}

GG_HD uint32_t f16_bits(float x)
{
    const __half_raw h = __float2half_rn(x);
    return h.x;
}

// numpy's float32 -> (u)int8 cast on x86-64: int32 truncation, then the low byte
GG_HD uint32_t code_byte(float v)
{
    const int32_t i = (v >= -2147483648.0f && v < 2147483648.0f) ? (int32_t)v : INT32_MIN;
    return (uint32_t)i & 0xFFu;
}

GG_HD void put16(uint8_t *o, uint32_t v)
{
    o[0] = (uint8_t)v;
    o[1] = (uint8_t)(v >> 8);
}

// Q4_0 / Q5_0: d = x[argmax |x|] / -2^(BITS-1), codes trunc(x / d + 2^(BITS-1) + 0.5) clipped to [0, 2^BITS - 1]
template <int BITS> GG_HD void quantize_sym(const float *x, uint8_t *o)
{
    constexpr float DIV = BITS == 4 ? -8.0f : -16.0f;
    constexpr float BIAS = BITS == 4 ? 8.5f : 16.5f;
    constexpr uint32_t QMAX = (1u << BITS) - 1;
    float amax = fabsf(x[0]), vmax = x[0];
    for (int i = 1; i < 32; ++i)
        if (fabsf(x[i]) > amax) {
            amax = fabsf(x[i]);
            vmax = x[i];
        }
    const float d = f32_div(vmax, DIV);
    const float id = d == 0.0f ? 0.0f : f32_div(1.0f, d);
    put16(o, f16_bits(d));
    uint8_t *qs = o + (BITS == 4 ? 2 : 6);
    uint32_t qh = 0;
    for (int j = 0; j < 16; ++j) {
        uint32_t lo = code_byte(f32_add(f32_mul(x[j], id), BIAS));
        uint32_t hi = code_byte(f32_add(f32_mul(x[j + 16], id), BIAS));
        lo = lo < QMAX ? lo : QMAX;
        hi = hi < QMAX ? hi : QMAX;
        qs[j] = (uint8_t)((lo & 0xFu) | (hi << 4));
        qh |= ((lo >> 4) & 1u) << j;
        qh |= ((hi >> 4) & 1u) << (j + 16);
    }
    if constexpr (BITS == 5) {
        put16(o + 2, qh);
        put16(o + 4, qh >> 16);
    }
}

// Q4_1 / Q5_1: d = (max - min) / (2^BITS - 1), m = min, codes trunc((x - min) / d + 0.5) clipped to [0, 2^BITS - 1]
template <int BITS> GG_HD void quantize_asym(const float *x, uint8_t *o)
{
    constexpr uint32_t QMAX = (1u << BITS) - 1;
    float mn = x[0], mx = x[0];
    for (int i = 1; i < 32; ++i) {
        if (x[i] <= mn) mn = x[i];
        if (x[i] >= mx) mx = x[i];
    }
    const float d = f32_div(f32_sub(mx, mn), (float)QMAX);
    const float id = d == 0.0f ? 0.0f : f32_div(1.0f, d);
    put16(o, f16_bits(d));
    put16(o + 2, f16_bits(mn));
    uint8_t *qs = o + (BITS == 4 ? 4 : 8);
    uint32_t qh = 0;
    for (int j = 0; j < 16; ++j) {
        uint32_t lo = code_byte(f32_add(f32_mul(f32_sub(x[j], mn), id), 0.5f));
        uint32_t hi = code_byte(f32_add(f32_mul(f32_sub(x[j + 16], mn), id), 0.5f));
        lo = lo < QMAX ? lo : QMAX;
        hi = hi < QMAX ? hi : QMAX;
        qs[j] = (uint8_t)((lo & 0xFu) | (hi << 4));
        qh |= ((lo >> 4) & 1u) << j;
        qh |= ((hi >> 4) & 1u) << (j + 16);
    }
    if constexpr (BITS == 5) {
        put16(o + 4, qh);
        put16(o + 6, qh >> 16);
    }
}

// Q8_0: d = max |x| / 127, codes np_roundf(x / d) (half away from zero, in gguf-py's float sequence) as int8
GG_HD void quantize_q8_0(const float *x, uint8_t *o)
{
    float amax = fabsf(x[0]);
    for (int i = 1; i < 32; ++i)
        if (fabsf(x[i]) > amax) amax = fabsf(x[i]);
    const float d = f32_div(amax, 127.0f);
    const float id = d == 0.0f ? 0.0f : f32_div(1.0f, d);
    put16(o, f16_bits(d));
    for (int j = 0; j < 32; ++j) {
        const float v = f32_mul(x[j], id);
        const float a = fabsf(v);
        const float fl = floorf(a);
        const float b = f32_add(fl, floorf(f32_mul(2.0f, f32_sub(a, fl))));
        const float s = v > 0.0f ? 1.0f : (v < 0.0f ? -1.0f : (v == 0.0f ? 0.0f : v));   // np.sign (NaN stays NaN)
        o[2 + j] = (uint8_t)code_byte(f32_mul(s, b));
    }
}

// BF16: NaN quietened (payload's top bits kept, bit 22 set), then round to nearest even on the top 16 bits
GG_HD uint32_t bf16_bits_of(float x)
{
    uint32_t n;
    memcpy(&n, &x, 4);
    if ((n & 0x7FFFFFFFu) > 0x7F800000u) n = (n & 0xFFFF0000u) | (64u << 16);
    return (n + (0x7FFFu + ((n >> 16) & 1u))) >> 16;     // no carry out of 32 bits: a quietened NaN has a zero low half
}

template <int T> struct QuantBlock;
template <> struct QuantBlock<T_Q4_0> {
    static constexpr int BS = 32, TS = 18;
    static GG_HD void run(const float *x, uint8_t *o) { quantize_sym<4>(x, o); }
};
template <> struct QuantBlock<T_Q5_0> {
    static constexpr int BS = 32, TS = 22;
    static GG_HD void run(const float *x, uint8_t *o) { quantize_sym<5>(x, o); }
};
template <> struct QuantBlock<T_Q4_1> {
    static constexpr int BS = 32, TS = 20;
    static GG_HD void run(const float *x, uint8_t *o) { quantize_asym<4>(x, o); }
};
template <> struct QuantBlock<T_Q5_1> {
    static constexpr int BS = 32, TS = 24;
    static GG_HD void run(const float *x, uint8_t *o) { quantize_asym<5>(x, o); }
};
template <> struct QuantBlock<T_Q8_0> {
    static constexpr int BS = 32, TS = 34;
    static GG_HD void run(const float *x, uint8_t *o) { quantize_q8_0(x, o); }
};

// f(QuantBlock<T>{}) for the block formats above; `fallback` for any other type (BF16 included: it has its own kernel)
template <class R, class F> R with_quant_block(int type, R fallback, F &&f)
{
    switch (type) {
    case T_Q4_0: return f(QuantBlock<T_Q4_0>{});
    case T_Q4_1: return f(QuantBlock<T_Q4_1>{});
    case T_Q5_0: return f(QuantBlock<T_Q5_0>{});
    case T_Q5_1: return f(QuantBlock<T_Q5_1>{});
    case T_Q8_0: return f(QuantBlock<T_Q8_0>{});
    }
    return fallback;
}

}  // namespace ggufb200
