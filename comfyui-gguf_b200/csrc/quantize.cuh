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

// ==================================================================================================================================
// K-quant encoders (Q2_K ... Q6_K, 256-element super-blocks): llama.cpp's reference quantisers at tag b3962 without an importance
// matrix (quantize_row_q{2,3,4,5,6}_K_ref with make_qkx2_quants / make_q3_quants / make_qx_quants / nearest_int), restated so that
// the bytes are a function of the input alone:
//   * every multiply, add, subtract and divide is rounded on its own (f32_*), sums run in the reference's loop order and
//     w * l * l is evaluated left to right; sqrt and division are correctly rounded; fp16 is rounded to nearest even;
//   * nearest_int is the reference's `+ 12582912.f` bit trick, not rintf (they differ once |v| > 2^22).  A NaN argument gives 0:
//     on x86-64 every NaN an operation creates carries the payload 0x400000, which the trick maps to 0 (a device NaN would not).
// The work is cut where the kernel cuts it: a per-group fit (one thread per group of 16 or 32 values), a super-block header step
// (scales, mins, d, dmin), the per-group code pass from the quantised header, and byte-wise packing of the codes.  Each piece is a
// __host__ __device__ function: tests/host_quantize_k.cu runs the same lines on the CPU against a plain-C restatement.
constexpr float kGroupMaxEps = 1e-15f;   // llama.cpp's GROUP_MAX_EPS: a group below this magnitude is all zero

GG_HD float f32_sqrt(float a)
{
#ifdef __CUDA_ARCH__
    return __fsqrt_rn(a);
#else
    volatile float r = sqrtf(a);
    return r;
#endif
}

GG_HD int k_nearest_int(float v)
{
    if (v != v) return 0;
    const float r = f32_add(v, 12582912.0f);
    uint32_t b;
    memcpy(&b, &r, 4);
    return (int)(b & 0x007FFFFFu) - 0x00400000;
}

GG_HD int k_clamp(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
GG_HD float f16_value(uint32_t bits) { return __half2float(__ushort_as_half((unsigned short)bits)); }
GG_HD uint32_t ld16le(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }

// make_qkx2_quants: asymmetric fit of N values to [0, nmax] by a scale and a min, weighted (Q2_K: mean absolute deviation).
// Note that the search steps use the min of the best step so far, as the reference does.
template <int N>
GG_HD float make_qkx2_quants(int nmax, const float *x, const float *w, uint8_t *L, float *the_min, float rmin, float rdelta,
                             int nstep, bool use_mad)
{
    float mn = x[0], mx = x[0];
    float sum_w = w[0];
    float sum_x = f32_mul(sum_w, x[0]);
    for (int i = 1; i < N; ++i) {
        if (x[i] < mn) mn = x[i];
        if (x[i] > mx) mx = x[i];
        sum_w = f32_add(sum_w, w[i]);
        sum_x = f32_add(sum_x, f32_mul(w[i], x[i]));
    }
    if (mn > 0) mn = 0;
    if (mx == mn) {
        for (int i = 0; i < N; ++i) L[i] = 0;
        *the_min = -mn;
        return 0.0f;
    }
    float iscale = f32_div((float)nmax, f32_sub(mx, mn));
    float scale = f32_div(1.0f, iscale);
    float best_mad = 0;
    for (int i = 0; i < N; ++i) {
        L[i] = (uint8_t)k_clamp(k_nearest_int(f32_mul(iscale, f32_sub(x[i], mn))), 0, nmax);
        float diff = f32_sub(f32_add(f32_mul(scale, (float)L[i]), mn), x[i]);
        diff = use_mad ? fabsf(diff) : f32_mul(diff, diff);
        best_mad = f32_add(best_mad, f32_mul(w[i], diff));
    }
    for (int is = 0; is <= nstep; ++is) {
        iscale = f32_div(f32_add(f32_add(rmin, f32_mul(rdelta, (float)is)), (float)nmax), f32_sub(mx, mn));
        float sum_l = 0, sum_l2 = 0, sum_xl = 0;
        uint8_t Laux[N];
        for (int i = 0; i < N; ++i) {
            const int l = k_clamp(k_nearest_int(f32_mul(iscale, f32_sub(x[i], mn))), 0, nmax);
            Laux[i] = (uint8_t)l;
            const float wl = f32_mul(w[i], (float)l);
            sum_l = f32_add(sum_l, wl);
            sum_l2 = f32_add(sum_l2, f32_mul(wl, (float)l));
            sum_xl = f32_add(sum_xl, f32_mul(wl, x[i]));
        }
        const float D = f32_sub(f32_mul(sum_w, sum_l2), f32_mul(sum_l, sum_l));
        if (D > 0) {
            float this_scale = f32_div(f32_sub(f32_mul(sum_w, sum_xl), f32_mul(sum_x, sum_l)), D);
            float this_min = f32_div(f32_sub(f32_mul(sum_l2, sum_x), f32_mul(sum_l, sum_xl)), D);
            if (this_min > 0) {
                this_min = 0;
                this_scale = f32_div(sum_xl, sum_l2);
            }
            float mad = 0;
            for (int i = 0; i < N; ++i) {
                float diff = f32_sub(f32_add(f32_mul(this_scale, (float)Laux[i]), this_min), x[i]);
                diff = use_mad ? fabsf(diff) : f32_mul(diff, diff);
                mad = f32_add(mad, f32_mul(w[i], diff));
            }
            if (mad < best_mad) {
                for (int i = 0; i < N; ++i) L[i] = Laux[i];
                best_mad = mad;
                scale = this_scale;
                mn = this_min;
            }
        }
    }
    *the_min = -mn;
    return scale;
}

// make_q3_quants(n 16, nmax 4, do_rmse): signed fit to [-4, 3] weighted by x^2, refined element by element up to 5 passes
GG_HD float make_q3_quants16(const float *x, uint8_t *L)
{
    constexpr int N = 16, NMAX = 4;
    float mx = 0, amax = 0;
    for (int i = 0; i < N; ++i) {
        const float ax = fabsf(x[i]);
        if (ax > amax) {
            amax = ax;
            mx = x[i];
        }
    }
    if (amax < kGroupMaxEps) {
        for (int i = 0; i < N; ++i) L[i] = 0;
        return 0.0f;
    }
    const float iscale = f32_div((float)-NMAX, mx);
    float sumlx = 0, suml2 = 0;
    int l8[N];
    for (int i = 0; i < N; ++i) {
        const int l = k_clamp(k_nearest_int(f32_mul(iscale, x[i])), -NMAX, NMAX - 1);
        l8[i] = l;
        const float w = f32_mul(x[i], x[i]);
        sumlx = f32_add(sumlx, f32_mul(f32_mul(w, x[i]), (float)l));
        suml2 = f32_add(suml2, f32_mul(f32_mul(w, (float)l), (float)l));
    }
    for (int itry = 0; itry < 5; ++itry) {
        int n_changed = 0;
        for (int i = 0; i < N; ++i) {
            const float w = f32_mul(x[i], x[i]);
            float slx = f32_sub(sumlx, f32_mul(f32_mul(w, x[i]), (float)l8[i]));
            if (slx > 0) {
                float sl2 = f32_sub(suml2, f32_mul(f32_mul(w, (float)l8[i]), (float)l8[i]));
                const int new_l = k_clamp(k_nearest_int(f32_div(f32_mul(x[i], sl2), slx)), -NMAX, NMAX - 1);
                if (new_l != l8[i]) {
                    slx = f32_add(slx, f32_mul(f32_mul(w, x[i]), (float)new_l));
                    sl2 = f32_add(sl2, f32_mul(f32_mul(w, (float)new_l), (float)new_l));
                    if (sl2 > 0 && f32_mul(f32_mul(slx, slx), suml2) > f32_mul(f32_mul(sumlx, sumlx), sl2)) {
                        l8[i] = new_l;
                        sumlx = slx;
                        suml2 = sl2;
                        ++n_changed;
                    }
                }
            }
        }
        if (!n_changed) break;
    }
    for (int i = 0; i < N; ++i) L[i] = (uint8_t)(l8[i] + NMAX);
    return f32_div(sumlx, suml2);
}

// make_qx_quants(n 16, nmax 32, rmse_type 1, no importance weights): signed fit to [-32, 31] weighted by x^2, 18 scale trials
GG_HD float make_qx_quants16(const float *x, uint8_t *L)
{
    constexpr int N = 16, NMAX = 32;
    float mx = 0, amax = 0;
    for (int i = 0; i < N; ++i) {
        const float ax = fabsf(x[i]);
        if (ax > amax) {
            amax = ax;
            mx = x[i];
        }
    }
    if (amax < kGroupMaxEps) {
        for (int i = 0; i < N; ++i) L[i] = 0;
        return 0.0f;
    }
    float iscale = f32_div((float)-NMAX, mx);
    float sumlx = 0, suml2 = 0;
    for (int i = 0; i < N; ++i) {
        const int l = k_clamp(k_nearest_int(f32_mul(iscale, x[i])), -NMAX, NMAX - 1);
        L[i] = (uint8_t)(l + NMAX);
        const float w = f32_mul(x[i], x[i]);
        sumlx = f32_add(sumlx, f32_mul(f32_mul(w, x[i]), (float)l));
        suml2 = f32_add(suml2, f32_mul(f32_mul(w, (float)l), (float)l));
    }
    float scale = suml2 != 0.0f ? f32_div(sumlx, suml2) : 0.0f;
    float best = f32_mul(scale, sumlx);
    for (int is = -9; is <= 9; ++is) {
        if (is == 0) continue;
        iscale = f32_div(-f32_add((float)NMAX, f32_mul(0.1f, (float)is)), mx);
        sumlx = suml2 = 0;
        for (int i = 0; i < N; ++i) {
            const int l = k_clamp(k_nearest_int(f32_mul(iscale, x[i])), -NMAX, NMAX - 1);
            const float w = f32_mul(x[i], x[i]);
            sumlx = f32_add(sumlx, f32_mul(f32_mul(w, x[i]), (float)l));
            suml2 = f32_add(suml2, f32_mul(f32_mul(w, (float)l), (float)l));
        }
        if (suml2 > 0 && f32_mul(sumlx, sumlx) > f32_mul(best, suml2)) {
            for (int i = 0; i < N; ++i) L[i] = (uint8_t)(NMAX + k_clamp(k_nearest_int(f32_mul(iscale, x[i])), -NMAX, NMAX - 1));
            scale = f32_div(sumlx, suml2);
            best = f32_mul(scale, sumlx);
        }
    }
    return scale;
}

struct KFit {
    float scale, min;      // the group's fitted scale and (Q2_K / Q4_K / Q5_K) its negated min
};

// Per type: GS values per group, NG groups per super-block, TS bytes per super-block, and
//   fit(x, L)                 the group search (x: GS values, L: GS codes out)
//   header(fits, o)           the super-block step: quantised scales, d and dmin written into block o; true for a block that
//                             is all zero bytes (Q6_K's early exit)
//   group_scale(o, j, d, dm)  group j's decoded scale (d * sc) and min (dmin * m) from the written header
//   codes(x, d, dm, L)        the final code pass of a group whose decoded scale is not 0
//   code_byte(L, b)           payload byte b (0 .. PB - 1, written at offset PO) from the super-block's 256 codes
template <int T> struct KQuantBlock;

template <> struct KQuantBlock<T_Q2_K> {   // [scales 16][qs 64][d][dmin]
    static constexpr int GS = 16, NG = 16, TS = 84, PO = 16, PB = 64;
    static GG_HD KFit fit(const float *x, uint8_t *L)
    {
        float w[GS];
        for (int l = 0; l < GS; ++l) w[l] = fabsf(x[l]);
        KFit f;
        f.scale = make_qkx2_quants<GS>(3, x, w, L, &f.min, -0.5f, 0.1f, 15, true);
        return f;
    }
    static GG_HD bool header(const KFit *f, uint8_t *o)
    {
        float max_scale = 0, max_min = 0;
        for (int j = 0; j < NG; ++j) {
            if (f[j].scale > max_scale) max_scale = f[j].scale;
            if (f[j].min > max_min) max_min = f[j].min;
        }
        if (max_scale > 0) {
            const float iscale = f32_div(15.0f, max_scale);
            for (int j = 0; j < NG; ++j) o[j] = (uint8_t)k_nearest_int(f32_mul(iscale, f[j].scale));
            put16(o + 80, f16_bits(f32_div(max_scale, 15.0f)));
        } else {
            for (int j = 0; j < NG; ++j) o[j] = 0;
            put16(o + 80, f16_bits(0.0f));
        }
        if (max_min > 0) {
            const float iscale = f32_div(15.0f, max_min);
            for (int j = 0; j < NG; ++j) o[j] = (uint8_t)(o[j] | ((uint32_t)k_nearest_int(f32_mul(iscale, f[j].min)) << 4));
            put16(o + 82, f16_bits(f32_div(max_min, 15.0f)));
        } else {
            put16(o + 82, f16_bits(0.0f));
        }
        return false;
    }
    static GG_HD void group_scale(const uint8_t *o, int j, float &d, float &dm)
    {
        d = f32_mul(f16_value(ld16le(o + 80)), (float)(o[j] & 0xF));
        dm = f32_mul(f16_value(ld16le(o + 82)), (float)(o[j] >> 4));
    }
    static GG_HD void codes(const float *x, float d, float dm, uint8_t *L)
    {
        for (int i = 0; i < GS; ++i) L[i] = (uint8_t)k_clamp(k_nearest_int(f32_div(f32_add(x[i], dm), d)), 0, 3);
    }
    static GG_HD uint8_t code_byte(const uint8_t *L, int b)
    {
        const int j = (b >> 5) * 128, l = b & 31;
        return (uint8_t)(L[j + l] | (L[j + l + 32] << 2) | (L[j + l + 64] << 4) | (L[j + l + 96] << 6));
    }
};

template <> struct KQuantBlock<T_Q3_K> {   // [hmask 32][qs 64][scales 12][d]
    static constexpr int GS = 16, NG = 16, TS = 110, PO = 0, PB = 96;
    static GG_HD KFit fit(const float *x, uint8_t *L)
    {
        KFit f;
        f.scale = make_q3_quants16(x, L);
        f.min = 0;
        return f;
    }
    static GG_HD bool header(const KFit *f, uint8_t *o)
    {
        float max_scale = 0, amax = 0;
        for (int j = 0; j < NG; ++j) {
            const float s = fabsf(f[j].scale);
            if (s > amax) {
                amax = s;
                max_scale = f[j].scale;
            }
        }
        uint8_t *sc = o + 96;
        for (int k = 0; k < 12; ++k) sc[k] = 0;
        if (max_scale != 0.0f) {
            const float iscale = f32_div(-32.0f, max_scale);
            for (int j = 0; j < NG; ++j) {
                int l = (int8_t)k_nearest_int(f32_mul(iscale, f[j].scale));
                l = k_clamp(l, -32, 31) + 32;
                if (j < 8) sc[j] = (uint8_t)(l & 0xF);
                else sc[j - 8] = (uint8_t)(sc[j - 8] | ((l & 0xF) << 4));
                l >>= 4;
                sc[j % 4 + 8] = (uint8_t)(sc[j % 4 + 8] | (l << (2 * (j / 4))));
            }
            put16(o + 108, f16_bits(f32_div(1.0f, iscale)));
        } else {
            put16(o + 108, f16_bits(0.0f));
        }
        return false;
    }
    static GG_HD void group_scale(const uint8_t *o, int j, float &d, float &dm)
    {
        const uint8_t *sc = o + 96;
        int s = j < 8 ? (sc[j] & 0xF) : (sc[j - 8] >> 4);
        s = (int)(int8_t)((s | (((sc[8 + j % 4] >> (2 * (j / 4))) & 3) << 4)) - 32);
        d = f32_mul(f16_value(ld16le(o + 108)), (float)s);
        dm = 0;
    }
    static GG_HD void codes(const float *x, float d, float, uint8_t *L)
    {
        for (int i = 0; i < GS; ++i) L[i] = (uint8_t)(k_clamp(k_nearest_int(f32_div(x[i], d)), -4, 3) + 4);
    }
    static GG_HD uint8_t code_byte(const uint8_t *L, int b)
    {
        if (b < 32) {      // hmask: bit k of byte m is the high bit of code 32 k + m
            uint32_t h = 0;
            for (int k = 0; k < 8; ++k) h |= (L[32 * k + b] > 3 ? 1u : 0u) << k;
            return (uint8_t)h;
        }
        b -= 32;
        const int j = (b >> 5) * 128, l = b & 31;
        auto lo = [&](int i) { return L[i] > 3 ? L[i] - 4 : L[i]; };
        return (uint8_t)(lo(j + l) | (lo(j + l + 32) << 2) | (lo(j + l + 64) << 4) | (lo(j + l + 96) << 6));
    }
};

// Q4_K / Q5_K share the super-block step: 6-bit scales and mins against max / 63, packed as get_scale_min_k4 reads them
template <int NMAX> struct KQuant45 {
    static constexpr int GS = 32, NG = 8;
    static GG_HD KFit fit(const float *x, uint8_t *L)
    {
        float sum_x2 = 0;
        for (int l = 0; l < GS; ++l) sum_x2 = f32_add(sum_x2, f32_mul(x[l], x[l]));
        const float av_x = f32_sqrt(f32_div(sum_x2, 32.0f));
        float w[GS];
        for (int l = 0; l < GS; ++l) w[l] = f32_add(av_x, fabsf(x[l]));
        KFit f;
        f.scale = NMAX == 15 ? make_qkx2_quants<GS>(15, x, w, L, &f.min, -1.0f, 0.1f, 20, false)
                             : make_qkx2_quants<GS>(31, x, w, L, &f.min, -0.5f, 0.1f, 15, false);
        return f;
    }
    static GG_HD bool header(const KFit *f, uint8_t *o)
    {
        float max_scale = 0, max_min = 0;
        for (int j = 0; j < NG; ++j) {
            if (f[j].scale > max_scale) max_scale = f[j].scale;
            if (f[j].min > max_min) max_min = f[j].min;
        }
        const float inv_scale = max_scale > 0 ? f32_div(63.0f, max_scale) : 0.0f;
        const float inv_min = max_min > 0 ? f32_div(63.0f, max_min) : 0.0f;
        uint8_t *sc = o + 4;
        for (int j = 0; j < NG; ++j) {
            uint8_t ls = (uint8_t)k_nearest_int(f32_mul(inv_scale, f[j].scale));
            uint8_t lm = (uint8_t)k_nearest_int(f32_mul(inv_min, f[j].min));
            ls = ls < 63 ? ls : 63;
            lm = lm < 63 ? lm : 63;
            if (j < 4) {
                sc[j] = ls;
                sc[j + 4] = lm;
            } else {
                sc[j + 4] = (uint8_t)((ls & 0xF) | ((lm & 0xF) << 4));
                sc[j - 4] = (uint8_t)(sc[j - 4] | ((ls >> 4) << 6));
                sc[j] = (uint8_t)(sc[j] | ((lm >> 4) << 6));
            }
        }
        put16(o, f16_bits(f32_div(max_scale, 63.0f)));
        put16(o + 2, f16_bits(f32_div(max_min, 63.0f)));
        return false;
    }
    static GG_HD void group_scale(const uint8_t *o, int j, float &d, float &dm)
    {
        const uint8_t *q = o + 4;
        const uint32_t s = j < 4 ? (q[j] & 63u) : ((q[j + 4] & 0xFu) | ((q[j - 4] >> 6) << 4));
        const uint32_t m = j < 4 ? (q[j + 4] & 63u) : ((q[j + 4] >> 4) | ((q[j] >> 6) << 4));
        d = f32_mul(f16_value(ld16le(o)), (float)s);
        dm = f32_mul(f16_value(ld16le(o + 2)), (float)m);
    }
    static GG_HD void codes(const float *x, float d, float dm, uint8_t *L)
    {
        for (int i = 0; i < GS; ++i) L[i] = (uint8_t)k_clamp(k_nearest_int(f32_div(f32_add(x[i], dm), d)), 0, NMAX);
    }
};

template <> struct KQuantBlock<T_Q4_K> : KQuant45<15> {   // [d][dmin][scales 12][qs 128]
    static constexpr int TS = 144, PO = 16, PB = 128;
    static GG_HD uint8_t code_byte(const uint8_t *L, int b)
    {
        const int j = (b >> 5) * 64, l = b & 31;
        return (uint8_t)(L[j + l] | (L[j + l + 32] << 4));
    }
};

template <> struct KQuantBlock<T_Q5_K> : KQuant45<31> {   // [d][dmin][scales 12][qh 32][qs 128]
    static constexpr int TS = 176, PO = 16, PB = 160;
    static GG_HD uint8_t code_byte(const uint8_t *L, int b)
    {
        if (b < 32) {      // qh: bits 2k and 2k + 1 of byte j are the high bits of codes 64 k + j and 64 k + j + 32
            uint32_t h = 0;
            for (int k = 0; k < 4; ++k) {
                h |= (L[64 * k + b] > 15 ? 1u : 0u) << (2 * k);
                h |= (L[64 * k + b + 32] > 15 ? 2u : 0u) << (2 * k);
            }
            return (uint8_t)h;
        }
        b -= 32;
        const int j = (b >> 5) * 64, l = b & 31;
        return (uint8_t)((L[j + l] & 0xF) | ((L[j + l + 32] & 0xF) << 4));
    }
};

template <> struct KQuantBlock<T_Q6_K> {   // [ql 128][qh 64][scales i8 16][d]
    static constexpr int GS = 16, NG = 16, TS = 210, PO = 0, PB = 192;
    static GG_HD KFit fit(const float *x, uint8_t *L)
    {
        KFit f;
        f.scale = make_qx_quants16(x, L);
        f.min = 0;
        return f;
    }
    static GG_HD bool header(const KFit *f, uint8_t *o)
    {
        float max_scale = 0, max_abs_scale = 0;
        for (int j = 0; j < NG; ++j) {
            const float a = fabsf(f[j].scale);
            if (a > max_abs_scale) {
                max_abs_scale = a;
                max_scale = f[j].scale;
            }
        }
        if (max_abs_scale < kGroupMaxEps) {      // the whole block is zero bytes (d included)
            for (int k = 192; k < TS; ++k) o[k] = 0;
            return true;
        }
        const float iscale = f32_div(-128.0f, max_scale);
        put16(o + 208, f16_bits(f32_div(1.0f, iscale)));
        for (int j = 0; j < NG; ++j) {
            const int l = k_nearest_int(f32_mul(iscale, f[j].scale));
            o[192 + j] = (uint8_t)(int8_t)(l < 127 ? l : 127);
        }
        return false;
    }
    static GG_HD void group_scale(const uint8_t *o, int j, float &d, float &dm)
    {
        d = f32_mul(f16_value(ld16le(o + 208)), (float)(int8_t)o[192 + j]);
        dm = 0;
    }
    static GG_HD void codes(const float *x, float d, float, uint8_t *L)
    {
        for (int i = 0; i < GS; ++i) L[i] = (uint8_t)(k_clamp(k_nearest_int(f32_div(x[i], d)), -32, 31) + 32);
    }
    static GG_HD uint8_t code_byte(const uint8_t *L, int b)
    {
        if (b < 128) {     // ql: half h = b / 64; byte r of a half holds codes r and r + 64 (r < 32), r and r + 64 shifted by 32
            const int j = (b >> 6) * 128, r = b & 63;
            return (uint8_t)((L[j + r] & 0xF) | ((L[j + r + 64] & 0xF) << 4));
        }
        b -= 128;
        const int j = (b >> 5) * 128, l = b & 31;
        return (uint8_t)((L[j + l] >> 4) | ((L[j + l + 32] >> 4) << 2) | ((L[j + l + 64] >> 4) << 4) | ((L[j + l + 96] >> 4) << 6));
    }
};

// One super-block, serially: what the kernel does with NG threads and a shared tile.  x: 256 values, o: TS bytes.
template <class KQ> GG_HD void quantize_k_superblock(const float *x, uint8_t *o)
{
    uint8_t L[256];
    KFit f[KQ::NG];
    for (int j = 0; j < KQ::NG; ++j) f[j] = KQ::fit(x + KQ::GS * j, L + KQ::GS * j);
    const bool zero = KQ::header(f, o);
    for (int j = 0; j < KQ::NG; ++j) {
        float d, dm;
        KQ::group_scale(o, j, d, dm);
        if (zero) {
            for (int i = 0; i < KQ::GS; ++i) L[KQ::GS * j + i] = 0;
        } else if (d != 0.0f) {
            KQ::codes(x + KQ::GS * j, d, dm, L + KQ::GS * j);
        }
    }
    for (int b = 0; b < KQ::PB; ++b) o[KQ::PO + b] = KQ::code_byte(L, b);
}

// f(KQuantBlock<T>{}) for the K types; `fallback` for any other type
template <class R, class F> R with_kquant_block(int type, R fallback, F &&f)
{
    switch (type) {
    case T_Q2_K: return f(KQuantBlock<T_Q2_K>{});
    case T_Q3_K: return f(KQuantBlock<T_Q3_K>{});
    case T_Q4_K: return f(KQuantBlock<T_Q4_K>{});
    case T_Q5_K: return f(KQuantBlock<T_Q5_K>{});
    case T_Q6_K: return f(KQuantBlock<T_Q6_K>{});
    }
    return fallback;
}

}  // namespace ggufb200
