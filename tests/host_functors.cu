// host_functors.cu -- TEST INFRASTRUCTURE: runs the product's per-format unpack functors and math policies
// (comfyui-gguf_b200/csrc/blocks.cuh, common.cuh -- the very code the CUDA kernels inline) on the CPU, so that
// `pytest -m "not gpu"` can compare the device arithmetic bit for bit with the oracle (oracle/gguf_oracle.c), which in turn
// is pinned to the unmodified reference (dequant.py:61-285).  Nothing in the product links or loads this file.
#include <type_traits>

#include "../comfyui-gguf_b200/csrc/produce.cuh"

using namespace ggufb200;

namespace {

template <class Q, int MATH, int OUT> int run_generic(const uint8_t *blocks, long long n_blocks, void *out)
{
    using M = Math<MATH>;
    for (long long b = 0; b < n_blocks; ++b) {
        const uint8_t *blk = blocks + b * Q::TS;
        for (int e0 = 0; e0 < Q::BS; e0 += 8) {
            const GroupScale<MATH> g = group_scale<Q, MATH>(blk, e0);
            typename M::T2 v[4];
            dequant_elems<Q, MATH, 8>(blk, e0, g, v);
            const long long at = b * Q::BS + e0;
            for (int j = 0; j < 4; ++j) {
                if constexpr (OUT == kF32) {
                    const float2 f = M::to_f32x2(v[j]);
                    reinterpret_cast<float *>(out)[at + 2 * j] = f.x;
                    reinterpret_cast<float *>(out)[at + 2 * j + 1] = f.y;
                } else {
                    reinterpret_cast<uint32_t *>(out)[(at >> 1) + j] = pack16<OUT, MATH>(v[j]);
                }
            }
        }
    }
    return 0;
}

template <class Q, int MATH> int run_out(const uint8_t *blocks, long long n, void *out, int out_dtype)
{
    switch (out_dtype) {
    case kF16: return run_generic<Q, MATH, kF16>(blocks, n, out);
    case kBF16: return run_generic<Q, MATH, kBF16>(blocks, n, out);
    case kF32: return run_generic<Q, MATH, kF32>(blocks, n, out);
    }
    return -2;
}

template <class Q> int run_math(const uint8_t *blocks, long long n, void *out, int out_dtype, int math)
{
    switch (math) {
    case kF16: return run_out<Q, kF16>(blocks, n, out, out_dtype);
    case kBF16: return run_out<Q, kBF16>(blocks, n, out, out_dtype);
    case kF32: return run_out<Q, kF32>(blocks, n, out, out_dtype);
    }
    return -2;
}

template <class Q, int ACT> int run_fast16(const uint8_t *blocks, long long n_blocks, uint32_t *out)
{
    if constexpr (!Fast16<Q, ACT>::available) {
        return -8;
    } else {
        for (long long b = 0; b < n_blocks; ++b)
            for (int e0 = 0; e0 < Q::BS; e0 += 16) {
                uint32_t o[8];
                Fast16<Q, ACT>::run(blocks + b * Q::TS, e0, o);
                for (int j = 0; j < 8; ++j) out[(b * Q::BS + e0) / 2 + j] = o[j];
            }
        return 0;
    }
}

// W producers of the fused kernels (produce.cuh): spans of `span_bytes` per row, 16-byte aligned, rows of
// 256 elements; out: fp16 bit patterns, n_spans * 256 elements
template <class Q, int PROD> int run_produce(const uint8_t *spans, long long n_spans, int pitch, uint16_t *out)
{
    using P = typename std::conditional<PROD == 0, Producer<Q>, FastProducer<Q, PROD == 1>>::type;
    for (long long s = 0; s < n_spans; ++s)
        for (int kq = 0; kq < 4; ++kq)
            P::run64(spans + s * pitch, kq, [&](int half, const uint32_t (&o)[16]) {
                uint32_t *dst = reinterpret_cast<uint32_t *>(out + s * 256 + kq * 64 + half * 32);
                for (int j = 0; j < 16; ++j) dst[j] = o[j];
            });
    return 0;
}

}  // namespace

#define HOSTF_TYPES(X) X(T_Q4_0) X(T_Q4_1) X(T_Q5_0) X(T_Q5_1) X(T_Q8_0) X(T_Q2_K) X(T_Q3_K) X(T_Q4_K) X(T_Q5_K) X(T_Q6_K) X(T_IQ4_NL) X(T_IQ4_XS)

extern "C" {

// group_scale + dequant_elems + pack16 over whole blocks (the standalone-dequant arithmetic); out: n_blocks * BS elements
int hostf_dequant(int type, const uint8_t *blocks, long long n_blocks, void *out, int out_dtype, int math_dtype)
{
    switch (type) {
#define X(T) case T: return run_math<Block<T>>(blocks, n_blocks, out, out_dtype, math_dtype);
        HOSTF_TYPES(X)
#undef X
    }
    return -1;
}

// the hand-scheduled 16-element producers of the Linear kernels (fp16 math, activation-dtype output); blocks 16-byte aligned
int hostf_fast16(int type, const uint8_t *blocks, long long n_blocks, uint32_t *out, int act_dtype)
{
    switch (type) {
#define X(T) case T: return act_dtype == kBF16 ? run_fast16<Block<T>, kBF16>(blocks, n_blocks, out) : run_fast16<Block<T>, kF16>(blocks, n_blocks, out);
        HOSTF_TYPES(X)
#undef X
    }
    return -1;
}

// produce.cuh: fast = 0 generic Producer<Q>; 1 hand-written with the fused multiply-add step; 2 hand-written with the reference
// sequence (falls back to the generic one for formats without a hand-written producer).
// Returns 1 when the request was served by a hand-written producer, 0 when by the generic one.
int hostf_produce(int type, const uint8_t *spans, long long n_spans, int pitch, uint16_t *out, int fast)
{
    switch (type) {
#define X(T) case T: if (fast == 1) { run_produce<Block<T>, 1>(spans, n_spans, pitch, out); return FastProducer<Block<T>>::fast ? 1 : 0; } \
                     if (fast == 2) { run_produce<Block<T>, 2>(spans, n_spans, pitch, out); return FastProducer<Block<T>>::fast ? 1 : 0; } \
                     run_produce<Block<T>, 0>(spans, n_spans, pitch, out); return 0;
        HOSTF_TYPES(X)
#undef X
    }
    return -1;
}

// 6-bit scale / min decode and the IQ4 value table, exposed for direct checks
void hostf_k_scale_min(const uint8_t *s12, int j, int *sc, int *mn) { k_scale_min(s12, j, *sc, *mn); }
uint32_t hostf_iq4_lookup4(uint32_t idx4) { return iq4_lookup4(idx4); }
uint32_t hostf_prmt(uint32_t a, uint32_t b, uint32_t sel) { return prmt(a, b, sel); }

}  // extern "C"
