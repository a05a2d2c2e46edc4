// host_fallback.cu -- TEST INFRASTRUCTURE: runs the product's decoders of the numpy-fallback types
// (comfyui-gguf_b200/csrc/fallback.cuh, the code the K1 kernel inlines for them) on the CPU, so that `pytest -m "not gpu"`
// compares them bit for bit with gguf-py's `gguf.quants.dequantize` + the torch cast.  Built with -ffp-contract=off, like
// the device code's non-contractible f32_mul / f32_add.  Nothing in the product links or loads this file.
#include "../comfyui-gguf_b200/csrc/fallback.cuh"

using namespace ggufb200;

namespace {

template <class Q, int OUT> int run(const uint8_t *blocks, long long n_blocks, void *out)
{
    for (long long b = 0; b < n_blocks; ++b) {
        for (int e0 = 0; e0 < Q::BS; e0 += 32) {
            float v[32];
            Q::run32(blocks + b * Q::TS, e0, v);
            const long long at = b * Q::BS + e0;
            for (int j = 0; j < 32; j += 2) {
                if constexpr (OUT == kF32) {
                    reinterpret_cast<float *>(out)[at + j] = v[j];
                    reinterpret_cast<float *>(out)[at + j + 1] = v[j + 1];
                } else {
                    reinterpret_cast<uint32_t *>(out)[(at + j) >> 1] = pack16<OUT, kF32>(make_float2(v[j], v[j + 1]));
                }
            }
        }
    }
    return 0;
}

}  // namespace

extern "C" {

// out: n_blocks * BS elements of out_dtype (0 fp16, 1 bf16, 2 fp32); -1 for a type outside fallback.cuh, -2 for a bad dtype
int hostfb_dequant(int type, const uint8_t *blocks, long long n_blocks, void *out, int out_dtype)
{
    return with_fallback_block(type, -1, [&](auto blk) {
        using Q = decltype(blk);
        switch (out_dtype) {
        case kF16: return run<Q, kF16>(blocks, n_blocks, out);
        case kBF16: return run<Q, kBF16>(blocks, n_blocks, out);
        case kF32: return run<Q, kF32>(blocks, n_blocks, out);
        }
        return -2;
    });
}

// block geometry as the decoders declare it
int hostfb_geometry(int type, int *bs, int *ts)
{
    return with_fallback_block(type, -1, [&](auto blk) {
        *bs = decltype(blk)::BS;
        *ts = decltype(blk)::TS;
        return 0;
    });
}

}  // extern "C"
