// host_quantize.cu -- TEST INFRASTRUCTURE: runs the product's quantiser functors (comfyui-gguf_b200/csrc/quantize.cuh, the very
// code the quantize kernels inline) on the CPU, so that `pytest -m "not gpu"` can compare the device arithmetic bit for bit with
// gguf-py's `gguf.quants.quantize`.  Nothing in the product links or loads this file.
#include "../comfyui-gguf_b200/csrc/quantize.cuh"

using namespace ggufb200;

extern "C" {

// x: n_blocks * 32 fp32 values (BF16: n_blocks values); out: n_blocks * type_size bytes.  Returns -1 for other types.
int hostq_quantize(int type, const float *x, long long n_blocks, uint8_t *out)
{
    if (type == T_BF16) {
        for (long long i = 0; i < n_blocks; ++i) put16(out + 2 * i, bf16_bits_of(x[i]));
        return 0;
    }
    return with_quant_block(type, -1, [&](auto blk) {
        using QZ = decltype(blk);
        for (long long b = 0; b < n_blocks; ++b) QZ::run(x + b * QZ::BS, out + b * QZ::TS);
        return 0;
    });
}

}  // extern "C"
