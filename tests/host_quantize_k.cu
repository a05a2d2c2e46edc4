// host_quantize_k.cu -- TEST INFRASTRUCTURE: runs the product's K-quant encoder pieces (comfyui-gguf_b200/csrc/quantize.cuh, the
// very code quantize_k_kernel inlines) on the CPU, one super-block at a time, so that `pytest -m "not gpu"` can compare the device
// arithmetic bit for bit with the plain-C restatement in tests/kquant_oracle.c.  Nothing in the product links or loads this file.
#include "../comfyui-gguf_b200/csrc/quantize.cuh"

using namespace ggufb200;

extern "C" {

// x: n_blocks * 256 fp32 values; out: n_blocks * type_size bytes.  Returns -1 for a type that is not a K type.
int hostk_quantize(int type, const float *x, long long n_blocks, uint8_t *out)
{
    return with_kquant_block(type, -1, [&](auto blk) {
        using KQ = decltype(blk);
        for (long long b = 0; b < n_blocks; ++b) quantize_k_superblock<KQ>(x + b * 256, out + b * KQ::TS);
        return 0;
    });
}

}  // extern "C"
