// quantize.cu -- dense fp32 / fp16 / bf16 values -> packed GGUF blocks (ggufb200_quantize), the inverse of K1.
//
// One pass, bound by HBM: algorithmic bytes per element = sizeof(src) read + TS / 32 written.
//   * block formats (Q4_0 ... Q8_0): one tile of 256 blocks (8192 elements) per CTA.  The CTA reads the tile's source span with
//     consecutive 16-byte loads (scalar loads for a source that is not 16-byte aligned), widens it exactly to fp32 and stages it
//     in shared memory one block per 33-float row (the pad keeps both the staging stores and the per-thread row reads free of
//     bank conflicts).  Each thread then quantises one block (quantize.cuh) into the packed output tile in shared memory, and the
//     CTA writes that tile out with consecutive 16-byte stores: every global access of a warp covers whole contiguous lines.
//   * BF16: elementwise, 8 elements per thread with 16-byte loads and stores when both pointers allow them.
//   * K types (ggufb200_quantize_k, Q2_K ... Q6_K): the same staging and stores around a per-group search (quantize_k_kernel
//     below).  Not bound by HBM: the searches run hundreds of separately rounded fp32 operations per element.
// All kernels are launched with programmatic stream serialization, like K1: they wait for the preceding kernel
// (griddepcontrol.wait) before their first global access, and let the next kernel launch (griddepcontrol.launch_dependents)
// only after their last global store, fenced and joined across the CTA (publish_and_release).  A consumer that promises a
// stable source (GGUFB200_DEQUANT_SRC_STABLE, GGUFB200_FLAG_W_STABLE) may read the packed bytes before its own wait, so the
// quantiser must not release it any earlier: its output is a packed weight.
#include "internal.h"
#include "quantize.cuh"

namespace ggufb200 {

namespace {

constexpr int kQThreads = 256;           // blocks per tile = threads per CTA
constexpr int kRow = 33;                 // staged floats per block: 32 + 1 pad

// Every thread's global stores are visible device-wide before any thread of the CTA lets the dependent grid launch.
__device__ __forceinline__ void publish_and_release()
{
    __threadfence();
    __syncthreads();
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

template <int SRC> __device__ __forceinline__ float widen(const void *p, long long i)
{
    if constexpr (SRC == kF32) return reinterpret_cast<const float *>(p)[i];
    else if constexpr (SRC == kF16) return __half2float(reinterpret_cast<const __half *>(p)[i]);
    else return __bfloat162float(reinterpret_cast<const __nv_bfloat16 *>(p)[i]);
}

// 16 bytes of source = 4 (fp32) or 8 (fp16 / bf16) values
template <int SRC> __device__ __forceinline__ void widen16(const uint4 &v, float *f)
{
    if constexpr (SRC == kF32) {
        f[0] = __uint_as_float(v.x), f[1] = __uint_as_float(v.y), f[2] = __uint_as_float(v.z), f[3] = __uint_as_float(v.w);
    } else {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if constexpr (SRC == kF16) {
                f[2 * j] = __half2float(__ushort_as_half((unsigned short)(w[j] & 0xFFFFu)));
                f[2 * j + 1] = __half2float(__ushort_as_half((unsigned short)(w[j] >> 16)));
            } else {
                f[2 * j] = __uint_as_float(w[j] << 16);
                f[2 * j + 1] = __uint_as_float(w[j] & 0xFFFF0000u);
            }
        }
    }
}

// flags: bit 0 = src 16-byte aligned, bit 1 = dst 16-byte aligned
template <class QZ, int SRC>
__global__ void __launch_bounds__(kQThreads) quantize_kernel(const void *__restrict__ src, long long n_blocks, uint8_t *__restrict__ dst,
                                                             int flags)
{
    constexpr int EB = SRC == kF32 ? 4 : 2;              // source bytes per element
    constexpr int VE = 16 / EB;                          // elements per 16-byte load
    constexpr int TILE_BYTES = kQThreads * QZ::TS;       // a multiple of 16: every tile starts 16-byte aligned if dst does
    __shared__ float stage[kQThreads * kRow];
    __shared__ __align__(16) uint8_t otile[TILE_BYTES];

    const int tid = threadIdx.x;
    const long long b0 = (long long)blockIdx.x * kQThreads;
    const int nb = n_blocks - b0 < kQThreads ? (int)(n_blocks - b0) : kQThreads;
    const int n = nb * 32;
    const long long e0 = b0 * 32;

    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (flags & 1) {
        const uint4 *s = reinterpret_cast<const uint4 *>(reinterpret_cast<const uint8_t *>(src) + e0 * EB);
        for (int v = tid; v < n / VE; v += kQThreads) {
            float f[VE];
            widen16<SRC>(__ldg(s + v), f);
            const int e = v * VE;                        // VE divides 32: the vector stays inside one block's row
            float *row = stage + (e >> 5) * kRow + (e & 31);
#pragma unroll
            for (int j = 0; j < VE; ++j) row[j] = f[j];
        }
    } else {
        for (int e = tid; e < n; e += kQThreads) stage[(e >> 5) * kRow + (e & 31)] = widen<SRC>(src, e0 + e);
    }
    __syncthreads();
    if (tid < nb) QZ::run(stage + tid * kRow, otile + tid * QZ::TS);
    __syncthreads();
    const int bytes = nb * QZ::TS;
    uint8_t *out = dst + b0 * QZ::TS;
    int done = 0;
    if (flags & 2) {
        done = bytes & ~15;
        for (int i = tid; i < done / 16; i += kQThreads)
            reinterpret_cast<uint4 *>(out)[i] = reinterpret_cast<const uint4 *>(otile)[i];
    }
    for (int i = done + tid; i < bytes; i += kQThreads) out[i] = otile[i];
    publish_and_release();
}

constexpr int kB16Threads = 256;

// flags: bit 0 = src and dst both 16-byte aligned; dst holds two bytes per element
template <int SRC> __global__ void __launch_bounds__(kB16Threads) bf16_quantize_kernel(const void *__restrict__ src, long long n, uint8_t *__restrict__ dst,
                                                                                     int flags)
{
    constexpr int EB = SRC == kF32 ? 4 : 2;
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const long long i0 = ((long long)blockIdx.x * kB16Threads + threadIdx.x) * 8;
    // threads past the end do not return early: publish_and_release joins the whole CTA
    if ((flags & 1) && i0 + 8 <= n) {
        const uint4 *s = reinterpret_cast<const uint4 *>(reinterpret_cast<const uint8_t *>(src) + i0 * EB);
        float f[8];
        widen16<SRC>(__ldg(s), f);
        if constexpr (SRC == kF32) widen16<SRC>(__ldg(s + 1), f + 4);
        uint32_t w[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) w[j] = bf16_bits_of(f[2 * j]) | (bf16_bits_of(f[2 * j + 1]) << 16);
        *reinterpret_cast<uint4 *>(dst + 2 * i0) = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
        // byte stores: `dst` need not be 2-byte aligned
        const long long end = i0 + 8 < n ? i0 + 8 : n;     // empty for a thread past the end
        for (long long i = i0; i < end; ++i) put16(dst + 2 * i, bf16_bits_of(widen<SRC>(src, i)));
    }
    publish_and_release();
}

// K types: one thread per group of 16 (Q2_K, Q3_K, Q6_K) or 32 (Q4_K, Q5_K) values, so a CTA of 128 threads holds 8 or 16
// super-blocks.  The source tile is staged like the legacy kernel's, one group per padded row.  Each thread runs its group's
// serial search (the sums must stay in the reference's order, so they are not split across lanes); one thread per super-block
// then writes the header (scales, mins, d, dmin); each thread recomputes its group's codes from the quantised header into a
// shared code tile; the CTA packs the code bytes into the output tile and writes it with 16-byte stores.
constexpr int kKThreads = 128;

template <class KQ, int SRC>
__global__ void __launch_bounds__(kKThreads) quantize_k_kernel(const void *__restrict__ src, long long n_blocks, uint8_t *__restrict__ dst,
                                                               int flags)
{
    constexpr int GS = KQ::GS, NG = KQ::NG, SB = kKThreads / NG, ROW = GS + 1;
    constexpr int EB = SRC == kF32 ? 4 : 2;
    constexpr int VE = 16 / EB;                          // divides GS: a vector stays inside one group's row
    constexpr int TILE_BYTES = SB * KQ::TS;              // a multiple of 16 for every K type
    static_assert(TILE_BYTES % 16 == 0 && GS % VE == 0, "tile geometry");
    __shared__ float stage[kKThreads * ROW];
    __shared__ KFit fits[kKThreads];
    __shared__ uint8_t codes[SB * 256];
    __shared__ bool zero[SB];
    __shared__ __align__(16) uint8_t otile[TILE_BYTES];

    const int tid = threadIdx.x;
    const long long b0 = (long long)blockIdx.x * SB;
    const int nb = n_blocks - b0 < SB ? (int)(n_blocks - b0) : SB;
    const int n = nb * 256;
    const long long e0 = b0 * 256;

    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (flags & 1) {
        const uint4 *s = reinterpret_cast<const uint4 *>(reinterpret_cast<const uint8_t *>(src) + e0 * EB);
        for (int v = tid; v < n / VE; v += kKThreads) {
            float f[VE];
            widen16<SRC>(__ldg(s + v), f);
            const int e = v * VE;
            float *row = stage + (e / GS) * ROW + (e % GS);
#pragma unroll
            for (int j = 0; j < VE; ++j) row[j] = f[j];
        }
    } else {
        for (int e = tid; e < n; e += kKThreads) stage[(e / GS) * ROW + (e % GS)] = widen<SRC>(src, e0 + e);
    }
    __syncthreads();
    const int sb = tid / NG, j = tid % NG;
    const bool live = sb < nb;
    const float *x = stage + tid * ROW;
    uint8_t *L = codes + sb * 256 + j * GS;
    if (live) fits[tid] = KQ::fit(x, L);
    __syncthreads();
    if (live && j == 0) zero[sb] = KQ::header(fits + sb * NG, otile + sb * KQ::TS);
    __syncthreads();
    if (live) {
        float d, dm;
        KQ::group_scale(otile + sb * KQ::TS, j, d, dm);
        if (zero[sb]) {
            for (int i = 0; i < GS; ++i) L[i] = 0;
        } else if (d != 0.0f) {
            KQ::codes(x, d, dm, L);
        }
    }
    __syncthreads();
    for (int i = tid; i < nb * KQ::PB; i += kKThreads) {
        const int s = i / KQ::PB, b = i % KQ::PB;
        otile[s * KQ::TS + KQ::PO + b] = KQ::code_byte(codes + s * 256, b);
    }
    __syncthreads();
    const int bytes = nb * KQ::TS;
    uint8_t *out = dst + b0 * KQ::TS;
    int done = 0;
    if (flags & 2) {
        done = bytes & ~15;
        for (int i = tid; i < done / 16; i += kKThreads)
            reinterpret_cast<uint4 *>(out)[i] = reinterpret_cast<const uint4 *>(otile)[i];
    }
    for (int i = done + tid; i < bytes; i += kKThreads) out[i] = otile[i];
    publish_and_release();
}

template <class Kernel, class... Args> int launch_pdl(Kernel kern, long long grid, int threads, cudaStream_t st, Args... args)
{
    if (grid > 0x7fffffffll) return GGUFB200_E_SHAPE;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, args...) == cudaSuccess ? GGUFB200_OK : GGUFB200_E_CUDA;
}

bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <int SRC> int quantize_src(int type, const void *src, long long n_blocks, void *packed, cudaStream_t st)
{
    if (type == T_BF16) {
        const int flags = aligned16(src) && aligned16(packed) ? 1 : 0;
        const long long grid = (n_blocks + 8ll * kB16Threads - 1) / (8ll * kB16Threads);
        return launch_pdl(bf16_quantize_kernel<SRC>, grid, kB16Threads, st, src, n_blocks, reinterpret_cast<uint8_t *>(packed), flags);
    }
    const int flags = (aligned16(src) ? 1 : 0) | (aligned16(packed) ? 2 : 0);
    return with_quant_block(type, (int)GGUFB200_E_TYPE, [&](auto blk) {
        using QZ = decltype(blk);
        const long long grid = (n_blocks + kQThreads - 1) / kQThreads;
        return launch_pdl(quantize_kernel<QZ, SRC>, grid, kQThreads, st, src, n_blocks, reinterpret_cast<uint8_t *>(packed), flags);
    });
}

template <int SRC> int quantize_k_src(int type, const void *src, long long n_blocks, void *packed, cudaStream_t st)
{
    const int flags = (aligned16(src) ? 1 : 0) | (aligned16(packed) ? 2 : 0);
    return with_kquant_block(type, (int)GGUFB200_E_TYPE, [&](auto blk) {
        using KQ = decltype(blk);
        constexpr int SB = kKThreads / KQ::NG;
        const long long grid = (n_blocks + SB - 1) / SB;
        return launch_pdl(quantize_k_kernel<KQ, SRC>, grid, kKThreads, st, src, n_blocks, reinterpret_cast<uint8_t *>(packed), flags);
    });
}

}  // namespace

bool quantize_supported(int type) { return type == T_BF16 || with_quant_block(type, false, [](auto) { return true; }); }

int quantize_dispatch(int type, const void *src, int src_dtype, long long n_blocks, void *packed, cudaStream_t st)
{
    if (n_blocks == 0) return GGUFB200_OK;
    switch (src_dtype) {
    case kF32: return quantize_src<kF32>(type, src, n_blocks, packed, st);
    case kF16: return quantize_src<kF16>(type, src, n_blocks, packed, st);
    case kBF16: return quantize_src<kBF16>(type, src, n_blocks, packed, st);
    }
    return GGUFB200_E_DTYPE;
}

bool quantize_k_supported(int type) { return with_kquant_block(type, false, [](auto) { return true; }); }

int quantize_k_dispatch(int type, const void *src, int src_dtype, long long n_blocks, void *packed, cudaStream_t st)
{
    if (n_blocks == 0) return GGUFB200_OK;
    switch (src_dtype) {
    case kF32: return quantize_k_src<kF32>(type, src, n_blocks, packed, st);
    case kF16: return quantize_k_src<kF16>(type, src, n_blocks, packed, st);
    case kBF16: return quantize_k_src<kBF16>(type, src, n_blocks, packed, st);
    }
    return GGUFB200_E_DTYPE;
}

}  // namespace ggufb200
