// repack.cu -- one-time re-layout of a packed GGUF weight into the SPAN-MAJOR shadow layout whose rows the producers of
// GGUFB200_ALGO_FUSED_TMEM (linear_sm90.cu) read with 16-byte loads, whatever the block size is (SURVEY 8f rank 3).
//
// Canonical layout (loader.py:96-120, gguf-py): N rows of K/bs blocks, row stride = K/bs*ts bytes.  Block sizes of
// 84 / 110 / 136 / 210 bytes (Q2_K / Q3_K / IQ4_XS / Q6_K) and row strides that are not multiples of 16 bytes (Q8_0 at
// K = 2432: 2584 B) leave a row's span without 16-byte alignment, so the FUSED_TMEM producers cannot read those weights
// from the canonical rows.  Shadow layout:
//
//     out[s][n][PITCH]      s = 256-wide K-span index (ceil(K/256)), n = row index padded to a multiple of 256,
//                           PITCH = SpanOf<Q>::PITCH >= the span's packed bytes, a multiple of 16 (odd multiple of 16
//                           for the formats that need padding: conflict-free 16-byte shared-memory reads at lane = row)
//
// The 128 rows of one CTA for one span are then 128*PITCH contiguous, 16-byte aligned bytes.  Pad bytes, rows >= N and the
// tail of a ragged last span are zero (a zero block dequantises to 0 in every format).  The canonical bytes stay where
// they are: GGMLTensor / state_dict semantics are untouched, the shadow is a cache the host layer may drop at any time.
//
// A straddled weight (straddled_rows(), internal.h: 256-element blocks, K % 256 != 0) is a flat stream of N*K/256 blocks
// with no row boundaries to keep, so its shadow is BLOCK-major:
//
//     out[b][PITCH]         b = block index < N*K/256, zero padded (no row or span padding)
//
// and the FUSED_TMEM producers read block b at b * PITCH.
#include "internal.h"
#include "produce.cuh"

namespace ggufb200 {

template <int SPAN, int PITCH>
__global__ void __launch_bounds__(256) repack_kernel(const uint8_t *__restrict__ W, long long N, long long n_pad, long long row_bytes, int spans,
                                                     uint8_t *__restrict__ out)
{
    // one thread = one 2-byte unit (every block size and row stride is even): unit u of shadow row (s, n)
    constexpr int UNITS = PITCH / 2;
    const long long total = (long long)spans * n_pad * UNITS;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const int u = (int)(i % UNITS);
        const long long sn = i / UNITS;
        const long long n = sn % n_pad;
        const long long s = sn / n_pad;
        const long long src = s * SPAN + 2 * u;                 // byte offset inside the canonical row
        uint16_t v = 0;
        if (n < N && 2 * u < SPAN && src + 1 < row_bytes) v = *reinterpret_cast<const uint16_t *>(W + n * row_bytes + src);
        reinterpret_cast<uint16_t *>(out)[i] = v;
    }
}

template <class Q> static int repack_run(const void *W, long long N, long long K, void *out, cudaStream_t st)
{
    constexpr int SPAN = SpanOf<Q>::BYTES, PITCH = SpanOf<Q>::PITCH;
    // a straddled weight is copied as N*K/256 one-block "rows" of one span each (SPAN = TS for 256-element blocks)
    const bool straddled = straddled_rows(Q::BS, N, K);
    const long long rows = straddled ? N * K / 256 : N;
    const long long n_pad = straddled ? rows : (N + 255) / 256 * 256;
    const int spans = straddled ? 1 : (int)((K + 255) / 256);
    const long long row_bytes = straddled ? Q::TS : K / Q::BS * Q::TS;
    const long long total = (long long)spans * n_pad * (PITCH / 2);
    long long blocks = (total + 255) / 256;
    const long long cap = (long long)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    repack_kernel<SPAN, PITCH><<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const uint8_t *>(W), rows, n_pad, row_bytes, spans,
                                                                   reinterpret_cast<uint8_t *>(out));
    return cudaGetLastError() == cudaSuccess ? GGUFB200_OK : GGUFB200_E_CUDA;
}

// bytes of the shadow buffer and its geometry; 0 for types without a block layout
size_t repack_bytes(int type, long long N, long long K, int *pitch, long long *span_stride)
{
    int bs = 0;
    const int pt = with_block(type, 0, [&](auto blk) {
        bs = decltype(blk)::BS;
        return SpanOf<decltype(blk)>::PITCH;
    });
    if (pt == 0) return 0;
    if (pitch) *pitch = pt;
    if (straddled_rows(bs, N, K)) {                 // block-major
        if (span_stride) *span_stride = pt;
        return (size_t)(N * K / 256) * (size_t)pt;
    }
    const long long n_pad = (N + 255) / 256 * 256;
    if (span_stride) *span_stride = n_pad * pt;
    return (size_t)((K + 255) / 256) * (size_t)n_pad * (size_t)pt;
}

int repack_dispatch(int type, const void *W, long long N, long long K, void *out, cudaStream_t st)
{
    return with_block(type, GGUFB200_E_TYPE, [&](auto blk) { return repack_run<decltype(blk)>(W, N, K, out, st); });
}

}  // namespace ggufb200
