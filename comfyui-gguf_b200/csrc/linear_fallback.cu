// linear_fallback.cu -- GGUFB200_ALGO_FUSED_SYNC: the fused Linear of the numpy-fallback types (fallback.cuh: IQ2_XXS ...
// NVFP4) at prompt-length token counts.
//
//   Y[M, N] = X[M, K] * W[N, K]^T (+ bias)     W decoded from the packed rows in registers, never written to memory
//
// Numerics: every weight element is Fallback<T>::run32's fp32 value (gguf-py's, the values ggufb200_dequant_fallback writes),
// rounded once to the activation dtype, so the weight operand is bit-identical to that kernel's output.  fp32 accumulation;
// the bias is rounded to the activation dtype first (load_bias).
//
// Shape (the mma.sync scheme of gemv.cu, widened to 64 tokens): a CTA = 8 warps x 16 features = 128 features and 64 tokens.
// The K loop runs in steps of 128: thread (g = lane / 4, c = lane % 4) decodes the run of 32 consecutive k
// [128 step + 32 c, +32) of weight rows g and g + 8 of its warp (run32, one header decode per run) into A fragments, and
// reuses them over the 8 token tiles of 8 rows (mma.sync.m16n8k16: 8 MMAs per token tile and step).  The 64 x 128 activation
// chunk of each step is staged in shared memory by 16-byte cp.async, double-buffered, zero-filled past M and K, so the 8 warps
// share one copy; it is fetched while the warps decode the step's weight runs.  Each step's 8 MMAs of a token tile accumulate
// into fresh registers that are added to the fp32 total (the GEMV's per-span partials: a long K is never one tensor-core
// accumulation chain).
// Split K: when the feature x token tile grid does not fill the SMs, K is cut into ranges whose fp32 partial tiles go to the
// caller's workspace and are summed in ascending order by the finalize kernel of linear_sm90.cu (no atomics: reproducible).
#include "fallback.cuh"
#include "internal.h"
#include "mma_sync.cuh"

namespace ggufb200 {

constexpr int kFbThreads = 256;
constexpr int kFbFeat = 16 * (kFbThreads / 32);     // features per CTA: 128
constexpr int kFbTiles = 8;                         // token tiles of 8 rows per CTA
constexpr int kFbTok = 8 * kFbTiles;                // tokens per CTA: 64
constexpr int kFbStep = 128;                        // k per step: 4 lanes x 32
constexpr int kFbRowBytes = kFbStep * 2;            // one staged activation row
constexpr int kFbStage = kFbTok * kFbRowBytes;      // 16 KB per buffer
constexpr int kFbMinSteps = 4;                      // a K range spans at least 512 k
constexpr int kFbMaxSplits = 16;

struct FbParams {
    const uint8_t *W;
    long long row_bytes;
    long long M, N, K;
    const uint8_t *X;
    long long ldx;
    const void *bias;
    int bias_dtype;
    uint8_t *Y;
    long long ldy;
    float *partial;         // split K: fp32 [splits, M, N]; nullptr: final output
    int ftiles, ttiles;     // CTA = (split, feature tile, token tile), token tile fastest (CTAs that read the same rows run together)
    long long steps, steps_per_split;
};

// 16-byte chunk `ch` (0 .. 15) of staged row `row`: bits 0-1 of the chunk index are XOR-ed with (chunk bit 3, row bit 0), so
// the eight 16-byte reads of a quarter warp (g = 0, 1 x c = 0 .. 3, chunk 4 c + j) hit eight different bank groups
__device__ __forceinline__ uint32_t fb_chunk(int row, int ch) { return (uint32_t)(row * kFbRowBytes + ((ch ^ (((ch >> 3) & 1) | ((row & 1) << 1))) * 16)); }

__device__ __forceinline__ void fb_cp_async16(uint32_t dst, const void *src, bool valid)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}

__device__ __forceinline__ uint4 fb_ld_shared_v4(uint32_t addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}

// activation rows m0 .. m0 + 63, k0 .. k0 + 127 into the stage at `sbase`: 1024 chunks of 8 elements, 4 per thread
__device__ __forceinline__ void fb_stage_x(uint32_t sbase, const FbParams &p, long long m0, long long k0, int tid)
{
#pragma unroll
    for (int i = 0; i < kFbTok * (kFbStep / 8) / kFbThreads; ++i) {
        const int q = tid + kFbThreads * i;
        const int row = q >> 4, ch = q & 15;
        const long long m = m0 + row, k = k0 + ch * 8;
        const bool valid = m < p.M && k < p.K;          // K % 8 == 0: a chunk is wholly inside or outside
        fb_cp_async16(sbase + fb_chunk(row, ch), valid ? p.X + (m * p.ldx + k) * 2 : p.X, valid);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

// the 32 weights k .. k + 31 of the row at `row` as 16 activation-dtype pairs (zeros where !ok: past N or past K)
template <class Q, int ACT> __device__ __forceinline__ void fb_decode(const uint8_t *row, long long k, bool ok, uint32_t (&a)[16])
{
    if (ok) {
        float v[32];
        Q::run32(row + (k / Q::BS) * Q::TS, (int)(k % Q::BS), v);
#pragma unroll
        for (int j = 0; j < 16; ++j) a[j] = pack16<ACT, kF32>(make_float2(v[2 * j], v[2 * j + 1]));
    } else {
#pragma unroll
        for (int j = 0; j < 16; ++j) a[j] = 0u;
    }
}

template <class Q, int ACT> __global__ void __launch_bounds__(kFbThreads, 1) fb_linear_kernel(const FbParams p)
{
    __shared__ __align__(128) uint8_t xs[2 * kFbStage];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, c = lane & 3;
    long long cta = blockIdx.x;
    const long long tt = cta % p.ttiles;
    cta /= p.ttiles;
    const long long ft = cta % p.ftiles, split = cta / p.ftiles;
    const long long m0 = tt * kFbTok;
    const long long nA = ft * kFbFeat + warp * 16 + g, nB = nA + 8;
    const bool okA = nA < p.N, okB = nB < p.N;
    const uint8_t *wA = p.W + (okA ? nA : 0) * p.row_bytes, *wB = p.W + (okB ? nB : 0) * p.row_bytes;
    const long long s0 = split * p.steps_per_split;
    const long long s1 = s0 + p.steps_per_split < p.steps ? s0 + p.steps_per_split : p.steps;
    const long long left = p.M - m0;
    const int ntl = left >= kFbTok ? kFbTiles : (int)((left + 7) / 8);     // token tiles with rows (warp-uniform)
    const uint32_t sbase = smem_u32(xs);

    float acc[kFbTiles][4];
#pragma unroll
    for (int t = 0; t < kFbTiles; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;

    fb_stage_x(sbase, p, m0, s0 * kFbStep, tid);
    for (long long step = s0; step < s1; ++step) {
        const uint32_t xb = sbase + (uint32_t)((step - s0) & 1) * kFbStage;
        if (step + 1 < s1) fb_stage_x(sbase + (uint32_t)((step + 1 - s0) & 1) * kFbStage, p, m0, (step + 1) * kFbStep, tid);
        else asm volatile("cp.async.commit_group;" ::: "memory");           // an empty group keeps the wait below uniform
        // K % 32 == 0, so a run is wholly inside or outside K; lanes outside still take part in the warp-wide mma.sync
        const long long k = step * kFbStep + c * 32;
        uint32_t a[16], b[16];
        fb_decode<Q, ACT>(wA, k, okA && k < p.K, a);
        fb_decode<Q, ACT>(wB, k, okB && k < p.K, b);
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncthreads();
#pragma unroll
        for (int t = 0; t < kFbTiles; ++t) {
            if (t < ntl) {
                float sp[4] = {0.f, 0.f, 0.f, 0.f};
                const int row = 8 * t + g;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint4 xv = fb_ld_shared_v4(xb + fb_chunk(row, 4 * c + j));
                    mma_16x8x16<ACT>(sp, a[4 * j], b[4 * j], a[4 * j + 1], b[4 * j + 1], xv.x, xv.y);
                    mma_16x8x16<ACT>(sp, a[4 * j + 2], b[4 * j + 2], a[4 * j + 3], b[4 * j + 3], xv.z, xv.w);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[t][i] += sp[i];
            }
        }
        __syncthreads();        // the next step's cp.async overwrites the buffer just read
    }

    // acc[t]: (feature nA, tokens 2c, 2c + 1 of tile t), (feature nB, the same tokens)
#pragma unroll
    for (int t = 0; t < kFbTiles; ++t) {
        if (t < ntl) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const long long n = i < 2 ? nA : nB, m = m0 + 8 * t + 2 * c + (i & 1);
                if (n < p.N && m < p.M) {
                    if (p.partial) {
                        p.partial[(split * p.M + m) * p.N + n] = acc[t][i];
                    } else {
                        float v = acc[t][i];
                        if (p.bias) v += load_bias<ACT>(p.bias, p.bias_dtype, n);
                        if constexpr (ACT == kBF16) reinterpret_cast<__nv_bfloat16 *>(p.Y)[m * p.ldy + n] = __float2bfloat16_rn(v);
                        else reinterpret_cast<__half *>(p.Y)[m * p.ldy + n] = __float2half_rn(v);
                    }
                }
            }
        }
    }
}

// K ranges for a call with `ws_bytes` of workspace (SIZE_MAX in a query): enough to fill the SMs once when the tile grid does
// not, each range at least kFbMinSteps steps long, no empty range, and as many fp32 [M, N] slices as the workspace holds
static int fb_splits(long long M, long long N, long long K, bool nosplit, size_t ws_bytes)
{
    const long long tiles = ((N + kFbFeat - 1) / kFbFeat) * ((M + kFbTok - 1) / kFbTok);
    const long long steps = (K + kFbStep - 1) / kFbStep;
    const long long sms = sm_count();
    if (nosplit || tiles == 0 || tiles >= sms) return 1;          // tiles == 0: M == 0, nothing to split
    long long s = sms / tiles;
    if (s > steps / kFbMinSteps) s = steps / kFbMinSteps;
    if (s > kFbMaxSplits) s = kFbMaxSplits;
    const size_t slice = (size_t)M * (size_t)N * 4;
    if ((size_t)s > ws_bytes / slice) s = (long long)(ws_bytes / slice);
    if (s < 2) return 1;
    const long long per = (steps + s - 1) / s;
    return (int)((steps + per - 1) / per);
}

size_t fallback_linear_workspace(long long M, long long N, long long K, bool nosplit)
{
    const int s = fb_splits(M, N, K, nosplit, (size_t)-1);
    return s > 1 ? (size_t)s * (size_t)M * (size_t)N * 4 : 0;
}

template <class Q, int ACT> static int fb_launch(const FbParams &p, int splits, cudaStream_t st)
{
    const long long ctas = (long long)p.ftiles * p.ttiles * splits;
    if (ctas <= 0 || ctas > 0x7fffffffll) return GGUFB200_E_SHAPE;
    fb_linear_kernel<Q, ACT><<<(unsigned)ctas, kFbThreads, 0, st>>>(p);
    return cudaGetLastError() == cudaSuccess ? GGUFB200_OK : GGUFB200_E_CUDA;
}

int fallback_linear(int type, const void *W, long long N, long long K, const void *X, long long M, long long ldx, int act_dtype, const void *bias,
                    int bias_dtype, void *Y, long long ldy, void *ws, size_t ws_bytes, bool nosplit, cudaStream_t st)
{
    const int splits = fb_splits(M, N, K, nosplit, ws ? ws_bytes : 0);
    FbParams p{};
    p.W = reinterpret_cast<const uint8_t *>(W);
    p.M = M;
    p.N = N;
    p.K = K;
    p.X = reinterpret_cast<const uint8_t *>(X);
    p.ldx = ldx;
    p.bias = bias;
    p.bias_dtype = bias_dtype;
    p.Y = reinterpret_cast<uint8_t *>(Y);
    p.ldy = ldy;
    p.partial = splits > 1 ? reinterpret_cast<float *>(ws) : nullptr;
    p.ftiles = (int)((N + kFbFeat - 1) / kFbFeat);
    p.ttiles = (int)((M + kFbTok - 1) / kFbTok);
    p.steps = (K + kFbStep - 1) / kFbStep;
    p.steps_per_split = (p.steps + splits - 1) / splits;
    const int rc = with_fallback_block(type, (int)GGUFB200_E_TYPE, [&](auto blk) {
        using Q = decltype(blk);
        p.row_bytes = K / Q::BS * Q::TS;
        return act_dtype == kBF16 ? fb_launch<Q, kBF16>(p, splits, st) : fb_launch<Q, kF16>(p, splits, st);
    });
    if (rc != GGUFB200_OK || splits == 1) return rc;
    return split_k_finalize(p.partial, splits, bias, bias_dtype, Y, M, N, ldy, act_dtype, st);
}

}  // namespace ggufb200
