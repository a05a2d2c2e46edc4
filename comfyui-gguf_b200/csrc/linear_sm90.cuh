// linear_sm90.cuh -- the warpgroup-MMA Linear kernel shared by the dense GEMM (gemm3.cu), the smem-fed fused kernel
// (gemm2.cu) and the span-fed fused kernel (gemm4.cu).
//
//   Y[M,N] = X[M,K] * W[N,K]^T (+ bias)      X fp16 / bf16, W dense (TMA) or packed GGUF rows dequantised on chip, fp32 accumulation
//
// One CTA computes one output tile for one K range.  Both operands are K-major 64-wide k-blocks in shared memory in the
// 128-byte swizzle layout: the activation tile is loaded by the TMA engine (zero-filled past M and K), the weight tile either
// by the TMA engine (Q = Prod = void) or by a producer warpgroup that runs Prod::run64 (produce.cuh) on the packed row bytes and
// stores the result in the swizzled layout.  Orientation:
//   TRANS = false   A = 128 activation rows, B = TN weight rows       (D = token x feature)
//   TRANS = true    A = 128 weight rows, B = TN activation rows       (D = feature x token; token tiles of 32 .. 256)
// Warpgroup 0 produces, warpgroups 1 and 2 each own 64 rows of A and issue wgmma.m64nTNk16, keeping one k-block in flight.
// Ring: full[s] (TMA bytes + one arrive per producer warp), empty[s] (one arrive per consumer thread).
// The epilogue either stores fp32 partial sums (split-K, summed by a finalize kernel in a fixed order) or adds the bias,
// rounds to the activation dtype and writes the tile through shared memory with 16-byte stores.
#pragma once
#include <type_traits>

#include "produce.cuh"
#include "wgmma.cuh"

namespace ggufb200 {

constexpr int kWgThreads = 384;

struct WgParams {
    long long M, N, K;
    const void *bias;
    int bias_dtype;
    uint8_t *Y;
    long long ldy;
    float *partial;          // split-K: fp32 [splits, M, N] (nullptr: final output)
    const uint8_t *W;        // canonical packed rows (Prod != void)
    long long row_bytes;
    const uint8_t *Wspan;    // span-major copy (repack.cu) or nullptr
    long long span_stride;   // bytes between consecutive spans of the span-major copy
    const uint16_t *loraU;   // fp16 [N, 64] = scale * up: one extra k-block on the K range 0 (TRANS only)
    int ttiles, ftiles;      // output tiles along tokens / features; CTA = (split, ftile, ttile), token tile fastest
    int kb_per_split, kb_total;
};

template <int TN, bool TRANS> struct WgCfg {
    static constexpr int TOK = TRANS ? TN : 128;
    static constexpr int FEAT = TRANS ? 128 : TN;
    static constexpr int A_BYTES = 128 * 128;
    static constexpr int B_BYTES = TN * 128;
    static constexpr int STAGE = A_BYTES + B_BYTES;
    static constexpr int RAW_STAGES = (227 * 1024 - 2048) / STAGE;
    static constexpr int STAGES = RAW_STAGES > 8 ? 8 : RAW_STAGES;
    static constexpr int YPITCH = FEAT * 2 + 16;                       // epilogue staging row (one token), padded
    static constexpr int SMEM = STAGES * STAGE + 1024 + 256;
    static_assert(TOK * YPITCH <= STAGES * STAGE, "epilogue staging reuses the operand ring");
    static_assert(B_BYTES % 1024 == 0, "swizzled tiles need 1024-byte alignment");
};

template <int ACT> __device__ __forceinline__ uint32_t wg_h2_to_act(uint32_t h)
{
    if constexpr (ACT == kBF16) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&h));
        const __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
        return *reinterpret_cast<const uint32_t *>(&b);
    } else {
        return h;
    }
}

template <class Q, class Prod, int ACT, int TN, bool TRANS>
__global__ void __launch_bounds__(kWgThreads, 1)
wg_linear_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmT,
                 const WgParams p)
{
    using Cfg = WgCfg<TN, TRANS>;
    constexpr bool DENSE = std::is_same<Prod, void>::value;
    constexpr int STAGES = Cfg::STAGES, TOK = Cfg::TOK, FEAT = Cfg::FEAT;
    constexpr int WROWS = TRANS ? 128 : TN;                   // weight rows of a stage

    const int per = p.ftiles * p.ttiles;
    const int split = blockIdx.x / per;
    const int rem = blockIdx.x - split * per;
    const long long feat0 = (long long)(rem / p.ttiles) * FEAT;
    const long long tok0 = (long long)(rem % p.ttiles) * TOK;
    if (tok0 >= p.M || feat0 >= p.N) return;                 // tile of the plan past the edge (uniform over the CTA)
    const int kb0 = split * p.kb_per_split;
    const int nkb_main = min(p.kb_per_split, p.kb_total - kb0);
    const bool lora = p.loraU != nullptr && split == 0;
    const int nkb = nkb_main + (lora ? 1 : 0);

    extern __shared__ uint8_t wg_smem_raw[];
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(wg_smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t *full = reinterpret_cast<uint64_t *>(tiles + STAGES * Cfg::STAGE);
    uint64_t *empty = full + STAGES;

    const int wg = threadIdx.x >> 7;
    const int t = threadIdx.x & 127;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full[s], DENSE ? 1 : 1 + 4);
            mbar_init(&empty[s], 256);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ===================== producer warpgroup
        for (int i = 0; i < nkb; ++i) {
            const int s = i % STAGES;
            mbar_wait(&empty[s], (uint32_t)(((i / STAGES) & 1) ^ 1));
            uint8_t *a_tile = tiles + s * Cfg::STAGE;
            uint8_t *b_tile = a_tile + Cfg::A_BYTES;
            uint8_t *x_tile = TRANS ? b_tile : a_tile;
            uint8_t *w_tile = TRANS ? a_tile : b_tile;
            const int kb = kb0 + i;
            const bool lora_kb = i == nkb_main;                // the extra k-block: X -> T = x * down^T, W -> U = scale * up
            if (t == 0) {
                mbar_arrive_expect_tx(&full[s], TOK * 128 + (DENSE ? WROWS * 128 : 0));
                tma_load_2d(x_tile, lora_kb ? &tmT : &tmX, &full[s], lora_kb ? 0 : kb * kG2BK, (int)tok0);
                if constexpr (DENSE) tma_load_2d(w_tile, &tmW, &full[s], kb * kG2BK, (int)feat0);
            }
            if constexpr (!DENSE) {
#pragma unroll 1
                for (int r = t; r < WROWS; r += 128) {
                    const long long n = feat0 + r;
                    const uint32_t dst = smem_u32(w_tile) + (uint32_t)r * 128;
                    auto emit = [&](int half, const uint32_t (&o)[16]) {
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const int chunk = half * 4 + c;
                            st_shared_v4(dst + (uint32_t)((chunk ^ (r & 7)) << 4), wg_h2_to_act<ACT>(o[4 * c]), wg_h2_to_act<ACT>(o[4 * c + 1]),
                                         wg_h2_to_act<ACT>(o[4 * c + 2]), wg_h2_to_act<ACT>(o[4 * c + 3]));
                        }
                    };
                    if (n >= p.N || (!lora_kb && (long long)kb * kG2BK >= p.K)) {
#pragma unroll
                        for (int c = 0; c < 8; ++c) st_shared_v4(dst + (uint32_t)(c << 4), 0, 0, 0, 0);
                    } else if (lora_kb) {
                        const uint4 *urow = reinterpret_cast<const uint4 *>(p.loraU + n * 64);
#pragma unroll
                        for (int half = 0; half < 2; ++half) {
                            uint32_t o[16];
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                const uint4 v = urow[half * 4 + q];
                                o[4 * q] = v.x; o[4 * q + 1] = v.y; o[4 * q + 2] = v.z; o[4 * q + 3] = v.w;
                            }
                            emit(half, o);
                        }
                    } else {
                        const int span = kb >> 2;
                        const uint8_t *src = p.Wspan ? p.Wspan + (long long)span * p.span_stride + n * SpanOf<Q>::PITCH
                                                     : p.W + n * p.row_bytes + (long long)span * SpanOf<Q>::BYTES;
                        Prod::run64(src, kb & 3, emit);
                    }
                }
                fence_proxy_async_smem();      // generic-proxy stores -> visible to wgmma (async proxy)
                __syncwarp();
                if ((t & 31) == 0) mbar_arrive(&full[s]);
            }
        }
        return;
    }

    // ===================== consumer warpgroups: 64 rows of A each
    const int cw = wg - 1;
    constexpr int NR = TN / 2;
    float acc[NR];
#pragma unroll
    for (int j = 0; j < NR; ++j) acc[j] = 0.f;
    const uint32_t base = smem_u32(tiles);
    for (int i = 0; i < nkb; ++i) {
        const int s = i % STAGES;
        mbar_wait(&full[s], (uint32_t)((i / STAGES) & 1));
        const uint32_t a_addr = base + (uint32_t)(s * Cfg::STAGE) + (uint32_t)(cw * 64 * 128);
        const uint32_t b_addr = base + (uint32_t)(s * Cfg::STAGE + Cfg::A_BYTES);
        const uint64_t da = wg_desc_sw128(a_addr), db = wg_desc_sw128(b_addr);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < kG2BK / 16; ++j) Wgmma<ACT, TN>::mma(acc, da + (uint64_t)(2 * j), db + (uint64_t)(2 * j));
        wgmma_commit();
        if (i > 0) {
            wgmma_wait<1>();                                   // k-block i-1 has been read: hand its stage back
            mbar_arrive(&empty[(i - 1) % STAGES]);
        }
    }
    wgmma_wait<0>();

    const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int arow0 = cw * 64 + warp * 16 + (lane >> 2);
    const int bcol0 = 2 * (lane & 3);
    if (p.partial) {
        float *P = p.partial + (long long)split * p.M * p.N;
#pragma unroll
        for (int j = 0; j < NR / 4; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int ar = arow0 + 8 * h, bc = 8 * j + bcol0 + e;
                    const long long tok = tok0 + (TRANS ? bc : ar), f = feat0 + (TRANS ? ar : bc);
                    if (tok < p.M && f < p.N) P[tok * p.N + f] = acc[4 * j + 2 * h + e];
                }
        return;
    }
    // every wgmma of both consumer warpgroups has completed: the ring is free for the [TOK][FEAT] output tile
    asm volatile("bar.sync 1, 256;" ::: "memory");
    const uint32_t ystage = base;
#pragma unroll
    for (int j = 0; j < NR / 4; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int ar = arow0 + 8 * h, bc = 8 * j + bcol0 + e;
                const int tk = TRANS ? bc : ar, f = TRANS ? ar : bc;
                float v = acc[4 * j + 2 * h + e];
                if (p.bias && feat0 + f < p.N) v += g2_bias<ACT>(p.bias, p.bias_dtype, feat0 + f);
                uint16_t hb;
                if constexpr (ACT == kBF16) hb = __bfloat16_as_ushort(__float2bfloat16_rn(v));
                else hb = __half_as_ushort(__float2half_rn(v));
                asm volatile("st.shared.u16 [%0], %1;" ::"r"(ystage + (uint32_t)(tk * Cfg::YPITCH + f * 2)), "h"(hb) : "memory");
            }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    constexpr int CPR = FEAT / 8;                              // 16-byte chunks per token row
    for (int c = threadIdx.x - 128; c < TOK * CPR; c += 256) {
        const int tk = c / CPR, f = (c % CPR) * 8;
        const long long m = tok0 + tk, n = feat0 + f;
        if (m < p.M && n < p.N) {
            uint32_t a, b, cc, d;
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(cc), "=r"(d) : "r"(ystage + (uint32_t)(tk * Cfg::YPITCH + f * 2)));
            st_global_v4(p.Y + (m * p.ldy + n) * 2, a, b, cc, d);
        }
    }
}

// Launch one CTA per (split, feature tile, token tile).  tmT: LoRA T tile map (or a copy of tmX).
template <class Q, class Prod, int ACT, int TN, bool TRANS>
static int wg_launch(const CUtensorMap &tmX, const CUtensorMap &tmW, const CUtensorMap &tmT, const WgParams &p, int splits, cudaStream_t st)
{
    using Cfg = WgCfg<TN, TRANS>;
    auto kern = wg_linear_kernel<Q, Prod, ACT, TN, TRANS>;
    static unsigned char attr[64] = {};
    if (!ensure_dynamic_smem(kern, Cfg::SMEM, attr)) return GGUFB200_E_CUDA;
    const long long ctas = (long long)p.ftiles * p.ttiles * splits;
    if (ctas <= 0 || ctas > 0x7fffffffll) return GGUFB200_E_SHAPE;
    kern<<<(unsigned)ctas, kWgThreads, Cfg::SMEM, st>>>(tmX, tmW, tmT, p);
    return cudaGetLastError() == cudaSuccess ? GGUFB200_OK : GGUFB200_E_CUDA;
}

// split-K finalize: Y = act(sum_s P[s] + bias), slices added in ascending order (bit-reproducible)
template <int ACT>
__global__ void __launch_bounds__(256) wg_finalize_kernel(const float *__restrict__ P, int splits, const void *__restrict__ bias, int bias_dtype,
                                                          uint8_t *__restrict__ Y, long long M, long long N, long long ldy)
{
    const long long n8 = N / 8;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < M * n8; i += (long long)gridDim.x * 256) {
        const long long m = i / n8, n = (i % n8) * 8;
        float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int sp = 0; sp < splits; ++sp) {
            const float *src = P + ((long long)sp * M + m) * N + n;
            const float4 a = *reinterpret_cast<const float4 *>(src), b = *reinterpret_cast<const float4 *>(src + 4);
            v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w;
            v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
        }
        if (bias) {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] += g2_bias<ACT>(bias, bias_dtype, n + j);
        }
        st_global_v4(Y + (m * ldy + n) * 2, g2_pack<ACT>(v[0], v[1]), g2_pack<ACT>(v[2], v[3]), g2_pack<ACT>(v[4], v[5]), g2_pack<ACT>(v[6], v[7]));
    }
}

template <int ACT>
static int wg_finalize(const float *P, int splits, const void *bias, int bias_dtype, void *Y, long long M, long long N, long long ldy, cudaStream_t st)
{
    const long long work = M * (N / 8);
    const long long cap = (long long)sm_count() * 8;
    const unsigned grid = (unsigned)((work + 255) / 256 < cap ? (work + 255) / 256 : cap);
    wg_finalize_kernel<ACT><<<grid, 256, 0, st>>>(P, splits, bias, bias_dtype, reinterpret_cast<uint8_t *>(Y), M, N, ldy);
    return cudaGetLastError() == cudaSuccess ? GGUFB200_OK : GGUFB200_E_CUDA;
}

}  // namespace ggufb200
