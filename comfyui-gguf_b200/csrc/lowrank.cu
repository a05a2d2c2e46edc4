// lowrank.cu -- K1 with LoRA / LoCon and LoHa patches: the patched [N, K] weight in one launch (ggufb200_dequant_lowrank).
//
// Replaces, for a Conv2d whose weight carries LoRA / LoHa patches, the reference's dequantise + comfy.lora.calculate_weight
// (an fp32 torch.mm writing a full-size fp32 delta, a scale, a cast and an in-place add).  The weight is the logical matrix
// [N, K] = [Cout, Cin * kh * kw] of the flat block stream, so a straddled SD1.5 / SDXL K-quant conv (K % 256 != 0) is read the
// same way as any other.
//
// One CTA = one 2-D tile of kRows x kCols weight elements:
//   * the packed bytes of the tile's row segments are staged into shared memory (one 16-byte aligned slot per row, the block
//     bytes keeping their stream alignment mod 16, as the unpackers of blocks.cuh expect) and unpacked run by run (32 elements
//     per thread, K % 32 == 0 so a run never leaves its block) into an output-dtype tile in shared memory;
//   * per patch, the tile's rows of `up` and columns of `down` are staged rank chunk by rank chunk (the factors are read once per
//     tile, not once per element); each thread forms a 4 x 8 block of rank sums, ascending j, one fp32 FMA chain per element;
//   * w = out(w + out(fp32(scale) * d)) in list order, with d the rank sum (LoRA) or fp32(m1 * m2) of two (LoHa);
//   * the tile leaves by 16-byte stores.
// A kernel of its own: the K1 / kron / rows instances are untouched.
//
// ggufb200_dequant_patched runs the same tile with a third patch kind, Kronecker (LoKr), interleaved with LoRA / LoHa in list
// order: d = fp32(A[n / b1, k / b2] * B[n % b1, k % b2]), A and B read through the read-only cache (one product per element, no
// rank loop, nothing staged).  It is a kernel of its own (dequant_patched_kernel, the body shared as a compile-time variant), so
// the dequant_lowrank_kernel instances compile exactly as without it.
//
// ggufb200_dequant_patched_dora is a third variant (dequant_patched_dora_kernel): any patch of the list may carry a DoRA step
// (ComfyUI's weight_decompose with its factor s, computed by the caller), applied per element after the patch's delta:
//     wc = out(w + out(fp32(scale) * d));  wc = out(wc * s[i]);  w = wc (strength 1) or out(w + out(st * out(wc - w)))
// with i = n (output axis) or k / group (input axis: one factor per Conv2d input channel, group = kh kw); s read through the
// read-only cache.  The two other variants compile exactly as without it.
#include <type_traits>

#include "blocks.cuh"
#include "fallback.cuh"
#include "internal.h"

namespace ggufb200 {

namespace {

constexpr int kThreads = 256;
constexpr int kRows = 64;                 // weight rows per tile
constexpr int kCols = 128;                // weight columns per tile
constexpr int kChunk = 32;                // rank chunk staged at a time
constexpr int kUpPitch = kRows + 4;       // floats per staged `up` column (16-byte rows for the float4 reads)
constexpr int kStageBytes = kChunk * (kUpPitch + kCols) * 4;
static_assert((kRows / 4) * (kCols / 8) == kThreads, "one 4 x 8 block of the tile per thread");
static_assert(kRows * (kCols / 32) == kThreads, "one 32-element run of the tile per thread");

struct LowrankOp {
    const float *a1, *b1, *a2, *b2;       // LoRA: a1 = up [N, r1], b1 = down [r1, K]; LoHa adds a2 [N, r2], b2 [r2, K]
    int r1, r2;                           // r2 = 0: LoRA
    float scale;
};
struct LowrankArgs {
    LowrankOp op[kLowrankMaxPatches];
    int n;
};
// ggufb200_dequant_patched: a LowrankOp, or (kron != 0) a Kronecker patch with A = lr.a1 [N / b1, a2], B = lr.b1 [b1, b2] and
// lr.scale (N = a1 b1, K = a2 b2: the whole weight)
struct PatchedOp {
    LowrankOp lr;
    int kron, a2, b1, b2;
};
struct PatchedArgs {
    PatchedOp op[kLowrankMaxPatches];
    int n;
};
// ggufb200_dequant_patched_dora: the PatchedOp list plus one DoRA step per patch (s == nullptr: a plain patch)
struct DoraOp {
    const float *s;                       // [N] (axis 0) or [K / group] (axis 1)
    int axis, group, blend;               // blend: strength != 1
    float strength;
};
struct DoraArgs {
    PatchedOp op[kLowrankMaxPatches];
    DoraOp dora[kLowrankMaxPatches];
    int n;
};
__device__ __forceinline__ const LowrankOp &lowrank_of(const LowrankOp &op) { return op; }
__device__ __forceinline__ const LowrankOp &lowrank_of(const PatchedOp &op) { return op.lr; }

// shared-memory geometry of one (format, output dtype)
template <class Q, int OUT> struct LrGeometry {
    static constexpr int OB = OutT<OUT>::bytes;
    static constexpr int PITCH = kCols * OB + 16;                                 // bytes per output-tile row (+16: fewer bank conflicts)
    static constexpr int NBLK = (Q::BS - 32 + kCols - 1) / Q::BS + 1;             // blocks one row segment can touch (it starts at a run)
    static constexpr int SLOT = (NBLK * Q::TS + 30) & ~15;                        // + the segment's offset in its first 16 bytes, + the last partial chunk
    static constexpr int PACKED = kRows * SLOT;
    static constexpr int SMEM = kRows * PITCH + (PACKED > kStageBytes ? PACKED : kStageBytes);
};

__device__ __forceinline__ void st_shared_v4(uint32_t saddr, uint32_t a, uint32_t b, uint32_t c, uint32_t d)
{
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(a), "r"(b), "r"(c), "r"(d));
}

template <int OUT> __device__ __forceinline__ float to_f32(uint32_t bits)
{
    if constexpr (OUT == kF32) return __uint_as_float(bits);
    else if constexpr (OUT == kF16) return __half2float(__ushort_as_half((unsigned short)bits));
    else return __bfloat162float(__ushort_as_bfloat16((unsigned short)bits));
}
template <int OUT> __device__ __forceinline__ uint32_t to_out(float x)
{
    if constexpr (OUT == kF32) return __float_as_uint(x);
    else if constexpr (OUT == kF16) return __half_as_ushort(__float2half_rn(x));
    else return __bfloat16_as_ushort(__float2bfloat16_rn(x));
}

// Unpack one run of 32 elements (its block at `blk` in shared memory, element e0 of the block) into the output tile at `orow`.
template <class Q, int MATH, int OUT> __device__ __forceinline__ void unpack_run(const uint8_t *blk, int e0, uint8_t *orow)
{
    constexpr int OB = OutT<OUT>::bytes;
    constexpr int EPC = 16 / OB;
    constexpr int CH = 32 / EPC;
    const uint32_t obase = smem_u32(orow);
    if constexpr (IsFallback<Q>::value) {
        static_assert(MATH == kF32, "the fallback formats are decoded in fp32 only");
        float v[32];
        Q::run32(blk, e0, v);
#pragma unroll
        for (int c = 0; c < CH; ++c) {
            const float *f = v + c * EPC;
            if constexpr (OUT == kF32) {
                st_shared_v4(obase + c * 16, __float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
            } else {
                st_shared_v4(obase + c * 16, pack16<OUT, kF32>(make_float2(f[0], f[1])), pack16<OUT, kF32>(make_float2(f[2], f[3])),
                             pack16<OUT, kF32>(make_float2(f[4], f[5])), pack16<OUT, kF32>(make_float2(f[6], f[7])));
            }
        }
    } else {
        constexpr int GROUP = GroupOf<Q>::value;
        const GroupScale<MATH> g0 = group_scale<Q, MATH>(blk, e0);
        GroupScale<MATH> g1 = g0;
        if constexpr (GROUP == 16) g1 = group_scale<Q, MATH>(blk, e0 + 16);
#pragma unroll
        for (int c = 0; c < CH; ++c) {
            const bool second = (GROUP == 16) && (c * EPC >= 16);
            typename Math<MATH>::T2 v[EPC / 2];
            dequant_elems<Q, MATH, EPC>(blk, e0 + c * EPC, second ? g1 : g0, v);
            if constexpr (OUT == kF32) {
                const float2 f0 = Math<MATH>::to_f32x2(v[0]), f1 = Math<MATH>::to_f32x2(v[1]);
                st_shared_v4(obase + c * 16, __float_as_uint(f0.x), __float_as_uint(f0.y), __float_as_uint(f1.x), __float_as_uint(f1.y));
            } else {
                st_shared_v4(obase + c * 16, pack16<OUT, MATH>(v[0]), pack16<OUT, MATH>(v[1]), pack16<OUT, MATH>(v[2]), pack16<OUT, MATH>(v[3]));
            }
        }
    }
}

// 4 bytes global -> shared without a register round trip; `in` false: the 4 bytes are zero-filled (nothing is read)
__device__ __forceinline__ void cp_async4(float *dst, const float *src, bool in)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(in ? 4 : 0) : "memory");
}

// d[i][c] = sum_j a[n0 + 4 rg + i, j] * b[j, k0 + 8 cg + c], j ascending, one fp32 FMA chain per element.  The tile's rows of `a`
// and columns of `b` are staged kChunk ranks at a time (rows past N and columns past K read as zero).
__device__ __forceinline__ void rank_sums(const float *__restrict__ a, const float *__restrict__ b, int r, int N, int K, int n0, int k0,
                                          float *stage, int tid, float (&d)[4][8])
{
    float *up = stage;                         // [kChunk][kUpPitch]: up[j][i] = a[n0 + i, j0 + j]
    float *dn = stage + kChunk * kUpPitch;     // [kChunk][kCols]:    dn[j][c] = b[j0 + j, k0 + c]
    const int rg = tid / (kCols / 8), cg = tid % (kCols / 8);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < 8; ++c) d[i][c] = -0.0f;     // x + -0 == x for every x: the first FMA is the plain product
    for (int j0 = 0; j0 < r; j0 += kChunk) {
        const int rc = r - j0 < kChunk ? r - j0 : kChunk;
        __syncthreads();                                  // the previous chunk (or the unpack of the packed tile) is done
        // cp.async: every thread's loads are in flight at once (a load + store loop would wait for each load in turn)
        for (int idx = tid; idx < kRows * rc; idx += kThreads) {
            const int i = idx / rc, j = idx - i * rc;
            const bool in = n0 + i < N;
            cp_async4(up + j * kUpPitch + i, a + (in ? (size_t)(n0 + i) * r + j0 + j : 0), in);
        }
        for (int idx = tid; idx < rc * kCols; idx += kThreads) {
            const int j = idx / kCols, c = idx - j * kCols;
            const bool in = k0 + c < K;
            cp_async4(dn + idx, b + (size_t)(j0 + j) * K + (in ? k0 + c : 0), in);
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncthreads();
        for (int j = 0; j < rc; ++j) {
            const float4 u = *reinterpret_cast<const float4 *>(up + j * kUpPitch + 4 * rg);
            const float4 v0 = *reinterpret_cast<const float4 *>(dn + j * kCols + 8 * cg);
            const float4 v1 = *reinterpret_cast<const float4 *>(dn + j * kCols + 8 * cg + 4);
            const float uu[4] = {u.x, u.y, u.z, u.w};
            const float vv[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int c = 0; c < 8; ++c) d[i][c] = __fmaf_rn(uu[i], vv[c], d[i][c]);
        }
    }
}

// The Kronecker patch on this thread's 4 x 8 block (rows n0 + 4 rg .., columns k0 + 8 cg ..; rows past N are skipped, the
// caller skips a block past the tile's columns): w = out(w + out(fp32(scale) * fp32(A[i1, i2] * B[j1, j2]))), (i1, j1) =
// divmod(n, b1), (i2, j2) = divmod(k, b2).
template <int OUT, int PITCH>
__device__ __forceinline__ void kron_block(uint8_t *otile, const PatchedOp &op, int N, int n0, int k0, int rg, int cg)
{
    constexpr int OB = OutT<OUT>::bytes;
    const float *__restrict__ A = op.lr.a1;
    const float *__restrict__ B = op.lr.b1;
    const int kb = k0 + 8 * cg;
    const int i2_0 = kb / op.b2, j2_0 = kb - i2_0 * op.b2;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int n = n0 + 4 * rg + i;
        if (n >= N) break;
        const int i1 = n / op.b1, j1 = n - i1 * op.b1;
        const float *arow = A + (size_t)i1 * op.a2;
        const float *brow = B + (size_t)j1 * op.b2;
        uint8_t *w = otile + (4 * rg + i) * PITCH + 8 * cg * OB;
        int i2 = i2_0, j2 = j2_0;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float d = __fmul_rn(__ldg(arow + i2), __ldg(brow + j2));
            const float delta = to_f32<OUT>(to_out<OUT>(__fmul_rn(op.lr.scale, d)));
            if constexpr (OUT == kF32) {
                float &x = reinterpret_cast<float *>(w)[c];
                x = __fadd_rn(x, delta);
            } else {
                uint16_t &x = reinterpret_cast<uint16_t *>(w)[c];
                x = (uint16_t)to_out<OUT>(__fadd_rn(to_f32<OUT>(x), delta));
            }
            if (++j2 == op.b2) {
                j2 = 0;
                ++i2;
            }
        }
    }
}

// DoRA variant: d[i][c] = fp32(A[i1, i2] * B[j1, j2]) of the Kronecker patch for this thread's 4 x 8 block (rows past N are
// left as they are: `dora_block` skips them)
__device__ __forceinline__ void kron_deltas(const PatchedOp &op, int N, int n0, int k0, int rg, int cg, float (&d)[4][8])
{
    const int kb = k0 + 8 * cg;
    const int i2_0 = kb / op.b2, j2_0 = kb - i2_0 * op.b2;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int n = n0 + 4 * rg + i;
        if (n >= N) break;
        const int i1 = n / op.b1, j1 = n - i1 * op.b1;
        const float *arow = op.lr.a1 + (size_t)i1 * op.a2;
        const float *brow = op.lr.b1 + (size_t)j1 * op.b2;
        int i2 = i2_0, j2 = j2_0;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            d[i][c] = __fmul_rn(__ldg(arow + i2), __ldg(brow + j2));
            if (++j2 == op.b2) {
                j2 = 0;
                ++i2;
            }
        }
    }
}

// DoRA variant: one patch on this thread's 4 x 8 block (rows past N skipped; the caller skips a block past the tile's columns):
// wc = out(w + out(fp32(scale) * d)), then, for a DoRA patch, wc = out(wc * s[i]) and w = wc or out(w + out(st * out(wc - w))).
// Every step rounds to the output dtype, as the reference's tensors of that dtype do.
template <int OUT, int PITCH>
__device__ __forceinline__ void dora_block(uint8_t *otile, const float (&d)[4][8], float scale, const DoraOp &dr, int N, int n0, int k0,
                                           int rg, int cg)
{
    constexpr int OB = OutT<OUT>::bytes;
    const bool in_axis = dr.s != nullptr && dr.axis == 1;
    const int kb = k0 + 8 * cg;
    // input axis: g = the channel of column kb + c, gk = the column's place in it (one division per patch, not per element)
    int g = in_axis ? kb / dr.group : 0, gk = in_axis ? kb - g * dr.group : 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const float s_col = in_axis ? __ldg(dr.s + g) : 0.0f;
        if (in_axis && ++gk == dr.group) {
            gk = 0;
            ++g;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int n = n0 + 4 * rg + i;
            if (n >= N) break;
            uint8_t *w = otile + (4 * rg + i) * PITCH + 8 * cg * OB;
            float x;
            if constexpr (OUT == kF32) x = reinterpret_cast<const float *>(w)[c];
            else x = to_f32<OUT>(reinterpret_cast<const uint16_t *>(w)[c]);
            const float delta = to_f32<OUT>(to_out<OUT>(__fmul_rn(scale, d[i][c])));
            float wc = to_f32<OUT>(to_out<OUT>(__fadd_rn(x, delta)));
            if (dr.s != nullptr) {
                const float s = in_axis ? s_col : __ldg(dr.s + n);
                wc = to_f32<OUT>(to_out<OUT>(__fmul_rn(wc, s)));
                if (dr.blend) {
                    const float t = to_f32<OUT>(to_out<OUT>(__fmul_rn(dr.strength, to_f32<OUT>(to_out<OUT>(__fsub_rn(wc, x))))));
                    wc = to_f32<OUT>(to_out<OUT>(__fadd_rn(x, t)));
                }
            }
            if constexpr (OUT == kF32) reinterpret_cast<float *>(w)[c] = wc;
            else reinterpret_cast<uint16_t *>(w)[c] = (uint16_t)to_out<OUT>(wc);
        }
    }
}

// The tile of one CTA; Args = LowrankArgs (ggufb200_dequant_lowrank), PatchedArgs (ggufb200_dequant_patched, Kronecker
// patches as well) or DoraArgs (ggufb200_dequant_patched_dora, a DoRA step per patch as well).
template <class Q, int MATH, int OUT, class Args>
__device__ __forceinline__ void lowrank_tile(const uint8_t *__restrict__ src, long long total_bytes, int aligned, int N, int K,
                                             uint8_t *__restrict__ dst, const Args &la)
{
    constexpr bool KRON = std::is_same<Args, PatchedArgs>::value;
    constexpr bool DORA = std::is_same<Args, DoraArgs>::value;
    using G = LrGeometry<Q, OUT>;
    constexpr int OB = G::OB;
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t *otile = smem;                                   // [kRows][PITCH]: the tile in the output dtype
    uint8_t *packed = smem + kRows * G::PITCH;               // [kRows][SLOT], later the factor stage
    float *stage = reinterpret_cast<float *>(packed);
    const int tid = threadIdx.x;
    const int k0 = blockIdx.x * kCols, n0 = blockIdx.y * kRows;
    const int cols = K - k0 < kCols ? K - k0 : kCols;        // a multiple of 32

    // 1. the packed bytes of every row segment: block bytes b_lo * TS .. (b_hi + 1) * TS of the stream, from the 16-byte boundary
    //    at or below, into the row's slot (16-byte chunks from a 16-byte aligned stream, bytes otherwise; never past the stream)
    constexpr int CPR = G::SLOT / 16;
    for (int idx = tid; idx < kRows * CPR; idx += kThreads) {
        const int i = idx / CPR, ch = idx - i * CPR;
        if (n0 + i >= N) continue;
        const long long e = (long long)(n0 + i) * K + k0;
        const long long s16 = (e / Q::BS * Q::TS) & ~15ll;
        const long long end = ((e + cols - 1) / Q::BS + 1) * Q::TS;
        const long long at = s16 + 16ll * ch;
        if (at >= end) continue;
        uint8_t *to = packed + i * G::SLOT + 16 * ch;
        if (aligned && at + 16 <= total_bytes) {
            *reinterpret_cast<uint4 *>(to) = __ldg(reinterpret_cast<const uint4 *>(src + at));
        } else {
            for (int q = 0; q < 16 && at + q < total_bytes; ++q) to[q] = src[at + q];
        }
    }
    __syncthreads();

    // 2. unpack: thread = one run of 32 elements, row tid / 4, columns 32 (tid % 4) ..
    {
        const int i = tid / (kCols / 32), run = tid % (kCols / 32);
        if (n0 + i < N && 32 * run < cols) {
            const long long e = (long long)(n0 + i) * K + k0 + 32 * run;
            const long long s16 = ((long long)(n0 + i) * K + k0) / Q::BS * Q::TS & ~15ll;
            const uint8_t *blk = packed + i * G::SLOT + (e / Q::BS * Q::TS - s16);
            unpack_run<Q, MATH, OUT>(blk, (int)(e % Q::BS), otile + i * G::PITCH + 32 * run * OB);
        }
    }

    // 3. the patches, in list order, on each thread's 4 x 8 block (rows 4 rg .., columns 8 cg ..)
    const int rg = tid / (kCols / 8), cg = tid % (kCols / 8);
    for (int p = 0; p < la.n; ++p) {
        if constexpr (DORA) {
            const PatchedOp &op = la.op[p];
            float d[4][8];
            if (op.kron) {
                __syncthreads();                                  // the unpack (or the previous patch) of other threads' elements is done
                if (8 * cg < cols) kron_deltas(op, N, n0, k0, rg, cg, d);
            } else {
                rank_sums(op.lr.a1, op.lr.b1, op.lr.r1, N, K, n0, k0, stage, tid, d);
                if (op.lr.r2 > 0) {
                    float d2[4][8];
                    rank_sums(op.lr.a2, op.lr.b2, op.lr.r2, N, K, n0, k0, stage, tid, d2);
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int c = 0; c < 8; ++c) d[i][c] = __fmul_rn(d[i][c], d2[i][c]);
                }
            }
            if (8 * cg < cols) dora_block<OUT, G::PITCH>(otile, d, op.lr.scale, la.dora[p], N, n0, k0, rg, cg);
            continue;
        }
        if constexpr (KRON) {
            if (la.op[p].kron) {
                __syncthreads();                                  // the unpack (or the previous patch) of other threads' elements is done
                if (8 * cg < cols) kron_block<OUT, G::PITCH>(otile, la.op[p], N, n0, k0, rg, cg);
                continue;
            }
        }
        const LowrankOp &op = lowrank_of(la.op[p]);
        float d[4][8];
        rank_sums(op.a1, op.b1, op.r1, N, K, n0, k0, stage, tid, d);
        if (op.r2 > 0) {
            float d2[4][8];
            rank_sums(op.a2, op.b2, op.r2, N, K, n0, k0, stage, tid, d2);
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int c = 0; c < 8; ++c) d[i][c] = __fmul_rn(d[i][c], d2[i][c]);
        }
        if (8 * cg >= cols) continue;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint8_t *w = otile + (4 * rg + i) * G::PITCH + 8 * cg * OB;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const float delta = to_f32<OUT>(to_out<OUT>(__fmul_rn(op.scale, d[i][c])));
                if constexpr (OUT == kF32) {
                    float &x = reinterpret_cast<float *>(w)[c];
                    x = __fadd_rn(x, delta);
                } else {
                    uint16_t &x = reinterpret_cast<uint16_t *>(w)[c];
                    x = (uint16_t)to_out<OUT>(__fadd_rn(to_f32<OUT>(x), delta));
                }
            }
        }
    }
    __syncthreads();

    // 4. store: each thread its 4 x 8 block, 16 bytes at a time
    if (8 * cg < cols) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int n = n0 + 4 * rg + i;
            if (n >= N) break;
            const uint4 *from = reinterpret_cast<const uint4 *>(otile + (4 * rg + i) * G::PITCH + 8 * cg * OB);
            uint8_t *to = dst + ((long long)n * K + k0 + 8 * cg) * OB;
#pragma unroll
            for (int q = 0; q < OB / 2; ++q) {
                const uint4 v = from[q];
                st_global_v4(to + 16 * q, v.x, v.y, v.z, v.w);
            }
        }
    }
}

template <class Q, int MATH, int OUT>
__global__ void __launch_bounds__(kThreads) dequant_lowrank_kernel(const uint8_t *__restrict__ src, long long total_bytes, int aligned, int N,
                                                                   int K, uint8_t *__restrict__ dst, const __grid_constant__ LowrankArgs la)
{
    lowrank_tile<Q, MATH, OUT>(src, total_bytes, aligned, N, K, dst, la);
}

template <class Q, int MATH, int OUT>
__global__ void __launch_bounds__(kThreads) dequant_patched_kernel(const uint8_t *__restrict__ src, long long total_bytes, int aligned, int N,
                                                                   int K, uint8_t *__restrict__ dst, const __grid_constant__ PatchedArgs la)
{
    lowrank_tile<Q, MATH, OUT>(src, total_bytes, aligned, N, K, dst, la);
}

template <class Q, int MATH, int OUT>
__global__ void __launch_bounds__(kThreads) dequant_patched_dora_kernel(const uint8_t *__restrict__ src, long long total_bytes, int aligned,
                                                                        int N, int K, uint8_t *__restrict__ dst,
                                                                        const __grid_constant__ DoraArgs la)
{
    lowrank_tile<Q, MATH, OUT>(src, total_bytes, aligned, N, K, dst, la);
}

template <class Args, class Q, int MATH, int OUT> struct KernelOf {
    static constexpr auto value = dequant_lowrank_kernel<Q, MATH, OUT>;
};
template <class Q, int MATH, int OUT> struct KernelOf<PatchedArgs, Q, MATH, OUT> {
    static constexpr auto value = dequant_patched_kernel<Q, MATH, OUT>;
};
template <class Q, int MATH, int OUT> struct KernelOf<DoraArgs, Q, MATH, OUT> {
    static constexpr auto value = dequant_patched_dora_kernel<Q, MATH, OUT>;
};

template <class Q, int MATH, int OUT, class Args>
int launch_lowrank(const void *packed, long long N, long long K, void *out, const Args &la, cudaStream_t st)
{
    using G = LrGeometry<Q, OUT>;
    auto kern = KernelOf<Args, Q, MATH, OUT>::value;
    static unsigned char smem_set[64] = {};
    if (!ensure_dynamic_smem(kern, G::SMEM, smem_set)) return GGUFB200_E_CUDA;
    const dim3 grid((unsigned)((K + kCols - 1) / kCols), (unsigned)((N + kRows - 1) / kRows));
    const long long total_bytes = N * K / Q::BS * Q::TS;
    const int aligned = (reinterpret_cast<uintptr_t>(packed) & 15) == 0;
    kern<<<grid, kThreads, G::SMEM, st>>>(reinterpret_cast<const uint8_t *>(packed), total_bytes, aligned, (int)N, (int)K,
                                          reinterpret_cast<uint8_t *>(out), la);
    return cudaGetLastError() == cudaSuccess ? GGUFB200_OK : GGUFB200_E_CUDA;
}

template <class Q, int MATH, class Args> int lowrank_out(const void *p, long long N, long long K, void *out, int od, const Args &la, cudaStream_t st)
{
    switch (od) {
    case kF16: return launch_lowrank<Q, MATH, kF16>(p, N, K, out, la, st);
    case kBF16: return launch_lowrank<Q, MATH, kBF16>(p, N, K, out, la, st);
    case kF32: return launch_lowrank<Q, MATH, kF32>(p, N, K, out, la, st);
    }
    return GGUFB200_E_DTYPE;
}

// every block format with K1's math dtypes, every fallback format in fp32, fp16 / bf16 / fp32 output
template <class Args>
int lowrank_dispatch(int type, const void *packed, long long N, long long K, void *out, int out_dtype, int math_dtype, const Args &la,
                     cudaStream_t st)
{
    const int fb = with_fallback_block(type, (int)GGUFB200_E_TYPE, [&](auto blk) {     // fp32 math: the reference ignores dequant_dtype there
        return lowrank_out<decltype(blk), kF32>(packed, N, K, out, out_dtype, la, st);
    });
    if (fb != GGUFB200_E_TYPE) return fb;
    return with_block(type, (int)GGUFB200_E_TYPE, [&](auto blk) {
        using Q = decltype(blk);
        switch (math_dtype) {
        case kF16: return lowrank_out<Q, kF16>(packed, N, K, out, out_dtype, la, st);
        case kBF16: return lowrank_out<Q, kBF16>(packed, N, K, out, out_dtype, la, st);
        case kF32: return lowrank_out<Q, kF32>(packed, N, K, out, out_dtype, la, st);
        }
        return (int)GGUFB200_E_DTYPE;
    });
}

LowrankOp lowrank_op(const ggufb200_lowrank_patch &p)
{
    return LowrankOp{p.a1, p.b1, p.a2, p.b2, (int)p.r1, p.a2 ? (int)p.r2 : 0, p.scale};
}

PatchedOp patched_op(const ggufb200_weight_patch &p)
{
    PatchedOp op{};
    if (p.kind == GGUFB200_PATCH_KRON) {
        const ggufb200_kron_patch &k = p.kron;
        op.lr = LowrankOp{k.A, k.B, nullptr, nullptr, 0, 0, k.scale};
        op.kron = 1;
        op.a2 = (int)k.a2;
        op.b1 = (int)k.b1;
        op.b2 = (int)k.b2;
    } else {
        op.lr = lowrank_op(p.lowrank);
    }
    return op;
}

}  // namespace

int dequant_lowrank_dispatch(int type, const void *packed, long long N, long long K, void *out, int out_dtype, int math_dtype,
                             const ggufb200_lowrank_patch *patches, int n_patches, cudaStream_t st)
{
    LowrankArgs la{};
    la.n = n_patches;
    for (int i = 0; i < n_patches; ++i) la.op[i] = lowrank_op(patches[i]);
    return lowrank_dispatch(type, packed, N, K, out, out_dtype, math_dtype, la, st);
}

int dequant_patched_dispatch(int type, const void *packed, long long N, long long K, void *out, int out_dtype, int math_dtype,
                             const ggufb200_weight_patch *patches, int n_patches, cudaStream_t st)
{
    PatchedArgs la{};
    la.n = n_patches;
    for (int i = 0; i < n_patches; ++i) la.op[i] = patched_op(patches[i]);
    return lowrank_dispatch(type, packed, N, K, out, out_dtype, math_dtype, la, st);
}

int dequant_patched_dora_dispatch(int type, const void *packed, long long N, long long K, void *out, int out_dtype, int math_dtype,
                                  const ggufb200_weight_patch *patches, const ggufb200_dora_patch *dora, int n_patches, cudaStream_t st)
{
    DoraArgs la{};
    la.n = n_patches;
    for (int i = 0; i < n_patches; ++i) {
        la.op[i] = patched_op(patches[i]);
        const ggufb200_dora_patch &d = dora[i];
        la.dora[i] = DoraOp{d.factor, (int)d.axis, d.axis == 1 ? (int)d.group : 1, d.strength != 1.0f, d.strength};
    }
    return lowrank_dispatch(type, packed, N, K, out, out_dtype, math_dtype, la, st);
}

}  // namespace ggufb200
