// dequant.cu -- K1: standalone GGUF block dequant (HBM-bound streaming kernel).
//
// Replaces dequant.py:30-44 + every dequantize_blocks_* (dequant.py:61-285) + the final
// `.to(dtype)` (dequant.py:23) with ONE kernel launch per tensor.
//
// Data movement (algorithmic bytes per element = TS/BS read + sizeof(out) written):
//   * the packed block stream is treated as a flat byte stream (block sizes 18/22/34/84/110/
//     210 B are not 16 B multiples, so 2-D tensor maps are illegal for most shapes); it is cut
//     into tiles of 4096 elements whose byte span is always a multiple of 16 B
//   * ONE TILE PER CTA (128 threads), CTAs handed out by the hardware in address order: the write front stays
//     compact, an SM that happens to be slower simply takes fewer tiles, and 16 CTAs per SM cover each other's load
//     latency (instead of persistent CTAs walking strided tiles through a prefetch ring, whose write fronts spread out).
//   * the tile is staged into shared memory by thread 0 with the TMA engine (cp.async.bulk, SASS UBLKCP), completion on
//     an mbarrier that only thread 0 polls; the other threads sleep in the CTA barrier
//   * every thread unpacks one run of 32 consecutive elements from shared memory (blocks.cuh) into its row of the output
//     tile in shared memory, which leaves through ONE swizzled tensor-map store (cp.async.bulk.tensor.2d, SASS UTMASTG): no
//     thread computes a global address, every HBM write is a full line, and the unpack runs with immediate offsets
#include <type_traits>

#include "blocks.cuh"
#include "internal.h"
#include "wgmma.cuh"

namespace ggufb200 {

constexpr int kThreads = 128;       // threads per CTA of the dequant kernel = 4096-element tiles (256: 0.929, 64: 0.80 of the copy peak on the Flux-shape sweep)

int g_dequant_pdl = 1;          // programmatic dependent launch of the dequant kernel; ggufb200_set_tuning(1, 0/1)

// Store into the OUTPUT tile.  No "memory" clobber: the output tile never aliases the packed tile the unpack reads, so the
// compiler may keep the bytes it has already loaded (the high nibbles of a 4-bit block sit in the same bytes as the low ones)
// across these stores; `volatile` keeps them in order before the fence + barrier that publish the tile.
__device__ __forceinline__ void st_otile_v4(uint32_t saddr, uint32_t a, uint32_t b, uint32_t c, uint32_t d)
{
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(a), "r"(b), "r"(c), "r"(d));
}

// One thread = one run of 32 consecutive elements of the packed tile at `tile` (shared memory).  The output tile is laid out for
// a swizzled 2-D tensor-map store, one row per thread (fp16 / bf16: 64-byte rows, CU_TENSOR_MAP_SWIZZLE_64B; fp32: 128-byte rows,
// SWIZZLE_128B): 16-byte chunk p of a row sits at chunk p ^ (address bits 7.. of the row), so the chunks are processed in their
// natural order -- every byte offset and shift of the unpack is an immediate -- and the STS.128 of a quarter-warp still hit eight
// different bank groups.  (A linear tile needs the chunk ORDER rotated per lane instead: dynamic offsets and shifts, more
// instructions.)
template <class Q, int MATH, int OUT>
__device__ __forceinline__ void dequant_tile(const uint8_t *tile, uint8_t *otile, int tile_elems, int tid)
{
    constexpr int OB = OutT<OUT>::bytes;
    constexpr int EPC = 16 / OB;                           // elements per 16-byte chunk: 8 or 4
    constexpr int CH = 32 / EPC;                           // chunks per thread: 4 or 8
    constexpr int GROUP = GroupOf<Q>::value;
    const int blk_in_tile = (tid * 32) / Q::BS;
    const int e0 = (tid * 32) % Q::BS;
    if (tid * 32 < tile_elems) {
        const uint8_t *blk = tile + blk_in_tile * Q::TS;
        const GroupScale<MATH> g0 = group_scale<Q, MATH>(blk, e0);
        GroupScale<MATH> g1 = g0;
        if constexpr (GROUP == 16) g1 = group_scale<Q, MATH>(blk, e0 + 16);
        const uint32_t obase = smem_u32(otile) + tid * (32 * OB);
        const uint32_t sw = (obase >> 7) & (CH - 1);       // the engine's swizzle key: shared-memory address bits 7-8 (64B mode) / 7-9 (128B mode)
#pragma unroll
        for (int c = 0; c < CH; ++c) {
            const int e = e0 + c * EPC;
            const bool second = (GROUP == 16) && (c * EPC >= 16);
            typename Math<MATH>::T2 v[EPC / 2];
            dequant_elems<Q, MATH, EPC>(blk, e, second ? g1 : g0, v);
            const uint32_t oaddr = obase + ((uint32_t)c ^ sw) * 16;
            if constexpr (OUT == kF32) {
                float2 f0 = Math<MATH>::to_f32x2(v[0]), f1 = Math<MATH>::to_f32x2(v[1]);
                st_otile_v4(oaddr, __float_as_uint(f0.x), __float_as_uint(f0.y), __float_as_uint(f1.x), __float_as_uint(f1.y));
            } else {
                st_otile_v4(oaddr, pack16<OUT, MATH>(v[0]), pack16<OUT, MATH>(v[1]), pack16<OUT, MATH>(v[2]), pack16<OUT, MATH>(v[3]));
            }
        }
    }
}

// One tile per CTA (see the file header).  flags: bit 0 = the packed pointer is 16-byte aligned (bulk copy legal),
// bit 1 = GGUFB200_DEQUANT_SRC_STABLE.
template <class Q, int MATH, int OUT, int THREADS>
__global__ void __launch_bounds__(THREADS) dequant_kernel(const __grid_constant__ CUtensorMap tmOut, const uint8_t *__restrict__ src,
                                                          void *__restrict__ dst, long long n_blocks, int flags)
{
    constexpr int OB = OutT<OUT>::bytes;
    constexpr int TILE_ELEMS = THREADS * 32;
    constexpr int TILE_BLOCKS = TILE_ELEMS / Q::BS;
    constexpr int TILE_BYTES = TILE_BLOCKS * Q::TS;
    static_assert(TILE_BYTES % 16 == 0, "tile byte span must be a multiple of 16");
    static_assert(TILE_ELEMS % Q::BS == 0, "tile shape");
    const int bulk_ok = flags & 1;
    const bool early = bulk_ok && (flags & 2);

    // output tile first (the swizzle pattern of the tensor-map store is a function of the shared-memory ADDRESS bits; the
    // threads derive their key from the address too, so the two agree wherever the window starts)
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *otile = smem;
    uint8_t *tile = smem + TILE_ELEMS * OB;
    uint64_t *full = reinterpret_cast<uint64_t *>(tile + ((TILE_BYTES + 16 + 15) & ~15));

    const int tid = threadIdx.x;
    const long long t = blockIdx.x;
    const long long total_bytes = n_blocks * (long long)Q::TS;
    const long long n_elems = n_blocks * (long long)Q::BS;
    long long off = t * (long long)TILE_BYTES;
    long long len = total_bytes - off;
    if (len > TILE_BYTES) len = TILE_BYTES;

    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (bulk_ok) {
        // Only thread 0 touches the mbarrier (init, copy, wait); the other 255 threads sleep in the CTA barrier instead of
        // polling, so the warps of the SM's other CTAs that are unpacking get the issue slots.
        if (tid == 0) {
            mbar_init(full, 1);
            fence_mbar_init();
            if (!early) asm volatile("griddepcontrol.wait;" ::: "memory");
            uint32_t bytes = (uint32_t)((len + 15) & ~15LL);
            mbar_arrive_expect_tx(full, bytes);
            bulk_g2s(tile, src + off, bytes, full);
            mbar_wait(full, 0);
        }
    } else {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        for (int i = tid; i < (int)len; i += THREADS) tile[i] = src[off + i];
    }
    __syncthreads();
    const long long elem_base = t * (long long)TILE_ELEMS;
    const long long left = n_elems - elem_base;
    const int tile_elems = left < TILE_ELEMS ? (int)left : TILE_ELEMS;
    dequant_tile<Q, MATH, OUT>(tile, otile, tile_elems, tid);
    fence_proxy_async_smem();
    __syncthreads();
    if (tid == 0) {
        if (early) asm volatile("griddepcontrol.wait;" ::: "memory");
        // one box = this tile's THREADS rows; rows past the end of the tensor (short last tile) are clipped by the TMA engine
        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(&tmOut)),
                     "r"(smem_u32(otile)), "r"(0), "r"((int)(t * THREADS))
                     : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");      // the shared-memory tile must outlive the engine's read of it
    }
}

// ------------------------------------------------------------------ K1 with LoKr patches (ggufb200_dequant_kron)
// One patch as the kernel reads it: band rows r0 .. r0 + rows, columns c0 .. c0 + cols; `staged`: the tile's B rows are copied
// to shared memory first (host decision: they fit kKronStageBytes).
struct KronOp {
    const float *A, *B;
    int a2, b1, b2, r0, rows, c0, cols, staged;
    float scale;
};
struct KronArgs {
    KronOp op[kKronMaxPatches];
    int n, K;
};
constexpr int kKronStageBytes = 32 * 1024;

// element j of a 16-byte chunk of the output tile: its bit pattern, and its value in fp32
template <int OUT> __device__ __forceinline__ uint32_t out_bits(const uint32_t (&w)[4], int j)
{
    if constexpr (OUT == kF32) return w[j];
    else return (w[j >> 1] >> (16 * (j & 1))) & 0xFFFFu;
}
template <int OUT> __device__ __forceinline__ float out_value(uint32_t bits)
{
    if constexpr (OUT == kF32) return __uint_as_float(bits);
    else if constexpr (OUT == kF16) return __half2float(__ushort_as_half((unsigned short)bits));
    else return __bfloat162float(__ushort_as_bfloat16((unsigned short)bits));
}
// round to the output dtype; the result is returned as the fp32 value and, through `bits`, as the output pattern
template <int OUT> __device__ __forceinline__ float out_round(float x, uint32_t &bits)
{
    if constexpr (OUT == kF32) {
        bits = __float_as_uint(x);
        return x;
    } else if constexpr (OUT == kF16) {
        const __half h = __float2half_rn(x);
        bits = __half_as_ushort(h);
        return __half2float(h);
    } else {
        const __nv_bfloat16 h = __float2bfloat16_rn(x);
        bits = __bfloat16_as_ushort(h);
        return __bfloat162float(h);
    }
}

// The patch pass over one dequantised output tile (its rows as dequant_tile left them; each thread rewrites its own 32 elements,
// so no barrier is needed before it).  Per element, in list order:  w = out(w + out(fp32(s) * fp32(A[i1, i2] * B[j1, j2]))),
// the sequence of `weight += ((s * alpha) * torch.kron(w1, w2)).to(weight.dtype)` with fp32 factors.  Chunks of EPC elements
// never cross a row (K % 8 == 0).  `stage`: room for the B rows of every weight row the tile touches.
template <int OUT, int THREADS>
__device__ __forceinline__ void kron_tile(uint8_t *otile, float *stage, const KronArgs &ka, long long elem_base, int tile_elems, int tid)
{
    constexpr int OB = OutT<OUT>::bytes;
    constexpr int EPC = 16 / OB;
    constexpr int CH = 32 / EPC;
    const int K = ka.K;
    const int n_first = (int)(elem_base / K);
    const int n_last = (int)((elem_base + tile_elems - 1) / K);
    const bool active = tid * 32 < tile_elems;
    const long long e_t = elem_base + tid * 32;
    const int n_t = (int)(e_t / K), k_t = (int)(e_t - (long long)n_t * K);
    const uint32_t obase = smem_u32(otile) + tid * (32 * OB);
    const uint32_t sw = (obase >> 7) & (CH - 1);
    for (int p = 0; p < ka.n; ++p) {
        const KronOp &op = ka.op[p];
        const int lo = max(n_first, op.r0), hi = min(n_last, op.r0 + op.rows - 1);
        if (op.staged) {
            __syncthreads();                                   // the previous patch is done with the stage
            for (int n = lo; n <= hi; ++n) {
                const float *brow = op.B + (size_t)((n - op.r0) % op.b1) * op.b2;
                float *srow = stage + (n - lo) * op.b2;
                for (int j = tid; j < op.b2; j += THREADS) srow[j] = __ldg(brow + j);
            }
            __syncthreads();
        }
        if (!active) continue;
        int n = n_t, k = k_t;
#pragma unroll
        for (int c = 0; c < CH; ++c, k += EPC) {
            if (k >= K) {
                k -= K;
                ++n;
            }
            int kk = k - op.c0;
            if (n < lo || n > hi || kk + EPC <= 0 || kk >= op.cols) continue;
            const int nn = n - op.r0;
            const int i1 = nn / op.b1;
            const float *arow = op.A + (size_t)i1 * op.a2;
            const float *brow = op.staged ? stage + (n - lo) * op.b2 : op.B + (size_t)(nn - i1 * op.b1) * op.b2;
            int i2 = 0, j2 = 0;
            if (kk > 0) {
                i2 = kk / op.b2;
                j2 = kk - i2 * op.b2;
            }
            const uint32_t oaddr = obase + ((uint32_t)c ^ sw) * 16;
            uint32_t w[4];
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(oaddr));
            uint32_t o[EPC];
#pragma unroll
            for (int j = 0; j < EPC; ++j, ++kk) {
                o[j] = out_bits<OUT>(w, j);
                if (kk >= 0 && kk < op.cols) {
                    const float prod = __fmul_rn(__ldg(arow + i2), brow[j2]);
                    uint32_t dbits;
                    const float d = out_round<OUT>(__fmul_rn(op.scale, prod), dbits);
                    out_round<OUT>(__fadd_rn(out_value<OUT>(o[j]), d), o[j]);
                    if (++j2 == op.b2) {
                        j2 = 0;
                        ++i2;
                    }
                }
            }
            if constexpr (OUT == kF32) st_otile_v4(oaddr, o[0], o[1], o[2], o[3]);
            else st_otile_v4(oaddr, o[0] | (o[1] << 16), o[2] | (o[3] << 16), o[4] | (o[5] << 16), o[6] | (o[7] << 16));
        }
    }
}

// dequant_kernel with the patch pass between the unpack and the store (a kernel of its own, so that the plain K1 instances
// are not touched).  Shared memory: dequant_kernel's layout, then the B-row stage.
template <class Q, int MATH, int OUT, int THREADS>
__global__ void __launch_bounds__(THREADS) dequant_kron_kernel(const __grid_constant__ CUtensorMap tmOut, const uint8_t *__restrict__ src,
                                                               long long n_blocks, int flags, const __grid_constant__ KronArgs kron)
{
    constexpr int OB = OutT<OUT>::bytes;
    constexpr int TILE_ELEMS = THREADS * 32;
    constexpr int TILE_BLOCKS = TILE_ELEMS / Q::BS;
    constexpr int TILE_BYTES = TILE_BLOCKS * Q::TS;
    constexpr int TB = (TILE_BYTES + 16 + 15) & ~15;
    const int bulk_ok = flags & 1;
    const bool early = bulk_ok && (flags & 2);

    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *otile = smem;
    uint8_t *tile = smem + TILE_ELEMS * OB;
    uint64_t *full = reinterpret_cast<uint64_t *>(tile + TB);
    float *stage = reinterpret_cast<float *>(tile + TB + 16);

    const int tid = threadIdx.x;
    const long long t = blockIdx.x;
    const long long total_bytes = n_blocks * (long long)Q::TS;
    const long long n_elems = n_blocks * (long long)Q::BS;
    long long off = t * (long long)TILE_BYTES;
    long long len = total_bytes - off;
    if (len > TILE_BYTES) len = TILE_BYTES;

    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (bulk_ok) {
        if (tid == 0) {
            mbar_init(full, 1);
            fence_mbar_init();
            if (!early) asm volatile("griddepcontrol.wait;" ::: "memory");
            uint32_t bytes = (uint32_t)((len + 15) & ~15LL);
            mbar_arrive_expect_tx(full, bytes);
            bulk_g2s(tile, src + off, bytes, full);
            mbar_wait(full, 0);
        }
    } else {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        for (int i = tid; i < (int)len; i += THREADS) tile[i] = src[off + i];
    }
    __syncthreads();
    const long long elem_base = t * (long long)TILE_ELEMS;
    const long long left = n_elems - elem_base;
    const int tile_elems = left < TILE_ELEMS ? (int)left : TILE_ELEMS;
    dequant_tile<Q, MATH, OUT>(tile, otile, tile_elems, tid);
    kron_tile<OUT, THREADS>(otile, stage, kron, elem_base, tile_elems, tid);
    fence_proxy_async_smem();
    __syncthreads();
    if (tid == 0) {
        if (early) asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(&tmOut)),
                     "r"(smem_u32(otile)), "r"(0), "r"((int)(t * THREADS))
                     : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
}

// BF16 "quantised" type (dequant.py:61-62): widen to fp32, then cast to the output dtype
template <int OUT> __global__ void __launch_bounds__(kThreads) bf16_kernel(const uint16_t *__restrict__ src, void *__restrict__ dst, long long n)
{
    using O = typename OutT<OUT>::type;
    O *out = reinterpret_cast<O *>(dst);
    const long long stride = (long long)gridDim.x * kThreads;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
    const long long n8 = vec_ok ? n / 8 : 0;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n8; i += stride) {
        uint4 w = *reinterpret_cast<const uint4 *>(src + i * 8);
        uint32_t ws[4] = {w.x, w.y, w.z, w.w};
        if constexpr (OUT == kBF16) {
            st_global_v4(out + i * 8, ws[0], ws[1], ws[2], ws[3]);
        } else if constexpr (OUT == kF32) {
            st_global_v4(out + i * 8, ws[0] << 16, ws[0] & 0xFFFF0000u, ws[1] << 16, ws[1] & 0xFFFF0000u);
            st_global_v4(out + i * 8 + 4, ws[2] << 16, ws[2] & 0xFFFF0000u, ws[3] << 16, ws[3] & 0xFFFF0000u);
        } else {
            uint32_t r[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                __half2 h = __floats2half2_rn(__uint_as_float(ws[j] << 16), __uint_as_float(ws[j] & 0xFFFF0000u));
                r[j] = *reinterpret_cast<uint32_t *>(&h);
            }
            st_global_v4(out + i * 8, r[0], r[1], r[2], r[3]);
        }
    }
    for (long long i = n8 * 8 + (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
        float f = __uint_as_float((uint32_t)src[i] << 16);
        if constexpr (OUT == kF16) out[i] = __float2half_rn(f);
        else if constexpr (OUT == kBF16) out[i] = __float2bfloat16_rn(f);
        else out[i] = f;
    }
}

// integer-unpack debug kernel: exercises exactly the q4()/scales() the product kernels use
template <class Q>
__global__ void unpack_int_kernel(const uint8_t *__restrict__ src, long long n_blocks, int16_t *q, int16_t *sc, int16_t *mn)
{
    const long long n4 = n_blocks * (Q::BS / 4);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / (Q::BS / 4);
        const int e0 = (int)(i % (Q::BS / 4)) * 4;
        // global pointers carry no alignment guarantee here -> byte-assemble through a local copy
        uint8_t local[Q::TS + 2] __attribute__((aligned(16)));
        for (int k = 0; k < Q::TS; ++k) local[k] = src[b * Q::TS + k];
        uint32_t u = Q::q4(local, e0);
        int s, m;
        Q::scales(local, e0, s, m);
        for (int j = 0; j < 4; ++j) {
            long long o = b * Q::BS + e0 + j;
            if (q) q[o] = (int16_t)((int)((u >> (8 * j)) & 0xFF) - Q::BIAS);
            if (sc) sc[o] = (int16_t)s;
            if (mn) mn[o] = (int16_t)m;
        }
    }
}

// ------------------------------------------------------------------ host-side dispatch
// The K1 launch geometry of one (format, output dtype): shared memory of dequant_kernel, tiles, and the output tensor map.
template <class Q, int OUT> struct K1Geometry {
    static constexpr int THREADS = kThreads;
    static constexpr int TILE_BLOCKS = THREADS * 32 / Q::BS;
    static constexpr int OB = OutT<OUT>::bytes;
    static constexpr int TB = ((TILE_BLOCKS * Q::TS + 16 + 15) & ~15);
    static constexpr int SMEM = THREADS * 32 * OB + TB + 16;

    // the output as [runs of 32 elements][64 | 128 bytes]: one row per thread, one box of THREADS rows per tile
    static int encode(CUtensorMap *tmOut, void *out, long long n_blocks)
    {
        TensorMapEncodeFn fn = tensor_map_encode_fn();
        const long long n_rows = n_blocks * (long long)Q::BS / 32;
        if (!fn || n_rows > 0x7fffffffll) return GGUFB200_E_CUDA;
        cuuint64_t dims[2] = {(cuuint64_t)(32 * OB), (cuuint64_t)n_rows};
        cuuint64_t strides[1] = {(cuuint64_t)(32 * OB)};
        cuuint32_t box[2] = {(cuuint32_t)(32 * OB), (cuuint32_t)THREADS};
        cuuint32_t estr[2] = {1, 1};
        if (fn(tmOut, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, out, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               OB == 2 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return GGUFB200_E_CUDA;
        return GGUFB200_OK;
    }
};

// One CTA per tile, programmatic stream serialization as set by ggufb200_set_tuning(1, .): shared by both K1 kernels.
template <class Kernel, class... Args>
static int launch_k1(Kernel kern, long long n_tiles, int smem, cudaStream_t st, Args... args)
{
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)n_tiles);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = g_dequant_pdl ? 1 : 0;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, args...);
    return e == cudaSuccess ? GGUFB200_OK : GGUFB200_E_CUDA;
}

template <class Q, int MATH, int OUT> static int launch_dequant(const void *packed, long long n_blocks, void *out, bool src_stable, cudaStream_t st)
{
    using G = K1Geometry<Q, OUT>;
    auto kern = dequant_kernel<Q, MATH, OUT, G::THREADS>;
    static unsigned char smem_set[64] = {};
    if (!ensure_dynamic_smem(kern, G::SMEM, smem_set)) return GGUFB200_E_CUDA;
    const long long n_tiles = (n_blocks + G::TILE_BLOCKS - 1) / G::TILE_BLOCKS;
    if (n_tiles > 0x7fffffffll) return GGUFB200_E_SHAPE;
    CUtensorMap tmOut{};
    if (int rc = G::encode(&tmOut, out, n_blocks)) return rc;
    int flags = ((reinterpret_cast<uintptr_t>(packed) & 15) == 0) ? 1 : 0;
    if (src_stable) flags |= 2;
    return launch_k1(kern, n_tiles, G::SMEM, st, tmOut, reinterpret_cast<const uint8_t *>(packed), out, (long long)n_blocks, flags);
}

// `stage_bytes`: room for the B rows of the weight rows one tile touches (the largest staged patch)
template <class Q, int MATH, int OUT>
static int launch_dequant_kron(const void *packed, long long n_blocks, void *out, bool src_stable, const KronArgs &kron, int stage_bytes,
                               cudaStream_t st)
{
    using G = K1Geometry<Q, OUT>;
    auto kern = dequant_kron_kernel<Q, MATH, OUT, G::THREADS>;
    static unsigned char smem_set[64] = {};
    if (!ensure_dynamic_smem(kern, G::SMEM + kKronStageBytes, smem_set)) return GGUFB200_E_CUDA;
    const long long n_tiles = (n_blocks + G::TILE_BLOCKS - 1) / G::TILE_BLOCKS;
    if (n_tiles > 0x7fffffffll) return GGUFB200_E_SHAPE;
    CUtensorMap tmOut{};
    if (int rc = G::encode(&tmOut, out, n_blocks)) return rc;
    int flags = ((reinterpret_cast<uintptr_t>(packed) & 15) == 0) ? 1 : 0;
    if (src_stable) flags |= 2;
    return launch_k1(kern, n_tiles, G::SMEM + stage_bytes, st, tmOut, reinterpret_cast<const uint8_t *>(packed), (long long)n_blocks, flags, kron);
}

// the (format, math, output) instance of either K1 kernel: f(Q{}, MathTag, OutTag)
template <class Q, class F> static int dispatch_math_out(int math_dtype, int out_dtype, F &&f)
{
    auto by_out = [&](auto math) {
        switch (out_dtype) {
        case kF16: return f(math, std::integral_constant<int, kF16>{});
        case kBF16: return f(math, std::integral_constant<int, kBF16>{});
        case kF32: return f(math, std::integral_constant<int, kF32>{});
        }
        return (int)GGUFB200_E_DTYPE;
    };
    switch (math_dtype) {
    case kF16: return by_out(std::integral_constant<int, kF16>{});
    case kBF16: return by_out(std::integral_constant<int, kBF16>{});
    case kF32: return by_out(std::integral_constant<int, kF32>{});
    }
    return GGUFB200_E_DTYPE;
}

template <class Q> static int dispatch_math(const void *packed, long long n_blocks, void *out, int out_dtype, int math_dtype, bool stable, cudaStream_t st)
{
    return dispatch_math_out<Q>(math_dtype, out_dtype, [&](auto math, auto o) {
        return launch_dequant<Q, decltype(math)::value, decltype(o)::value>(packed, n_blocks, out, stable, st);
    });
}

int dequant_dispatch(int type, const void *packed, long long n_blocks, void *out, int out_dtype, int math_dtype, cudaStream_t st, bool stable)
{
    if (n_blocks == 0) return GGUFB200_OK;
    if (type == T_BF16) {
        // one 8-element vector per thread, CTAs in address order (the grid-stride loop of the kernel only runs past the first
        // iteration for tensors beyond 2^31 CTAs): same reasoning as for the block formats above
        long long blocks = (n_blocks + (long long)kThreads * 8 - 1) / ((long long)kThreads * 8);
        long long cap = 0x7fffffffll;
        unsigned grid = (unsigned)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
        const uint16_t *s = reinterpret_cast<const uint16_t *>(packed);
        if (out_dtype == kF16) bf16_kernel<kF16><<<grid, kThreads, 0, st>>>(s, out, n_blocks);
        else if (out_dtype == kBF16) bf16_kernel<kBF16><<<grid, kThreads, 0, st>>>(s, out, n_blocks);
        else if (out_dtype == kF32) bf16_kernel<kF32><<<grid, kThreads, 0, st>>>(s, out, n_blocks);
        else return GGUFB200_E_DTYPE;
        return cudaGetLastError() == cudaSuccess ? GGUFB200_OK : GGUFB200_E_CUDA;
    }
    return with_block(type, GGUFB200_E_TYPE, [&](auto blk) {
        return dispatch_math<decltype(blk)>(packed, n_blocks, out, out_dtype, math_dtype, stable, st);
    });
}

int dequant_kron_dispatch(int type, const void *packed, long long N, long long K, void *out, int out_dtype, int math_dtype,
                          const ggufb200_kron_patch *patches, int n_patches, cudaStream_t st, bool stable)
{
    // weight rows one 4096-element tile can touch
    const long long tile_rows = (kThreads * 32 - 1) / K + 2;
    KronArgs ka{};
    ka.n = n_patches;
    ka.K = (int)K;
    int stage_bytes = 0;
    for (int i = 0; i < n_patches; ++i) {
        const ggufb200_kron_patch &p = patches[i];
        KronOp &op = ka.op[i];
        op.A = p.A;
        op.B = p.B;
        op.a2 = (int)p.a2;
        op.b1 = (int)p.b1;
        op.b2 = (int)p.b2;
        op.r0 = p.band_dim == 0 ? (int)p.band_start : 0;
        op.rows = (int)(p.a1 * p.b1);
        op.c0 = p.band_dim == 1 ? (int)p.band_start : 0;
        op.cols = (int)(p.a2 * p.b2);
        op.scale = p.scale;
        const long long bytes = (tile_rows < op.rows ? tile_rows : op.rows) * p.b2 * 4;
        op.staged = bytes <= kKronStageBytes;
        if (op.staged && bytes > stage_bytes) stage_bytes = (int)bytes;
    }
    return with_block(type, GGUFB200_E_TYPE, [&](auto blk) {
        using Q = decltype(blk);
        return dispatch_math_out<Q>(math_dtype, out_dtype, [&](auto math, auto o) {
            return launch_dequant_kron<Q, decltype(math)::value, decltype(o)::value>(packed, N * K / Q::BS, out, stable, ka, stage_bytes, st);
        });
    });
}

template <class Q> static int launch_unpack(const void *packed, long long n_blocks, int16_t *q, int16_t *sc, int16_t *mn, cudaStream_t st)
{
    long long n4 = n_blocks * (Q::BS / 4);
    long long blocks = (n4 + 127) / 128;
    if (blocks > 65535) blocks = 65535;
    unpack_int_kernel<Q><<<(unsigned)blocks, 128, 0, st>>>(reinterpret_cast<const uint8_t *>(packed), n_blocks, q, sc, mn);
    return cudaGetLastError() == cudaSuccess ? GGUFB200_OK : GGUFB200_E_CUDA;
}

int unpack_dispatch(int type, const void *packed, long long n_blocks, int16_t *q, int16_t *sc, int16_t *mn, cudaStream_t st)
{
    if (n_blocks == 0) return GGUFB200_OK;
    return with_block(type, GGUFB200_E_TYPE, [&](auto blk) { return launch_unpack<decltype(blk)>(packed, n_blocks, q, sc, mn, st); });
}

}  // namespace ggufb200
