"""GPU parity tests of the tensor-core Linear kernels: dense TMA-fed GEMM (csrc/gemm3.cu), the shared-memory-fed fused
kernel (csrc/gemm2.cu, reference-exact W) and the FUSED_TMEM kernel (csrc/gemm4.cu, the AUTO default).

Reference: fp32-accumulated x @ W^T (+bias) rounded to the activation dtype, where W is the bit-exact dequantised weight
(validated separately against the reference's golden outputs).

Tolerances (DESIGN.md section 3), relative Frobenius:
  * routes whose weight operand is bit-identical to the reference's (GEMV, FUSED_MMA, DEQUANT_MMA): 1e-3 in every dtype
    (north_star's figure; only the fp32 summation order differs).
  * FUSED_TMEM with FLAG_GENERIC (functor producers) or FLAG_EXACT_W (hand-written producers, reference sequence): the weight
    operand is bit-identical as well (fp16 chain, then the cast to bf16 for bf16 activations) -> 3e-4 asserted.
  * FUSED_TMEM default ("fast": Q4_K / Q5_K use ONE fused multiply-add per element instead of multiply + subtract):
      fp16 activations:  1e-3 against the reference arithmetic (measured ~4e-4);
      bf16 activations:  8e-3 = the same bound expressed in bf16 ulps (2^3 coarser than fp16), because ANY weight that is not
                         bit-identical to bf16(W_ref) moves a bf16 Linear by ~2e-3 (measured 1.9e-3) -- even the exactly
                         dequantised weight would.  What is asserted in addition: the result is as close to the fp64 product
                         of the exact weight as the reference's own result is (within 5 %)."""
import numpy as np
import pytest
import torch
import gguf

import oracle
from util import Q, rel_fro

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-3
TOL_TMEM = {torch.float16: 1e-3, torch.bfloat16: 8e-3}
BLOCK_TYPES = [Q.Q4_0, Q.Q4_1, Q.Q5_0, Q.Q5_1, Q.Q8_0, Q.Q2_K, Q.Q3_K, Q.Q4_K, Q.Q5_K, Q.Q6_K, Q.IQ4_NL, Q.IQ4_XS]
TMEM_TYPES = [Q.Q4_0, Q.Q4_1, Q.Q5_0, Q.Q5_1, Q.Q8_0, Q.Q4_K, Q.Q5_K, Q.IQ4_NL]     # canonical row layout is TMA-legal (span % 16 == 0)


def _ref(x, W, bias):
    y = x.float() @ W.float().t()
    if bias is not None:
        y = y + bias.to(x.dtype).float()
    return y.to(x.dtype)


def _weight(pkg, qt, N, K, seed=0):
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    raw = oracle.random_blocks(int(qt), N * K // bs, seed=seed, scale=0.02).reshape(N, K // bs * ts)
    return raw, pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=qt, tensor_shape=torch.Size((N, K)))


def _ideal(pkg, x, w, bias):
    """fp64 product with the EXACT dequantised weight d*sc*q - dmin*mn (fp32 math: no fp16 rounding anywhere); no output
    rounding.  The yardstick for 'at least as accurate as the reference'."""
    w32 = pkg.dequant.dequantize_tensor(w, torch.float32, torch.float32)
    y = x.double() @ w32.double().t()
    if bias is not None:
        y = y + bias.to(x.dtype).double()
    return y


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (300, 264, 512), (1000, 128, 3072), (24, 512, 256), (513, 1032, 1024), (300, 264, 200)])
def test_dense_gemm_matches_torch(pkg, dt, M, N, K):
    """(300, 264, 200): K not a multiple of the 64-wide k-block -- the ragged tail is zero-filled by the TMA engine."""
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    x = torch.randn(M, K, device=DEV, dtype=dt, generator=g)
    W = (torch.randn(N, K, device=DEV, generator=g) * 0.05).to(dt)
    b = torch.randn(N, device=DEV, generator=g) * 0.1
    y = pkg.ops.linear_dense(x, W, b)
    ref = _ref(x, W, b)
    assert rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy()) <= TOL
    y2 = pkg.ops.linear_dense(x, W, None)
    assert rel_fro(y2.float().cpu().numpy(), _ref(x, W, None).float().cpu().numpy()) <= TOL


# ---------------------------------------------------------------- shared-memory-fed fused kernel (reference-exact W)
@pytest.mark.parametrize("staged", [True, False], ids=["staged", "direct"])
@pytest.mark.parametrize("qt", BLOCK_TYPES, ids=lambda q: q.name)
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_fused_gemm_all_types(pkg, qt, dt, staged):
    M, N, K = 300, 264, 1024
    _raw, w = _weight(pkg, qt, N, K, seed=int(qt))
    x = torch.randn(M, K, device=DEV, dtype=dt)
    b = torch.randn(N, device=DEV) * 0.1
    algo = pkg.lib.ALGO_FUSED_MMA | (0 if staged else pkg.lib.FLAG_UNSTAGED)
    y = pkg.ops.linear_packed(x, w, b, None, algo)
    W = pkg.dequant.dequantize_tensor(w, dt)
    assert rel_fro(y.float().cpu().numpy(), _ref(x, W, b).float().cpu().numpy()) <= TOL


@pytest.mark.parametrize("qt", [Q.Q4_K, Q.Q8_0, Q.Q6_K, Q.Q5_0], ids=lambda q: q.name)
@pytest.mark.parametrize("M,N,K", [(64, 512, 4096), (300, 264, 2048), (513, 520, 1280), (1000, 256, 5120), (24, 1032, 768)])
def test_fused_gemm_split_k(pkg, qt, M, N, K):
    """Short activations: the fused kernel cuts K into ranges of whole 256-wide spans, one SM pair per (tile, range), keeps
    fp32 partial tiles in the workspace and sums them in a fixed order (bit-reproducible).  Checked against the reference
    arithmetic and against the unsplit kernel (same tiles, no workspace): the two may differ only by fp32 summation order."""
    L = pkg.lib.lib()
    _raw, w = _weight(pkg, qt, N, K, seed=int(qt) + K)
    W = pkg.dequant.dequantize_tensor(w, torch.bfloat16)
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    b = torch.randn(N, device=DEV) * 0.1
    need = L.ggufb200_linear_workspace(int(qt), M, N, K, 1, pkg.lib.ALGO_FUSED_MMA)
    assert need % (M * N * 4) == 0 and need >= 2 * M * N * 4, "these shapes leave SM pairs idle without split-K"
    y = pkg.ops.linear_packed(x, w, b, None, pkg.lib.ALGO_FUSED_MMA)
    assert torch.equal(y, pkg.ops.linear_packed(x, w, b, None, pkg.lib.ALGO_FUSED_MMA)), "split-K must be reproducible"
    nosplit = pkg.lib.ALGO_FUSED_MMA | pkg.lib.FLAG_NOSPLIT
    assert L.ggufb200_linear_workspace(int(qt), M, N, K, 1, nosplit) == 0
    y1 = pkg.ops.linear_packed(x, w, b, None, nosplit)
    ref = _ref(x, W, b).float().cpu().numpy()
    assert rel_fro(y.float().cpu().numpy(), ref) <= TOL
    assert rel_fro(y1.float().cpu().numpy(), ref) <= TOL
    assert rel_fro(y.float().cpu().numpy(), y1.float().cpu().numpy()) <= 2e-3   # bf16 output rounding of two fp32 orders
    ya = pkg.ops.linear_packed(x, w, None, None, pkg.lib.ALGO_AUTO | pkg.lib.FLAG_EXACT_W)
    assert rel_fro(ya.float().cpu().numpy(), _ref(x, W, None).float().cpu().numpy()) <= TOL


def test_fused_split_k_without_workspace_runs_unsplit(pkg):
    """The C ABI never allocates: FUSED_MMA with a NULL workspace must still be correct (one pair per tile)."""
    qt, M, N, K = Q.Q4_K, 64, 512, 4096
    raw = oracle.random_blocks(int(qt), N * K // 256, seed=9, scale=0.02).reshape(N, K // 256 * 144)
    w = torch.from_numpy(raw).to(DEV)
    x = torch.randn(M, K, device=DEV, dtype=torch.float16)
    L = pkg.lib.lib()
    gw = pkg.ops.GGMLTensor(w, tensor_type=qt, tensor_shape=torch.Size((N, K)))
    W = pkg.dequant.dequantize_tensor(gw, torch.float16)
    for algo in (pkg.lib.ALGO_FUSED_MMA, pkg.lib.ALGO_FUSED_TMEM):
        y = torch.empty(M, N, device=DEV, dtype=torch.float16)
        rc = L.ggufb200_linear(int(qt), w.data_ptr(), N, K, x.data_ptr(), M, K, 0, 0, None, 0, y.data_ptr(), N, None, 0,
                               algo, torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        assert rel_fro(y.float().cpu().numpy(), _ref(x, W, None).float().cpu().numpy()) <= TOL


@pytest.mark.parametrize("route", ["fused", "dequant+mma", "auto", "auto-exact"])
def test_sd35_shape_q8_0_unaligned_rows(pkg, route):
    """SD3.5-large hidden size 2432: Q8_0 rows are 2584 bytes (not a multiple of 16), so no tensor map over the packed bytes
    is legal; the fused kernel must take its direct-load producer and K1 its flat byte-stream tiling."""
    M, N, K = 700, 7296, 2432
    _raw, w = _weight(pkg, Q.Q8_0, N, K, seed=2)
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    b = torch.randn(N, device=DEV) * 0.1
    algo = {"fused": pkg.lib.ALGO_FUSED_MMA, "dequant+mma": pkg.lib.ALGO_DEQUANT_MMA, "auto": pkg.lib.ALGO_AUTO,
            "auto-exact": pkg.lib.ALGO_AUTO | pkg.lib.FLAG_EXACT_W}[route]
    y = pkg.ops.linear_packed(x, w, b, None, algo)
    W = pkg.dequant.dequantize_tensor(w, torch.bfloat16)
    assert rel_fro(y.float().cpu().numpy(), _ref(x, W, b).float().cpu().numpy()) <= TOL      # (AUTO cannot take the TMEM route here)


@pytest.mark.parametrize("M,N,K", [(4608, 3072, 3072), (512, 9216, 3072), (4096, 3072, 12288)])
def test_fused_gemm_flux_shapes_q4k(pkg, M, N, K):
    """Full Flux.1 Linear sizes: the oracle is too slow here, so compare against fp32-accumulated products of the same
    bit-exact K1 weight: bf16(W) for the reference-exact routes, and the fp64 ideal for the TMEM route."""
    qt = Q.Q4_K
    _raw, w = _weight(pkg, qt, N, K, seed=1)
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    W = pkg.dequant.dequantize_tensor(w, torch.bfloat16)
    ref = torch.nn.functional.linear(x, W)
    for algo in (pkg.lib.ALGO_FUSED_MMA, pkg.lib.ALGO_DEQUANT_MMA):
        y = pkg.ops.linear_packed(x, w, None, None, algo)
        assert rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy()) <= TOL
    W32 = pkg.dequant.dequantize_tensor(w, torch.float32, torch.float32)
    ideal = (x.float() @ W32.t()).double()                  # exact weight, fp32 accumulate: ~1e-6 from the fp64 product
    del W32
    for algo in (pkg.lib.ALGO_FUSED_TMEM, pkg.lib.ALGO_FUSED_TMEM | pkg.lib.FLAG_TILE384, pkg.lib.ALGO_FUSED_TMEM | pkg.lib.FLAG_GENERIC,
                 pkg.lib.ALGO_FUSED_TMEM | pkg.lib.FLAG_EXACT_W):
        y = pkg.ops.linear_packed(x, w, None, None, algo)
        exact = bool(algo & (pkg.lib.FLAG_GENERIC | pkg.lib.FLAG_EXACT_W))
        assert rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy()) <= (3e-4 if exact else TOL_TMEM[torch.bfloat16])
        err_ours = (y.double() - ideal).norm().item()
        err_ref = (ref.double() - ideal).norm().item()
        assert err_ours <= 1.05 * err_ref, (algo, err_ours, err_ref)


# ---------------------------------------------------------------- FUSED_TMEM kernel (csrc/gemm4.cu)
PRODUCERS = {"fast": 0, "generic": 0x200, "exact": 0x100}      # default / GGUFB200_FLAG_GENERIC / GGUFB200_FLAG_EXACT_W


@pytest.mark.parametrize("producers", list(PRODUCERS))
@pytest.mark.parametrize("qt", TMEM_TYPES, ids=lambda q: q.name)
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_tmem_fused_all_types(pkg, qt, dt, producers):
    """Every format whose canonical rows can be staged by a 2-D tensor map, all three producer families, ragged M and N."""
    M, N, K = 300, 264, 1024
    _raw, w = _weight(pkg, qt, N, K, seed=int(qt) + 3)
    x = torch.randn(M, K, device=DEV, dtype=dt)
    b = torch.randn(N, device=DEV) * 0.1
    y = pkg.ops.linear_packed(x, w, b, None, pkg.lib.ALGO_FUSED_TMEM | PRODUCERS[producers])
    W = pkg.dequant.dequantize_tensor(w, dt)
    ref = _ref(x, W, b)
    assert rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy()) <= TOL_TMEM[dt]
    ideal = _ideal(pkg, x, w, b)
    assert (y.double() - ideal).norm().item() <= 1.05 * (ref.double() - ideal).norm().item()
    if producers != "fast" or qt not in (Q.Q4_K, Q.Q5_K):
        # reference rounding sequence: the weight operand IS the reference's (in fp16 and in bf16) -> only summation order differs
        assert rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy()) <= 3e-4


@pytest.mark.parametrize("M,N,K", [(1, 512, 1024), (3, 200, 768), (8, 1032, 4096), (24, 512, 256), (33, 264, 512), (128, 256, 256),
                                   (129, 512, 1280), (192, 256, 512), (193, 264, 1024), (385, 520, 768), (513, 1032, 1024),
                                   (1000, 128, 3072), (64, 512, 4096), (700, 768, 320)])
@pytest.mark.parametrize("tile384", [False, True], ids=["tile192", "tile384"])
def test_tmem_fused_shapes(pkg, M, N, K, tile384):
    """Token tiles of 32 / 128 / 192 (and 384), ragged edges, K ranges (split-K) for short activations, K % 256 != 0."""
    qt = Q.Q4_K if K % 256 == 0 else Q.Q5_1      # Q5_1 rows of 320 elements are 240 bytes: TMA-legal with a ragged last span
    _raw, w = _weight(pkg, qt, N, K, seed=M + N + K)
    x = torch.randn(M, K, device=DEV, dtype=torch.float16)
    b = torch.randn(N, device=DEV) * 0.1
    algo = pkg.lib.ALGO_FUSED_TMEM | (pkg.lib.FLAG_TILE384 if tile384 else 0)
    y = pkg.ops.linear_packed(x, w, b, None, algo)
    assert torch.equal(y, pkg.ops.linear_packed(x, w, b, None, algo)), "must be run-to-run reproducible (no atomics)"
    W = pkg.dequant.dequantize_tensor(w, torch.float16)
    ref = _ref(x, W, b)
    assert rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy()) <= TOL
    y1 = pkg.ops.linear_packed(x, w, b, None, algo | pkg.lib.FLAG_NOSPLIT)
    assert rel_fro(y1.float().cpu().numpy(), ref.float().cpu().numpy()) <= TOL


def test_tmem_fused_many_items_per_pair(pkg):
    """More CTAs than SMs: several waves of (feature tile, token tile) CTAs, with 192- and 384-token items -- exercises the
    tile decode of the grid and the ring parities over long K loops."""
    M, N, K = 1536, 8192, 512          # 32 feature tiles x 8 token tiles = 256 items, 512 CTAs on 132 SMs
    _raw, w = _weight(pkg, Q.Q4_K, N, K, seed=77)
    x = torch.randn(M, K, device=DEV, dtype=torch.float16)
    W = pkg.dequant.dequantize_tensor(w, torch.float16)
    ref = _ref(x, W, None)
    for flags in (0, pkg.lib.FLAG_TILE384):
        y = pkg.ops.linear_packed(x, w, None, None, pkg.lib.ALGO_FUSED_TMEM | flags)
        assert rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy()) <= TOL


def test_auto_route_large_m_through_layer(pkg):
    lin = pkg.ops.GGMLOps.Linear(1024, 264)
    raw = oracle.random_blocks(int(Q.Q5_K), 264 * 4, seed=3, scale=0.02).reshape(264, 4 * 176)
    w = pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=Q.Q5_K, tensor_shape=torch.Size((264, 1024)))
    lin.load_state_dict({"weight": w})
    x = torch.randn(2, 200, 1024, device=DEV, dtype=torch.bfloat16)
    W = pkg.dequant.dequantize_tensor(w, torch.bfloat16)
    ref = _ref(x.reshape(-1, 1024), W, None).float().cpu().numpy()
    y = lin(x)
    assert tuple(y.shape) == (2, 200, 264)
    assert rel_fro(y.float().cpu().numpy(), ref) <= TOL_TMEM[torch.bfloat16]
    lin.linear_numerics = "exact"
    assert rel_fro(lin(x).float().cpu().numpy(), ref) <= TOL


# ---------------------------------------------------------------- span-major shadow layout (csrc/repack.cu, SURVEY 8f rank 3)
def _pitch(qt):
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    span = 256 // bs * ts
    if span % 16 == 0:
        return span, span
    pad = (span + 15) // 16 * 16
    return span, pad if (pad // 16) % 2 == 1 else pad + 16


@pytest.mark.parametrize("qt", BLOCK_TYPES, ids=lambda q: q.name)
@pytest.mark.parametrize("N,K", [(300, 768), (264, 1280), (130, 320)])
def test_repack_layout_is_a_pure_byte_permutation(pkg, qt, N, K):
    """out[span][row padded to 256][pitch]: the canonical bytes of (row, span), zero padding everywhere else -- bit-exact."""
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    if K % bs:
        pytest.skip("K must be a multiple of the block size")
    raw, w = _weight(pkg, qt, N, K, seed=int(qt) + N)
    got = pkg.ops.span_layout(w, pkg.ops._plain(w)).cpu().numpy()
    span, pitch = _pitch(qt)
    spans, n_pad, row_bytes = -(-K // 256), -(-N // 256) * 256, K // bs * ts
    want = np.zeros((spans, n_pad, pitch), dtype=np.uint8)
    for s in range(spans):
        chunk = raw[:, s * span:min((s + 1) * span, row_bytes)]
        want[s, :N, :chunk.shape[1]] = chunk
    assert got.size == want.size == pkg.lib.lib().ggufb200_repack_bytes(int(qt), N, K)
    assert np.array_equal(got.reshape(want.shape), want)
    assert pkg.ops.span_layout(w, pkg.ops._plain(w)).data_ptr() == pkg.ops.span_layout(w, pkg.ops._plain(w)).data_ptr()   # cached


@pytest.mark.parametrize("producers", list(PRODUCERS))
@pytest.mark.parametrize("qt", BLOCK_TYPES, ids=lambda q: q.name)
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_tmem_fused_from_span_layout_all_types(pkg, qt, dt, producers):
    """Every block format -- including the ones no tensor map can stage (Q2_K / Q3_K / Q6_K / IQ4_XS) -- on the FUSED_TMEM kernel."""
    M, N, K = 300, 264, 1024
    _raw, w = _weight(pkg, qt, N, K, seed=int(qt) + 5)
    x = torch.randn(M, K, device=DEV, dtype=dt)
    b = torch.randn(N, device=DEV) * 0.1
    algo = pkg.lib.ALGO_FUSED_TMEM | PRODUCERS[producers]
    y = pkg.ops.linear_packed(x, w, b, None, algo, use_spans=True)
    W = pkg.dequant.dequantize_tensor(w, dt)
    ref = _ref(x, W, b)
    assert rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy()) <= TOL_TMEM[dt]
    ideal = _ideal(pkg, x, w, b)
    assert (y.double() - ideal).norm().item() <= 1.05 * (ref.double() - ideal).norm().item()
    if producers != "fast" or qt not in (Q.Q4_K, Q.Q5_K):
        assert rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy()) <= 3e-4
    if qt in TMEM_TYPES:
        assert torch.equal(y, pkg.ops.linear_packed(x, w, b, None, algo)), "span-major and canonical staging must agree bit for bit"


@pytest.mark.parametrize("M", [2, 700])
def test_sd35_shape_q8_0_rows_run_on_the_tmem_kernel_through_the_layer(pkg, M):
    """SD3.5-large hidden size 2432: 2584-byte Q8_0 rows.  The layer builds the span-major copy on first use and the FUSED_TMEM
    kernel serves it (K = 2432 is not a multiple of 256: the last span is half empty); at M = 2 this 17.7 M-element weight stays on
    the mma.sync GEMV."""
    N, K = 7296, 2432
    _raw, w = _weight(pkg, Q.Q8_0, N, K, seed=2)
    lin = pkg.ops.GGMLOps.Linear(K, N)
    lin.load_state_dict({"weight": w})
    x = torch.randn(M, K, device=DEV, dtype=torch.float16)
    y = lin(x)
    # the span-major copy is built for the FUSED_TMEM kernel only: M > 8, or M <= 8 on a weight large enough for that kernel to win
    assert ("_gg_spans" in lin.weight.__dict__) == (M > 8)
    W = pkg.dequant.dequantize_tensor(w, torch.float16)
    assert rel_fro(y.float().cpu().numpy(), _ref(x, W, None).float().cpu().numpy()) <= TOL
    lin.repack_spans = False
    y2 = lin(x)
    assert rel_fro(y2.float().cpu().numpy(), _ref(x, W, None).float().cpu().numpy()) <= TOL
