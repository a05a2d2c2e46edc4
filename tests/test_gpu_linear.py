"""GPU parity tests of the Linear path (csrc/gemv.cu, gemv2.cu, linear_sm90.cu) through the plugin surface.

Tolerance (written here, from BASELINE.json north_star): ||y - y_ref||_F / ||y_ref||_F <= 1e-3 for fp16/bf16 Linear
outputs; y_ref is the unmodified reference's GGMLOps.Linear output (golden files) or the CPU oracle.
Every layer-level test runs under both numerics contracts of GGMLOps.Linear (`linear_numerics`): "exact" (the default: weight
operand bit-identical to the reference's: 1e-3 in every dtype) and "fast" (fused-multiply-add producers on the FUSED_TMEM
kernel: 1e-3 for fp16 activations, 8e-3 = the same bound in bf16 ulps for bf16 activations -- see tests/test_gpu_gemm.py and
DESIGN.md section 3)."""
import os

import numpy as np
import pytest
import torch
import gguf

import oracle
from util import Q, bits_to_f32, rel_fro, torch_bits

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-3


@pytest.fixture(params=["exact", "fast"], autouse=True)
def numerics(request, pkg):
    """Layer-level tests run under both numerics contracts (a class attribute, like dequant_dtype / patch_dtype)."""
    cls = pkg.ops.GGMLOps.Linear
    before = cls.linear_numerics
    cls.linear_numerics = request.param
    yield request.param
    cls.linear_numerics = before


def _tol(numerics, dt):
    return 8e-3 if (numerics == "fast" and dt == torch.bfloat16) else TOL


def _weight(pkg, qt, N, K, seed=0, scale=0.02):
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    raw = oracle.random_blocks(int(qt), N * K // bs, seed=seed, scale=scale).reshape(N, K // bs * ts)
    return raw, pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=qt, tensor_shape=torch.Size((N, K)))


def _layer(pkg, qt, N, K, bias=True, seed=0):
    raw, w = _weight(pkg, qt, N, K, seed)
    lin = pkg.ops.GGMLOps.Linear(K, N)
    sd = {"weight": w}
    b = None
    if bias:
        b = np.random.default_rng(seed + 1).normal(0, 0.02, size=N).astype(np.float32)
        sd["bias"] = pkg.ops.GGMLTensor(torch.from_numpy(b).to(DEV), tensor_type=Q.F32, tensor_shape=torch.Size((N,)))
    lin.load_state_dict(sd)
    return lin, raw, b


@pytest.mark.parametrize("name", ["Q4_K", "Q8_0", "Q5_K", "Q6_K", "Q4_0", "BF16"])
@pytest.mark.parametrize("act,code,dt", [("bf16", 1, torch.bfloat16), ("f16", 0, torch.float16), ("f32", 2, torch.float32)])
def test_linear_matches_reference_ops_golden(pkg, name, act, code, dt, golden_dir, numerics):
    """x (24 rows) through the drop-in GGMLOps.Linear vs the y the reference's GGMLOps.Linear produced."""
    g = np.load(os.path.join(golden_dir, f"linear_{name}_{act}.npz"))
    qt = Q(int(g["qtype"]))
    N, K, M = int(g["N"]), int(g["K"]), int(g["M"])
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    lin = pkg.ops.GGMLOps.Linear(K, N)
    w = pkg.ops.GGMLTensor(torch.from_numpy(g["packed"].reshape(N, K // bs * ts)).to(DEV), tensor_type=qt, tensor_shape=torch.Size((N, K)))
    b = pkg.ops.GGMLTensor(torch.from_numpy(g["bias"]).to(DEV), tensor_type=Q.F32, tensor_shape=torch.Size((N,)))
    lin.load_state_dict({"weight": w, "bias": b})
    xb = g["x"]
    x = torch.from_numpy(xb.view(np.float32) if code == 2 else xb.view(np.int16)).to(DEV)
    x = x.view(dt).reshape(M, K)
    want = bits_to_f32(g["y"].reshape(-1), code)
    for rows in (M, 5, 1):                       # M=24 -> large-M route, 5 and 1 -> fused GEMV
        y = lin(x[:rows])
        assert type(y) is torch.Tensor and y.dtype == dt and tuple(y.shape) == (rows, N)
        got = y.float().cpu().numpy().reshape(-1)
        assert rel_fro(got, want[: rows * N]) <= _tol(numerics, dt), (name, act, rows)


@pytest.mark.parametrize("qt", [Q.Q4_0, Q.Q4_1, Q.Q5_0, Q.Q5_1, Q.Q8_0, Q.Q2_K, Q.Q3_K, Q.Q4_K, Q.Q5_K, Q.Q6_K, Q.IQ4_NL, Q.IQ4_XS],
                         ids=lambda q: q.name)
@pytest.mark.parametrize("M", [1, 3, 8])
def test_gemv_all_types_vs_oracle(pkg, qt, M):
    N, K = 200, 1024
    raw, w = _weight(pkg, qt, N, K, seed=int(qt))
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    bias = torch.randn(N, device=DEV, dtype=torch.float32) * 0.1
    y = pkg.ops.linear_packed(x, w, bias, None, pkg.lib.ALGO_GEMV)
    bias_bits = torch_bits(bias.to(torch.bfloat16))
    want = oracle.linear(raw, int(qt), N, K, torch_bits(x), oracle.DT_BF16, oracle.DT_F16, bias_bits)
    assert rel_fro(y.float().cpu().numpy(), bits_to_f32(want.reshape(-1), 1)) <= TOL


def test_gemv_dequant_dtype_modes_and_fp16(pkg):
    raw, w = _weight(pkg, Q.Q4_K, 128, 512, seed=5)
    for act, code in ((torch.float16, 0), (torch.bfloat16, 1)):
        x = torch.randn(2, 512, device=DEV, dtype=act)
        for mode, mcode in ((None, 0), ("target", code), (torch.float32, 2)):
            y = pkg.ops.linear_packed(x, w, None, mode, pkg.lib.ALGO_GEMV)
            want = oracle.linear(raw, int(Q.Q4_K), 128, 512, torch_bits(x), code, mcode, None)
            assert rel_fro(y.float().cpu().numpy(), bits_to_f32(want.reshape(-1), code)) <= TOL


def test_linear_strided_and_batched_input(pkg, numerics):
    lin, raw, b = _layer(pkg, Q.Q8_0, 96, 256)
    x = torch.randn(2, 3, 512, device=DEV, dtype=torch.bfloat16)[..., :256]   # non-contiguous rows, ld=512
    y = lin(x)
    assert tuple(y.shape) == (2, 3, 96)
    W = pkg.dequant.dequantize_tensor(lin.weight, torch.bfloat16)
    ref = torch.nn.functional.linear(x.float(), W.float(), torch.from_numpy(b).to(DEV).to(torch.bfloat16).float())
    assert rel_fro(y.float().cpu().numpy(), ref.cpu().numpy()) <= max(2e-3, _tol(numerics, torch.bfloat16))   # ref: fp32 math on bf16 W, unrounded output


def test_offloaded_weight_is_moved_packed(pkg):
    """lowvram: module on the CPU, activations on the GPU -> packed bytes cross PCIe, result on the GPU (ops.py:209)."""
    lin, raw, b = _layer(pkg, Q.Q4_K, 64, 512)
    lin.weight = torch.nn.Parameter(lin.weight.to("cpu"), requires_grad=False)
    x = torch.randn(4, 512, device=DEV, dtype=torch.float16)
    y = lin(x)
    want = oracle.linear(raw, int(Q.Q4_K), 64, 512, torch_bits(x), 0, 0, torch_bits(torch.from_numpy(b).to(torch.float16)))
    assert y.is_cuda and rel_fro(y.float().cpu().numpy(), bits_to_f32(want.reshape(-1), 0)) <= TOL


def _lora_case(pkg, M, N, K, dtype, n_loras=1, rank=4):
    lin, raw, b = _layer(pkg, Q.Q4_K, N, K)
    g = torch.Generator(device="cpu").manual_seed(N + K + M)
    loras = [(torch.randn(N, rank, generator=g).to(DEV) * 0.05, torch.randn(rank, K, generator=g).to(DEV) * 0.05, 0.8 - 0.3 * i, 2.0 + i)
             for i in range(n_loras)]
    lin.weight.patches = [([(s, ("lora", (up, down, alpha, None, None, None)), 1.0, None, None)], "w") for up, down, s, alpha in loras]
    x = torch.randn(M, K, generator=g).to(DEV).to(dtype)
    W = pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, dtype))   # GGMLTensor.clone() returns self (ops.py:64-68)
    delta = [s * (alpha / rank) * (up @ down) for up, down, s, alpha in loras]
    # what the reference computes (ops.py:184-190): W rounded to the activation dtype after every patch, then F.linear
    Wref = W.clone()
    for d in delta:
        Wref += d.to(dtype)
    bias = torch.from_numpy(b).to(DEV)
    ref = torch.nn.functional.linear(x.double(), Wref.double(), bias.to(dtype).double())
    # the unrounded ideal
    ideal = torch.nn.functional.linear(x.double(), W.double() + sum(delta).double(), bias.to(dtype).double())
    return lin, x, ref, ideal


def _rel(a, b):
    return float((a.double() - b).norm() / b.norm())


@pytest.mark.parametrize("M,N,K,dtype,n_loras", [(6, 64, 512, torch.bfloat16, 1), (6, 64, 512, torch.float16, 2),
                                                (300, 264, 1024, torch.bfloat16, 1), (300, 264, 1024, torch.float16, 3)])
def test_lora_on_packed_weight_runs_as_side_gemms(pkg, M, N, K, dtype, n_loras, numerics):
    """SURVEY 8f rank 1: LoRA-only patch lists are served by the packed-weight Linear plus rank-r side GEMMs.
    Parity budget: the side-GEMM result must be (a) within 3e-3 (fp16) / 1e-2 (bf16) relative Frobenius of the reference's
    dequant + calculate_weight + F.linear arithmetic and (b) no further from the unrounded ideal than 1.5x the reference is
    (the reference additionally rounds W + delta to the activation dtype)."""
    lin, x, ref, ideal = _lora_case(pkg, M, N, K, dtype, n_loras)
    assert lin._lora_terms(x.device), "LoRA-only patch list must be recognised"
    if numerics == "fast":
        # default route (GGMLOps.Linear.lora_in_kernel = True): base product AND the rank-r update inside the FUSED_TMEM kernel (one
        # extra k-block: U = scale*up rows as the weight tile, T = x*down^T TMA-fed); same budget against the reference arithmetic,
        # and within bf16 / fp16 output rounding of the side-GEMM formulation
        y_in = lin(x)
        lin.lora_in_kernel = False
        try:
            y_side = lin(x)
        finally:
            del lin.lora_in_kernel
        assert "_gg_lora" in lin.__dict__, "the LoRA operands should have been prepared for the in-kernel path"
        assert _rel(y_in, ref) <= (3e-3 if dtype == torch.float16 else 1e-2)
        assert _rel(y_in, y_side.double()) <= (1.5e-3 if dtype == torch.float16 else 8e-3)
    lin.linear_numerics = "exact"
    y = lin(x)
    assert type(y) is torch.Tensor and y.dtype == dtype
    budget = 3e-3 if dtype == torch.float16 else 1e-2
    assert _rel(y, ref) <= budget
    ref_rounded = ref.to(dtype)          # the reference's own output rounding
    assert _rel(y, ideal) <= 1.5 * _rel(ref_rounded, ideal) + 1e-4
    # knob off -> the reference's two-step arithmetic
    lin.lora_side_gemm = False
    try:
        y2 = lin(x)
    finally:
        del lin.lora_side_gemm
    assert _rel(y2, ref) <= (2e-3 if dtype == torch.float16 else 6e-3)
    lin.weight.patches = []
    assert lin._lora_terms(x.device) == []


def test_non_lora_patch_takes_two_step_route(pkg):
    """Anything calculate_weight-specific (diff patches, strength_model, offsets ...) keeps the reference route
    (ops.py:171-190): dequant + comfy.lora.calculate_weight + F.linear."""
    lin, raw, _ = _layer(pkg, Q.Q4_K, 64, 512, bias=False)
    diff = torch.randn(64, 512, device=DEV) * 0.01
    lin.weight.patches = [([(0.5, ("diff", (diff,)), 1.0, None, None)], "w")]
    assert lin._lora_terms(torch.device(DEV)) is None
    x = torch.randn(6, 512, device=DEV, dtype=torch.bfloat16)
    y = lin(x)
    W = pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, torch.bfloat16))
    ref = torch.nn.functional.linear(x.double(), (W + (0.5 * diff).to(torch.bfloat16)).double())
    assert _rel(y, ref) <= 6e-3
    up, down = torch.randn(64, 4, device=DEV), torch.randn(4, 512, device=DEV)
    lin.weight.patches = [([(0.5, ("lora", (up, down, None, None, None, None)), 0.9, None, None)], "w")]   # strength_model != 1
    assert lin._lora_terms(torch.device(DEV)) is None
    lin.weight.patches = [([(0.5, ("lora", (up, down, None, None, torch.ones(64, device=DEV), None)), 1.0, None, None)], "w")]  # DoRA
    assert lin._lora_terms(torch.device(DEV)) is None


@pytest.mark.parametrize("M", [3, 300])
def test_q4k_producer_is_exact_for_huge_scales(pkg, M):
    """The hand-scheduled Q4_K producer folds `fp16(D*q)` into one fma, which needs 2^k*D to be representable; sub-blocks
    with |d*sc| >= 32 must fall back to the plain sequence instead of overflowing to NaN.  d = 4.0 gives D = 4*sc in
    [0, 252]: lanes of both kinds inside the same warp."""
    N, K = 264, 1024
    raw = oracle.random_blocks(int(Q.Q4_K), N * K // 256, seed=11, scale=0.02).reshape(-1, 144).copy()
    raw[:, 0:2] = np.frombuffer(np.float16(4.0).tobytes(), dtype=np.uint8)
    raw = raw.reshape(N, K // 256 * 144)
    w = pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=Q.Q4_K, tensor_shape=torch.Size((N, K)))
    W = pkg.ops._plain(pkg.dequant.dequantize_tensor(w, torch.bfloat16))       # K1: bit-exact vs the reference
    assert torch.isfinite(W).all() and W.abs().max() > 1000
    x = (torch.randn(M, K, device=DEV) * 0.01).to(torch.bfloat16)
    ref = torch.nn.functional.linear(x.double(), W.double())
    algos = [pkg.lib.ALGO_GEMV] if M <= 8 else [pkg.lib.ALGO_FUSED_MMA, pkg.lib.ALGO_DEQUANT_MMA]
    for algo in algos + [pkg.lib.ALGO_FUSED_TMEM]:
        y = pkg.ops.linear_packed(x, w, None, None, algo)
        assert torch.isfinite(y).all()
        # bf16 output rounding of values ~1e2; the TMEM route keeps W in fp16 (8e-3 = 1e-3 in bf16 ulps)
        assert float((y.double() - ref).norm() / ref.norm()) <= (8e-3 if algo == pkg.lib.ALGO_FUSED_TMEM else 3e-3)


def test_embedding_row_gather_equals_reference_semantics(pkg):
    emb = pkg.ops.GGMLOps.Embedding(500, 1024, device="meta")
    raw, w = _weight(pkg, Q.Q5_K, 500, 1024, seed=8)
    emb.load_state_dict({"weight": w}, assign=True)
    idx = torch.tensor([[1, 499, 7, 7]], device=DEV)
    full = pkg.dequant.dequantize_tensor(w, torch.float32)
    out = emb(idx)
    assert out.dtype == torch.float32 and torch.equal(out, torch.nn.functional.embedding(idx, full))
    out16 = emb(idx, out_dtype=torch.bfloat16)
    assert out16.dtype == torch.bfloat16
    assert torch.equal(out16, torch.nn.functional.embedding(idx, pkg.dequant.dequantize_tensor(w, torch.bfloat16)))


def test_error_paths_raise(pkg):
    raw, w = _weight(pkg, Q.Q4_K, 32, 512)
    with pytest.raises(ValueError):
        pkg.ops.linear_packed(torch.randn(2, 256, device=DEV, dtype=torch.bfloat16), w, None)
    with pytest.raises(pkg.lib.GGUFB200Error):
        pkg.ops.linear_packed(torch.randn(64, 512, device=DEV, dtype=torch.bfloat16), w, None, None, pkg.lib.ALGO_GEMV)


@pytest.mark.parametrize("M", [2, 300])
def test_unaligned_packed_weight_view(pkg, M):
    """A packed weight that does not start on a 16-byte boundary (a byte-offset view): every 16-byte fast path (TMA staging,
    Fast16 producers, bulk loads) must step aside for the alignment-agnostic routes and still match."""
    qt, N, K = Q.Q4_K, 136, 1024
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    raw = oracle.random_blocks(int(qt), N * K // bs, seed=11, scale=0.02).reshape(-1)
    buf = torch.zeros(raw.size + 64, dtype=torch.uint8, device=DEV)
    buf[6:6 + raw.size] = torch.from_numpy(raw).to(DEV)
    view = buf[6:6 + raw.size].view(N, K // bs * ts)
    assert view.data_ptr() % 16 != 0
    w = pkg.ops.GGMLTensor(view, tensor_type=qt, tensor_shape=torch.Size((N, K)))
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    want = oracle.linear(raw, int(qt), N, K, torch_bits(x), oracle.DT_BF16, oracle.DT_F16, None)
    for algo in ((pkg.lib.ALGO_GEMV,) if M <= 8 else (pkg.lib.ALGO_FUSED_MMA, pkg.lib.ALGO_DEQUANT_MMA)) + (pkg.lib.ALGO_AUTO, pkg.lib.ALGO_FUSED_TMEM):
        y = pkg.ops.linear_packed(x, w, None, None, algo)     # whatever is asked for, an unaligned weight is served by dequant + GEMM
        assert rel_fro(y.float().cpu().numpy(), bits_to_f32(want.reshape(-1), 1)) <= TOL


def test_conv2d_and_norms_with_quantised_parameters(pkg):
    """Non-Linear consumers of the standalone dequant (ops.py:246-271): Conv2d with a Q8_0 kernel, LayerNorm / GroupNorm with
    BF16-typed affine parameters.  Reference semantics = the stock functional op on the dequantised parameters."""
    ops = pkg.ops.GGMLOps
    g = torch.Generator(device=DEV).manual_seed(0)
    # Conv2d: logical weight [8, 32, 3, 3] = 2304 elements = 72 Q8_0 blocks
    raw = oracle.random_blocks(int(Q.Q8_0), 72, seed=21, scale=0.02)
    w = pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=Q.Q8_0, tensor_shape=torch.Size((8, 32, 3, 3)))
    b = pkg.ops.GGMLTensor(torch.randn(8, device=DEV, generator=g), tensor_type=Q.F32, tensor_shape=torch.Size((8,)))
    conv = ops.Conv2d(32, 8, 3, padding=1, device="meta")
    conv.load_state_dict({"weight": w, "bias": b}, assign=True)
    x = torch.randn(2, 32, 16, 16, device=DEV, generator=g).to(torch.bfloat16)
    y = conv(x)
    W = torch.from_numpy(oracle.dequant(raw, int(Q.Q8_0), oracle.DT_BF16, oracle.DT_F16).view(np.int16)).to(DEV).view(torch.bfloat16).reshape(8, 32, 3, 3)
    ref = torch.nn.functional.conv2d(x, W, b.as_subclass(torch.Tensor).to(torch.bfloat16), padding=1)
    assert type(y) is torch.Tensor and torch.equal(y, ref)

    def bf16_param(n, seed):
        v = (torch.randn(n, generator=torch.Generator().manual_seed(seed)) * 0.5 + 1).to(torch.bfloat16)
        return v, pkg.ops.GGMLTensor(v.view(torch.uint8).to(DEV), tensor_type=Q.BF16, tensor_shape=torch.Size((n,)))
    wv, wq = bf16_param(64, 1)
    bv, bq = bf16_param(64, 2)
    ln = ops.LayerNorm(64, device="meta")
    ln.load_state_dict({"weight": wq, "bias": bq}, assign=True)
    xs = torch.randn(5, 64, device=DEV, generator=g).to(torch.float16)
    torch.testing.assert_close(ln(xs), torch.nn.functional.layer_norm(xs, (64,), wv.to(DEV).half(), bv.to(DEV).half(), ln.eps))
    gn = ops.GroupNorm(8, 64, device="meta")
    gn.load_state_dict({"weight": wq, "bias": bq}, assign=True)
    xg = torch.randn(2, 64, 4, 4, device=DEV, generator=g).to(torch.float16)
    torch.testing.assert_close(gn(xg), torch.nn.functional.group_norm(xg, 8, wv.to(DEV).half(), bv.to(DEV).half(), gn.eps))


# ---------------------------------------------------------------- K3 v2: integer patterns on mma.sync, scales applied to partial sums (csrc/gemv2.cu)
@pytest.mark.parametrize("qt", [Q.Q4_K, Q.Q5_K], ids=lambda q: q.name)
@pytest.mark.parametrize("dt,code", [(torch.bfloat16, 1), (torch.float16, 0)], ids=["bf16", "f16"])
@pytest.mark.parametrize("M,N,K", [(1, 200, 1024), (3, 264, 256), (8, 5000, 4096), (5, 1032, 3072), (2, 16, 15360)])
def test_gemv_fast_kernel_vs_oracle_and_ideal(pkg, qt, dt, code, M, N, K):
    """GGUFB200_ALGO_GEMV_FAST never forms W (DESIGN.md section 3, `fast` contract): within 1e-3 of the reference Linear for
    fp16 activations, 8e-3 for bf16 -- and at least as close to the fp64 product of the exactly dequantised weight as the
    reference's own result.  Shapes: partial last row tile, a single super-block, several K-chunks, persistent CTAs."""
    raw, w = _weight(pkg, qt, N, K, seed=int(qt) + M + N)
    x = torch.randn(M, K, device=DEV, dtype=dt)
    bias = torch.randn(N, device=DEV, dtype=torch.float32) * 0.1
    y = pkg.ops.linear_packed(x, w, bias, None, pkg.lib.ALGO_GEMV_FAST)
    assert torch.equal(y, pkg.ops.linear_packed(x, w, bias, None, pkg.lib.ALGO_GEMV_FAST)), "fixed summation order: reproducible"
    # W_STABLE only lets the weight ring fill before the preceding kernel has drained: same bits, also back to back with a
    # kernel that has just written the activations
    for _ in range(3):
        x2 = x + 0
        assert torch.equal(y, pkg.ops.linear_packed(x2, w, bias, None, pkg.lib.ALGO_GEMV_FAST | pkg.lib.FLAG_W_STABLE))
    want = oracle.linear(raw, int(qt), N, K, torch_bits(x), code, oracle.DT_F16, torch_bits(bias.to(dt)))
    ref = torch.from_numpy(bits_to_f32(want.reshape(-1), code).reshape(M, N)).to(DEV)
    assert rel_fro(y.float().cpu().numpy(), ref.cpu().numpy()) <= (1e-3 if dt == torch.float16 else 8e-3)
    w32 = pkg.dequant.dequantize_tensor(w, torch.float32, torch.float32)
    ideal = x.double() @ w32.double().t() + bias.to(dt).double()
    assert (y.double() - ideal).norm().item() <= 1.02 * (ref.double() - ideal).norm().item()
    # AUTO takes it exactly when the caller did not ask for a reference-exact weight
    ya = pkg.ops.linear_packed(x, w, bias, None, pkg.lib.ALGO_AUTO)
    assert torch.equal(ya, y)
    ye = pkg.ops.linear_packed(x, w, bias, None, pkg.lib.ALGO_AUTO | pkg.lib.FLAG_EXACT_W)
    assert rel_fro(ye.float().cpu().numpy(), ref.cpu().numpy()) <= TOL


def test_gemv_fast_kernel_rejects_what_it_cannot_do(pkg):
    raw, w = _weight(pkg, Q.Q8_0, 64, 512)
    x = torch.randn(2, 512, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(pkg.lib.GGUFB200Error):
        pkg.ops.linear_packed(x, w, None, None, pkg.lib.ALGO_GEMV_FAST)               # only Q4_K / Q5_K
    raw, w = _weight(pkg, Q.Q4_K, 64, 512)
    with pytest.raises(pkg.lib.GGUFB200Error):
        pkg.ops.linear_packed(torch.randn(9, 512, device=DEV, dtype=torch.bfloat16), w, None, None, pkg.lib.ALGO_GEMV_FAST)   # M > 8
    with pytest.raises(pkg.lib.GGUFB200Error):
        pkg.ops.linear_packed(x, w, None, None, pkg.lib.ALGO_GEMV_FAST | pkg.lib.FLAG_EXACT_W)                                 # contract conflict
