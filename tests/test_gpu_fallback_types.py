"""GPU tests of the numpy-fallback types (IQ2_XXS ... NVFP4) on an H100: K1 (ggufb200_dequant_fallback) bit for bit against
gguf-py and the golden files, the reference's `dequantize_tensor` semantics for these types, and the layers built on them
(Linear, Embedding, Conv2d, a qwen3-arch text-encoder GGUF)."""
import os

import gguf
import numpy as np
import pytest
import torch

from fallback_cases import FALLBACK, TORCH_DT, gguf_values, random_blocks, reference_tensor
from util import Q, canon_nan, rel_fro, torch_bits

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _same_bits(got, want, code):
    return np.array_equal(canon_nan(torch_bits(got), code), canon_nan(torch_bits(want), code))


def _ragged_blocks(qt):
    """Three whole 4096-element tiles and a partial one."""
    bs = gguf.GGML_QUANT_SIZES[qt][0]
    return 3 * (4096 // bs) + max(1, 4096 // bs // 3)


@pytest.mark.parametrize("code", [0, 1, 2], ids=["f16", "bf16", "f32"])
@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_k1_bit_exact_vs_gguf_py(pkg, qt, code):
    blocks = random_blocks(qt, _ragged_blocks(qt), seed=5, specials=True)
    with np.errstate(all="ignore"):
        want = reference_tensor(blocks, qt, code)
    bs = gguf.GGML_QUANT_SIZES[qt][0]
    got = pkg.dequant.dequantize_fallback(torch.from_numpy(blocks).to(DEV), qt, (blocks.shape[0] * bs,), TORCH_DT[code])
    assert got.dtype == TORCH_DT[code] and got.device == DEV
    assert _same_bits(got, want, code)


@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_k1_matches_golden(pkg, qt, golden_dir):
    g = np.load(os.path.join(golden_dir, f"fallback_{qt.name}.npz"))
    got = pkg.dequant.dequantize_fallback(torch.from_numpy(g["blocks"]).to(DEV), qt, g["f32"].shape)
    assert got.dtype == torch.float32
    assert np.array_equal(canon_nan(torch_bits(got), 2), canon_nan(g["f32"].view(np.uint32).copy(), 2))


@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_k1_unaligned_packed_view(pkg, qt):
    """A byte-offset view of the packed bytes takes the kernel's byte-copy staging path: same bits."""
    blocks = random_blocks(qt, _ragged_blocks(qt), seed=6, scale=0.01)
    flat = torch.from_numpy(blocks.reshape(-1))
    buf = torch.zeros(flat.numel() + 16, dtype=torch.uint8, device=DEV)
    for shift in (1, 3, 8):
        view = buf[shift:shift + flat.numel()]
        view.copy_(flat.to(DEV))
        assert view.data_ptr() % 16 != 0
        got = pkg.dequant.dequantize_fallback(view, qt, (-1,), torch.bfloat16)
        assert _same_bits(got, reference_tensor(blocks, qt, 1), 1), shift


def test_k1_src_stable_after_a_torch_kernel_that_rewrites_the_packed_bytes(pkg):
    """dequantize_fallback passes SRC_STABLE by default: a torch kernel rewrites the packed tensor in place and the dequant
    follows at once on the same stream; the result must always be the dequant of the new bytes."""
    qt = Q.IQ2_XS
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    seed = torch.from_numpy(random_blocks(qt, 1 << 12, seed=21, scale=0.01)).to(DEV)
    n_blocks = 10240 * 4096 // bs
    base = seed.repeat(n_blocks // (1 << 12), 1).contiguous()
    mask = torch.zeros(ts, dtype=torch.uint8, device=DEV)
    work = base.clone()
    torch.cuda.synchronize()
    for i in range(12):
        mask.zero_()
        mask[2 + (i * 5) % 64] = 1 + i                                   # quant bytes only: the f16 scale stays finite
        torch.bitwise_xor(base, mask, out=work)
        got = pkg.dequant.dequantize_fallback(work, qt, (-1,), torch.float16, src_stable=True)
        torch.cuda.synchronize()
        want = pkg.dequant.dequantize_fallback(work, qt, (-1,), torch.float16, src_stable=False)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"iteration {i}: stale packed bytes were read"
    last = work[:64].cpu().numpy()
    assert _same_bits(got[:64 * bs], reference_tensor(last, qt, 0), 0)


def test_dequantize_tensor_semantics(pkg):
    qt = Q.IQ3_S
    N, K = 64, 512
    raw = random_blocks(qt, N * K // 256, seed=8, scale=0.01)
    t = pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=qt, tensor_shape=torch.Size((N, K)))
    y = pkg.dequant.dequantize_tensor(t)                                  # the reference's .to(dtype=None): float32
    assert y.dtype == torch.float32 and tuple(y.shape) == (N, K)
    assert _same_bits(y, reference_tensor(raw, qt, 2), 2)
    base = pkg.dequant.dequantize_tensor(t, torch.float16)
    for dq in (None, "target", torch.float16, torch.float32, torch.bfloat16):   # dequant_dtype is ignored on this branch
        again = pkg.dequant.dequantize_tensor(t, torch.float16, dq)
        assert torch.equal(again.view(torch.int16), base.view(torch.int16)), dq
    cpu = pkg.ops.GGMLTensor(torch.from_numpy(raw), tensor_type=qt, tensor_shape=torch.Size((N, K)))
    back = pkg.dequant.dequantize_tensor(cpu, torch.bfloat16)             # packed bytes on the host: result on the host
    assert back.device.type == "cpu" and _same_bits(back, reference_tensor(raw, qt, 1), 1)
    # a tensor the converter reshaped to [n / 256, 256] (comfy.gguf.orig_shape): the logical shape, not the byte shape
    conv = random_blocks(qt, 320 * 320 * 9 // 256, seed=9, scale=0.01)
    c = pkg.ops.GGMLTensor(torch.from_numpy(conv).to(DEV), tensor_type=qt, tensor_shape=torch.Size((320, 320, 3, 3)))
    w = pkg.dequant.dequantize_tensor(c, torch.float16)
    assert tuple(w.shape) == (320, 320, 3, 3)
    assert _same_bits(w, reference_tensor(conv, qt, 0), 0)


def _linear(pkg, qt, N, K, seed, bias=True):
    raw = random_blocks(qt, N * K // gguf.GGML_QUANT_SIZES[qt][0], seed=seed, scale=0.002)
    w = pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=qt, tensor_shape=torch.Size((N, K)))
    lin = pkg.ops.GGMLOps.Linear(K, N)
    sd = {"weight": w}
    if bias:
        sd["bias"] = pkg.ops.GGMLTensor(torch.randn(N, device=DEV) * 0.1, tensor_type=Q.F32, tensor_shape=torch.Size((N,)))
    lin.load_state_dict(sd)
    w32 = torch.from_numpy(gguf_values(raw, qt).reshape(N, K)).to(DEV)
    return lin, w32, (sd["bias"].as_subclass(torch.Tensor) if bias else None)


def _reference(x, w32, bias):
    """What the reference computes: F.linear with the weight rounded once from fp32 to the activation dtype (summed in fp64
    here), its output in the activation dtype."""
    dt = x.dtype
    y = x.double() @ w32.to(dt).double().t()
    if bias is not None:
        y = y + bias.to(dt).double()
    return y.to(dt)


def _rel(y, ref):
    return rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy())


@pytest.mark.parametrize("M", [1, 8, 77, 512, 4096])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_linear_matches_reference(pkg, qt, dtype, M):
    N, K = 384, 1024
    g = torch.Generator().manual_seed(M)
    for bias in (True, False):
        lin, w32, b = _linear(pkg, qt, N, K, seed=M + int(bias), bias=bias)
        x = torch.randn(M, K, generator=g).to(DEV).to(dtype)
        y = lin(x)
        assert y.dtype == dtype and tuple(y.shape) == (M, N)
        assert _rel(y, _reference(x, w32, b)) <= 1e-3, (M, bias)


def test_linear_runs_k1_then_the_dense_gemm(pkg, monkeypatch):
    """Route evidence: one ggufb200_dequant_fallback into the activation dtype, then ggufb200_gemm; no packed-weight Linear."""
    calls = []
    real = pkg.lib.lib()

    class Spy:
        def __getattr__(self, name):
            fn = getattr(real, name)
            if name.startswith("ggufb200_linear") or name in ("ggufb200_dequant_fallback", "ggufb200_gemm", "ggufb200_dequant"):
                def wrapped(*a):
                    calls.append((name, a[4] if name == "ggufb200_dequant_fallback" else None))
                    return fn(*a)
                return wrapped
            return fn
    lin, _w, _b = _linear(pkg, Q.IQ2_XXS, 256, 512, seed=1)
    monkeypatch.setattr(pkg.lib, "lib", lambda: Spy())
    lin(torch.randn(5, 512, device=DEV, dtype=torch.bfloat16))
    assert calls == [("ggufb200_dequant_fallback", pkg.lib.BF16), ("ggufb200_gemm", None)]


@pytest.mark.parametrize("qt", [Q.IQ1_M, Q.IQ2_S, Q.MXFP4], ids=lambda q: q.name)
def test_linear_with_lora_patch(pkg, qt):
    """A LoRA-only patch list: K1 + GEMM plus the side GEMMs, within the LoRA budget of the reference's two-step result."""
    N, K, r = 512, 1024, 16
    g = torch.Generator().manual_seed(3)
    lin, w32, b = _linear(pkg, qt, N, K, seed=3)
    up = (torch.randn(N, r, generator=g) * 0.02).to(DEV)
    down = (torch.randn(r, K, generator=g) * 0.02).to(DEV)
    lin.weight.patches = [([(0.8, ("lora", (up, down, 8.0, None, None, None)), 1.0, None, None)], "w")]
    try:
        for M, dtype in ((3, torch.float16), (300, torch.bfloat16)):
            x = torch.randn(M, K, generator=g).to(DEV).to(dtype)
            y = lin(x)
            lin.lora_side_gemm = False                                    # the reference's two-step arithmetic
            ref = lin(x)
            lin.lora_side_gemm = True
            ideal = x.double() @ (w32.double() + 0.8 * 8.0 / r * (up.double() @ down.double())).t() + b.to(dtype).double()
            assert _rel(y, ref) <= (3e-3 if dtype == torch.float16 else 1e-2), (M, dtype)
            assert _rel(y, ideal) <= 1.5 * _rel(ref, ideal) + 1e-4, (M, dtype)
    finally:
        lin.weight.patches = []


def test_linear_two_step_route_for_unaligned_shapes(pkg):
    """N % 8 != 0: the two-step route (dequantize_tensor + F.linear), which now works for these types."""
    N, K = 100, 512
    lin, w32, b = _linear(pkg, Q.IQ3_XXS, N, K, seed=4)
    x = torch.randn(33, K, device=DEV, dtype=torch.float16)
    y = lin(x)
    assert tuple(y.shape) == (33, N)
    assert _rel(y, _reference(x, w32, b)) <= 1e-3


def test_embedding_with_an_iq_table(pkg):
    qt = Q.IQ2_XXS
    V, D = 1000, 512
    raw = random_blocks(qt, V * D // 256, seed=12, scale=0.01)
    emb = pkg.ops.GGMLOps.Embedding(V, D, device="meta")
    w = pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=qt, tensor_shape=torch.Size((V, D)))
    emb.load_state_dict({"weight": w}, assign=True)
    ids = torch.randint(0, V, (3, 17), device=DEV)
    table = reference_tensor(raw, qt, 2).reshape(V, D).to(DEV)
    for out_dtype in (None, torch.float16):
        got = emb(ids, out_dtype=out_dtype)
        want = torch.nn.functional.embedding(ids, table).to(dtype=out_dtype)
        assert got.dtype == want.dtype and torch.equal(got, want), out_dtype


def test_conv2d_reshaped_sdxl_weight(pkg):
    """An SDXL-style 3x3 conv the converter reshaped to [n / 256, 256]: Conv2d through dequantize_tensor, logical shape."""
    qt = Q.IQ2_S
    shape = (320, 320, 3, 3)
    raw = random_blocks(qt, int(np.prod(shape)) // 256, seed=13, scale=0.002)
    conv = pkg.ops.GGMLOps.Conv2d(320, 320, 3, padding=1, device="meta")
    w = pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=qt, tensor_shape=torch.Size(shape))
    bias = torch.randn(320, device=DEV) * 0.1
    conv.load_state_dict({"weight": w, "bias": bias}, assign=True)
    x = torch.randn(2, 320, 16, 16, device=DEV, dtype=torch.float16)
    w16 = reference_tensor(raw, qt, 0).reshape(shape).to(DEV)
    want = torch.nn.functional.conv2d(x.double(), w16.double(), bias.half().double(), padding=1)
    y = conv(x)
    assert y.dtype == torch.float16 and _rel(y, want) <= 1e-3


def test_qwen3_gguf_end_to_end(pkg, tmp_path):
    """A small qwen3-arch text-encoder GGUF with i-quant, ternary and FP4 tensors, written by gguf.GGUFWriter, loaded by
    gguf_clip_loader; every Linear runs and matches the reference arithmetic."""
    path = str(tmp_path / "qwen3_iq.gguf")
    H, F = 512, 1536
    tensors = {
        "blk.0.attn_q.weight": (Q.IQ2_XXS, (H, H)), "blk.0.attn_k.weight": (Q.IQ3_XXS, (H, H)),
        "blk.0.attn_v.weight": (Q.IQ1_S, (H, H)), "blk.0.attn_output.weight": (Q.IQ3_S, (H, H)),
        "blk.0.ffn_gate.weight": (Q.IQ2_XS, (F, H)), "blk.0.ffn_up.weight": (Q.IQ1_M, (F, H)),
        "blk.0.ffn_down.weight": (Q.IQ2_S, (H, F)), "blk.1.ffn_gate.weight": (Q.TQ1_0, (F, H)),
        "blk.1.ffn_up.weight": (Q.TQ2_0, (F, H)), "blk.1.ffn_down.weight": (Q.MXFP4, (H, F)),
        "blk.1.attn_q.weight": (Q.NVFP4, (H, H)), "token_embd.weight": (Q.IQ2_XXS, (1024, H)),
    }
    w = gguf.GGUFWriter(path, "qwen3")
    raws = {}
    for i, (name, (qt, shape)) in enumerate(tensors.items()):
        bs, ts = gguf.GGML_QUANT_SIZES[qt]
        raw = random_blocks(qt, shape[0] * shape[1] // bs, seed=70 + i, scale=0.002).reshape(shape[0], shape[1] // bs * ts)
        w.add_tensor(name, raw, raw_dtype=qt)
        raws[name] = (qt, shape, raw)
    w.add_tensor("output_norm.weight", np.ones(H, dtype=np.float32))
    w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()

    sd = pkg.loader.gguf_clip_loader(path)
    g = torch.Generator().manual_seed(0)
    for name, (qt, shape, raw) in raws.items():
        key = next(iter(pkg.loader.sd_map_replace({name: None}, pkg.loader.LLAMA_SD_MAP)))     # e.g. model.layers.0.self_attn.q_proj.weight
        w = sd[key]
        assert w.tensor_type == qt and tuple(w.tensor_shape) == shape
        assert np.array_equal(w.as_subclass(torch.Tensor).numpy(), raw)
        if name == "token_embd.weight":
            continue
        lin = pkg.ops.GGMLOps.Linear(shape[1], shape[0])
        lin.load_state_dict({"weight": w})                             # packed bytes on the host: the Linear moves them over
        x = torch.randn(77, shape[1], generator=g).to(DEV).to(torch.bfloat16)
        w32 = torch.from_numpy(gguf_values(raw, qt).reshape(shape)).to(DEV)
        assert _rel(lin(x), _reference(x, w32, None)) <= 1e-3, name
    emb = pkg.ops.GGMLOps.Embedding(1024, H, device="meta")
    emb.load_state_dict({"weight": sd["model.embed_tokens.weight"]}, assign=True)
    ids = torch.arange(0, 1024, 13, device=DEV)
    qt, shape, raw = raws["token_embd.weight"]
    want = torch.nn.functional.embedding(ids, reference_tensor(raw, qt, 2).reshape(shape).to(DEV))
    assert torch.equal(emb(ids), want)
