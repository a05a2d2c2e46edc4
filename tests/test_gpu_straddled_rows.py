"""GPU tests of straddled K-quant weights on the packed-weight Linear.

For SD1.5 / SDXL the GGUF converter reshapes every tensor whose last dimension is not a multiple of 256 to [n / 256, 256]
before quantising and records the logical shape in `comfy.gguf.orig_shape.<key>`.  A Linear [N, K] with K % 256 != 0 (K = 320
or 640 in those UNets) is then a flat stream of N * K / 256 super-blocks, and row n starts at element n * K, often inside a
block.  FUSED_TMEM reads k-block kb of row n as one quarter of block (n K + 64 kb) / 256: Q4_K / Q5_K from the canonical
bytes, Q2_K / Q3_K / Q6_K / IQ4_XS from the block-major copy of ggufb200_repack.

Reference: the oracle's dequant of the flat stream reshaped to [N, K] (the reference's `dequantize_tensor`), cast to the
activation dtype, x @ W^T + bias in float64, rounded to the activation dtype.  Bounds: 1e-3 relative Frobenius (8e-3 for the
`fast` producers with bf16 activations); the reference-exact FUSED_TMEM producers 3e-4, as for whole-block rows
(tests/test_gpu_gemm.py)."""
import functools
import os

import gguf
import numpy as np
import pytest
import torch

import oracle
from util import Q, bits_to_f32, rel_fro

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N = 264                                    # 264 * 320 and 264 * 640 are whole numbers of blocks; odd rows start mid-block
K_QUANTS = [Q.Q2_K, Q.Q3_K, Q.Q4_K, Q.Q5_K, Q.Q6_K, Q.IQ4_XS]
PITCH = {Q.Q2_K: 112, Q.Q3_K: 112, Q.Q4_K: 144, Q.Q5_K: 176, Q.Q6_K: 240, Q.IQ4_XS: 144}


@pytest.fixture(params=["exact", "fast"])
def numerics(request, pkg):
    cls = pkg.ops.GGMLOps.Linear
    before = cls.linear_numerics
    cls.linear_numerics = request.param
    yield request.param
    cls.linear_numerics = before


@functools.lru_cache(maxsize=None)
def _stream(qt, n, K, seed=0):
    """Packed stream [n K / 256, ts] and its dequantised fp16 weight [n, K] (oracle, flat block order)."""
    raw = oracle.random_blocks(int(qt), n * K // 256, seed=seed + int(qt) + K, scale=0.02)
    w16 = bits_to_f32(oracle.dequant(raw, int(qt), oracle.DT_F16, oracle.DT_F16), 0).reshape(n, K)
    return raw, torch.from_numpy(w16)


def _layer(pkg, qt, n, K, seed=0):
    raw, w16 = _stream(qt, n, K, seed)
    lin = pkg.ops.GGMLOps.Linear(K, n)
    w = pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=qt, tensor_shape=torch.Size((n, K)))
    b = (torch.randn(n, generator=torch.Generator().manual_seed(seed + 7)) * 0.02).to(DEV)
    lin.load_state_dict({"weight": w, "bias": pkg.ops.GGMLTensor(b, tensor_type=Q.F32, tensor_shape=torch.Size((n,)))})
    return lin, w16.to(DEV), b


def _reference(x, w16, bias):
    dt = x.dtype
    y = x.double() @ w16.to(dt).double().t()
    if bias is not None:
        y = y + bias.to(dt).double()
    return y.to(dt)


def _rel(y, ref):
    return rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy())


@pytest.mark.parametrize("M", [3, 300, 4096])
@pytest.mark.parametrize("K", [320, 640])
@pytest.mark.parametrize("qt", K_QUANTS, ids=lambda q: q.name)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_straddled_linear_matches_the_oracle(pkg, qt, K, M, dtype, numerics):
    A = pkg.lib
    lin, w16, b = _layer(pkg, qt, N, K)
    x = (torch.randn(M, K, generator=torch.Generator().manual_seed(M + K)) * 0.5).to(DEV).to(dtype)
    ref = _reference(x, w16, b)
    tol = 8e-3 if (numerics == "fast" and dtype == torch.bfloat16) else 1e-3
    y = lin(x)
    assert y.dtype == dtype and tuple(y.shape) == (M, N)
    assert _rel(y, ref) <= tol, "layer"
    spans = pkg.ops.needs_span_layout(qt, K)
    exact = A.FLAG_EXACT_W if numerics == "exact" else 0
    y = pkg.ops.linear_packed(x, lin.weight, b, None, A.ALGO_FUSED_TMEM | exact, use_spans=spans)
    assert _rel(y, ref) <= (3e-4 if numerics == "exact" else tol), "FUSED_TMEM"
    y = pkg.ops.linear_packed(x, lin.weight, b, None, A.ALGO_DEQUANT_MMA | exact)
    assert _rel(y, ref) <= 1e-3, "DEQUANT_MMA"


@pytest.mark.parametrize("qt", K_QUANTS, ids=lambda q: q.name)
def test_fused_tmem_needs_a_readable_layout(pkg, qt):
    """Without the block-major copy, FUSED_TMEM reads only Q4_K / Q5_K (16-byte blocks); the others are refused, not
    misread, and the copy has one padded block per block of the stream."""
    lin, _w16, _b = _layer(pkg, qt, N, 640)
    x = torch.randn(64, 640, device=DEV, dtype=torch.float16)
    if pkg.ops.needs_span_layout(qt, 640):
        with pytest.raises(pkg.lib.GGUFB200Error):
            pkg.ops.linear_packed(x, lin.weight, None, None, pkg.lib.ALGO_FUSED_TMEM)
        spans = pkg.ops.span_layout(lin.weight, pkg.ops._plain(lin.weight))
        assert spans.numel() == N * 640 // 256 * PITCH[qt]
    else:
        pkg.ops.linear_packed(x, lin.weight, None, None, pkg.lib.ALGO_FUSED_TMEM)


@pytest.mark.parametrize("name", ["Q4_K", "Q6_K"])
@pytest.mark.parametrize("act,code,dt", [("bf16", 1, torch.bfloat16), ("f16", 0, torch.float16)])
def test_straddled_layer_matches_the_reference_golden(pkg, golden_dir, name, act, code, dt, numerics):
    """The drop-in GGMLOps.Linear vs the y the reference's GGMLOps.Linear produced on the same straddled GGMLTensor."""
    g = np.load(os.path.join(golden_dir, f"linear_straddled_{name}_{act}.npz"))
    qt = Q(int(g["qtype"]))
    n, K, M = int(g["N"]), int(g["K"]), int(g["M"])
    ts = gguf.GGML_QUANT_SIZES[qt][1]
    lin = pkg.ops.GGMLOps.Linear(K, n)
    w = pkg.ops.GGMLTensor(torch.from_numpy(g["packed"].reshape(n * K // 256, ts)).to(DEV), tensor_type=qt, tensor_shape=torch.Size((n, K)))
    b = pkg.ops.GGMLTensor(torch.from_numpy(g["bias"]).to(DEV), tensor_type=Q.F32, tensor_shape=torch.Size((n,)))
    lin.load_state_dict({"weight": w, "bias": b})
    x = torch.from_numpy(g["x"].view(np.int16)).to(DEV).view(dt).reshape(M, K)
    want = bits_to_f32(g["y"].reshape(-1), code)
    tol = 8e-3 if (numerics == "fast" and dt == torch.bfloat16) else 1e-3
    for rows in (M, 5, 1):                       # AUTO: dequant + GEMM at every M
        y = lin(x[:rows])
        assert rel_fro(y.float().cpu().numpy().reshape(-1), want[: rows * n]) <= tol, rows


@pytest.fixture
def calls(pkg, monkeypatch):
    """Records the library calls the package makes (name, args)."""
    L = pkg.lib.lib()
    seen = []
    for name in ("ggufb200_linear", "ggufb200_linear_spans", "ggufb200_dequant", "ggufb200_repack", "ggufb200_linear_lora",
                 "ggufb200_linear_lora_ex"):
        real = getattr(L, name)

        def wrapped(*args, _real=real, _name=name):
            seen.append((_name, args))
            return _real(*args)
        monkeypatch.setattr(L, name, wrapped)
    return seen


def test_route_evidence(pkg, calls):
    """AUTO serves a straddled weight by dequant + GEMM inside one ggufb200_linear call (its workspace is the dense weight), and
    the layer builds no block-major copy for it; an explicit FUSED_TMEM call with the copy reads the block-major layout."""
    A = pkg.lib
    K = 640
    for qt in (Q.Q6_K, Q.Q4_K):
        lin, _w, _b = _layer(pkg, qt, N, K)
        for M in (300, 4):
            calls.clear()
            lin(torch.randn(M, K, device=DEV, dtype=torch.float16))
            assert [c[0] for c in calls] == ["ggufb200_linear"], (qt, M, calls)
            args = calls[0][1]
            assert args[14] == N * K * 2 == pkg.lib.lib().ggufb200_linear_workspace_ex(int(qt), M, N, K, 0, 0, args[15]), (qt, M)
        assert "_gg_spans" not in lin.weight.__dict__
    calls.clear()
    lin6, _w, _b = _layer(pkg, Q.Q6_K, N, K)
    pkg.ops.linear_packed(torch.randn(300, K, device=DEV, dtype=torch.float16), lin6.weight, None, None, A.ALGO_FUSED_TMEM, use_spans=True)
    assert [c[0] for c in calls] == ["ggufb200_repack", "ggufb200_linear_spans"]
    spans = lin6.weight.__dict__["_gg_spans"][1]
    assert spans.numel() == N * K // 256 * 240 and calls[1][1][2] == spans.data_ptr() and calls[1][1][15] == 0


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


def _lora_reference(pkg, lin, x, patches):
    dtype = x.dtype
    W = pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, dtype))
    Wref, Wideal = W.clone(), W.double()
    for s, up, down, alpha, offset in patches:
        d = (s * alpha / down.shape[0]) * (up.float() @ down.float())
        rows = slice(None) if offset is None else slice(offset[1], offset[1] + offset[2])
        Wref[rows] += d.to(dtype)
        Wideal[rows] += d.double()
    bias = pkg.ops._plain(lin.bias).to(dtype).double()
    return (torch.nn.functional.linear(x.double(), Wref.double(), bias), torch.nn.functional.linear(x.double(), Wideal, bias))


@pytest.mark.parametrize("M", [3, 300])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", ["rank16", "stack128", "band"])
def test_lora_runs_in_the_kernel_on_a_straddled_weight(pkg, calls, case, dtype, M):
    """SDXL attention projection [640, 640] in Q4_K with LoRA: Σr = 16 (one k-block), Σr = 128 (two), and three
    row bands (to_q / to_k / to_v style offsets on a fused weight).  Budget of tests/test_gpu_lora_slices.py."""
    K = 640
    n = 640 if case != "band" else 3 * 640 // 2           # 960 rows: three bands of 320
    lin, _w, _b = _layer(pkg, Q.Q4_K, n, K, seed=3)
    g = torch.Generator().manual_seed(11)

    def factors(rows, r):
        return (torch.randn(rows, r, generator=g) * 0.05).to(DEV), (torch.randn(r, K, generator=g) * 0.05).to(DEV)
    if case == "rank16":
        patches = [(0.8, *factors(n, 16), 8.0, None)]
    elif case == "stack128":
        patches = [(0.8, *factors(n, 64), 16.0, None), (0.5, *factors(n, 64), 64.0, None)]
    else:
        patches = [(0.9 - 0.1 * i, *factors(320, 24), 12.0, (0, 320 * i, 320)) for i in range(3)]
    entries = []
    for i, (s, up, down, alpha, offset) in enumerate(patches):
        value = (up, down, alpha, None, None, None)
        entries.append((s, LoRAAdapter(value) if i % 2 else ("lora", value), 1.0, offset, None))
    lin.weight.patches = [(entries, "diffusion_model.w")]
    x = (torch.randn(M, K, generator=g) * 0.5).to(DEV).to(dtype)
    y = lin(x)
    want = "ggufb200_linear_lora" if case == "rank16" else "ggufb200_linear_lora_ex"
    assert [c[0] for c in calls] == [want], [c[0] for c in calls]
    ref, ideal = _lora_reference(pkg, lin, x, patches)
    err = float((y.double() - ref).norm() / ref.norm())
    assert err <= (3e-3 if dtype == torch.float16 else 1e-2), err
    e_ours = float((y.double() - ideal).norm() / ideal.norm())
    e_ref = float((ref.to(dtype).double() - ideal).norm() / ideal.norm())
    assert e_ours <= 1.5 * e_ref + 1e-4, (e_ours, e_ref)
    lin.weight.patches = []


def _write_sdxl_gguf(path):
    """Tensors the way the converter writes an SDXL UNet: 640-wide Linears and a 3x3 conv reshaped to [n / 256, 256] before
    quantising (random payloads stand in for the quantiser), logical shapes in comfy.gguf.orig_shape.*"""
    w = gguf.GGUFWriter(path, "sdxl")
    tensors = {
        "model.diffusion_model.attn.to_q.weight": (Q.Q4_K, (640, 640)),
        "model.diffusion_model.attn.to_k.weight": (Q.Q6_K, (640, 640)),
        "model.diffusion_model.ff.net.0.proj.weight": (Q.Q4_K, (5120, 640)),
        "model.diffusion_model.conv.weight": (Q.Q4_K, (640, 640, 3, 3)),
    }
    raws = {}
    for i, (name, (qt, shape)) in enumerate(tensors.items()):
        n = int(np.prod(shape))
        assert shape[-1] % 256 != 0 and n % 256 == 0
        raw = oracle.random_blocks(int(qt), n // 256, seed=50 + i, scale=0.02)          # [n / 256, ts]: the reshaped tensor
        w.add_tensor(name, raw, raw_dtype=qt)
        w.add_array(f"comfy.gguf.orig_shape.{name}", list(shape))
        raws[name[len("model.diffusion_model."):-len(".weight")]] = (qt, shape, raw)
    bias = np.random.default_rng(1).normal(0, 0.02, size=640).astype(np.float32)
    w.add_tensor("model.diffusion_model.conv.bias", bias)
    w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()
    return raws, bias


def test_sdxl_gguf_loads_and_runs(pkg, tmp_path):
    path = str(tmp_path / "sdxl_straddled.gguf")
    raws, conv_bias = _write_sdxl_gguf(path)
    sd, arch = pkg.loader.gguf_sd_loader(path, return_arch=True)
    assert arch == "sdxl"
    g = torch.Generator().manual_seed(0)
    for key in ("attn.to_q", "attn.to_k", "ff.net.0.proj"):
        qt, shape, raw = raws[key]
        w = sd[key + ".weight"]
        assert w.tensor_type == qt and tuple(w.tensor_shape) == shape
        lin = pkg.ops.GGMLOps.Linear(shape[1], shape[0])
        lin.load_state_dict({"weight": w.to(DEV)})
        w16 = torch.from_numpy(bits_to_f32(oracle.dequant(raw, int(qt), oracle.DT_F16, oracle.DT_F16), 0).reshape(shape)).to(DEV)
        for M, dtype in ((4096, torch.float16), (300, torch.bfloat16), (2, torch.float16)):
            x = (torch.randn(M, shape[1], generator=g) * 0.5).to(DEV).to(dtype)
            assert _rel(lin(x), _reference(x, w16, None)) <= 1e-3, (key, M, dtype)
    qt, shape, raw = raws["conv"]
    conv = pkg.ops.GGMLOps.Conv2d(640, 640, 3, padding=1, device="meta")
    conv.load_state_dict({"weight": sd["conv.weight"].to(DEV), "bias": sd["conv.bias"].to(DEV)}, assign=True)
    x = (torch.randn(2, 640, 16, 16, generator=g) * 0.5).to(DEV).to(torch.float16)
    w16 = torch.from_numpy(bits_to_f32(oracle.dequant(raw, int(qt), oracle.DT_F16, oracle.DT_F16), 0).reshape(shape)).to(DEV)
    want = torch.nn.functional.conv2d(x.double(), w16.double(), torch.from_numpy(conv_bias).to(DEV).half().double(), padding=1)
    y = conv(x)
    assert y.dtype == torch.float16
    assert _rel(y, want) <= 1e-3
