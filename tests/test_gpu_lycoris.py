"""GPU tests of LoKr and LoHa (LyCORIS) patches on a packed weight.

LoKr runs as ggufb200_dequant_kron (the patched weight in one dequant launch) + ggufb200_gemm; its weight must be bit-identical
to the reference's, the restated `calculate_weight` below:  W = dequantize_tensor(...).to(dtype), then per patch in list order
`W[band] += ((strength * alpha) * torch.kron(A, B)).to(dtype)` with fp32 A / B (a decomposed factor = fp32 torch.mm of its
halves).  The Linear must then meet the exact-route budget of tests/test_gpu_linear.py (1e-3 relative Frobenius) against
F.linear(x, W').  LoHa runs as a LoRA of rank r1 r2 on the LoRA machinery and meets the LoRA budget of
tests/test_gpu_lora_slices.py."""
import pytest
import torch

import oracle
from util import Q

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class LoKrAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoKrAdapter):
    pass


def _raw(qt, N, K, seed):
    bs, ts = oracle.type_info(int(qt))
    return torch.from_numpy(oracle.random_blocks(int(qt), N * K // bs, seed=seed, scale=0.02).reshape(-1)).to(DEV)


def _layer(pkg, qt, N, K, seed=0):
    lin = pkg.ops.GGMLOps.Linear(K, N)
    w = pkg.ops.GGMLTensor(_raw(qt, N, K, seed), tensor_type=qt, tensor_shape=torch.Size((N, K)))
    b = (torch.randn(N, generator=torch.Generator().manual_seed(seed + 1)) * 0.02).to(DEV)
    lin.load_state_dict({"weight": w, "bias": pkg.ops.GGMLTensor(b, tensor_type=Q.F32, tensor_shape=torch.Size((N,)))})
    return lin


def _factors(shape, g, rank=None):
    """A full factor, or (rank given) the two halves of a decomposed one."""
    if rank is None:
        return (torch.randn(*shape, generator=g) * 0.3).to(DEV)
    return (torch.randn(shape[0], rank, generator=g) * 0.3).to(DEV), (torch.randn(rank, shape[1], generator=g) * 0.3).to(DEV)


def _lokr(a, b, g, alpha=None, rank1=None, rank2=None):
    """A LoKr payload (w1, w2, alpha, w1_a, w1_b, w2_a, w2_b, t2, dora_scale) with A of shape a and B of shape b."""
    w1, w2 = _factors(a, g, rank1), _factors(b, g, rank2)
    w1, (w1_a, w1_b) = (None, w1) if rank1 else (w1, (None, None))
    w2, (w2_a, w2_b) = (None, w2) if rank2 else (w2, (None, None))
    return (w1, w2, alpha, w1_a, w1_b, w2_a, w2_b, None, None)


def _restated_weight(W, entries, dtype):
    """The reference's calculate_weight for LoRA, LoHa and LoKr entries (in place on the act-dtype W)."""
    for strength, value, _sm, offset, _fn in entries:
        kind, v = (value.__class__.__name__[:4].lower(), value.weights) if not isinstance(value, tuple) else value
        if offset is not None:
            W_ = W.narrow(offset[0], offset[1], offset[2])
        else:
            W_ = W
        if kind == "lokr":
            w1, w2, alpha, w1_a, w1_b, w2_a, w2_b = v[:7]
            dim = None
            if w1 is None:
                dim = w1_b.shape[0]
                w1 = torch.mm(w1_a.float(), w1_b.float())
            if w2 is None:
                dim = w2_b.shape[0]
                w2 = torch.mm(w2_a.float(), w2_b.float())
            alpha = alpha / dim if alpha is not None and dim is not None else 1.0
            delta = torch.kron(w1.float(), w2.float()).reshape(W_.shape)
        elif kind == "loha":
            w1a, w1b, alpha, w2a, w2b = v[:5]
            alpha = 1.0 if alpha is None else alpha / w1b.shape[0]
            delta = (torch.mm(w1a.float(), w1b.float()) * torch.mm(w2a.float(), w2b.float())).reshape(W_.shape)
        else:
            up, down, alpha = v[:3]
            alpha = 1.0 if alpha is None else alpha / down.shape[0]
            delta = torch.mm(up.float(), down.float()).reshape(W_.shape)
        W_ += ((strength * alpha) * delta).type(dtype)
    return W


def _ideal_weight(W, entries):
    """The same patches in float64, never rounded."""
    W = W.double()
    for strength, value, _sm, offset, _fn in entries:
        kind, v = (value.__class__.__name__[:4].lower(), value.weights) if not isinstance(value, tuple) else value
        W_ = W.narrow(offset[0], offset[1], offset[2]) if offset is not None else W
        if kind == "lokr":
            w1, w2, alpha, w1_a, w1_b, w2_a, w2_b = v[:7]
            dim = None
            if w1 is None:
                dim, w1 = w1_b.shape[0], w1_a.double() @ w1_b.double()
            if w2 is None:
                dim, w2 = w2_b.shape[0], w2_a.double() @ w2_b.double()
            alpha = alpha / dim if alpha is not None and dim is not None else 1.0
            W_ += strength * alpha * torch.kron(w1.double(), w2.double())
        elif kind == "loha":
            w1a, w1b, alpha, w2a, w2b = v[:5]
            alpha = 1.0 if alpha is None else alpha / w1b.shape[0]
            W_ += strength * alpha * ((w1a.double() @ w1b.double()) * (w2a.double() @ w2b.double()))
        else:
            up, down, alpha = v[:3]
            alpha = 1.0 if alpha is None else alpha / down.shape[0]
            W_ += strength * alpha * (up.double() @ down.double())
    return W


@pytest.fixture
def calls(pkg, monkeypatch):
    """Names of the library entry points the package calls, in order; and a calculate_weight that knows LoHa / LoKr."""
    L = pkg.lib.lib()
    seen = []
    for name in ("ggufb200_dequant_kron", "ggufb200_gemm", "ggufb200_linear_lora", "ggufb200_linear_lora_ex", "ggufb200_linear",
                 "ggufb200_dequant"):
        real = getattr(L, name)

        def wrapped(*args, _real=real, _name=name):
            seen.append(_name)
            return _real(*args)
        monkeypatch.setattr(L, name, wrapped)
    monkeypatch.setattr(pkg.ops.comfy_lora, "calculate_weight",
                        lambda patches, weight, key, intermediate_dtype=torch.float32, original_weights=None:
                        _restated_weight(weight, patches, weight.dtype))
    return seen


def _kron_call(pkg, qt, raw, N, K, out_dtype, math_dtype, patches):
    """ggufb200_dequant_kron with [(scale, A, B, band)] patches."""
    descs = (pkg.lib.KronPatch * len(patches))(*[
        pkg.lib.KronPatch(A.data_ptr(), B.data_ptr(), A.shape[0], A.shape[1], B.shape[0], B.shape[1], -1 if band is None else band[0], scale,
                          0 if band is None else band[1], 0 if band is None else band[2]) for scale, A, B, band in patches])
    out = torch.empty(N, K, dtype=out_dtype, device=DEV)
    rc = pkg.lib.lib().ggufb200_dequant_kron(int(qt), raw.data_ptr(), N, K, out.data_ptr(), pkg.dequant.dtype_code(out_dtype),
                                             pkg.dequant.dtype_code(math_dtype), descs, len(patches), torch.cuda.current_stream().cuda_stream)
    pkg.lib.check(rc, "ggufb200_dequant_kron")
    return out


SHAPES = [(Q.Q4_K, 384, 1024), (Q.Q6_K, 384, 1024), (Q.Q8_0, 384, 1024), (Q.Q4_K, 64, 640)]   # the last one straddled


@pytest.mark.parametrize("qt,N,K", SHAPES, ids=lambda v: getattr(v, "name", str(v)))
@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("math", ["f16", "target"])
@pytest.mark.parametrize("band", [None, 0, 1], ids=["whole", "rows", "cols"])
def test_dequant_kron_is_the_reference_weight(pkg, qt, N, K, out_dtype, math, band):
    g = torch.Generator().manual_seed(N + K + int(qt))
    raw = _raw(qt, N, K, seed=K)
    math_dtype = torch.float16 if math == "f16" else out_dtype
    W = pkg.dequant.dequantize(raw, qt, (N, K), dtype=math_dtype, out_dtype=out_dtype)
    rows, cols = N, K
    offsets = [None, None]
    if band == 0:
        rows = N // 2
        offsets = [(0, N // 4, rows), (0, N // 2, rows)]
    elif band == 1:
        cols = K // 2
        offsets = [(1, K // 2 - 64, cols), (1, K // 2, cols)]
    # two LoKr patches: a full w2 with alpha ignored, and one with w2 decomposed (scale = alpha / rank)
    entries = [(0.8, ("lokr", _lokr((16, 4), (rows // 16, cols // 4), g, alpha=3.0)), 1.0, offsets[0], None),
               (1.3, ("lokr", _lokr((8, 8), (rows // 8, cols // 8), g, alpha=4.0, rank2=4)), 1.0, offsets[1], None)]
    ops = []
    for kind, scale, factors, bnd in pkg.ops.lycoris_terms(entries):
        ops.append((scale, *pkg.ops.lokr_operands(factors, torch.device(DEV)), bnd))
    want = _restated_weight(W.clone(), entries, out_dtype)
    got = _kron_call(pkg, qt, raw, N, K, out_dtype, math_dtype, ops)
    assert torch.equal(got, want)
    # one patch alone, and none: the plain dequant
    one = _restated_weight(W.clone(), entries[:1], out_dtype)
    assert torch.equal(_kron_call(pkg, qt, raw, N, K, out_dtype, math_dtype, ops[:1]), one)
    assert torch.equal(_kron_call(pkg, qt, raw, N, K, out_dtype, math_dtype, []), W)


def _rel(a, b):
    return float((a.double() - b).norm() / b.norm())


@pytest.mark.parametrize("qt,N,K", SHAPES, ids=lambda v: getattr(v, "name", str(v)))
@pytest.mark.parametrize("M", [3, 300])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_lokr_linear_meets_the_exact_budget(pkg, qt, N, K, M, dtype, calls):
    lin = _layer(pkg, qt, N, K, seed=M)
    g = torch.Generator().manual_seed(M + N)
    entries = [(0.7, ("lokr", _lokr((16, 16), (N // 16, K // 16), g, alpha=2.0, rank1=4)), 1.0, None, None),
               (1.1, LoKrAdapter(_lokr((4, 8), (N // 8, K // 8), g, alpha=None, rank2=8)), 1.0, (0, N // 2, N // 2), None)]
    lin.weight.patches = [(entries, "diffusion_model.w")]
    x = (torch.randn(M, K, generator=g) * 0.5).to(DEV).to(dtype)
    y = lin(x)
    assert calls == ["ggufb200_dequant_kron", "ggufb200_gemm"], calls
    W = _restated_weight(pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, dtype)).clone(), entries, dtype)
    ref = torch.nn.functional.linear(x, W, pkg.ops._plain(lin.bias).to(dtype)).double()   # what the reference's Linear returns
    assert y.dtype == dtype and _rel(y, ref) <= 1e-3
    # the two-step route (lora_side_gemm = False) computes the same weight through calculate_weight
    calls.clear()
    lin.lora_side_gemm = False
    try:
        y2 = lin(x)
    finally:
        del lin.lora_side_gemm
    assert "ggufb200_dequant_kron" not in calls and _rel(y2, ref) <= 1e-3
    lin.weight.patches = []


def _check_lora_budget(y, ref, ideal, dtype, what):
    err = _rel(y, ref)
    assert err <= (3e-3 if dtype == torch.float16 else 1e-2), (what, err)
    assert _rel(y, ideal) <= 1.5 * _rel(ref.to(dtype), ideal) + 1e-4, (what, _rel(y, ideal), _rel(ref.to(dtype), ideal))


def _loha(rows, cols, dim, g, alpha):
    f = [(torch.randn(*s, generator=g) * 0.2).to(DEV) for s in ((rows, dim), (dim, cols), (rows, dim), (dim, cols))]
    return (f[0], f[1], alpha, f[2], f[3], None, None, None)


def _references(pkg, lin, x, entries):
    dtype = x.dtype
    W = pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, dtype))
    bias = pkg.ops._plain(lin.bias).to(dtype).double()
    ref = torch.nn.functional.linear(x.double(), _restated_weight(W.clone(), entries, dtype).double(), bias)
    return ref, torch.nn.functional.linear(x.double(), _ideal_weight(W, entries), bias)


@pytest.mark.parametrize("dim,route", [(4, "ggufb200_linear_lora"), (16, "ggufb200_linear_lora_ex"), (32, "ggufb200_linear")])
@pytest.mark.parametrize("M", [3, 300])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_loha_runs_as_lora(pkg, dim, route, M, dtype, calls):
    """dim 4 / 16: rank 16 / 256 in the fused kernel's LoRA k-blocks; dim 32 = rank 1024 > 512: the side GEMMs."""
    N, K = 512, 1024
    lin = _layer(pkg, Q.Q4_K, N, K, seed=dim)
    g = torch.Generator().manual_seed(dim + M)
    entries = [(0.9, ("loha", _loha(N, K, dim, g, float(dim) / 2)), 1.0, None, None)]
    lin.weight.patches = [(entries, "diffusion_model.w")]
    x = (torch.randn(M, K, generator=g) * 0.5).to(DEV).to(dtype)
    y = lin(x)
    assert calls[-1] == route and "ggufb200_dequant_kron" not in calls and "ggufb200_dequant" not in calls, calls
    ref, ideal = _references(pkg, lin, x, entries)
    _check_lora_budget(y, ref, ideal, dtype, dim)
    # cached: the second forward builds nothing and gives the same result
    assert torch.equal(lin(x), y)
    lin.weight.patches = []


@pytest.mark.parametrize("M", [3, 300])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_mixed_lora_loha_lokr(pkg, M, dtype, calls):
    """LoRA + LoHa (row band) + LoKr in one list: the patched weight by dequant_kron + GEMM, the rest as side GEMMs."""
    N, K = 768, 1024
    H = N // 3
    lin = _layer(pkg, Q.Q4_K, N, K, seed=5)
    g = torch.Generator().manual_seed(M)
    up, down = (torch.randn(N, 16, generator=g) * 0.05).to(DEV), (torch.randn(16, K, generator=g) * 0.05).to(DEV)
    entries = [(0.6, ("lora", (up, down, 8.0, None, None, None)), 1.0, None, None),
               (0.8, LoHaAdapter(_loha(H, K, 8, g, 4.0)), 1.0, (0, H, H), None),
               (1.2, ("lokr", _lokr((16, 16), (N // 16, K // 16), g, alpha=8.0, rank2=16)), 1.0, None, None)]
    lin.weight.patches = [(entries, "diffusion_model.w")]
    x = (torch.randn(M, K, generator=g) * 0.5).to(DEV).to(dtype)
    y = lin(x)
    assert calls[:2] == ["ggufb200_dequant_kron", "ggufb200_gemm"] and "ggufb200_linear_lora_ex" not in calls, calls
    ref, ideal = _references(pkg, lin, x, entries)
    _check_lora_budget(y, ref, ideal, dtype, "mixed")
    lin.weight.patches = []
