"""GPU tests of DoRA (weight-decomposed LoRA) patches on a packed weight.

The layer keeps the patched weight in the compact form diag(r) W0 diag(c) + sum_j diag(rho_j) a_j st_j up_j down_j diag(gamma_j)
(ops.dora_compact) with the reference's own DoRA factors, and runs it either inside the fused kernel
(ggufb200_linear_lora_scaled: feature scale r, input columns scaled by ggufb200_scale_columns) or as the dequantised weight +
ggufb200_gemm_scaled + side GEMMs.  Its output must meet the LoRA budget of tests/test_gpu_lora_slices.py against the two-step
route, which runs `calculate_weight` with the reference's `weight_decompose` restated below.

DoRA magnitudes are drawn as the dequantised weight's own row / column norms times U(0.8, 1.2), as trainers initialise them
(factors s near 1).  Far from that (s ~ 0.005 with unit magnitudes on these random weights) the reference's own bf16 blend
`W + 0.8 (Wc - W)` cancels and lands ~1.2e-2 from the float64 weight, while this route stays within ~2e-3 of it."""
import pytest
import torch

import oracle
from fallback_cases import random_blocks as fallback_blocks
from util import Q

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


def _delta(kind, v, dtype=torch.float32):
    """The entry's delta and alpha / rank as calculate_weight forms them (fp32, or float64 for the ideal weight)."""
    if kind == "lora":
        up, down, alpha = v[:3]
        return torch.mm(up.to(dtype), down.to(dtype)), 1.0 if alpha is None else alpha / down.shape[0], v[4] if len(v) > 4 else None
    if kind == "loha":
        w1a, w1b, alpha, w2a, w2b = v[:5]
        d = torch.mm(w1a.to(dtype), w1b.to(dtype)) * torch.mm(w2a.to(dtype), w2b.to(dtype))
        return d, 1.0 if alpha is None else alpha / w1b.shape[0], v[7] if len(v) > 7 else None
    w1, w2, alpha = v[:3]                                 # lokr, whole factors only
    return torch.kron(w1.to(dtype), w2.to(dtype)), 1.0, v[8]


def weight_decompose(dora_scale, weight, lora_diff, alpha, strength):
    """ComfyUI's weight_decompose (comfy/weight_adapter/base.py), restated for 2-D weights."""
    dora_scale = dora_scale.to(device=weight.device, dtype=torch.float32)
    lora_diff *= alpha
    weight_calc = weight + lora_diff.type(weight.dtype)
    if dora_scale.shape[0] == weight_calc.shape[0]:
        weight_norm = weight.reshape(weight.shape[0], -1).norm(dim=1, keepdim=True).reshape(weight.shape[0], 1)
    else:
        weight_norm = (weight_calc.transpose(0, 1).reshape(weight_calc.shape[1], -1).norm(dim=1, keepdim=True)
                       .reshape(weight_calc.shape[1], 1).transpose(0, 1))
    weight_norm = weight_norm + torch.finfo(weight.dtype).eps
    weight_calc *= (dora_scale / weight_norm).type(weight.dtype)
    if strength != 1.0:
        weight_calc -= weight
        weight += strength * weight_calc
    else:
        weight[:] = weight_calc
    return weight


def restated_calculate_weight(patches, weight, key, intermediate_dtype=torch.float32, original_weights=None):
    for entry in patches:
        strength, value = entry[0], entry[1]
        offset = entry[3] if len(entry) > 3 else None
        kind, v = (value.__class__.__name__[:4].lower(), value.weights) if not isinstance(value, tuple) else value
        W = weight.narrow(offset[0], offset[1], offset[2]) if offset is not None else weight
        delta, alpha, dora_scale = _delta(kind, v)
        delta = delta.reshape(W.shape)
        if dora_scale is not None:
            weight_decompose(dora_scale, W, delta, alpha, strength)
        else:
            W += ((strength * alpha) * delta).type(W.dtype)
    return weight


def ideal_weight(W, entries):
    """The same patches in float64, never rounded (DoRA norms in float64 too, plus the eps of W's dtype as the reference adds)."""
    eps = torch.finfo(W.dtype).eps
    W = W.double()
    N = W.shape[0]
    for strength, value, *_rest in entries:
        kind, v = (value.__class__.__name__[:4].lower(), value.weights) if not isinstance(value, tuple) else value
        delta, alpha, dora_scale = _delta(kind, v, torch.float64)
        delta = alpha * delta
        if dora_scale is None:
            W = W + strength * delta
            continue
        Wc = W + delta
        out = dora_scale.shape[0] == N
        nrm = (W.norm(dim=1) if out else Wc.norm(dim=0)) + eps
        s = dora_scale.double().reshape(-1) / nrm
        Wc = Wc * (s[:, None] if out else s[None, :])
        W = W + strength * (Wc - W)
    return W


@pytest.fixture
def calls(pkg, monkeypatch):
    """Names of the library entry points the package calls, in order (calculate_weight included)."""
    L = pkg.lib.lib()
    seen = []
    for name in ("ggufb200_gemm", "ggufb200_gemm_scaled", "ggufb200_linear_lora", "ggufb200_linear_lora_ex", "ggufb200_linear_lora_scaled",
                 "ggufb200_linear", "ggufb200_linear_spans", "ggufb200_dequant", "ggufb200_dequant_fallback", "ggufb200_scale_columns"):
        real = getattr(L, name)

        def wrapped(*args, _real=real, _name=name):
            seen.append(_name)
            return _real(*args)
        monkeypatch.setattr(L, name, wrapped)

    def counted(*args, **kwargs):
        seen.append("calculate_weight")
        return restated_calculate_weight(*args, **kwargs)
    monkeypatch.setattr(pkg.ops.comfy_lora, "calculate_weight", counted)
    return seen


def _rel(a, b):
    return float((a.double() - b).norm() / b.norm())


# ------------------------------------------------------------------ the kernels
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("M,K", [(1, 8), (77, 1024), (4096, 3072)])
def test_scale_columns_is_torch(pkg, dtype, M, K):
    g = torch.Generator().manual_seed(M + K)
    x = (torch.randn(M, K + 8, generator=g) * 3).to(DEV).to(dtype)[:, :K]              # strided rows (ldx = K + 8)
    c = (torch.rand(K, generator=g) * 4 - 2).to(DEV)
    c[0] = 0.0
    y = pkg.ops.scale_columns(x, c)
    assert y.dtype == dtype and torch.equal(y, (x.float() * c).to(dtype))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [4, 300, 2048])
def test_gemm_scaled(pkg, dtype, M):
    N, K = 512, 1024
    g = torch.Generator().manual_seed(M)
    x = torch.randn(M, K, generator=g).to(DEV).to(dtype)
    W = (torch.randn(N, K, generator=g) * 0.05).to(DEV).to(dtype)
    b = (torch.randn(N, generator=g) * 0.1).to(DEV)
    scale = (torch.rand(N, generator=g) * 2 - 0.5).to(DEV)
    L = pkg.lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    code = pkg.dequant.dtype_code(dtype)

    def gemm_scaled(s):
        y = torch.empty(M, N, dtype=dtype, device=DEV)
        pkg.lib.check(L.ggufb200_gemm_scaled(W.data_ptr(), N, K, K, x.data_ptr(), M, K, code, b.data_ptr(), 2, s, y.data_ptr(), N, st), "gemm")
        return y
    assert torch.equal(gemm_scaled(None), pkg.ops.linear_dense(x, W, b))
    want = scale.double() * (x.double() @ W.double().t()) + b.to(dtype).double()
    assert _rel(gemm_scaled(scale.data_ptr()), want) <= 1e-3 + (4e-3 if dtype == torch.bfloat16 else 0)
    assert torch.equal(gemm_scaled(scale.data_ptr()), pkg.ops.linear_dense(x, W, b, scale))


@pytest.mark.parametrize("qt,N,K", [(Q.Q4_K, 512, 1024), (Q.Q6_K, 384, 1024), (Q.Q4_K, 64, 640)], ids=["Q4_K", "Q6_K", "Q4_K_straddled"])
@pytest.mark.parametrize("M", [4, 300, 4096])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_linear_lora_scaled(pkg, qt, N, K, M, dtype):
    """NULL scale: ggufb200_linear_lora_ex bit for bit; a scale: within 1e-3 of the float64 product for fp16 outputs, 5e-3 for bf16
    (the output rounding alone is ~1.5e-3 there); split K and its finalize are included (M = 4)."""
    g = torch.Generator().manual_seed(M + N)
    bs, _ts = oracle.type_info(int(qt))
    raw = torch.from_numpy(oracle.random_blocks(int(qt), N * K // bs, seed=M, scale=0.02).reshape(-1)).to(DEV)
    w = pkg.ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size((N, K)))
    spans = pkg.ops.span_layout(w, raw) if pkg.ops.needs_span_layout(qt, K) else None
    x = torch.randn(M, K, generator=g).to(DEV).to(dtype)
    down = (torch.randn(96, K, generator=g) * 0.05).to(DEV)
    up = (torch.randn(N, 96, generator=g) * 0.05).to(DEV)
    b = (torch.randn(N, generator=g) * 0.1).to(DEV)
    down_pad, u_pad, _tiles = pkg.ops.lora_kernel_operands([(1.0, up, down, None)], N, K, dtype, torch.device(DEV))
    t = pkg.ops.linear_dense(x, down_pad)
    algo = pkg.lib.ALGO_FUSED_TMEM | pkg.lib.FLAG_EXACT_W
    plain = pkg.ops._launch_linear(x, raw, qt, N, K, b, pkg.lib.F16, algo, spans, (t, u_pad, None))
    none = pkg.ops._launch_linear(x, raw, qt, N, K, b, pkg.lib.F16, algo, spans, (t, u_pad, None), None)
    assert torch.equal(none, plain)
    scale = (torch.rand(N, generator=g) * 2 - 0.5).to(DEV)
    y = pkg.ops._launch_linear(x, raw, qt, N, K, b, pkg.lib.F16, algo, spans, (t, u_pad, None), scale)
    W = pkg.dequant.dequantize(raw, qt, (N, K), out_dtype=dtype).double()
    want = scale.double() * (x.double() @ W.t() + t.double() @ u_pad.double().t()) + b.to(dtype).double()
    assert _rel(y, want) <= 1e-3 + (4e-3 if dtype == torch.bfloat16 else 0)


# ------------------------------------------------------------------ the layer
def _layer(pkg, qt, N, K, seed, bias):
    if qt == Q.BF16:
        raw = (torch.randn(N, K, generator=torch.Generator().manual_seed(seed)) * 0.02).bfloat16().view(torch.uint8).to(DEV)
    elif qt == Q.IQ2_XXS:
        raw = torch.from_numpy(fallback_blocks(qt, N * K // 256, seed=seed, scale=0.002).reshape(-1)).to(DEV)
    else:
        bs, _ts = oracle.type_info(int(qt))
        raw = torch.from_numpy(oracle.random_blocks(int(qt), N * K // bs, seed=seed, scale=0.02).reshape(-1)).to(DEV)
    lin = pkg.ops.GGMLOps.Linear(K, N)
    sd = {"weight": pkg.ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size((N, K)))}
    if bias:
        b = (torch.randn(N, generator=torch.Generator().manual_seed(seed + 1)) * 0.02).to(DEV)
        sd["bias"] = pkg.ops.GGMLTensor(b, tensor_type=Q.F32, tensor_shape=torch.Size((N,)))
    lin.load_state_dict(sd)
    return lin


def _magnitude(W, axis, g):
    """A DoRA magnitude for weight W: its row (axis 0, [N, 1]) or column (axis 1, [1, K]) norms times U(0.8, 1.2)."""
    nrm = W.float().norm(dim=1 - axis, keepdim=True)
    return nrm * (torch.rand(*nrm.shape, generator=g) * 0.4 + 0.8).to(nrm.device)


def _entries(N, K, axis, st, g, W):
    """DoRA entry on `axis` with strength st, then a plain LoRA, then a DoRA LoHa on the same axis (W: the dequantised weight)."""
    def ds():
        return _magnitude(W, axis, g)
    up, down = (torch.randn(N, 16, generator=g) * 0.05).to(DEV), (torch.randn(16, K, generator=g) * 0.05).to(DEV)
    up2, down2 = (torch.randn(N, 8, generator=g) * 0.05).to(DEV), (torch.randn(8, K, generator=g) * 0.05).to(DEV)
    loha = [(torch.randn(*s, generator=g) * 0.2).to(DEV) for s in ((N, 2), (2, K), (N, 2), (2, K))]
    return [(st, ("lora", (up, down, 8.0, None, ds(), None)), 1.0, None, None),
            (0.9, LoRAAdapter((up2, down2, None, None, None, None)), 1.0, None, None),
            (st, LoHaAdapter((loha[0], loha[1], 1.0, loha[2], loha[3], None, None, ds())), 1.0, None, None)]


def _weight(pkg, lin, dtype):
    return pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, dtype))


def _references(pkg, lin, x, entries):
    dtype = x.dtype
    W = pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, dtype))
    bias = pkg.ops._plain(lin.bias).to(dtype).double() if lin.bias is not None else None
    ref = torch.nn.functional.linear(x.double(), restated_calculate_weight(entries, W.clone(), None).double(), bias)
    return ref, torch.nn.functional.linear(x.double(), ideal_weight(W, entries), bias)


def _in_kernel(pkg, qt, K, M):
    if qt in (Q.BF16, Q.IQ2_XXS):
        return False
    spans = M > pkg.ops.GEMV_MAX_M and not pkg.ops.straddled_rows(qt, K)
    return spans or not pkg.ops.needs_span_layout(qt, K)


LAYERS = [(Q.Q4_K, 384, 1024), (Q.Q6_K, 384, 1024), (Q.Q8_0, 384, 1024), (Q.Q4_K, 64, 640), (Q.IQ2_XXS, 256, 512), (Q.BF16, 256, 512)]


@pytest.mark.parametrize("qt,N,K", LAYERS, ids=["Q4_K", "Q6_K", "Q8_0", "Q4_K_straddled", "IQ2_XXS", "BF16"])
@pytest.mark.parametrize("M", [1, 4, 77, 512, 4096])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("axis", [0, 1], ids=["out", "in"])
@pytest.mark.parametrize("st", [1.0, 0.8])
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
def test_dora_linear_meets_the_lora_budget(pkg, qt, N, K, M, dtype, axis, st, bias, calls):
    lin = _layer(pkg, qt, N, K, seed=M + axis, bias=bias)
    g = torch.Generator().manual_seed(M * 4 + axis * 2 + int(st == 1.0))
    entries = _entries(N, K, axis, st, g, _weight(pkg, lin, dtype))
    lin.weight.patches = [(entries, "diffusion_model.w")]
    x = (torch.randn(M, K, generator=g) * 0.5).to(DEV).to(dtype)
    y = lin(x)
    route = "ggufb200_linear_lora_scaled" if _in_kernel(pkg, qt, K, M) else "ggufb200_gemm_scaled"
    assert "calculate_weight" not in calls and route in calls, calls
    assert ("ggufb200_scale_columns" in calls) == (axis == 1), calls
    ref, ideal = _references(pkg, lin, x, entries)
    err = _rel(y, ref)
    assert y.dtype == dtype and err <= (3e-3 if dtype == torch.float16 else 1e-2), err
    assert _rel(y, ideal) <= 1.5 * _rel(ref.to(dtype), ideal) + 1e-4, (_rel(y, ideal), _rel(ref.to(dtype), ideal))
    lin.weight.patches = []


def test_plan_is_built_once_and_rebuilt_on_change(pkg, calls):
    N, K = 384, 1024
    lin = _layer(pkg, Q.Q4_K, N, K, seed=1, bias=True)
    g = torch.Generator().manual_seed(1)
    entries = _entries(N, K, 0, 0.8, g, _weight(pkg, lin, torch.float16))
    lin.weight.patches = [(entries, "w")]
    x = torch.randn(77, K, generator=g).to(DEV).half()
    calls.clear()                                                               # (the magnitudes above dequantised the weight)
    y = lin(x)
    first = list(calls)
    assert first.count("ggufb200_dequant") == 1 and first[-1] == "ggufb200_linear_lora_scaled", first      # K1 for the plan
    plan = lin._gg_dora[1]
    calls.clear()
    assert torch.equal(lin(x), y)
    assert calls == ["ggufb200_gemm", "ggufb200_linear_lora_scaled"] and lin._gg_dora[1] is plan, calls      # T, then the fused call
    entries[0][1][1][4].mul_(1.5)                                               # dora_scale modified in place: a new plan
    calls.clear()
    y2 = lin(x)
    assert "ggufb200_dequant" in calls and lin._gg_dora[1] is not plan and not torch.equal(y2, y)
    ref, _ideal = _references(pkg, lin, x, entries)
    assert _rel(y2, ref) <= 3e-3
    # the same patch set in bf16: the factors depend on the activation dtype, so another plan
    plan16 = lin._gg_dora[1]
    lin(x.bfloat16())
    assert lin._gg_dora[1] is not plan16
    lin.weight.patches = []


@pytest.mark.parametrize("case", ["lora_in_kernel_off", "rank_above_512", "zero_row"])
def test_side_form(pkg, case, calls):
    N, K = 384, 1024
    lin = _layer(pkg, Q.Q4_K, N, K, seed=2, bias=True)
    g = torch.Generator().manual_seed(2)
    entries = _entries(N, K, 0, 1.0, g, _weight(pkg, lin, torch.float16))
    if case == "lora_in_kernel_off":
        lin.lora_in_kernel = False
    elif case == "rank_above_512":
        entries.append((0.5, ("lora", ((torch.randn(N, 520, generator=g) * 0.01).to(DEV), (torch.randn(520, K, generator=g) * 0.01).to(DEV),
                                        None, None, None, None)), 1.0, None, None))
    else:
        entries[0][1][1][4][5] = 0.0                                            # s = 0 on row 5 at strength 1: r_5 = 0
    lin.weight.patches = [(entries, "w")]
    x = torch.randn(300, K, generator=g).to(DEV).half()
    y = lin(x)
    assert "ggufb200_gemm_scaled" in calls and "ggufb200_linear_lora_scaled" not in calls and "calculate_weight" not in calls, calls
    ref, ideal = _references(pkg, lin, x, entries)
    assert _rel(y, ref) <= 3e-3 and _rel(y, ideal) <= 1.5 * _rel(ref.half(), ideal) + 1e-4
    if case == "zero_row":
        assert lin._gg_dora[1].kernel is None and _rel(y[:, 5], ref[:, 5]) <= 3e-3
    lin.weight.patches = []


@pytest.mark.parametrize("case", ["banded", "lokr", "side_gemm_off", "patch_dtype"])
def test_rejected_lists_keep_the_two_step_route(pkg, case, calls):
    N, K = 256, 512
    lin = _layer(pkg, Q.Q4_K, N, K, seed=3, bias=False)
    g = torch.Generator().manual_seed(3)
    W = _weight(pkg, lin, torch.float16)
    entries = _entries(N, K, 0, 1.0, g, W)[:1]
    if case == "banded":
        up, down = (torch.randn(N // 2, 4, generator=g) * 0.05).to(DEV), (torch.randn(4, K, generator=g) * 0.05).to(DEV)
        entries = [(1.0, ("lora", (up, down, None, None, _magnitude(W[:N // 2], 0, g), None)), 1.0, (0, 0, N // 2), None)]
    elif case == "lokr":
        w1, w2 = (torch.randn(4, 4, generator=g) * 0.2).to(DEV), (torch.randn(N // 4, K // 4, generator=g) * 0.2).to(DEV)
        entries = [(1.0, ("lokr", (w1, w2, None, None, None, None, None, None, _magnitude(W, 0, g))), 1.0, None, None)]
    elif case == "side_gemm_off":
        lin.lora_side_gemm = False
    else:
        lin.patch_dtype = torch.float32
    lin.weight.patches = [(entries, "w")]
    x = torch.randn(77, K, generator=g).to(DEV).half()
    y = lin(x)
    assert "calculate_weight" in calls and "ggufb200_gemm_scaled" not in calls and "ggufb200_linear_lora_scaled" not in calls, calls
    if case != "patch_dtype":
        ref = torch.nn.functional.linear(x.double(), restated_calculate_weight(entries, W.clone(), None).double())
        assert _rel(y, ref) <= 1e-3
    lin.weight.patches = []
