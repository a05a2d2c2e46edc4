"""GPU tests of LoRA / LoCon and LoHa patches on a packed Conv2d weight (ggufb200_dequant_lowrank through GGMLOps.Conv2d).

The reference is the layer's own two-step route (`conv_patches_in_kernel = False`): dequantize_tensor, then calculate_weight, here
restated for LoRA and LoHa as ComfyUI's adapters compute them:
    LoRA  diff = torch.mm(up.flatten(start_dim=1), down.flatten(start_dim=1)).reshape(weight.shape)      (fp32)
    LoHa  diff = (torch.mm(w1a, w1b) * torch.mm(w2a, w2b)).reshape(weight.shape)                          (fp32)
          weight += ((strength * alpha) * diff).type(weight.dtype)
The kernel follows the same per-element rounding sequence; only the order of the fp32 rank sums differs from cuBLAS, so the
patched weights must be bit-identical except for a small fraction of elements, each at most 1 ulp of the activation dtype apart at
the element's magnitude |W0| + sum |s d| (where w + delta cancels, that is more than one ulp of the small result).
Each element is also checked against a float64 restatement with a bound derived from the rounding sequence."""
import gguf
import pytest
import torch

import oracle
from fallback_cases import random_blocks as fallback_blocks
from util import Q

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FALLBACK = (Q.IQ2_XXS, Q.MXFP4)
MAX_DIFF_FRACTION = 0.01       # elements of the patched weight that may differ from the two-step route (by one ulp at their magnitude)


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


def _payload(v):
    return (v[0], tuple(v[1])) if isinstance(v, tuple) else (type(v).__name__[:4].lower(), tuple(v.weights))


@pytest.fixture
def restated(pkg, monkeypatch):
    """calculate_weight with ComfyUI's LoRA and LoHa arithmetic (the package's test double knows LoRA only)."""
    original = pkg.ops.comfy_lora.calculate_weight

    def calculate_weight(patches, weight, key, intermediate_dtype=torch.float32, original_weights=None):
        if not all(_payload(p[1])[0] in ("lora", "loha") and p[2] == 1.0 for p in patches):
            return original(patches, weight, key, intermediate_dtype, original_weights)
        for p in patches:
            strength, (kind, v) = p[0], _payload(p[1])
            f = [t.to(device=weight.device, dtype=intermediate_dtype) for t in (v[:2] if kind == "lora" else v[:2] + v[3:5])]
            if kind == "lora":
                alpha = 1.0 if v[2] is None else v[2] / f[1].shape[0]
                diff = torch.mm(f[0].flatten(start_dim=1), f[1].flatten(start_dim=1)).reshape(weight.shape)
            else:
                alpha = 1.0 if v[2] is None else v[2] / f[1].shape[0]
                diff = (torch.mm(f[0], f[1]) * torch.mm(f[2], f[3])).reshape(weight.shape)
            weight += ((strength * alpha) * diff).type(weight.dtype)
        return weight
    monkeypatch.setattr(pkg.ops.comfy_lora, "calculate_weight", calculate_weight)


@pytest.fixture
def kernel(pkg, monkeypatch):
    """The layer takes ggufb200_dequant_lowrank wherever it can, whatever its cost model (`lowrank_pays`) would pick: these tests
    check the kernel, including ranks where the two-step route is faster."""
    monkeypatch.setattr(pkg.ops, "lowrank_pays", lambda N, K, terms: True)


@pytest.fixture
def calls(pkg, monkeypatch):
    """Names of the dequant entry points the package calls, in order."""
    L = pkg.lib.lib()
    seen = []
    for name in ("ggufb200_dequant_lowrank", "ggufb200_dequant", "ggufb200_dequant_fallback", "ggufb200_dequant_kron"):
        real = getattr(L, name)

        def wrapped(*args, _real=real, _name=name):
            seen.append(_name)
            return _real(*args)
        monkeypatch.setattr(L, name, wrapped)
    return seen


def _raw(qt, numel, seed):
    bs, _ts = gguf.GGML_QUANT_SIZES[qt]
    blocks = fallback_blocks(qt, numel // bs, seed=seed, scale=0.02) if qt in FALLBACK else oracle.random_blocks(int(qt), numel // bs, seed=seed, scale=0.02)
    return torch.from_numpy(blocks.reshape(-1)).to(DEV)


def _entries(spec, shape, seed, factor_dtype=torch.float32):
    """Patch entries of (kind, rank(s), strength, alpha) specs for a conv weight of `shape`: LoRA / LoCon as 4-D factors, LoHa as
    the 2-D factors LyCORIS stores."""
    g = torch.Generator().manual_seed(seed)
    cout, cin, kh, kw = shape
    K = cin * kh * kw
    out = []
    for i, (kind, ranks, strength, alpha) in enumerate(spec):
        def f(*s):
            return (torch.randn(*s, generator=g) * 0.1).to(factor_dtype).to(DEV)
        if kind == "lora":
            r = ranks
            payload = (f(cout, r, 1, 1), f(r, cin, kh, kw), alpha, None, None, None)
            value = ("lora", payload) if i % 2 == 0 else LoRAAdapter(payload)
        else:
            r1, r2 = ranks
            payload = (f(cout, r1), f(r1, K), alpha, f(cout, r2), f(r2, K), None, None, None)
            value = ("loha", payload) if i % 2 == 0 else LoHaAdapter(payload)
        out.append((strength, value, 1.0, None, None))
    return out


def _conv(pkg, qt, shape, entries, seed=0, raw=None):
    cout, cin, kh, kw = shape
    conv = pkg.ops.GGMLOps.Conv2d(cin, cout, (kh, kw), padding=kh // 2, device="meta")
    raw = _raw(qt, cout * cin * kh * kw, seed) if raw is None else raw
    w = pkg.ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size(shape), patches=[(entries, "diffusion_model.conv.weight")])
    bias = (torch.randn(cout, generator=torch.Generator().manual_seed(seed + 7)) * 0.05).to(DEV)
    conv.load_state_dict({"weight": w, "bias": bias}, assign=True)
    return conv


def _weight(conv, x, in_kernel):
    """The (weight, bias) the layer hands to _conv_forward with the class switch set to `in_kernel`, and the output."""
    seen = {}
    real = conv._conv_forward

    def spy(inp, w, b):
        seen["w"], seen["b"] = w, b
        return real(inp, w, b)
    conv._conv_forward = spy
    conv.conv_patches_in_kernel = in_kernel
    try:
        y = conv(x)
    finally:
        del conv._conv_forward
        del conv.conv_patches_in_kernel
    return seen["w"], seen["b"], y


def _ideal(pkg, conv, dtype, entries):
    """(float64 patched weight, per-element error bound) from the act-dtype dequantised weight and the patch factors."""
    w = conv.weight
    W0 = pkg.dequant.dequantize_tensor(w, dtype, conv.dequant_dtype)
    W0 = W0.as_subclass(torch.Tensor).double().reshape(W0.shape[0], -1)
    ideal, mag, fp32_err = W0.clone(), W0.abs(), torch.zeros_like(W0)
    for strength, value, *_ in entries:
        kind, v = _payload(value)
        if kind == "lora":
            up, down = v[0].double().flatten(1), v[1].double().flatten(1)
            a = 1.0 if v[2] is None else v[2] / down.shape[0]
            d, m, r = up @ down, up.abs() @ down.abs(), down.shape[0]
        else:
            w1a, w1b, w2a, w2b = (t.double() for t in v[:2] + v[3:5])
            a = 1.0 if v[2] is None else v[2] / w1b.shape[0]
            d, m, r = (w1a @ w1b) * (w2a @ w2b), (w1a.abs() @ w1b.abs()) * (w2a.abs() @ w2b.abs()), w1b.shape[0] + w2b.shape[0] + 1
        s = strength * a
        ideal += s * d
        mag += abs(s) * m
        fp32_err += abs(s) * (r + 1) * 2.0 ** -23 * m
    n = len(entries)
    u, tiny = {torch.float16: (2.0 ** -11, 2.0 ** -24), torch.bfloat16: (2.0 ** -8, 2.0 ** -133), torch.float32: (2.0 ** -24, 2.0 ** -149)}[dtype]
    return ideal, 2 * n * (u * mag + tiny) + fp32_err, mag, fp32_err


def _ulp(mag, dtype):
    """One ulp of the activation dtype at magnitude `mag` (float64 tensor), subnormals included."""
    bits, emin = {torch.float16: (10, -14), torch.bfloat16: (7, -126), torch.float32: (23, -126)}[dtype]
    e = torch.floor(torch.log2(mag.clamp_min(2.0 ** emin))).clamp_min(emin)
    return torch.exp2(e - bits)


# (format, conv shape, patch specs, activation dtype, dequant_dtype).  K = Cin kh kw: 320 and 2880 / 5760 are straddled for the
# 256-element formats, 11520 (SDXL 3x3 at 1280 channels) is not.
CASES = [
    (Q.Q4_0, (320, 320, 1, 1), [("lora", 16, 1.0, 8.0)], torch.float16, None),
    (Q.Q8_0, (640, 320, 3, 3), [("lora", 64, 1.0, 32.0)], torch.bfloat16, None),
    (Q.Q8_0, (320, 320, 1, 1), [("lora", 128, -0.8, 64.0)], torch.float16, None),
    (Q.Q4_K, (1280, 1280, 3, 3), [("lora", 128, 1.0, 64.0)], torch.float16, None),
    (Q.Q6_K, (1280, 1280, 3, 3), [("loha", (16, 16), 1.0, 8.0)], torch.bfloat16, None),
    (Q.Q4_K, (640, 320, 3, 3), [("lora", 1, 1.0, None)], torch.float16, None),
    (Q.Q4_K, (320, 320, 1, 1), [("lora", 16, 1.0, 16.0)], torch.bfloat16, "target"),
    (Q.Q6_K, (640, 640, 3, 3), [("lora", 64, 0.7, 32.0), ("loha", (8, 4), -1.0, 4.0)], torch.float16, None),
    (Q.Q4_K, (640, 640, 3, 3), [("loha", (16, 8), -0.5, 16.0)], torch.bfloat16, None),
    (Q.Q6_K, (320, 320, 1, 1), [("lora", 16, 1.0, 8.0), ("lora", 1, 1.0, 1.0)], torch.bfloat16, None),
    (Q.IQ2_XXS, (640, 320, 3, 3), [("lora", 16, 1.0, 8.0)], torch.float16, None),
    (Q.MXFP4, (320, 320, 1, 1), [("lora", 64, 1.0, 32.0), ("loha", (4, 4), 0.5, 2.0)], torch.bfloat16, None),
    (Q.Q8_0, (640, 640, 3, 3), [("lora", 80, 1.0, 32.0)], torch.float16, None),                          # rank tail: 32 + 32 + 16
    (Q.Q6_K, (640, 320, 3, 3), [("lora", 48, 1.0, 16.0), ("loha", (40, 8), -0.5, 8.0)], torch.float32, None),   # fp32 output
]


def _case_id(c):
    qt, shape, spec, dtype, math = c
    kinds = "+".join(f"{k}{r if isinstance(r, int) else 'x'.join(map(str, r))}" for k, r, *_ in spec)
    return f"{qt.name}-{'x'.join(map(str, shape))}-{kinds}-{str(dtype)[6:]}" + (f"-{math}" if math else "")


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_patched_weight_matches_the_two_step_route(pkg, restated, kernel, calls, case):
    qt, shape, spec, dtype, math = case
    entries = _entries(spec, shape, seed=shape[0] + shape[1] + int(qt), factor_dtype=torch.float16 if len(spec) > 1 else torch.float32)
    conv = _conv(pkg, qt, shape, entries, seed=int(qt))
    conv.dequant_dtype = math
    x = (torch.randn(2, shape[1], 16, 16, generator=torch.Generator().manual_seed(3)) * 0.5).to(DEV).to(dtype)
    calls.clear()
    W, b, y = _weight(conv, x, True)
    assert calls == ["ggufb200_dequant_lowrank"], calls                  # one launch, no K1 + calculate_weight
    W_ref, b_ref, y_ref = _weight(conv, x, False)
    assert W.dtype == dtype and tuple(W.shape) == shape and torch.equal(b, b_ref)
    assert bool(torch.isfinite(W).all())
    # 16-bit outputs: bit-identical but for a small fraction, each within one activation-dtype ulp at the element's magnitude
    # (|W0| + sum |s d|: where w + delta cancels, one ulp of delta is many ulps of the small result).  fp32 output keeps the fp32
    # rank sums' own rounding, which differs between the two summation orders in most elements: within twice its bound.
    ideal, bound, mag, fp32_err = _ideal(pkg, conv, dtype, entries)
    diff = (W.reshape(shape[0], -1).double() - W_ref.reshape(shape[0], -1).double()).abs()
    if dtype == torch.float32:
        assert bool((diff <= _ulp(mag, dtype) + 2 * fp32_err).all())
    else:
        frac = (W.view(torch.int16) != W_ref.view(torch.int16)).double().mean().item()
        assert bool((diff <= _ulp(mag, dtype)).all()) and frac <= MAX_DIFF_FRACTION, ((diff / _ulp(mag, dtype)).max().item(), frac)
    # element by element against float64
    err = (W.reshape(shape[0], -1).double() - ideal).abs()
    assert bool((err <= bound).all()), (err / bound).max().item()
    # the convolution on top
    rel = ((y.float() - y_ref.float()).norm() / y_ref.float().norm()).item()
    assert rel <= 1e-3, rel


def _lowrank(pkg, conv, x, raw, out, n_patches=None):
    """ggufb200_dequant_lowrank of the layer's cached operands into `out` from the packed bytes `raw`."""
    ops, descs = conv._conv_patch_operands(x)
    shape = tuple(conv.weight.tensor_shape)
    N, K = shape[0], shape[1] * shape[2] * shape[3]
    rc = pkg.lib.lib().ggufb200_dequant_lowrank(int(conv.weight.tensor_type), raw.data_ptr(), N, K, out.data_ptr(),
                                                pkg.dequant.dtype_code(x.dtype), pkg.dequant.math_code(conv.dequant_dtype, x.dtype), descs,
                                                len(ops) if n_patches is None else n_patches, torch.cuda.current_stream().cuda_stream)
    pkg.lib.check(rc, "ggufb200_dequant_lowrank")
    return out


@pytest.mark.parametrize("qt,shape", [(Q.Q4_K, (640, 320, 3, 3)), (Q.Q8_0, (320, 320, 1, 1)), (Q.IQ2_XXS, (320, 320, 1, 1)),
                                      (Q.Q6_K, (332, 320, 3, 3))], ids=lambda v: v.name if hasattr(v, "name") else "x".join(map(str, v)))
def test_every_element_written_and_nothing_else(pkg, restated, kernel, qt, shape):
    """Output pre-filled with NaN (an unwritten element stays NaN) inside a sentinel-filled buffer; an unaligned packed view gives
    the same bits; zero patches give exactly K1's weight.  332 rows: a partial last row tile."""
    entries = _entries([("lora", 16, 1.0, 8.0), ("loha", (4, 2), -0.5, 2.0)], shape, seed=5)
    raw = _raw(qt, shape[0] * shape[1] * shape[2] * shape[3], seed=9)
    conv = _conv(pkg, qt, shape, entries, raw=raw)
    x = torch.randn(1, shape[1], 8, 8, device=DEV).to(torch.float16)
    numel = shape[0] * shape[1] * shape[2] * shape[3]
    buf = torch.full((numel + 64,), float("nan"), dtype=torch.float16, device=DEV)
    buf[numel:] = 1234.0
    out = _lowrank(pkg, conv, x, raw, buf[:numel])
    assert not bool(out.isnan().any()) and bool((buf[numel:] == 1234.0).all())
    W, _b, _y = _weight(conv, x, True)
    assert torch.equal(out.view(torch.int16), W.reshape(-1).view(torch.int16))
    shifted = torch.empty(raw.numel() + 1, dtype=torch.uint8, device=DEV)
    shifted[1:] = raw
    assert shifted[1:].data_ptr() % 16 == 1
    unaligned = _lowrank(pkg, conv, x, shifted[1:], torch.full((numel,), float("nan"), dtype=torch.float16, device=DEV))
    assert torch.equal(unaligned.view(torch.int16), out.view(torch.int16))
    plain = _lowrank(pkg, conv, x, raw, torch.full((numel,), float("nan"), dtype=torch.float16, device=DEV), n_patches=0)
    k1 = pkg.dequant.dequantize_tensor(conv.weight, torch.float16, None).reshape(-1)
    assert torch.equal(plain.view(torch.int16), k1.as_subclass(torch.Tensor).view(torch.int16))


def test_non_finite_weight_blocks(pkg, restated, kernel):
    """Q8_0 blocks with an Inf / NaN scale: NaN and Inf land where the two-step route puts them, the rest as in the main test."""
    shape = (320, 320, 1, 1)
    raw = _raw(Q.Q8_0, 320 * 320, seed=4).view(-1, 34)
    raw[3, 0:2] = torch.tensor([0x00, 0x7C], dtype=torch.uint8)            # d = +Inf
    raw[700, 0:2] = torch.tensor([0x00, 0x7E], dtype=torch.uint8)          # d = NaN
    raw[1601, 0:2] = torch.tensor([0x00, 0xFC], dtype=torch.uint8)         # d = -Inf
    entries = _entries([("lora", 16, 1.0, 8.0)], shape, seed=6)
    conv = _conv(pkg, Q.Q8_0, shape, entries, raw=raw.reshape(-1))
    x = torch.randn(1, 320, 8, 8, device=DEV).to(torch.float16)
    W, _b, _y = _weight(conv, x, True)
    W_ref, _b, _y = _weight(conv, x, False)
    assert bool(W_ref.isnan().any()) and bool(W_ref.isinf().any())
    assert torch.equal(W.isnan(), W_ref.isnan()) and torch.equal(W.isinf() & (W > 0), W_ref.isinf() & (W_ref > 0))
    fin = torch.isfinite(W_ref)
    _i, _b, mag, _e = _ideal(pkg, conv, torch.float16, entries)
    mag = mag.reshape(W.shape)
    assert bool(torch.isfinite(W[fin]).all()) and bool(((W[fin].double() - W_ref[fin].double()).abs() <= _ulp(mag[fin], torch.float16)).all())


def test_factor_modified_in_place_refreshes_the_operands(pkg, restated, kernel):
    shape = (320, 320, 1, 1)
    entries = _entries([("lora", 16, 1.0, 8.0)], shape, seed=8)
    conv = _conv(pkg, Q.Q4_0, shape, entries)
    x = torch.randn(1, 320, 8, 8, device=DEV).to(torch.float16)
    W1, _b, _y = _weight(conv, x, True)
    _payload(entries[0][1])[1][0].mul_(3.0)                                  # up, in place
    W2, _b, _y = _weight(conv, x, True)
    W_ref, _b, _y = _weight(conv, x, False)
    _i, _b, mag, _e = _ideal(pkg, conv, torch.float16, entries)
    assert not torch.equal(W1, W2) and bool(((W2 - W_ref).double().abs().reshape(mag.shape) <= _ulp(mag, torch.float16)).all())


def test_declined_lists_take_the_two_step_route_bit_for_bit(pkg, restated, calls):
    shape = (320, 320, 1, 1)
    base = _entries([("lora", 8, 1.0, 4.0)], shape, seed=11)
    strength, value, *_ = base[0]
    declined = [
        [(strength, value, 0.9, None, None)],                                # strength_model != 1
        [(strength, ("lora", _payload(value)[1][:5] + ((320, 320, 1, 1),)), 1.0, None, None)],      # reshape
        base * 9,                                                            # more than 8 patches
    ]
    for entries in declined:
        conv = _conv(pkg, Q.Q4_K, shape, entries)
        x = torch.randn(1, 320, 8, 8, device=DEV).to(torch.bfloat16)
        calls.clear()
        W, _b, y = _weight(conv, x, True)
        assert "ggufb200_dequant_lowrank" not in calls and "ggufb200_dequant" in calls
        W_ref, _b, y_ref = _weight(conv, x, False)
        assert torch.equal(W, W_ref) and torch.equal(y, y_ref)


def test_offloaded_weight_and_unpatched_route(pkg, restated, kernel, calls):
    """Packed bytes on the host are copied for the call; an unpatched conv keeps K1 + conv."""
    shape = (640, 320, 3, 3)
    entries = _entries([("lora", 16, 1.0, 8.0)], shape, seed=12)
    conv = _conv(pkg, Q.Q4_K, shape, entries)
    x = torch.randn(1, 320, 8, 8, device=DEV).to(torch.float16)
    W, _b, y = _weight(conv, x, True)
    host = _conv(pkg, Q.Q4_K, shape, entries, raw=conv.weight.as_subclass(torch.Tensor).cpu())
    calls.clear()
    W_host, _b, y_host = _weight(host, x, True)
    assert calls == ["ggufb200_dequant_lowrank"] and host.weight.device.type == "cpu"
    assert torch.equal(W_host, W) and torch.equal(y_host, y)
    plain = _conv(pkg, Q.Q4_K, shape, [])
    plain.weight.patches = []
    calls.clear()
    plain(x)
    assert calls == ["ggufb200_dequant"]


@pytest.mark.parametrize("shape,spec,in_kernel", [
    ((320, 320, 1, 1), [("lora", 16, 1.0, 8.0)], True),
    ((320, 320, 1, 1), [("lora", 128, 1.0, 64.0)], False),              # the rank loop costs more than cuBLAS's product here
    ((320, 320, 1, 1), [("loha", (32, 32), 1.0, 16.0)], True),          # LoHa's two-step route pays two products and a full-size one
    ((1280, 1280, 3, 3), [("lora", 64, 1.0, 32.0)], True),
    ((1280, 1280, 3, 3), [("lora", 256, 1.0, 64.0)], False),
], ids=["proj_in-r16", "proj_in-r128", "proj_in-loha32", "sdxl3x3-r64", "sdxl3x3-r256"])
def test_cost_model_picks_the_route(pkg, restated, calls, shape, spec, in_kernel):
    """By default the layer takes the kernel only where `lowrank_pays` expects it to win; elsewhere the two-step route, bit for bit."""
    entries = _entries(spec, shape, seed=21)
    conv = _conv(pkg, Q.Q4_K, shape, entries)
    x = torch.randn(1, shape[1], 8, 8, device=DEV).to(torch.float16)
    calls.clear()
    y = conv(x)
    assert calls == (["ggufb200_dequant_lowrank"] if in_kernel else ["ggufb200_dequant"]), calls
    conv.conv_patches_in_kernel = False
    y_ref = conv(x)
    if not in_kernel:
        assert torch.equal(y, y_ref)
