"""GPU tests of LoKr, LoCon `mid` and Tucker LoHa patches on a packed Conv2d weight (ggufb200_dequant_patched and
ggufb200_dequant_kron through GGMLOps.Conv2d).

The reference is the layer's own two-step route (`conv_patches_in_kernel = False`): dequantize_tensor, then calculate_weight,
here restated as ComfyUI's LoRA / LoHa / LoKr adapters compute it (every factor cast to fp32 on the weight's device):
    LoCon mid   down = mm(down.T.flatten(1), mid.T.flatten(1)).reshape(Cin, r, kh, kw).T;  diff = mm(up.flatten(1), down.flatten(1))
    LoHa        diff = m1 * m2, m = einsum('i j k l, j r, i p -> p r k l', t, wb, wa) with Tucker factors, else wa @ wb
    LoKr        diff = kron(w1 (or w1_a @ w1_b) [unsqueezed for a 4-D w2], w2 (or w2_a @ w2_b, or einsum(t2, w2_b, w2_a)));
                an exception of kron / reshape is logged and the entry skipped
    weight += ((strength * alpha) * diff.reshape(weight.shape)).type(weight.dtype)
LoKr lists are bit-identical to it (one fp32 product per element, the same rounding sequence).  Lists with rank sums differ from
it only in the order of the fp32 sums: bit-identical but for at most 1 % of elements, each within one activation-dtype ulp at
the element's magnitude |W0| + sum |s d|, and every element within a float64 bound."""
import gguf
import pytest
import torch

import oracle
from fallback_cases import random_blocks as fallback_blocks
from util import Q

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FALLBACK = (Q.IQ2_XXS, Q.MXFP4)
MAX_DIFF_FRACTION = 0.01


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


class LoKrAdapter(LoRAAdapter):
    pass


def _payload(v):
    return (v[0], tuple(v[1])) if isinstance(v, tuple) else (type(v).__name__[:4].lower(), tuple(v.weights))


def ref_diff(kind, v, shape, dev, dtype=torch.float32):
    """(alpha, diff [shape] or None when the reference skips the entry) of one payload, as ComfyUI's adapters form it (factors
    cast to `dtype`: the reference's fp32, or float64 for the ideal)."""
    def _f32(t, dev):
        return None if t is None else t.to(device=dev, dtype=dtype)
    if kind == "lora":
        up, down, alpha, mid = _f32(v[0], dev), _f32(v[1], dev), v[2], _f32(v[3] if len(v) > 3 else None, dev)
        alpha = 1.0 if alpha is None else alpha / down.shape[0]
        if mid is not None:
            final_shape = [down.shape[1], down.shape[0], mid.shape[2], mid.shape[3]]
            down = torch.mm(down.transpose(0, 1).flatten(start_dim=1), mid.transpose(0, 1).flatten(start_dim=1)).reshape(final_shape).transpose(0, 1)
        return alpha, torch.mm(up.flatten(start_dim=1), down.flatten(start_dim=1)).reshape(shape)
    if kind == "loha":
        w1a, w1b, alpha, w2a, w2b = _f32(v[0], dev), _f32(v[1], dev), v[2], _f32(v[3], dev), _f32(v[4], dev)
        t1, t2 = (_f32(v[5], dev), _f32(v[6], dev)) if len(v) > 6 else (None, None)
        alpha = 1.0 if alpha is None else alpha / w1b.shape[0]
        if t1 is not None:
            m1 = torch.einsum("i j k l, j r, i p -> p r k l", t1, w1b, w1a)
            m2 = torch.einsum("i j k l, j r, i p -> p r k l", t2, w2b, w2a)
        else:
            m1, m2 = torch.mm(w1a, w1b), torch.mm(w2a, w2b)
        return alpha, (m1 * m2).reshape(shape)
    w1, w2, alpha, w1_a, w1_b, w2_a, w2_b, t2 = (_f32(t, dev) if torch.is_tensor(t) else t for t in (v + (None,) * 2)[:8])
    dim = None
    if w1 is None:
        dim = w1_b.shape[0]
        w1 = torch.mm(w1_a, w1_b)
    if w2 is None:
        dim = w2_b.shape[0]
        w2 = torch.mm(w2_a, w2_b) if t2 is None else torch.einsum("i j k l, j r, i p -> p r k l", t2, w2_b, w2_a)
    if w2.dim() == 4:
        w1 = w1.unsqueeze(2).unsqueeze(2)
    alpha = alpha / dim if (alpha is not None and dim is not None) else 1.0
    try:
        return alpha, torch.kron(w1, w2).reshape(shape)
    except RuntimeError:
        return alpha, None


@pytest.fixture
def restated(pkg, monkeypatch):
    """calculate_weight with ComfyUI's LoRA, LoHa and LoKr arithmetic (whole-weight entries without hooks)."""
    original = pkg.ops.comfy_lora.calculate_weight

    def calculate_weight(patches, weight, key, intermediate_dtype=torch.float32, original_weights=None):
        if not all(_payload(p[1])[0] in ("lora", "loha", "lokr") and (len(p) < 4 or p[3] is None) for p in patches):
            return original(patches, weight, key, intermediate_dtype, original_weights)
        for p in patches:
            strength, (kind, v), strength_model = p[0], _payload(p[1]), p[2]
            if strength_model != 1.0:
                weight *= strength_model
            alpha, diff = ref_diff(kind, v, weight.shape, weight.device, intermediate_dtype)
            if diff is not None:
                weight += ((strength * alpha) * diff).type(weight.dtype)
        return weight
    monkeypatch.setattr(pkg.ops.comfy_lora, "calculate_weight", calculate_weight)


@pytest.fixture
def kernel(pkg, monkeypatch):
    """The layer takes the kernels wherever it can, whatever its cost model says."""
    monkeypatch.setattr(pkg.ops, "lowrank_pays", lambda N, K, terms: True)


@pytest.fixture
def calls(pkg, monkeypatch):
    L = pkg.lib.lib()
    seen = []
    for name in ("ggufb200_dequant_patched", "ggufb200_dequant_lowrank", "ggufb200_dequant", "ggufb200_dequant_fallback",
                 "ggufb200_dequant_kron"):
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


def _entry(spec, shape, g, i):
    """One patch entry of (kind, form / rank, strength, alpha) for a conv weight of `shape`."""
    kind, form, strength, alpha = spec
    cout, cin, kh, kw = shape

    def f(*s):
        return (torch.randn(*s, generator=g) * 0.1).to(DEV)
    if kind == "lokr":
        fac, how = form
        b1, c2 = cout // fac, cin // fac
        w1 = f(fac, fac)
        payload = {"full4d": (w1, f(b1, c2, kh, kw), alpha, None, None, None, None, None, None),
                   "full2d": (w1, f(b1, c2 * kh * kw), alpha, None, None, None, None, None, None),
                   "decomposed": (w1, None, alpha, None, None, f(b1, 16), f(16, c2 * kh * kw), None, None),
                   "tucker": (w1, None, alpha, None, None, f(8, b1), f(8, c2), f(8, 8, kh, kw), None),
                   "w1dec": (None, f(b1, c2, kh, kw), alpha, f(fac, 2), f(2, fac), None, None, None, None)}[how]
        cls = LoKrAdapter
    elif kind == "lora":
        payload, cls = (f(cout, form, 1, 1), f(form, cin, kh, kw), alpha, None, None, None), LoRAAdapter
    elif kind == "locon_mid":
        payload, cls, kind = (f(cout, form, 1, 1), f(form, cin, 1, 1), alpha, f(form, form, kh, kw), None, None), LoRAAdapter, "lora"
    elif kind == "loha":
        payload, cls = (f(cout, form), f(form, cin * kh * kw), alpha, f(cout, form), f(form, cin * kh * kw), None, None, None), LoHaAdapter
    else:
        payload = (f(form, cout), f(form, cin), alpha, f(form, cout), f(form, cin), f(form, form, kh, kw), f(form, form, kh, kw), None)
        cls, kind = LoHaAdapter, "loha"
    return (strength, (kind, payload) if i % 2 == 0 else cls(payload), 1.0, None, None)


def _entries(spec, shape, seed):
    g = torch.Generator().manual_seed(seed)
    return [_entry(s, shape, g, i) for i, s in enumerate(spec)]


def _conv(pkg, qt, shape, entries, seed=0, raw=None):
    cout, cin, kh, kw = shape
    conv = pkg.ops.GGMLOps.Conv2d(cin, cout, (kh, kw), padding=kh // 2, device="meta")
    raw = _raw(qt, cout * cin * kh * kw, seed) if raw is None else raw
    w = pkg.ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size(shape), patches=[(entries, "diffusion_model.conv.weight")])
    bias = (torch.randn(cout, generator=torch.Generator().manual_seed(seed + 7)) * 0.05).to(DEV)
    conv.load_state_dict({"weight": w, "bias": bias}, assign=True)
    return conv


def _x(*shape):
    """A seeded activation: these tests leave the global random state to the tests that run after them."""
    return torch.randn(*shape, generator=torch.Generator().manual_seed(sum(shape))).to(DEV)


def _weight(conv, x, in_kernel):
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


def _patched(pkg, conv, x, raw, out, n=None):
    """ggufb200_dequant_patched of the layer's terms (`conv_lycoris_operands`) into `out` from the packed bytes `raw`."""
    terms = pkg.ops.conv_lycoris_terms(pkg.ops._patch_entries(conv.weight))
    _keep, descs = pkg.ops.conv_lycoris_operands(terms, DEV)
    shape = tuple(conv.weight.tensor_shape)
    rc = pkg.lib.lib().ggufb200_dequant_patched(int(conv.weight.tensor_type), raw.data_ptr(), shape[0], out.numel() // shape[0],
                                                out.data_ptr(), pkg.dequant.dtype_code(x.dtype),
                                                pkg.dequant.math_code(conv.dequant_dtype, x.dtype), descs, len(terms) if n is None else n,
                                                torch.cuda.current_stream().cuda_stream)
    pkg.lib.check(rc, "ggufb200_dequant_patched")
    return out


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _ideal(pkg, conv, dtype, entries):
    """(float64 patched weight, per-element bound, magnitude) from the act-dtype dequantised weight and the factors."""
    W0 = pkg.dequant.dequantize_tensor(conv.weight, dtype, conv.dequant_dtype)
    W0 = W0.as_subclass(torch.Tensor).double().reshape(W0.shape[0], -1)
    shape = tuple(conv.weight.tensor_shape)
    ideal, mag, fp32_err = W0.clone(), W0.abs(), torch.zeros_like(W0)
    for strength, value, *_ in entries:
        kind, v = _payload(value)
        alpha, d = ref_diff(kind, v, shape, DEV, torch.float64)
        if d is None:
            continue
        vabs = tuple(t.abs() if torch.is_tensor(t) else t for t in v)
        m = ref_diff(kind, vabs, shape, DEV, torch.float64)[1].reshape(ideal.shape)
        terms = sum(t.shape[0] for t in v if torch.is_tensor(t)) + 4        # a generous count of fp32 roundings per element
        s = strength * alpha
        ideal += s * d.reshape(ideal.shape)
        mag += abs(s) * m
        fp32_err += abs(s) * terms * 2.0 ** -23 * m
    n = len(entries)
    u, tiny = {torch.float16: (2.0 ** -11, 2.0 ** -24), torch.bfloat16: (2.0 ** -8, 2.0 ** -133), torch.float32: (2.0 ** -24, 2.0 ** -149)}[dtype]
    return ideal, 2 * n * (u * mag + tiny) + fp32_err, mag


def _ulp(mag, dtype):
    bits, emin = {torch.float16: (10, -14), torch.bfloat16: (7, -126), torch.float32: (23, -126)}[dtype]
    e = torch.floor(torch.log2(mag.clamp_min(2.0 ** emin))).clamp_min(emin)
    return torch.exp2(e - bits)


# ---------------------------------------------------------------- LoKr only: bit for bit
# (format, conv shape, LoKr specs, activation dtype, dequant_dtype).  K = 2880 is straddled for the 256-element formats.
LOKR_CASES = [
    (Q.Q4_0, (320, 320, 1, 1), [("lokr", (4, "full4d"), 1.0, None)], torch.float16, None),
    (Q.Q8_0, (640, 320, 3, 3), [("lokr", (8, "decomposed"), 1.0, 8.0)], torch.bfloat16, None),
    (Q.Q4_K, (640, 320, 3, 3), [("lokr", (16, "full4d"), 0.8, None)], torch.float16, None),
    (Q.Q6_K, (640, 320, 3, 3), [("lokr", (4, "tucker"), 1.0, 4.0)], torch.bfloat16, None),
    (Q.Q4_K, (1280, 1280, 3, 3), [("lokr", (8, "full2d"), 1.0, None)], torch.float32, None),
    (Q.Q6_K, (640, 640, 1, 1), [("lokr", (4, "w1dec"), -1.0, 2.0), ("lokr", (8, "decomposed"), 0.5, 16.0)], torch.float16, "target"),
    (Q.Q8_0, (320, 320, 3, 3), [("lokr", (8, "full4d"), 1.0, None)], torch.bfloat16, "target"),
    (Q.IQ2_XXS, (640, 320, 3, 3), [("lokr", (8, "full4d"), 1.0, None)], torch.float16, None),
    (Q.MXFP4, (320, 320, 1, 1), [("lokr", (4, "decomposed"), 1.0, 8.0), ("lokr", (16, "full4d"), -0.5, None)], torch.float32, None),
]


def _case_id(c):
    qt, shape, spec, dtype, math = c
    kinds = "+".join(f"{k}{r if isinstance(r, int) else '-'.join(map(str, r))}" for k, r, *_ in spec)
    return f"{qt.name}-{'x'.join(map(str, shape))}-{kinds}-{str(dtype)[6:]}" + (f"-{math}" if math else "")


@pytest.mark.parametrize("case", LOKR_CASES, ids=_case_id)
def test_lokr_lists_are_bit_identical(pkg, restated, kernel, calls, case):
    qt, shape, spec, dtype, math = case
    entries = _entries(spec, shape, seed=shape[0] + int(qt))
    conv = _conv(pkg, qt, shape, entries, seed=int(qt))
    conv.dequant_dtype = math
    x = (torch.randn(2, shape[1], 8, 8, generator=torch.Generator().manual_seed(3)) * 0.5).to(DEV).to(dtype)
    W_ref, b_ref, y_ref = _weight(conv, x, False)
    skipped = any(ref_diff(*_payload(e[1]), shape, DEV)[1] is None for e in entries)
    calls.clear()
    W, b, y = _weight(conv, x, True)
    if skipped:                          # the reference skips the entry (its torch.kron raises): the layer keeps the two-step route
        assert "ggufb200_dequant" in calls or "ggufb200_dequant_fallback" in calls, calls
        assert torch.equal(_bits(W), _bits(W_ref)) and torch.equal(y, y_ref)
        return
    assert calls == ["ggufb200_dequant_patched"], calls
    assert W.dtype == dtype and tuple(W.shape) == shape and torch.equal(b, b_ref)
    assert torch.equal(_bits(W), _bits(W_ref))
    assert torch.equal(y, y_ref)
    if qt not in FALLBACK:               # K1 with the Kronecker patch gives the same bits
        _keep, descs = pkg.ops.conv_lycoris_operands(pkg.ops.conv_lycoris_terms(entries), DEV)
        kron = (pkg.lib.KronPatch * len(entries))(*[d.kron for d in descs[:len(entries)]])
        out = torch.full((W.numel(),), float("nan"), dtype=dtype, device=DEV)
        rc = pkg.lib.lib().ggufb200_dequant_kron(int(qt), conv.weight.as_subclass(torch.Tensor).data_ptr(), shape[0], W.numel() // shape[0],
                                                 out.data_ptr(), pkg.dequant.dtype_code(dtype), pkg.dequant.math_code(math, dtype), kron,
                                                 len(entries), torch.cuda.current_stream().cuda_stream)
        pkg.lib.check(rc, "ggufb200_dequant_kron")
        assert torch.equal(_bits(out), _bits(W_ref.reshape(-1)))


# ---------------------------------------------------------------- mixed lists: the conv budget
MIXED_CASES = [
    (Q.Q4_K, (640, 320, 3, 3), [("lokr", (8, "full4d"), 1.0, None), ("lora", 32, 1.0, 16.0)], torch.float16, None),
    (Q.Q8_0, (320, 320, 1, 1), [("lora", 16, 1.0, 8.0), ("lokr", (4, "decomposed"), 0.5, 8.0), ("loha", 8, -1.0, 4.0)], torch.bfloat16, None),
    (Q.Q6_K, (640, 320, 3, 3), [("locon_mid", 16, 1.0, 8.0)], torch.float16, None),
    (Q.Q4_0, (640, 640, 3, 3), [("locon_mid", 32, 0.7, 16.0), ("lokr", (16, "full2d"), 1.0, None)], torch.bfloat16, "target"),
    (Q.Q4_K, (1280, 1280, 3, 3), [("loha_tucker", 8, 1.0, 4.0)], torch.float16, None),
    (Q.IQ2_XXS, (640, 320, 3, 3), [("loha_tucker", 16, 1.0, 8.0), ("lora", 8, 1.0, 4.0)], torch.float16, None),
    (Q.Q6_K, (320, 320, 3, 3), [("loha_tucker", 4, -0.5, 2.0), ("lokr", (4, "w1dec"), 1.0, 2.0), ("locon_mid", 8, 1.0, None)],
     torch.float32, None),
]


@pytest.mark.parametrize("case", MIXED_CASES, ids=_case_id)
def test_mixed_lists_stay_within_the_conv_budget(pkg, restated, kernel, calls, case):
    qt, shape, spec, dtype, math = case
    entries = _entries(spec, shape, seed=shape[1] + int(qt))
    conv = _conv(pkg, qt, shape, entries, seed=int(qt) + 1)
    conv.dequant_dtype = math
    x = (torch.randn(2, shape[1], 8, 8, generator=torch.Generator().manual_seed(4)) * 0.5).to(DEV).to(dtype)
    calls.clear()
    W, b, y = _weight(conv, x, True)
    assert calls == ["ggufb200_dequant_patched"], calls
    W_ref, b_ref, y_ref = _weight(conv, x, False)
    assert torch.equal(b, b_ref) and bool(torch.isfinite(W).all())
    ideal, bound, mag = _ideal(pkg, conv, dtype, entries)
    W2, R2 = W.reshape(shape[0], -1).double(), W_ref.reshape(shape[0], -1).double()
    diff = (W2 - R2).abs()
    if dtype == torch.float32:
        assert bool((diff <= _ulp(mag, dtype) + 2 * (bound - 2 * len(entries) * 2.0 ** -24 * mag)).all())
    else:
        frac = (_bits(W) != _bits(W_ref)).double().mean().item()
        assert bool((diff <= _ulp(mag, dtype)).all()) and frac <= MAX_DIFF_FRACTION, ((diff / _ulp(mag, dtype)).max().item(), frac)
    err = (W2 - ideal).abs()
    assert bool((err <= bound).all()), (err / bound).max().item()
    rel = ((y.float() - y_ref.float()).norm() / y_ref.float().norm()).item()
    assert rel <= 1e-3, rel


def test_lowrank_descriptors_match_dequant_lowrank(pkg, kernel):
    """ggufb200_dequant_patched with LOWRANK descriptors only = ggufb200_dequant_lowrank, bit for bit."""
    shape = (640, 320, 3, 3)
    for qt, dtype in ((Q.Q4_K, torch.float16), (Q.MXFP4, torch.bfloat16), (Q.Q8_0, torch.float32)):
        entries = _entries([("lora", 32, 1.0, 16.0), ("loha", 8, -0.5, 4.0)], shape, seed=13)
        conv = _conv(pkg, qt, shape, entries)
        x = _x(1, 320, 8, 8).to(dtype)
        ops, descs = conv._conv_patch_operands(x)
        L = pkg.lib
        wp = (L.WeightPatch * len(ops))(*[L.WeightPatch(L.PATCH_LOWRANK, descs[i], L.KronPatch()) for i in range(len(ops))])
        raw = conv.weight.as_subclass(torch.Tensor)
        N, K = shape[0], shape[1] * 9
        outs = []
        for fn, d in (("ggufb200_dequant_lowrank", descs), ("ggufb200_dequant_patched", wp)):
            out = torch.full((N * K,), float("nan"), dtype=dtype, device=DEV)
            rc = getattr(L.lib(), fn)(int(qt), raw.data_ptr(), N, K, out.data_ptr(), pkg.dequant.dtype_code(dtype),
                                      pkg.dequant.math_code(None, dtype), d, len(ops), torch.cuda.current_stream().cuda_stream)
            L.check(rc, fn)
            outs.append(out)
        assert not bool(outs[0].isnan().any()) and torch.equal(_bits(outs[0]), _bits(outs[1]))


@pytest.mark.parametrize("qt,shape", [(Q.Q4_K, (332, 320, 3, 3)), (Q.Q8_0, (320, 320, 1, 1)), (Q.IQ2_XXS, (640, 320, 3, 3))],
                         ids=lambda v: v.name if hasattr(v, "name") else "x".join(map(str, v)))
def test_every_element_written_and_nothing_else(pkg, restated, kernel, qt, shape):
    """NaN-poisoned output inside a sentinel-filled buffer; an unaligned packed view gives the same bits.  332 rows: a partial
    last row tile (and a LoKr factor of 4: b1 = 83)."""
    entries = _entries([("lokr", (4, "full4d"), 1.0, None), ("lora", 16, 1.0, 8.0), ("lokr", (4, "decomposed"), -0.5, 4.0)], shape, seed=5)
    raw = _raw(qt, shape[0] * shape[1] * shape[2] * shape[3], seed=9)
    conv = _conv(pkg, qt, shape, entries, raw=raw)
    x = _x(1, shape[1], 8, 8).to(torch.float16)
    numel = shape[0] * shape[1] * shape[2] * shape[3]
    buf = torch.full((numel + 64,), float("nan"), dtype=torch.float16, device=DEV)
    buf[numel:] = 1234.0
    out = _patched(pkg, conv, x, raw, buf[:numel])
    assert not bool(out.isnan().any()) and bool((buf[numel:] == 1234.0).all())
    W, _b, _y = _weight(conv, x, True)
    assert torch.equal(_bits(out), _bits(W.reshape(-1)))
    shifted = torch.empty(raw.numel() + 1, dtype=torch.uint8, device=DEV)
    shifted[1:] = raw
    assert shifted[1:].data_ptr() % 16 == 1
    unaligned = _patched(pkg, conv, x, shifted[1:], torch.full((numel,), float("nan"), dtype=torch.float16, device=DEV))
    assert torch.equal(_bits(unaligned), _bits(out))
    plain = _patched(pkg, conv, x, raw, torch.full((numel,), float("nan"), dtype=torch.float16, device=DEV), n=0)
    k1 = pkg.dequant.dequantize_tensor(conv.weight, torch.float16, None).reshape(-1)
    assert torch.equal(_bits(plain), _bits(k1.as_subclass(torch.Tensor)))


def test_offloaded_weight_and_cache_refresh(pkg, restated, kernel, calls):
    shape = (640, 320, 3, 3)
    for spec in ([("lokr", (8, "decomposed"), 1.0, 8.0)], [("lokr", (8, "full4d"), 1.0, None), ("locon_mid", 8, 1.0, 4.0)]):
        entries = _entries(spec, shape, seed=12)
        conv = _conv(pkg, Q.Q4_K, shape, entries)
        x = _x(1, 320, 8, 8).to(torch.float16)
        W, _b, y = _weight(conv, x, True)
        host = _conv(pkg, Q.Q4_K, shape, entries, raw=conv.weight.as_subclass(torch.Tensor).cpu())
        calls.clear()
        W_host, _b, y_host = _weight(host, x, True)
        assert calls == ["ggufb200_dequant_patched"] and host.weight.device.type == "cpu"
        assert torch.equal(W_host, W) and torch.equal(y_host, y)
        # a factor edited in place: the cached operands are rebuilt
        lokr = _payload(entries[0][1])[1]
        (lokr[0] if lokr[0] is not None else lokr[3]).mul_(3.0)
        W2, _b, _y = _weight(conv, x, True)
        W_ref, _b, _y = _weight(conv, x, False)
        assert not torch.equal(W, W2)
        if len(spec) == 1:
            assert torch.equal(W2, W_ref)
        else:
            _i, _bd, mag = _ideal(pkg, conv, torch.float16, entries)
            assert bool(((W2 - W_ref).double().abs().reshape(mag.shape) <= _ulp(mag, torch.float16)).all())


def test_class_switch_and_declined_lists_take_the_two_step_route_bit_for_bit(pkg, restated, calls):
    shape = (64, 32, 3, 3)
    g = torch.Generator().manual_seed(31)
    lokr = _entry(("lokr", (4, "full4d"), 1.0, None), shape, g, 0)
    misfit = _entry(("lokr", (4, "full4d"), 1.0, None), (32, 64, 3, 3), g, 0)            # kron [32, 64, 3, 3] on a [64, 32, 3, 3] weight
    declined = [
        [(lokr[0], lokr[1], 0.5, None, None)],                                           # strength_model != 1
        [lokr] * 9,                                                                      # more than 8 entries
        [misfit],                                                                        # a1 b1 != Cout: the reshape mixes rows
    ]
    x = _x(1, 32, 8, 8).to(torch.bfloat16)
    for entries in declined:
        conv = _conv(pkg, Q.Q4_K, shape, entries)
        calls.clear()
        W, _b, y = _weight(conv, x, True)
        assert calls == ["ggufb200_dequant"], calls
        W_ref, _b, y_ref = _weight(conv, x, False)
        assert torch.equal(W, W_ref) and torch.equal(y, y_ref)
    conv = _conv(pkg, Q.Q4_K, shape, [lokr])
    calls.clear()
    _weight(conv, x, False)
    assert calls == ["ggufb200_dequant"]                                                 # the class switch
    calls.clear()
    _weight(conv, x, True)
    assert calls == ["ggufb200_dequant_patched"]
