"""GPU tests of DoRA (weight-decomposed LoRA) patches on a packed Conv2d weight (ggufb200_dequant_patched_dora through
GGMLOps.Conv2d).

The reference is the layer's own two-step route (`conv_patches_in_kernel = False`): dequantize_tensor, then calculate_weight with
ComfyUI's LoRA / LoHa / LoKr adapters and weight_decompose restated (every factor cast to fp32 on the weight's device):
    diff as in tests/test_gpu_conv_lycoris.py
    plain   weight += ((strength * alpha) * diff).type(weight.dtype)
    DoRA    diff *= alpha;  Wc = weight + diff.type(weight.dtype);  norm = per output channel of weight, or per input channel of Wc
            Wc *= (dora_scale / (norm + eps)).type(weight.dtype);   weight = Wc, or weight += strength * (Wc - weight)
The layer replays the factors s once per patch set and the kernel applies the same per-element rounding sequence, so LoKr lists
(one fp32 product per element) are bit-identical to it, and lists with rank sums differ only through the order of the fp32 sums:
at most 1 % of elements, each by at most one activation-dtype ulp at the element's magnitude (fp32 output: within the rank sums'
own rounding).  DoRA magnitudes are the weight's own channel norms times U(0.8, 1.2), as trainers initialise them."""
import gguf
import pytest
import torch

import oracle
from fallback_cases import random_blocks as fallback_blocks
from test_gpu_conv_lycoris import LoHaAdapter, LoKrAdapter, LoRAAdapter, _payload, ref_diff
from util import Q

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FALLBACK = (Q.IQ2_XXS, Q.MXFP4)
MAX_DIFF_FRACTION = 0.01
DORA_AT = {"lora": 4, "loha": 7, "lokr": 8}


def weight_decompose(dora_scale, weight, lora_diff, alpha, strength):
    """ComfyUI's weight_decompose (comfy/weight_adapter/base.py), restated."""
    dora_scale = dora_scale.to(device=weight.device, dtype=torch.float32)
    lora_diff *= alpha
    weight_calc = weight + lora_diff.type(weight.dtype)
    if dora_scale.shape[0] == weight_calc.shape[0]:
        weight_norm = weight.reshape(weight.shape[0], -1).norm(dim=1, keepdim=True).reshape(weight.shape[0], *[1] * (weight.dim() - 1))
    else:
        weight_norm = (weight_calc.transpose(0, 1).reshape(weight_calc.shape[1], -1).norm(dim=1, keepdim=True)
                       .reshape(weight_calc.shape[1], *[1] * (weight_calc.dim() - 1)).transpose(0, 1))
    weight_norm = weight_norm + torch.finfo(weight.dtype).eps
    weight_calc *= (dora_scale / weight_norm).type(weight.dtype)
    if strength != 1.0:
        weight_calc -= weight
        weight += strength * weight_calc
    else:
        weight[:] = weight_calc
    return weight


@pytest.fixture
def restated(pkg, monkeypatch):
    """calculate_weight with ComfyUI's LoRA, LoHa and LoKr arithmetic and weight_decompose (whole-weight entries, no hooks)."""
    original = pkg.ops.comfy_lora.calculate_weight

    def calculate_weight(patches, weight, key, intermediate_dtype=torch.float32, original_weights=None):
        if not all(_payload(p[1])[0] in DORA_AT and (len(p) < 4 or p[3] is None) for p in patches):
            return original(patches, weight, key, intermediate_dtype, original_weights)
        for p in patches:
            strength, (kind, v), strength_model = p[0], _payload(p[1]), p[2]
            if strength_model != 1.0:
                weight *= strength_model
            alpha, diff = ref_diff(kind, v, weight.shape, weight.device, intermediate_dtype)
            if diff is None:
                continue
            ds = v[DORA_AT[kind]] if len(v) > DORA_AT[kind] else None
            if ds is not None:
                weight = weight_decompose(ds, weight, diff, alpha, strength)
            else:
                weight += ((strength * alpha) * diff).type(weight.dtype)
        return weight
    monkeypatch.setattr(pkg.ops.comfy_lora, "calculate_weight", calculate_weight)


@pytest.fixture
def kernel(pkg, monkeypatch):
    """The layer takes the kernel wherever it can, whatever its cost model says."""
    monkeypatch.setattr(pkg.ops, "conv_dora_pays", lambda N, K, terms: True)


@pytest.fixture
def calls(pkg, monkeypatch):
    L = pkg.lib.lib()
    seen = []
    for name in ("ggufb200_dequant_patched_dora", "ggufb200_dequant_patched", "ggufb200_dequant_lowrank", "ggufb200_dequant",
                 "ggufb200_dequant_fallback", "ggufb200_dequant_kron"):
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


def _conv(pkg, qt, shape, seed=0, raw=None):
    cout, cin, kh, kw = shape
    conv = pkg.ops.GGMLOps.Conv2d(cin, cout, (kh, kw), padding=kh // 2, device="meta")
    raw = _raw(qt, cout * cin * kh * kw, seed) if raw is None else raw
    w = pkg.ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size(shape), patches=[([], "diffusion_model.conv.weight")])
    bias = (torch.randn(cout, generator=torch.Generator().manual_seed(seed + 7)) * 0.05).to(DEV)
    conv.load_state_dict({"weight": w, "bias": bias}, assign=True)
    return conv


def _norms(pkg, conv, axis):
    """The dequantised weight's output- (axis 0) or input-channel (axis 1) norms, in the dora_scale shape of that axis."""
    W = pkg.dequant.dequantize_tensor(conv.weight, torch.float32).as_subclass(torch.Tensor)
    if axis == 0:
        return W.reshape(W.shape[0], -1).norm(dim=1).reshape(-1, 1, 1, 1)
    return W.transpose(0, 1).reshape(W.shape[1], -1).norm(dim=1).reshape(1, -1, 1, 1)


def _entry(pkg, conv, spec, g, i):
    """One patch entry of (kind, form / rank, strength, alpha, DoRA axis or None) for the layer's weight."""
    kind, form, strength, alpha, axis = spec
    cout, cin, kh, kw = tuple(conv.weight.tensor_shape)

    def f(*s):
        return (torch.randn(*s, generator=g) * 0.1).to(DEV)
    ds = None
    if axis is not None:
        ds = _norms(pkg, conv, axis) * (0.8 + 0.4 * torch.rand(*((cout, 1, 1, 1) if axis == 0 else (1, cin, 1, 1)), generator=g).to(DEV))
    if kind == "lokr":
        fac, how = form
        b1, c2 = cout // fac, cin // fac
        w1 = f(fac, fac) * 10
        payload = {"full4d": (w1, f(b1, c2, kh, kw), alpha, None, None, None, None, None, ds),
                   "decomposed": (w1, None, alpha, None, None, f(b1, 16), f(16, c2 * kh * kw), None, ds)}[how]
        cls = LoKrAdapter
    elif kind == "lora":
        payload, cls = (f(cout, form, 1, 1), f(form, cin, kh, kw), alpha, None, ds, None), LoRAAdapter
    elif kind == "locon_mid":
        payload, cls, kind = (f(cout, form, 1, 1), f(form, cin, 1, 1), alpha, f(form, form, kh, kw), ds, None), LoRAAdapter, "lora"
    elif kind == "loha":
        payload, cls = (f(cout, form), f(form, cin * kh * kw), alpha, f(cout, form), f(form, cin * kh * kw), None, None, ds), LoHaAdapter
    else:                                                            # Tucker LoHa
        payload = (f(form, cout), f(form, cin), alpha, f(form, cout), f(form, cin), f(form, form, kh, kw), f(form, form, kh, kw), ds)
        cls, kind = LoHaAdapter, "loha"
    return (strength, (kind, payload) if i % 2 == 0 else cls(payload), 1.0, None, None)


def _patch(pkg, conv, spec, seed):
    g = torch.Generator().manual_seed(seed)
    entries = [_entry(pkg, conv, s, g, i) for i, s in enumerate(spec)]
    conv.weight.patches = [(entries, "diffusion_model.conv.weight")]
    return entries


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


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _ulp(mag, dtype):
    bits, emin = {torch.float16: (10, -14), torch.bfloat16: (7, -126), torch.float32: (23, -126)}[dtype]
    e = torch.floor(torch.log2(mag.clamp_min(2.0 ** emin))).clamp_min(emin)
    return torch.exp2(e - bits)


def _magnitude(pkg, conv, dtype, entries, W_ref):
    """(magnitude, fp32 rank-sum error bound) per element of the patched weight: |W0| + |alpha d| through each entry, scaled by
    |s| for a DoRA entry (s read off the reference weight's chain in float64), and the fp32 rounding of the rank sums carried
    along the same way."""
    W0 = pkg.dequant.dequantize_tensor(conv.weight, dtype, conv.dequant_dtype).as_subclass(torch.Tensor).double()
    shape = W0.shape
    W, mag, err = W0.clone(), W0.abs(), torch.zeros_like(W0)
    eps = torch.finfo(dtype).eps
    for strength, value, *_ in entries:
        kind, v = _payload(value)
        alpha, d = ref_diff(kind, v, shape, DEV, torch.float64)
        vabs = tuple(t.abs() if torch.is_tensor(t) else t for t in v)
        m = ref_diff(kind, vabs, shape, DEV, torch.float64)[1]
        at = DORA_AT[kind]
        ranks = sum(t.shape[0] for j, t in enumerate(v) if torch.is_tensor(t) and j != at) + 4
        ds = v[at] if len(v) > at else None
        if ds is None:
            W, mag, err = W + strength * alpha * d, mag + abs(strength * alpha) * m, err + abs(strength * alpha) * ranks * 2.0 ** -23 * m
            continue
        Wc = W + alpha * d
        if ds.shape[0] == shape[0]:
            s = ds.double() / (W.reshape(shape[0], -1).norm(dim=1).reshape(-1, 1, 1, 1) + eps)
        else:
            s = ds.double() / (Wc.transpose(0, 1).reshape(shape[1], -1).norm(dim=1).reshape(1, -1, 1, 1) + eps)
        s = s.abs()
        mag_c, err_c = (mag + abs(alpha) * m) * s, (err + abs(alpha) * ranks * 2.0 ** -23 * m) * s
        W = W + strength * (Wc * s - W) if strength != 1.0 else Wc * s
        mag, err = (mag_c, err_c) if strength == 1.0 else (mag + abs(strength) * (mag_c + mag), err + abs(strength) * (err_c + err))
    return mag.reshape(W_ref.shape), err.reshape(W_ref.shape)


def _check_budget(pkg, conv, dtype, entries, W, W_ref):
    mag, err = _magnitude(pkg, conv, dtype, entries, W_ref)
    diff = (W.double() - W_ref.double()).abs()
    if dtype == torch.float32:
        assert bool((diff <= 2 * _ulp(mag, dtype) + 2 * err).all()), (diff / (_ulp(mag, dtype) + err)).max().item()
    else:
        frac = (_bits(W) != _bits(W_ref)).double().mean().item()
        assert bool((diff <= _ulp(mag, dtype)).all()) and frac <= MAX_DIFF_FRACTION, ((diff / _ulp(mag, dtype)).max().item(), frac)


def _case_id(c):
    qt, shape, spec, dtype = c
    kinds = "+".join(f"{k}{r if isinstance(r, int) else r[0]}" + ("" if ax is None else f"-{'out' if ax == 0 else 'in'}{st}")
                     for k, r, st, _a, ax in spec)
    return f"{qt.name}-{'x'.join(map(str, shape))}-{kinds}-{str(dtype)[6:]}"


# ---------------------------------------------------------------- DoRA LoKr only: bit for bit
LOKR_CASES = [
    (Q.Q4_K, (640, 320, 3, 3), [("lokr", (8, "full4d"), 1.0, None, 0)], torch.float16),
    (Q.Q8_0, (320, 320, 1, 1), [("lokr", (4, "decomposed"), 0.8, 8.0, 1)], torch.bfloat16),
    (Q.Q6_K, (640, 320, 3, 3), [("lokr", (8, "full4d"), 1.0, None, 1)], torch.float32),
    (Q.IQ2_XXS, (640, 320, 3, 3), [("lokr", (4, "full4d"), 0.8, None, 0), ("lokr", (8, "decomposed"), 1.0, 4.0, 1)], torch.float16),
]


@pytest.mark.parametrize("case", LOKR_CASES, ids=_case_id)
def test_dora_lokr_lists_are_bit_identical(pkg, restated, kernel, calls, case):
    qt, shape, spec, dtype = case
    conv = _conv(pkg, qt, shape, seed=int(qt))
    entries = _patch(pkg, conv, spec, seed=shape[0] + int(qt))
    x = (torch.randn(2, shape[1], 8, 8, generator=torch.Generator().manual_seed(3)) * 0.5).to(DEV).to(dtype)
    W_ref, b_ref, y_ref = _weight(conv, x, False)
    _weight(conv, x, True)                                             # builds the plan (K1 for the factors s)
    calls.clear()
    W, b, y = _weight(conv, x, True)
    assert calls == ["ggufb200_dequant_patched_dora"], calls          # the cached forward: one launch, no K1
    assert W.dtype == dtype and tuple(W.shape) == shape and torch.equal(b, b_ref)
    assert bool(torch.isfinite(W).all()) and torch.equal(_bits(W), _bits(W_ref)) and torch.equal(y, y_ref)


# ---------------------------------------------------------------- lists with rank sums: the conv budget
CASES = [
    (Q.Q4_K, (640, 320, 3, 3), [("lora", 16, 1.0, 8.0, 0)], torch.float16),
    (Q.Q8_0, (320, 320, 1, 1), [("lora", 32, 0.8, 16.0, 1)], torch.bfloat16),
    (Q.Q6_K, (640, 320, 3, 3), [("loha", 8, 1.0, 4.0, 1)], torch.float16),
    (Q.Q4_K, (332, 320, 3, 3), [("lora", 16, 0.8, 8.0, 0)], torch.bfloat16),                         # Cout not a multiple of 64
    (Q.Q8_0, (640, 640, 3, 3), [("locon_mid", 8, 1.0, 4.0, 0), ("loha_tucker", 4, 0.8, 2.0, 1)], torch.float16),
    (Q.Q6_K, (640, 320, 3, 3), [("lora", 32, 0.7, 16.0, None), ("lora", 16, 1.0, 8.0, 1), ("lokr", (8, "full4d"), 1.0, None, None)],
     torch.bfloat16),
    (Q.Q4_K, (640, 320, 3, 3), [("lora", 16, 0.8, 8.0, 0), ("lora", 8, 1.0, 4.0, 1)], torch.float16),   # two DoRA entries, two axes
    (Q.IQ2_XXS, (640, 320, 3, 3), [("lora", 16, 1.0, 8.0, 1), ("loha", 4, 0.5, None, None)], torch.float32),
    (Q.Q8_0, (320, 320, 1, 1), [("loha", 8, 0.8, 4.0, 0)], torch.float32),
]


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_patched_weight_meets_the_conv_budget(pkg, restated, kernel, calls, case):
    qt, shape, spec, dtype = case
    conv = _conv(pkg, qt, shape, seed=int(qt) + 1)
    entries = _patch(pkg, conv, spec, seed=shape[1] + int(qt))
    x = (torch.randn(2, shape[1], 8, 8, generator=torch.Generator().manual_seed(4)) * 0.5).to(DEV).to(dtype)
    calls.clear()
    W, b, y = _weight(conv, x, True)
    assert calls == ["ggufb200_dequant", "ggufb200_dequant_patched_dora"] or (
        qt in FALLBACK and calls == ["ggufb200_dequant_fallback", "ggufb200_dequant_patched_dora"]), calls
    W_ref, b_ref, y_ref = _weight(conv, x, False)
    assert W.dtype == dtype and torch.equal(b, b_ref) and bool(torch.isfinite(W).all())
    _check_budget(pkg, conv, dtype, entries, W, W_ref)
    rel = ((y.float() - y_ref.float()).norm() / y_ref.float().norm()).item()
    assert rel <= 1e-3, rel


def test_plan_cache_and_offloaded_weight(pkg, restated, kernel, calls, monkeypatch):
    shape = (640, 320, 3, 3)
    conv = _conv(pkg, Q.Q4_K, shape, seed=12)
    entries = _patch(pkg, conv, [("lora", 16, 0.8, 8.0, 1), ("lokr", (8, "full4d"), 1.0, None, 0)], seed=12)
    builds = []
    real = pkg.ops.build_conv_dora_plan
    monkeypatch.setattr(pkg.ops, "build_conv_dora_plan", lambda W, terms: builds.append(W.dtype) or real(W, terms))
    x = torch.randn(1, 320, 8, 8, generator=torch.Generator().manual_seed(5)).to(DEV)
    W16, _b, y16 = _weight(conv, x.half(), True)
    Wb, _b, _y = _weight(conv, x.bfloat16(), True)
    W16b, _b, y16b = _weight(conv, x.half(), True)
    assert builds == [torch.float16, torch.bfloat16] and torch.equal(W16b, W16) and torch.equal(y16b, y16)   # one plan per dtype, kept
    # an offloaded (host) weight: the packed bytes are copied for the call, the result is the same
    host = _conv(pkg, Q.Q4_K, shape, seed=12, raw=conv.weight.as_subclass(torch.Tensor).cpu())
    host.weight.patches = conv.weight.patches
    calls.clear()
    W_host, _b, y_host = _weight(host, x.half(), True)
    assert calls[-1] == "ggufb200_dequant_patched_dora" and host.weight.device.type == "cpu"
    assert torch.equal(W_host, W16) and torch.equal(y_host, y16)
    # in-place changes rebuild the plan: a dora_scale, a factor, the packed bytes
    changes = [lambda: _payload(entries[0][1])[1][4].mul_(1.1), lambda: _payload(entries[1][1])[1][0].mul_(0.5),
               lambda: conv.weight.as_subclass(torch.Tensor)[:144].copy_(_raw(Q.Q4_K, 256, seed=99))]
    for change in changes:
        before = list(builds)
        change()
        W2, _b, _y = _weight(conv, x.half(), True)
        assert builds == before + [torch.float16] and not torch.equal(W2, W16)
        W_ref, _b, _y = _weight(conv, x.half(), False)
        _check_budget(pkg, conv, torch.float16, entries, W2, W_ref)
        W16 = W2


def test_every_element_written_and_nothing_else(pkg, restated, kernel):
    """NaN-poisoned output inside a sentinel-filled buffer, 332 rows (a partial last row tile)."""
    shape = (332, 320, 3, 3)
    conv = _conv(pkg, Q.Q6_K, shape, seed=9)
    _patch(pkg, conv, [("lora", 16, 0.8, 8.0, 0), ("lokr", (4, "full4d"), 1.0, None, 1)], seed=5)
    x = torch.randn(1, 320, 8, 8, generator=torch.Generator().manual_seed(6)).to(DEV).half()
    W, _b, _y = _weight(conv, x, True)
    (_keep, _s), descs, dora = conv._conv_dora_plan(x)
    numel = W.numel()
    buf = torch.full((numel + 64,), float("nan"), dtype=torch.float16, device=DEV)
    buf[numel:] = 1234.0
    raw = conv.weight.as_subclass(torch.Tensor)
    rc = pkg.lib.lib().ggufb200_dequant_patched_dora(int(Q.Q6_K), raw.data_ptr(), shape[0], numel // shape[0], buf.data_ptr(),
                                                     pkg.dequant.dtype_code(torch.float16), pkg.dequant.math_code(None, torch.float16),
                                                     descs, dora, 2, torch.cuda.current_stream().cuda_stream)
    pkg.lib.check(rc, "ggufb200_dequant_patched_dora")
    assert not bool(buf[:numel].isnan().any()) and bool((buf[numel:] == 1234.0).all())
    assert torch.equal(_bits(buf[:numel]), _bits(W.reshape(-1)))


def test_class_switch_and_declined_lists_take_the_two_step_route(pkg, restated, calls):
    shape = (320, 320, 3, 3)
    conv = _conv(pkg, Q.Q4_K, shape, seed=21)
    entries = _patch(pkg, conv, [("lora", 16, 1.0, 8.0, 0)], seed=21)
    x = torch.randn(1, 320, 8, 8, generator=torch.Generator().manual_seed(7)).to(DEV).half()
    calls.clear()
    W, _b, y = _weight(conv, x, True)
    assert calls[-1] == "ggufb200_dequant_patched_dora", calls         # the layer's own cost model takes the kernel here
    calls.clear()
    W_ref, _b, y_ref = _weight(conv, x, False)
    assert calls == ["ggufb200_dequant"], calls                        # the class switch: K1 + calculate_weight
    strength, value, *_ = entries[0]
    for declined in ([(strength, value, 0.5, None, None)], [entries[0]] * 9):
        conv.weight.patches = [(declined, "w")]
        calls.clear()
        W, _b, y = _weight(conv, x, True)
        assert calls == ["ggufb200_dequant"], calls
        W_ref, _b, y_ref = _weight(conv, x, False)
        assert torch.equal(W, W_ref) and torch.equal(y, y_ref)
    conv.weight.patches = [(entries, "w")]
    conv.patch_dtype = torch.float32                                   # the reference forms the patch in another dtype
    calls.clear()
    _weight(conv, x, True)
    assert "ggufb200_dequant_patched_dora" not in calls


@pytest.mark.parametrize("case", ["zero_row", "zero_dora_scale", "nan_block"])
def test_non_finite_and_degenerate_weights(pkg, restated, kernel, case):
    """A zero output channel (norm = eps), a zero dora_scale and a NaN-scale block: non-finite values where the two-step route
    puts them, the rest within the budget."""
    shape = (320, 320, 1, 1)
    raw = _raw(Q.Q8_0, 320 * 320, seed=4).view(-1, 34)
    if case == "zero_row":
        raw[10 * 10:11 * 10, 2:] = 0                                  # row 10: every quant zero
    if case == "nan_block":
        raw[700, 0:2] = torch.tensor([0x00, 0x7E], dtype=torch.uint8)
    conv = _conv(pkg, Q.Q8_0, shape, raw=raw.reshape(-1))
    spec = [("lora", 16, 0.8, 8.0, 0), ("lora", 8, 1.0, 4.0, 1)]
    entries = _patch(pkg, conv, spec, seed=6)
    if case == "zero_dora_scale":
        _payload(entries[0][1])[1][4][5] = 0.0
    if case == "zero_row":                                           # the weight's own zero norm would give dora_scale 0 there
        _payload(entries[0][1])[1][4][10] = 1.0
    x = torch.randn(1, 320, 8, 8, generator=torch.Generator().manual_seed(8)).to(DEV).half()
    W, _b, _y = _weight(conv, x, True)
    W_ref, _b, _y = _weight(conv, x, False)
    assert torch.equal(W.isnan(), W_ref.isnan()) and torch.equal(W.isinf(), W_ref.isinf())
    assert torch.equal(W[W.isinf()], W_ref[W_ref.isinf()])
    if case == "nan_block":
        assert bool(W_ref.isnan().any())
    fin = torch.isfinite(W_ref)
    if case != "nan_block":
        _check_budget(pkg, conv, torch.float16, entries, torch.where(fin, W, 0), torch.where(fin, W_ref, 0))
