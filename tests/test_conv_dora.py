"""CPU tests of DoRA (weight-decomposed LoRA) patches on a packed Conv2d weight: the recogniser (`conv_dora_terms`) and its
refusals, the 4-D replay of weight_decompose (`dora_replay` with `conv_term_delta`) against ComfyUI's calculate_weight restated,
the plan's descriptors, and ggufb200_dequant_patched_dora's argument codes and descriptor layout without a device.

The reference restated (ComfyUI's LoRA / LoHa / LoKr adapters and weight_decompose, every factor cast to fp32 first):
    diff = mm(up.flatten(1), down.flatten(1)) | mm(w1a, w1b) * mm(w2a, w2b) | kron(w1 [, 1, 1], w2), reshaped to the weight
    plain   weight += ((strength * alpha) * diff).type(weight.dtype)
    DoRA    diff *= alpha;  Wc = weight + diff.type(weight.dtype)
            norm = weight.reshape(Cout, -1).norm(dim=1) (dora_scale [Cout, 1, 1, 1]) or
                   Wc.transpose(0, 1).reshape(Cin, -1).norm(dim=1) (dora_scale [1, Cin, 1, 1]), + eps(weight.dtype)
            Wc *= (dora_scale / norm).type(weight.dtype);  weight = Wc (strength 1) or weight += strength * (Wc - weight)"""
import ctypes
import os
import re

import pytest
import torch

E_TYPE, E_DTYPE, E_ALIGN, E_SHAPE, E_NULL, E_UNSUPPORTED = -1, -2, -3, -4, -5, -8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


class LoKrAdapter(LoRAAdapter):
    pass


def _r(*shape, seed=0, scale=0.1):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed + 3 * sum(shape))) * scale


def _ds_out(cout, seed=0):
    return _r(cout, 1, 1, 1, seed=seed, scale=1.0).abs() + 0.5


def _ds_in(cin, seed=0):
    return _r(1, cin, 1, 1, seed=seed, scale=1.0).abs() + 0.5


def _locon(cout, cin, k, r, alpha=None, ds=None, seed=0):
    return ("lora", (_r(cout, r, 1, 1, seed=seed), _r(r, cin, k, k, seed=seed + 1), alpha, None, ds, None))


def _locon_mid(cout, cin, k, r, alpha=None, ds=None, seed=0):
    return ("lora", (_r(cout, r, 1, 1, seed=seed), _r(r, cin, 1, 1, seed=seed + 1), alpha, _r(r, r, k, k, seed=seed + 2), ds, None))


def _loha(cout, cin, k, r, alpha=None, ds=None, seed=0):
    return ("loha", (_r(cout, r, seed=seed), _r(r, cin * k * k, seed=seed + 1), alpha, _r(cout, r, seed=seed + 2),
                     _r(r, cin * k * k, seed=seed + 3), None, None, ds))


def _loha_tucker(cout, cin, k, r, alpha=None, ds=None, seed=0):
    return ("loha", (_r(r, cout, seed=seed), _r(r, cin, seed=seed + 1), alpha, _r(r, cout, seed=seed + 2), _r(r, cin, seed=seed + 3),
                     _r(r, r, k, k, seed=seed + 4), _r(r, r, k, k, seed=seed + 5), ds))


def _lokr(cout, cin, k, f, alpha=None, ds=None, seed=0, decomposed=False):
    w1, b1, c2 = _r(f, f, seed=seed, scale=1.0), cout // f, cin // f
    if decomposed:
        return ("lokr", (w1, None, alpha, None, None, _r(b1, 4, seed=seed + 1), _r(4, c2 * k * k, seed=seed + 2), None, ds))
    return ("lokr", (w1, _r(b1, c2, k, k, seed=seed + 1), alpha, None, None, None, None, None, ds))


def _adapter(value):
    return {"lora": LoRAAdapter, "loha": LoHaAdapter, "lokr": LoKrAdapter}[value[0]](value[1])


# ---------------------------------------------------------------- the reference, restated
def ref_diff(kind, v, shape):
    """(alpha, fp32 diff of the weight's shape) of one payload as ComfyUI's adapters form it."""
    f = [t.float() if torch.is_tensor(t) else t for t in v]
    if kind == "lora":
        up, down, alpha, mid = f[0], f[1], f[2], f[3]
        a = 1.0 if alpha is None else alpha / down.shape[0]
        if mid is not None:
            final_shape = [down.shape[1], down.shape[0], mid.shape[2], mid.shape[3]]
            down = torch.mm(down.transpose(0, 1).flatten(start_dim=1), mid.transpose(0, 1).flatten(start_dim=1)).reshape(final_shape).transpose(0, 1)
        return a, torch.mm(up.flatten(start_dim=1), down.flatten(start_dim=1)).reshape(shape)
    if kind == "loha":
        w1a, w1b, alpha, w2a, w2b, t1, t2 = f[:7]
        a = 1.0 if alpha is None else alpha / w1b.shape[0]
        if t1 is not None:
            m1 = torch.einsum("i j k l, j r, i p -> p r k l", t1, w1b, w1a)
            m2 = torch.einsum("i j k l, j r, i p -> p r k l", t2, w2b, w2a)
        else:
            m1, m2 = torch.mm(w1a, w1b), torch.mm(w2a, w2b)
        return a, (m1 * m2).reshape(shape)
    w1, w2, alpha, w1_a, w1_b, w2_a, w2_b = f[:7]
    dim = None
    if w1 is None:
        dim, w1 = w1_b.shape[0], torch.mm(w1_a, w1_b)
    if w2 is None:
        dim, w2 = w2_b.shape[0], torch.mm(w2_a, w2_b)
    if w2.dim() == 4:
        w1 = w1.unsqueeze(2).unsqueeze(2)
    a = alpha / dim if (alpha is not None and dim is not None) else 1.0
    return a, torch.kron(w1, w2).reshape(shape)


def weight_decompose(dora_scale, weight, lora_diff, alpha, strength):
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


def calculate_weight(patches, weight):
    for strength, value, *_ in patches:
        kind, v = (value[0], tuple(value[1])) if isinstance(value, tuple) else (type(value).__name__[:4].lower(), tuple(value.weights))
        alpha, diff = ref_diff(kind, v, weight.shape)
        ds = v[{"lora": 4, "loha": 7, "lokr": 8}[kind]]
        if ds is not None:
            weight = weight_decompose(ds, weight, diff, alpha, strength)
        else:
            weight += ((strength * alpha) * diff).type(weight.dtype)
    return weight


# ---------------------------------------------------------------- the recogniser
def test_recogniser_accepts_dora_lists(pkg):
    o = pkg.ops
    shape = (64, 32, 3, 3)
    out, inp = _ds_out(64), _ds_in(32)
    entries = [(1.0, _locon(64, 32, 3, 4, 8.0, out), 1.0), (0.8, _adapter(_loha(64, 32, 3, 2, None, inp)), 1.0, None, None),
               (1.0, _lokr(64, 32, 3, 4, 2.0, out, decomposed=True), 1.0), (0.5, _locon(64, 32, 3, 8, 4.0), 1.0),
               (1.0, _locon_mid(64, 32, 3, 4, None, inp), 1.0), (1.2, _loha_tucker(64, 32, 3, 2, 1.0, out), 1.0),
               (1.0, _adapter(_lokr(64, 32, 3, 8, None, inp)), 1.0)]
    terms = o.conv_dora_terms(entries, shape)
    assert [t[0] for t in terms] == ["lora", "loha", "lokr", "lora", "locon_mid", "loha_tucker", "lokr"]
    assert [t[6] for t in terms] == [0, 1, 0, None, 1, 0, 1]                                 # axes; None for the plain entry
    assert terms[0][1:3] == (1.0, 2.0) and terms[0][5] is out                                # alpha / rank, apart from the strength
    assert terms[1][1:3] == (0.8, 1.0) and terms[1][5] is inp
    assert terms[2][1:3] == (1.0, 0.5)                                                      # LoKr: alpha / w2_b.shape[0]
    assert terms[3][1:3] == (0.5, 0.5) and terms[3][5] is None
    assert terms[5][1:3] == (1.2, 0.5)
    assert all(t[5] is None or t[5] is t[4][-1] for t in terms)                            # dora_scale is a cache key
    assert o.conv_dora_terms([entries[3]], shape) is None                                   # no DoRA entry: the other recognisers' list
    # the other conv recognisers keep refusing every list with DoRA
    for e in entries[:3] + entries[4:]:
        assert o.conv_patch_terms([e]) is None and o.conv_lycoris_terms([e]) is None
    # the recognised terms (without dora_scale) are exactly what the other recognisers make of the entry without it
    plain = o.conv_lycoris_terms([(0.8, _loha(64, 32, 3, 2, None, None), 1.0), (1.0, _lokr(64, 32, 3, 4, 2.0, None, decomposed=True), 1.0)])
    assert [(k, s) for k, s, _f, _src in plain] == [("loha", 0.8), ("lokr", 0.5)]


def test_recogniser_declines_what_needs_calculate_weight(pkg):
    o = pkg.ops
    shape = (64, 32, 3, 3)
    ds = _ds_out(64)
    ok = _locon(64, 32, 3, 4, 4.0, ds)
    assert o.conv_dora_terms([(1.0, ok, 1.0)], shape) is not None
    assert o.conv_dora_terms([(1.0, ok, 0.5)], shape) is None                                              # strength_model
    assert o.conv_dora_terms([(1.0, ok, 1.0, None, lambda w: w)], shape) is None                           # function hook
    assert o.conv_dora_terms([(1.0, ok, 1.0, (0, 0, 32), None)], shape) is None                            # offset
    assert o.conv_dora_terms([(1.0, ("lora", ok[1][:5] + ((64, 288),)), 1.0)], shape) is None               # reshape
    assert o.conv_dora_terms([(1.0, ok, 1.0)] * 9, shape) is None                                           # more than 8 entries
    assert o.conv_dora_terms([(1.0, _locon(32, 32, 3, 4, None, ds), 1.0)], shape) is None                   # misfit (Cout 32)
    assert o.conv_dora_terms([(1.0, _locon(64, 32, 1, 4, None, ds), 1.0)], shape) is None                   # misfit (1x1 factors)
    assert o.conv_dora_terms([(1.0, _lokr(64, 64, 3, 4, None, ds), 1.0)], shape) is None                    # LoKr misfit
    assert o.conv_dora_terms([(1.0, _locon(64, 32, 3, 1025, None, ds), 1.0)], shape) is None                # rank limit
    assert o.conv_dora_terms([(1.0, ("lora", ok[1][:4] + ([1.0] * 64, None)), 1.0)], shape) is None         # dora_scale not a tensor
    for bad in (torch.ones(64), torch.ones(64, 1), torch.ones(1, 32), torch.ones(1, 32, 1), torch.ones(64, 32, 1, 1),
                torch.ones(1, 16, 1, 1), torch.ones(64, 1, 3, 3), torch.ones(1, 32, 3, 3)):
        assert o.conv_dora_terms([(1.0, ("lora", ok[1][:4] + (bad, None)), 1.0)], shape) is None, bad.shape  # other dora_scale shapes
    assert o.conv_dora_terms([(1.0 + 1e-12, ok, 1.0)], shape) is None                                       # st != 1 but fp32(st) == 1
    assert o.conv_dora_terms([(1.0, ok, 1.0), (1.0, ("diff", (torch.ones(64, 32, 3, 3),)), 1.0)], shape) is None   # another kind
    lone_t1 = ("loha", _loha_tucker(64, 32, 3, 2, None, ds)[1][:6] + (None, ds))
    assert o.conv_dora_terms([(1.0, lone_t1, 1.0)], shape) is None                                          # Tucker LoHa with t1 only
    assert o.conv_dora_axis(torch.ones(1, 1, 1, 1), (1, 1, 3, 3)) == 0                                     # shape[0] == Cout: output axis
    assert o.conv_dora_axis(torch.ones(1, 8, 1, 1), (1, 8, 3, 3)) is None


# ---------------------------------------------------------------- the 4-D replay, bit for bit
def _lists(cout, cin, k):
    out, inp = _ds_out(cout, 1), _ds_in(cin, 2)
    return {
        "out-st1": [(1.0, _locon(cout, cin, k, 4, 2.0, out), 1.0)],
        "in-st1": [(1.0, _locon(cout, cin, k, 4, None, inp), 1.0)],
        "out-st0.8": [(0.8, _loha(cout, cin, k, 3, 1.5, out), 1.0)],
        "in-st0.8": [(0.8, _adapter(_lokr(cout, cin, k, 4, None, inp)), 1.0)],
        "mixed": [(0.7, _locon(cout, cin, k, 8, 4.0), 1.0), (1.0, _locon_mid(cout, cin, k, 4, 2.0, out), 1.0),
                  (0.6, _loha_tucker(cout, cin, k, 2, 1.0, inp), 1.0), (1.0, _lokr(cout, cin, k, 8, 8.0, out, decomposed=True), 1.0)],
    }


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("name", ["out-st1", "in-st1", "out-st0.8", "in-st0.8", "mixed"])
def test_replay_is_the_reference_weight_bit_for_bit(pkg, dtype, name):
    o = pkg.ops
    shape = (64, 32, 3, 3)
    entries = _lists(*shape[:3])[name]
    terms = o.conv_dora_terms(entries, shape)
    assert terms is not None
    W0 = _r(*shape, seed=5).to(dtype)
    want = calculate_weight(entries, W0.clone())
    factors, patched = o.dora_replay(W0, [(k, st, a, f, ds) for k, st, a, f, _src, ds, _ax in terms], o.conv_term_delta)
    assert patched.dtype == dtype and patched.shape == shape and torch.equal(patched, want)
    assert [s is None for s in factors] == [t[5] is None for t in terms]
    for s, t in zip(factors, terms):
        if s is not None:
            assert s.dtype == dtype and s.shape == (shape[0] if t[6] == 0 else shape[1],)
    # the plan: s in fp32 holding the dtype values, one DoRA descriptor per entry, deltas scaled by alpha (DoRA) or st * alpha
    keep_s, descs, dora = o.build_conv_dora_plan(W0, terms)
    keep, s32 = keep_s
    assert len(keep) == len(terms)
    for i, ((kind, st, a, _f, _src, ds, axis), s) in enumerate(zip(terms, factors)):
        scale = descs[i].kron.scale if kind == "lokr" else descs[i].lowrank.scale
        if ds is None:
            assert dora[i].factor is None and scale == pytest.approx(st * a, rel=1e-7)
            continue
        assert scale == pytest.approx(a, rel=1e-7)
        assert dora[i].factor == s32[i].data_ptr() and dora[i].axis == axis and dora[i].group == 9
        assert dora[i].strength == pytest.approx(st, rel=1e-7)
        assert s32[i].dtype == torch.float32 and torch.equal(s32[i].to(dtype), s)


def test_linear_replay_is_unchanged(pkg):
    """The Linear's 2-D replay takes the same ops as before the 4-D generalisation: calculate_weight restated on [N, K]."""
    o = pkg.ops
    N, K = 48, 80
    for ds in (_r(N, 1, seed=1, scale=1.0).abs() + 0.5, _r(1, K, seed=2, scale=1.0).abs() + 0.5):
        entries = [(0.8, ("lora", (_r(N, 4, seed=3), _r(4, K, seed=4), 2.0, None, ds, None)), 1.0),
                   (1.0, ("lora", (_r(N, 4, seed=5), _r(4, K, seed=6), None, None, None, None)), 1.0)]
        W0 = _r(N, K, seed=7).half()
        _f, patched = o.dora_replay(W0, o.dora_terms(entries))
        assert torch.equal(patched, calculate_weight(entries, W0.clone()))


def test_cost_model(pkg):
    o = pkg.ops
    for shape in ((320, 320, 1, 1), (640, 320, 3, 3), (1280, 1280, 3, 3)):
        cout, cin, k = shape[:3]
        N, K = cout, cin * k * k
        for r in (16, 32, 64):
            terms = o.conv_dora_terms([(1.0, _locon(cout, cin, k, r, None, _ds_out(cout)), 1.0)], shape)
            plain = [(kind, st * a, f, src) for kind, st, a, f, src, _ds, _ax in terms]
            # weight_decompose's passes only add to the two-step side: where the plain LoRA takes the kernel, its DoRA form does
            if o.lowrank_pays(N, K, plain):
                assert o.conv_dora_pays(N, K, terms)


# ---------------------------------------------------------------- the C entry point, without a device
def test_dora_argument_codes_without_gpu(pkg):
    import gguf
    Q = gguf.GGMLQuantizationType
    L = pkg.lib.lib()
    W, LR, KP, DP = pkg.lib.WeightPatch, pkg.lib.LowrankPatch, pkg.lib.KronPatch, pkg.lib.DoraPatch
    buf = (ctypes.c_uint8 * 4096)()
    p16 = (ctypes.addressof(buf) + 15) & ~15
    ok_lr = W(pkg.lib.PATCH_LOWRANK, LR(p16, p16, None, None, 4, 0, 1.0), KP())
    ok_kr = W(pkg.lib.PATCH_KRON, LR(), KP(p16, p16, 2, 8, 4, 36, -1, 1.0, 0, 0))

    def call(patches, dora, qt=Q.Q4_K, N=8, K=288, out=p16, od=0, md=0, packed=p16, n=None):
        arr = (W * max(1, len(patches)))(*patches)
        darr = None if dora is None else (DP * max(1, len(dora)))(*dora)
        return L.ggufb200_dequant_patched_dora(int(qt), packed, N, K, out, od, md, arr, darr, len(patches) if n is None else n, None)
    plain, out_ax, in_ax = DP(), DP(p16, 0, 0, 1.0), DP(p16, 1, 9, 0.8)
    # the checks of ggufb200_dequant_patched come first
    assert call([ok_kr], [out_ax], qt=999) == E_TYPE
    assert call([ok_kr], [out_ax], qt=Q.BF16) == E_UNSUPPORTED
    assert call([ok_kr], [out_ax], od=3) == E_DTYPE
    assert call([ok_kr], [out_ax], K=280) == E_SHAPE
    assert call([ok_kr, ok_lr] * 4 + [ok_kr], [plain] * 9) == E_SHAPE                           # more than 8
    assert call([ok_kr], [out_ax], out=p16 + 4) == E_ALIGN
    assert call([ok_kr], [out_ax], packed=None) == E_NULL
    # then the DoRA descriptors
    assert call([ok_kr], None) == E_NULL
    assert call([ok_kr], [DP(p16, 2, 9, 1.0)]) == E_SHAPE and call([ok_kr], [DP(p16, -1, 9, 1.0)]) == E_SHAPE    # axis
    assert call([ok_kr], [DP(p16, 1, 0, 1.0)]) == E_SHAPE                                      # group < 1
    assert call([ok_kr], [DP(p16, 1, 7, 1.0)]) == E_SHAPE                                      # K % group
    assert call([ok_kr], [DP(p16 + 2, 0, 0, 1.0)]) == E_ALIGN and call([ok_lr, ok_kr], [plain, DP(p16 + 1, 1, 9, 1.0)]) == E_ALIGN
    # no factor: a plain patch whose other fields are not read (the next descriptor's misaligned factor is what is reported)
    assert call([ok_kr, ok_kr], [DP(None, 7, -3, 1.0), DP(p16 + 2, 0, 0, 1.0)]) == E_ALIGN
    # valid lists pass every check and reach the device check (an error other than the argument codes without a GPU); the
    # host buffers here must never reach a kernel, so only where there is no device
    if not torch.cuda.is_available():
        codes = (E_TYPE, E_DTYPE, E_ALIGN, E_SHAPE, E_NULL, E_UNSUPPORTED, 0)
        assert call([ok_lr, ok_kr], [out_ax, in_ax]) not in codes and call([ok_kr], [DP(None, 7, -3, 1.0)]) not in codes
        assert call([], None, n=0) not in codes                                               # nothing to describe


def test_header_and_binding_agree(pkg):
    hdr = open(os.path.join(ROOT, "include", "ggufb200.h")).read()
    assert int(re.search(r"#define GGUFB200_DORA_AXIS_OUT (\d+)", hdr).group(1)) == pkg.lib.DORA_AXIS_OUT
    assert int(re.search(r"#define GGUFB200_DORA_AXIS_IN (\d+)", hdr).group(1)) == pkg.lib.DORA_AXIS_IN
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct ggufb200_dora_patch \{(.*?)\} ggufb200_dora_patch;", hdr, re.S).group(1))
    decls = [re.match(r"(?:const\s+)?(\w+)\s*(\*?)\s*(\w+)", d.strip()).groups() for d in body.split(";") if d.strip()]
    want = {("float", "*"): ctypes.c_void_p, ("int32_t", ""): ctypes.c_int32, ("float", ""): ctypes.c_float}
    assert [(n, want[(t, p)]) for t, p, n in decls] == list(pkg.lib.DoraPatch._fields_)
    assert ctypes.sizeof(pkg.lib.DoraPatch) == 24
    m = re.search(r"\bggufb200_dequant_patched_dora\s*\(([^;]*)\)\s*;", hdr)
    args = [a.strip() for a in m.group(1).split(",")]
    assert args[8] == "const ggufb200_dora_patch *dora" and len(args) == 11
    patched = [a.strip() for a in re.search(r"\bggufb200_dequant_patched\s*\(([^;]*)\)\s*;", hdr).group(1).split(",")]
    assert args[:8] + args[9:] == patched                                       # ggufb200_dequant_patched plus the DoRA array
    assert "ggufb200_dequant_patched_dora" in pkg.lib.EXPORTS and len(pkg.lib.lib().ggufb200_dequant_patched_dora.argtypes) == 11
