"""CPU tests of LoRA / LoCon and LoHa patches on a packed Conv2d weight: the recogniser (`conv_patch_terms`), its refusals, the
Linear recognisers' unchanged refusal of 4-D factors, the layer's route conditions, and argument validation of
ggufb200_dequant_lowrank without a device.

The reference (comfy.lora.calculate_weight) multiplies a LoRA's `up.flatten(start_dim=1) @ down.flatten(start_dim=1)` and a LoHa's
`(w1a @ w1b) * (w2a @ w2b)` as given, reshapes the delta to the conv weight and adds `((strength * alpha) * delta).type(dtype)`
with alpha = alpha / rank."""
import ctypes

import pytest
import torch

E_TYPE, E_DTYPE, E_ALIGN, E_SHAPE, E_NULL, E_UNSUPPORTED = -1, -2, -3, -4, -5, -8


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


def _m(*shape):
    return torch.ones(*shape)


def _locon(cout, cin, k, r, alpha=None):
    return (_m(cout, r, 1, 1), _m(r, cin, k, k), alpha, None, None, None)


def _loha(cout, cin, k, r1, r2, alpha=None):
    return (_m(cout, r1), _m(r1, cin * k * k), alpha, _m(cout, r2), _m(r2, cin * k * k), None, None, None)


@pytest.mark.parametrize("k", [1, 3])
def test_recogniser_flattens_lora_and_locon(pkg, k):
    locon = _locon(64, 32, k, 8, alpha=4.0)
    terms = pkg.ops.conv_patch_terms([(0.5, ("lora", locon), 1.0, None, None), (2.0, LoRAAdapter(locon), 1.0)])
    assert [t[0] for t in terms] == ["lora", "lora"]
    kind, scale, (up, down), sources = terms[0]
    assert scale == 0.5 * 4.0 / 8 and terms[1][1] == 2.0 * 4.0 / 8
    assert tuple(up.shape) == (64, 8) and tuple(down.shape) == (8, 32 * k * k)
    assert sources[0] is locon[0] and sources[1] is locon[1]                          # cache keys follow the entry's own tensors
    # 2-D LoRA factors (already flat) are taken as they are
    flat = (_m(64, 8), _m(8, 32 * k * k), None, None, None, None)
    (_kind, scale, factors, sources), = pkg.ops.conv_patch_terms([(1.5, ("lora", flat), 1.0)])
    assert scale == 1.5 and factors == flat[:2] and sources == flat[:2]


def test_recogniser_loha_and_mixed_lists(pkg):
    loha = _loha(64, 32, 3, 4, 2, alpha=6.0)
    mixed = [(1.0, ("lora", _locon(64, 32, 3, 2)), 1.0, None, None), (0.5, LoHaAdapter(loha), 1.0, None, None),
             (-1.0, ("loha", loha), 1.0)]
    terms = pkg.ops.conv_patch_terms(mixed)
    assert [t[0] for t in terms] == ["lora", "loha", "loha"]
    assert terms[0][1] == 1.0 and terms[1][1] == 0.5 * 6.0 / 4 and terms[2][1] == -1.0 * 6.0 / 4
    assert terms[1][2] == loha[:2] + loha[3:5] and terms[1][3] == terms[1][2]
    assert all(pkg.ops._fits_weight(kind, f, None, 64, 288) for kind, _s, f, _src in terms)
    assert not pkg.ops._fits_weight("lora", terms[0][2], None, 64, 320)               # misfit: delta is [64, 288]
    assert not pkg.ops._fits_weight("loha", terms[1][2], None, 32, 288)


def test_recogniser_declines_what_needs_calculate_weight(pkg):
    f = pkg.ops.conv_patch_terms
    locon, loha = _locon(64, 32, 3, 4), _loha(64, 32, 3, 4, 2)
    assert f([(0.5, ("lora", locon), 0.7, None, None)]) is None                              # strength_model
    assert f([(0.5, ("lora", locon), 1.0, None, lambda w: w)]) is None                       # function hook
    assert f([(0.5, ("lora", locon), 1.0, (0, 0, 32), None)]) is None                        # offset
    assert f([(0.5, ("lora", locon[:3] + (_m(4, 4, 3, 3),) + locon[4:]), 1.0)]) is None       # LoCon mid (Tucker)
    assert f([(0.5, ("lora", locon[:4] + (_m(64, 1, 1, 1),) + locon[5:]), 1.0)]) is None      # dora_scale
    assert f([(0.5, ("lora", locon[:5] + ((64, 32, 3, 3),)), 1.0)]) is None                   # reshape
    assert f([(0.5, ("loha", loha[:5] + (_m(4, 2, 3, 3), None, None)), 1.0)]) is None         # Tucker t1
    assert f([(0.5, ("loha", loha[:7] + (_m(64, 1),)), 1.0)]) is None                         # DoRA
    assert f([(0.5, ("loha", (_m(64, 4, 1, 1),) + loha[1:]), 1.0)]) is None                   # 4-D LoHa: torch.mm would refuse it
    assert f([(0.5, ("lora", (_m(64, 4, 3, 3), _m(4, 32, 3, 3), None)), 1.0)]) is None        # up [Cout, r, 3, 3] does not chain
    assert f([(0.5, ("lokr", (_m(8, 8), _m(8, 36), None, None, None, None, None, None, None)), 1.0)]) is None
    assert f([(0.5, ("diff", (_m(64, 32, 3, 3),)), 1.0)]) is None
    assert f([(1.0, ("lora", locon), 1.0), (1.0, ("glora", loha), 1.0)]) is None            # one refusal declines the list
    assert f([]) == []


def test_linear_recognisers_still_refuse_4d_factors(pkg):
    """The Linear routes are unchanged: the same conv entries stay None for them."""
    o = pkg.ops
    locon, loha = _locon(64, 32, 3, 4), _loha(64, 32, 3, 4, 2)
    entries = [[(0.5, ("lora", locon), 1.0)], [(0.5, LoRAAdapter(_locon(64, 32, 1, 4)), 1.0)],
               [(0.5, ("loha", (_m(64, 4, 1, 1),) + loha[1:]), 1.0)]]
    for e in entries:
        assert o.lora_band_terms(e) is None and o.lycoris_terms(e) is None and o.dora_terms(e) is None, e
        assert o.lora_side_terms(e) is None


def _conv(pkg, qt, shape, patches, bias=True):
    conv = pkg.ops.GGMLOps.Conv2d(shape[1], shape[0], shape[2], padding=shape[2] // 2, device="meta")
    import gguf
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    n = shape[0] * shape[1] * shape[2] * shape[3] // bs * ts
    w = pkg.ops.GGMLTensor(torch.zeros(n, dtype=torch.uint8), tensor_type=qt, tensor_shape=torch.Size(shape),
                           patches=[(patches, "k")] if patches else [])
    sd = {"weight": w}
    if bias:
        sd["bias"] = torch.zeros(shape[0])
    conv.load_state_dict(sd, assign=True, strict=False)
    return conv


def test_layer_route_conditions(pkg, monkeypatch):
    """`_conv_patch_operands` is consulted only where the kernel serves the weight; every other case is the two-step route."""
    import gguf
    Q = gguf.GGMLQuantizationType
    ops = pkg.ops
    monkeypatch.setattr(ops, "conv_patch_operands", lambda terms, dev: ("built", len(terms)))
    assert _conv(pkg, Q.Q4_0, (320, 320, 1, 1), [(1.0, ("lora", _locon(320, 320, 1, 128)), 1.0)])._conv_patch_operands(
        type("CudaLike", (), {"is_cuda": True, "dtype": torch.float16, "device": torch.device("cuda", 0)})()) is None   # cost model
    monkeypatch.setattr(ops, "lowrank_pays", lambda N, K, terms: True)          # the other conditions, whatever the cost
    x = torch.zeros(1, 32, 8, 8)
    cuda_like = type("CudaLike", (), {"is_cuda": True, "dtype": torch.float16, "device": torch.device("cuda", 0)})()
    lora = [(1.0, ("lora", _locon(64, 32, 3, 4)), 1.0)]
    conv = _conv(pkg, Q.Q4_K, (64, 32, 3, 3), lora)
    assert conv._conv_patch_operands(x) is None                                              # CPU input
    assert conv._conv_patch_operands(cuda_like) == ("built", 1)
    conv.conv_patches_in_kernel = False
    assert conv._conv_patch_operands(cuda_like) is None                                      # the class switch
    conv = _conv(pkg, Q.Q4_K, (64, 32, 3, 3), lora)
    conv.patch_dtype = torch.float32
    assert conv._conv_patch_operands(cuda_like) is None                                      # patch_dtype set
    assert _conv(pkg, Q.Q4_K, (64, 32, 3, 3), [])._conv_patch_operands(cuda_like) is None    # unpatched: the plain route
    assert _conv(pkg, Q.BF16, (64, 32, 3, 3), lora)._conv_patch_operands(cuda_like) is None  # BF16 weight
    assert _conv(pkg, Q.Q8_0, (64, 32, 3, 3), [(1.0, ("lora", _locon(64, 32, 1, 4)), 1.0)])._conv_patch_operands(cuda_like) is None  # misfit
    odd = [(1.0, ("lora", _locon(64, 12, 1, 4)), 1.0)]
    assert _conv(pkg, Q.Q8_0, (64, 12, 1, 1), odd)._conv_patch_operands(cuda_like) is None   # K = 12: not a multiple of 32
    assert _conv(pkg, Q.IQ2_XXS, (64, 32, 3, 3), lora)._conv_patch_operands(cuda_like) == ("built", 1)
    many = lora * 9
    assert _conv(pkg, Q.Q4_0, (64, 32, 3, 3), many)._conv_patch_operands(cuda_like) is None  # more than 8 patches
    big = [(1.0, ("lora", _locon(64, 32, 3, 1025)), 1.0)]
    assert _conv(pkg, Q.Q4_0, (64, 32, 3, 3), big)._conv_patch_operands(cuda_like) is None   # rank above the limit


def test_operand_descriptors(pkg):
    terms = pkg.ops.conv_patch_terms([(1.0, ("lora", _locon(64, 32, 3, 4, 2.0)), 1.0), (0.25, ("loha", _loha(64, 32, 3, 4, 2)), 1.0)])
    ops, descs = pkg.ops.conv_patch_operands(terms, torch.device("cpu"))
    assert [o[0] for o in ops] == ["lora", "loha"] and all(t.dtype == torch.float32 and t.is_contiguous() for o in ops for t in o[2])
    assert descs[0].r1 == 4 and descs[0].r2 == 0 and descs[0].a2 is None and descs[0].scale == 0.5
    assert descs[1].r1 == 4 and descs[1].r2 == 2 and descs[1].a2 == ops[1][2][2].data_ptr() and descs[1].b2 == ops[1][2][3].data_ptr()
    assert ops[0][2][1].shape == (4, 288)


def test_lowrank_argument_codes_without_gpu(pkg):
    import gguf
    Q = gguf.GGMLQuantizationType
    L = pkg.lib.lib()
    buf = (ctypes.c_uint8 * 4096)()
    p16 = (ctypes.addressof(buf) + 15) & ~15
    P = pkg.lib.LowrankPatch

    def call(qt=Q.Q4_K, N=8, K=256, out=p16, od=0, md=0, patches=None, n=None, packed=p16):
        arr = (P * max(1, len(patches or [])))(*(patches or []))
        return L.ggufb200_dequant_lowrank(int(qt), packed, N, K, out, od, md, arr, len(patches or []) if n is None else n, None)
    ok = P(p16, p16, None, None, 4, 0, 1.0)
    assert call(qt=999, patches=[ok]) == E_TYPE
    assert call(qt=Q.BF16, patches=[ok]) == E_UNSUPPORTED
    assert call(od=3, patches=[ok]) == E_DTYPE and call(md=5, patches=[ok]) == E_DTYPE
    assert call(K=240, patches=[ok]) == E_SHAPE                                                    # K % 32
    assert call(N=3, K=96, patches=[ok]) == E_SHAPE                                                # N * K not whole blocks
    assert call(N=0, patches=[ok]) == E_SHAPE
    assert call(patches=[ok] * 9) == E_SHAPE                                                       # more than 8 patches
    assert call(patches=[P(p16, p16, None, None, 0, 0, 1.0)]) == E_SHAPE                           # rank 0
    assert call(patches=[P(p16, p16, None, None, 1025, 0, 1.0)]) == E_SHAPE                        # rank above the limit
    assert call(patches=[P(p16, p16, p16, p16, 4, 0, 1.0)]) == E_SHAPE                             # LoHa without r2
    assert call(patches=[P(p16, None, None, None, 4, 0, 1.0)]) == E_NULL
    assert call(patches=[P(p16, p16, p16, None, 4, 2, 1.0)]) == E_NULL                             # LoHa without b2
    assert call(patches=[P(p16 + 2, p16, None, None, 4, 0, 1.0)]) == E_ALIGN
    assert call(packed=None, patches=[P(p16, p16, None, p16 + 1, 4, 0, 1.0)]) == E_NULL            # LoRA: b2 is not read, not checked
    assert call(packed=None, patches=[P(p16, p16, p16, p16 + 1, 4, 2, 1.0)]) == E_ALIGN            # LoHa: it is
    assert call(out=p16 + 4, patches=[ok]) == E_ALIGN
    assert call(packed=None, patches=[ok]) == E_NULL
    assert L.ggufb200_dequant_lowrank(int(Q.Q4_K), p16, 8, 256, p16, 0, 0, None, 1, None) == E_NULL
    assert call(qt=Q.IQ2_XXS, N=3, K=96, patches=[ok]) == E_SHAPE                                  # fallback types: same shape rule
    assert call(qt=Q.MXFP4, K=240, patches=[ok]) == E_SHAPE


def test_header_binding_and_constants_agree(pkg):
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "ggufb200.h")).read()
    assert int(re.search(r"#define GGUFB200_LOWRANK_MAX_PATCHES (\d+)", hdr).group(1)) == pkg.lib.LOWRANK_MAX_PATCHES
    assert int(re.search(r"#define GGUFB200_LOWRANK_MAX_RANK (\d+)", hdr).group(1)) == pkg.lib.LOWRANK_MAX_RANK
    fields = re.search(r"typedef struct ggufb200_lowrank_patch \{(.*?)\} ggufb200_lowrank_patch;", hdr, re.S).group(1)
    names = re.findall(r"(\w+)(?:,\s*(\w+))?;", re.sub(r"/\*.*?\*/", "", fields))
    flat = [n for pair in names for n in pair if n]
    assert flat == [f[0] for f in pkg.lib.LowrankPatch._fields_]
    assert "ggufb200_dequant_lowrank" in pkg.lib.EXPORTS and len(pkg.lib.lib().ggufb200_dequant_lowrank.argtypes) == 10


def test_cost_model_follows_the_measured_crossovers(pkg):
    """`lowrank_pays` against the H100 measurements it was fitted to (DESIGN.md section 9): LoRA crosses over near rank 40 on
    the 320-channel 1x1 conv and near rank 120 on the SDXL 1280-channel 3x3; LoHa (whose two-step route forms two products and
    a full-size elementwise one) keeps the kernel at every measured shape."""
    def lora(shape, r):
        return pkg.ops.conv_patch_terms([(1.0, ("lora", _locon(shape[0], shape[1], shape[2], r)), 1.0)])

    def loha(shape, r):
        return pkg.ops.conv_patch_terms([(1.0, ("loha", _loha(shape[0], shape[1], shape[2], r, r)), 1.0)])

    def pays(shape, terms):
        return pkg.ops.lowrank_pays(shape[0], shape[1] * shape[2] * shape[3], terms)
    proj_in, sd3x3, sdxl3x3, proj1280 = (320, 320, 1, 1), (640, 320, 3, 3), (1280, 1280, 3, 3), (1280, 1280, 1, 1)
    assert pays(proj_in, lora(proj_in, 16)) and not pays(proj_in, lora(proj_in, 64)) and not pays(proj_in, lora(proj_in, 128))
    assert pays(sd3x3, lora(sd3x3, 64)) and not pays(sd3x3, lora(sd3x3, 128))
    assert pays(proj1280, lora(proj1280, 64)) and not pays(proj1280, lora(proj1280, 128))
    assert pays(sdxl3x3, lora(sdxl3x3, 64)) and not pays(sdxl3x3, lora(sdxl3x3, 256))
    for shape in (proj_in, sd3x3, sdxl3x3, proj1280):
        assert pays(shape, loha(shape, 16)) and pays(shape, loha(shape, 32))
    # a stack is priced as a whole: the kernel pays the sum of the ranks, the two-step route a product and an add per entry
    assert pays(proj_in, lora(proj_in, 16) * 2) and not pays(proj_in, lora(proj_in, 128) * 2)
