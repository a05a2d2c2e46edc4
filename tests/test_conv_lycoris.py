"""CPU tests of LoKr, LoCon `mid` and Tucker LoHa patches on a packed Conv2d weight: the recogniser (`conv_lycoris_terms`), its
scale rules and refusals, the composed operands against ComfyUI's own expressions, the layer's route conditions, the cost model's
LoKr term, and ggufb200_dequant_patched's argument codes and descriptor layout without a device.

The reference (ComfyUI's LoRA / LoHa / LoKr adapters) restated, every factor cast to fp32 first:
    LoCon mid   down = mm(down.T.flatten(1), mid.T.flatten(1)).reshape(Cin, r, kh, kw).T;   diff = up.flatten(1) @ down.flatten(1)
    LoHa t1/t2  m = einsum('i j k l, j r, i p -> p r k l', t, wb, wa) per half;             diff = m1 * m2
    LoKr        w1 = w1 or w1_a @ w1_b;  w2 = w2 or w2_a @ w2_b or einsum(t2, w2_b, w2_a);  diff = kron(w1 [, 1, 1], w2)
    weight += ((strength * alpha) * diff.reshape(weight.shape)).type(weight.dtype)"""
import ctypes
import os
import re

import pytest
import torch

E_TYPE, E_DTYPE, E_ALIGN, E_SHAPE, E_NULL, E_UNSUPPORTED = -1, -2, -3, -4, -5, -8


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


class LoKrAdapter(LoRAAdapter):
    pass


def _r(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed + sum(shape)))


def _lokr(cout, cin, k, f, form, r=4, alpha=None, seed=0):
    """LoKr payload (w1, w2, alpha, w1_a, w1_b, w2_a, w2_b, t2, dora_scale) of factor f: A [f, f], w2 on [cout / f, cin / f, k, k]."""
    b1, c2 = cout // f, cin // f
    w1 = _r(f, f, seed=seed)
    if form == "full4d":
        return (w1, _r(b1, c2, k, k, seed=seed + 1), alpha, None, None, None, None, None, None)
    if form == "full2d":
        return (w1, _r(b1, c2 * k * k, seed=seed + 1), alpha, None, None, None, None, None, None)
    if form == "decomposed":
        return (w1, None, alpha, None, None, _r(b1, r, seed=seed + 2), _r(r, c2 * k * k, seed=seed + 3), None, None)
    if form == "tucker":
        return (w1, None, alpha, None, None, _r(r, b1, seed=seed + 2), _r(r, c2, seed=seed + 3), _r(r, r, k, k, seed=seed + 4), None)
    if form == "w1_decomposed":
        return (None, _r(b1, c2, k, k, seed=seed + 1), alpha, _r(f, 2, seed=seed + 5), _r(2, f, seed=seed + 6), None, None, None, None)
    raise ValueError(form)


def _locon_mid(cout, cin, k, r, alpha=None, seed=0):
    return (_r(cout, r, 1, 1, seed=seed), _r(r, cin, 1, 1, seed=seed + 1), alpha, _r(r, r, k, k, seed=seed + 2), None, None)


def _loha_tucker(cout, cin, k, r, alpha=None, seed=0):
    return (_r(r, cout, seed=seed), _r(r, cin, seed=seed + 1), alpha, _r(r, cout, seed=seed + 2), _r(r, cin, seed=seed + 3),
            _r(r, r, k, k, seed=seed + 4), _r(r, r, k, k, seed=seed + 5), None)


def _locon(cout, cin, k, r, alpha=None):
    return (_r(cout, r, 1, 1), _r(r, cin, k, k), alpha, None, None, None)


def _loha(cout, cin, k, r, alpha=None):
    return (_r(cout, r), _r(r, cin * k * k), alpha, _r(cout, r), _r(r, cin * k * k), None, None, None)


# ---------------------------------------------------------------- the reference, restated
def ref_lokr_diff(v, shape):
    w1, w2, alpha, w1_a, w1_b, w2_a, w2_b, t2, _ds = v
    dim = None
    if w1 is None:
        dim = w1_b.shape[0]
        w1 = torch.mm(w1_a.float(), w1_b.float())
    if w2 is None:
        dim = w2_b.shape[0]
        w2 = torch.mm(w2_a.float(), w2_b.float()) if t2 is None else torch.einsum("i j k l, j r, i p -> p r k l", t2.float(), w2_b.float(),
                                                                                     w2_a.float())
    w1, w2 = w1.float(), w2.float()
    if w2.dim() == 4:
        w1 = w1.unsqueeze(2).unsqueeze(2)
    alpha = alpha / dim if (alpha is not None and dim is not None) else 1.0
    try:
        return alpha, torch.kron(w1, w2).reshape(shape)
    except RuntimeError:                   # ComfyUI logs the error and skips the entry (torch.kron of a non-contiguous einsum result)
        return alpha, None


def ref_locon_mid_diff(v, shape):
    up, down, alpha, mid = (t.float() if torch.is_tensor(t) else t for t in v[:4])
    alpha = 1.0 if alpha is None else alpha / down.shape[0]
    final_shape = [down.shape[1], down.shape[0], mid.shape[2], mid.shape[3]]
    down = torch.mm(down.transpose(0, 1).flatten(start_dim=1), mid.transpose(0, 1).flatten(start_dim=1)).reshape(final_shape).transpose(0, 1)
    return alpha, torch.mm(up.flatten(start_dim=1), down.flatten(start_dim=1)).reshape(shape)


def ref_loha_tucker_diff(v, shape):
    w1a, w1b, alpha, w2a, w2b, t1, t2 = (t.float() if torch.is_tensor(t) else t for t in v[:7])
    alpha = 1.0 if alpha is None else alpha / w1b.shape[0]
    m1 = torch.einsum("i j k l, j r, i p -> p r k l", t1, w1b, w1a)
    m2 = torch.einsum("i j k l, j r, i p -> p r k l", t2, w2b, w2a)
    return alpha, (m1 * m2).reshape(shape)


def _kron2d(A, B):
    """Element (n, k) = A[n // b1, k // b2] * B[n % b1, k % b2], one fp32 product each."""
    b1, b2 = B.shape
    n = torch.arange(A.shape[0] * b1)[:, None]
    k = torch.arange(A.shape[1] * b2)[None, :]
    return A[n // b1, k // b2] * B[n % b1, k % b2]


# ---------------------------------------------------------------- the recogniser
LOKR_FORMS = ["full4d", "full2d", "decomposed", "tucker", "w1_decomposed"]


@pytest.mark.parametrize("form", LOKR_FORMS)
@pytest.mark.parametrize("k", [1, 3])
def test_lokr_forms_are_recognised_with_the_reference_scale(pkg, form, k):
    v = _lokr(64, 32, k, 4, form, alpha=8.0)
    terms = pkg.ops.conv_lycoris_terms([(0.5, ("lokr", v), 1.0, None, None), (2.0, LoKrAdapter(v), 1.0)])
    assert [t[0] for t in terms] == ["lokr", "lokr"]
    alpha, _diff = ref_lokr_diff(v, (64, 32, k, k))
    assert terms[0][1] == 0.5 * alpha and terms[1][1] == 2.0 * alpha
    assert pkg.ops.conv_term_shape("lokr", terms[0][2]) == (64, 32 * k * k) and pkg.ops.conv_term_ranks("lokr", terms[0][2]) == ()
    assert all(any(s is t for t in v if torch.is_tensor(t)) for s in terms[0][3])      # cache keys: the entry's own tensors
    if form in ("full4d", "full2d", "tucker"):
        assert terms[0][1] == (0.5 * 8.0 / 4 if form == "tucker" else 0.5)            # alpha / dim only with a decomposed factor


def test_scale_rules_for_alpha_and_dim(pkg):
    f = pkg.ops.conv_lycoris_terms
    whole = _lokr(64, 32, 3, 4, "full4d", alpha=8.0)
    assert f([(0.5, ("lokr", whole), 1.0)])[0][1] == 0.5                               # no decomposed factor: dim None -> 1.0
    w1dec = _lokr(64, 32, 3, 4, "w1_decomposed", alpha=8.0)
    assert f([(0.5, ("lokr", w1dec), 1.0)])[0][1] == 0.5 * 8.0 / 2                     # dim = w1_b.shape[0]
    both = (None, None, 8.0, w1dec[3], w1dec[4]) + _lokr(64, 32, 3, 4, "decomposed", r=16)[5:]
    assert f([(0.5, ("lokr", both), 1.0)])[0][1] == 0.5 * 8.0 / 16                    # w2's dim wins
    assert f([(0.5, ("lokr", _lokr(64, 32, 3, 4, "decomposed")), 1.0)])[0][1] == 0.5   # alpha None -> 1.0
    assert f([(0.5, ("lora", _locon_mid(64, 32, 3, 8, alpha=4.0)), 1.0)])[0][1] == 0.5 * 4.0 / 8
    assert f([(0.5, ("loha", _loha_tucker(64, 32, 3, 4, alpha=6.0)), 1.0)])[0][1] == 0.5 * 6.0 / 4


def test_mixed_lists_keep_list_order(pkg):
    o = pkg.ops
    entries = [(1.0, ("lora", _locon(64, 32, 3, 4)), 1.0, None, None), (0.5, LoKrAdapter(_lokr(64, 32, 3, 8, "tucker")), 1.0),
               (0.25, LoHaAdapter(_loha(64, 32, 3, 2)), 1.0), (1.0, ("lora", _locon_mid(64, 32, 3, 4)), 1.0),
               (-1.0, ("loha", _loha_tucker(64, 32, 3, 2)), 1.0)]
    terms = o.conv_lycoris_terms(entries)
    assert [t[0] for t in terms] == ["lora", "lokr", "loha", "locon_mid", "loha_tucker"]
    assert all(o.conv_term_shape(kind, f) == (64, 288) for kind, _s, f, _src in terms)
    assert [o.conv_term_ranks(kind, f) for kind, _s, f, _src in terms] == [(4,), (), (2, 2), (4,), (2, 2)]
    # plain LoRA / LoHa lists are not this recogniser's: conv_patch_terms keeps serving them exactly as before
    plain = [entries[0], entries[2]]
    assert o.conv_lycoris_terms(plain) is None and o.conv_patch_terms(plain) is not None
    # and the existing recognisers keep refusing every new form
    for e in entries[1:2] + entries[3:]:
        assert o.conv_patch_terms([e]) is None and o.lycoris_terms([e]) is None and o.lora_band_terms([e]) is None


def test_declines(pkg):
    f = pkg.ops.conv_lycoris_terms
    lokr = _lokr(64, 32, 3, 4, "full4d")
    good = (1.0, ("lokr", lokr), 1.0)
    assert f([good]) is not None
    assert f([(1.0, ("lokr", lokr), 1.0, (0, 0, 32), None)]) is None                          # offset
    assert f([(1.0, ("lokr", lokr), 0.5)]) is None                                            # strength_model != 1
    assert f([(1.0, ("lokr", lokr), 1.0, None, lambda w: w)]) is None                         # function hook
    assert f([(1.0, ("lokr", lokr[:8] + (_r(64, 1),)), 1.0)]) is None                         # DoRA
    assert f([(1.0, ("lora", _locon_mid(64, 32, 3, 4)[:4] + (_r(64, 1), None)), 1.0)]) is None        # DoRA on LoCon mid
    assert f([(1.0, ("lora", _locon_mid(64, 32, 3, 4)[:5] + ((64, 32, 3, 3),)), 1.0)]) is None         # reshape
    t = _loha_tucker(64, 32, 3, 4)
    assert f([(1.0, ("loha", t[:6] + (None, None)), 1.0)]) is None                            # only t1
    assert f([(1.0, ("loha", t[:5] + (None, t[6], None)), 1.0)]) is None                      # only t2
    assert f([(1.0, ("loha", t[:7] + (_r(64, 1),)), 1.0)]) is None                            # Tucker LoHa with DoRA
    assert f([(1.0, ("lokr", (_r(4, 4, 1, 1),) + lokr[1:]), 1.0)]) is None                    # 4-D w1
    assert f([(1.0, ("lokr", (None, lokr[1], None, None, None, None, None, None, None)), 1.0)]) is None  # no w1 at all
    assert f([good, (1.0, ("diff", (_r(64, 32, 3, 3),)), 1.0)]) is None                      # one refusal declines the list
    assert f([good, (1.0, ("lora", _locon(64, 32, 3, 4)), 0.5)]) is None
    assert f([]) is None


def test_misfit_shapes_are_not_served(pkg):
    """a1 b1 != Cout or a2 b2 != Cin kh kw: the reference's reshape fails or mixes rows; the layer leaves that to the two-step
    route."""
    o = pkg.ops
    v = _lokr(64, 32, 3, 4, "full4d")
    (kind, _s, factors, _src), = o.conv_lycoris_terms([(1.0, ("lokr", v), 1.0)])
    assert o.conv_term_shape(kind, factors) == (64, 288)
    assert o.conv_term_shape(kind, factors) != (32, 576)                  # same numel, another [Cout, K]: declined by the layer
    skew = (_r(2, 8), _r(32, 4, 3, 3)) + v[2:]                             # kron [64, 32, 3, 3] from a1 = 2, a2 = 8: Cout 64, K 288
    (kind, _s, factors, _src), = o.conv_lycoris_terms([(1.0, ("lokr", skew), 1.0)])
    assert o.conv_term_shape(kind, factors) == (64, 288)


# ---------------------------------------------------------------- the composed operands, bit for bit
@pytest.mark.parametrize("form", LOKR_FORMS)
@pytest.mark.parametrize("k", [1, 3])
def test_lokr_operands_equal_the_reference_kron(pkg, form, k):
    shape = (64, 32, k, k)
    v = _lokr(*shape[:3], 4, form)
    (_kind, _s, factors, _src), = pkg.ops.conv_lycoris_terms([(1.0, ("lokr", v), 1.0)])
    (a1, a2), (b1, b2) = pkg.ops.conv_lokr_shapes(factors)
    _alpha, diff = ref_lokr_diff(v, shape)
    AB = pkg.ops.conv_lokr_operands(factors, torch.device("cpu"))
    if diff is None:                       # the reference skips this entry: the layer leaves it to the two-step route
        assert AB is None
        return
    A, B = AB
    assert tuple(A.shape) == (a1, a2) and tuple(B.shape) == (b1, b2) and a1 * b1 == 64 and a2 * b2 == 32 * k * k
    assert A.dtype == B.dtype == torch.float32 and A.is_contiguous() and B.is_contiguous()
    assert torch.equal(_kron2d(A, B), diff.reshape(64, -1))


def test_locon_mid_and_tucker_loha_operands(pkg):
    o = pkg.ops
    shape = (64, 32, 3, 3)
    cpu = torch.device("cpu")
    v = _locon_mid(64, 32, 3, 8)
    (_k, _s, factors, _src), = o.conv_lycoris_terms([(1.0, ("lora", v), 1.0)])
    down = o.locon_mid_down(factors[1], factors[2], cpu)
    up, dn, _a, mid = v[:4]
    final_shape = [dn.shape[1], dn.shape[0], mid.shape[2], mid.shape[3]]
    ref_down = torch.mm(dn.transpose(0, 1).flatten(start_dim=1), mid.transpose(0, 1).flatten(start_dim=1)).reshape(final_shape).transpose(0, 1)
    assert torch.equal(down, ref_down.flatten(start_dim=1))                              # the reference's own expression
    _alpha, diff = ref_locon_mid_diff(v, shape)
    assert torch.equal(torch.mm(up.flatten(start_dim=1), down), diff.reshape(64, -1))
    t = _loha_tucker(64, 32, 3, 4)
    (_k, _s, factors, _src), = o.conv_lycoris_terms([(1.0, ("loha", t), 1.0)])
    a1, b1 = o.loha_tucker_half(*factors[:3], cpu)
    a2, b2 = o.loha_tucker_half(*factors[3:], cpu)
    assert tuple(a1.shape) == (64, 4) and tuple(b1.shape) == (4, 288)
    _alpha, diff = ref_loha_tucker_diff(t, shape)
    got = (a1 @ b1) * (a2 @ b2)                                   # only the order of the fp32 sums differs from the einsum
    assert torch.allclose(got, diff.reshape(64, -1), rtol=1e-5, atol=1e-5)


def test_operand_descriptors(pkg):
    o, L = pkg.ops, pkg.lib
    entries = [(1.0, ("lora", _locon(64, 32, 3, 4, 2.0)), 1.0), (0.5, ("lokr", _lokr(64, 32, 3, 8, "decomposed", alpha=4.0)), 1.0),
               (0.25, ("loha", _loha_tucker(64, 32, 3, 2)), 1.0), (1.0, ("lora", _locon_mid(64, 32, 3, 4)), 1.0)]
    terms = o.conv_lycoris_terms(entries)
    keep, descs = o.conv_lycoris_operands(terms, torch.device("cpu"))
    assert [d.kind for d in descs] == [L.PATCH_LOWRANK, L.PATCH_KRON, L.PATCH_LOWRANK, L.PATCH_LOWRANK]
    assert descs[0].lowrank.r1 == 4 and descs[0].lowrank.a2 is None and descs[0].lowrank.scale == 0.5
    k = descs[1].kron
    A, B = keep[1]
    assert (k.A, k.B, k.a1, k.a2, k.b1, k.b2, k.band_dim) == (A.data_ptr(), B.data_ptr(), 8, 8, 8, 36, -1) and k.scale == 0.5 * 4.0 / 4
    lh = descs[2].lowrank
    assert lh.r1 == 2 and lh.r2 == 2 and lh.b2 == keep[2][3].data_ptr() and tuple(keep[2][1].shape) == (2, 288)
    assert descs[3].lowrank.r1 == 4 and tuple(keep[3][1].shape) == (4, 288)
    assert all(t.dtype == torch.float32 and t.is_contiguous() for f in keep for t in f)
    # a LoKr entry whose reference kron raises makes the whole list the two-step route's
    tucker = (0.5, ("lokr", _lokr(64, 32, 3, 8, "tucker")), 1.0)
    if ref_lokr_diff(tucker[1][1], (64, 32, 3, 3))[1] is None:
        assert o.conv_lycoris_operands(o.conv_lycoris_terms(entries + [tucker]), torch.device("cpu")) is None


# ---------------------------------------------------------------- the layer's route conditions
def _conv(pkg, qt, shape, patches, bias=True):
    import gguf
    conv = pkg.ops.GGMLOps.Conv2d(shape[1], shape[0], shape[2], padding=shape[2] // 2, device="meta")
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    n = shape[0] * shape[1] * shape[2] * shape[3] // bs * ts
    w = pkg.ops.GGMLTensor(torch.zeros(n, dtype=torch.uint8), tensor_type=qt, tensor_shape=torch.Size(shape),
                           patches=[(patches, "k")] if patches else [])
    sd = {"weight": w}
    if bias:
        sd["bias"] = torch.zeros(shape[0])
    conv.load_state_dict(sd, assign=True, strict=False)
    return conv


CUDA_LIKE = type("CudaLike", (), {"is_cuda": True, "dtype": torch.float16, "device": torch.device("cuda", 0)})()


def test_layer_route_conditions(pkg, monkeypatch):
    """`_conv_lycoris_operands` serves a list only where ggufb200_dequant_patched can; every other case is the two-step route."""
    import gguf
    Q = gguf.GGMLQuantizationType
    ops = pkg.ops
    monkeypatch.setattr(ops, "conv_lycoris_operands", lambda terms, dev: ("built", len(terms)))
    shape = (64, 32, 3, 3)
    lokr = [(1.0, ("lokr", _lokr(64, 32, 3, 4, "full4d")), 1.0)]
    mixed = lokr + [(1.0, ("lora", _locon(64, 32, 3, 4)), 1.0)]

    def route(conv, x=CUDA_LIKE):
        return conv._conv_lycoris_operands(x)
    assert route(_conv(pkg, Q.Q4_K, shape, lokr)) == ("built", 1)                            # LoKr only, block format: one route
    assert route(_conv(pkg, Q.IQ2_XXS, shape, lokr)) == ("built", 1)                         # fallback format
    assert route(_conv(pkg, Q.Q4_K, shape, mixed)) == ("built", 2)                           # mixed list
    assert route(_conv(pkg, Q.Q4_K, shape, lokr), torch.zeros(1, 32, 8, 8)) is None          # CPU input
    conv = _conv(pkg, Q.Q4_K, shape, lokr)
    conv.conv_patches_in_kernel = False
    assert route(conv) is None                                                               # the class switch
    conv = _conv(pkg, Q.Q4_K, shape, lokr)
    conv.patch_dtype = torch.float32
    assert route(conv) is None                                                               # patch_dtype set
    assert route(_conv(pkg, Q.BF16, shape, lokr)) is None                                    # BF16 weight
    odd = [(1.0, ("lokr", _lokr(64, 12, 1, 4, "full4d")), 1.0)]
    assert route(_conv(pkg, Q.Q8_0, (64, 12, 1, 1), odd)) is None                            # K = 12
    assert route(_conv(pkg, Q.Q8_0, (32, 64, 3, 3), lokr)) is None                           # a1 b1 != Cout (numel agrees)
    assert route(_conv(pkg, Q.Q4_0, shape, lokr * 9)) is None                                # more than 8 entries
    big = [(1.0, ("lora", _locon_mid(64, 32, 3, 1025)), 1.0)] + lokr
    assert route(_conv(pkg, Q.Q4_0, shape, big)) is None                                     # rank above 1024
    # plain lists never reach this recogniser's route; the cost model gates every list
    assert route(_conv(pkg, Q.Q4_K, shape, [(1.0, ("lora", _locon(64, 32, 3, 4)), 1.0)])) is None
    monkeypatch.setattr(ops, "lowrank_pays", lambda N, K, terms: False)
    assert route(_conv(pkg, Q.Q4_K, shape, mixed)) is None and route(_conv(pkg, Q.Q4_K, shape, lokr)) is None


def test_cost_model_follows_the_measured_runs(pkg):
    """`lowrank_pays` against tools/bench_conv_lycoris.py on the H100 (DESIGN.md section 9): the kernel won every measured LoKr
    list (factors 4 / 8 / 16, whole or decomposed w2, alone or with a rank-32 LoRA), every Tucker LoHa (dim 8 / 16) and every
    Tucker LoCon (rank 16 / 32: its two-step route pays the mid composition on top of the LoRA product).  The LoRA / LoHa
    arithmetic is unchanged: a rank-256 LoRA next to a LoKr on proj_in still keeps the two-step route."""
    o = pkg.ops

    def pays(shape, *entries):
        return o.lowrank_pays(shape[0], shape[1] * shape[2] * shape[3], o.conv_lycoris_terms(list(entries)))
    for shape in [(320, 320, 1, 1), (640, 640, 1, 1), (1280, 1280, 1, 1), (640, 320, 3, 3), (1280, 1280, 3, 3)]:
        cout, cin, k = shape[:3]
        for f in (4, 8, 16):
            for form in ("full4d", "decomposed"):
                assert pays(shape, (1.0, ("lokr", _lokr(cout, cin, k, f, form, r=16)), 1.0)), (shape, f, form)
        assert pays(shape, (1.0, ("lokr", _lokr(cout, cin, k, 8, "full4d")), 1.0), (1.0, ("lora", _locon(cout, cin, k, 32)), 1.0))
        for r in (16, 32):
            assert pays(shape, (1.0, ("lora", _locon_mid(cout, cin, k, r)), 1.0)), (shape, r)
        for r in (8, 16):
            assert pays(shape, (1.0, ("loha", _loha_tucker(cout, cin, k, r)), 1.0)), (shape, r)
    proj_in = (320, 320, 1, 1)
    assert not pays(proj_in, (1.0, ("lokr", _lokr(320, 320, 1, 4, "full4d")), 1.0), (1.0, ("lora", _locon(320, 320, 1, 256)), 1.0))
    assert o.conv_patch_terms([(1.0, ("lora", _locon(320, 320, 1, 32)), 1.0)]) is not None
    assert not o.lowrank_pays(320, 320, o.conv_patch_terms([(1.0, ("lora", _locon(320, 320, 1, 64)), 1.0)]))   # plain LoRA: as before


# ---------------------------------------------------------------- the C entry point, without a device
def test_patched_argument_codes_without_gpu(pkg):
    import gguf
    Q = gguf.GGMLQuantizationType
    L = pkg.lib.lib()
    W, LR, KP = pkg.lib.WeightPatch, pkg.lib.LowrankPatch, pkg.lib.KronPatch
    buf = (ctypes.c_uint8 * 4096)()
    p16 = (ctypes.addressof(buf) + 15) & ~15

    def lr(*a):
        return W(pkg.lib.PATCH_LOWRANK, LR(*a), KP())

    def kr(A=p16, B=p16, a1=2, a2=8, b1=4, b2=32, band=-1, kind=None):
        return W(pkg.lib.PATCH_KRON if kind is None else kind, LR(), KP(A, B, a1, a2, b1, b2, band, 1.0, 0, 0))

    def call(patches, qt=Q.Q4_K, N=8, K=256, out=p16, od=0, md=0, packed=p16, n=None):
        arr = (W * max(1, len(patches)))(*patches)
        return L.ggufb200_dequant_patched(int(qt), packed, N, K, out, od, md, arr, len(patches) if n is None else n, None)
    ok_lr, ok_kr = lr(p16, p16, None, None, 4, 0, 1.0), kr()
    assert call([ok_kr], qt=999) == E_TYPE
    assert call([ok_kr], qt=Q.BF16) == E_UNSUPPORTED
    assert call([ok_kr], od=3) == E_DTYPE and call([ok_kr], md=5) == E_DTYPE
    assert call([ok_kr], K=240) == E_SHAPE and call([ok_kr], N=0) == E_SHAPE
    assert call([ok_kr, ok_lr] * 4 + [ok_kr]) == E_SHAPE                                         # more than 8
    assert call([kr(kind=2)]) == E_UNSUPPORTED and call([kr(kind=-1)]) == E_UNSUPPORTED         # unknown kind
    assert call([kr(band=0)]) == E_UNSUPPORTED and call([kr(band=1)]) == E_UNSUPPORTED          # bands: not on this entry point
    assert call([kr(a1=0, b1=8)]) == E_SHAPE and call([kr(b2=-32, a2=-8)]) == E_SHAPE          # non-positive
    assert call([kr(a1=4, b1=4)]) == E_SHAPE                                                    # a1 b1 != N
    assert call([kr(a2=4, b2=32)]) == E_SHAPE                                                   # a2 b2 != K
    assert call([lr(p16, p16, None, None, 0, 0, 1.0)]) == E_SHAPE                               # LOWRANK rank 0
    assert call([lr(p16, p16, None, None, 1025, 0, 1.0)]) == E_SHAPE
    assert call([ok_lr, kr(B=None)]) == E_NULL and call([kr(A=None)]) == E_NULL
    assert call([lr(p16, None, None, None, 4, 0, 1.0)]) == E_NULL
    assert call([kr(A=p16 + 2)]) == E_ALIGN and call([kr(B=p16 + 1)]) == E_ALIGN
    assert call([lr(p16 + 2, p16, None, None, 4, 0, 1.0)]) == E_ALIGN
    assert call([ok_kr], out=p16 + 4) == E_ALIGN
    assert call([ok_kr], packed=None) == E_NULL
    assert L.ggufb200_dequant_patched(int(Q.Q4_K), p16, 8, 256, p16, 0, 0, None, 1, None) == E_NULL
    assert call([kr(a1=1, b1=3, a2=1, b2=96)], qt=Q.IQ2_XXS, N=3, K=96) == E_SHAPE              # N K not whole 256-element blocks
    # a valid list passes every check and reaches the device check (an error other than the argument codes without a GPU)
    if not torch.cuda.is_available():
        assert call([ok_lr, ok_kr]) not in (E_TYPE, E_DTYPE, E_ALIGN, E_SHAPE, E_NULL, E_UNSUPPORTED, 0)


def test_header_structs_and_binding_agree(pkg):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "ggufb200.h")).read()
    assert int(re.search(r"#define GGUFB200_PATCH_LOWRANK (\d+)", hdr).group(1)) == pkg.lib.PATCH_LOWRANK
    assert int(re.search(r"#define GGUFB200_PATCH_KRON (\d+)", hdr).group(1)) == pkg.lib.PATCH_KRON

    def fields(name):
        """[(C type, field name), ...] of a header struct, pointers as 'T *'."""
        body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), hdr, re.S).group(1))
        out = []
        for decl in filter(None, (d.strip() for d in body.split(";"))):
            m = re.match(r"(?:const\s+)?(\w+)\s*(\*?)\s*(.*)", decl)
            ctype = m.group(1) + (" *" if m.group(2) else "")
            out += [(ctype, n.strip().lstrip("*")) for n in m.group(3).split(",")]
        return out
    want = {"int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "float": ctypes.c_float, "float *": ctypes.c_void_p,
            "ggufb200_lowrank_patch": pkg.lib.LowrankPatch, "ggufb200_kron_patch": pkg.lib.KronPatch}
    for name, cls in (("ggufb200_weight_patch", pkg.lib.WeightPatch), ("ggufb200_kron_patch", pkg.lib.KronPatch),
                      ("ggufb200_lowrank_patch", pkg.lib.LowrankPatch)):
        got = fields(name)
        assert [n for _t, n in got] == [f[0] for f in cls._fields_], (name, got)
        assert [want[t] for t, _n in got] == [f[1] for f in cls._fields_], (name, got)
    assert ctypes.sizeof(pkg.lib.WeightPatch) == 8 + ctypes.sizeof(pkg.lib.LowrankPatch) + ctypes.sizeof(pkg.lib.KronPatch)
    assert "ggufb200_dequant_patched" in pkg.lib.EXPORTS and len(pkg.lib.lib().ggufb200_dequant_patched.argtypes) == 10
