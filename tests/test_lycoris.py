"""CPU tests of LoHa and LoKr (LyCORIS) patches on a packed weight: the recogniser and its scaling rules, LoHa as one LoRA of
rank r1 r2, the layer's shape checks, and argument validation of ggufb200_dequant_kron without a device.

Scaling, as comfy.lora.calculate_weight applies it (restated here, the reference of these tests):
    LoHa  delta = (w1a @ w1b) * (w2a @ w2b),  scale = strength * alpha / w1b.shape[0]  (strength when alpha is None)
    LoKr  delta = kron(w1, w2), a decomposed factor being the fp32 torch.mm of its halves;  dim = w1_b.shape[0] when w1 is
          decomposed, overwritten by w2_b.shape[0] when w2 is;  scale = strength * alpha / dim, or strength when alpha is None
          or nothing is decomposed;  W += ((strength * alpha) * delta).to(W.dtype)"""
import ctypes

import pytest
import torch

import oracle
from util import Q

E_TYPE, E_DTYPE, E_ALIGN, E_SHAPE, E_NULL, E_UNSUPPORTED = -1, -2, -3, -4, -5, -8


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


class LoKrAdapter(LoRAAdapter):
    pass


def _m(*shape):
    return torch.ones(*shape)


def test_recogniser_loha_scaling_and_forms(pkg):
    f = pkg.ops.lycoris_terms
    w1a, w1b, w2a, w2b = _m(8, 4), _m(4, 16), _m(8, 2), _m(2, 16)
    loha = (w1a, w1b, 6.0, w2a, w2b, None, None, None)
    terms = f([(0.5, ("loha", loha), 1.0, None, None), (2.0, LoHaAdapter(loha[:2] + (None,) + loha[3:]), 1.0, (0, 8, 8), None)])
    assert [t[0] for t in terms] == ["loha", "loha"]
    assert terms[0][1] == 0.5 * 6.0 / 4 and terms[1][1] == 2.0               # alpha / w1b.shape[0]; no alpha -> strength
    assert terms[0][2][0] is w1a and terms[0][2][3] is w2b and terms[0][3] is None and terms[1][3] == (0, 8, 8)


def test_recogniser_lokr_scaling_rules(pkg):
    f = pkg.ops.lycoris_terms
    w1, w2 = _m(4, 4), _m(2, 4)
    w1_a, w1_b, w2_a, w2_b = _m(4, 3), _m(3, 4), _m(2, 5), _m(5, 4)

    def scale(payload, strength=0.5):
        terms = f([(strength, ("lokr", payload), 1.0, None, None)])
        assert terms is not None and terms[0][0] == "lokr"
        return terms[0][1]
    assert scale((w1, w2, 8.0, None, None, None, None, None, None)) == 0.5                    # nothing decomposed: alpha ignored
    assert scale((None, w2, 8.0, w1_a, w1_b, None, None, None, None)) == 0.5 * 8.0 / 3        # dim = w1_b.shape[0]
    assert scale((w1, None, 8.0, None, None, w2_a, w2_b, None, None)) == 0.5 * 8.0 / 5        # dim = w2_b.shape[0]
    assert scale((None, None, 8.0, w1_a, w1_b, w2_a, w2_b, None, None)) == 0.5 * 8.0 / 5      # w2's dim wins
    assert scale((None, None, None, w1_a, w1_b, w2_a, w2_b, None, None)) == 0.5               # no alpha
    terms = f([(1.5, LoKrAdapter((None, w2, 2.0, w1_a, w1_b, None, None, None, None)), 1.0, (1, 0, 16), None)])
    assert terms[0][1] == 1.5 * 2.0 / 3 and terms[0][3] == (1, 0, 16)
    assert pkg.ops.lokr_factor_shapes(terms[0][2]) == ((4, 4), (2, 4))


def test_recogniser_mixes_kinds_in_list_order(pkg):
    up, down = _m(8, 2), _m(2, 16)
    mixed = [(1.0, ("lora", (up, down, 4.0, None, None, None)), 1.0, None, None),
             (1.0, ("lokr", (_m(2, 4), _m(4, 4), None, None, None, None, None, None, None)), 1.0, None, None),
             (1.0, LoHaAdapter((_m(8, 1), _m(1, 16), None, _m(8, 1), _m(1, 16), None, None, None)), 1.0)]
    terms = pkg.ops.lycoris_terms(mixed)
    assert [t[0] for t in terms] == ["lora", "lokr", "loha"] and terms[0][1] == 2.0 and terms[0][2] == (up, down)


def test_recogniser_rejects_what_needs_calculate_weight(pkg):
    f = pkg.ops.lycoris_terms
    loha = (_m(8, 4), _m(4, 16), 6.0, _m(8, 2), _m(2, 16), None, None, None)
    lokr = (_m(4, 4), _m(2, 4), None, None, None, None, None, None, None)
    assert f([(0.5, ("loha", loha), 0.7, None, None)]) is None                                      # strength_model
    assert f([(0.5, ("lokr", lokr), 1.0, None, lambda w: w)]) is None                               # function hook
    assert f([(0.5, ("lokr", lokr), 1.0, (2, 0, 4), None)]) is None                                 # offset on another dim
    assert f([(0.5, ("lokr", lokr), 1.0, (0, -1, 4), None)]) is None
    assert f([(0.5, ("loha", loha[:5] + (_m(4, 4), None, None)), 1.0)]) is None                     # Tucker t1
    assert f([(0.5, ("loha", loha[:6] + (_m(2, 2), None)), 1.0)]) is None                           # Tucker t2
    assert f([(0.5, ("loha", loha[:7] + (_m(8),)), 1.0)]) is None                                   # DoRA
    assert f([(0.5, ("lokr", lokr[:7] + (_m(2, 2), None)), 1.0)]) is None                           # Tucker t2
    assert f([(0.5, LoKrAdapter(lokr[:8] + (_m(8),)), 1.0)]) is None                                # DoRA
    assert f([(0.5, ("loha", (torch.ones(8, 4, 1, 1),) + loha[1:]), 1.0)]) is None                  # conv (4-D) factor
    assert f([(0.5, ("lokr", (torch.ones(4, 4, 1, 1),) + lokr[1:]), 1.0)]) is None
    assert f([(0.5, ("lokr", (None,) + lokr[1:]), 1.0)]) is None                                     # neither w1 nor its halves
    assert f([(0.5, ("loha", (_m(8, 4), _m(3, 16)) + loha[2:]), 1.0)]) is None                      # factors do not chain
    assert f([(0.5, ("diff", (_m(8, 16),)), 1.0)]) is None
    assert f([(0.5, ("glora", loha), 1.0)]) is None
    assert f([(0.5, ("lora", (_m(8, 2), _m(2, 16), 4.0, None, _m(8), None)), 1.0)]) is None         # DoRA LoRA in the list
    # lora_band_terms keeps rejecting the LyCORIS kinds
    assert pkg.ops.lora_band_terms([(0.5, ("loha", loha), 1.0)]) is None
    assert pkg.ops.lora_band_terms([(0.5, LoKrAdapter(lokr), 1.0)]) is None


@pytest.mark.parametrize("r1,r2", [(1, 1), (4, 4), (8, 3)])
def test_loha_is_a_lora_of_rank_r1_r2(pkg, r1, r2):
    g = torch.Generator().manual_seed(r1 * 10 + r2)
    N, K = 48, 80
    w1a, w1b, w2a, w2b = (torch.randn(*s, generator=g) for s in ((N, r1), (r1, K), (N, r2), (r2, K)))
    up, down = pkg.ops.loha_as_lora(w1a, w1b, w2a, w2b, torch.device("cpu"))
    assert up.dtype == down.dtype == torch.float32 and tuple(up.shape) == (N, r1 * r2) and tuple(down.shape) == (r1 * r2, K)
    assert torch.equal(up[:, (r1 - 1) * r2 + r2 - 1], w1a[:, r1 - 1] * w2a[:, r2 - 1])
    assert torch.equal(down[(r1 - 1) * r2], w1b[r1 - 1] * w2b[0])
    want = (w1a.double() @ w1b.double()) * (w2a.double() @ w2b.double())
    got = up.double() @ down.double()
    # the fp32 products are the only roundings: a few fp32 ulps of the summed magnitudes
    bound = 8 * 2.0 ** -24 * ((w1a.abs().double() @ w1b.abs().double()) * (w2a.abs().double() @ w2b.abs().double()))
    assert bool(((got - want).abs() <= bound + 1e-30).all())


def _linear(pkg, N, K):
    raw = oracle.random_blocks(int(Q.Q4_K), N * K // 256, seed=3).reshape(N, K // 256 * 144)
    lin = pkg.ops.GGMLOps.Linear(K, N)
    lin.load_state_dict({"weight": pkg.ops.GGMLTensor(torch.from_numpy(raw), tensor_type=Q.Q4_K, tensor_shape=torch.Size((N, K)))})
    return lin


def test_layer_checks_shapes_and_knobs(pkg):
    N, K = 64, 512
    lin = _linear(pkg, N, K)
    cpu = torch.device("cpu")

    def patch(value, offset=None):
        lin.weight.patches = [([(1.0, value, 1.0, offset, None)], "w")]
        return lin._lycoris_terms(cpu)
    lokr = ("lokr", (torch.randn(4, 8), torch.randn(16, 64), 2.0, None, None, None, None, None, None))
    lora, kron = patch(lokr)
    assert lora == [] and len(kron[0]) == 1 and kron[1][0].a1 == 4 and kron[1][0].b2 == 64 and kron[1][0].band_dim == -1
    assert patch(lokr) == (lora, kron) and lin._lycoris_terms(cpu)[1] is kron               # built once per patch set
    assert patch(lokr, (0, 32, 64)) is None                                                   # band past N
    assert patch(("lokr", (torch.randn(2, 8), torch.randn(16, 64), None, None, None, None, None, None, None)), (0, 16, 32))[1][1][0].band_start == 16
    assert patch(("lokr", (torch.randn(4, 4), torch.randn(16, 64), None, None, None, None, None, None, None))) is None   # 4 * 64 != K
    loha = ("loha", (torch.randn(N, 2), torch.randn(2, 256), None, torch.randn(N, 3), torch.randn(3, 256), None, None, None))
    lora, kron = patch(loha, (1, 256, 256))
    assert kron is None and len(lora) == 1 and lora[0][1].shape == (N, 6) and lora[0][3] == (1, 256, 256)
    assert patch(loha) is None                                                                # 256 columns != K
    lin.patch_dtype = "target"                                                                # the reference forms the delta in another dtype
    assert patch(lokr) is None
    del lin.patch_dtype
    lin.lora_side_gemm = False
    assert patch(lokr) is None
    del lin.lora_side_gemm
    assert lin._lora_terms(cpu) is None                                                       # the LoRA recogniser is unchanged
    lin.weight.patches = []


def _kron(pkg, p16, *, qt=int(Q.Q4_K), N=8, K=256, out=None, out_dtype=0, math=0, patches=None, n=None, packed=True):
    if patches is None:
        patches = [dict()]
    L = pkg.lib.lib()
    arr = (pkg.lib.KronPatch * max(1, len(patches)))()
    for i, kw in enumerate(patches):
        d = dict(A=p16, B=p16, a1=2, a2=16, b1=4, b2=16, band_dim=-1, scale=1.0, band_start=0, band_size=0)
        d.update(kw)
        for k, v in d.items():
            setattr(arr[i], k, v)
    return L.ggufb200_dequant_kron(qt, p16 if packed else None, N, K, p16 if out is None else out, out_dtype, math,
                                   arr if patches else None, len(patches) if n is None else n, None)


def test_dequant_kron_validates_without_gpu(pkg):
    L = pkg.lib.lib()
    assert ctypes.sizeof(pkg.lib.KronPatch) == 72
    buf = (ctypes.c_uint8 * 4096)()
    p16 = (ctypes.addressof(buf) + 15) & ~15
    assert _kron(pkg, p16, qt=99) == E_TYPE
    assert _kron(pkg, p16, qt=int(Q.BF16)) == E_UNSUPPORTED
    assert _kron(pkg, p16, out_dtype=3) == E_DTYPE
    assert _kron(pkg, p16, math=3) == E_DTYPE
    assert _kron(pkg, p16, K=100) == E_SHAPE                                      # not whole blocks, not straddled
    assert _kron(pkg, p16, N=3, K=264) == E_SHAPE                                 # N * K not a multiple of 256
    assert _kron(pkg, p16, K=0) == E_SHAPE
    assert _kron(pkg, p16, N=-8) == E_SHAPE
    assert _kron(pkg, p16, patches=[dict()] * 9) == E_SHAPE                       # at most 8 patches
    assert _kron(pkg, p16, n=-1) == E_SHAPE
    assert L.ggufb200_dequant_kron(int(Q.Q4_K), p16, 8, 256, p16, 0, 0, None, 1, None) == E_NULL
    assert _kron(pkg, p16, patches=[dict(a1=4)]) == E_SHAPE                       # a1 * b1 != N
    assert _kron(pkg, p16, patches=[dict(b2=8)]) == E_SHAPE                       # a2 * b2 != K
    assert _kron(pkg, p16, patches=[dict(a1=0, b1=0)]) == E_SHAPE
    assert _kron(pkg, p16, patches=[dict(band_dim=2)]) == E_SHAPE
    assert _kron(pkg, p16, patches=[dict(band_dim=0, band_start=6, band_size=4, a1=1)]) == E_SHAPE   # band past N
    assert _kron(pkg, p16, patches=[dict(band_dim=0, band_start=0, band_size=4)]) == E_SHAPE         # 2 * 4 != 4 band rows
    assert _kron(pkg, p16, patches=[dict(band_dim=1, band_start=128, band_size=256)]) == E_SHAPE    # band past K
    assert _kron(pkg, p16, patches=[dict(band_dim=1, band_start=-1, band_size=256)]) == E_SHAPE
    assert _kron(pkg, p16, patches=[dict(A=None)]) == E_NULL
    assert _kron(pkg, p16, patches=[dict(B=None)]) == E_NULL
    assert _kron(pkg, p16, patches=[dict(A=p16 + 2)]) == E_ALIGN
    assert _kron(pkg, p16, patches=[dict(), dict(B=p16 + 1)]) == E_ALIGN                              # every patch is checked
    assert _kron(pkg, p16, out=p16 + 8) == E_ALIGN
    assert _kron(pkg, p16, packed=False) == E_NULL
    assert _kron(pkg, p16, out_dtype=1, math=1 | pkg.lib.DEQUANT_SRC_STABLE, patches=[dict(a1=0)]) == E_SHAPE   # the flag is accepted
