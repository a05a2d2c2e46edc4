"""CPU tests of DoRA (weight-decomposed LoRA) patches on a packed weight: the recogniser and its rejections, the axis rule, the
compact form of the patched weight against a float64 replay of the reference's sequence, the plan's route decision, and
argument validation of the three entry points the route adds, without a device.

The reference's sequence (ComfyUI `weight_decompose`, restated in ops.dora_replay) for one entry with strength st on the
running weight W:
    Wc = W + (delta * alpha).to(W.dtype)
    nrm = W's row norms (dora_scale [N, 1], output axis; the weight BEFORE this patch) or Wc's column norms (input axis) + eps
    s = (fp32(dora_scale) / nrm).to(W.dtype);  Wc *= s;  W = Wc if st == 1 else W + st * (Wc - W)"""
import ctypes
import os
import re

import pytest
import torch

import oracle
from util import Q

E_TYPE, E_DTYPE, E_ALIGN, E_SHAPE, E_NULL, E_UNSUPPORTED = -1, -2, -3, -4, -5, -8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


class LoKrAdapter(LoRAAdapter):
    pass


def _m(*shape):
    return torch.ones(*shape)


def _lora(N, K, r, g, alpha=None, dora=None):
    up, down = torch.randn(N, r, generator=g) * 0.2, torch.randn(r, K, generator=g) * 0.2
    return ("lora", (up, down, alpha, None, dora, None))


def _loha(N, K, d, g, alpha=None, dora=None):
    f = [torch.randn(*s, generator=g) * 0.3 for s in ((N, d), (d, K), (N, d), (d, K))]
    return ("loha", (f[0], f[1], alpha, f[2], f[3], None, None, dora))


def test_recogniser_accepts_dora_lists(pkg):
    f = pkg.ops.dora_terms
    up, down, ds = _m(8, 2), _m(2, 16), _m(8, 1)
    plain = (1.0, ("lora", (up, down, 4.0, None, None, None)), 1.0, None, None)
    dora = (0.5, LoRAAdapter((up, down, None, None, ds, None)), 1.0)
    loha = (0.8, ("loha", (_m(8, 3), _m(3, 16), 6.0, _m(8, 1), _m(1, 16), None, None, _m(1, 16))), 1.0, None, None)
    terms = f([plain, dora, loha])
    assert [t[0] for t in terms] == ["lora", "lora", "loha"]
    assert terms[0][1:3] == (1.0, 2.0) and terms[0][4] is None                     # alpha / rank, kept apart from the strength
    assert terms[1][1:3] == (0.5, 1.0) and terms[1][4] is ds                       # no alpha -> 1
    assert terms[2][1:3] == (0.8, 2.0) and terms[2][3][0].shape == (8, 3)          # LoHa: alpha / w1b.shape[0]
    assert f([dora]) is not None and f([loha]) is not None
    assert f([plain]) is None                                                     # no DoRA entry: the LoRA recogniser's list
    # the existing recognisers keep refusing DoRA
    assert pkg.ops.lora_band_terms([dora]) is None and pkg.ops.lycoris_terms([loha]) is None


def test_recogniser_rejects_what_needs_calculate_weight(pkg):
    f = pkg.ops.dora_terms
    up, down, ds = _m(8, 2), _m(2, 16), _m(8, 1)
    lora = ("lora", (up, down, None, None, ds, None))
    assert f([(1.0, lora, 0.7)]) is None                                                            # strength_model
    assert f([(1.0, lora, 1.0, None, lambda w: w)]) is None                                         # function hook
    assert f([(1.0, lora, 1.0, (0, 0, 8), None)]) is None                                           # offset (banded DoRA)
    assert f([(1.0, ("lora", (up, down, None, _m(2, 2), ds, None)), 1.0)]) is None                  # LoCon mid
    assert f([(1.0, ("lora", (up, down, None, None, ds, (8, 16))), 1.0)]) is None                   # reshape
    assert f([(1.0, ("lora", (torch.ones(8, 2, 1, 1), down, None, None, ds, None)), 1.0)]) is None  # conv factor
    assert f([(1.0, ("lora", (up, _m(3, 16), None, None, ds, None)), 1.0)]) is None                 # does not chain
    assert f([(1.0, ("lora", (up, down, None, None, [1.0], None)), 1.0)]) is None                   # not a tensor
    loha = (_m(8, 3), _m(3, 16), None, _m(8, 1), _m(1, 16))
    assert f([(1.0, ("loha", loha + (_m(3, 3), None, ds)), 1.0)]) is None                           # Tucker t1
    assert f([(1.0, ("loha", loha + (None, _m(1, 1), ds)), 1.0)]) is None                           # Tucker t2
    assert f([(1.0, ("loha", (_m(8, 3), _m(2, 16)) + loha[2:] + (None, None, ds)), 1.0)]) is None   # does not chain
    lokr = (_m(2, 4), _m(4, 4), None, None, None, None, None, None, ds)
    assert f([(1.0, ("lokr", lokr), 1.0)]) is None                                                  # LoKr + DoRA
    assert f([(1.0, LoKrAdapter(lokr), 1.0)]) is None
    assert f([(1.0, lora, 1.0), (1.0, ("diff", (_m(8, 16),)), 1.0)]) is None                        # another kind in the list
    assert f([(1.0, lora, 1.0), (1.0, ("lokr", lokr[:8] + (None,)), 1.0)]) is None


def test_axis_follows_the_reference_rule(pkg):
    axis = pkg.ops.dora_axis
    assert axis(_m(64, 1), 64, 128) == 0 and axis(_m(1, 128), 64, 128) == 1 and axis(_m(128), 64, 128) == 1
    assert axis(_m(64, 1), 64, 64) == 0 and axis(_m(1, 64), 64, 64) == 1          # square: dora_scale.shape[0] decides
    assert axis(_m(64), 64, 128) is None                                            # [N]: the reference broadcasts to [N, N]
    assert axis(_m(64), 64, 64) is None
    assert axis(_m(128, 1), 64, 128) is None and axis(_m(1, 64), 64, 128) is None and axis(_m(64, 2), 64, 128) is None


def _replay64(W0, terms, factors):
    """The reference's sequence in float64 with the given DoRA factors s (never rounded)."""
    W = W0.double().clone()
    N = W.shape[0]
    for (kind, st, a, fac, ds), s in zip(terms, factors):
        f = [t.double() for t in fac]
        delta = f[0] @ f[1] if kind == "lora" else (f[0] @ f[1]) * (f[2] @ f[3])
        if ds is None:
            W += st * a * delta
            continue
        Wc = W + a * delta
        Wc = Wc * (s.double()[:, None] if ds.shape[0] == N else s.double()[None, :])
        W = W + st * (Wc - W)
    return W


def _compact64(W0, terms, r, c, compact):
    W = r[:, None] * W0.double() * c[None, :]
    for (kind, _st, _a, fac, _ds), (coef, rho, gamma) in zip(terms, compact):
        f = [t.double() for t in fac]
        delta = f[0] @ f[1] if kind == "lora" else (f[0] @ f[1]) * (f[2] @ f[3])
        if rho is not None:
            delta = rho[:, None] * delta
        if gamma is not None:
            delta = delta * gamma[None, :]
        W += coef * delta
    return W


def _lists(N, K, g):
    """Mixed lists: DoRA then LoRA, LoRA then DoRA, two DoRA entries on different axes, LoHa + DoRA, strengths != 1."""
    def ds_out():
        return torch.rand(N, 1, generator=g) * 2 + 0.5

    def ds_in():
        return torch.rand(1, K, generator=g) * 2 + 0.5
    return {
        "dora_then_lora": [(1.0, _lora(N, K, 4, g, 2.0, ds_out()), 1.0), (0.7, _lora(N, K, 8, g, 4.0), 1.0)],
        "lora_then_dora": [(0.9, _lora(N, K, 8, g, 4.0), 1.0), (1.0, _lora(N, K, 4, g, None, ds_in()), 1.0)],
        "two_axes": [(0.8, _lora(N, K, 4, g, 2.0, ds_out()), 1.0), (1.2, LoRAAdapter(_lora(N, K, 6, g, 3.0, ds_in().reshape(K))[1]), 1.0)],
        "loha_dora": [(0.6, _loha(N, K, 3, g, 1.5, ds_out()), 1.0), (1.0, _lora(N, K, 4, g, 2.0), 1.0),
                      (0.8, LoHaAdapter(_loha(N, K, 2, g, None, ds_in())[1]), 1.0)],
        "strength": [(0.8, _lora(N, K, 4, g, 2.0, ds_in()), 1.0), (0.5, _lora(N, K, 4, g, 2.0, ds_out()), 1.0),
                     (1.3, _lora(N, K, 4, g, 8.0, ds_out()), 1.0)],
    }


@pytest.mark.parametrize("name", ["dora_then_lora", "lora_then_dora", "two_axes", "loha_dora", "strength"])
def test_compact_form_is_the_reference_weight(pkg, name):
    N, K = 48, 80
    g = torch.Generator().manual_seed(len(name))
    entries = _lists(N, K, g)[name]
    terms = pkg.ops.dora_terms(entries)
    assert terms is not None and all(t[4] is None or pkg.ops.dora_axis(t[4], N, K) is not None for t in terms)
    W0 = torch.randn(N, K, generator=g) * 0.1
    factors, patched = pkg.ops.dora_replay(W0, terms)
    assert [s is None for s in factors] == [t[4] is None for t in terms]
    r, c, compact = pkg.ops.dora_compact(terms, factors, N, K)
    want = _replay64(W0, terms, factors)
    # the algebra itself: the compact form with the same s equals the float64 replay up to float64 rounding
    assert float((_compact64(W0, terms, r, c, compact) - want).norm() / want.norm()) < 1e-12
    # the fp32 replay (the reference's own arithmetic) is the same weight up to fp32 rounding
    assert float((patched.double() - want).norm() / want.norm()) < 1e-5
    # the factors are the reference's: s recomputed in float64 from the float64 running weight differs by fp32 rounding only
    W = W0.double()
    for (kind, st, a, fac, ds), s in zip(terms, factors):
        f = [t.double() for t in fac]
        delta = a * (f[0] @ f[1] if kind == "lora" else (f[0] @ f[1]) * (f[2] @ f[3]))
        if ds is None:
            W = W + st * delta
            continue
        Wc = W + delta
        out = ds.shape[0] == N
        nrm = (W.norm(dim=1) if out else Wc.norm(dim=0)) + torch.finfo(torch.float32).eps
        s64 = ds.double().reshape(-1) / nrm
        assert float(((s.double() - s64).abs() / s64).max()) < 1e-5
        Wc = Wc * (s64[:, None] if out else s64[None, :])
        W = W + st * (Wc - W)
    # the plan's operands compose back to the same weight: r W0 c + up @ down
    plan = pkg.ops.build_dora_plan(W0, terms, torch.float32)
    assert plan.r.dtype == torch.float32 and plan.r.shape == (N,)
    has_in = any(t[4] is not None and t[4].shape[0] != N for t in terms)
    assert (plan.c is not None) == has_in
    c_plan = plan.c.double() if plan.c is not None else torch.ones(K, dtype=torch.float64)
    got = plan.r.double()[:, None] * W0.double() * c_plan[None, :] + plan.up.double() @ plan.down.double()
    assert float((got - want).norm() / want.norm()) < 1e-5
    assert plan.kernel is not None
    down_pad, u_pad = plan.kernel
    R = plan.down.shape[0]
    assert u_pad.dtype == torch.float16 and torch.equal(down_pad[:R], plan.down)
    assert torch.allclose((u_pad[:, :R].double() * plan.r.double()[:, None]), plan.up.double(), rtol=2e-3, atol=1e-6)


def test_fp16_replay_matches_the_reference_ops(pkg):
    """In fp16 the factors are the fp16 quotient of the fp32 dora_scale by the fp16 norm + fp16 eps, as the reference forms them."""
    N, K = 32, 64
    g = torch.Generator().manual_seed(3)
    ds = torch.rand(N, 1, generator=g) + 0.5
    entries = [(1.0, _lora(N, K, 4, g, 2.0, ds), 1.0)]
    terms = pkg.ops.dora_terms(entries)
    W = (torch.randn(N, K, generator=g) * 0.1).half()
    (s,), patched = pkg.ops.dora_replay(W, terms)
    nrm = W.reshape(N, -1).norm(dim=1, keepdim=True) + torch.finfo(torch.float16).eps
    assert s.dtype == torch.float16 and torch.equal(s, (ds / nrm).half().reshape(-1))
    delta = (terms[0][3][0] @ terms[0][3][1]) * 2.0 / 4
    assert torch.equal(patched, (W + delta.half()) * (ds / nrm).half())


def test_zero_row_factor_sends_the_plan_to_the_side_form(pkg):
    N, K = 32, 64
    g = torch.Generator().manual_seed(5)
    ds = torch.rand(N, 1, generator=g) + 0.5
    ds[3] = 0.0                                                       # s = 0 on row 3: r_3 = 1 - st + st * 0 = 0 at st = 1
    terms = pkg.ops.dora_terms([(1.0, _lora(N, K, 4, g, None, ds), 1.0)])
    W0 = torch.randn(N, K, generator=g) * 0.1
    plan = pkg.ops.build_dora_plan(W0, terms, torch.float32)
    assert plan.r[3] == 0 and plan.kernel is None
    want = _replay64(W0, terms, pkg.ops.dora_replay(W0, terms)[0])
    got = plan.r.double()[:, None] * W0.double() + plan.up.double() @ plan.down.double()
    assert float((got - want).norm() / want.norm()) < 1e-5
    # rank above 512 also takes the side form
    big = pkg.ops.dora_terms([(1.0, _lora(N, K, 520, g, None, ds.abs() + 1), 1.0)])
    assert pkg.ops.build_dora_plan(W0, big, torch.float32).kernel is None


def _linear(pkg, N, K):
    raw = oracle.random_blocks(int(Q.Q4_K), N * K // 256, seed=3).reshape(N, K // 256 * 144)
    lin = pkg.ops.GGMLOps.Linear(K, N)
    lin.load_state_dict({"weight": pkg.ops.GGMLTensor(torch.from_numpy(raw), tensor_type=Q.Q4_K, tensor_shape=torch.Size((N, K)))})
    return lin


def test_layer_checks_shapes_and_knobs(pkg):
    N, K = 64, 512
    lin = _linear(pkg, N, K)
    g = torch.Generator().manual_seed(1)

    def patch(*entries):
        lin.weight.patches = [(list(entries), "w")]
        return lin._dora_terms()
    assert len(patch((1.0, _lora(N, K, 4, g, None, _m(N, 1)), 1.0))) == 1
    assert len(patch((1.0, _lora(N, K, 4, g, None, _m(1, K)), 1.0), (1.0, _loha(N, K, 2, g), 1.0))) == 2
    assert patch((1.0, _lora(N, K, 4, g, None, _m(N)), 1.0)) is None                  # [N]: not one factor per row
    assert patch((1.0, _lora(N, K, 4, g, None, _m(K, 1)), 1.0)) is None
    assert patch((1.0, _lora(N, 256, 4, g, None, _m(N, 1)), 1.0)) is None               # factors of another shape
    assert patch((1.0, _lora(32, K, 4, g, None, _m(N, 1)), 1.0)) is None
    ok = (1.0, _lora(N, K, 4, g, None, _m(N, 1)), 1.0)
    lin.patch_dtype = "target"                                                          # the reference forms the delta in another dtype
    assert patch(ok) is None
    del lin.patch_dtype
    lin.lora_side_gemm = False
    assert patch(ok) is None
    del lin.lora_side_gemm
    assert lin._lora_terms(torch.device("cpu")) is None and lin._lycoris_terms(torch.device("cpu")) is None   # unchanged recognisers
    lin.weight.patches = []


def _buf():
    buf = (ctypes.c_uint8 * 8192)()
    return buf, (ctypes.addressof(buf) + 15) & ~15


def test_scale_columns_validates_without_gpu(pkg):
    L = pkg.lib.lib()
    _keep, p = _buf()
    assert L.ggufb200_scale_columns(p, 4, 64, 64, 2, p, p + 1024, 64, None) == E_DTYPE        # fp32 activations
    assert L.ggufb200_scale_columns(p, 4, 60, 64, 0, p, p + 1024, 64, None) == E_SHAPE        # K % 8
    assert L.ggufb200_scale_columns(p, 4, 0, 64, 0, p, p + 1024, 64, None) == E_SHAPE
    assert L.ggufb200_scale_columns(p, -1, 64, 64, 0, p, p + 1024, 64, None) == E_SHAPE
    assert L.ggufb200_scale_columns(p, 4, 64, 56, 0, p, p + 1024, 64, None) == E_SHAPE        # ldx < K
    assert L.ggufb200_scale_columns(p, 4, 64, 64, 0, p, p + 1024, 56, None) == E_SHAPE        # ldy < K
    assert L.ggufb200_scale_columns(p, 0, 64, 64, 0, None, None, 64, None) == 0               # nothing to do
    assert L.ggufb200_scale_columns(None, 4, 64, 64, 0, p, p + 1024, 64, None) == E_NULL
    assert L.ggufb200_scale_columns(p, 4, 64, 64, 0, None, p + 1024, 64, None) == E_NULL
    assert L.ggufb200_scale_columns(p, 4, 64, 64, 0, p, None, 64, None) == E_NULL
    assert L.ggufb200_scale_columns(p + 8, 4, 64, 64, 0, p, p + 1024, 64, None) == E_ALIGN
    assert L.ggufb200_scale_columns(p, 4, 64, 64, 0, p + 4, p + 1024, 64, None) == E_ALIGN    # col_scale: 16-byte vectors
    assert L.ggufb200_scale_columns(p, 4, 64, 64, 1, p, p + 1032, 64, None) == E_ALIGN
    assert L.ggufb200_scale_columns(p, 4, 64, 68, 1, p, p + 1024, 64, None) == E_ALIGN        # ldx % 8


def test_gemm_scaled_validates_without_gpu(pkg):
    L = pkg.lib.lib()
    _keep, p = _buf()
    args = dict(W=p, N=64, K=64, ldw=64, X=p, M=4, ldx=64, act=0, bias=None, bias_dtype=0, scale=p + 4096, Y=p + 2048, ldy=64)

    def call(**kw):
        a = dict(args, **kw)
        return L.ggufb200_gemm_scaled(a["W"], a["N"], a["K"], a["ldw"], a["X"], a["M"], a["ldx"], a["act"], a["bias"], a["bias_dtype"],
                                      a["scale"], a["Y"], a["ldy"], None)
    assert call(act=2) == E_DTYPE
    assert call(bias=p, bias_dtype=3) == E_DTYPE
    assert call(K=60) == E_SHAPE and call(ldw=32) == E_SHAPE and call(M=-1) == E_SHAPE
    assert call(M=0) == 0
    assert call(W=None) == E_NULL
    assert call(scale=p + 4100) == E_ALIGN                            # feature_scale: 16-byte aligned
    assert call(scale=p + 4100, act=2) == E_DTYPE                     # dtype checked first, as in ggufb200_gemm
    assert call(Y=p + 2050) == E_ALIGN


def test_linear_lora_scaled_validates_without_gpu(pkg):
    L = pkg.lib.lib()
    _keep, p = _buf()
    N, K = 64, 256

    def call(scale, algo=pkg.lib.ALGO_FUSED_TMEM, kblocks=1, T=p, qt=int(Q.Q4_K)):
        return L.ggufb200_linear_lora_scaled(qt, p, None, N, K, p, 4, K, 0, None, 0, T, 64, p, 64, kblocks, None, scale, p, N, None, 0,
                                             algo, None)
    assert call(p + 4) == E_ALIGN                                     # a misaligned feature scale
    assert call(p + 4, kblocks=9) == E_SHAPE                          # LoRA operands checked first
    assert call(p + 4, T=None) == E_NULL
    assert call(p, algo=pkg.lib.ALGO_DEQUANT_MMA) == E_UNSUPPORTED    # only FUSED_TMEM carries the LoRA k-blocks
    assert call(None, algo=pkg.lib.ALGO_DEQUANT_MMA) == E_UNSUPPORTED
    assert call(p, qt=99) == E_TYPE


def _prototype(header, name):
    m = re.search(r"\b" + name + r"\s*\(([^;]*)\)\s*;", header)
    assert m, name
    return [a.strip() for a in m.group(1).split(",")]


def test_header_and_binding_agree(pkg):
    header = open(os.path.join(ROOT, "include", "ggufb200.h")).read()
    assert re.search(r"#define\s+GGUFB200_VERSION\s+200\b", header)
    L = pkg.lib.lib()
    for name, scale_at in (("ggufb200_linear_lora_scaled", 17), ("ggufb200_gemm_scaled", 10), ("ggufb200_scale_columns", 5)):
        args = _prototype(header, name)
        assert name in pkg.lib.EXPORTS and len(getattr(L, name).argtypes) == len(args), name
        assert re.match(r"const float \*\s*(feature|col)_scale$", args[scale_at]), (name, args[scale_at])
    # the scaled calls are the unscaled ones plus the scale argument
    lora_ex, scaled = _prototype(header, "ggufb200_linear_lora_ex"), _prototype(header, "ggufb200_linear_lora_scaled")
    assert scaled[:17] + scaled[18:] == lora_ex
    gemm, gemm_s = _prototype(header, "ggufb200_gemm"), _prototype(header, "ggufb200_gemm_scaled")
    assert gemm_s[:10] + gemm_s[11:] == gemm
