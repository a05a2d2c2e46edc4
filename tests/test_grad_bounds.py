"""CPU checks of the input-gradient bound of tests/grad_bounds.py: it accepts the correctly rounded product dY.W, and it
rejects each fault the backward's K1 + B_MN GEMM could plausibly make -- one k-block of N dropped in a tile, the N tail
dropped, dY's padding columns read, a 64-column box taken from the neighbouring offset, W rounded to the other 16-bit type,
the math dtype ignored, partial sums rounded to the activation dtype per k-block -- at the shapes named below, and stops
seeing it where the bound has grown past the fault (stated and shown per fault).  Also: the case list against its axes and
against the GEMM's narrow / wide tile choice."""
import functools
import math
import os

import numpy as np
import pytest
import torch

import grad_bounds as gb
import linear_bounds as lb
import oracle
from fallback_cases import FALLBACK
from util import Q

HERE = os.path.dirname(os.path.abspath(__file__))


@functools.lru_cache(maxsize=32)
def _operands(qt, M, N, K, act, math_=0):
    """(raw, dY [M, ldy] with NaN padding, dY [M, N] float64, W float64, v, a, cls) of a case, on the CPU."""
    case = gb.make_case(qt, M, N, K, act, math_)
    raw = gb.weight_bytes(case)
    W = gb.grad_weight(raw, qt, N, K, act, math_)
    dy_buf = gb.grad_dy(case)
    dy = lb.to_f64(dy_buf[:, :N])
    v, a, cls = gb.grad_reference(dy, W)
    return raw, dy_buf, dy, W, v, a, cls


def _passes(y, qt, M, N, K, act, math_=0):
    """True when the fault's float64 output, rounded once to the activation dtype, passes the bound of its case."""
    _raw, _b, _dy, _W, v, a, cls = _operands(qt, M, N, K, act, math_)
    return lb.check(lb.round_act(y, act), v, a, cls, act).ok


SMALL = [c for c in gb.CASES if c.M * c.N * c.K <= 3e7]


@pytest.mark.parametrize("case", SMALL, ids=lambda c: c.id)
def test_the_correctly_rounded_product_is_accepted(case):
    raw = gb.weight_bytes(case)
    W = gb.grad_weight(raw, case.qt, case.N, case.K, case.act, case.math)
    dy = lb.to_f64(gb.grad_dy(case)[:, :case.N])
    v, a, cls = gb.grad_reference(dy, W)
    y = lb.round_act(dy @ torch.where(torch.isfinite(W), W, torch.zeros_like(W)), case.act)
    y = torch.where(cls == lb.NAN, torch.full_like(y, float("nan")), y)
    y = torch.where(cls == lb.PINF, torch.full_like(y, float("inf")), y)
    y = torch.where(cls == lb.NINF, torch.full_like(y, float("-inf")), y)
    verdict = lb.check(y, v, a, cls, case.act, case.id)
    assert verdict.ok and verdict.used < 1e-6, verdict.message
    assert (case.edge in ("none", "subnormal_col")) == bool((cls == lb.FIN).all()), "the edge values must reach dX"


def test_it_is_the_forward_bound_with_n_as_the_reduction():
    """grad_reference(dY, W) = linear_bounds.reference(dY, W^T): v = dY.W, a = 2 N u |dY|.|W| + u |v|, classes of dY.W."""
    _raw, _b, dy, W, v, a, cls = _operands(Q.Q8_0, 65, 130, 96, lb.F16)
    assert torch.equal(v, dy @ W)
    assert torch.allclose(a, 2 * 130 * lb.U * (dy.abs() @ W.abs()) + lb.U * v.abs(), rtol=1e-14, atol=0)
    dy2, W2 = dy.clone(), W.clone()
    dy2[4, 7] = float("nan")
    W2[9, 11] = float("inf")
    _v, _a, c2 = gb.grad_reference(dy2, W2)
    assert bool((c2[4] == lb.NAN).all()), "a NaN in dY's row 4 reaches every column of dX's row 4"
    inf_col = (c2[:, 11] == lb.PINF) | (c2[:, 11] == lb.NINF)
    assert bool(inf_col[torch.arange(65) != 4].all()), "an Inf in W's column 11 reaches every other row of dX's column 11"
    assert int((c2 != lb.FIN).sum()) == 96 + 65 - 1


# ---------------------------------------------------------------- simulated faults
def _fault_dropped_kblock(qt, M, N, K, act):
    """The first 128 x 128 tile of dX misses k-block 0 (rows 0..63 of W)."""
    _raw, _b, dy, W, v, _a, _c = _operands(qt, M, N, K, act)
    y = v.clone()
    y[:128, :128] -= dy[:128, :64] @ W[:64, :128]
    return y


def _fault_dropped_tail(qt, M, N, K, act):
    """The last N % 64 rows of W (the partial k-block) never reach the product."""
    _raw, _b, dy, W, v, _a, _c = _operands(qt, M, N, K, act)
    t = N % 64
    return v - dy[:, N - t:] @ W[N - t:]


def _fault_padding_read(qt, M, N, K, act, pad_value=float("nan")):
    """dY's columns [N, ldy) read into the partial k-block; W's rows past N are zero-filled by TMA, so they multiply zeros."""
    _raw, dy_buf, dy, W, _v, _a, _c = _operands(qt, M, N, K, act)
    width = min(dy_buf.shape[1], (N + 63) // 64 * 64)
    ext = lb.to_f64(dy_buf[:, :width]).clone()
    ext[:, N:] = pad_value
    Wext = torch.cat([W, torch.zeros(width - N, K, dtype=W.dtype)])
    return ext @ Wext


def _fault_neighbour_box(qt, M, N, K, act):
    """Columns 0..63 of the first tile computed from W's columns 64..127 (the next box's offset; zero-filled past K)."""
    _raw, _b, dy, W, v, _a, _c = _operands(qt, M, N, K, act)
    Wn = torch.nn.functional.pad(W, (0, max(0, 128 - K)))
    y = v.clone()
    w = min(64, K)
    y[:128, :w] = (dy[:128] @ Wn[:, 64:128])[:, :w]
    return y


def _fault_other_type(qt, M, N, K, act):
    """W in the other 16-bit type: the fp16 chain's value kept under bf16 activations, bf16(W) under fp16 activations."""
    raw, _b, dy, W, _v, _a, _c = _operands(qt, M, N, K, act)
    if act == lb.F16:
        return dy @ lb.to_f64(W.to(torch.bfloat16))
    return dy @ gb.grad_weight(raw, qt, N, K, lb.F16, 0)


def _fault_math_ignored(qt, M, N, K, act):
    """fp32 math asked for, the fp16 chain run."""
    raw, _b, dy, _W, _v, _a, _c = _operands(qt, M, N, K, act, oracle.DT_F32)
    return dy @ gb.grad_weight(raw, qt, N, K, act, oracle.DT_F16)


def _fault_kblock_rounding(qt, M, N, K, act):
    """The fp32 accumulator rounded to the activation dtype after every 64-row k-block of N."""
    _raw, _b, dy, W, v, _a, _c = _operands(qt, M, N, K, act)
    acc = torch.zeros_like(v)
    for k in range(0, N, 64):
        acc = lb.round_act(acc + dy[:, k:k + 64] @ W[k:k + 64], act)
    return acc


# fault -> (visible shapes, invisible shapes), each (qt, M, N, K, act).  Sizes are M x N x K of dX = dY[M, N] . W[N, K].
FAULTS = {
    # a k-block moves an element by about 8 sigma (64 products); the bound grows as 1.3 N^2 u sigma: past N ~ 10^4 it is
    # wider than the largest such move over a 128 x 128 tile
    "dropped_kblock": ([(Q.Q8_0, 128, 130, 128, lb.F16), (Q.BF16, 129, 2432, 200, lb.BF16), (Q.Q8_0, 128, 8192, 128, lb.BF16)],
                       [(Q.Q8_0, 128, 16384, 128, lb.F16)]),
    # the tail of t rows moves an element by about sqrt(t) sigma: seen at every case of the list (N <= 2432, t >= 2)
    "dropped_tail": ([(Q.Q8_0, 65, 130, 96, lb.F16), (Q.BF16, 63, 72, 56, lb.BF16), (Q.BF16, 129, 200, 1000, lb.F16),
                      (Q.Q4_K, 64, 2440, 256, lb.BF16)], []),
    # NaN padding turns every element NaN at every shape; finite padding meets W's zero-filled rows and is invisible --
    # which is why the padding of dY holds NaN in every case
    "padding_read": ([(Q.Q8_0, 65, 130, 96, lb.F16), (Q.BF16, 2, 1, 8, lb.BF16), (Q.Q4_K, 127, 200, 512, lb.F16)], []),
    # another column offset shares no product with this one: seen at every shape with a non-zero box
    "neighbour_box": ([(Q.Q8_0, 65, 130, 96, lb.F16), (Q.BF16, 1, 1, 8, lb.BF16), (Q.Q4_K, 128, 2432, 256, lb.BF16)], []),
    # a relative change of up to 2^-9 per weight: under the bound from N ~ 2400 on (M = K = 128)
    "other_type": ([(Q.Q8_0, 128, 64, 128, lb.F16), (Q.Q8_0, 128, 1024, 128, lb.F16), (Q.Q8_0, 128, 200, 128, lb.BF16),
                    (Q.Q8_0, 128, 1024, 128, lb.BF16)],
                   [(Q.Q8_0, 128, 2432, 128, lb.F16), (Q.Q8_0, 128, 2432, 128, lb.BF16)]),
    # one or two fp16 ulps on some weights: seen up to N ~ 200 under fp16 activations, ~ 1000 under bf16 (Q4_K)
    "math_ignored": ([(Q.Q4_K, 128, 64, 256, lb.F16), (Q.Q4_K, 128, 200, 256, lb.F16), (Q.Q4_K, 128, 1024, 256, lb.BF16)],
                     [(Q.Q4_K, 128, 1024, 256, lb.F16), (Q.Q4_K, 128, 2432, 256, lb.BF16)]),
    # needs two k-blocks (N > 64); an fp16 rounding per k-block is seen up to N ~ 200, a bf16 one up to N ~ 8192
    "kblock_rounding": ([(Q.Q8_0, 128, 130, 128, lb.F16), (Q.Q8_0, 128, 200, 128, lb.F16), (Q.Q8_0, 128, 2432, 128, lb.BF16),
                         (Q.Q8_0, 128, 8192, 128, lb.BF16)],
                        [(Q.Q8_0, 128, 64, 128, lb.F16), (Q.Q8_0, 128, 1024, 128, lb.F16), (Q.Q8_0, 128, 16384, 128, lb.BF16)]),
}
SIMULATE = {name: globals()[f"_fault_{name}"] for name in FAULTS}
MATH = {"math_ignored": oracle.DT_F32}          # the math dtype the case asks for (default fp16)


def _shape_id(s):
    qt, M, N, K, act = s
    return f"{qt.name}-{M}x{N}x{K}-{'f16' if act == lb.F16 else 'bf16'}"


@pytest.mark.parametrize("fault,shape", [(f, s) for f, (vis, _inv) in FAULTS.items() for s in vis],
                         ids=lambda v: _shape_id(v) if isinstance(v, tuple) else v)
def test_the_fault_is_rejected(fault, shape):
    y = SIMULATE[fault](*shape)
    assert not _passes(y, *shape, MATH.get(fault, 0)), f"{fault} passes the bound at {_shape_id(shape)}"


@pytest.mark.parametrize("fault,shape", [(f, s) for f, (_vis, inv) in FAULTS.items() for s in inv],
                         ids=lambda v: _shape_id(v) if isinstance(v, tuple) else v)
def test_where_the_fault_stops_being_visible(fault, shape):
    """The stated limit: past it the fault fits inside the bound (the kernel's own rounding freedom is that large there)."""
    y = SIMULATE[fault](*shape)
    assert _passes(y, *shape, MATH.get(fault, 0)), f"{fault} is still rejected at {_shape_id(shape)}: the stated limit is out of date"


def test_finite_padding_is_invisible_which_is_why_it_holds_nan():
    shape = (Q.Q8_0, 65, 130, 96, lb.F16)
    assert _passes(_fault_padding_read(*shape, pad_value=3.0), *shape)


# ---------------------------------------------------------------- the case list
def test_case_list_covers_its_axes():
    cases = gb.CASES
    assert len({c.id for c in cases}) == len(cases)
    assert {c.M for c in cases} >= set(gb.M_ALL)
    assert {c.N for c in cases} >= set(gb.N_ALL)
    assert {c.K for c in cases if c.qt == Q.BF16} >= set(gb.K_BF16)
    assert {c.K % 64 for c in cases if c.qt == Q.BF16} == set(range(0, 64, 8)), "every residue of K mod 64 a BF16 weight allows"
    assert {c.K for c in cases if c.qt in (Q.Q8_0, Q.Q4_0)} >= set(gb.K_32)
    for t in gb.TABLE12:
        assert {(c.act, c.math) for c in cases if c.qt == t and c.edge == "none"} >= {(a, m) for a in (lb.F16, lb.BF16) for m in gb.MATHS}, t
    for t in FALLBACK:
        assert {c.act for c in cases if c.qt == t} == {lb.F16, lb.BF16}, t
    assert {c.weight for c in cases if c.qt == Q.BF16} == {"in_place", "workspace"}
    for t in (Q.Q2_K, Q.Q3_K, Q.Q4_K, Q.Q5_K, Q.Q6_K):
        assert {(c.N, c.K) for c in cases if c.qt == t and c.straddled} >= set(gb.STRADDLED), t
    assert any(c.straddled for c in cases if c.qt in FALLBACK)
    assert {(c.qt, c.N, c.K) for c in cases if c.M == 4096} >= {(t, N, K) for t in (Q.Q4_K, Q.Q8_0) for N, K in gb.FLUX}
    assert set(gb.EDGES) == {c.edge for c in cases}
    for c in cases:
        bs = gb.block_size(c.qt)
        assert c.K % 8 == 0 and (c.N * c.K) % bs == 0, c.id
        assert c.straddled == (c.K % bs != 0)
        assert c.qt in FALLBACK or not c.straddled or (bs == 256 and c.N * c.K % 256 == 0), c.id
        assert c.ldy > c.N and c.ldy % 8 == 0 and c.ldx > c.K and c.ldx % 8 == 0, c.id
        assert c.weight == ("in_place" if c.qt == Q.BF16 and c.act == lb.BF16 else "workspace"), c.id


def test_the_tile_predicate_is_the_kernels():
    """narrow_tile restates dense_gemm_nn's choice; the source line it restates must still be there."""
    with open(os.path.join(HERE, "..", "comfyui-gguf_b200", "csrc", "linear_sm90.cu")) as f:
        src = f.read()
    assert "const bool narrow = ((M + 127) / 128) * ((Kout + 255) / 256) < sm_count();" in src
    assert gb.narrow_tile(128, 256, 2) and not gb.narrow_tile(129, 256, 2) and not gb.narrow_tile(128, 257, 2)


@pytest.mark.parametrize("sms", [132, 114, 78, 7])
def test_switch_cases_sit_on_either_side_of_the_switch(sms):
    below, at = gb.switch_cases(sms, lb.BF16)
    for c, tiles in ((below, sms - 1), (at, sms)):
        assert math.ceil(c.M / 128) * math.ceil(c.K / 256) == tiles, (sms, c.id)
        assert c.K % 8 == 0 and c.M % 128 != 0 and c.K % 256 != 0 and c.K > 128, c.id
    assert gb.narrow_tile(below.M, below.K, sms) and not gb.narrow_tile(at.M, at.K, sms)


def test_the_list_reaches_partial_tiles_of_both_widths():
    """On a 132-SM H100 (SXM) the list alone has narrow and wide launches whose last tile column is partial."""
    narrow = [c for c in gb.CASES if gb.narrow_tile(c.M, c.K, 132)]
    wide = [c for c in gb.CASES if not gb.narrow_tile(c.M, c.K, 132)]
    assert any(c.K % 128 and c.K > 128 for c in narrow)
    assert any(c.K % 256 and c.K > 256 for c in wide)
    assert any(c.M % 128 and c.M > 128 for c in narrow) and any(c.M % 128 for c in wide)
