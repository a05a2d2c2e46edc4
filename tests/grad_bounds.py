"""Per-element error bound of the packed Linear's input gradient (ggufb200_linear_grad_input: dX[M, K] = dY[M, N] . W[N, K]),
the weight it must use and its shape / type case list.

No GPU here: tests/test_grad_bounds.py checks these helpers on the CPU, tests/test_gpu_grad_bounds.py applies them to the
C ABI and to the layer's backward.

The bound is the forward's (tests/linear_bounds.py) with the roles renamed: x -> dY, W -> W^T, and the reduction runs over N
instead of K.  It carries over unchanged because the backward has less arithmetic than any forward route:
  * no bias and no split-K: the dense GEMM's B_MN mode runs every k-block of N in one CTA and writes the tile once, so the
    fp32 chain is the tensor-core steps alone, at most N steps that combine non-zero products (at most N + 2 with the
    forward's bias and finalize terms, which are absent), inside c N u (|dY|.|W|) with c = 2 for N >= 2; at N = 1 the single
    product is exact in fp32;
  * one fp32 -> act rounding in the epilogue, covered by rounding the interval ends once (`round_act`) plus u |v|;
  * TMA's zero fill past N (dY's columns, W's rows) and past K (W's columns) adds exact zeros: products of zeros, and
    tensor-core steps whose terms are all zero, leave the accumulator as it is.
So with v = dY.W exactly (float64), a = 2 N u (|dY|.|W|) + u |v|, every element of dX lies in [rnd(v - a), rnd(v + a)], and
its NaN / Inf class is that of the float64 product (`linear_bounds.classes` on dY and W^T)."""
import math as _math
from dataclasses import dataclass

import gguf
import numpy as np
import torch

import fallback_cases
import linear_bounds as lb
import oracle
from fallback_cases import FALLBACK
from util import Q

F16, BF16 = lb.F16, lb.BF16
MATHS = (oracle.DT_F16, oracle.DT_BF16, oracle.DT_F32)


def grad_reference(dy, W):
    """(v, a, cls) of dX = dY.W for float64 dY [M, N] and W [N, K] on any device: `linear_bounds.reference(dy, W^T)`, so the
    reduction length of the bound is N (module docstring)."""
    return lb.reference(dy, W.t().contiguous())


# ---------------------------------------------------------------- the weight the kernel must use
def grad_weight(raw, qt, N, K, act, math):
    """The exact [N, K] weight of the backward as float64 (CPU): what the reference's F.linear saved, W = dequantize_tensor(w,
    act dtype, dequant dtype).
      * the 12 table types: the oracle's chain in the math dtype, then the activation dtype (one flat stream, so rows that
        start inside a block -- straddled rows -- come out right);
      * the 11 numpy-fallback types: gguf-py's fp32 values rounded once to the activation dtype (math is ignored);
      * BF16: the stored bf16 values cast to the activation dtype (under fp16 activations K1 turns values past 65504 into
        Inf, as the cast does)."""
    raw = np.ascontiguousarray(raw).reshape(-1)
    qt = Q(qt)
    if qt == Q.BF16:
        w = torch.from_numpy(raw.view(np.int16).copy()).view(torch.bfloat16).to(lb.TORCH_ACT[act])
    elif qt in FALLBACK:
        w = fallback_cases.reference_tensor(raw, qt, act)
    else:
        bits = oracle.dequant(raw, int(qt), act, math)
        w = torch.from_numpy(bits.view(np.int16).copy()).view(lb.TORCH_ACT[act])
    return lb.to_f64(w).reshape(N, K)


def block_size(qt):
    return gguf.GGML_QUANT_SIZES[Q(qt)][0]


def narrow_tile(M, K, sms):
    """dense_gemm_nn's tile choice (csrc/linear_sm90.cu), restated: 128-wide output tiles when the 256-wide ones (128 rows
    of dX each) number fewer than the SMs, else 256-wide."""
    return _math.ceil(M / 128) * _math.ceil(K / 256) < sms


# ---------------------------------------------------------------- case list
TABLE12 = list(lb.ALL12)
M_ALL = (1, 2, 63, 64, 65, 127, 128, 129, 255, 1000, 4097)
N_ALL = (1, 8, 56, 64, 72, 130, 136, 200, 2432)
K_BF16 = (8, 56, 72, 200, 1000, 16, 24, 96, 40, 112, 64)     # with 1000 and 200: every residue of K mod 64 (multiples of 8)
K_32 = (96, 1056)                                            # 32-element blocks: K % 64 = 32, one partial box / tile
K_256 = (256, 512, 1280)
K_FALLBACK = (256, 512, 768)
STRADDLED = ((264, 320), (640, 320), (320, 640))
FLUX = ((3072, 12288), (12288, 3072))
EDGES = ("none", "bf16_overflow", "subnormal_col", "nonfinite_scales", "nonfinite_dy")


@dataclass(frozen=True)
class GradCase:
    qt: Q
    M: int
    N: int
    K: int
    act: int
    math: int           # the dequant's math dtype code (ignored by the fallback types and BF16)
    ldy: int            # dY's row pitch in elements, > N: columns [N, ldy) hold NaN
    ldx: int            # dX's row pitch, > K: columns [K, ldx) must come back untouched
    weight: str         # "in_place" (BF16 weight, bf16 activations: W's bytes are the operand) or "workspace" (K1 first)
    edge: str = "none"

    @property
    def straddled(self):
        """Blocks start inside rows (K % block size != 0): the weight is one flat block stream."""
        return self.K % block_size(self.qt) != 0

    @property
    def id(self):
        act = "f16" if self.act == F16 else "bf16"
        e = "" if self.edge == "none" else f"-{self.edge}"
        return f"{self.qt.name}-{self.M}x{self.N}x{self.K}-{act}-m{self.math}-ldy{self.ldy}-ldx{self.ldx}{e}"


def make_case(qt, M, N, K, act, math=0, edge="none", i=0):
    """A GradCase with dY / dX pitches 8, 16 or 24 elements past the row (by i), and the weight path the ABI takes."""
    qt = Q(qt)
    pad = 8 * (1 + i % 3)
    weight = "in_place" if qt == Q.BF16 and act == BF16 else "workspace"
    return GradCase(qt, M, N, K, act, math, (N + 7) // 8 * 8 + pad, K + pad, weight, edge)


_Cycle = lb._Cycle


def _cases():
    cases = []
    m, n = _Cycle(M_ALL, 11), _Cycle(N_ALL, 12)
    k32, k256, kfb = _Cycle(K_32, 13), _Cycle(K_256, 14), _Cycle(K_FALLBACK, 15)

    def add(*args, **kw):
        cases.append(make_case(*args, i=len(cases), **kw))
    # the 12 table types, both activation dtypes, the three math dtypes
    for t in TABLE12:
        for act in (F16, BF16):
            for math in MATHS:
                add(t, m(), n(), k32() if block_size(t) == 32 else k256(), act, math)
    # the 11 fallback types, both activation dtypes
    for t in FALLBACK:
        for act in (F16, BF16):
            add(t, m(), n(), kfb(), act, MATHS[len(cases) % 3])
    # BF16 weights: every K (every residue mod 64), bf16 read in place and fp16 through K1
    for K in K_BF16:
        for act in (F16, BF16):
            add(Q.BF16, m(), n(), K, act, MATHS[len(cases) % 3])
    # straddled rows: Q2_K .. Q6_K at the SD1.5 / SDXL shapes, and two fallback types whose blocks straddle rows
    act = _Cycle((F16, BF16), 17)
    for t in (Q.Q2_K, Q.Q3_K, Q.Q4_K, Q.Q5_K, Q.Q6_K):
        for N, K in STRADDLED:
            add(t, m(), N, K, act(), MATHS[len(cases) % 3])
    add(Q.IQ2_XS, 300, 264, 320, F16)
    add(Q.TQ2_0, 77, 640, 320, BF16)
    # wide (256-column) launches whose last tile column is partial, on any H100
    add(Q.BF16, 4097, 200, 1000, F16)
    add(Q.Q8_0, 4097, 136, 1056, BF16, oracle.DT_F32)
    # Flux.1 scale: full-size weights at 4096 tokens
    for t in (Q.Q4_K, Q.Q8_0):
        for j, (N, K) in enumerate(FLUX):
            add(t, 4096, N, K, (F16, BF16)[j], oracle.DT_F16)
    # edge values
    add(Q.BF16, 65, 130, 200, F16, edge="bf16_overflow")
    add(Q.BF16, 129, 8, 72, F16, edge="subnormal_col")
    add(Q.BF16, 2, 64, 1000, F16, edge="subnormal_col")
    add(Q.Q8_0, 127, 136, 1056, F16, edge="nonfinite_scales")
    add(Q.Q8_0, 255, 200, 1056, BF16, oracle.DT_F32, edge="nonfinite_scales")
    add(Q.Q4_K, 64, 264, 320, BF16, edge="nonfinite_scales")
    add(Q.IQ2_XS, 129, 72, 2048, F16, edge="nonfinite_scales")
    add(Q.Q4_0, 255, 200, 1056, BF16, oracle.DT_BF16, edge="nonfinite_dy")
    add(Q.BF16, 63, 72, 56, BF16, edge="nonfinite_dy")
    add(Q.Q6_K, 1000, 130, 512, F16, edge="nonfinite_dy")
    return cases


CASES = _cases()


def switch_cases(sms, act):
    """Two BF16 cases on either side of dense_gemm_nn's narrow / wide switch on an `sms`-SM device: 256-wide tiles numbering
    sms - 1 (narrow, the last tile row and column partial) and exactly sms (wide)."""
    out = []
    for tiles in (sms - 1, sms):
        f = max(d for d in range(1, 9) if tiles % d == 0)     # tiles = ceil(M / 128) * ceil(K / 256)
        t = tiles // f
        out.append(make_case(Q.BF16, 128 * t - 37, 136, 256 * f - 56, act, i=len(out)))
    return out


# ---------------------------------------------------------------- operands
NAN16, PINF16, NINF16 = 0x7E00, 0x7C00, 0xFC00


def _seed(case):
    return (int(case.qt) * 7919 + case.M * 131 + case.N * 31 + case.K + case.act) % 100003


def weight_bytes(case):
    """The packed bytes of the case's [N, K] weight (flat uint8): seeded random blocks with finite scales of about 0.02 (every
    |dX| stays far inside the fp16 range), then the case's edge values."""
    qt, N, K = case.qt, case.N, case.K
    bs = block_size(qt)
    seed = _seed(case)
    if qt in FALLBACK:
        blocks = fallback_cases.random_blocks(qt, N * K // bs, seed=seed, scale=0.02)
    else:
        blocks = oracle.random_blocks(int(qt), N * K // bs, seed=seed, scale=0.02)
    if case.edge == "bf16_overflow":
        w = blocks.reshape(-1).view(np.uint16).reshape(N, K)
        w[3, 17] = 0x4789          # 70144: past 65504, Inf in fp16
        w[N - 1, K - 1] = 0xC7C3   # -99840
    elif case.edge == "subnormal_col":
        w = blocks.reshape(-1).view(np.uint16).reshape(N, K)
        w[:, 5] = _bf16_subnormals(N, np.random.default_rng(seed))
    elif case.edge == "nonfinite_scales":
        _poison_scales(blocks, case)
    return blocks.reshape(-1)


def _bf16_subnormals(n, rng):
    """n bf16 bit patterns of random sign in [2^-17, 2^-15): 8-bit mantissas on a 2^-24 grid, so every one is an fp16
    subnormal exactly (a flush to zero anywhere in K1 or the MMA shows in that column of dX)."""
    exps = rng.integers(127 - 17, 127 - 15, size=n)          # 2^-17 <= |w| < 2^-15
    mant = rng.integers(0, 128, size=n)
    sign = rng.integers(0, 2, size=n)
    return ((sign << 15) | (exps << 7) | mant).astype(np.uint16)


def nonfinite_blocks(case):
    """(block index, fp16 scale pattern) pairs of a nonfinite_scales case: the last block (last row of W, last column box of
    dX), the first block of the last row and one in the middle of row 3 -- three column ranges of dX, the others stay
    finite.  Straddled rows: the middle block only (one block reaches 256 columns)."""
    bs = block_size(case.qt)
    nb = case.N * case.K // bs
    if case.straddled:
        return [(nb // 2, PINF16)]
    per_row = case.K // bs
    return list(zip((nb - 1, (case.N - 1) * per_row, 3 * per_row + per_row // 2), (PINF16, NAN16, NINF16)))


def _poison_scales(blocks, case):
    for b, bits in nonfinite_blocks(case):
        if case.qt in FALLBACK:
            fallback_cases._set_f16_scale(blocks[b:b + 1], case.qt, [bits])
        else:
            assert case.qt in (Q.Q8_0, Q.Q4_K), case.qt      # d is the block's first field
            blocks[b, 0:2] = np.frombuffer(np.uint16(bits).tobytes(), np.uint8)
            if case.qt == Q.Q4_K:
                blocks[b, 4:16] = 0x05            # every 6-bit scale non-zero: d * sc is +-Inf / NaN, not Inf * 0


def grad_dy(case, device="cpu", seed=0):
    """dY as a [M, ldy] activation-dtype buffer: N(0, 1) in [:, :N], NaN in the padding [N, ldy); nonfinite_dy cases also get
    a NaN, a +Inf (in the last column, the N tail) and a -Inf in three rows."""
    g = torch.Generator(device=device).manual_seed(_seed(case) + seed)
    dt = lb.TORCH_ACT[case.act]
    buf = torch.full((case.M, case.ldy), float("nan"), dtype=dt, device=device)
    buf[:, :case.N] = torch.randn(case.M, case.N, generator=g, device=device).to(dt)
    if case.edge == "nonfinite_dy":
        M, N = case.M, case.N
        buf[0, 3 % N] = float("nan")
        buf[M - 1, N - 1] = float("inf")
        buf[M // 2, N // 2] = float("-inf")
    return buf
