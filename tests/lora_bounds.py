"""Per-element error bound of the patched packed Linear -- the FUSED_TMEM kernel with LoRA k-blocks, the per-tile k-block
table and the per-feature scale (ggufb200_linear_lora, _lora_ex, _lora_scaled) and the scaled dense GEMM
(ggufb200_gemm_scaled) -- its case list and its operands.  It extends the unpatched bound of tests/linear_bounds.py.

No GPU here: tests/test_lora_bounds.py checks these helpers on the CPU, tests/test_gpu_lora_bounds.py applies them to the
C ABI and to the layer's own calls."""
from dataclasses import dataclass

import numpy as np
import torch

import linear_bounds as lb
import oracle
from util import Q


def workspace_bytes(L, case):
    """The workspace a LoraCase hands the kernel: what the unpatched route asks for, or room for two K ranges ("two")."""
    if case.ws == "two":
        return 2 * case.M * case.N * 4             # two fp32 partial slices: at most two K ranges
    return L.ggufb200_linear_workspace(int(case.qt), case.M, case.N, case.K, case.act, case.algo)


def random_weight(qt, N, K):
    """The packed bytes of the seeded random [N, K] weight the bound tests use (flat uint8, read-only)."""
    bs, _ts = oracle.type_info(int(qt))
    raw = oracle.random_blocks(int(qt), N * K // bs, seed=(int(qt) * 7919 + N * 31 + K) % 100003, scale=0.02).reshape(-1)
    raw.flags.writeable = False
    return raw


# ---------------------------------------------------------------- the bound
def clamp_tiles(tiles, J):
    """The (first, count) pairs the kernel runs: first clamped to [0, J], count to [0, J - first] (csrc/linear_sm90.cuh)."""
    out = []
    for f, c in (tiles.tolist() if torch.is_tensor(tiles) else tiles):
        f = min(max(int(f), 0), J)
        out.append((f, min(max(int(c), 0), J - f)))
    return out


def lora_u_model(U, act, tiles=None):
    """(Û, run): U [N, 64 J] as the warpgroup MMA sees it -- fp16 in memory, then the activation dtype (bf16(fp16(U)) under
    bf16 activations) -- as float64, with the columns of the k-blocks a 128-feature tile's clamped table entry does not run
    set to zero on that tile's rows; run [N, 64 J] marks the entries that are read."""
    N, width = U.shape
    J = width // 64
    Um = lb.to_f64(U.to(torch.float16).to(lb.TORCH_ACT[act]))
    run = torch.ones(N, width, dtype=torch.bool, device=U.device)
    if tiles is not None:
        for i, (f, c) in enumerate(clamp_tiles(tiles, J)):
            run[128 * i:128 * i + 128] = False
            run[128 * i:128 * i + 128, 64 * f:64 * (f + c)] = True
    return torch.where(run, Um, torch.zeros_like(Um)), run


def _scaled_classes(c, scale, bias):
    """Class of r * p + b from the class c of p: a negative r swaps the infinities, r = 0 turns them into NaN; then the bias."""
    if scale is not None:
        r = lb.to_f64(scale)[None, :].expand(c.shape)
        inf = (c == lb.PINF) | (c == lb.NINF)
        c = torch.where(inf & (r < 0), lb.PINF + lb.NINF - c, c)
        c = torch.where(inf & (r == 0), torch.full_like(c, lb.NAN), c)
    if bias is not None:
        b = bias[None, :].expand(c.shape)
        pos = (c == lb.PINF) | (b == float("inf"))
        neg = (c == lb.NINF) | (b == float("-inf"))
        nan = (c == lb.NAN) | torch.isnan(b) | (pos & neg)
        c = torch.where(pos, torch.full_like(c, lb.PINF), torch.where(neg, torch.full_like(c, lb.NINF), c))
        c = torch.where(nan, torch.full_like(c, lb.NAN), c)
    return c


def lora_reference(x, W, T, U, act, bias=None, scale=None, tiles=None):
    """(v, a, cls) of the patched route, y = rnd_act(r * (x.W^T + T.Û^T) + b), as float64 tensors on x's device.

    x [M, K], W [N, K] the route's weight model, T [M, >= 64 J] the LoRA activations (already in the activation dtype: the
    layer makes them with this library's dense GEMM), U [N, 64 J] (rounded through fp16 and then the activation dtype,
    `lora_u_model`), tiles None or ceil(N / 128) pairs (first, count), bias [N] float64 (already rounded to the activation
    dtype) or None, scale r [N] (fp32) or None.  T = U = None: no LoRA k-blocks (J = 0).

    The bound.  The kernel runs the J LoRA k-blocks after the main loop of the K range 0 only: k-block j reads T columns 64 j ..
    64 j + 63 (zero past M) against those columns of U, skipped on the tiles whose table entry excludes it.  So with the
    extended operands  x^ = [x | T],  W^ = [W | Û]  over K' = K + 64 J, the fp32 accumulator holds some evaluation of
    x^.W^^T by the same tensor-core steps and split-K adds as the unpatched route (linear_bounds module docstring):
    |acc - x^.W^^T| <= n u (|x^|.|W^|^T), n <= K' + S + 1.  The epilogue (or the split-K finalize, once, to the summed
    ranges) then computes fl(fl(r acc) + b) -- or one fused multiply-add, which nvcc may contract it into -- and rounds once
    to the activation dtype.  The multiply adds at most u/2 |r| |acc| <= u |r| (|x^|.|W^|^T), one more step of the chain
    scaled by |r|; the bias add at most u |fl(r acc) + b|.  With n + 2 <= 2 K' (K' >= 320) and v = r (x^.W^^T) + b in
    float64,

        a = c * K' * u * (|r| (|x^|.|W^|^T) + |b|) + 2 u |v|,   c = 2,

    where the second u |v| (absent without a scale, so that r = None, J = 0 is `reference` exactly) is kept for the rounding
    of the product r acc when the fused multiply-add is not formed.  cls: `linear_bounds.classes` on the extended operands, per tile on
    the k-blocks that tile runs (an excluded k-block multiplies nothing, not zero), then the sign of r and the bias."""
    if U is None:
        xh, Wh, run = x, W, None
    else:
        Uh, run = lora_u_model(U, act, tiles)
        xh = torch.cat([x, lb.to_f64(T[:, :U.shape[1]])], 1)
        Wh = torch.cat([W, Uh], 1)
    Kx = xh.shape[1]
    xf = torch.where(torch.isfinite(xh), xh, torch.zeros_like(xh))
    Wf = torch.where(torch.isfinite(Wh), Wh, torch.zeros_like(Wh))
    v = xf @ Wf.T
    s = xf.abs() @ Wf.abs().T
    if scale is not None:
        r = lb.to_f64(scale)[None, :]
        v = v * r
        s = s * r.abs()
    if bias is not None:
        v = v + bias[None, :]
        s = s + bias.abs()[None, :]
    a = lb.C_BOUND * Kx * lb.U * s + (2.0 if scale is not None else 1.0) * lb.U * v.abs()
    if run is None or bool(run.all()) or (bool(torch.isfinite(xh).all()) and bool(torch.isfinite(Wh).all())):
        cls = lb.classes(xh, Wh)
    else:
        K = x.shape[1]
        cls = torch.empty(v.shape, dtype=torch.int8, device=v.device)
        for n0 in range(0, W.shape[0], 128):
            cols = run[n0].nonzero().reshape(-1)
            cls[:, n0:n0 + 128] = lb.classes(torch.cat([x, xh[:, K:][:, cols]], 1), torch.cat([W[n0:n0 + 128], Wh[n0:n0 + 128, K:][:, cols]], 1))
    return v, a, _scaled_classes(cls, scale, bias)


N_LORA = tuple(sorted(set(lb.N_FUSED) | {384, 520}))        # 520, 8 ...: a partial last 128-feature tile
J_ALL = (1, 2, 5, 8)
TABLES = ("none", "banded", "zero", "clamp")
WORKSPACES = ("auto", "two")


@dataclass(frozen=True)
class LoraCase:
    """One call of the patched FUSED_TMEM route: ggufb200_linear_lora_scaled when scale == "r", else
    ggufb200_linear_lora_ex (and, for J = 1 without a table, ggufb200_linear_lora too)."""
    qt: Q
    M: int
    N: int
    K: int
    act: int
    J: int                  # LoRA k-blocks
    table: str              # none | banded | zero | clamp (values outside [0, J])
    scale: str              # none | r (drawn in [0.5, 2])
    bias: str               # none | f32 | act
    producers: str          # fast | exact | generic
    spans: bool = False
    flags: int = 0          # TILE384 / TILE192 / NOSPLIT
    ws: str = "auto"        # auto: the workspace the plain route asks for; two: room for two K ranges
    route = "tmem"

    @property
    def R(self):
        """Total rank: U columns R .. 64 J are zero (a ragged last k-block, as the layer's zero padding)."""
        return 64 * self.J - 13

    @property
    def straddled(self):
        return self.K % oracle.type_info(int(self.qt))[0] != 0

    @property
    def algo(self):
        return lb.ALGO["tmem"] | lb.PRODUCER_FLAG[self.producers] | self.flags

    @property
    def weight_model(self):
        return "fast" if self.producers == "fast" else "exact"

    @property
    def entry(self):
        return "lora_scaled" if self.scale == "r" else "lora_ex"

    @property
    def id(self):
        s = "-spans" if self.spans else ""
        f = {lb.FLAG_TILE384: "-t384", lb.FLAG_TILE192: "-t192", lb.FLAG_NOSPLIT: "-nosplit"}.get(self.flags, "")
        act = "f16" if self.act == lb.F16 else "bf16"
        return (f"{self.producers}{s}{f}-{self.qt.name}-{self.M}x{self.N}x{self.K}-J{self.J}-{self.table}-scale_{self.scale}"
                f"-{act}-bias_{self.bias}-ws_{self.ws}")


def lora_table(kind, N, J):
    """The per-tile table of a case: None, or ceil(N / 128) (first, count) pairs."""
    n = -(-N // 128)
    if kind == "none":
        return None
    if kind == "zero":
        return [(0, 0)] * n
    if kind == "banded":                       # tile i: one or two k-blocks, moving along the columns with i
        return [((i * J) // n, min(1 + i % 2, J - (i * J) // n)) for i in range(n)]
    raw = [(J + 3, 2), (-2, 1), (J - 1, 5), (1, -4), (-7, J + 7), (J, 1)]        # clamped: (J, 0) (0, 1) (J-1, 1) (1|J, 0) (0, J) (J, 0)
    return [raw[i % len(raw)] for i in range(n)]


def _lora_cases():
    cases = []
    act, bias, scale = lb._Cycle((lb.F16, lb.BF16), 11), lb._Cycle(lb.BIAS_KINDS, 12), lb._Cycle(("none", "r"), 13)
    n, k, qt = lb._Cycle(N_LORA, 14), lb._Cycle(lb.K_ALL, 15), lb._Cycle(lb.TMEM_CANON, 16)
    J, table, ws = lb._Cycle(J_ALL, 17), lb._Cycle(TABLES, 18), lb._Cycle(WORKSPACES, 19)

    def shape(t):
        N = n()
        K = 320 if t == Q.Q5_1 else k()
        while N * K > 4 << 20:                 # weight models on the CPU oracle stay at N K <= 4 M elements
            K //= 2
        return N, K
    # canonical rows: every M, two producer families each
    for i, M in enumerate(lb.M_ALL):
        for j, prod in enumerate((lb.PRODUCERS[i % 3], lb.PRODUCERS[(i + 1) % 3])):
            t = qt()
            N, K = shape(t)
            flags = (lb.FLAG_TILE384, lb.FLAG_TILE192, 0)[(i + j) % 3] if M > 192 else (lb.FLAG_NOSPLIT if (i + j) % 5 == 0 else 0)
            cases.append(LoraCase(t, M, N, K, act(), J(), table(), scale(), bias(), prod, flags=flags, ws=ws()))
    # the span-major copy: all 12 formats
    m = lb._Cycle(lb.M_ALL, 20)
    for i, t in enumerate(lb.ALL12):
        N, K = shape(t)
        cases.append(LoraCase(t, m(), N, K, act(), J(), table(), scale(), bias(), lb.PRODUCERS[i % 3], spans=True, ws=ws()))
    # straddled rows: Q4_K from the canonical stream, Q6_K from the block-major copy
    for j, (N, K) in enumerate(lb.STRADDLED):
        for t in (Q.Q4_K, Q.Q6_K):
            cases.append(LoraCase(t, m(), N, K, act(), J(), table(), scale(), bias(), lb.PRODUCERS[(j + int(t)) % 3], spans=t == Q.Q6_K))
    # ggufb200_linear_lora: J = 1, no table, no scale, split and unsplit
    for M, prod, flags in ((5, "fast", 0), (300, "exact", 0), (129, "generic", lb.FLAG_NOSPLIT)):
        N, K = shape(Q.Q4_K)
        cases.append(LoraCase(Q.Q4_K, M, N, K, act(), 1, "none", "none", bias(), prod, flags=flags))
    return cases


LORA_CASES = _lora_cases()


@dataclass
class LoraOperands:
    """Operands of one patched call, on the CPU: x [M, K], T [M, 64 J] (activation dtype), U [N, 64 J] fp16, the bias as the
    kernel takes it (bias, bias_code) and as the reference takes it (b_ref, float64 rounded to the activation dtype), the
    feature scale (fp32 [N] or None) and the table (int32 [ceil(N / 128), 2] or None)."""
    x: torch.Tensor
    T: torch.Tensor
    U: torch.Tensor
    bias: object
    bias_code: int
    b_ref: object
    scale: object
    tiles: object


def lora_operands(case, w_rms, seed=0):
    """Seeded operands of a LoraCase, sized so that the faults the bound must catch exceed it: with s0 = sqrt(K) w_rms the
    rms of x.W^T, each of T.U^T (rank R), the bias and r - 1 is of the order of s0 (typical LoRA magnitudes would hide a
    dropped k-block below one output ulp)."""
    g = torch.Generator().manual_seed(case.M * 1009 + case.N * 17 + case.K * 3 + case.J + seed)
    dt = lb.TORCH_ACT[case.act]
    s0 = float(np.sqrt(case.K)) * w_rms
    x = torch.randn(case.M, case.K, generator=g).to(dt)
    T = torch.randn(case.M, 64 * case.J, generator=g).to(dt)
    U = torch.randn(case.N, 64 * case.J, generator=g) * (s0 / np.sqrt(case.R))
    U[:, case.R:] = 0.0
    U = U.to(torch.float16)
    b32 = torch.randn(case.N, generator=g) * s0
    scale = (torch.rand(case.N, generator=g) * 1.5 + 0.5) if case.scale == "r" else None
    table = lora_table(case.table, case.N, case.J)
    tiles = None if table is None else torch.tensor(table, dtype=torch.int32)
    if case.bias == "none":
        return LoraOperands(x, T, U, None, 0, None, scale, tiles)
    b_ref = lb.to_f64(b32.to(dt))
    if case.bias == "f32":
        return LoraOperands(x, T, U, b32, oracle.DT_F32, b_ref, scale, tiles)
    return LoraOperands(x, T, U, b32.to(dt), case.act, b_ref, scale, tiles)
