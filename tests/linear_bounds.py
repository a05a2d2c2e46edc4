"""Per-element error bounds of the packed Linear, the weight models they are taken against and the shape / route case list.

No GPU here: tests/test_linear_bounds.py checks these helpers on the CPU, tests/test_gpu_linear_bounds.py applies them to
every route of the C ABI.

The bound.  A route computes y = rnd_act(fl(sum_k x_k W_k + b)), where W is the route's weight operand (below), every
product x_k W_k is exact in fp32 (fp16 x fp16 and bf16 x bf16 products have at most 22 / 16 significant bits) and fl() is
some fp32 evaluation of the sum: tensor-core steps (wgmma / mma.sync add 16 products to the accumulator, aligning to the
largest exponent and TRUNCATING: at most 2^-23 of the largest magnitude per term and step), fp32 partial tiles of a K range,
the split-K finalize (one fp32 add per range, then the bias) and the bias add.  Every fp32 add or tensor-core step loses at
most 2^-23 times the sum of the magnitudes it combines, and a chain of at most n such steps over K products therefore
satisfies  |fl(s) - s| <= n * 2^-23 * (sum_k |x_k| |W_k| + |b|).  Here n <= K + S + 2 <= 2K for K >= 64 (one step per
product, one per K range S <= K / 256, the bias, the final fp32 add), so with  v = x.W^T + b  exactly (float64) and

    a = c * K * 2^-23 * (|x|.|W|^T + |b|),   c = 2,

the fp32 value lies in [v - a, v + a] and, rounding being monotone,  rnd_act(v - a) <= y <= rnd_act(v + a)  holds for every
element.  rnd_act here is ONE correctly rounded step from float64 (`round_act`); the kernels round fp32 -> fp16 / bf16 once,
so no extra term is needed for the output, but the last fp32 add itself rounds to nearest: 2^-23 |v| is added to a for it.
On the exact-weight routes this is sharp: the only freedom left is the fp32 summation order, and a dropped k-block, a wrong
bias or a stale split-K slice moves an element by far more than a.

The weight operand W per contract:
  * exact (GEMV, FUSED_MMA, DEQUANT_MMA, FUSED_TMEM | EXACT_W or | GENERIC, the dense GEMM): `exact_weight`, the reference's
    fp16 chain cast to the activation dtype (oracle.dequant), bit for bit.
  * fast FUSED_TMEM: `fast_weight`, the bits of FastProducer<Q> (produce.cuh, run on the host by tests/host_functors.cu)
    cast to the activation dtype; only Q4_K / Q5_K differ from the exact weight (one fused multiply-add per element).
  * GEMV_FAST (csrc/gemv2.cu): W is never formed.  `gemv_fast_model` holds W = D*q - M exactly in float64 with the
    reference's sub-block products D = fp16(d*sc), M = fp16(dmin*mn).  The kernel does not sum x_k W_k: per 32-element
    sub-block it sums the integer PATTERNS (BIAS + q_k) * x_k on the tensor core and the activations x_k in fp32, then adds
    D * S - E * Xs with E = fp32(BIAS*D + M) (one fp32 fused multiply-add, rounded) by fp32 fused multiply-adds; BIAS is the
    exponent-trick offset of the pattern (1024 for fp16, 128 for bf16, 64 for the high nibbles of Q4_K in fp16).  With
    u = 2^-23, S* = sum (BIAS + q_k) x_k, Xs* = sum x_k exactly, D*S* - E*Xs* = sum x_k W_k: the large pattern terms cancel
    INSIDE one sub-block, and only the cancelled contribution travels the long accumulator chain.  Per sub-block:
      - S: two mma.sync k16 steps (16 + 17 terms, truncating): |S - S*| <= 33 u sum (BIAS + q_k) |x_k|;
      - Xs: 32 sequential fp32 adds: |Xs - Xs*| <= 16 u sum |x_k|;  E: one rounding, |E - E*| <= u/2 |E*|;
      - t = fma(D, S, acc): rounding <= u/2 (|D| |S| + |acc|);  acc' = fma(-E, Xs, t): rounding <= u/2 |acc'|.
    The terms in |D| (BIAS + q_k) |x_k| and |E| |x_k| add up to at most 35 u sum_k |x_k| mag_k with the model's magnitude
    mag_k = |D| (BIAS + q_k) + |BIAS*D + M| (second-order terms below u^2), summed over the sub-blocks once: |x|.mag^T.
    The accumulator itself (|acc|, |acc'| <= the running partial sums, bounded by |x|.|W|^T) goes through at most K/16 + 8 + 2
    roundings (two per sub-block per warp, the 8-warp reduction, the bias, the final add), inside the c K u (|x|.|W|^T + |b|)
    term above.  So for GEMV_FAST

        a = c * K * u * (|x|.|W|^T + |b|) + c_sub * u * (|x|.mag^T) + u |v|,   c = 2,  c_sub = 64 (35 doubled),

    `reference(..., mag=...)`; tests/test_linear_bounds.py shows this bound rejects a zeroed output and one dropped sub-block."""
import ctypes
import os
import random
import shutil
import subprocess
from dataclasses import dataclass

import numpy as np
import torch

import oracle
from util import Q

U = 2.0 ** -23
C_BOUND = 2.0
C_SUB = 64.0                 # GEMV_FAST: the sub-block sums of the pattern magnitudes, charged once
F16, BF16 = oracle.DT_F16, oracle.DT_BF16
TORCH_ACT = {F16: torch.float16, BF16: torch.bfloat16}
# mantissa bits, smallest normal exponent, first power of two that rounds to infinity
_FMT = {F16: (10, -14, 2.0 ** 16), BF16: (7, -126, 2.0 ** 128)}
FIN, NAN, PINF, NINF = 0, 1, 2, 3

HERE = os.path.dirname(os.path.abspath(__file__))
HOSTF_SRC = os.path.join(HERE, "host_functors.cu")
HOSTF_OUT = os.path.join(HERE, "_build", "libhostfunctors.so")
CSRC = os.path.join(os.path.dirname(HERE), "comfyui-gguf_b200", "csrc")


# ---------------------------------------------------------------- rounding
def _ulp_exp(v, act):
    mant, emin, _ = _FMT[act]
    _, e = torch.frexp(v)                                   # v = m * 2^e, 0.5 <= |m| < 1
    return torch.clamp(e.to(torch.int64) - 1, min=emin) - mant


def round_act(v, act):
    """float64 -> the nearest fp16 / bf16 value (ties to even, overflow to +-Inf), as float64; one rounding step."""
    v = torch.as_tensor(v, dtype=torch.float64)
    e = _ulp_exp(torch.where(torch.isfinite(v), v, torch.zeros_like(v)), act)
    r = torch.ldexp(torch.round(torch.ldexp(v, -e)), e)
    r = torch.where(r.abs() >= _FMT[act][2], torch.copysign(torch.full_like(v, float("inf")), v), r)
    return torch.where(torch.isfinite(v), r, v)


def half_ulp(y, act):
    """Half the spacing of the fp16 / bf16 grid at the finite values y (float64)."""
    y = torch.where(torch.isfinite(y), y, torch.zeros_like(y))
    return torch.ldexp(torch.full_like(y, 0.5), _ulp_exp(y, act))


def to_f64(t):
    return t.to(torch.float64)


# ---------------------------------------------------------------- weight models (CPU)
def exact_weight(raw, qt, N, K, act):
    """The reference's weight: fp16 dequant chain, then the cast to the activation dtype -- [N, K] float64."""
    bits = oracle.dequant(np.ascontiguousarray(raw).reshape(-1), int(qt), act, oracle.DT_F16)
    return to_f64(torch.from_numpy(bits.view(np.int16).copy()).view(TORCH_ACT[act])).reshape(N, K)


def build_hostf():
    """tests/host_functors.cu as a shared library (the command of tests/test_host_functors.py); None without nvcc."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        return None
    deps = [HOSTF_SRC] + [os.path.join(CSRC, f) for f in ("blocks.cuh", "common.cuh", "produce.cuh")]
    if not os.path.exists(HOSTF_OUT) or any(os.path.getmtime(d) > os.path.getmtime(HOSTF_OUT) for d in deps):
        os.makedirs(os.path.dirname(HOSTF_OUT), exist_ok=True)
        tmp = HOSTF_OUT + f".{os.getpid()}.tmp"
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-o", tmp, HOSTF_SRC], check=True)
        os.replace(tmp, HOSTF_OUT)
    L = ctypes.CDLL(HOSTF_OUT)
    L.hostf_produce.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    return L


def fast_bits(hostf, raw, qt):
    """FastProducer<Q> (FMA step) over a flat stream of Q4_K / Q5_K blocks (one block = one 256-wide span): fp16 bits."""
    assert qt in (Q.Q4_K, Q.Q5_K)
    ts = oracle.type_info(int(qt))[1]
    blocks = np.ascontiguousarray(raw).reshape(-1, ts)
    pitch = (ts + 15) // 16 * 16
    buf = np.zeros(blocks.shape[0] * pitch + 16, dtype=np.uint8)
    off = (-buf.ctypes.data) % 16
    view = buf[off:off + blocks.shape[0] * pitch].reshape(-1, pitch)
    view[:, :ts] = blocks
    out = np.empty(blocks.shape[0] * 256, dtype=np.uint16)
    assert hostf.hostf_produce(int(qt), view.ctypes.data, blocks.shape[0], pitch, out.ctypes.data, 1) == 1
    return out


def fast_weight(hostf, raw, qt, N, K, act):
    """Weight operand of FUSED_TMEM without EXACT_W: the FMA producers' fp16 value for Q4_K / Q5_K, cast to the activation
    dtype; every other format's hand-written or generic producer is the reference's (tests/test_host_functors.py)."""
    if qt not in (Q.Q4_K, Q.Q5_K):
        return exact_weight(raw, qt, N, K, act)
    h = torch.from_numpy(fast_bits(hostf, raw, qt).view(np.int16).copy()).view(torch.float16)
    return to_f64(h.to(TORCH_ACT[act])).reshape(N, K)


def k_quant_parts(raw, qt):
    """Per element of a flat Q4_K / Q5_K stream: q (integer unpack), D = fp16(d*sc), M = fp16(dmin*mn), as float64 arrays."""
    ts = oracle.type_info(int(qt))[1]
    blocks = np.ascontiguousarray(raw).reshape(-1, ts)
    q, sc, mn = oracle.unpack_int(blocks, int(qt))
    nb = blocks.shape[0]
    d = blocks[:, 0:2].copy().view(np.float16).astype(np.float32)
    dmin = blocks[:, 2:4].copy().view(np.float16).astype(np.float32)
    with np.errstate(all="ignore"):
        D = (d * sc.reshape(nb, -1).astype(np.float32)).astype(np.float16).astype(np.float64)
        Mm = (dmin * mn.reshape(nb, -1).astype(np.float32)).astype(np.float16).astype(np.float64)
    return q.reshape(nb, -1).astype(np.float64), D, Mm


def fma_model(raw, qt):
    """fp16(D*q - M) with D*q - M exact in float64 (fp16 operands: at most 45 significant bits), one rounding: the value the
    fused multiply-add producer must give, NaN / Inf included.  fp16 bits, flat."""
    q, D, Mm = k_quant_parts(raw, qt)
    with np.errstate(all="ignore"):
        return (D * q - Mm).astype(np.float16).reshape(-1).view(np.uint16)


def gemv_fast_model(raw, qt, N, K, act):
    """GEMV_FAST: (W, mag) as [N, K] float64 -- W = D*q - M exactly, mag = |D| (BIAS + q) + |BIAS*D + M| (module docstring)."""
    q, D, Mm = k_quant_parts(raw, qt)
    sub = (np.arange(256) // 32)[None, :]
    if act == BF16:
        bias = np.full((1, 256), 128.0)
    elif qt == Q.Q4_K:
        bias = np.where(sub % 2 == 1, 64.0, 1024.0)      # high nibbles kept in place: pattern 64 + q
    else:
        bias = np.full((1, 256), 1024.0)
    with np.errstate(all="ignore"):
        W = D * q - Mm
        mag = np.abs(D) * (bias + q) + np.abs(bias * D + Mm)
    return torch.from_numpy(W.reshape(N, K)), torch.from_numpy(mag.reshape(N, K))


# ---------------------------------------------------------------- the per-element check
def _ind(t):
    return t.to(torch.float64)


def classes(x, W, bias=None):
    """Class of every element of x.W^T (+ bias) in exact arithmetic: FIN, NAN, PINF or NINF.  Counted with 0/1 matrix
    products, independent of any summation order: NaN if a term is NaN (NaN operand, Inf * 0) or terms of both infinite
    signs meet; +-Inf if an infinite term of one sign exists."""
    if bool(torch.isfinite(x).all()) and bool(torch.isfinite(W).all()) and (bias is None or bool(torch.isfinite(bias).all())):
        return torch.full((x.shape[0], W.shape[0]), FIN, dtype=torch.int8, device=x.device)
    nan = (torch.isnan(x).any(1)[:, None] | torch.isnan(W).any(1)[None, :]
           | (_ind(torch.isinf(x)) @ _ind(W == 0).T > 0) | (_ind(x == 0) @ _ind(torch.isinf(W)).T > 0))
    inf = float("inf")
    pos = (_ind(x == inf) @ _ind(W > 0).T + _ind(x == -inf) @ _ind(W < 0).T + _ind(x > 0) @ _ind(W == inf).T
           + _ind(x < 0) @ _ind(W == -inf).T) > 0
    neg = (_ind(x == inf) @ _ind(W < 0).T + _ind(x == -inf) @ _ind(W > 0).T + _ind(x > 0) @ _ind(W == -inf).T
           + _ind(x < 0) @ _ind(W == inf).T) > 0
    if bias is not None:
        nan = nan | torch.isnan(bias)[None, :]
        pos = pos | (bias == inf)[None, :]
        neg = neg | (bias == -inf)[None, :]
    nan = nan | (pos & neg)
    c = torch.full(nan.shape, FIN, dtype=torch.int8, device=x.device)
    c[pos] = PINF
    c[neg] = NINF
    c[nan] = NAN
    return c


def value_classes(y):
    c = torch.full(y.shape, FIN, dtype=torch.int8, device=y.device)
    c[y == float("inf")] = PINF
    c[y == float("-inf")] = NINF
    c[torch.isnan(y)] = NAN
    return c


def reference(x, W, bias=None, mag=None):
    """(v, a, cls) for y ~ x.W^T + bias: float64 tensors on any device (x [M, K], W / mag [N, K], bias [N] or None).  v and a
    are taken over the finite operands (an element whose class is FIN involves no other), cls from `classes`.  mag: the
    per-element magnitudes of GEMV_FAST's sub-block sums (`gemv_fast_model`), charged once (module docstring)."""
    K = x.shape[1]
    xf = torch.where(torch.isfinite(x), x, torch.zeros_like(x))
    Wf = torch.where(torch.isfinite(W), W, torch.zeros_like(W))
    v = xf @ Wf.T
    s = xf.abs() @ Wf.abs().T
    if bias is not None:
        v = v + bias[None, :]
        s = s + bias.abs()[None, :]
    a = C_BOUND * K * U * s + U * v.abs()
    if mag is not None:
        a = a + C_SUB * U * (xf.abs() @ torch.where(torch.isfinite(mag), mag, torch.zeros_like(mag)).T)
    return v, a, classes(x, W, bias)


@dataclass
class Verdict:
    ok: bool
    used: float          # largest fraction of the bound used by a finite element
    message: str


def check(y, v, a, cls, act, what="", match_nonfinite=True):
    """rnd_act(v - a) <= y <= rnd_act(v + a) for every element of class FIN; y's NaN / +Inf / -Inf exactly where cls says
    (match_nonfinite=False: only the FIN elements must be finite, the others may hold anything)."""
    y = to_f64(y).reshape(v.shape)
    yc = value_classes(y)
    wrong_class = yc != cls
    if not match_nonfinite:
        wrong_class = wrong_class & (cls == FIN)
    fin = cls == FIN
    lo, hi = round_act(v - a, act), round_act(v + a, act)
    out = fin & ~wrong_class & ~((lo <= y) & (y <= hi))
    dist = torch.clamp((y - v).abs() - half_ulp(y, act), min=0.0)
    frac = torch.where(a > 0, dist / a, torch.where(dist > 0, torch.full_like(a, float("inf")), torch.zeros_like(a)))
    frac = torch.where(fin & ~wrong_class, frac, torch.zeros_like(frac))
    used = float(frac.max()) if frac.numel() else 0.0
    n_cls, n_out = int(wrong_class.sum()), int(out.sum())
    msg = f"{what}: {n_out} elements outside the bound, {n_cls} with the wrong NaN/Inf class, largest fraction of the bound {used:.3g}"
    if n_cls:
        idx = wrong_class.nonzero()[:4].tolist()
        msg += "; class (got, want) at " + ", ".join(f"{tuple(i)}: ({int(yc[tuple(i)])}, {int(cls[tuple(i)])})" for i in idx)
    if n_out:
        idx = out.nonzero()[:4].tolist()
        msg += "; out of bound at " + ", ".join(f"{tuple(i)}: y={float(y[tuple(i)]):.6g} v={float(v[tuple(i)]):.6g} a={float(a[tuple(i)]):.3g}"
                                                for i in idx)
    return Verdict(n_cls == 0 and n_out == 0, used, msg)


# ---------------------------------------------------------------- shape / route case list
ALL12 = [Q.Q4_0, Q.Q4_1, Q.Q5_0, Q.Q5_1, Q.Q8_0, Q.Q2_K, Q.Q3_K, Q.Q4_K, Q.Q5_K, Q.Q6_K, Q.IQ4_NL, Q.IQ4_XS]
TMEM_CANON = [Q.Q4_0, Q.Q4_1, Q.Q5_0, Q.Q5_1, Q.Q8_0, Q.Q4_K, Q.Q5_K, Q.IQ4_NL]      # canonical rows a tensor map can stage
M_ALL = (1, 5, 8, 9, 31, 32, 33, 127, 128, 129, 191, 192, 193, 383, 384, 385, 1000)
N_FUSED = (8, 120, 136, 248, 264, 520)
N_GEMV = N_FUSED + (130, 13)
K_ALL = (256, 1024, 4096, 12288)
STRADDLED = ((640, 320), (2560, 320), (320, 640))
BIAS_KINDS = ("none", "f32", "act")
PRODUCERS = ("fast", "exact", "generic")
FLAG_EXACT_W, FLAG_GENERIC, FLAG_TILE384, FLAG_NOSPLIT, FLAG_TILE192 = 0x100, 0x200, 0x400, 0x800, 0x2000
ALGO = {"gemv": 1, "fused_mma": 2, "dequant_mma": 3, "tmem": 4, "gemv_fast": 5}
PRODUCER_FLAG = {"fast": 0, "exact": FLAG_EXACT_W, "generic": FLAG_GENERIC}


@dataclass(frozen=True)
class Case:
    route: str              # gemv | gemv_fast | fused_mma | tmem | dequant_mma | dense
    qt: Q
    M: int
    N: int
    K: int
    act: int
    bias: str               # none | f32 | act
    producers: str = ""     # tmem: fast | exact | generic
    spans: bool = False     # tmem: read the span-major (block-major if straddled) copy
    flags: int = 0          # extra GGUFB200_FLAG_* bits (TILE384 / TILE192 / NOSPLIT)

    @property
    def straddled(self):
        return self.K % oracle.type_info(int(self.qt))[0] != 0

    @property
    def algo(self):
        return ALGO.get(self.route, 0) | PRODUCER_FLAG.get(self.producers, 0) | self.flags

    @property
    def weight_model(self):
        if self.route == "gemv_fast":
            return "gemv_fast"
        return "fast" if self.route == "tmem" and self.producers == "fast" else "exact"

    @property
    def id(self):
        p = f"-{self.producers}" if self.producers else ""
        s = "-spans" if self.spans else ""
        f = {FLAG_TILE384: "-t384", FLAG_TILE192: "-t192", FLAG_NOSPLIT: "-nosplit"}.get(self.flags, "")
        act = "f16" if self.act == F16 else "bf16"
        return f"{self.route}{p}{s}{f}-{self.qt.name}-{self.M}x{self.N}x{self.K}-{act}-bias_{self.bias}"


class _Cycle:
    """Values of `seq` in successive seeded shuffles: every value appears once per len(seq) draws, in varying company."""

    def __init__(self, seq, seed):
        self.seq, self.rng, self.buf = list(seq), random.Random(seed), []

    def __call__(self):
        if not self.buf:
            self.buf = self.seq[:]
            self.rng.shuffle(self.buf)
        return self.buf.pop()


def _cases():
    cases = []
    act, bias = _Cycle((F16, BF16), 1), _Cycle(BIAS_KINDS, 2)
    # FUSED_TMEM, canonical rows: every M with every producer family
    n, k, qt = _Cycle(N_FUSED, 3), _Cycle(K_ALL, 4), _Cycle(TMEM_CANON, 5)
    for i, M in enumerate(M_ALL):
        for prod in PRODUCERS:
            t = qt()
            K = 320 if t == Q.Q5_1 else k()
            flags = (FLAG_TILE384, FLAG_TILE192, 0)[i % 3] if M > 192 else (FLAG_NOSPLIT if (i + len(cases)) % 7 == 0 else 0)
            cases.append(Case("tmem", t, M, n(), K, act(), bias(), prod, flags=flags))
    # FUSED_TMEM from the span-major copy: all 12 formats
    m = _Cycle(M_ALL, 6)
    for t in ALL12:
        K = 320 if t == Q.Q5_1 else k()
        cases.append(Case("tmem", t, m(), n(), K, act(), bias(), PRODUCERS[len(cases) % 3], spans=True))
    # straddled rows (SD1.5 / SDXL): Q4_K from the canonical stream, Q6_K from the block-major copy
    for j, (N, K) in enumerate(STRADDLED):
        for t in (Q.Q4_K, Q.Q6_K):
            cases.append(Case("tmem", t, m(), N, K, act(), bias(), PRODUCERS[(j + int(t)) % 3], spans=t == Q.Q6_K))
        cases.append(Case("dequant_mma", (Q.Q4_K, Q.Q6_K)[j % 2], m(), N, K, act(), bias()))
    # FUSED_MMA: every M, all 12 formats
    t12 = _Cycle(ALL12, 7)
    for i, M in enumerate(M_ALL):
        t = t12()
        K = 320 if t == Q.Q5_1 else k()
        cases.append(Case("fused_mma", t, M, n(), K, act(), bias(), flags=FLAG_NOSPLIT if i % 5 == 4 else 0))
    # DEQUANT_MMA: all 12 formats
    for t in ALL12:
        K = 320 if t == Q.Q5_1 else k()
        cases.append(Case("dequant_mma", t, m(), n(), K, act(), bias()))
    # the mma.sync GEMV (M <= 8, any N): all 12 formats
    mg, ng = _Cycle((1, 5, 8), 8), _Cycle(N_GEMV, 9)
    for t in ALL12:
        K = 320 if t == Q.Q5_1 else k()
        cases.append(Case("gemv", t, mg(), ng(), K, act(), bias()))
    # GEMV_FAST (Q4_K / Q5_K, M <= 8, any N)
    for t in (Q.Q4_K, Q.Q5_K):
        for M in (1, 5, 8):
            cases.append(Case("gemv_fast", t, M, ng(), k(), act(), bias()))
    # the dense GEMM on the exact weight
    for M in (1, 33, 129, 385, 1000):
        cases.append(Case("dense", Q.Q8_0, M, n(), k(), act(), bias()))
    return cases


CASES = _cases()


def plan(L, case, ws_bytes):
    """ggufb200_linear_plan of a fused case: (tile rows / tokens, K ranges, k-blocks per range, CTAs / items)."""
    vals = [ctypes.c_int() for _ in range(4)]
    rc = L.ggufb200_linear_plan(int(case.qt), case.M, case.N, case.K, ws_bytes, case.algo, *[ctypes.byref(v) for v in vals])
    assert rc == 0, (case.id, rc)
    return tuple(v.value for v in vals)


def workspace_bytes(L, case):
    if case.route == "dense":
        return 0
    return L.ggufb200_linear_workspace(int(case.qt), case.M, case.N, case.K, case.act, case.algo)
