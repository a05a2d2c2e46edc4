"""The patched packed Linear, element by element, against a float64 product (bound and derivation: `lora_reference` in
tests/lora_bounds.py): ggufb200_linear_lora, _lora_ex and _lora_scaled -- the FUSED_TMEM kernel with J LoRA k-blocks, the
per-tile k-block table and the DoRA feature scale in its epilogue and in the split-K finalize -- and ggufb200_gemm_scaled,
called through the C ABI into caller-owned buffers; then the layer's own calls of them, captured from real forwards.

Beyond the bound: outputs start as NaN; `_lora_scaled` with a NULL scale is `_lora_ex` and `_lora_ex` with J = 1 and no table
is `_lora`, bit for bit; a table that excludes only all-zero U columns changes no bit; unsplit runs meet the bound as split
ones do; NaN in X's row pad, in T and U past 64 J, in the U entries a tile's table excludes and in the split-K workspace is
never read, and bytes around Y stay as they were; NaN / Inf in one U row and one T row stay in that feature column and that
token row."""
import functools
import inspect

import numpy as np
import pytest
import torch

import linear_bounds as lb
import lora_bounds as lob
from util import Q

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = {lb.F16: 0x7D5A, lb.BF16: 0x7FA5}          # NaN patterns no kernel writes
USED = {}                                              # entry point -> largest fraction of the bound used


@pytest.fixture(scope="module", autouse=True)
def report_bound_use():
    yield
    if USED:
        print("\nlargest fraction of the per-element bound used, per entry point:")
        for k in sorted(USED):
            print(f"  {k:28s} {USED[k]:.3f}")


def _record(key, used):
    USED[key] = max(USED.get(key, 0.0), used)


@pytest.fixture(scope="module")
def hostf():
    L = lb.build_hostf()
    assert L is not None, "nvcc is needed to run the fast producers on the host"
    return L


@functools.lru_cache(maxsize=8)
def _model(qt, N, K, act, model, hostf=None):
    """The route's weight operand, float64 on the CPU, and its rms."""
    raw = lob.random_weight(qt, N, K)
    W = lb.fast_weight(hostf, raw, qt, N, K, act) if model == "fast" else lb.exact_weight(raw, qt, N, K, act)
    return W, float(W.pow(2).mean().sqrt())


def _weight(case, hostf):
    return _model(case.qt, case.N, case.K, case.act, case.weight_model, hostf if case.weight_model == "fast" else None)


def _packed(pkg, case):
    """(packed bytes, span-major / block-major copy or None) on the GPU."""
    w = torch.from_numpy(np.array(lob.random_weight(case.qt, case.N, case.K))).to(DEV)
    spans = None
    if case.spans:
        L = pkg.lib.lib()
        spans = torch.empty(L.ggufb200_repack_bytes(int(case.qt), case.N, case.K), dtype=torch.uint8, device=DEV)
        assert L.ggufb200_repack(int(case.qt), w.data_ptr(), case.N, case.K, spans.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
    return w, spans


def _device(ops):
    return lob.LoraOperands(*[t.to(DEV) if torch.is_tensor(t) else t for t in
                             (ops.x, ops.T, ops.U, ops.bias, ops.bias_code, ops.b_ref, ops.scale, ops.tiles)])


def _ptr(t):
    return None if t is None else t.data_ptr()


def _call(pkg, entry, case, w, spans, d, Y, ldy, ws, ws_bytes, X=None, ldx=None, T=None, ldt=None, U=None, ldu=None, tiles="d",
          scale="d", algo=None):
    """One call of `entry` (lora | lora_ex | lora_scaled); pointers default to the operands d, contiguous."""
    L = pkg.lib.lib()
    head = (int(case.qt), w.data_ptr(), _ptr(spans), case.N, case.K, X or d.x.data_ptr(), case.M, ldx or case.K, case.act, _ptr(d.bias),
            d.bias_code, T or d.T.data_ptr(), ldt or 64 * case.J, U or d.U.data_ptr())
    tail = (ws, ws_bytes, case.algo if algo is None else algo, torch.cuda.current_stream().cuda_stream)
    tiles = _ptr(d.tiles) if tiles == "d" else tiles
    scale = _ptr(d.scale) if scale == "d" else scale
    if entry == "lora":
        return L.ggufb200_linear_lora(*head, Y, ldy, *tail)
    if entry == "lora_ex":
        return L.ggufb200_linear_lora_ex(*head, ldu or 64 * case.J, case.J, tiles, Y, ldy, *tail)
    return L.ggufb200_linear_lora_scaled(*head, ldu or 64 * case.J, case.J, tiles, scale, Y, ldy, *tail)


def _run(pkg, entry, case, w, spans, d, **kw):
    """`_call` into a fresh NaN-filled [M, N] output with a zeroed workspace of the case's size."""
    L = pkg.lib.lib()
    Y = torch.full((case.M, case.N), float("nan"), dtype=lb.TORCH_ACT[case.act], device=DEV)
    need = lob.workspace_bytes(L, case)
    ws = torch.zeros(max(need, 16), dtype=torch.uint8, device=DEV)
    rc = _call(pkg, entry, case, w, spans, d, Y.data_ptr(), case.N, ws.data_ptr(), need, **kw)
    assert rc == 0, (entry, case.id, L.ggufb200_strerror(rc))
    return Y


def _reference(case, d, W):
    return lob.lora_reference(lb.to_f64(d.x), W.to(DEV), d.T, d.U, case.act, d.b_ref, d.scale, d.tiles)


# ---------------------------------------------------------------- 1. every element within the bound, and the bit identities
@pytest.mark.parametrize("case", lob.LORA_CASES, ids=lambda c: c.id)
def test_every_element_within_the_bound(pkg, hostf, case):
    L = pkg.lib.lib()
    W, w_rms = _weight(case, hostf)
    d = _device(lob.lora_operands(case, w_rms))
    w, spans = _packed(pkg, case)
    v, a, cls = _reference(case, d, W)
    y = _run(pkg, case.entry, case, w, spans, d)
    verdict = lb.check(y, v, a, cls, case.act, f"{case.entry} {case.id}")
    _record(case.entry, verdict.used)
    assert verdict.ok, verdict.message
    if case.scale == "none":
        assert torch.equal(_run(pkg, "lora_scaled", case, w, spans, d, scale=None), y), "_lora_scaled with a NULL scale is not _lora_ex"
        if case.J == 1 and case.table == "none":
            y1 = _run(pkg, "lora", case, w, spans, d)
            assert torch.equal(y1, y), "_lora_ex with J = 1 and no table is not _lora"
            _record("lora", lb.check(y1, v, a, cls, case.act).used)
    if d.tiles is not None:
        # zero the U entries the table excludes: running every k-block everywhere must then give the same bits
        _Uh, run = lob.lora_u_model(d.U, case.act, d.tiles)
        dz = lob.LoraOperands(d.x, d.T, torch.where(run, d.U, torch.zeros_like(d.U)), d.bias, d.bias_code, d.b_ref, d.scale, d.tiles)
        assert torch.equal(_run(pkg, case.entry, case, w, spans, dz), y), "the table changed bits on zero U columns"
        assert torch.equal(_run(pkg, case.entry, case, w, spans, dz, tiles=None), y), "a table that skips only zero U columns changed bits"
    if lb.plan(L, case, lob.workspace_bytes(L, case))[1] > 1:
        y_ns = _run(pkg, case.entry, case, w, spans, d, algo=case.algo | lb.FLAG_NOSPLIT)
        verdict = lb.check(y_ns, v, a, cls, case.act, f"{case.entry} unsplit {case.id}")
        _record(case.entry, verdict.used)
        assert verdict.ok, verdict.message


# ---------------------------------------------------------------- 2. poison that must never be read
GUARDED = [
    lob.LoraCase(Q.Q4_K, 33, 264, 4096, lb.F16, 5, "banded", "r", "f32", "fast"),                     # split K, scale in the finalize
    lob.LoraCase(Q.Q8_0, 5, 520, 4096, lb.BF16, 8, "clamp", "r", "act", "exact"),                      # split K, 32-token items
    lob.LoraCase(Q.Q5_1, 385, 136, 320, lb.BF16, 2, "banded", "none", "f32", "generic", flags=lb.FLAG_TILE384),
    lob.LoraCase(Q.Q3_K, 129, 248, 1024, lb.F16, 1, "zero", "r", "act", "fast", spans=True),
    lob.LoraCase(Q.Q4_K, 200, 640, 320, lb.BF16, 2, "banded", "r", "f32", "fast"),                     # straddled rows
    lob.LoraCase(Q.Q6_K, 31, 320, 640, lb.F16, 1, "none", "none", "none", "exact", spans=True),       # straddled, block-major copy
    lob.LoraCase(Q.Q4_K, 300, 264, 1024, lb.BF16, 1, "none", "none", "act", "exact", ws="two"),
]


@pytest.mark.parametrize("case", GUARDED, ids=lambda c: c.id)
def test_poisoned_buffers_are_never_read(pkg, hostf, case):
    L = pkg.lib.lib()
    M, N, K, J = case.M, case.N, case.K, case.J
    dt = lb.TORCH_ACT[case.act]
    W, w_rms = _weight(case, hostf)
    d = _device(lob.lora_operands(case, w_rms, seed=1))
    w, spans = _packed(pkg, case)
    y_clean = _run(pkg, case.entry, case, w, spans, d)
    # X: row pitch K + 16, NaN in [K, ldx) and in two rows after M; T and U: pitch 64 J + 8, NaN past 64 J (and in T's rows
    # after M); U: NaN in the entries the table excludes
    ldx, ldt, ldu = K + 16, 64 * J + 8, 64 * J + 8
    xbuf = torch.full((M + 2, ldx), float("nan"), dtype=dt, device=DEV)
    xbuf[:M, :K] = d.x
    tbuf = torch.full((M + 2, ldt), float("nan"), dtype=dt, device=DEV)
    tbuf[:M, :64 * J] = d.T
    ubuf = torch.full((N, ldu), float("nan"), dtype=torch.float16, device=DEV)
    _Uh, run = lob.lora_u_model(d.U, case.act, d.tiles)
    ubuf[:, :64 * J] = torch.where(run, d.U, torch.full_like(d.U, float("nan")))
    if d.tiles is not None and case.table != "none":
        assert not bool(run.all()), "meant to poison excluded U entries"
    # Y: a view inside a sentinel-filled buffer -- 8-element lead, pitch N + 8 or N + 24, three trailing rows
    lead, ldy = 8, N + (8 if N % 16 else 24)
    ybuf = torch.empty(lead + (M + 3) * ldy, dtype=torch.int16, device=DEV)
    inside = torch.zeros(ybuf.numel(), dtype=torch.bool, device=DEV)
    inside[lead:lead + M * ldy].view(M, ldy)[:, :N] = True
    ybuf.fill_(SENTINEL[case.act])
    need = lob.workspace_bytes(L, case)
    tail = 4096
    wsbuf = torch.empty(need + tail, dtype=torch.uint8, device=DEV)
    wsbuf[:need].fill_(0xFF)                                      # 0xFFFFFFFF: an fp32 NaN in every partial slot
    wsbuf[need:].fill_(0xA5)
    if case.M <= 64 and not case.straddled:
        assert lb.plan(L, case, need)[1] > 1, "meant to cover the split-K finalize"
    rc = _call(pkg, case.entry, case, w, spans, d, ybuf.data_ptr() + 2 * lead, ldy, wsbuf.data_ptr() if need else None, need,
               X=xbuf.data_ptr(), ldx=ldx, T=tbuf.data_ptr(), ldt=ldt, U=ubuf.data_ptr(), ldu=ldu)
    assert rc == 0, (case.id, L.ggufb200_strerror(rc))
    torch.cuda.synchronize()
    assert bool((wsbuf[need:] == 0xA5).all()), "bytes past the workspace the route asked for were written"
    assert bool((ybuf[~inside] == SENTINEL[case.act]).all()), "bytes of Y outside the [M, N] view changed"
    y = ybuf[inside].view(dt).view(M, N)
    assert torch.equal(y, y_clean), "poisoned padding, excluded U entries or stale partials changed the result"
    v, a, cls = _reference(case, d, W)
    verdict = lb.check(y, v, a, cls, case.act, case.id)
    assert verdict.ok, verdict.message


# ---------------------------------------------------------------- 3. non-finite LoRA operands
NONFINITE = [
    lob.LoraCase(Q.Q4_K, 33, 264, 4096, lb.BF16, 2, "none", "r", "f32", "fast"),            # split K
    lob.LoraCase(Q.Q8_0, 300, 520, 1024, lb.F16, 5, "banded", "r", "act", "exact"),
    lob.LoraCase(Q.Q6_K, 129, 384, 1024, lb.BF16, 1, "none", "none", "none", "generic", spans=True),
    lob.LoraCase(Q.Q4_K, 200, 640, 320, lb.F16, 2, "clamp", "none", "f32", "exact"),       # straddled rows
]


@pytest.mark.parametrize("case", NONFINITE, ids=lambda c: c.id)
def test_nonfinite_lora_values_stay_in_their_row_and_column(pkg, hostf, case):
    """NaN in one U row, +Inf in another; +Inf in one T row, NaN in another: each in a column the row's tile runs."""
    M, N, J = case.M, case.N, case.J
    W, w_rms = _weight(case, hostf)
    d = _device(lob.lora_operands(case, w_rms, seed=2))
    _Uh, run = lob.lora_u_model(d.U, case.act, d.tiles)
    rows = [n for n in (N - 3, 130, 7, 255) if bool(run[n, :case.R].any())][:2]
    assert len(rows) == 2, "needs two features whose tiles run a k-block"
    for n, val in zip(rows, (float("nan"), float("inf"))):
        d.U[n, int(run[n, :case.R].nonzero()[-1])] = val
    cols = run[:, :case.R].any(0).nonzero().reshape(-1)
    d.T[1, int(cols[0])] = float("inf")
    d.T[M - 1, int(cols[-1])] = float("nan")
    w, spans = _packed(pkg, case)
    y = _run(pkg, case.entry, case, w, spans, d)
    v, a, cls = _reference(case, d, W)
    bad = torch.zeros(M, N, dtype=torch.bool, device=DEV)
    bad[[1, M - 1], :] = True
    bad[:, rows] = True
    assert bool((cls[~bad] == lb.FIN).all()) and int((cls != lb.FIN).sum()) >= M
    verdict = lb.check(y, v, a, cls, case.act, case.id)
    assert verdict.ok, verdict.message


# ---------------------------------------------------------------- 4. the dense GEMM with a feature scale
@pytest.mark.parametrize("act", [lb.F16, lb.BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("M,N,K,bias", [(1, 8, 1024, "f32"), (127, 136, 4096, "act"), (128, 264, 1000, "none"), (129, 520, 256, "f32"),
                                        (385, 264, 4096, "act"), (1000, 120, 72, "f32"), (64, 384, 2048, "none")])
def test_gemm_scaled_within_the_bound(pkg, act, M, N, K, bias):
    """r drawn log-uniform in [1/8, 8]; N past the last full 128 / 256-feature tile in most shapes, so the scale must reach the
    features of a partial tile."""
    g = torch.Generator().manual_seed(M * 7 + N + K + act)
    dt = lb.TORCH_ACT[act]
    x = torch.randn(M, K, generator=g).to(dt).to(DEV)
    W = (torch.randn(N, K, generator=g) * 0.05).to(dt).to(DEV)
    r = torch.exp2(torch.rand(N, generator=g) * 6 - 3).to(DEV)
    b32 = (torch.randn(N, generator=g) * 0.5).to(DEV)
    b = None if bias == "none" else (b32 if bias == "f32" else b32.to(dt))
    code = 0 if b is None else pkg.dequant.dtype_code(b.dtype)
    b_ref = None if b is None else lb.to_f64(b32.to(dt))
    L = pkg.lib.lib()
    st = torch.cuda.current_stream().cuda_stream

    def gemm_scaled(s):
        y = torch.full((M, N), float("nan"), dtype=dt, device=DEV)
        rc = L.ggufb200_gemm_scaled(W.data_ptr(), N, K, K, x.data_ptr(), M, K, act, _ptr(b), code, s, y.data_ptr(), N, st)
        assert rc == 0, L.ggufb200_strerror(rc)
        return y
    y = gemm_scaled(r.data_ptr())
    v, a, cls = lob.lora_reference(lb.to_f64(x), lb.to_f64(W), None, None, act, b_ref, r)
    verdict = lb.check(y, v, a, cls, act, f"gemm_scaled {M}x{N}x{K}")
    _record("gemm_scaled", verdict.used)
    assert verdict.ok, verdict.message
    assert torch.equal(gemm_scaled(None), pkg.ops.linear_dense(x, W, b)), "NULL scale is not ggufb200_gemm"
    edge = N // 128 * 128
    if edge < N:                                    # the partial tile's features carry a scale far from 1
        assert float((r[edge:] - 1).abs().max()) > 0.25


# ---------------------------------------------------------------- 5. the layer's own calls
class LoRAAdapter:                      # the objects newer ComfyUI puts in a patch entry
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


_LAUNCH = inspect.signature(lambda x, wraw, qtype, N, K, bias, math, algo, spans=None, lora=None, scale=None: None)


@pytest.fixture
def launches(pkg, monkeypatch):
    """Every ops._launch_linear call of a forward: (bound arguments, result).  Wraps the function, never replaces it."""
    real = pkg.ops._launch_linear
    seen = []

    def spy(*args, **kwargs):
        y = real(*args, **kwargs)
        seen.append((_LAUNCH.bind(*args, **kwargs).arguments, y))
        return y
    monkeypatch.setattr(pkg.ops, "_launch_linear", spy)
    return seen


def _layer(pkg, N, K, seed):
    raw = lob.random_weight(Q.Q4_K, N, K)
    lin = pkg.ops.GGMLOps.Linear(K, N)
    w = pkg.ops.GGMLTensor(torch.from_numpy(np.array(raw)).to(DEV).view(N, K // 256 * 144), tensor_type=Q.Q4_K, tensor_shape=torch.Size((N, K)))
    b = (torch.randn(N, generator=torch.Generator().manual_seed(seed)) * 0.5).to(DEV)
    lin.load_state_dict({"weight": w, "bias": pkg.ops.GGMLTensor(b, tensor_type=Q.F32, tensor_shape=torch.Size((N,)))})
    return lin, raw


def _factors(g, *shapes, s=0.2):
    return [(torch.randn(*sh, generator=g) * s).to(DEV) for sh in shapes]


def _entries(kind, N, K, g, W=None):
    """Patch entries: Flux linear1 slices (four row bands), a LoHa, or DoRA lists on the output or the input axis."""
    if kind == "slices":
        H = N // 7
        out = []
        for i, (start, size) in enumerate([(0, H), (H, H), (2 * H, H), (3 * H, 4 * H)]):
            up, down = _factors(g, (size, 24), (24, K))
            out.append((0.8 - 0.1 * i, ("lora", (up, down, 12.0, None, None, None)) if i % 2 else LoRAAdapter((up, down, 12.0, None, None, None)),
                        1.0, (0, start, size), None))
        return out
    if kind == "loha":
        w1a, w1b, w2a, w2b = _factors(g, (N, 4), (4, K), (N, 6), (6, K))
        return [(0.9, LoHaAdapter((w1a, w1b, 2.0, w2a, w2b, None, None, None)), 1.0, None, None)]
    axis = 0 if kind == "dora_out" else 1

    def magnitude():
        nrm = W.float().norm(dim=1 - axis, keepdim=True)
        return nrm * (torch.rand(*nrm.shape, generator=g) * 0.4 + 0.8).to(DEV)
    up, down, up2, down2 = _factors(g, (N, 16), (16, K), (N, 8), (8, K), s=0.05)
    w1a, w1b, w2a, w2b = _factors(g, (N, 2), (2, K), (N, 2), (2, K))
    return [(0.8, ("lora", (up, down, 8.0, None, magnitude(), None)), 1.0, None, None),
            (0.9, LoRAAdapter((up2, down2, None, None, None, None)), 1.0, None, None),
            (1.0, LoHaAdapter((w1a, w1b, 1.0, w2a, w2b, None, None, magnitude())), 1.0, None, None)]


@pytest.mark.parametrize("M", [5, 300])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("kind", ["slices", "loha", "dora_out", "dora_in"])
def test_the_layers_patched_calls_within_the_bound(pkg, launches, kind, dtype, M):
    """A forward's ggufb200_linear_lora* call, captured with its operands (T, U, table, feature scale as the layer built
    them), against `lora_reference` on those operands; the layer returns exactly that call's output.  For DoRA the call gets
    the plan's r, U and input scale c."""
    N, K = (1792, 1024) if kind == "slices" else (384, 1024)
    act = pkg.dequant.dtype_code(dtype)
    lin, raw = _layer(pkg, N, K, seed=M + N)
    g = torch.Generator().manual_seed(M * 3 + act)
    W0 = pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, dtype))
    lin.weight.patches = [(_entries(kind, N, K, g, W0), "diffusion_model.w")]
    x = (torch.randn(2, M, K, generator=g) * 0.5).to(DEV).to(dtype)
    y = lin(x)
    assert len(launches) == 1 and launches[0][0].get("lora") is not None, "the in-kernel route was not taken"
    args, y_call = launches[0]
    assert torch.equal(y.reshape(-1, N), y_call.reshape(-1, N))
    T, U, tiles = args["lora"]
    scale = args.get("scale")
    assert args["algo"] & pkg.lib.FLAG_EXACT_W and args["spans"] is None
    assert (tiles is not None) == (kind == "slices") and (scale is not None) == kind.startswith("dora")
    xk = args["x"].reshape(-1, K)
    if kind.startswith("dora"):
        plan = lin._gg_dora[1]
        down_pad, u_pad = plan.kernel
        assert scale is plan.r and U is u_pad
        assert torch.equal(T, pkg.ops.linear_dense(x.reshape(-1, K), down_pad))
        assert (plan.c is None) == (kind == "dora_out")
        want_x = x.reshape(-1, K) if plan.c is None else pkg.ops.scale_columns(x.reshape(-1, K), plan.c)
        assert torch.equal(xk, want_x)
    Wm = lb.exact_weight(raw, Q.Q4_K, N, K, act).to(DEV)
    b_ref = lb.to_f64(args["bias"].to(dtype))
    v, a, cls = lob.lora_reference(lb.to_f64(xk), Wm, T, U, act, b_ref, scale, tiles)
    verdict = lb.check(y_call.reshape(-1, N), v, a, cls, act, f"layer {kind}")
    _record(f"layer-{kind}", verdict.used)
    assert verdict.ok, verdict.message
    lin.weight.patches = []


# ---------------------------------------------------------------- 6. refusals
def test_refusals(pkg):
    """J = 0 / 9: E_SHAPE; ldu below 64 J or not a multiple of 8, a tile table not 4-byte aligned, a feature scale not 16-byte
    aligned: E_ALIGN; an algo that resolves away from FUSED_TMEM: E_UNSUPPORTED.  The unmodified call runs."""
    A = pkg.lib
    E_ALIGN, E_SHAPE, E_UNSUPPORTED = -3, -4, -8
    case = lob.LoraCase(Q.Q4_K, 40, 264, 1024, lb.F16, 2, "banded", "r", "f32", "exact")
    d = _device(lob.lora_operands(case, 0.05))
    w, _spans = _packed(pkg, case)
    big = torch.zeros(case.N * 9 * 64 + 64, dtype=torch.float16, device=DEV)       # room for J = 9 and wide pitches
    tbig = torch.zeros(case.M * 9 * 64 + 64, dtype=torch.float16, device=DEV)
    Y = torch.empty(case.M, case.N, dtype=torch.float16, device=DEV)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    sbuf = torch.ones(case.N + 8, dtype=torch.float32, device=DEV)

    def rc(entry="lora_scaled", **kw):
        return _call(pkg, entry, case, w, None, d, Y.data_ptr(), case.N, ws.data_ptr(), ws.numel(), **kw)
    assert rc() == 0 and rc("lora_ex") == 0
    torch.cuda.synchronize()
    j9 = lob.LoraCase(Q.Q4_K, 40, 264, 1024, lb.F16, 9, "none", "r", "f32", "exact")
    for entry in ("lora_ex", "lora_scaled"):
        assert _call(pkg, entry, j9, w, None, d, Y.data_ptr(), case.N, ws.data_ptr(), ws.numel(), T=tbig.data_ptr(), U=big.data_ptr(),
                     tiles=None) == E_SHAPE, entry
        assert _j0(pkg, entry, case, w, d, Y, ws) == E_SHAPE, entry
        assert rc(entry, ldu=64 * case.J - 8, U=big.data_ptr()) == E_ALIGN
        assert rc(entry, ldu=64 * case.J + 4, U=big.data_ptr()) == E_ALIGN
        assert rc(entry, tiles=d.tiles.data_ptr() + 2) == E_ALIGN
        for algo in (A.ALGO_GEMV, A.ALGO_FUSED_MMA, A.ALGO_DEQUANT_MMA):
            assert rc(entry, algo=algo) == E_UNSUPPORTED, (entry, algo)
    assert rc(scale=sbuf.data_ptr() + 4) == E_ALIGN
    assert rc(scale=sbuf.data_ptr() + 16) == 0
    # AUTO: under EXACT_W at M <= 8 it resolves to the mma.sync GEMV, without it to the integer-pattern GEMV
    small = lob.LoraCase(Q.Q4_K, 4, 264, 1024, lb.F16, 2, "banded", "r", "f32", "exact")
    for algo in (A.ALGO_AUTO | A.FLAG_EXACT_W, A.ALGO_AUTO):
        for entry in ("lora_ex", "lora_scaled"):
            assert _call(pkg, entry, small, w, None, d, Y.data_ptr(), case.N, ws.data_ptr(), ws.numel(), algo=algo) == E_UNSUPPORTED
    torch.cuda.synchronize()


def _j0(pkg, entry, case, w, d, Y, ws):
    """The call with J = 0 (lora_kblocks out of range below)."""
    L = pkg.lib.lib()
    head = (int(case.qt), w.data_ptr(), None, case.N, case.K, d.x.data_ptr(), case.M, case.K, case.act, _ptr(d.bias), d.bias_code,
            d.T.data_ptr(), 64 * case.J, d.U.data_ptr(), 64 * case.J, 0, None)
    tail = (Y.data_ptr(), case.N, ws.data_ptr(), ws.numel(), case.algo, torch.cuda.current_stream().cuda_stream)
    if entry == "lora_ex":
        return L.ggufb200_linear_lora_ex(*head, *tail)
    return L.ggufb200_linear_lora_scaled(*head, _ptr(d.scale), *tail)
