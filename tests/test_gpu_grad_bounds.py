"""The packed Linear's input gradient, element by element, against a float64 product (bound and derivation:
tests/grad_bounds.py): ggufb200_linear_grad_input for every weight type and math dtype, at tile, box and reduction edges and
on both sides of the dense GEMM's narrow / wide switch, and the layer's own backward calls.

Beyond the bound: dY's padding columns hold NaN and must never reach the product; dX lives in a sentinel-filled buffer
with a row pitch past K and guard rows before and after it, which must come back bit for bit; the workspace starts as NaN
and is oversized (bytes past what the call asked for must stay), and a second call on a 16-byte-offset, exactly sized
workspace must give the same bits; W_STABLE against flags = 0, two back-to-back calls, and a NaN- against a zero-filled
workspace are bit-identical; NaN / Inf in the weight's blocks and in dY's rows stay in their own columns and rows."""
import functools
import inspect

import pytest
import torch

import grad_bounds as gb
import linear_bounds as lb
from util import Q

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = {lb.F16: 0x7D5A, lb.BF16: 0x7FA5}          # NaN patterns no kernel writes
GUARD = 3                                              # guard rows of dX's buffer before and after the [M, ldx] rows
TAIL = 4096                                            # workspace bytes past the size the call asks for
USED = {}                                              # entry point / layer group -> largest fraction of the bound used


@pytest.fixture(scope="module", autouse=True)
def report_bound_use():
    yield
    if USED:
        print("\nlargest fraction of the per-element bound used:")
        for k in sorted(USED):
            print(f"  {k:28s} {USED[k]:.3f}")


def _record(key, used):
    USED[key] = max(USED.get(key, 0.0), used)


@functools.lru_cache(maxsize=4)
def _weight(case):
    """(packed bytes as numpy, the same on the GPU, the exact W as float64 on the GPU)."""
    raw = gb.weight_bytes(case)
    W = gb.grad_weight(raw, case.qt, case.N, case.K, case.act, case.math).to(DEV)
    return raw, torch.from_numpy(raw.copy()).to(DEV), W


def _call(pkg, case, wraw, dy_buf, dx_ptr, ws_ptr, ws_bytes, flags=None, ldx=None):
    L = pkg.lib.lib()
    flags = pkg.lib.FLAG_W_STABLE if flags is None else flags
    return L.ggufb200_linear_grad_input(int(case.qt), wraw.data_ptr(), case.N, case.K, dy_buf.data_ptr(), case.M, case.ldy, case.act,
                                        case.math, dx_ptr, case.ldx if ldx is None else ldx, ws_ptr, ws_bytes, flags,
                                        torch.cuda.current_stream().cuda_stream)


class _Out:
    """dX's [M, ldx] rows inside a sentinel-filled buffer with GUARD rows before and after."""

    def __init__(self, case):
        self.case = case
        self.buf = torch.empty((case.M + 2 * GUARD) * case.ldx, dtype=torch.int16, device=DEV)
        self.inside = torch.zeros(self.buf.numel(), dtype=torch.bool, device=DEV)
        self.inside[GUARD * case.ldx:(GUARD + case.M) * case.ldx].view(case.M, case.ldx)[:, :case.K] = True

    def reset(self):
        self.buf.fill_(SENTINEL[self.case.act])
        return self.buf.data_ptr() + 2 * GUARD * self.case.ldx

    def dx(self):
        assert bool((self.buf[~self.inside] == SENTINEL[self.case.act]).all()), "dX's padding or guard rows were written"
        return self.buf[self.inside].clone().view(lb.TORCH_ACT[self.case.act]).view(self.case.M, self.case.K)


def _workspace_need(pkg, case):
    need = pkg.lib.lib().ggufb200_linear_grad_input_workspace(int(case.qt), case.N, case.K, case.act)
    assert (need == 0) == (case.weight == "in_place") and need in (0, case.N * case.K * 2), (case.id, need)
    return need


def _run(pkg, case, out, dy_buf, wraw, ws_fill=0xFF, offset=0, exact=False, flags=None):
    """One call; workspace NaN-filled (0xFF) or zeroed, `offset` bytes into its buffer, sized exactly or TAIL bytes over.
    Returns dX; asserts that the bytes past the asked-for workspace are untouched."""
    need = _workspace_need(pkg, case)
    ws = torch.empty(offset + need + TAIL, dtype=torch.uint8, device=DEV)
    ws[:offset + need].fill_(ws_fill)
    ws[offset + need:].fill_(0xA5)
    size = need if exact else need + TAIL
    rc = _call(pkg, case, wraw, dy_buf, out.reset(), ws.data_ptr() + offset if size else None, size, flags)
    assert rc == 0, (case.id, pkg.lib.lib().ggufb200_strerror(rc))
    torch.cuda.synchronize()
    assert bool((ws[offset + need:] == 0xA5).all()), "bytes past the workspace the call needs were written"
    return out.dx()


def _check(case, dx, W, dy_buf, key):
    v, a, cls = gb.grad_reference(lb.to_f64(dy_buf[:, :case.N]), W)
    verdict = lb.check(dx, v, a, cls, case.act, case.id)
    _record(key, verdict.used)
    assert verdict.ok, verdict.message
    return cls


# ---------------------------------------------------------------- 1. every case within the bound
@pytest.mark.parametrize("case", gb.CASES, ids=lambda c: c.id)
def test_every_element_within_the_bound(pkg, case):
    _raw, wraw, W = _weight(case)
    dy_buf = gb.grad_dy(case, DEV)
    out = _Out(case)
    dx = _run(pkg, case, out, dy_buf, wraw)
    dx2 = _run(pkg, case, out, dy_buf, wraw, offset=16, exact=True)
    assert torch.equal(dx.view(torch.int16), dx2.view(torch.int16)), "a 16-byte-offset, exactly sized workspace changed dX"
    _check(case, dx, W, dy_buf, f"abi-{case.weight}" + ("" if case.edge == "none" else "-edge"))


@pytest.mark.parametrize("act", [lb.F16, lb.BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("side", ["below", "at"])
def test_either_side_of_the_tile_switch(pkg, act, side):
    """dense_gemm_nn's narrow / wide choice at this device's SM count: 256-wide tiles numbering SMs - 1 and exactly SMs."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    case = gb.switch_cases(sms, act)[side == "at"]
    assert gb.narrow_tile(case.M, case.K, sms) == (side == "below")
    _raw, wraw, W = _weight(case)
    dy_buf = gb.grad_dy(case, DEV)
    dx = _run(pkg, case, _Out(case), dy_buf, wraw)
    _check(case, dx, W, dy_buf, "abi-tile-switch")


# ---------------------------------------------------------------- 2. bit identities
IDENTITY = [gb.make_case(Q.Q4_K, 300, 264, 320, lb.BF16, 2), gb.make_case(Q.Q8_0, 129, 2432, 1056, lb.F16, 1, i=1),
            gb.make_case(Q.IQ2_XS, 65, 136, 512, lb.BF16, i=2), gb.make_case(Q.BF16, 1000, 200, 1000, lb.F16),
            gb.make_case(Q.BF16, 4097, 72, 1000, lb.BF16, i=1)]


@pytest.mark.parametrize("case", IDENTITY, ids=lambda c: c.id)
def test_bit_identities(pkg, case):
    """W_STABLE against flags = 0; two back-to-back calls (no split, no atomics); a NaN- against a zero-filled workspace (K1
    writes every element the GEMM reads)."""
    _raw, wraw, _W = _weight(case)
    dy_buf = gb.grad_dy(case, DEV, seed=1)
    out = _Out(case)
    bits = lambda t: t.view(torch.int16)
    stable = _run(pkg, case, out, dy_buf, wraw)
    assert torch.equal(bits(stable), bits(_run(pkg, case, out, dy_buf, wraw, flags=0))), "W_STABLE changed dX"
    assert torch.equal(bits(stable), bits(_run(pkg, case, out, dy_buf, wraw))), "two calls gave different bits"
    assert torch.equal(bits(stable), bits(_run(pkg, case, out, dy_buf, wraw, ws_fill=0))), "the workspace's old contents reached dX"


# ---------------------------------------------------------------- 3. non-finite containment
NONFINITE = [c for c in gb.CASES if c.edge in ("bf16_overflow", "nonfinite_scales", "nonfinite_dy")]


@pytest.mark.parametrize("case", NONFINITE, ids=lambda c: c.id)
def test_nonfinite_values_stay_in_their_columns_and_rows(pkg, case):
    """A non-finite weight element reaches only its column of dX, a non-finite dY element only its row; inside them the
    NaN / Inf pattern is that of the float64 product."""
    _raw, wraw, W = _weight(case)
    dy_buf = gb.grad_dy(case, DEV)
    dx = _run(pkg, case, _Out(case), dy_buf, wraw)
    cls = _check(case, dx, W, dy_buf, "abi-nonfinite")
    bad_cols = ~torch.isfinite(W).all(0)
    bad_rows = ~torch.isfinite(dy_buf[:, :case.N].double()).all(1)
    assert bool(bad_cols.any() or bad_rows.any())
    nonfinite = ~torch.isfinite(dx.double())
    assert not bool((nonfinite & ~(bad_rows[:, None] | bad_cols[None, :])).any()), "a non-finite value left its row / column"
    assert 0 < int((cls == lb.FIN).sum()) < case.M * case.K


# ---------------------------------------------------------------- 4. the layer's own backward calls
_GRAD = inspect.signature(lambda dy, wraw, qtype, N, K, math: None)


@pytest.fixture
def grads(pkg, monkeypatch):
    """Every ops.linear_grad_input call of a backward: (bound arguments, dX).  Wraps the function, never replaces it."""
    real = pkg.ops.linear_grad_input
    seen = []

    def spy(*args, **kwargs):
        dx = real(*args, **kwargs)
        seen.append((_GRAD.bind(*args, **kwargs).arguments, dx))
        return dx
    monkeypatch.setattr(pkg.ops, "linear_grad_input", spy)
    return seen


def _layer(pkg, qt, N, K, device=DEV, offload=False, dequant_dtype=None):
    case = gb.make_case(qt, 1, N, K, lb.F16)
    raw = torch.from_numpy(gb.weight_bytes(case).copy())
    lin = pkg.ops.GGMLOps.Linear(K, N)
    w = pkg.ops.GGMLTensor(raw if offload else raw.to(device), tensor_type=qt, tensor_shape=torch.Size((N, K)))
    b = (torch.randn(N, generator=torch.Generator().manual_seed(N)) * 0.1).to(device)
    lin.load_state_dict({"weight": w, "bias": pkg.ops.GGMLTensor(b, tensor_type=Q.F32, tensor_shape=torch.Size((N,)))})
    lin.dequant_dtype = dequant_dtype
    return lin


def _check_call(pkg, call, dtype, key):
    args, dx = call
    dy, wraw, qtype, N, K, math = (args[k] for k in ("dy", "wraw", "qtype", "N", "K", "math"))
    act = pkg.dequant.dtype_code(dtype)
    assert dy.dtype == dtype and dx.dtype == dtype and dx.device == dy.device
    W = gb.grad_weight(wraw.cpu().numpy(), qtype, N, K, act, math).to(dy.device)
    v, a, cls = gb.grad_reference(lb.to_f64(dy.reshape(-1, N)), W)
    verdict = lb.check(dx.reshape(-1, K), v, a, cls, act, f"{key} {Q(qtype).name} N={N} K={K}")
    _record(key, verdict.used)
    assert verdict.ok, verdict.message
    return math


LAYER = {
    # name: (qt, N, K, M (tokens), input shape kind, extra)
    "sum0-broadcast-n130": (Q.Q8_0, 130, 512, 5, "sum0", {}),
    "sum0-broadcast": (Q.Q4_K, 264, 1024, 300, "sum0", {}),
    "3d-input": (Q.Q6_K, 264, 1024, 150, "3d", {}),
    "offloaded": (Q.Q4_K, 512, 512, 40, "2d", {"offload": True}),
    "dequant-f32": (Q.Q5_K, 264, 512, 77, "2d", {"dequant_dtype": torch.float32}),
    "dequant-bf16": (Q.Q4_1, 136, 1056, 129, "2d", {"dequant_dtype": torch.bfloat16}),
    "dequant-target": (Q.Q3_K, 136, 512, 64, "2d", {"dequant_dtype": "target"}),
    "fast-forward": (Q.Q4_K, 3072, 1024, 256, "2d", {"fast": True}),
    "sdxl-straddled": (Q.Q5_K, 640, 320, 300, "3d", {}),
    "fallback-IQ2_XS": (Q.IQ2_XS, 264, 512, 100, "2d", {}),
    "fallback-TQ2_0": (Q.TQ2_0, 136, 1024, 9, "3d", {}),
}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("name", list(LAYER))
def test_the_layers_backward_calls_within_the_bound(pkg, grads, monkeypatch, name, dtype):
    qt, N, K, M, kind, extra = LAYER[name]
    if extra.get("fast"):
        monkeypatch.setattr(pkg.ops.GGMLOps.Linear, "linear_numerics", "fast")
    lin = _layer(pkg, qt, N, K, offload=extra.get("offload", False), dequant_dtype=extra.get("dequant_dtype"))
    g = torch.Generator(device=DEV).manual_seed(M + N)
    shape = (2, M, K) if kind == "3d" else (M, K)
    x = torch.randn(*shape, device=DEV, generator=g).to(dtype).requires_grad_(True)
    y = lin(x)
    if kind == "sum0":
        c = torch.randn(N, device=DEV, generator=g)
        (y.sum(0).float() * c).sum().backward()
    else:
        y.backward(torch.randn(y.shape, device=DEV, generator=g).to(dtype))
    assert len(grads) == 1, "the backward did not call ops.linear_grad_input once"
    args, dx = grads[0]
    assert torch.equal(x.grad.reshape(-1, K), dx.reshape(-1, K)), "the layer's gradient is not the call's dX"
    if kind == "sum0":
        assert args["dy"].stride(0) == 0, "meant to cover the broadcast dY the backward copies into rows"
    math = _check_call(pkg, grads[0], dtype, "layer")
    assert math == pkg.dequant.math_code(lin.dequant_dtype, dtype)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_backward_on_the_second_device(pkg, grads):
    """The backward runs on autograd's worker thread for cuda:1: the entry point binds that device's primary context."""
    dev = torch.device("cuda:1")
    lin = _layer(pkg, Q.Q4_K, 264, 1024, device=dev)
    x = torch.randn(300, 1024, device=dev).to(torch.bfloat16).requires_grad_(True)
    lin(x).backward(torch.randn(300, 264, device=dev).to(torch.bfloat16))
    assert len(grads) == 1 and grads[0][1].device == dev
    _check_call(pkg, grads[0], torch.bfloat16, "layer-cuda1")


# ---------------------------------------------------------------- 5. refusals
def test_refusals(pkg):
    """A workspace not 16-byte aligned, and a dX pitch that is not a multiple of 8: E_ALIGN.  The unmodified call runs."""
    E_ALIGN = -3
    case = gb.make_case(Q.Q4_K, 16, 264, 512, lb.F16)
    _raw, wraw, _W = _weight(case)
    dy_buf = gb.grad_dy(case, DEV)
    need = _workspace_need(pkg, case)
    ws = torch.zeros(need + 64, dtype=torch.uint8, device=DEV)
    dx = torch.empty(case.M, case.ldx + 8, dtype=torch.float16, device=DEV)
    assert _call(pkg, case, wraw, dy_buf, dx.data_ptr(), ws.data_ptr(), need) == 0
    assert _call(pkg, case, wraw, dy_buf, dx.data_ptr(), ws.data_ptr() + 8, need) == E_ALIGN
    assert _call(pkg, case, wraw, dy_buf, dx.data_ptr(), ws.data_ptr(), need, ldx=case.K + 4) == E_ALIGN
    torch.cuda.synchronize()
