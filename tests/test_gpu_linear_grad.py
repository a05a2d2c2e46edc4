"""GPU tests of the packed-weight Linear's backward on an H100: the MN-major dense GEMM of ggufb200_linear_grad_input against a
float64 product, the layer's input gradient for every weight type against the float64 dY . W_ref (W_ref = the reference's
`dequantize_tensor(weight, act_dtype, dequant_dtype)`, bit-exact to the reference through the committed goldens), the
untouched no-grad launch sequence, the memory the backward keeps alive, LoRA factor gradients, the two-step route of the
other patch lists, a small LoRA training run and the entry point's refusals."""
import gguf
import pytest
import torch

import oracle
from fallback_cases import FALLBACK, random_blocks as fallback_blocks
from linear_bounds import check, reference
from util import ALL_QTYPES, Q, rel_fro

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ACT = {torch.float16: 0, torch.bfloat16: 1}


def _raw(qt, n_elems, seed=0, scale=0.02):
    bs = gguf.GGML_QUANT_SIZES[qt][0]
    if qt in FALLBACK:
        return fallback_blocks(qt, n_elems // bs, seed=seed, scale=scale)
    return oracle.random_blocks(int(qt), n_elems // bs, seed=seed + int(qt), scale=scale)


def _weight(pkg, qt, N, K, seed=0, patches=(), scale=0.02):
    raw = torch.from_numpy(_raw(qt, N * K, seed, scale).reshape(-1)).to(DEV)
    return pkg.ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size((N, K)), patches=list(patches))


def _linear(pkg, qt, N, K, seed=0, bias=False, patches=(), scale=0.02):
    lin = pkg.ops.GGMLOps.Linear(K, N)
    sd = {"weight": _weight(pkg, qt, N, K, seed, patches, scale)}
    if bias:
        b = (torch.randn(N, generator=torch.Generator().manual_seed(seed + 3)) * 0.05).to(DEV)
        sd["bias"] = pkg.ops.GGMLTensor(b, tensor_type=Q.F32, tensor_shape=torch.Size((N,)))
    lin.load_state_dict(sd)
    return lin


def _w_ref(pkg, lin, dtype):
    return pkg.dequant.dequantize_tensor(lin.weight, dtype, lin.dequant_dtype)


def _rel(a, b):
    """Relative Frobenius distance; the 1e-3 checks take it against the float64 product rounded once to the output dtype, as
    the reference's own output is (a bf16 result cannot be nearer than its rounding, about 1.6e-3 here)."""
    return rel_fro(a.double().cpu().numpy(), b.double().cpu().numpy())


def _grad_input(pkg, qt, wraw, N, K, dy, M, ldy, act, dx, ldx, ws=None, ws_bytes=None, flags=0, math=0):
    L = pkg.lib.lib()
    if ws_bytes is None:
        ws_bytes = L.ggufb200_linear_grad_input_workspace(int(qt), N, K, act)
    if ws is None and ws_bytes:
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV).data_ptr()
    return L.ggufb200_linear_grad_input(int(qt), wraw, N, K, dy, M, ldy, act, math, dx, ldx, ws, ws_bytes, flags,
                                        torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------- the GEMM mode
@pytest.mark.parametrize("NK", [(3072, 12288), (12288, 3072), (18432, 3072), (640, 640), (320, 2560)], ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("M", [1, 7, 64, 300, 4096])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_gemm_mode_against_float64(pkg, dtype, M, NK):
    """dX = dY . W through ggufb200_linear_grad_input on a BF16 weight (bf16: the bytes are the operand, the GEMM alone; fp16:
    one exact-contract dequant first), with strided dY and dX: 1e-3 relative Frobenius and the per-element bound of
    tests/linear_bounds.py (the reduction runs over N)."""
    N, K = NK
    g = torch.Generator(device=DEV).manual_seed(M + N)
    w = (torch.randn(N, K, device=DEV, generator=g) * 0.02).to(torch.bfloat16)
    wraw = w.view(torch.uint8).reshape(-1)
    W = w.to(dtype)
    ldy, ldx = N + 24, K + 16
    dy_buf = torch.randn(M, ldy, device=DEV, generator=g).to(dtype)
    dx_buf = torch.full((M, ldx), float("nan"), device=DEV, dtype=dtype)
    rc = _grad_input(pkg, Q.BF16, wraw.data_ptr(), N, K, dy_buf.data_ptr(), M, ldy, ACT[dtype], dx_buf.data_ptr(), ldx)
    assert rc == 0, pkg.lib.lib().ggufb200_strerror(rc)
    torch.cuda.synchronize()
    dy = dy_buf[:, :N]
    dx = dx_buf[:, :K]
    assert torch.isnan(dx_buf[:, K:]).all(), "the kernel wrote past the row length"
    v, a, cls = reference(dy.double(), W.double().t().contiguous())
    assert _rel(dx, v.to(dtype)) <= 1e-3                  # against the product rounded once to the output dtype
    verdict = check(dx, v, a, cls, ACT[dtype], f"M={M} N={N} K={K}")
    assert verdict.ok, verdict.message


# ---------------------------------------------------------------- the layer's input gradient
TYPES = ALL_QTYPES + list(FALLBACK)


@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("M", [1, 8, 77, 512, 4096])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("qt", TYPES, ids=lambda q: q.name)
def test_layer_input_gradient(pkg, qt, dtype, M, bias):
    N, K = 136, 512
    lin = _linear(pkg, qt, N, K, seed=int(qt), bias=bias)
    g = torch.Generator(device=DEV).manual_seed(M)
    x = torch.randn(M, K, device=DEV, generator=g).to(dtype)
    with torch.no_grad():
        y0 = lin(x)
    xr = x.clone().requires_grad_(True)
    y = lin(xr)
    assert y.requires_grad and torch.equal(y, y0), "the forward with grad must be bit-identical to the no-grad call"
    dy = torch.randn(M, N, device=DEV, generator=g).to(dtype)
    y.backward(dy)
    want = dy.double() @ _w_ref(pkg, lin, dtype).double()
    assert xr.grad is not None and xr.grad.dtype == dtype
    assert _rel(xr.grad, want.to(dtype)) <= 1e-3


@pytest.mark.parametrize("case", [(Q.Q4_K, 264, 320), (Q.Q4_K, 264, 640), (Q.Q6_K, 264, 320), (Q.Q6_K, 264, 640), (Q.Q8_0, 136, 2432),
                                  (Q.Q8_0, 130, 512)], ids=lambda c: f"{c[0].name}-{c[1]}x{c[2]}")
@pytest.mark.parametrize("M", [5, 300])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_layer_input_gradient_straddled_and_odd_rows(pkg, case, M, dtype):
    """Straddled SD1.5 / SDXL K-quant rows, Q8_0 rows the tensor map cannot stage, and N % 8 != 0 (at M <= 8 the GEMV serves
    it and the backward pads dY's rows; above, the two-step route)."""
    qt, N, K = case
    lin = _linear(pkg, qt, N, K, seed=3, bias=True)
    x = torch.randn(1, M, K, device=DEV).to(dtype).requires_grad_(True)
    y = lin(x)
    dy = torch.randn_like(y)
    y.backward(dy)
    want = dy.double().reshape(-1, N) @ _w_ref(pkg, lin, dtype).double()
    assert x.grad.shape == x.shape and _rel(x.grad.reshape(-1, K), want.to(dtype)) <= 1e-3


@pytest.mark.parametrize("case", [(Q.Q4_K, 136, 5), (Q.Q4_K, 136, 300), (Q.Q8_0, 130, 5)], ids=lambda c: f"{c[0].name}-N{c[1]}-M{c[2]}")
@pytest.mark.parametrize("pool", ["sum0-2d", "sum1-batch1"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_layer_input_gradient_of_a_pooled_output(pkg, case, pool, dtype):
    """A loss pooled over the tokens hands the layer a broadcast gradient whose rows overlap (row stride 0): y.sum(0) of an
    [M, N] output, y.sum(1) of a [1, T, N] one.  The backward copies it into proper rows (padded when N % 8 != 0)."""
    qt, N, M = case
    K = 512
    lin = _linear(pkg, qt, N, K, seed=4, bias=True)
    shape = (M, K) if pool == "sum0-2d" else (1, M, K)
    x = torch.randn(*shape, device=DEV).to(dtype).requires_grad_(True)
    c = torch.randn(N, device=DEV)
    y = lin(x)
    strides = []
    y.register_hook(lambda g: strides.append(g.stride()))
    pooled = y.sum(0) if pool == "sum0-2d" else y.sum(1)
    (pooled.float() * c).sum().backward()
    assert strides and strides[0][-2] == 0, strides
    want = c.to(dtype).double().expand(M, N) @ _w_ref(pkg, lin, dtype).double()
    assert x.grad.shape == x.shape and _rel(x.grad.reshape(-1, K), want.to(dtype)) <= 1e-3


def test_fast_contract_backward_uses_the_exact_weight(pkg, monkeypatch):
    monkeypatch.setattr(pkg.ops.GGMLOps.Linear, "linear_numerics", "fast")
    lin = _linear(pkg, Q.Q4_K, 3072, 1024)
    x = torch.randn(256, 1024, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    dy = torch.randn(256, 3072, device=DEV, dtype=torch.bfloat16)
    lin(x).backward(dy)
    W = _w_ref(pkg, lin, torch.bfloat16)
    v, a, cls = reference(dy.double(), W.double().t().contiguous())
    verdict = check(x.grad, v, a, cls, 1, "fast forward, exact backward")
    assert verdict.ok, verdict.message


# ---------------------------------------------------------------- the no-grad path and the calls
SPIED = ("ggufb200_linear", "ggufb200_linear_spans", "ggufb200_linear_lora", "ggufb200_linear_lora_ex", "ggufb200_gemm", "ggufb200_dequant",
         "ggufb200_dequant_fallback", "ggufb200_dequant_kron", "ggufb200_dequant_lowrank", "ggufb200_dequant_patched", "ggufb200_repack",
         "ggufb200_linear_grad_input")


@pytest.fixture
def calls(pkg, monkeypatch):
    L = pkg.lib.lib()
    seen = []
    for name in SPIED:
        real = getattr(L, name)

        def wrapped(*args, _real=real, _name=name):
            seen.append(_name)
            return _real(*args)
        monkeypatch.setattr(L, name, wrapped)
    return seen


@pytest.mark.parametrize("qt", [Q.Q4_K, Q.Q6_K, Q.BF16, Q.IQ2_XS], ids=lambda q: q.name)
@pytest.mark.parametrize("M", [4, 300])
def test_no_grad_path_unchanged(pkg, calls, qt, M):
    """Under no_grad, and with grad enabled but nothing requiring it, the same launches run and give the same bits; the new
    entry point is called by the backward only."""
    lin = _linear(pkg, qt, 256, 512, bias=True)
    x = torch.randn(M, 512, device=DEV, dtype=torch.bfloat16)
    lin(x)                                           # first use builds the span copy of Q6_K
    calls.clear()
    with torch.no_grad():
        y0 = lin(x)
    seq0, calls[:] = list(calls), []
    y1 = lin(x)
    seq1, calls[:] = list(calls), []
    assert seq0 == seq1 and seq0 and "ggufb200_linear_grad_input" not in seq0, (seq0, seq1)
    assert not y1.requires_grad and torch.equal(y0, y1)
    xr = x.clone().requires_grad_(True)
    y2 = lin(xr)
    assert list(calls) == seq0 and torch.equal(y2, y0)
    calls.clear()
    y2.sum().backward()
    assert calls == ["ggufb200_linear_grad_input"]


def test_offloaded_weight_saves_the_device_copy(pkg):
    """A module whose packed weight stays on the host: the forward copies it to the GPU and the backward reads that copy."""
    N, K = 512, 512
    raw = torch.from_numpy(_raw(Q.Q4_K, N * K).reshape(-1))
    lin = pkg.ops.GGMLOps.Linear(K, N)
    lin.load_state_dict({"weight": pkg.ops.GGMLTensor(raw, tensor_type=Q.Q4_K, tensor_shape=torch.Size((N, K)))})
    assert lin.weight.device.type == "cpu"
    w_dev = pkg.dequant.dequantize_tensor(pkg.ops.GGMLTensor(raw.to(DEV), tensor_type=Q.Q4_K, tensor_shape=torch.Size((N, K))),
                                          torch.float16)
    x = torch.randn(40, K, device=DEV, dtype=torch.float16, requires_grad=True)
    dy = torch.randn(40, N, device=DEV, dtype=torch.float16)
    lin(x).backward(dy)
    assert _rel(x.grad, (dy.double() @ w_dev.double()).half()) <= 1e-3


def test_double_backward_raises(pkg):
    lin = _linear(pkg, Q.Q8_0, 256, 256)
    x = torch.randn(16, 256, device=DEV, dtype=torch.float16, requires_grad=True)
    (gx,) = torch.autograd.grad(lin(x).float().square().sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.float().sum().backward()


# ---------------------------------------------------------------- memory
def _stack_growth(pkg, two_step, monkeypatch):
    N, K, M = 12288, 3072, 512
    layers = [_linear(pkg, Q.Q4_K, N, K, seed=i) for i in range(8)]
    if two_step:
        monkeypatch.setattr(pkg.ops.GGMLOps.Linear, "_fused_ok", lambda self, x: False)
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    ys = [lin(x) for lin in layers]
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    sum(y.float().sum() for y in ys).backward()
    monkeypatch.undo()
    return grown, sum(y.numel() * y.element_size() for y in ys), N * K * 2


def test_memory_packed_backward_keeps_no_dense_weight(pkg, monkeypatch):
    grown, activations, _dense = _stack_growth(pkg, False, monkeypatch)
    assert grown <= activations + (1 << 20), (grown, activations)


def test_memory_two_step_route_keeps_every_dense_weight(pkg, monkeypatch):
    grown, _activations, dense = _stack_growth(pkg, True, monkeypatch)
    assert grown >= 8 * dense, (grown, dense)


# ---------------------------------------------------------------- LoRA factor gradients
def _lora_entries(N, K, ranks, bands, seed=0):
    g = torch.Generator().manual_seed(seed)
    entries, factors = [], []
    for i, (r, band) in enumerate(zip(ranks, bands)):
        rows = band[2] if band is not None and band[0] == 0 else N
        cols = band[2] if band is not None and band[0] == 1 else K
        up = (torch.randn(rows, r, generator=g) * 0.05).to(DEV).requires_grad_(True)
        down = (torch.randn(r, cols, generator=g) * 0.05).to(DEV).requires_grad_(True)
        alpha, strength = float(r) / 2, 0.5 + 0.25 * i
        entries.append((strength, ("lora", (up, down, alpha, None, None, None)), 1.0, band, None))
        factors.append((strength * alpha / r, up, down, band))
    return entries, factors


def _delta64(N, K, factors):
    D = torch.zeros(N, K, dtype=torch.float64, device=DEV)
    for s, up, down, band in factors:
        d = s * (up.double() @ down.double())
        if band is None:
            D = D + d
        elif band[0] == 0:
            D = D + torch.nn.functional.pad(d, (0, 0, band[1], N - band[1] - band[2]))
        else:
            D = D + torch.nn.functional.pad(d, (band[1], K - band[1] - band[2]))
    return D


LORA_CASES = {
    "whole-r16": ([16], [None]),
    "stack-r96": ([32, 48, 16], [None, None, None]),
    "banded": ([16, 16, 8], [(0, 0, 512), (0, 512, 512), (1, 256, 256)]),
}


@pytest.mark.parametrize("case", list(LORA_CASES))
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_lora_factor_gradients(pkg, calls, case, dtype):
    N, K, M = 1536, 1024, 300
    ranks, bands = LORA_CASES[case]
    entries, factors = _lora_entries(N, K, ranks, bands)
    lin = _linear(pkg, Q.Q4_K, N, K, bias=True, patches=[(entries, "diffusion_model.x.weight")])
    x = torch.randn(M, K, device=DEV).to(dtype).requires_grad_(True)
    dy = torch.randn(M, N, device=DEV).to(dtype)
    lin(x).backward(dy)
    assert "ggufb200_linear_grad_input" in calls
    W = _w_ref(pkg, lin, dtype).double()
    x64 = x.detach().double().requires_grad_(True)
    f64 = [(s, u.detach().double().requires_grad_(True), d.detach().double().requires_grad_(True), b) for s, u, d, b in factors]
    (x64 @ (W + _delta64(N, K, f64)).t()).backward(dy.double())
    tol = 3e-3 if dtype == torch.float16 else 1e-2
    assert _rel(x.grad, x64.grad) <= tol
    for (_s, up, down, _b), (_s64, up64, down64, _b64) in zip(factors, f64):
        assert _rel(up.grad, up64.grad) <= tol and _rel(down.grad, down64.grad) <= tol


# ---------------------------------------------------------------- declined lists: the two-step route
def _restated_calculate_weight(patches, weight, key, intermediate_dtype=torch.float32, original_weights=None):
    """comfy.lora.calculate_weight for diff, LoRA, LoHa and LoKr entries, written with differentiable (out-of-place) torch ops."""
    for strength, value, _sm, *_rest in patches:
        kind, v = value
        f = [t.to(device=weight.device, dtype=intermediate_dtype) if torch.is_tensor(t) else t for t in v]
        if kind == "diff":
            d, s = f[0], 1.0
        elif kind == "lora":
            d, s = (f[0] @ f[1]).reshape(weight.shape), 1.0 if f[2] is None else f[2] / f[1].shape[0]
        elif kind == "loha":
            d, s = (f[0] @ f[1]) * (f[3] @ f[4]), 1.0 if f[2] is None else f[2] / f[1].shape[0]
        else:
            d, s = torch.kron(f[0], f[1]).reshape(weight.shape), 1.0
        weight = weight + ((strength * s) * d).to(weight.dtype)
    return weight


def _declined(kind, N, K, g):
    def f(*shape, scale=0.1):
        return (torch.randn(*shape, generator=g) * scale).to(DEV).requires_grad_(True)
    if kind == "diff":
        return ("diff", (f(N, K, scale=0.01),))
    if kind == "loha":
        return ("loha", (f(N, 8), f(8, K), 4.0, f(N, 8), f(8, K), None, None, None))
    return ("lokr", (f(N // 16, K // 16), f(16, 16), None, None, None, None, None, None, None))


def _factors(value):
    return [t for t in value[1] if torch.is_tensor(t)]


@pytest.mark.parametrize("kind", ["diff", "loha", "lokr"])
def test_declined_linear_lists_take_the_two_step_route(pkg, calls, monkeypatch, kind):
    monkeypatch.setattr(pkg.ops.comfy_lora, "calculate_weight", _restated_calculate_weight)
    N, K, M = 512, 512, 64
    grads = []
    for kernels in (True, False):
        g = torch.Generator().manual_seed(1)
        value = _declined(kind, N, K, g)
        lin = _linear(pkg, Q.Q4_K, N, K, bias=True, patches=[([(0.7, value, 1.0, None, None)], "k")])
        lin.lora_side_gemm = kernels
        x = (torch.randn(M, K, generator=g) * 0.5).to(DEV, torch.float16).requires_grad_(True)
        calls.clear()
        y = lin(x)
        assert calls == ["ggufb200_dequant"], calls
        y.float().square().sum().backward()
        grads.append([x.grad] + [t.grad for t in _factors(value)])
    for a, b in zip(*grads):
        assert a is not None and torch.equal(a, b)


def _conv(pkg, qt, shape, entries, seed=0):
    cout, cin, kh, kw = shape
    conv = pkg.ops.GGMLOps.Conv2d(cin, cout, (kh, kw), padding=kh // 2, device="meta")
    raw = torch.from_numpy(_raw(qt, cout * cin * kh * kw, seed).reshape(-1)).to(DEV)
    w = pkg.ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size(shape), patches=[(entries, "diffusion_model.conv.weight")])
    bias = (torch.randn(cout, generator=torch.Generator().manual_seed(seed + 7)) * 0.05).to(DEV)
    conv.load_state_dict({"weight": w, "bias": bias}, assign=True)
    return conv


@pytest.mark.parametrize("kind", ["lora", "lokr"])
@pytest.mark.parametrize("x_grad", [True, False], ids=["x", "factors-only"])
def test_declined_conv_lists_take_the_two_step_route(pkg, calls, monkeypatch, kind, x_grad):
    monkeypatch.setattr(pkg.ops.comfy_lora, "calculate_weight", _restated_calculate_weight)
    shape = (64, 32, 3, 3)
    grads = []
    for kernels in (True, False):
        g = torch.Generator().manual_seed(2)
        if kind == "lora":
            value = ("lora", ((torch.randn(64, 8, generator=g) * 0.1).to(DEV).requires_grad_(True),
                              (torch.randn(8, 288, generator=g) * 0.1).to(DEV).requires_grad_(True), 4.0, None, None, None))
        else:
            value = ("lokr", ((torch.randn(4, 8, generator=g) * 0.1).to(DEV).requires_grad_(True),
                              (torch.randn(16, 36, generator=g) * 0.1).to(DEV).requires_grad_(True), None, None, None, None, None, None, None))
        conv = _conv(pkg, Q.Q8_0, shape, [(0.8, value, 1.0, None, None)])
        conv.conv_patches_in_kernel = kernels
        x = torch.randn(2, 32, 16, 16, generator=g).to(DEV, torch.bfloat16).requires_grad_(x_grad)
        calls.clear()
        y = conv(x)
        assert calls == ["ggufb200_dequant"], calls
        y.float().square().sum().backward()
        grads.append(([x.grad] if x_grad else []) + [t.grad for t in _factors(value)])
    for a, b in zip(*grads):
        assert a is not None and torch.equal(a, b)


# ---------------------------------------------------------------- a small training run
def _train(pkg, monkeypatch, two_step, steps=10):
    if two_step:
        monkeypatch.setattr(pkg.ops.GGMLOps.Linear, "_fused_ok", lambda self, x: False)
    D, r = 1024, 16
    layers = [_linear(pkg, Q.Q4_K, D, D, seed=10 + i, bias=True, scale=1e-4) for i in range(4)]   # unit-size activations
    g = torch.Generator().manual_seed(5)
    adapters = []
    for lin in layers:
        A = (torch.randn(r, D, generator=g) * 0.02).to(DEV).requires_grad_(True)
        B = (torch.randn(D, r, generator=g) * 0.02).to(DEV).requires_grad_(True)
        adapters += [A, B]

        def hook(mod, inputs, out, A=A, B=B):       # LoRA added to the layer's output: the packed weight is never patched
            return out + ((inputs[0].float() @ A.t()) @ B.t()).to(out.dtype)
        lin.register_forward_hook(hook)
    x = torch.randn(256, D, generator=g).to(DEV, torch.bfloat16)
    target = torch.randn(256, D, generator=g).to(DEV)
    opt = torch.optim.SGD(adapters, lr=0.05)
    losses, first = [], None
    for step in range(steps):
        h = x
        for lin in layers:
            h = torch.nn.functional.layer_norm(torch.nn.functional.gelu(lin(h)), (D,))
        loss = torch.nn.functional.mse_loss(h.float(), target)
        opt.zero_grad()
        loss.backward()
        if step == 0:
            first = [a.grad.clone() for a in adapters]
        opt.step()
        losses.append(loss.item())
    monkeypatch.undo()
    return losses, first


def test_training_smoke_lora_adapters(pkg, monkeypatch):
    losses, grads = _train(pkg, monkeypatch, False)
    want_losses, want_grads = _train(pkg, monkeypatch, True)
    for i, (g, w) in enumerate(zip(grads, want_grads)):
        assert float(g.abs().max()) > 0, f"adapter tensor {i} got no gradient"
        assert _rel(g, w) <= 2e-2, i
    assert all(torch.isfinite(torch.tensor(losses))), losses
    for a, b in zip(losses, want_losses):
        assert abs(a - b) <= 1e-2 * abs(b), (losses, want_losses)


# ---------------------------------------------------------------- refusals
def test_refusals(pkg):
    L = pkg.lib.lib()
    N, K, M = 256, 512, 16
    w = _weight(pkg, Q.Q4_K, N, K).as_subclass(torch.Tensor)
    dy = torch.randn(M + 1, N, device=DEV, dtype=torch.float16)
    dx = torch.empty(M + 1, K, device=DEV, dtype=torch.float16)
    ok = _grad_input(pkg, Q.Q4_K, w.data_ptr(), N, K, dy.data_ptr(), M, N, 0, dx.data_ptr(), K)
    assert ok == 0
    assert _grad_input(pkg, Q.Q4_K, None, N, K, dy.data_ptr(), M, N, 0, dx.data_ptr(), K) == -5
    assert _grad_input(pkg, Q.Q4_K, w.data_ptr(), N, K, dy.data_ptr() + 2, M, N, 0, dx.data_ptr(), K) == -3
    assert _grad_input(pkg, Q.Q4_K, w.data_ptr(), N, K, dy.data_ptr(), M, N - 1, 0, dx.data_ptr(), K) == -4
    assert _grad_input(pkg, 1, w.data_ptr(), N, K, dy.data_ptr(), M, N, 0, dx.data_ptr(), K) == -1
    assert _grad_input(pkg, Q.Q4_K, w.data_ptr(), N, K, dy.data_ptr(), M, N, 0, dx.data_ptr(), K, ws_bytes=N * K * 2 - 16) == -7
    assert _grad_input(pkg, Q.Q4_K, w.data_ptr(), N, K, dy.data_ptr(), M, N, 0, dx.data_ptr(), K, flags=pkg.lib.FLAG_EXACT_W) == -8
    assert L.ggufb200_linear_grad_input_workspace(int(Q.BF16), N, K, 1) == 0
    assert L.ggufb200_linear_grad_input_workspace(int(Q.Q4_K), N, K, 1) == N * K * 2
    torch.cuda.synchronize()
