"""GPU tests of the Linear and the row gather of the numpy-fallback types (IQ2_XXS ... NVFP4): ggufb200_linear_fallback's two
routes bit for bit on the weight operand and element by element against a float64 product, its split-K reproducibility and
unaligned views, ggufb200_dequant_rows_fallback bit for bit, and the layers that call them."""
import gguf
import numpy as np
import pytest
import torch

from fallback_cases import FALLBACK, gguf_values, random_blocks
from linear_bounds import BF16, F16, TORCH_ACT, check, reference
from linear_fallback_cases import CROSSOVER, splits_of
from util import Q, canon_nan, torch_bits

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ALGOS = {"fused_sync": 6, "dequant_mma": 3}
OK, E_ALIGN = 0, -3


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _packed(qt, N, K, seed, specials=False):
    raw = random_blocks(qt, N * K // gguf.GGML_QUANT_SIZES[qt][0], seed=seed, scale=0.01, specials=specials)
    return raw, torch.from_numpy(raw).to(DEV).reshape(-1)


def _call(pkg, qt, w, N, K, x, ldx, act, y, ldy, bias=None, bias_code=0, ws=None, algo=0):
    """ggufb200_linear_fallback on device tensors: x [M, ldx], y [M, ldy]; ws None, a tensor, or (pointer, bytes)."""
    L = pkg.lib.lib()
    ws_ptr, ws_bytes = (None, 0) if ws is None else ((ws.data_ptr(), ws.numel()) if torch.is_tensor(ws) else ws)
    return L.ggufb200_linear_fallback(int(qt), w.data_ptr(), N, K, x.data_ptr(), x.shape[0], ldx, act, None if bias is None else bias.data_ptr(),
                                      bias_code, y.data_ptr(), ldy, ws_ptr, ws_bytes, algo, _stream())


def _workspace(pkg, qt, M, N, K, act, algo, fill=float("nan")):
    need = pkg.lib.lib().ggufb200_linear_fallback_workspace(int(qt), M, N, K, act, algo)
    return torch.full((max(need, 16) // 4,), fill, dtype=torch.float32, device=DEV).view(torch.uint8)


def _onehot_check(pkg, qt, w, N, K, act, algo):
    """Y = X W^T with one-hot rows X (M = 64 per call, every k once): Y[m, n] = W[n, k_m], bit for bit with the dequant."""
    dt = TORCH_ACT[act]
    want = pkg.dequant.dequantize_fallback(w, qt, (N, K), dt)
    for k0 in range(0, K, 64):
        x = torch.zeros(64, K, dtype=dt, device=DEV)
        x[torch.arange(64), k0 + torch.arange(64)] = 1
        y = torch.empty(64, N, dtype=dt, device=DEV)
        ws = _workspace(pkg, qt, 64, N, K, act, algo)
        assert _call(pkg, qt, w, N, K, x, K, act, y, N, ws=ws, algo=algo) == OK
        assert torch.equal(y.float(), want[:, k0:k0 + 64].t().float()), (qt.name, algo, k0)     # +0 / -0 alike


@pytest.mark.parametrize("route", list(ALGOS))
@pytest.mark.parametrize("act", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_weight_operand_bit_exact(pkg, qt, act, route):
    N, K = 136, 512
    _raw, w = _packed(qt, N, K, seed=1)
    _onehot_check(pkg, qt, w, N, K, act, ALGOS[route])


# ---------------------------------------------------------------- per-element bound against a float64 product
M_LIST = (1, 8, 9, 31, 32, 33, 64, 65, 127, 128, 129, 1000)
N_LIST = (8, 120, 136, 264)


def _bound_cases():
    cases = []
    i = 0
    for qt in FALLBACK:
        c = CROSSOVER[qt]
        bs = gguf.GGML_QUANT_SIZES[qt][0]
        ks = (256, 4096) + ((96 if bs == 32 else 192, 1088 if bs == 32 else 1216) if bs < 256 else ())
        for M in sorted(m for m in set(M_LIST + (c - 1, c, c + 1)) if m >= 1):
            N = N_LIST[i % len(N_LIST)]
            K = ks[i % len(ks)]
            act = (F16, BF16)[(i // 2) % 2]
            bias = ("none", "f32", "act")[i % 3]
            specials = i % 4 == 3 and qt != Q.MXFP4          # Inf / NaN / subnormal block scales (MXFP4's e8m0 has none)
            cases.append((qt, M, N, K, act, bias, specials))
            i += 1
    return cases


CASES = _bound_cases()


def _case_id(c):
    qt, M, N, K, act, bias, specials = c
    return f"{qt.name}-{M}x{N}x{K}-{'f16' if act == F16 else 'bf16'}-bias_{bias}{'-specials' if specials else ''}"


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_within_bound(pkg, case):
    qt, M, N, K, act, bias_kind, specials = case
    dt = TORCH_ACT[act]
    raw, w = _packed(qt, N, K, seed=M + N + K, specials=specials)
    W = torch.from_numpy(gguf_values(raw, qt).reshape(N, K)).to(DEV).to(dt).double()   # gguf-py fp32, rounded to the act dtype
    g = torch.Generator(device=DEV).manual_seed(M * 7 + N)
    ldx, ldy = K + 8, N + 8
    xbuf = torch.full((M, ldx), float("nan"), dtype=dt, device=DEV)
    xbuf[:, :K] = torch.randn(M, K, generator=g, device=DEV).to(dt)
    b, bcode, bref = None, 0, None
    if bias_kind != "none":
        b = torch.randn(N, generator=g, device=DEV) * 0.5
        b = b if bias_kind == "f32" else b.to(dt)
        bcode = 2 if bias_kind == "f32" else act
        bref = b.to(dt).double()
    v, a, cls = reference(xbuf[:, :K].double(), W, bref)
    for name, algo in (("auto", 0), ("fused_sync", ALGOS["fused_sync"])):
        ybuf = torch.full((M, ldy), float("nan"), dtype=dt, device=DEV)
        ws = _workspace(pkg, qt, M, N, K, act, algo)
        assert _call(pkg, qt, w, N, K, xbuf, ldx, act, ybuf, ldy, b, bcode, ws, algo) == OK
        verdict = check(ybuf[:, :N], v, a, cls, act, f"{_case_id(case)} {name}")
        assert verdict.ok, verdict.message
        assert torch.isnan(ybuf[:, N:]).all(), "padding columns of Y were written"


def test_split_k_engages_and_is_reproducible(pkg):
    qt, M, N, K, act = Q.IQ3_XXS, 40, 136, 8192, BF16
    need = pkg.lib.lib().ggufb200_linear_fallback_workspace(int(qt), M, N, K, act, ALGOS["fused_sync"])
    assert splits_of(need, M, N) > 1                       # the library's own plan on this device
    _raw, w = _packed(qt, N, K, seed=3)
    x = torch.randn(M, K, device=DEV).to(torch.bfloat16)
    b = torch.randn(N, device=DEV)
    outs = []
    for fill in (float("nan"), 1e30, 0.0):
        ws = _workspace(pkg, qt, M, N, K, act, ALGOS["fused_sync"], fill)
        assert ws.numel() >= need
        y = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        assert _call(pkg, qt, w, N, K, x, K, act, y, N, b, 2, ws, ALGOS["fused_sync"]) == OK
        outs.append(y)
    for y in outs[1:]:
        assert torch.equal(y.view(torch.int16), outs[0].view(torch.int16))
    # unsplit (NOSPLIT, or no workspace at all) is as close to the float64 product
    W = pkg.dequant.dequantize_fallback(w, qt, (N, K), torch.bfloat16).double()
    v, a, cls = reference(x.double(), W, b.to(torch.bfloat16).double())
    for algo, ws in ((ALGOS["fused_sync"] | pkg.lib.FLAG_NOSPLIT, None), (ALGOS["fused_sync"], None)):
        y = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        assert _call(pkg, qt, w, N, K, x, K, act, y, N, b, 2, ws, algo) == OK
        verdict = check(y, v, a, cls, act, "unsplit")
        assert verdict.ok, verdict.message


@pytest.mark.parametrize("qt", [q for q in FALLBACK if q != Q.MXFP4], ids=lambda q: q.name)
def test_unaligned_packed_view(pkg, qt):
    """A byte-offset view below the type's block alignment: AUTO and FUSED_SYNC take DEQUANT_MMA (same bits as the one-hot
    check); without the workspace the call is refused."""
    N, K = 136, 512
    raw, _w = _packed(qt, N, K, seed=4)
    buf = torch.zeros(raw.size + 32, dtype=torch.uint8, device=DEV)
    view = buf[1:1 + raw.size]
    view.copy_(torch.from_numpy(raw.reshape(-1)).to(DEV))
    for algo in (0, ALGOS["fused_sync"]):
        for act in (F16, BF16):
            dt = TORCH_ACT[act]
            want = pkg.dequant.dequantize_fallback(view, qt, (N, K), dt)
            x = torch.zeros(64, K, dtype=dt, device=DEV)
            x[torch.arange(64), torch.arange(64) * 3] = 1
            y = torch.empty(64, N, dtype=dt, device=DEV)
            ws = torch.empty(N * K * 2, dtype=torch.uint8, device=DEV)
            assert _call(pkg, qt, view, N, K, x, K, act, y, N, ws=ws, algo=algo) == OK
            assert torch.equal(y.float(), want[:, torch.arange(64) * 3].t().float())
            assert _call(pkg, qt, view, N, K, x, K, act, y, N, ws=None, algo=algo) == E_ALIGN


# ---------------------------------------------------------------- row gather
@pytest.mark.parametrize("code", [0, 1, 2], ids=["f16", "bf16", "f32"])
@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_rows_bit_exact(pkg, qt, code):
    V, K = 300, 2560
    raw, w = _packed(qt, V, K, seed=6, specials=True)
    dt = {0: torch.float16, 1: torch.bfloat16, 2: torch.float32}[code]
    table = pkg.dequant.dequantize_fallback(w, qt, (V, K), dt)
    ids = torch.tensor([0, 5, 299, 17, -1, 300, 10**9, 5, 0, 1], dtype=torch.int64, device=DEV)
    out = torch.full((ids.numel(), K), float("nan"), dtype=dt, device=DEV)
    rc = pkg.lib.lib().ggufb200_dequant_rows_fallback(int(qt), w.data_ptr(), V, K, ids.data_ptr(), ids.numel(), out.data_ptr(), code, _stream())
    assert rc == OK
    inside = (ids >= 0) & (ids < V)
    want = table[ids.clamp(0, V - 1)]
    assert np.array_equal(canon_nan(torch_bits(out[inside]), code), canon_nan(torch_bits(want[inside]), code))
    assert torch.equal(out[~inside], torch.zeros_like(out[~inside]))
    assert not torch.signbit(out[~inside]).any()


def test_rows_beyond_the_grid_y_limit(pkg):
    qt, V, K = Q.IQ2_XXS, 512, 256
    _raw, w = _packed(qt, V, K, seed=7)
    table = pkg.dequant.dequantize_fallback(w, qt, (V, K), torch.bfloat16)
    ids = torch.randint(-3, V + 3, (70000,), device=DEV)
    got = pkg.dequant.dequantize_rows(pkg.ops.GGMLTensor(w, tensor_type=qt, tensor_shape=torch.Size((V, K))), ids, torch.bfloat16)
    inside = (ids >= 0) & (ids < V)
    assert torch.equal(got[inside].view(torch.int16), table[ids[inside]].view(torch.int16))
    assert (got[~inside].view(torch.int16) == 0).all()


# ---------------------------------------------------------------- the layers
def _spy(pkg, monkeypatch, names):
    calls = []
    real = pkg.lib.lib()

    class Spy:
        def __getattr__(self, name):
            fn = getattr(real, name)
            if name in names:
                def wrapped(*a):
                    calls.append(name)
                    return fn(*a)
                return wrapped
            return fn
    monkeypatch.setattr(pkg.lib, "lib", lambda: Spy())
    return calls


def _layer(pkg, qt, N, K, seed, bias=True):
    raw, w = _packed(qt, N, K, seed=seed)
    w = pkg.ops.GGMLTensor(w.reshape(N, -1), tensor_type=qt, tensor_shape=torch.Size((N, K)))
    lin = pkg.ops.GGMLOps.Linear(K, N)
    sd = {"weight": w}
    if bias:
        sd["bias"] = pkg.ops.GGMLTensor(torch.randn(N, device=DEV) * 0.1, tensor_type=Q.F32, tensor_shape=torch.Size((N,)))
    lin.load_state_dict(sd)
    return lin, raw


ROUTE_NAMES = {"ggufb200_linear_fallback", "ggufb200_dequant_fallback", "ggufb200_gemm", "ggufb200_dequant", "ggufb200_linear"}


@pytest.mark.parametrize("M", [32, 77])
@pytest.mark.parametrize("qt", [Q.IQ2_XS, Q.MXFP4, Q.TQ2_0], ids=lambda q: q.name)
def test_layer_runs_the_fused_linear(pkg, monkeypatch, qt, M):
    """Where ggufb200_linear_fallback's AUTO decodes the weight in the kernel (M = 32 here) the layer makes that one call; where
    AUTO would take K1 + the dense GEMM (M = 77, past every type's crossover) the layer runs those two steps itself."""
    N, K = 256, 1024
    lin, raw = _layer(pkg, qt, N, K, seed=8)
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    route = pkg.lib.lib().ggufb200_linear_fallback_route(int(qt), M, N, K, BF16, 0)
    assert route == (ALGOS["fused_sync"] if M <= CROSSOVER[qt] else ALGOS["dequant_mma"])
    calls = _spy(pkg, monkeypatch, ROUTE_NAMES)
    y = lin(x)
    monkeypatch.undo()
    assert calls == (["ggufb200_linear_fallback"] if M <= CROSSOVER[qt] else ["ggufb200_dequant_fallback", "ggufb200_gemm"])
    W = torch.from_numpy(gguf_values(raw, qt).reshape(N, K)).to(DEV).to(torch.bfloat16).double()
    v, a, cls = reference(x.double(), W, lin.bias.as_subclass(torch.Tensor).to(torch.bfloat16).double())
    verdict = check(y, v, a, cls, BF16, "layer")
    assert verdict.ok, verdict.message


def test_embedding_gathers_rows(pkg, monkeypatch):
    qt, V, D = Q.IQ2_XXS, 151936 // 16, 2560
    raw, w = _packed(qt, V, D, seed=9)
    emb = pkg.ops.GGMLOps.Embedding(V, D, device="meta")
    emb.load_state_dict({"weight": pkg.ops.GGMLTensor(w.reshape(V, -1), tensor_type=qt, tensor_shape=torch.Size((V, D)))}, assign=True)
    ids = torch.randint(0, V, (2, 256), device=DEV)
    calls = _spy(pkg, monkeypatch, {"ggufb200_dequant_rows_fallback", "ggufb200_dequant_fallback", "ggufb200_dequant_rows"})
    got32, got16 = emb(ids), emb(ids, out_dtype=torch.float16)
    monkeypatch.undo()
    assert calls == ["ggufb200_dequant_rows_fallback"] * 2
    table = pkg.dequant.dequantize_fallback(w, qt, (V, D))
    want = torch.nn.functional.embedding(ids, table)
    assert got32.dtype == torch.float32 and torch.equal(got32, want)
    assert got16.dtype == torch.float16 and torch.equal(got16, want.to(torch.float16))


def test_layer_backward(pkg, monkeypatch):
    qt, N, K, M = Q.IQ3_S, 512, 2048, 48
    lin, _raw = _layer(pkg, qt, N, K, seed=10)
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    dy = torch.randn(M, N, device=DEV, dtype=torch.bfloat16)
    calls = _spy(pkg, monkeypatch, ROUTE_NAMES | {"ggufb200_linear_grad_input"})
    before = torch.cuda.memory_allocated()
    y = lin(x)
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    assert grown <= y.numel() * y.element_size() + (1 << 20), grown      # no [N, K] weight is kept for the backward
    y.backward(dy)
    monkeypatch.undo()
    assert calls == ["ggufb200_linear_fallback", "ggufb200_linear_grad_input"]
    wraw = lin.weight.as_subclass(torch.Tensor)
    want = pkg.ops.linear_grad_input(dy, wraw, qt, N, K, pkg.dequant.math_code(None, torch.bfloat16))
    assert torch.equal(x.grad.view(torch.int16), want.view(torch.int16))
    with torch.no_grad():
        assert torch.equal(y.view(torch.int16), lin(x).view(torch.int16))


def test_layer_wrapper_routes_views_by_block_alignment(pkg):
    """ops.linear_fallback leaves the alignment decision to the library: a view aligned to the type's blocks but not to 16 bytes
    still takes FUSED_SYNC (same bits as the aligned tensor), a view below the block alignment takes DEQUANT_MMA with that
    route's workspace (same bits as DEQUANT_MMA on the aligned tensor)."""
    qt, N, K, M = Q.IQ2_XS, 256, 1024, 32                  # A_BLK = gcd(74, 16) = 2
    raw, w = _packed(qt, N, K, seed=11)
    x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    assert pkg.lib.lib().ggufb200_linear_fallback_route(int(qt), M, N, K, BF16, 0) == ALGOS["fused_sync"]
    fused = pkg.ops.linear_fallback(x, w, qt, N, K, None)
    ws = _workspace(pkg, qt, M, N, K, BF16, ALGOS["dequant_mma"])
    two_step = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    assert _call(pkg, qt, w, N, K, x, K, BF16, two_step, N, ws=ws, algo=ALGOS["dequant_mma"]) == OK
    assert not torch.equal(fused, two_step)                # the two routes sum in different orders: the bits tell them apart
    buf = torch.zeros(raw.size + 32, dtype=torch.uint8, device=DEV)
    for shift, want in ((2, fused), (6, fused), (1, two_step), (3, two_step)):
        view = buf[shift:shift + raw.size]
        view.copy_(w)
        y = pkg.ops.linear_fallback(x, view, qt, N, K, None)
        assert torch.equal(y.view(torch.int16), want.view(torch.int16)), shift
