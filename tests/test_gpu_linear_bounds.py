"""Every route of the packed Linear, element by element, against a float64 product (bound and derivation:
tests/linear_bounds.py): GEMV, GEMV_FAST, FUSED_MMA, FUSED_TMEM (fast / EXACT_W / GENERIC producers; canonical rows, span-major
copy, straddled rows), DEQUANT_MMA and the dense GEMM, called through the C ABI into caller-owned buffers.

Beyond the bound: outputs start as NaN, so a tile that is never stored fails; bytes around the [M, N] view of Y (leading pad,
row pitch ldy > N, trailing rows) and past the workspace the route asked for must be left alone; activation padding [K, ldx)
and the rows after M hold NaN and must never reach the product; a workspace full of NaN (stale partials) must give the same
bits as a zeroed one; NaN / Inf injected into chosen weight blocks and activation rows must stay in their own output columns
and rows, with the NaN / Inf pattern of the float64 product."""
import functools

import numpy as np
import pytest
import torch

import linear_bounds as lb
import oracle
from util import Q

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = {lb.F16: 0x7D5A, lb.BF16: 0x7FA5}          # NaN patterns no kernel writes
USED = {}                                              # route -> largest fraction of the bound used


@pytest.fixture(scope="module", autouse=True)
def report_bound_use():
    yield
    if USED:
        print("\nlargest fraction of the per-element bound used, per route:")
        for k in sorted(USED):
            print(f"  {k:28s} {USED[k]:.3f}")


def _record(key, used):
    USED[key] = max(USED.get(key, 0.0), used)


@pytest.fixture(scope="module")
def hostf():
    L = lb.build_hostf()
    assert L is not None, "nvcc is needed to run the fast producers on the host"
    return L


@functools.lru_cache(maxsize=16)
def _raw(qt, N, K):
    bs, ts = oracle.type_info(int(qt))
    raw = oracle.random_blocks(int(qt), N * K // bs, seed=(int(qt) * 7919 + N * 31 + K) % 100003, scale=0.02).reshape(-1)
    raw.flags.writeable = False
    return raw


@functools.lru_cache(maxsize=8)
def _model(qt, N, K, act, model, hostf=None):
    raw = _raw(qt, N, K)
    if model == "gemv_fast":
        return lb.gemv_fast_model(raw, qt, N, K, act)
    if model == "fast":
        return lb.fast_weight(hostf, raw, qt, N, K, act), None
    return lb.exact_weight(raw, qt, N, K, act), None


def _weights(pkg, case, raw):
    """(packed bytes, span-major / block-major copy or None, dense act-dtype weight for the dense GEMM or None) on the GPU."""
    w = torch.from_numpy(np.array(raw)).to(DEV)
    spans = None
    L = pkg.lib.lib()
    if case.spans:
        spans = torch.empty(L.ggufb200_repack_bytes(int(case.qt), case.N, case.K), dtype=torch.uint8, device=DEV)
        assert L.ggufb200_repack(int(case.qt), w.data_ptr(), case.N, case.K, spans.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
    dense = None
    if case.route == "dense":
        dense = _model(case.qt, case.N, case.K, case.act, "exact")[0].to(lb.TORCH_ACT[case.act]).to(DEV).contiguous()
    return w, spans, dense


def _operands(case, seed=0):
    g = torch.Generator(device=DEV).manual_seed(case.M * 1009 + case.N * 17 + case.K + seed)
    dt = lb.TORCH_ACT[case.act]
    x = torch.randn(case.M, case.K, device=DEV, generator=g).to(dt)
    if case.bias == "none":
        return x, None, 0, None
    b32 = torch.randn(case.N, device=DEV, generator=g) * 0.1
    b_ref = lb.to_f64(b32.to(dt))                     # the kernels round the bias to the activation dtype first
    if case.bias == "f32":
        return x, b32, oracle.DT_F32, b_ref
    return x, b32.to(dt), case.act, b_ref


def _launch(pkg, case, w, spans, dense, X, ldx, bias, bias_code, Y, ldy, ws, ws_bytes):
    L = pkg.lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    b = bias.data_ptr() if bias is not None else None
    if case.route == "dense":
        return L.ggufb200_gemm(dense.data_ptr(), case.N, case.K, case.K, X, case.M, ldx, case.act, b, bias_code, Y, ldy, st)
    if spans is not None:
        return L.ggufb200_linear_spans(int(case.qt), w.data_ptr(), spans.data_ptr(), case.N, case.K, X, case.M, ldx, case.act, oracle.DT_F16,
                                       b, bias_code, Y, ldy, ws, ws_bytes, case.algo, st)
    return L.ggufb200_linear(int(case.qt), w.data_ptr(), case.N, case.K, X, case.M, ldx, case.act, oracle.DT_F16, b, bias_code, Y, ldy,
                             ws, ws_bytes, case.algo, st)


def _reference(case, x, b_ref, raw=None, hostf=None):
    if raw is None:
        W, mag = _model(case.qt, case.N, case.K, case.act, case.weight_model, hostf if case.weight_model == "fast" else None)
    elif case.weight_model == "gemv_fast":
        W, mag = lb.gemv_fast_model(raw, case.qt, case.N, case.K, case.act)
    elif case.weight_model == "fast":
        W, mag = lb.fast_weight(hostf, raw, case.qt, case.N, case.K, case.act), None
    else:
        W, mag = lb.exact_weight(raw, case.qt, case.N, case.K, case.act), None
    W = W.to(DEV)
    return lb.reference(lb.to_f64(x), W, b_ref, None if mag is None else mag.to(DEV)), W


# ---------------------------------------------------------------- 1. every element within the bound
@pytest.mark.parametrize("case", lb.CASES, ids=lambda c: c.id)
def test_every_element_within_the_bound(pkg, hostf, case):
    L = pkg.lib.lib()
    raw = _raw(case.qt, case.N, case.K)
    w, spans, dense = _weights(pkg, case, raw)
    x, bias, bias_code, b_ref = _operands(case)
    Y = torch.full((case.M, case.N), float("nan"), dtype=lb.TORCH_ACT[case.act], device=DEV)
    need = lb.workspace_bytes(L, case)
    ws = torch.zeros(max(need, 16), dtype=torch.uint8, device=DEV)
    rc = _launch(pkg, case, w, spans, dense, x.data_ptr(), case.K, bias, bias_code, Y.data_ptr(), case.N, ws.data_ptr(), need)
    assert rc == 0, (case.id, L.ggufb200_strerror(rc))
    (v, a, cls), _W = _reference(case, x, b_ref, hostf=hostf)
    verdict = lb.check(Y, v, a, cls, case.act, case.id)
    _record(case.route + (f"-{case.producers}" if case.producers else ""), verdict.used)
    assert verdict.ok, verdict.message


# ---------------------------------------------------------------- 2. guarded memory
GUARDED = [
    lb.Case("gemv", Q.Q4_K, 5, 130, 1024, lb.BF16, "f32"),
    lb.Case("gemv", Q.Q6_K, 8, 136, 1024, lb.F16, "act"),
    lb.Case("gemv_fast", Q.Q5_K, 8, 264, 1024, lb.F16, "f32"),
    lb.Case("gemv_fast", Q.Q4_K, 3, 13, 4096, lb.BF16, "act"),
    lb.Case("fused_mma", Q.Q4_K, 64, 520, 4096, lb.BF16, "f32"),                  # split K
    lb.Case("fused_mma", Q.Q6_K, 300, 264, 1024, lb.F16, "none"),
    lb.Case("tmem", Q.Q4_K, 33, 264, 4096, lb.F16, "f32", "fast"),                 # split K, 128-token items
    lb.Case("tmem", Q.Q8_0, 5, 520, 12288, lb.BF16, "act", "exact"),               # split K, 32-token items
    lb.Case("tmem", Q.Q5_1, 385, 136, 320, lb.BF16, "f32", "generic", flags=lb.FLAG_TILE384),
    lb.Case("tmem", Q.Q3_K, 129, 248, 1024, lb.F16, "act", "fast", spans=True),
    lb.Case("tmem", Q.Q4_K, 200, 640, 320, lb.BF16, "f32", "fast"),               # straddled rows
    lb.Case("tmem", Q.Q6_K, 31, 320, 640, lb.F16, "none", "exact", spans=True),    # straddled rows, block-major copy
    lb.Case("dequant_mma", Q.Q5_0, 300, 248, 1024, lb.F16, "f32"),
    lb.Case("dequant_mma", Q.Q4_K, 9, 2560, 320, lb.BF16, "act"),                  # straddled rows
    lb.Case("dense", Q.Q8_0, 129, 120, 1024, lb.BF16, "f32"),
]


@pytest.mark.parametrize("case", GUARDED, ids=lambda c: c.id)
def test_guarded_memory(pkg, hostf, case):
    L = pkg.lib.lib()
    M, N, K = case.M, case.N, case.K
    dt = lb.TORCH_ACT[case.act]
    raw = _raw(case.qt, N, K)
    w, spans, dense = _weights(pkg, case, raw)
    x, bias, bias_code, b_ref = _operands(case, seed=1)
    # X: row pitch K + 16, NaN in [K, ldx) and in two rows after M
    ldx = K + 16
    xbuf = torch.full((M + 2, ldx), float("nan"), dtype=dt, device=DEV)
    xbuf[:M, :K] = x
    # Y: a view inside a sentinel-filled buffer -- 8-element lead, pitch N + 8 or N + 24, three trailing rows
    lead, ldy = 8, N + (8 if N % 2 else 24)
    ybuf = torch.empty(lead + (M + 3) * ldy, dtype=torch.int16, device=DEV)
    inside = torch.zeros(ybuf.numel(), dtype=torch.bool, device=DEV)
    inside[lead:lead + M * ldy].view(M, ldy)[:, :N] = True
    need = lb.workspace_bytes(L, case)
    tail = 4096
    wsbuf = torch.empty(need + tail, dtype=torch.uint8, device=DEV)
    if case.route in ("fused_mma", "tmem") and case.M <= 64 and not case.straddled:
        assert lb.plan(L, case, need)[1] > 1, "meant to cover the split-K finalize"
    results = []
    for stale in (False, True):
        ybuf.fill_(SENTINEL[case.act])
        wsbuf[:need].fill_(0xFF if stale else 0)                 # 0xFFFFFFFF: an fp32 NaN in every partial slot
        wsbuf[need:].fill_(0xA5)
        rc = _launch(pkg, case, w, spans, dense, xbuf.data_ptr(), ldx, bias, bias_code, ybuf.data_ptr() + 2 * lead, ldy,
                     wsbuf.data_ptr() if need else None, need)
        assert rc == 0, (case.id, L.ggufb200_strerror(rc))
        torch.cuda.synchronize()
        assert bool((wsbuf[need:] == 0xA5).all()), "bytes past the workspace the route asked for were written"
        assert bool((ybuf[~inside] == SENTINEL[case.act]).all()), f"bytes of Y outside the [M, N] view changed (stale workspace: {stale})"
        results.append(ybuf[inside].clone())
    assert torch.equal(results[0], results[1]), "a workspace holding stale partials changed the result"
    y = results[0].view(dt).view(M, N)
    (v, a, cls), _W = _reference(case, x, b_ref, hostf=hostf)
    verdict = lb.check(y, v, a, cls, case.act, case.id)
    assert verdict.ok, verdict.message


# ---------------------------------------------------------------- 3. non-finite containment
NAN16, INF16 = 0x7E00, 0x7C00


def _poke(blocks, b, kind):
    """Q4_K block b: NaN d | +Inf d with non-zero quants | +Inf d with zero quants | dmin = +Inf."""
    blk = blocks[b]
    if kind == "nan_d":
        blk[0:2] = np.frombuffer(np.uint16(NAN16).tobytes(), np.uint8)
    elif kind in ("inf_d", "inf_d_zero_q"):
        blk[0:2] = np.frombuffer(np.uint16(INF16).tobytes(), np.uint8)
        blk[4:16] = 0x05                                  # every 6-bit scale non-zero: D = Inf, not Inf * 0
        blk[16:144] = 0x11 if kind == "inf_d" else 0
    elif kind == "inf_dmin":
        blk[2:4] = np.frombuffer(np.uint16(INF16).tobytes(), np.uint8)


KINDS = ("nan_d", "inf_d", "inf_d_zero_q", "inf_dmin")
NONFINITE = [
    lb.Case("gemv", Q.Q4_K, 5, 264, 4096, lb.F16, "f32"),
    lb.Case("gemv_fast", Q.Q4_K, 5, 264, 4096, lb.BF16, "f32"),
    lb.Case("fused_mma", Q.Q4_K, 64, 264, 4096, lb.BF16, "act"),
    lb.Case("dequant_mma", Q.Q4_K, 300, 264, 4096, lb.F16, "none"),
    lb.Case("tmem", Q.Q4_K, 33, 264, 4096, lb.BF16, "f32", "fast"),
    lb.Case("tmem", Q.Q4_K, 33, 264, 4096, lb.F16, "f32", "exact"),
    lb.Case("tmem", Q.Q4_K, 300, 264, 4096, lb.BF16, "none", "generic"),
    lb.Case("tmem", Q.Q4_K, 200, 640, 320, lb.F16, "f32", "fast"),                 # straddled
    lb.Case("tmem", Q.Q4_K, 200, 640, 320, lb.BF16, "act", "exact"),               # straddled
    lb.Case("dequant_mma", Q.Q4_K, 40, 640, 320, lb.BF16, "f32"),                  # straddled
]


def _injections(pkg, case):
    """(block index, kind) pairs: a row of the last partial feature tile; the last span of the first (non-final) K range;
    a block interior to a 128-row producer tile; a dmin; and for straddled rows blocks shared by two rows."""
    per_row = case.K // 256
    if case.straddled:
        # (640, 320): block 6 = elements 1536..1791 (rows 4 and 5), 11 (rows 8, 9), 16 (rows 12, 13), 797 (rows 637, 638)
        return list(zip((6, 11, 16, 797), KINDS))
    L = pkg.lib.lib()
    span = per_row // 2
    if case.route in ("fused_mma", "tmem"):
        _rows, ranges, kb, _c = lb.plan(L, case, lb.workspace_bytes(L, case))
        if ranges > 1:
            span = kb // 4 - 1
    return [((case.N - 3) * per_row, "nan_d"), (10 * per_row + span, "inf_d"), (77 * per_row + 7, "inf_d_zero_q"),
            (150 * per_row + 3, "inf_dmin")]


@pytest.mark.parametrize("case", NONFINITE, ids=lambda c: c.id)
def test_nonfinite_values_stay_in_their_rows_and_columns(pkg, hostf, case):
    L = pkg.lib.lib()
    M, N, K = case.M, case.N, case.K
    raw = np.array(_raw(case.qt, N, K)).reshape(-1, 144)
    for b, kind in _injections(pkg, case):
        _poke(raw, b, kind)
    raw = raw.reshape(-1)
    w, spans, dense = _weights(pkg, case, raw)
    x, bias, bias_code, b_ref = _operands(case, seed=2)
    x[1, 100] = float("nan")
    x[M - 1, K - 7] = float("inf")
    Y = torch.full((M, N), float("nan"), dtype=lb.TORCH_ACT[case.act], device=DEV)
    need = lb.workspace_bytes(L, case)
    ws = torch.zeros(max(need, 16), dtype=torch.uint8, device=DEV)
    rc = _launch(pkg, case, w, spans, dense, x.data_ptr(), K, bias, bias_code, Y.data_ptr(), N, ws.data_ptr(), need)
    assert rc == 0, (case.id, L.ggufb200_strerror(rc))
    (v, a, cls), W = _reference(case, x, b_ref, raw=raw, hostf=hostf)
    bad_cols = ~torch.isfinite(W).all(1)
    bad_rows = ~torch.isfinite(lb.to_f64(x)).all(1)
    assert int(bad_cols.sum()) >= 4 and int(bad_rows.sum()) == 2
    assert int((cls == lb.FIN).sum()) > 0.9 * (M - 2) * (N - 8)
    if case.route == "gemv_fast":
        # scales applied to partial sums: which non-finite value comes out may differ from the float64 product, where it
        # appears may not
        verdict = lb.check(Y, v, a, cls, case.act, case.id, match_nonfinite=False)
        nonfinite = ~torch.isfinite(Y.double())
        assert not bool((nonfinite & ~(bad_rows[:, None] | bad_cols[None, :])).any()), "a non-finite value left its row / column"
    else:
        verdict = lb.check(Y, v, a, cls, case.act, case.id)
    assert verdict.ok, verdict.message


# ---------------------------------------------------------------- 4. AUTO through the layer, both numerics contracts
@pytest.mark.parametrize("numerics", ["exact", "fast"])
@pytest.mark.parametrize("qt,M,N,K,act", [(Q.Q4_K, 5, 264, 1024, lb.BF16), (Q.Q4_K, 300, 264, 1024, lb.F16), (Q.Q5_K, 129, 136, 4096, lb.BF16),
                                          (Q.Q5_K, 8, 520, 4096, lb.F16), (Q.Q6_K, 33, 520, 1024, lb.F16), (Q.Q8_0, 1, 130, 256, lb.BF16)],
                         ids=lambda v: v.name if isinstance(v, Q) else None)
def test_auto_route_through_the_layer(pkg, hostf, numerics, qt, M, N, K, act):
    raw = _raw(qt, N, K)
    bs, ts = oracle.type_info(int(qt))
    lin = pkg.ops.GGMLOps.Linear(K, N)
    b32 = torch.randn(N, generator=torch.Generator().manual_seed(N)) * 0.1
    w = pkg.ops.GGMLTensor(torch.from_numpy(np.array(raw)).to(DEV).view(N, K // bs * ts), tensor_type=qt, tensor_shape=torch.Size((N, K)))
    lin.load_state_dict({"weight": w, "bias": pkg.ops.GGMLTensor(b32.to(DEV), tensor_type=Q.F32, tensor_shape=torch.Size((N,)))})
    lin.linear_numerics = numerics
    case = lb.Case("auto", qt, M, N, K, act, "f32")
    x, _b, _c, _r = _operands(case)
    y = lin(x)
    # the route the contract implies (api.cu pick_route, ops.py span copy): M <= 8 -> the integer-pattern GEMV (`fast`, Q4_K /
    # Q5_K) or the mma.sync GEMV; M > 8 -> FUSED_TMEM with the fast or the reference-sequence producers.  The layer must give
    # exactly that route's bits, and y is checked against that route's weight model only.
    L = pkg.lib
    fast = numerics == "fast"
    if M <= 8:
        algo, model = (L.ALGO_GEMV_FAST, "gemv_fast") if fast and qt in (Q.Q4_K, Q.Q5_K) else (L.ALGO_GEMV, "exact")
    else:
        algo, model = L.ALGO_FUSED_TMEM | (0 if fast else L.FLAG_EXACT_W), "fast" if fast else "exact"
    y_route = pkg.ops.linear_packed(x, w, b32.to(DEV), None, algo, use_spans=M > 8 and qt == Q.Q6_K)
    assert torch.equal(y, y_route), f"AUTO ({numerics}) did not take route {algo:#x}"
    b_ref = lb.to_f64(b32.to(DEV).to(lb.TORCH_ACT[act]))
    W, mag = _model(qt, N, K, act, model, hostf if model == "fast" else None)
    v, a, cls = lb.reference(lb.to_f64(x), W.to(DEV), b_ref, None if mag is None else mag.to(DEV))
    verdict = lb.check(y, v, a, cls, act, f"AUTO {numerics} vs the {model} weight")
    _record(f"auto-{numerics}", verdict.used)
    assert verdict.ok, verdict.message
