"""CPU checks of tests/linear_bounds.py: the rounding helper against brute force, the fast-weight model against an
independent float64 evaluation on raw random bytes, and the case list against the fused kernels' own plans."""
import ctypes

import numpy as np
import pytest
import torch

import linear_bounds as lb
import oracle
from util import Q


# ---------------------------------------------------------------- round_act against brute force
def _grid(act):
    """Every finite value of the 16-bit format, ascending, with +Inf as the even neighbour past the largest finite one."""
    bits = np.arange(0x8000, dtype=np.uint16)           # non-negative patterns
    if act == lb.F16:
        vals = bits.view(np.float16).astype(np.float64)
    else:
        with np.errstate(invalid="ignore"):
            vals = (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    fin = np.isfinite(vals)
    return vals[fin], bits[fin]


def _brute(v, act):
    """Nearest grid value, ties to the even bit pattern, past the largest finite value + half an ulp: Inf."""
    vals, bits = _grid(act)
    top = 2.0 ** 16 if act == lb.F16 else 2.0 ** 128        # the next "value" after the largest finite one (even pattern 0x7C00 / 0x7F80)
    vals = np.append(vals, top)
    bits = np.append(bits, np.uint16(0x7C00 if act == lb.F16 else 0x7F80))
    a = np.abs(v)
    i = np.clip(np.searchsorted(vals, a), 1, len(vals) - 1)
    lo, hi = vals[i - 1], vals[i]
    pick_hi = (hi - a < a - lo) | ((hi - a == a - lo) & (bits[i] % 2 == 0))
    r = np.where(a >= hi, hi, np.where(pick_hi, hi, lo))
    r = np.where(a <= vals[0], vals[0], r)
    r = np.where(r == top, np.inf, r)
    return np.copysign(r, v)


@pytest.mark.parametrize("act", [lb.F16, lb.BF16], ids=["f16", "bf16"])
def test_round_act_equals_brute_force(act):
    vals, _ = _grid(act)
    top = 2.0 ** 16 if act == lb.F16 else 2.0 ** 128
    ext = np.append(vals, top)
    mids = (ext[:-1] + ext[1:]) / 2                                 # exact in float64: every tie, overflow threshold included
    eps = np.spacing(np.abs(mids)) * 4
    pts = np.concatenate([vals, mids, mids - eps, mids + eps, [top * 1.5, 1e300, np.spacing(0.0)]])
    pts = np.concatenate([pts, -pts])
    got = lb.round_act(torch.from_numpy(pts), act).numpy()
    want = _brute(pts, act)
    assert np.array_equal(got, want), pts[got != want][:8]
    # torch's own conversion of a value that is exact in fp32 is a correct single rounding: a second opinion
    p32 = pts[np.abs(pts) < 3e38].astype(np.float32).astype(np.float64)
    assert np.array_equal(lb.round_act(torch.from_numpy(p32), act).numpy(),
                          torch.from_numpy(p32).float().to(lb.TORCH_ACT[act]).double().numpy())
    special = torch.tensor([float("inf"), float("-inf"), float("nan"), 0.0, -0.0], dtype=torch.float64)
    r = lb.round_act(special, act)
    assert r[0] == float("inf") and r[1] == float("-inf") and torch.isnan(r[2]) and r[3] == 0 and r[4] == 0
    # named edges: the largest finite value, the first tie that overflows, the smallest subnormal and half of it (a tie to 0)
    big, sub = (65504.0, 2.0 ** -24) if act == lb.F16 else (float(torch.finfo(torch.bfloat16).max), 2.0 ** -133)
    over = 65520.0 if act == lb.F16 else 2.0 ** 127 * (2 - 2 ** -8)
    r = lb.round_act(torch.tensor([big, over, np.nextafter(over, 0), sub, sub / 2, sub * 0.75], dtype=torch.float64), act).tolist()
    assert r == [big, float("inf"), big, sub, 0.0, sub]


def test_check_reports_class_and_bound():
    """The check itself: an element one output ulp past the interval fails, a moved NaN fails, the fraction is reported."""
    x = torch.tensor([[1.0, 2.0], [3.0, float("nan")]], dtype=torch.float64)
    W = torch.tensor([[0.5, 0.25], [1.0, -1.0]], dtype=torch.float64)
    v, a, cls = lb.reference(x, W)
    assert cls.tolist() == [[lb.FIN, lb.FIN], [lb.NAN, lb.NAN]]
    y = torch.tensor([[1.0, -1.0], [float("nan"), float("nan")]], dtype=torch.float64)
    assert lb.check(y, v, a, cls, lb.F16).ok
    y2 = y.clone()
    y2[0, 0] = 1.0 + 2 ** -10
    assert not lb.check(y2, v, a, cls, lb.F16).ok
    y3 = y.clone()
    y3[1, 0] = 0.0
    assert not lb.check(y3, v, a, cls, lb.F16).ok
    Winf = W.clone()
    Winf[0, 0] = float("inf")
    assert lb.classes(x[:1], Winf).tolist() == [[lb.PINF, lb.FIN]]
    Winf[0, 1] = float("-inf")
    assert lb.classes(x[:1], Winf).tolist() == [[lb.NAN, lb.FIN]]
    assert lb.classes(torch.zeros(1, 2, dtype=torch.float64), Winf).tolist() == [[lb.NAN, lb.FIN]]      # Inf * 0


# ---------------------------------------------------------------- the fast-weight model on raw random bytes
@pytest.fixture(scope="module")
def hostf():
    L = lb.build_hostf()
    if L is None:
        pytest.skip("nvcc not available")
    return L


def _f16(bits):
    return bits.view(np.float16).astype(np.float64)


@pytest.mark.parametrize("qt", [Q.Q4_K, Q.Q5_K], ids=lambda q: q.name)
def test_fast_producers_on_raw_random_bytes(hostf, qt):
    """FastProducer<Q> (FMA step) on random bytes in every header field: each element is fp16(D*q - M) of the float64 model,
    NaN positions included.  Against the reference's fp16(fp16(D*q) - M) the NaN / Inf pattern differs only at fp16
    overflow: where the reference's intermediate fp16(D*q) overflows, the fused step is finite (M finite) or +-Inf (M
    infinite, where the reference has Inf - Inf = NaN); and where the exact step lies past 65504 but the reference's
    rounded intermediate keeps it finite.  The fused step is never NaN where the reference is not (DESIGN.md section 3)."""
    n = 4096
    ts = oracle.type_info(int(qt))[1]
    raw = np.random.default_rng(int(qt) + 40).integers(0, 256, size=n * ts, dtype=np.uint8)
    got = lb.fast_bits(hostf, raw, qt)
    want = lb.fma_model(raw, qt)
    g, w = _f16(got), _f16(want)
    assert np.array_equal(np.isnan(g), np.isnan(w))
    assert np.array_equal(got[~np.isnan(g)], want[~np.isnan(w)])
    assert np.isnan(g).sum() > 100 and np.isinf(g).sum() > 100           # the bytes do reach the non-finite cases
    ref = _f16(oracle.dequant(raw, int(qt), oracle.DT_F16, oracle.DT_F16))
    q, D, Mm = lb.k_quant_parts(raw, qt)
    with np.errstate(all="ignore"):
        prod_overflows = (np.isinf((D * q).astype(np.float16).astype(np.float64)) & np.isfinite(D * q)).reshape(-1)
        step_overflows = (np.abs(D * q - Mm) >= 65520.0).reshape(-1)           # the exact step rounds to +-Inf
    same_nan = np.isnan(g) == np.isnan(ref)
    same_inf = np.where(np.isinf(g) | np.isinf(ref), g == ref, True)
    differs = ~(same_nan & same_inf)
    assert differs.sum() > 100
    assert np.all((prod_overflows | step_overflows)[differs]), "fast and reference non-finite patterns differ away from fp16 overflow"
    assert not np.any(np.isnan(g) & ~np.isnan(ref)), "the fused step is NaN only where the reference is"
    both = np.isfinite(g) & np.isfinite(ref)
    with np.errstate(all="ignore"):
        prod = np.abs(D * q).reshape(-1)[both].astype(np.float16)
        bound = 0.5 * np.spacing(prod).astype(np.float64) + np.spacing(np.maximum(np.abs(g[both]), np.abs(ref[both])).astype(np.float16)).astype(np.float64)
    assert np.all(np.abs(g[both] - ref[both]) <= bound)


@pytest.mark.parametrize("qt", [Q.Q4_K, Q.Q5_K], ids=lambda q: q.name)
def test_gemv_fast_model_against_the_reference_weight(qt):
    """W = D*q - M of the GEMV_FAST model against the oracle's fp16 chain fp16(fp16(D*q) - M) (oracle/gguf_oracle.c): equal
    where q = 0 (then the chain is -M, exact) and, rounded once, where M = 0; elsewhere apart by at most the chain's two
    roundings."""
    N, K = 64, 1024
    raw = oracle.random_blocks(int(qt), N * K // 256, seed=3, scale=0.02)
    W, mag = lb.gemv_fast_model(raw, qt, N, K, lb.F16)
    W = W.numpy().reshape(-1)
    ref = _f16(oracle.dequant(raw, int(qt), oracle.DT_F16, oracle.DT_F16))
    q = oracle.unpack_int(raw, int(qt))[0].astype(np.float64)
    zero_q = q == 0
    assert zero_q.sum() > 100 and np.array_equal(W[zero_q], ref[zero_q])
    mn = oracle.unpack_int(raw, int(qt))[2]
    zero_m = (mn == 0) & ~zero_q
    assert zero_m.sum() > 100 and np.array_equal(W[zero_m].astype(np.float16).astype(np.float64), ref[zero_m])
    _q, D, _M = lb.k_quant_parts(raw, qt)
    half = lambda v: 0.5 * np.spacing(np.abs(v).astype(np.float16)).astype(np.float64)
    assert np.all(np.abs(W - ref) <= half((D * _q).reshape(-1)) + half(ref))
    assert np.all(mag.numpy().reshape(-1) >= np.abs(W))


@pytest.mark.parametrize("act", [lb.F16, lb.BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("qt", [Q.Q4_K, Q.Q5_K], ids=lambda q: q.name)
def test_gemv_fast_bound_rejects_a_zeroed_output_and_a_dropped_sub_block(qt, act):
    """The GEMV_FAST bound is tight enough to pin the route: the correctly rounded product passes, an all-zero output and an
    output missing one 32-element sub-block of K fail."""
    M, N, K = 8, 264, 4096
    raw = oracle.random_blocks(int(qt), N * K // 256, seed=int(qt) + act, scale=0.02)
    W, mag = lb.gemv_fast_model(raw, qt, N, K, act)
    x = lb.to_f64(torch.randn(M, K, generator=torch.Generator().manual_seed(act)).to(lb.TORCH_ACT[act]))
    v, a, cls = lb.reference(x, W, None, mag)
    good = lb.check(lb.round_act(v, act), v, a, cls, act, "rounded product")
    assert good.ok and good.used == 0.0, good.message
    assert float((a / v.abs()).median()) < 0.5
    assert not lb.check(torch.zeros_like(v), v, a, cls, act).ok
    sb = slice(37 * 32, 38 * 32)
    dropped = lb.round_act(v - x[:, sb] @ W[:, sb].T, act)
    assert not lb.check(dropped, v, a, cls, act).ok


# ---------------------------------------------------------------- the case list reaches what it claims
def test_case_list_covers_the_routes_and_their_plans(pkg):
    L = pkg.lib.lib()
    cases = lb.CASES
    assert len({c.id for c in cases}) == len(cases)
    for route in ("gemv", "fused_mma", "tmem", "dequant_mma"):
        assert {c.qt for c in cases if c.route == route} == set(lb.ALL12), route
    assert {c.qt for c in cases if c.route == "gemv_fast"} == {Q.Q4_K, Q.Q5_K}
    assert {c.M for c in cases if c.route == "tmem"} == set(lb.M_ALL) == {c.M for c in cases if c.route == "fused_mma"}
    assert {c.N for c in cases} >= set(lb.N_GEMV)
    assert {c.K for c in cases} >= set(lb.K_ALL) | {320}
    assert {(c.N, c.K) for c in cases if c.route == "tmem" and c.straddled and c.qt == Q.Q4_K} == set(lb.STRADDLED)
    assert {(c.N, c.K) for c in cases if c.route == "tmem" and c.straddled and c.qt == Q.Q6_K} == set(lb.STRADDLED)
    assert {c.producers for c in cases if c.route == "tmem"} == set(lb.PRODUCERS)
    assert {(c.act, c.bias) for c in cases} == {(a, b) for a in (lb.F16, lb.BF16) for b in lb.BIAS_KINDS}
    for c in cases:
        bs = oracle.type_info(int(c.qt))[0]
        assert c.K % bs == 0 or (c.route in ("tmem", "dequant_mma") and c.N * c.K % 256 == 0 and c.K % 64 == 0), c.id
        assert c.route not in ("gemv", "gemv_fast") or c.M <= 8
    tokens, ranges = {}, {"tmem": [], "fused_mma": []}
    ragged_span = partial_tile = 0
    for c in cases:
        if c.route not in ("tmem", "fused_mma"):
            continue
        rows, k_ranges, kb, ctas = lb.plan(L, c, lb.workspace_bytes(L, c))
        ranges[c.route].append(k_ranges)
        if c.route == "tmem":
            tokens.setdefault(rows, c.id)
            ragged_span += c.K % 256 != 0
            partial_tile += c.N % 128 != 0
    assert set(tokens) == {32, 128, 192, 384}, tokens
    assert max(ranges["tmem"]) > 1 and max(ranges["fused_mma"]) > 1, ranges
    assert ragged_span and partial_tile
