"""CPU checks of the patched-route bound of tests/lora_bounds.py (`lora_reference`): it reduces to the unpatched bound, it
accepts the correctly rounded product, and it rejects each fault the patched FUSED_TMEM kernel could plausibly make -- a tile
missing one LoRA k-block, the LoRA k-blocks added once per K range, the tile table ignored, the feature scale applied twice
or after the bias, U fed to a bf16 MMA as its fp16 value.  Also: the operands the layer builds for the kernel
(`ops.lora_kernel_operands`) against a restatement, and the case list of tests/test_gpu_lora_bounds.py against the kernel's
own plans."""
import functools

import numpy as np
import pytest
import torch

import linear_bounds as lb
import lora_bounds as lob
from util import Q


@functools.lru_cache(maxsize=4)
def _weight(qt, N, K, act):
    return lb.exact_weight(lob.random_weight(qt, N, K), qt, N, K, act)


@functools.lru_cache(maxsize=4)
def _simulated(case):
    """Operands, bound and the float64 pieces of the product: (ops, v, a, cls, main = x.W^T, lora = T.Û^T with the table)."""
    W = _weight(case.qt, case.N, case.K, case.act)
    ops = lob.lora_operands(case, float(W.pow(2).mean().sqrt()))
    x = lb.to_f64(ops.x)
    v, a, cls = lob.lora_reference(x, W, ops.T, ops.U, case.act, ops.b_ref, ops.scale, ops.tiles)
    Uh, _run = lob.lora_u_model(ops.U, case.act, ops.tiles)
    return ops, v, a, cls, x @ W.T, lb.to_f64(ops.T) @ Uh.T


def _assemble(case, main, lora, ops):
    """r * (main + lora) + b in float64, rounded once to the activation dtype: the kernel's output without a fault."""
    v = main + lora
    if ops.scale is not None:
        v = v * lb.to_f64(ops.scale)[None, :]
    if ops.b_ref is not None:
        v = v + ops.b_ref[None, :]
    return v


# the cases whose float64 product is cheap on the CPU, and two more that bring the faults the list draws rarely together
FAULT_CASES = [c for c in lob.LORA_CASES if c.M * c.N * (c.K + 64 * c.J) <= 40e6] + [
    lob.LoraCase(Q.Q4_K, 128, 264, 256, lb.BF16, 1, "banded", "r", "f32", "exact"),
    lob.LoraCase(Q.Q8_0, 77, 520, 1024, lb.BF16, 2, "banded", "r", "act", "exact"),
]


def _dropped_kblock(case, ops):
    """(tile, k-block) of the first tile that runs a k-block whose U columns are not all zero on it, or None."""
    if ops.tiles is None:
        return (0, 0)
    for i, (f, c) in enumerate(lob.clamp_tiles(ops.tiles, case.J)):
        if c > 0 and 128 * i < case.N:
            return (i, f)
    return None


def _fault(case, kind):
    """The kernel's output under fault `kind`, or None where the fault cannot arise in this case."""
    ops, v, a, cls, main, lora = _simulated(case)
    if kind == "dropped_kblock":
        hit = _dropped_kblock(case, ops)
        if hit is None:
            return None
        i, j = hit
        U = ops.U.clone()
        U[128 * i:128 * i + 128, 64 * j:64 * j + 64] = 0
        Uh, _run = lob.lora_u_model(U, case.act, ops.tiles)
        return _assemble(case, main, lb.to_f64(ops.T) @ Uh.T, ops)
    if kind == "lora_per_range":
        if not bool(lora.any()):
            return None
        return _assemble(case, main, 2 * lora, ops)                # split K: every K range adds the k-blocks (two ranges)
    if kind == "table_ignored":
        Uall, _run = lob.lora_u_model(ops.U, case.act, None)
        lora_all = lb.to_f64(ops.T) @ Uall.T
        if ops.tiles is None or torch.equal(lora_all, lora):
            return None
        return _assemble(case, main, lora_all, ops)
    if kind in ("scale_twice", "scale_after_bias"):
        if ops.scale is None or (kind == "scale_after_bias" and ops.b_ref is None):
            return None
        r = lb.to_f64(ops.scale)
        y = _assemble(case, main, lora, ops)
        if kind == "scale_twice":
            n = int(((r - 1).abs() * (main + lora).abs().amax(0)).argmax())
            y[:, n] = r[n] * r[n] * (main + lora)[:, n] + (0 if ops.b_ref is None else ops.b_ref[n])
        else:
            n = int(((r - 1).abs() * ops.b_ref.abs()).argmax())
            y[:, n] = r[n] * ((main + lora)[:, n] + ops.b_ref[n])
        return y
    if kind == "u_as_fp16":
        # the rounding of U to bf16 is a relative change of 2^-9 at most, against a bound that grows with K' and the rank:
        # visible only for short K' and a single k-block (here K' sqrt(R) <= 3000: K <= 256 + 64 at J = 1)
        if case.act != lb.BF16 or not bool(lora.any()) or (case.K + 64 * case.J) * np.sqrt(case.R) > 3e3:
            return None
        Uh, _run = lob.lora_u_model(ops.U, lb.F16, ops.tiles)          # fp16(U) as it is, no cast to bf16
        return _assemble(case, main, lb.to_f64(ops.T) @ Uh.T, ops)
    raise AssertionError(kind)


FAULTS = ("dropped_kblock", "lora_per_range", "table_ignored", "scale_twice", "scale_after_bias", "u_as_fp16")


@pytest.mark.parametrize("case", FAULT_CASES, ids=lambda c: c.id)
def test_the_correctly_rounded_product_is_accepted(case):
    ops, v, a, cls, main, lora = _simulated(case)
    y = lb.round_act(_assemble(case, main, lora, ops), case.act)
    verdict = lb.check(y, v, a, cls, case.act, case.id)
    assert verdict.ok and verdict.used < 1e-6, verdict.message
    # the sizing the faults rely on: the LoRA term is of the order of x.W^T (or switched off by the table)
    if bool(lora.any()):
        ratio = float(lora.pow(2).mean().sqrt() / main.pow(2).mean().sqrt())
        assert 0.05 < ratio < 20, ratio


@pytest.mark.parametrize("kind", FAULTS)
def test_every_fault_is_rejected(kind):
    hits = 0
    for case in FAULT_CASES:
        y = _fault(case, kind)
        if y is None:
            continue
        hits += 1
        _ops, v, a, cls, _m, _l = _simulated(case)
        verdict = lb.check(lb.round_act(y, case.act), v, a, cls, case.act, f"{kind} {case.id}")
        assert not verdict.ok, f"fault {kind} passes the bound in {case.id}: {verdict.message}"
    assert hits >= 2, f"fault {kind} arises in {hits} case(s) only"


def test_without_lora_and_scale_it_is_the_unpatched_bound():
    """J = 0, r = None: `reference` exactly.  r = 1: the same value and classes, and the bound grows by u |v| only.  J = 1
    with U = 0: the same value and classes, and the bound's first term is taken over K' = K + 64."""
    case = lob.LoraCase(Q.Q4_K, 33, 264, 1024, lb.F16, 1, "none", "none", "f32", "exact")
    W = _weight(case.qt, case.N, case.K, case.act)
    ops = lob.lora_operands(case, float(W.pow(2).mean().sqrt()))
    x = lb.to_f64(ops.x)
    x[3, 5] = float("nan")
    want = lb.reference(x, W, ops.b_ref)
    got = lob.lora_reference(x, W, None, None, case.act, ops.b_ref)
    assert all(torch.equal(g, w) for g, w in zip(got, want))
    one = lob.lora_reference(x, W, None, None, case.act, ops.b_ref, torch.ones(case.N))
    assert torch.equal(one[0], want[0]) and torch.equal(one[2], want[2])
    assert torch.allclose(one[1], want[1] + lb.U * want[0].abs(), rtol=1e-15, atol=0)
    zero = lob.lora_reference(x, W, ops.T, torch.zeros_like(ops.U), case.act, ops.b_ref)
    assert torch.equal(zero[0], want[0]) and torch.equal(zero[2], want[2])
    uv = lb.U * want[0].abs()
    assert torch.allclose(zero[1] - uv, (want[1] - uv) * (case.K + 64) / case.K, rtol=1e-12, atol=0)


def test_classes_follow_the_table_and_the_scale():
    """An Inf in a T column counts only on the tiles that run its k-block (an excluded k-block multiplies nothing, not zero);
    a negative r swaps the infinities; the bias is added after the scale."""
    N, K, J = 256, 64, 2
    x = torch.ones(2, K, dtype=torch.float64)
    W = torch.ones(N, K, dtype=torch.float64)
    T = torch.zeros(2, 64 * J, dtype=torch.float64)
    T[1, 64] = float("inf")                                   # k-block 1 of token 1
    U = torch.ones(N, 64 * J, dtype=torch.float16)
    tiles = torch.tensor([(0, 1), (0, 2)], dtype=torch.int32)  # tile 0 runs k-block 0 only
    r = torch.ones(N)
    r[200] = -1.0
    b = torch.zeros(N, dtype=torch.float64)
    b[201] = float("-inf")
    _v, _a, cls = lob.lora_reference(x, W, T, U, lb.F16, b, r, tiles)
    row0 = torch.full((N,), lb.FIN, dtype=torch.int8)
    row0[201] = lb.NINF
    assert torch.equal(cls[0], row0) and bool((cls[1, :128] == lb.FIN).all())
    want = torch.full((128,), lb.PINF, dtype=torch.int8)
    want[200 - 128] = lb.NINF
    want[201 - 128] = lb.NAN                                  # +Inf + (-Inf)
    assert torch.equal(cls[1, 128:], want)


# ---------------------------------------------------------------- the layer's kernel operands, restated
def _restated(terms, N, K, dtype):
    """ggufb200_linear_lora_ex's operands for LoRA terms [(scale, up, down, band)], from the header's definition: terms sorted
    by output band (a whole-weight term spans every row), each taking the next r columns; U = fp16(fp32(up) * scale) on the
    band's rows, down on the band's columns; tile i runs the k-blocks from the one holding its lowest column to the one
    holding its highest, (0, 0) without one; no table without bands."""
    def rows(band):
        return (band[1], band[1] + band[2]) if band is not None and band[0] == 0 else (0, N)
    order = sorted(terms, key=lambda t: rows(t[3]))
    R = sum(t[2].shape[0] for t in order)
    J = max(1, -(-R // 64))
    down_pad = torch.zeros(64 * J, K, dtype=dtype)
    u_pad = torch.zeros(N, 64 * J, dtype=torch.float16)
    cols = [set() for _ in range(-(-N // 128))]
    r0 = 0
    for scale, up, down, band in order:
        r = down.shape[0]
        k0, k1 = (band[1], band[1] + band[2]) if band is not None and band[0] == 1 else (0, K)
        n0, n1 = rows(band)
        for j in range(r):
            down_pad[r0 + j, k0:k1] = down[j].to(dtype)
            u_pad[n0:n1, r0 + j] = (up[:, j].float() * scale).half()
            for tile in range(n0 // 128, -(-n1 // 128)):
                cols[tile].add(r0 + j)
        r0 += r
    if all(t[3] is None for t in terms):
        return down_pad, u_pad, None
    pairs = [(min(c) // 64, max(c) // 64 - min(c) // 64 + 1) if c else (0, 0) for c in cols]
    return down_pad, u_pad, torch.tensor(pairs, dtype=torch.int32)


def _terms(spec, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for scale, r, band in spec:
        rows = band[2] if band is not None and band[0] == 0 else N
        cols = band[2] if band is not None and band[0] == 1 else K
        out.append((scale, torch.randn(rows, r, generator=g) * 0.05, torch.randn(r, cols, generator=g) * 0.05, band))
    return out


OPERAND_SPECS = {
    # Flux linear1 slices, listed out of order, with one overlapping band and a tile (rows 1408 .. 1535) no band reaches
    "bands_unsorted_overlapping": (1664, 256, [(0.7, 24, (0, 768, 256)), (0.8, 24, (0, 0, 256)), (0.5, 40, (0, 200, 300)),
                                              (0.6, 24, (0, 256, 512)), (0.9, 16, (0, 1024, 384))]),
    # R crossing 64 within one term, next to an input band and a whole-weight term
    "rank_across_kblocks": (384, 512, [(1.0, 80, (0, 128, 256)), (0.3, 12, (1, 256, 128)), (0.45, 8, None)]),
    # whole-weight terms only: no table
    "no_bands": (264, 256, [(0.25, 40, None), (1.5, 30, None)]),
}


@pytest.mark.parametrize("name", OPERAND_SPECS)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_lora_kernel_operands_match_the_restatement(pkg, name, dtype):
    N, K, spec = OPERAND_SPECS[name]
    terms = _terms(spec, N, K, seed=len(name))
    down_pad, u_pad, tiles = pkg.ops.lora_kernel_operands(terms, N, K, dtype, torch.device("cpu"))
    want = _restated(terms, N, K, dtype)
    assert down_pad.dtype == dtype and u_pad.dtype == torch.float16
    assert torch.equal(down_pad, want[0]) and torch.equal(u_pad, want[1])
    assert (tiles is None) == (want[2] is None)
    if tiles is not None:
        assert tiles.dtype == torch.int32 and torch.equal(tiles, want[2])
        # the table runs every k-block holding a non-zero U entry of the tile's rows: it changes the time, never the bits
        Uh, run = lob.lora_u_model(u_pad, lb.F16, tiles)
        assert torch.equal(Uh, lb.to_f64(u_pad))
        if name == "bands_unsorted_overlapping":
            assert tiles[11].tolist() == [0, 0] and tiles[2].tolist() == [0, 2]      # rows 256 .. 383: columns 24 .. 87


# ---------------------------------------------------------------- the GPU case list reaches what it claims
def test_lora_case_list_covers_its_axes_and_plans(pkg):
    L = pkg.lib.lib()
    cases = lob.LORA_CASES
    assert len({c.id for c in cases}) == len(cases)
    assert {c.M for c in cases} >= set(lb.M_ALL)
    assert {c.N for c in cases} >= set(lb.N_FUSED) | {384, 520}
    assert {c.J for c in cases} == set(lob.J_ALL)
    assert {c.table for c in cases} == set(lob.TABLES) and {c.scale for c in cases} == {"none", "r"}
    assert {(c.act, c.bias) for c in cases} == {(a, b) for a in (lb.F16, lb.BF16) for b in lb.BIAS_KINDS}
    assert {c.producers for c in cases} == set(lb.PRODUCERS)
    assert {c.qt for c in cases if c.spans and not c.straddled} == set(lb.ALL12)
    for t in (Q.Q4_K, Q.Q6_K):
        assert {(c.N, c.K) for c in cases if c.straddled and c.qt == t and c.spans == (t == Q.Q6_K)} == set(lb.STRADDLED)
    assert {c.N * c.K <= 4 << 20 for c in cases} == {True}
    for J in lob.J_ALL:
        # clamping values are drawn for every J: first past J, negative, count past J
        raw = lob.lora_table("clamp", 768, J)
        assert any(f > J for f, _c in raw) and any(f < 0 for f, _c in raw) and any(f + c > J for f, c in raw)
    lora_entry = [c for c in cases if c.J == 1 and c.table == "none" and c.scale == "none"]
    assert lora_entry and any(c.flags == lb.FLAG_NOSPLIT for c in lora_entry)
    tokens, ranges_by_ws = set(), {"auto": [], "two": []}
    for c in cases:
        rows, k_ranges, _kb, _items = lb.plan(L, c, lob.workspace_bytes(L, c))
        tokens.add(rows)
        ranges_by_ws[c.ws].append(k_ranges)
        if c.flags == lb.FLAG_NOSPLIT or c.straddled:
            assert k_ranges == 1, c.id
        if c.ws == "two":
            assert k_ranges <= 2, c.id
    assert tokens == {32, 128, 192, 384}, tokens
    assert max(ranges_by_ws["auto"]) > 2 and 2 in ranges_by_ws["two"]
    split_scaled = [c for c in cases if c.scale == "r" and lb.plan(L, c, lob.workspace_bytes(L, c))[1] > 1]
    split_tables = [c for c in cases if c.table != "none" and lb.plan(L, c, lob.workspace_bytes(L, c))[1] > 1]
    assert split_scaled and split_tables, "the finalize must see the scale, and split K the table"
