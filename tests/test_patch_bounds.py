"""CPU checks of tests/patch_bounds.py: the restatement of calculate_weight agrees with the restatements the other test files
carry, the case list names every route of the patched Linear, and each route's bound rejects the translation mistakes it
exists to catch, on float64-simulated outputs (the rejection margin, the largest fraction of the bound used, is printed)."""
import pytest
import torch

import linear_bounds as lb
import patch_bounds as pb
import test_gpu_dora as gd
import test_gpu_lycoris as gl

MARGINS = {}


@pytest.fixture(scope="module", autouse=True)
def report_margins():
    yield
    if MARGINS:
        print("\nrejection margins (largest fraction of the bound used by the mutated output):")
        for k in sorted(MARGINS):
            print(f"  {k:40s} {MARGINS[k]:.3g}")


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


class LoKrAdapter(LoRAAdapter):
    pass


def _r(g, *shape, s=0.1):
    return torch.randn(*shape, generator=g) * s


def _entries(g, N, K):
    """LoRA (alpha None and given), LoHa, LoKr whole / decomposed, on the whole weight, row bands and input bands."""
    return [
        (0.8, ("lora", (_r(g, N, 8), _r(g, 8, K), 4.0, None, None, None)), 1.0, None, None),
        (-0.6, LoRAAdapter((_r(g, 64, 4), _r(g, 4, K), None, None, None, None)), 1.0, (0, 40, 64), None),
        (1.1, ("lora", (_r(g, N, 4), _r(g, 4, 72), 2.0, None, None, None)), 1.0, (1, 24, 72), None),
        (0.9, LoHaAdapter((_r(g, N, 3), _r(g, 3, K), 6.0, _r(g, N, 3), _r(g, 3, K), None, None, None)), 1.0, None, None),
        (0.7, ("lokr", (_r(g, 8, 4, s=0.3), None, 3.0, None, None, _r(g, N // 8, 2), _r(g, 2, K // 4), None, None)), 1.0, None, None),
        (1.3, LoKrAdapter((_r(g, 4, 4, s=0.3), _r(g, 16, K // 4), 5.0, None, None, None, None, None, None)), 1.0, (0, 16, 64), None),
    ]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=["f16", "bf16", "f32"])
def test_restatement_equals_the_other_restatements(dtype):
    g = torch.Generator().manual_seed(3)
    N, K = 128, 256
    W0 = _r(g, N, K, s=0.05).to(dtype)
    entries = _entries(g, N, K)
    W_ref, W_star, factors = pb.reference_weights(W0, entries)
    assert factors == [None] * len(entries)
    assert torch.equal(W_ref, gl._restated_weight(W0.clone(), entries, dtype))
    assert torch.allclose(W_star, gl._ideal_weight(W0, entries), rtol=0, atol=1e-12)
    # the fake comfy.lora (LoRA only) and, with DoRA entries, test_gpu_dora's restated weight_decompose
    import comfy.lora
    lora_only = [e for e in entries if pb.parse(e)[1] == "lora" and e[3] is None]
    assert torch.equal(pb.calculate_weight(W0.clone(), lora_only)[0], comfy.lora.calculate_weight(lora_only, W0.clone(), "k"))
    up, down = _r(g, N, 8), _r(g, 8, K)
    dora = [(0.8, ("lora", (up, down, 4.0, None, W0.float().norm(dim=1, keepdim=True) * 1.1, None)), 1.0, None, None),
            (1.3, LoHaAdapter((_r(g, N, 2), _r(g, 2, K), 1.0, _r(g, N, 2), _r(g, 2, K), None, None,
                               W0.float().norm(dim=0, keepdim=True) * 0.9)), 1.0, None, None),
            (1.0, ("lora", (up, down, None, None, W0.float().norm(dim=1, keepdim=True), None)), 1.0, None, None)]
    W_ref, W_star, factors = pb.reference_weights(W0, dora)
    assert torch.equal(W_ref, gd.restated_calculate_weight(dora, W0.clone(), "k"))
    assert [s is None for s in factors] == [False, False, False] and factors[1].shape == (K,)
    # W*: with the s of the replay, the float64 weight is within a few activation ulps of the reference's
    assert float((W_star - W_ref.double()).abs().max()) <= 64 * pb.U_ACT[dtype] * float(W_star.abs().max())


def test_strength_model_scales_the_band_before_the_patch():
    g = torch.Generator().manual_seed(4)
    W0 = _r(g, 64, 32).double()
    up, down = _r(g, 16, 2).double(), _r(g, 2, 32).double()
    e = [(0.5, ("lora", (up, down, None, None, None, None)), 0.9, (0, 8, 16), None)]
    want = W0.clone()
    want[8:24] = 0.9 * want[8:24] + 0.5 * up @ down
    assert torch.allclose(pb.calculate_weight(W0.clone(), e)[0], want, rtol=0, atol=1e-7)       # the delta is fp32


def test_the_case_list_names_every_route():
    assert {c.route for c in pb.CASES} == set(pb.ROUTES)
    specs = {c.spec for c in pb.CASES}
    for need in ("bands_offgrid", "bands_overlap", "cols_non64", "rank_J2", "rank_J5", "rank_J8", "strength_zero_neg", "u_subnormal",
                 "u_above_f16", "loha_4", "loha_16", "loha_32", "dora_out", "dora_in", "dora_both", "dora_both_r0", "lokr_nine"):
        assert need in specs, need
    assert {1, 8, 9, 300} <= {c.M for c in pb.CASES} and any(c.x3d for c in pb.CASES) and any(c.N == 520 for c in pb.CASES)
    assert {dict(c.layer).get("lora_in_kernel") for c in pb.CASES} >= {False}
    assert any(dict(c.layer).get("patch_dtype") == "target" for c in pb.CASES)
    assert any(dict(c.layer).get("lora_side_gemm") is False for c in pb.CASES)


# ---------------------------------------------------------------- mutations the bounds reject
N, K, M = 520, 512, 48
BANDS = [(0, 3, 197), (0, 200, 136), (0, 336, N - 336), (1, 40, K - 104)]


def _setup(dtype, seed=5):
    g = torch.Generator().manual_seed(seed)
    x = lb.to_f64(torch.randn(M, K, generator=g).to(dtype))
    W0 = lb.to_f64((torch.randn(N, K, generator=g) * 0.02).to(dtype))
    b = lb.to_f64((torch.randn(N, generator=g) * 0.5).to(dtype))
    return g, x, W0, b


def _terms(g, strengths=(0.8, 0.7, 0.6, 0.5), ranks=(16, 24, 8, 12)):
    out = []
    for st, r, band in zip(strengths, ranks, BANDS):
        rows = band[2] if band[0] == 0 else N
        cols = band[2] if band[0] == 1 else K
        up = (torch.randn(rows, r, generator=g) * 0.1).double()
        down = (torch.randn(r, cols, generator=g) * (0.2 / r ** 0.5)).double()
        out.append(pb.Term(st, up, down, band))      # alpha = r: scale = strength
    return out


def _simulate_kernel(x, W0, terms, dtype, b):
    """The in-kernel route's roundings in float64: T = act(x act(down)^T), U = act(fp16(fp32(scale up))), one output rounding."""
    y = x @ W0.T + b
    for t in terms:
        rows = slice(t.band[1], t.band[1] + t.band[2]) if t.band and t.band[0] == 0 else slice(0, N)
        cols = slice(t.band[1], t.band[1] + t.band[2]) if t.band and t.band[0] == 1 else slice(0, K)
        T = lb.to_f64((x[:, cols] @ lb.to_f64(t.down.to(dtype)).T).to(dtype))
        U = lb.to_f64((t.up.float() * t.scale).half().to(dtype))
        y[:, rows] += T @ U.T
    return lb.round_act(y, pb.ACT_CODE[dtype])


def _verdict(y, v, a, dtype):
    return lb.check(y, v, a, torch.zeros(v.shape, dtype=torch.int8), pb.ACT_CODE[dtype])


def _rejects(name, y, v, a, dtype):
    verdict = _verdict(y, v, a, dtype)
    MARGINS[f"{name}-{'f16' if dtype == torch.float16 else 'bf16'}"] = verdict.used
    assert not verdict.ok and verdict.used > 2, (name, verdict.message)


def _moved(terms, shift):
    return [pb.Term(t.scale, t.up, t.down, (0, t.band[1] + shift, t.band[2]) if t.band[0] == 0 and t.band[1] + t.band[2] + shift <= N
                    else t.band) for t in terms]


DTYPES = pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])


@DTYPES
@pytest.mark.parametrize("route", ["kernel", "side"])
def test_lora_bounds_reject_translation_mistakes(dtype, route):
    g, x, W0, b = _setup(dtype)
    terms = _terms(g)
    bound = pb.kernel_bound if route == "kernel" else pb.side_bound
    v, a = bound(x, W0, terms, dtype, b)
    act = pb.ACT_CODE[dtype]
    clean = _verdict(_simulate_kernel(x, W0, terms, dtype, b), v, a, dtype)
    assert clean.ok and clean.used < 1, clean.message
    assert _verdict(lb.round_act(v, act), v, a, dtype).ok

    def y_of(ts):
        return lb.round_act(bound(x, W0, ts, dtype, b)[0], act)
    _rejects(f"{route}-band_shift_1", y_of(_moved(terms, 1)), v, a, dtype)
    _rejects(f"{route}-band_shift_8", y_of(_moved(terms, 8)), v, a, dtype)
    # one tile's table entry dropped: rows 128 .. 255 run no k-block
    dropped = []
    for t in terms:
        up = t.up.clone()
        if t.band[0] == 0:
            lo, hi = max(128 - t.band[1], 0), min(256 - t.band[1], t.band[2])
            if lo < hi:
                up[lo:hi] = 0
        else:
            up[128:256] = 0
        dropped.append(pb.Term(t.scale, up, t.down, t.band))
    _rejects(f"{route}-tile_dropped", y_of(dropped), v, a, dtype)
    _rejects(f"{route}-alpha_without_rank", y_of([pb.Term(t.scale * t.down.shape[0], t.up, t.down, t.band) for t in terms[:1]] + terms[1:]),
             v, a, dtype)
    _rejects(f"{route}-strength_twice", y_of([pb.Term(t.scale * t.scale, t.up, t.down, t.band) for t in terms]), v, a, dtype)


@DTYPES
def test_loha_bound_rejects_a_permuted_down(dtype):
    g, x, W0, b = _setup(dtype, seed=6)
    d1, d2 = 4, 3
    s = (0.02 / 4) ** 0.25
    w1a, w1b, w2a, w2b = (torch.randn(*sh, generator=g) * s for sh in ((N, d1), (d1, K), (N, d2), (d2, K)))
    up, down = pb.khatri_rao(w1a, w1b, w2a, w2b)
    assert torch.allclose(up @ down, (w1a.double() @ w1b.double()) * (w2a.double() @ w2b.double()), rtol=0, atol=1e-12)
    terms = [pb.Term(0.9, up, down)]
    v, a = pb.kernel_bound(x, W0, terms, dtype, b)
    assert _verdict(_simulate_kernel(x, W0, terms, dtype, b), v, a, dtype).ok
    perm = torch.einsum("ik,jk->jik", w1b.double(), w2b.double()).reshape(-1, K)     # (j, i) order against up's (i, j)
    _rejects("loha-down_permuted", lb.round_act(pb.kernel_bound(x, W0, [pb.Term(0.9, up, perm)], dtype, b)[0], pb.ACT_CODE[dtype]),
             v, a, dtype)


@DTYPES
def test_lokr_bounds_reject_swapped_bands(dtype):
    g, x, _W0, b = _setup(dtype, seed=7)
    W0 = (torch.randn(N, K, generator=g) * 0.02).to(dtype)
    e1 = (0.7, ("lokr", (_r(g, 8, 16, s=0.3), None, 2.0, None, None, _r(g, 32, 4), _r(g, 4, K // 16), None, None)), 1.0, (0, 8, 256), None)
    e2 = (1.1, ("lokr", (_r(g, 8, 16, s=0.3), _r(g, 32, K // 16), None, None, None, None, None, None, None)), 1.0, (0, 264, 256), None)
    W_ref, W_star, _s = pb.reference_weights(W0, [e1, e2])
    wb = pb.weight_bound(W0, [e1, e2], W_star)
    assert bool(((lb.to_f64(W_ref) - W_star).abs() <= wb).all())
    assert float(wb.max()) <= 8 * pb.U_ACT[dtype] * float(W_star.abs().max())       # a few roundings, not a blanket
    v, a, cls = lb.reference(x, lb.to_f64(W_ref), b)
    assert lb.check(lb.round_act(v, pb.ACT_CODE[dtype]), v, a, cls, pb.ACT_CODE[dtype]).ok
    swapped = [e1[:3] + (e2[3], None), e2[:3] + (e1[3], None)]
    W_mut = pb.calculate_weight(W0.clone(), swapped)[0]
    _rejects("lokr-bands_swapped", lb.round_act(x @ lb.to_f64(W_mut).T + b, pb.ACT_CODE[dtype]), v, a, dtype)


def _dora(g, W0, st_out=0.8, st_in=1.3):
    n = W0.shape[0]
    up, down = _r(g, n, 8, s=0.05), _r(g, 8, W0.shape[1], s=0.05)
    up2, down2 = _r(g, n, 4, s=0.05), _r(g, 4, W0.shape[1], s=0.05)
    return [(st_out, ("lora", (up, down, 8.0, None, W0.float().norm(dim=1, keepdim=True) * 1.15, None)), 1.0, None, None),
            (st_in, ("lora", (up2, down2, 4.0, None, W0.float().norm(dim=0, keepdim=True) * 0.85, None)), 1.0, None, None)]


@DTYPES
@pytest.mark.parametrize("route", ["kernel", "side"])
def test_dora_bounds_reject_translation_mistakes(dtype, route):
    g = torch.Generator().manual_seed(8)
    n = 256                                                      # square: r and c can be exchanged
    x = lb.to_f64(torch.randn(M, n, generator=g).to(dtype))
    W0 = (torch.randn(n, n, generator=g) * 0.02).to(dtype)
    b = lb.to_f64((torch.randn(n, generator=g) * 0.5).to(dtype))
    entries = _dora(g, W0)
    W_ref, W_star, factors = pb.reference_weights(W0, entries)
    pieces = pb.dora_pieces(entries, factors, n, n, "cpu")
    W_c = pieces.r[:, None] * lb.to_f64(W0) * pieces.c[None, :] + sum(
        (coef * rho[:, None] * up) @ (down * gam[None, :]) for coef, rho, gam, up, down in pieces.terms)
    assert torch.allclose(W_c, W_star, rtol=0, atol=1e-12)
    bound = pb.dora_kernel_bound if route == "kernel" else pb.dora_side_bound
    v, a = bound(x, lb.to_f64(W0), pieces, dtype, b)
    act = pb.ACT_CODE[dtype]
    assert _verdict(lb.round_act(x @ W_star.T + b, act), v, a, dtype).ok
    swapped = pb.DoraPieces(pieces.c, pieces.r, True, pieces.terms)
    _rejects(f"dora-{route}-r_c_exchanged", lb.round_act(bound(x, lb.to_f64(W0), swapped, dtype, b)[0], act), v, a, dtype)
    # the output-axis s from the norms of the patched weight instead of the weight before the patch
    W = lb.to_f64(W0)
    st, _k, p, _sm, _o = pb.parse(entries[0])
    Wc = W + 1.0 * (p[0].double() @ p[1].double())
    s_after = (p[4].double().reshape(-1) / (Wc.norm(dim=1) + torch.finfo(dtype).eps))
    wrong = [s_after.to(dtype)] + factors[1:]
    W_mut = pb.ideal_weight(W0, entries, wrong)
    _rejects(f"dora-{route}-s_after_patch", lb.round_act(x @ W_mut.T + b, act), v, a, dtype)
