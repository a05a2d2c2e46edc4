"""The patched packed Linear, driven as a user drives it (`lin(x)` on a GGMLOps.Linear with a packed weight and a patch list),
every output element against the float64 restatement of calculate_weight and the bound of the route the layer took
(tests/patch_bounds.py).  Spies on the library entry points assert the route; the largest fraction of the bound used is
printed per route.  Then three translation mistakes injected into the layer's own helpers (wrapped, not replaced) must be
flagged by the same check."""
import numpy as np
import pytest
import torch

import linear_bounds as lb
import oracle
import patch_bounds as pb
from fallback_cases import random_blocks as fallback_blocks
from util import Q

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
USED = {}
ENTRIES = ("ggufb200_linear", "ggufb200_linear_spans", "ggufb200_linear_lora", "ggufb200_linear_lora_ex", "ggufb200_linear_lora_scaled",
           "ggufb200_linear_fallback", "ggufb200_dequant_kron", "ggufb200_gemm", "ggufb200_gemm_scaled", "ggufb200_dequant",
           "ggufb200_dequant_fallback")


@pytest.fixture(scope="module", autouse=True)
def report_bound_use():
    yield
    if USED:
        print("\nlargest fraction of the per-element bound used, per route:")
        for k in sorted(USED):
            print(f"  {k:34s} {USED[k]:.3g}")


@pytest.fixture(scope="module")
def hostf():
    L = lb.build_hostf()
    assert L is not None, "nvcc is needed to run the fast producers on the host"
    return L


class LoRAAdapter:
    def __init__(self, weights):
        self.weights = weights


class LoHaAdapter(LoRAAdapter):
    pass


class LoKrAdapter(LoRAAdapter):
    pass


@pytest.fixture
def calls(pkg, monkeypatch):
    """Library entry points called, in order, "calculate_weight" for the two-step route (restated for LoHa / LoKr), and the
    weights handed to linear_dense / returned by cast_bias_weight."""
    L = pkg.lib.lib()
    seen, weights = [], {}
    for name in ENTRIES:
        real = getattr(L, name)

        def wrapped(*args, _real=real, _name=name):
            seen.append(_name)
            return _real(*args)
        monkeypatch.setattr(L, name, wrapped)

    def restated(patches, weight, key, intermediate_dtype=torch.float32, original_weights=None):
        seen.append("calculate_weight")
        return pb.calculate_weight(weight, patches, intermediate_dtype)[0]
    monkeypatch.setattr(pkg.ops.comfy_lora, "calculate_weight", restated)
    real_dense = pkg.ops.linear_dense

    def dense(x, weight, bias=None, feature_scale=None):
        weights.setdefault("dense", weight)
        return real_dense(x, weight, bias, feature_scale)
    monkeypatch.setattr(pkg.ops, "linear_dense", dense)
    return seen, weights


# ---------------------------------------------------------------- layer and patch lists
def _raw(qt, N, K):
    seed = int(qt) * 31 + N + K
    if qt == Q.BF16:
        w = (torch.randn(N, K, generator=torch.Generator().manual_seed(seed)) * 0.02).to(torch.bfloat16)
        return w.view(torch.uint8).reshape(-1)
    if qt in (Q.IQ2_XS, Q.TQ2_0):
        return torch.from_numpy(fallback_blocks(qt, N * K // 256, seed=seed, scale=0.002).reshape(-1))
    bs, _ts = oracle.type_info(int(qt))
    return torch.from_numpy(oracle.random_blocks(int(qt), N * K // bs, seed=seed, scale=0.02).reshape(-1))


def _layer(pkg, case):
    qt = Q[case.qt]
    N, K = case.N, case.K
    raw = _raw(qt, N, K)
    lin = pkg.ops.GGMLOps.Linear(K, N)
    w = pkg.ops.GGMLTensor(raw.to(DEV), tensor_type=qt, tensor_shape=torch.Size((N, K)))
    b = (torch.randn(N, generator=torch.Generator().manual_seed(N + K)) * 0.5).to(DEV)
    lin.load_state_dict({"weight": w, "bias": pkg.ops.GGMLTensor(b, tensor_type=Q.F32, tensor_shape=torch.Size((N,)))})
    for attr, value in case.layer:
        setattr(lin, attr, value)
    return lin, raw


def _lora(g, rows, cols, r, s_up=0.1, s_down=None):
    s_down = 0.2 / np.sqrt(r) if s_down is None else s_down
    return (torch.randn(rows, r, generator=g) * s_up).to(DEV), (torch.randn(r, cols, generator=g) * s_down).to(DEV)


def _lora_entry(g, N, K, r, band=None, strength=0.8, adapter=False, alpha="r", s_up=0.1, s_down=None):
    rows = band[2] if band is not None and band[0] == 0 else N
    cols = band[2] if band is not None and band[0] == 1 else K
    up, down = _lora(g, rows, cols, r, s_up, s_down)
    payload = (up, down, float(r) if alpha == "r" else alpha, None, None, None)
    return (strength, LoRAAdapter(payload) if adapter else ("lora", payload), 1.0, band, None)


def _loha_entry(g, rows, cols, d, band=None, strength=0.9):
    s = (0.02 / d) ** 0.25
    f = [(torch.randn(*sh, generator=g) * s).to(DEV) for sh in ((rows, d), (d, cols), (rows, d), (d, cols))]
    return (strength, LoHaAdapter((f[0], f[1], float(d), f[2], f[3], None, None, None)), 1.0, band, None)


def _lokr_entry(g, a, b, band=None, strength=0.7, rank2=None, alpha=2.0):
    w1 = (torch.randn(*a, generator=g) * 0.3).to(DEV)
    if rank2 is None:
        w2, w2_a, w2_b = (torch.randn(*b, generator=g) * 0.1).to(DEV), None, None
    else:
        w2, w2_a, w2_b = None, (torch.randn(b[0], rank2, generator=g) * 0.1).to(DEV), (torch.randn(rank2, b[1], generator=g) * 0.1).to(DEV)
    return (strength, ("lokr", (w1, w2, alpha, None, None, w2_a, w2_b, None, None)), 1.0, band, None)


def _magnitude(g, W0, axis):
    nrm = W0.float().norm(dim=1 - axis, keepdim=True)
    return nrm * (torch.rand(*nrm.shape, generator=g) * 0.4 + 0.8).to(DEV)


def _offgrid(N, K):
    return [(0, 3, 197), (0, 200, 136), (0, 336, N - 336), (1, 40, K - 104)]


def entries_for(spec, N, K, g, W0):
    if spec == "whole_r16":
        return [_lora_entry(g, N, K, 16)]
    if spec == "whole_two":
        return [_lora_entry(g, N, K, 16), _lora_entry(g, N, K, 24, adapter=True, alpha=None, s_up=0.05)]
    if spec in ("bands_offgrid", "nan_up_band", "inf_down_band"):
        out = [_lora_entry(g, N, K, (16, 24, 8, 12)[i], band, 0.8 - 0.1 * i, adapter=i % 2 == 1) for i, band in enumerate(_offgrid(N, K))]
        if spec == "nan_up_band":
            out[1][1].weights[0][5, 3] = float("nan")          # the band of rows 200 .. 335
        elif spec == "inf_down_band":
            out[2][1][1][1][2, 17] = float("inf")              # the band of rows 336 .. N - 1
        return out
    if spec == "bands_overlap":
        return [_lora_entry(g, N, K, 16, (0, 100, 300)), _lora_entry(g, N, K, 8, (0, 250, 200), -0.6), _lora_entry(g, N, K, 4)]
    if spec == "cols_non64":
        return [_lora_entry(g, N, K, 16, (1, 24, 488)), _lora_entry(g, N, K, 8, (1, 520, 488)), _lora_entry(g, N, K, 8, (0, 8, 120))]
    if spec == "rank_J2":
        return [_lora_entry(g, N, K, 100)]
    if spec == "rank_J5":
        return [_lora_entry(g, N, K, r, (0, 128 * i, 128)) for i, r in enumerate((100, 113, 100))]
    if spec == "rank_J8":
        return [_lora_entry(g, N, K, 125, strength=0.5, adapter=i % 2 == 0) for i in range(4)]
    if spec == "rank_513":
        return [_lora_entry(g, N, K, 256), _lora_entry(g, N, K, 257)]
    if spec == "strength_zero_neg":
        return [_lora_entry(g, N, K, 16, strength=0.0), _lora_entry(g, N, K, 16, (0, 64, 200), strength=-0.7)]
    if spec == "u_subnormal":
        return [_lora_entry(g, N, K, 16, strength=1.0, s_up=2e-6, s_down=100.0)]
    if spec == "u_above_f16":
        e = _lora_entry(g, N, K, 16, strength=1.0, s_up=3e4, s_down=2e-6)
        e[1][1][0][0, 0] = 1e5
        return [e]
    if spec == "inf_up_whole":
        e = _lora_entry(g, N, K, 16)
        e[1][1][0][7, 2] = float("inf")
        return [e]
    if spec == "slices_flux":
        H = N // 7
        return [_lora_entry(g, N, K, 16, (0, s, z), 0.8 - 0.1 * i, adapter=i % 2 == 1)
                for i, (s, z) in enumerate([(0, H), (H, H), (2 * H, H), (3 * H, 4 * H)])]
    if spec.startswith("loha_"):
        return [_loha_entry(g, N, K, int(spec[5:]))]
    if spec == "lokr_whole":
        return [_lokr_entry(g, (16, 16), (N // 16, K // 16), rank2=4)]
    if spec in ("lokr_bands", "nan_lokr"):
        out = [_lokr_entry(g, (8, 16), (32, K // 16), (0, 8, 256)), _lokr_entry(g, (8, 16), (32, K // 16), (0, 264, 256), 1.1, rank2=8)]
        if spec == "nan_lokr":
            out[0][1][1][0][1, 1] = float("nan")
        return out
    if spec == "lokr_mixed":
        H = N // 3
        return [_lora_entry(g, N, K, 16, strength=0.6), _loha_entry(g, H, K, 8, (0, H, H)),
                _lokr_entry(g, (16, 16), (N // 16, K // 16), strength=1.2, rank2=16)]
    if spec == "lokr_nine":
        return [_lokr_entry(g, (8, 8), (N // 8, K // 8), strength=0.2 + 0.1 * i) for i in range(9)]
    if spec == "mixed_whole":
        return [_lora_entry(g, N, K, 16), _loha_entry(g, N, K, 4), _lokr_entry(g, (16, 16), (N // 16, K // 16), rank2=4)]
    if spec == "strength_model":
        e = _lora_entry(g, N, K, 16)
        return [(e[0], e[1], 0.9, None, None)]
    up, down = _lora(g, N, K, 16, 0.05, 0.05)
    up2, down2 = _lora(g, N, K, 8, 0.05, 0.05)
    w = _loha_entry(g, N, K, 2)[1].weights
    if spec == "dora_out":
        return [(0.8, ("lora", (up, down, 8.0, None, _magnitude(g, W0, 0), None)), 1.0, None, None),
                (0.9, LoRAAdapter((up2, down2, None, None, None, None)), 1.0, None, None)]
    if spec == "dora_in":
        return [(1.3, ("lora", (up, down, 8.0, None, _magnitude(g, W0, 1), None)), 1.0, None, None)]
    if spec == "dora_both":
        return [(0.8, ("lora", (up, down, 8.0, None, _magnitude(g, W0, 0), None)), 1.0, None, None),
                (0.9, LoRAAdapter((up2, down2, None, None, None, None)), 1.0, None, None),
                (1.2, LoHaAdapter(tuple(w[:7]) + (_magnitude(g, W0, 1),)), 1.0, None, None)]
    if spec == "dora_both_r0":
        m = _magnitude(g, W0, 0)
        m[5] = 0.0                                     # s_5 = 0 at strength 1: r_5 = 0, the in-kernel U = up / r is not finite
        return [(1.0, ("lora", (up, down, 8.0, None, m, None)), 1.0, None, None),
                (1.2, LoHaAdapter(tuple(w[:7]) + (_magnitude(g, W0, 1),)), 1.0, None, None)]
    raise KeyError(spec)


def scaled(entries, spec, W0):
    """The entries with their first factor (LoRA up, LoHa w1a, LoKr w1) scaled in place so that each delta is of the order of
    the weight itself (the factors above are drawn for a weight of rms 0.02): a dropped or misplaced row then moves outputs by
    many times their bound in bf16 too.  The U-range cases keep their magnitudes."""
    if spec in ("u_subnormal", "u_above_f16"):
        return entries
    amp = float(W0.float().pow(2).mean().sqrt()) / 0.02
    for entry in entries:
        pb.parse(entry)[2][0].mul_(amp)
    return entries


# ---------------------------------------------------------------- the route the layer must take
def family(case, dtype, numerics):
    if case.route == "side_bf16_weight" and dtype == torch.float16:
        return "two_step"                             # a BF16 weight under fp16 activations above M = 8: the reference's route
    if case.spec == "u_above_f16":
        return "two_step" if dtype == torch.float16 else "side"
    if case.route in ("lokr_two_step", "two_step", "nonfinite"):
        return "two_step"
    if case.route.startswith("lokr"):
        return "kron"
    if case.route == "dora_kernel":
        return "dora_kernel"
    if case.route == "dora_side":
        return "dora_side"
    if case.route.startswith("kernel") or case.route == "loha_kernel":
        return "kernel"
    return "side"


def _assert_route(fam, seen, case):
    lora = {"ggufb200_linear_lora", "ggufb200_linear_lora_ex", "ggufb200_linear_lora_scaled"}
    if fam == "kernel":
        assert lora & set(seen) and "calculate_weight" not in seen, seen
    elif fam == "dora_kernel":
        assert "ggufb200_linear_lora_scaled" in seen and "calculate_weight" not in seen, seen
    elif fam == "dora_side":
        assert "ggufb200_gemm_scaled" in seen and not lora & set(seen) and "calculate_weight" not in seen, seen
    elif fam == "kron":
        assert seen[:2] == ["ggufb200_dequant_kron", "ggufb200_gemm"] and "calculate_weight" not in seen, seen
    elif fam == "two_step":
        assert "calculate_weight" in seen and "ggufb200_dequant_kron" not in seen and not lora & set(seen), seen
    else:
        assert not lora & set(seen) and "calculate_weight" not in seen and "ggufb200_dequant_kron" not in seen, seen
        if case.route == "side_fallback_sync":
            assert "ggufb200_linear_fallback" in seen or "ggufb200_dequant_fallback" in seen, seen
        if case.route == "side_fallback_k1":
            assert "ggufb200_dequant_fallback" in seen, seen


# ---------------------------------------------------------------- the check
def _weight_error(hostf, raw, qt, N, K, dtype, numerics, M, fam, W0):
    """(ew0, mag): what the fast contract lets the weight operand differ by, and GEMV_FAST's magnitudes."""
    if numerics != "fast" or qt not in (Q.Q4_K, Q.Q5_K) or fam not in ("kernel", "side", "dora_kernel"):
        return None, None
    act = pb.ACT_CODE[dtype]
    rawn = raw.numpy()
    ew0 = (lb.fast_weight(hostf, rawn, qt, N, K, act).to(DEV) - W0).abs()
    mag = None
    if M <= 8 and fam == "side":
        Wg, mag = lb.gemv_fast_model(rawn, qt, N, K, act)
        ew0 = torch.maximum(ew0, (Wg.to(DEV) - W0).abs())
        mag = mag.to(DEV)
    return ew0, mag


def run_case(pkg, hostf, case, dtype, numerics, calls, mutate=None):
    """Forward, route check and the per-element verdict of one case."""
    seen, weights = calls
    lin, raw = _layer(pkg, case)
    lin.linear_numerics = numerics
    N, K = case.N, case.K
    qt = Q[case.qt]
    W0a = pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, dtype, lin.dequant_dtype)).to(dtype)
    g = torch.Generator().manual_seed(N * 7 + K + len(case.spec) + case.M)
    entries = scaled(entries_for(case.spec, N, K, g, W0a), case.spec, W0a)
    lin.weight.patches = [(entries, "diffusion_model.w")]
    shape = (3, case.M // 3, K) if case.x3d else (case.M, K)
    x = torch.randn(*shape, generator=g).to(DEV).to(dtype)
    grad = case.route == "autograd"
    if grad:
        x.requires_grad_(True)
    fam = family(case, dtype, numerics)
    seen.clear()
    weights.clear()
    if mutate is not None:
        mutate()
    with torch.no_grad() if not grad else torch.enable_grad():
        y = lin(x)
    y = y.detach().reshape(-1, N)
    x2 = lb.to_f64(x.detach().reshape(-1, K))
    _assert_route(fam, seen, case)
    act = pb.ACT_CODE[dtype]
    b = lb.to_f64(pkg.ops._plain(lin.bias).to(dtype))
    W0 = lb.to_f64(W0a)
    inter = dtype if lin.patch_dtype == "target" else torch.float32
    W_ref, W_star, factors = pb.reference_weights(W0a, entries, inter)
    ew0, mag = _weight_error(hostf, raw, qt, N, K, dtype, numerics, x2.shape[0], fam, W0)
    cls = pb.reference_classes(x2, W_ref, b)
    if fam == "two_step":
        assert torch.equal(pkg.ops._plain(lin.cast_bias_weight(x.detach())[0]), W_ref) or bool((cls != lb.FIN).any()), "two-step weight"
        v, a, _c = lb.reference(x2, lb.to_f64(W_ref), b)
        if bool(torch.isfinite(W_ref).all()):
            wb = pb.weight_bound(W0a, entries, W_star, inter)
            assert bool(((lb.to_f64(W_ref) - W_star).abs() <= wb).all()), "the reference weight is outside its bound around W*"
    elif fam == "kron":
        kron = [e for e in entries if pb.parse(e)[1] == "lokr"]
        W_k = pb.calculate_weight(W0a.clone(), kron)[0]
        assert torch.equal(weights["dense"], W_k), "dequant_kron's weight is not the reference's"
        v, a = pb.side_bound(x2, lb.to_f64(W_k), pb.lora_terms(entries, DEV), dtype, b) if len(kron) < len(entries) else \
            lb.reference(x2, lb.to_f64(W_k), b)[:2]
        wb = pb.weight_bound(W0a, entries, W_star)
        assert bool(((lb.to_f64(W_ref) - W_star).abs() <= wb).all()), "the reference weight is outside its bound around W*"
    elif fam in ("kernel", "side"):
        terms = pb.lora_terms(entries, DEV)
        if fam == "kernel":
            v, a = pb.kernel_bound(x2, W0, terms, dtype, b, ew0)
        else:
            v, a = pb.side_bound(x2, W0, terms, dtype, b, ew0, mag, sidesum=grad)
    else:
        pieces = pb.dora_pieces(entries, factors, N, K, DEV)
        v, a = (pb.dora_kernel_bound(x2, W0, pieces, dtype, b, ew0) if fam == "dora_kernel" else pb.dora_side_bound(x2, W0, pieces, dtype, b))
    if fam in ("kernel", "side", "dora_kernel", "dora_side"):
        # the route's factorisation is the restated W*: the same exact value up to float64 rounding
        v_star = x2 @ W_star.T + b[None, :]
        assert float((v - v_star).abs().max()) <= 1e-9 * (float((x2.abs() @ W_star.abs().T).max()) + 1.0), "factorisation is not W*"
    verdict = lb.check(y, v, a, cls, act, f"{case.id} {dtype} {numerics}")
    lin.weight.patches = []
    return fam, verdict


@pytest.mark.parametrize("numerics", ["exact", "fast"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", pb.CASES, ids=lambda c: c.id)
def test_every_element_within_the_bound(pkg, hostf, calls, case, dtype, numerics):
    fam, verdict = run_case(pkg, hostf, case, dtype, numerics, calls)
    key = f"{case.route}-{'f16' if dtype == torch.float16 else 'bf16'}"
    USED[key] = max(USED.get(key, 0.0), verdict.used)
    assert verdict.ok, verdict.message


# ---------------------------------------------------------------- injected translation mistakes
def _shift_band(pkg, monkeypatch):
    real = pkg.ops.lora_kernel_operands

    def wrong(terms, N, K, dtype, device):
        moved = [(s, u, d, (0, band[1] + 8, band[2]) if band is not None and band[0] == 0 and band[1] + band[2] + 8 <= N else band)
                 for s, u, d, band in terms]
        return real(moved, N, K, dtype, device)
    monkeypatch.setattr(pkg.ops, "lora_kernel_operands", wrong)


def _drop_tile(pkg, monkeypatch):
    real = pkg.ops.lora_kernel_operands

    def wrong(terms, N, K, dtype, device):
        down_pad, u_pad, tiles = real(terms, N, K, dtype, device)
        tiles = tiles.clone()
        tiles[1] = 0
        return down_pad, u_pad, tiles
    monkeypatch.setattr(pkg.ops, "lora_kernel_operands", wrong)


def _swap_lokr_bands(pkg, monkeypatch):
    real = pkg.ops.lycoris_operands

    def wrong(terms, device):
        bands = [band for kind, _s, _f, band in terms if kind == "lokr"]
        it = iter(bands[::-1])
        return real([(k, s, f, next(it) if k == "lokr" else band) for k, s, f, band in terms], device)
    monkeypatch.setattr(pkg.ops, "lycoris_operands", wrong)


@pytest.mark.parametrize("mutation,case", [
    (_shift_band, pb.PatchCase("kernel", "bands_offgrid", N=520, M=64)),
    (_drop_tile, pb.PatchCase("kernel", "bands_offgrid", N=520, M=64)),
    (_swap_lokr_bands, pb.PatchCase("lokr_banded", "lokr_bands", N=520, M=64)),
], ids=["band_shift_8", "tile_dropped", "lokr_bands_swapped"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_injected_translation_mistakes_are_flagged(pkg, hostf, calls, monkeypatch, mutation, case, dtype):
    lokr = case.route == "lokr_banded"
    if lokr:
        seen, weights = calls
        # the bit-for-bit weight check would catch it first; the output bound must too: check it alone
        mutation(pkg, monkeypatch)
        lin, _raw_ = _layer(pkg, case)
        W0a = pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, dtype)).to(dtype)
        g = torch.Generator().manual_seed(case.N * 7 + case.K + len(case.spec) + case.M)
        entries = scaled(entries_for(case.spec, case.N, case.K, g, W0a), case.spec, W0a)
        lin.weight.patches = [(entries, "diffusion_model.w")]
        x = torch.randn(case.M, case.K, generator=g).to(DEV).to(dtype)
        y = lin(x)
        assert "ggufb200_dequant_kron" in seen
        W_ref = pb.reference_weights(W0a, entries)[0]
        v, a, cls = lb.reference(lb.to_f64(x), lb.to_f64(W_ref), lb.to_f64(pkg.ops._plain(lin.bias).to(dtype)))
        verdict = lb.check(y, v, a, cls, pb.ACT_CODE[dtype])
    else:
        _fam, verdict = run_case(pkg, hostf, case, dtype, "exact", calls, mutate=lambda: mutation(pkg, monkeypatch))
    USED[f"mutation-{mutation.__name__}-{'f16' if dtype == torch.float16 else 'bf16'}"] = verdict.used
    assert not verdict.ok and verdict.used > 2, verdict.message
