"""GPU tests of LoRA on bands of a packed weight and of LoRA stacks above rank 64 inside the FUSED_TMEM kernel
(ggufb200_linear_lora_ex: J <= 8 LoRA k-blocks, optional per-tile k-block ranges).

Shapes follow Flux: diffusers-format LoRAs patch `qkv` [3 H, K] as three row bands and a single block's `linear1` [3 H + 4 H, K]
as four, which ComfyUI hands over as patch entries with `offset = (0, start, size)`.  Reference = what ComfyUI computes for such
an entry: `W[band] += (strength * alpha / r * up @ down).to(dtype)` on the dequantised weight, then F.linear (here in float64).
Budget (the one of tests/test_gpu_linear.py::test_lora_on_packed_weight_runs_as_side_gemms): within 3e-3 (fp16) / 1e-2 (bf16)
relative Frobenius of the reference, and under the `exact` contract no further from the unrounded ideal than 1.5x the
reference's own rounded output is, + 1e-4."""
import pytest
import torch

import oracle
from util import Q

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K = 1024


class LoRAAdapter:                      # the object newer ComfyUI puts in a patch entry
    def __init__(self, weights):
        self.weights = weights


def _layer(pkg, N, seed=0):
    raw = oracle.random_blocks(int(Q.Q4_K), N * K // 256, seed=seed, scale=0.02).reshape(N, K // 256 * 144)
    lin = pkg.ops.GGMLOps.Linear(K, N)
    w = pkg.ops.GGMLTensor(torch.from_numpy(raw).to(DEV), tensor_type=Q.Q4_K, tensor_shape=torch.Size((N, K)))
    g = torch.Generator().manual_seed(seed + 1)
    b = pkg.ops.GGMLTensor((torch.randn(N, generator=g) * 0.02).to(DEV), tensor_type=Q.F32, tensor_shape=torch.Size((N,)))
    lin.load_state_dict({"weight": w, "bias": b})
    return lin


def _bands(kind, H):
    return [(0, H), (H, H), (2 * H, H)] + ([(3 * H, 4 * H)] if kind == "linear1" else [])


def _patches(kind, H, rank=None, total=None, seed=0):
    """(strength, up, down, alpha, offset) per entry: one diffusers-format LoRA of `rank` per slice, or a stack of Σr = total
    (one sliced LoRA of rank total / 8 per slice plus whole-weight LoRAs of rank <= 64 for the rest)."""
    g = torch.Generator().manual_seed(seed)
    N = sum(size for _s, size in _bands(kind, H))

    def factors(rows, r, cols=K):
        return (torch.randn(rows, r, generator=g) * 0.05).to(DEV), (torch.randn(r, cols, generator=g) * 0.05).to(DEV)
    out = []
    r_slice = rank if rank is not None else total // 8
    for i, (start, size) in enumerate(_bands(kind, H)):
        up, down = factors(size, r_slice)
        out.append((0.8 - 0.1 * i, up, down, float(r_slice) / 2, (0, start, size)))
    rest = 0 if total is None else total - r_slice * len(_bands(kind, H))
    while rest > 0:
        r = min(rest, 64)
        up, down = factors(N, r)
        out.append((0.6, up, down, 4.0, None))
        rest -= r
    return out


def _apply(lin, patches):
    entries = []
    for i, (s, up, down, alpha, offset) in enumerate(patches):
        value = (up, down, alpha, None, None, None)
        entries.append((s, LoRAAdapter(value) if i % 2 else ("lora", value), 1.0, offset, None))
    lin.weight.patches = [(entries, "diffusion_model.w")]


def _references(pkg, lin, x, patches):
    dtype = x.dtype
    W = pkg.ops._plain(pkg.dequant.dequantize_tensor(lin.weight, dtype))
    Wref, Wideal = W.clone(), W.double()
    for s, up, down, alpha, offset in patches:
        d = (s * alpha / down.shape[0]) * (up.float() @ down.float())
        if offset is None:
            Wref += d.to(dtype)
            Wideal += d.double()
        elif offset[0] == 0:
            Wref[offset[1]:offset[1] + offset[2]] += d.to(dtype)
            Wideal[offset[1]:offset[1] + offset[2]] += d.double()
        else:
            Wref[:, offset[1]:offset[1] + offset[2]] += d.to(dtype)
            Wideal[:, offset[1]:offset[1] + offset[2]] += d.double()
    bias = pkg.ops._plain(lin.bias).to(dtype).double()
    return (torch.nn.functional.linear(x.double(), Wref.double(), bias), torch.nn.functional.linear(x.double(), Wideal, bias))


def _rel(a, b):
    return float((a.double() - b).norm() / b.norm())


def _check(y, ref, ideal, dtype, numerics, what):
    assert y.dtype == dtype
    err = _rel(y, ref)
    assert err <= (3e-3 if dtype == torch.float16 else 1e-2), (what, err)
    if numerics == "exact":
        assert _rel(y, ideal) <= 1.5 * _rel(ref.to(dtype), ideal) + 1e-4, (what, _rel(y, ideal), _rel(ref.to(dtype), ideal))


@pytest.fixture
def ex_calls(pkg, monkeypatch):
    """Counts the calls of ggufb200_linear_lora_ex made through the package."""
    L = pkg.lib.lib()
    real = L.ggufb200_linear_lora_ex
    calls = []

    def counting(*args):
        calls.append(args)
        return real(*args)
    monkeypatch.setattr(L, "ggufb200_linear_lora_ex", counting)
    return calls


@pytest.fixture(params=["exact", "fast"])
def numerics(request, pkg):
    cls = pkg.ops.GGMLOps.Linear
    before = cls.linear_numerics
    cls.linear_numerics = request.param
    yield request.param
    cls.linear_numerics = before


CASES = [dict(rank=16), dict(rank=48), dict(rank=80), dict(total=128), dict(total=256), dict(total=512)]


@pytest.mark.parametrize("M", [3, 300, 1000])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("kind,H", [("qkv", 256), ("qkv", 384), ("linear1", 256), ("linear1", 384)])
def test_sliced_lora_runs_in_the_fused_kernel(pkg, kind, H, dtype, M, numerics, ex_calls):
    lin = _layer(pkg, sum(size for _s, size in _bands(kind, H)), seed=H)
    x = (torch.randn(M, K, generator=torch.Generator().manual_seed(M)) * 0.5).to(DEV).to(dtype)
    for case in CASES:
        patches = _patches(kind, H, seed=M + H, **case)
        _apply(lin, patches)
        assert lin._lora_terms(x.device), case
        n_before = len(ex_calls)
        y = lin(x)
        assert "_gg_lora" in lin.__dict__ and len(ex_calls) == n_before + 1, f"{case}: the in-kernel route was not taken"
        ref, ideal = _references(pkg, lin, x, patches)
        _check(y, ref, ideal, dtype, numerics, case)
    lin.weight.patches = []


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_input_band_and_whole_weight_terms(pkg, dtype, ex_calls):
    """A band of input features (offset dim 1) next to row bands and a whole-weight LoRA."""
    H = 256
    lin = _layer(pkg, 3 * H, seed=9)
    g = torch.Generator().manual_seed(2)
    patches = _patches("qkv", H, rank=32, seed=3)
    patches.append((0.7, (torch.randn(3 * H, 24, generator=g) * 0.05).to(DEV), (torch.randn(24, 256, generator=g) * 0.05).to(DEV), 12.0,
                    (1, 512, 256)))
    patches.append((1.0, (torch.randn(3 * H, 8, generator=g) * 0.05).to(DEV), (torch.randn(8, K, generator=g) * 0.05).to(DEV), 8.0, None))
    _apply(lin, patches)
    x = (torch.randn(300, K, generator=g) * 0.5).to(DEV).to(dtype)
    y = lin(x)
    assert len(ex_calls) == 1
    ref, ideal = _references(pkg, lin, x, patches)
    _check(y, ref, ideal, dtype, "exact", "dim 1")


def _direct(pkg, lin, x, terms, tiles, algo):
    """The fused call with the layer's packed operands and an explicit tile table (or none)."""
    N = lin.weight.tensor_shape[0]
    down_pad, u_pad, _tiles = pkg.ops.lora_kernel_operands(terms, N, K, x.dtype, x.device)
    t = pkg.ops.linear_dense(x, down_pad)
    return pkg.ops._launch_linear(x, pkg.ops._plain(lin.weight), Q.Q4_K, N, K, pkg.ops._plain(lin.bias), pkg.lib.F16, algo, None,
                                  (t, u_pad, tiles))


@pytest.mark.parametrize("M", [3, 300, 1000])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_tile_table_semantics(pkg, dtype, M):
    """count = 0 leaves a tile's features exactly as the unpatched kernel computes them, and the tight table of the packing gives
    the same bits as running every LoRA k-block on every tile (zero U rows add exact zeros)."""
    H = 384
    lin = _layer(pkg, 7 * H, seed=4)
    N = 7 * H
    x = (torch.randn(M, K, generator=torch.Generator().manual_seed(5)) * 0.5).to(DEV).to(dtype)
    algo = pkg.lib.ALGO_FUSED_TMEM | pkg.lib.FLAG_EXACT_W | pkg.lib.FLAG_W_STABLE
    _apply(lin, _patches("linear1", H, rank=48, seed=6))
    terms = lin._lora_terms(x.device)
    _d, u_pad, tight = pkg.ops.lora_kernel_operands(terms, N, K, dtype, x.device)
    J = u_pad.shape[1] // 64
    assert J == 3 and tight is not None
    y_tight = _direct(pkg, lin, x, terms, tight, algo)
    y_all = _direct(pkg, lin, x, terms, None, algo)
    assert torch.equal(y_tight, y_all)
    # switch LoRA off on every other tile
    masked = tight.clone()
    masked[::2, 1] = 0
    y_masked = _direct(pkg, lin, x, terms, masked, algo)
    y_plain = pkg.ops._launch_linear(x, pkg.ops._plain(lin.weight), Q.Q4_K, N, K, pkg.ops._plain(lin.bias), pkg.lib.F16, algo)
    off = torch.zeros(N, dtype=torch.bool, device=DEV)
    for i in range(0, -(-N // 128), 2):
        off[128 * i:128 * i + 128] = True
    assert torch.equal(y_masked[:, off], y_plain[:, off])
    assert torch.equal(y_masked[:, ~off], y_tight[:, ~off])
    assert not torch.equal(y_tight[:, off], y_plain[:, off])
    lin.weight.patches = []


@pytest.mark.parametrize("M", [3, 300])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_lora_ex_with_one_kblock_matches_lora(pkg, dtype, M):
    """ggufb200_linear_lora is ggufb200_linear_lora_ex(ldu = 64, J = 1, no table): the same bits."""
    N = 264
    lin = _layer(pkg, N, seed=11)
    g = torch.Generator().manual_seed(12)
    x = (torch.randn(M, K, generator=g) * 0.5).to(DEV).to(dtype)
    terms = [(0.5, (torch.randn(N, 40, generator=g) * 0.05).to(DEV), (torch.randn(40, K, generator=g) * 0.05).to(DEV), None)]
    down_pad, u_pad, tiles = pkg.ops.lora_kernel_operands(terms, N, K, dtype, x.device)
    assert tiles is None and u_pad.shape[1] == 64
    t = pkg.ops.linear_dense(x, down_pad)
    L = pkg.lib.lib()
    w, b = pkg.ops._plain(lin.weight), pkg.ops._plain(lin.bias)
    act = pkg.dequant.dtype_code(dtype)
    stream = torch.cuda.current_stream().cuda_stream
    for algo in (pkg.lib.ALGO_FUSED_TMEM, pkg.lib.ALGO_FUSED_TMEM | pkg.lib.FLAG_EXACT_W):
        need = L.ggufb200_linear_workspace_ex(int(Q.Q4_K), M, N, K, act, pkg.lib.F16, algo)
        ws = torch.empty(max(need, 16), dtype=torch.uint8, device=DEV)
        y0 = torch.empty(M, N, dtype=dtype, device=DEV)
        y1 = torch.full((M, N), float("nan"), dtype=dtype, device=DEV)
        head = (int(Q.Q4_K), w.data_ptr(), None, N, K, x.data_ptr(), M, K, act, b.data_ptr(), pkg.dequant.dtype_code(b.dtype), t.data_ptr(), 64,
                u_pad.data_ptr())
        tail = (ws.data_ptr(), need, algo, stream)
        pkg.lib.check(L.ggufb200_linear_lora(*head, y0.data_ptr(), N, *tail), "lora")
        pkg.lib.check(L.ggufb200_linear_lora_ex(*head, 64, 1, None, y1.data_ptr(), N, *tail), "lora_ex")
        assert torch.equal(y0, y1), algo


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [3, 300])
def test_above_the_cap_and_knob_off_use_band_aware_side_gemms(pkg, dtype, M, ex_calls):
    H = 256
    lin = _layer(pkg, 7 * H, seed=13)
    x = (torch.randn(M, K, generator=torch.Generator().manual_seed(14)) * 0.5).to(DEV).to(dtype)
    big = _patches("linear1", H, rank=144, seed=15)                  # Σr = 576 > 512
    _apply(lin, big)
    y = lin(x)
    assert not ex_calls and "_gg_lora" not in lin.__dict__
    ref, ideal = _references(pkg, lin, x, big)
    _check(y, ref, ideal, dtype, "exact", "above the cap")
    small = _patches("linear1", H, rank=32, seed=16)
    _apply(lin, small)
    lin.lora_in_kernel = False
    try:
        y = lin(x)
    finally:
        del lin.lora_in_kernel
    assert not ex_calls and "_gg_lora" not in lin.__dict__
    ref, ideal = _references(pkg, lin, x, small)
    _check(y, ref, ideal, dtype, "exact", "lora_in_kernel = False")
    lin.weight.patches = []
