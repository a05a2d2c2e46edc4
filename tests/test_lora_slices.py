"""CPU tests of LoRA patches on a band of a packed weight (diffusers-format slices such as Flux's q / k / v on `qkv`) and of
LoRA stacks above rank 64: argument validation of ggufb200_linear_lora_ex, the patch recogniser, the packing of the kernel
operands with the per-tile k-block table, and the band-aware side GEMMs."""
import ctypes

import pytest
import torch

import oracle
from util import Q

E_ALIGN, E_SHAPE, E_NULL, E_UNSUPPORTED = -3, -4, -5, -8


def _lora_ex(L, p16, algo, T=True, ldt=64, ldu=64, J=1, tiles=None):
    x = p16
    return L.ggufb200_linear_lora_ex(int(Q.Q4_K), p16, None, 8, 256, x, 4, 256, 1, None, 0, x if T else None, ldt, x, ldu, J, tiles,
                                     x, 8, None, 0, algo, None)


def test_lora_ex_validates_without_gpu(pkg):
    L = pkg.lib.lib()
    buf = (ctypes.c_uint8 * 4096)()
    p16 = (ctypes.addressof(buf) + 15) & ~15
    tmem = pkg.lib.ALGO_FUSED_TMEM
    for J in (0, 9, -1):
        assert _lora_ex(L, p16, tmem, ldt=64 * 9, ldu=64 * 9, J=J) == E_SHAPE
    assert _lora_ex(L, p16, pkg.lib.ALGO_GEMV) == E_UNSUPPORTED          # the update only rides on the FUSED_TMEM kernel
    assert _lora_ex(L, p16, tmem, T=False) == E_NULL
    assert _lora_ex(L, p16, tmem, ldt=48) == E_ALIGN
    assert _lora_ex(L, p16, tmem, ldu=48) == E_ALIGN
    assert _lora_ex(L, p16, tmem, J=2, ldt=128, ldu=64) == E_ALIGN       # U narrower than 64 J
    assert _lora_ex(L, p16, tmem, J=2, ldt=64, ldu=128) == E_ALIGN       # T narrower than 64 J
    assert _lora_ex(L, p16, tmem, J=2, ldt=132, ldu=128) == E_ALIGN      # not a multiple of 8
    assert _lora_ex(L, p16, tmem, J=2, ldt=128, ldu=130) == E_ALIGN
    assert _lora_ex(L, p16, tmem, J=1, tiles=p16 + 2) == E_ALIGN         # int32 pairs
    # the original entry point is the J = 1, ldu = 64, no-table call: same answers
    assert L.ggufb200_linear_lora(int(Q.Q4_K), p16, None, 8, 256, p16, 4, 256, 1, None, 0, p16, 48, p16, p16, 8, None, 0, tmem, None) == E_ALIGN


class LoRAAdapter:                  # newer ComfyUI wraps the (up, down, alpha, mid, dora_scale, reshape) tuple in an adapter object
    def __init__(self, weights):
        self.weights = weights


def test_band_recogniser_accepts_offsets_and_rejects_the_rest(pkg):
    f = pkg.ops.lora_band_terms
    up, down = torch.ones(8, 2), torch.ones(2, 16)
    lora = ("lora", (up, down, 4.0, None, None, None))
    terms = f([(0.5, lora, 1.0, (0, 8, 8), None), (1.0, LoRAAdapter((up, down, None, None, None, None)), 1.0, (1, 0, 16), None),
               (1.0, ("lora", (up, down, None)), 1.0)])
    assert [t[3] for t in terms] == [(0, 8, 8), (1, 0, 16), None]
    assert [t[0] for t in terms] == [0.5 * 4.0 / 2, 1.0, 1.0] and terms[0][1] is up and terms[0][2] is down
    assert f([]) == []
    # an offset is only a band when it names dim 0 or 1
    assert f([(0.5, lora, 1.0, (2, 0, 4), None)]) is None
    assert f([(0.5, lora, 1.0, (0, 0), None)]) is None
    assert f([(0.5, lora, 1.0, (0, -1, 4), None)]) is None
    # the kinds that keep the two-step route
    assert f([(0.5, lora, 0.7, (0, 0, 8), None)]) is None                                         # strength_model
    assert f([(0.5, lora, 1.0, (0, 0, 8), lambda w: w)]) is None                                  # function hook
    assert f([(0.5, ("diff", (up,)), 1.0, (0, 0, 8), None)]) is None
    assert f([(0.5, up, 1.0, None, None)]) is None                                                # bare tensor = diff
    assert f([(0.5, ("lora", (up, down, 4.0, torch.ones(2, 2), None, None)), 1.0, (0, 0, 8), None)]) is None   # LoCon mid
    assert f([(0.5, LoRAAdapter((up, down, 4.0, None, torch.ones(8), None)), 1.0, (0, 0, 8), None)]) is None   # DoRA
    assert f([(0.5, ("lora", (up, down, 4.0, None, None, (8, 16))), 1.0, None, None)]) is None    # reshape
    assert f([(0.5, ("loha", (up, down)), 1.0, None, None)]) is None

    class LoKrAdapter(LoRAAdapter):
        pass
    assert f([(0.5, LoKrAdapter((up, down, 4.0, None, None, None)), 1.0, None, None)]) is None
    # lora_side_terms keeps its contract: no band
    assert pkg.ops.lora_side_terms([(0.5, lora, 1.0, (0, 8, 8), None)]) is None


def _linear(pkg, N, K):
    raw = oracle.random_blocks(int(Q.Q4_K), N * K // 256, seed=3).reshape(N, K // 256 * 144)
    lin = pkg.ops.GGMLOps.Linear(K, N)
    lin.load_state_dict({"weight": pkg.ops.GGMLTensor(torch.from_numpy(raw), tensor_type=Q.Q4_K, tensor_shape=torch.Size((N, K)))})
    return lin


def test_layer_checks_band_shapes(pkg):
    N, K = 96, 512
    lin = _linear(pkg, N, K)
    cpu = torch.device("cpu")

    def patch(up, down, offset):
        lin.weight.patches = [([(1.0, ("lora", (up, down, None, None, None, None)), 1.0, offset, None)], "w")]
        return lin._lora_terms(cpu)
    assert patch(torch.ones(32, 4), torch.ones(4, K), (0, 64, 32))[0][3] == (0, 64, 32)
    assert patch(torch.ones(N, 4), torch.ones(4, 256), (1, 256, 256))[0][3] == (1, 256, 256)
    assert patch(torch.ones(32, 4), torch.ones(4, K), (0, 80, 32)) is None          # band past N
    assert patch(torch.ones(N, 4), torch.ones(4, 256), (1, 384, 256)) is None       # band past K
    assert patch(torch.ones(N, 4), torch.ones(4, K), (0, 0, 32)) is None            # up rows != band
    assert patch(torch.ones(N, 4), torch.ones(4, K), (1, 0, 256)) is None           # down columns != band
    lin.weight.patches = []


def _flux_terms(H, K, rank, g, dim1=False):
    """`qkv` + `proj_mlp` slices of a Flux single block's linear1 (N = 3 H + 4 H), in ComfyUI's offset form."""
    terms = []
    for start, size in ((0, H), (H, H), (2 * H, H), (3 * H, 4 * H)):
        terms.append((0.5 + 0.1 * len(terms), torch.randn(size, rank, generator=g), torch.randn(rank, K, generator=g), (0, start, size)))
    if dim1:
        terms.append((0.25, torch.randn(7 * H, 8, generator=g), torch.randn(8, K // 2, generator=g), (1, K // 4, K // 2)))
    return terms


def _dense_delta(terms, N, K, u_fp16=True):
    """The straightforward construction: each scale * up @ down added on its band of an [N, K] zero matrix (scale * up
    rounded to fp16 like the kernel operand when u_fp16)."""
    delta = torch.zeros(N, K, dtype=torch.float64)
    for scale, up, down, band in terms:
        u = up.float() * scale
        d = (u.half() if u_fp16 else u).double() @ down.double()
        if band is None:
            delta += d
        elif band[0] == 0:
            delta[band[1]:band[1] + band[2]] += d
        else:
            delta[:, band[1]:band[1] + band[2]] += d
    return delta


def _tight_table(u_pad):
    """(first, count) per 128-row tile: the k-blocks with a non-zero U entry on the tile's rows."""
    N, J = u_pad.shape[0], u_pad.shape[1] // 64
    out = []
    for i in range(-(-N // 128)):
        nz = [j for j in range(J) if bool((u_pad[128 * i:128 * i + 128, 64 * j:64 * j + 64] != 0).any())]
        out.append((nz[0], nz[-1] - nz[0] + 1) if nz else (0, 0))
    return out


@pytest.mark.parametrize("H,rank,dim1", [(256, 16, False), (384, 48, False), (256, 80, False), (384, 16, True), (256, 32, True)])
def test_operand_packing_and_tile_table(pkg, H, rank, dim1):
    g = torch.Generator().manual_seed(H + rank)
    N, K = 7 * H, 1024
    terms = _flux_terms(H, K, rank, g, dim1)
    down_pad, u_pad, tiles = pkg.ops.lora_kernel_operands(terms, N, K, torch.float32, torch.device("cpu"))
    R = sum(d.shape[0] for _s, _u, d, _b in terms)
    J = -(-R // 64)
    assert tuple(down_pad.shape) == (64 * J, K) and tuple(u_pad.shape) == (N, 64 * J) and u_pad.dtype == torch.float16
    assert torch.count_nonzero(down_pad[R:]) == 0 and torch.count_nonzero(u_pad[:, R:]) == 0      # padding past the total rank
    assert torch.allclose(u_pad.double() @ down_pad.double(), _dense_delta(terms, N, K), rtol=0, atol=1e-9)
    assert tiles is not None and tiles.dtype == torch.int32 and tuple(tiles.shape) == (-(-N // 128), 2)
    assert [tuple(p) for p in tiles.tolist()] == _tight_table(u_pad)
    if not dim1:
        # disjoint row bands: every tile runs only the k-blocks of the bands it overlaps
        for i, (first, count) in enumerate(tiles.tolist()):
            r0s = [sum(d.shape[0] for _s, _u, d, _b in terms[:t]) for t in range(len(terms))]
            own = [t for t, (_s, _u, _d, b) in enumerate(terms) if b[1] < 128 * (i + 1) and 128 * i < b[1] + b[2]]
            lo, hi = min(r0s[t] for t in own), max(r0s[t] + rank for t in own)
            assert (first, count) == (lo // 64, (hi - 1) // 64 - lo // 64 + 1)


def test_whole_weight_terms_pack_as_before(pkg):
    """Plain LoRA (no band) with total rank <= 64: one k-block, no table, the columns in patch order."""
    g = torch.Generator().manual_seed(0)
    N, K = 200, 256
    terms = [(0.5, torch.randn(N, 4, generator=g), torch.randn(4, K, generator=g), None),
             (2.0, torch.randn(N, 8, generator=g), torch.randn(8, K, generator=g), None)]
    down_pad, u_pad, tiles = pkg.ops.lora_kernel_operands(terms, N, K, torch.bfloat16, torch.device("cpu"))
    assert tiles is None and tuple(down_pad.shape) == (64, K) and tuple(u_pad.shape) == (N, 64)
    assert torch.equal(down_pad[:12], torch.cat([terms[0][2], terms[1][2]]).to(torch.bfloat16))
    assert torch.equal(u_pad[:, :12], torch.cat([(terms[0][1] * 0.5).half(), (terms[1][1] * 2.0).half()], 1))
    # a stack above rank 64 spans several k-blocks and still needs no table
    big = terms + [(1.0, torch.randn(N, 60, generator=g), torch.randn(60, K, generator=g), None)]
    down_pad, u_pad, tiles = pkg.ops.lora_kernel_operands(big, N, K, torch.float32, torch.device("cpu"))
    assert tiles is None and tuple(u_pad.shape) == (N, 128)
    assert torch.allclose(u_pad.double() @ down_pad.double(), _dense_delta(big, N, K), rtol=0, atol=1e-9)


def test_side_gemms_honour_the_bands(pkg):
    """`_add_lora` (Σr above the in-kernel cap, lora_in_kernel = False, no fused route) adds each term on its bands only."""
    g = torch.Generator().manual_seed(5)
    H, K = 64, 256
    N = 7 * H
    terms = _flux_terms(H, K, 8, g, dim1=True)
    lin = pkg.ops.GGMLOps.Linear(K, N)
    x = torch.randn(3, 5, K, generator=g)
    y = torch.zeros(3, 5, N)
    got = lin._add_lora(y, x, terms)
    want = x.double() @ _dense_delta(terms, N, K, u_fp16=False).t()
    assert got is y and torch.allclose(got.double(), want, rtol=1e-4, atol=1e-4)
