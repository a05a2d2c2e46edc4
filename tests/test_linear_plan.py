"""Host arithmetic of the fused Linear's tiling (csrc/linear_sm90.cu::mma_splits for
GGUFB200_ALGO_FUSED_MMA, exported as ggufb200_linear_plan).

A wrong plan is the kind of bug that HANGS a GPU (a K range with no k-blocks never signals its barriers), so the invariants
are checked here on the CPU over many shapes: every K range owns whole 256-wide spans, none is empty, together they cover K
exactly once, the slices fit the workspace, the grid fits one wave of the 132 SMs when K is split, and the workspace query, the plan
and the AUTO routing agree with each other."""
import ctypes

import pytest
from hypothesis import given, settings, strategies as st

from util import Q

SMS = 132           # an H100 SXM (sm_count() reports 132 without a device as well)
CAP = 24 << 20


FUSED_MMA, FUSED_TMEM, NOSPLIT, TILE384, TILE192 = 2, 4, 0x800, 0x400, 0x2000


def _plan(L, qt, M, N, K, ws, algo=FUSED_MMA):
    vals = [ctypes.c_int() for _ in range(4)]
    rc = L.ggufb200_linear_plan(int(qt), M, N, K, ws, algo, *[ctypes.byref(v) for v in vals])
    return rc, tuple(v.value for v in vals)


def _check(L, M, N, K, ws):
    rc, (rows, ranges, kb, ctas) = _plan(L, Q.Q4_K, M, N, K, ws)
    assert rc == 0
    assert rows == 128 and ranges >= 1 and kb >= 1
    total_kb = K // 64
    tiles = -(-M // rows) * -(-N // 256)
    assert ctas == tiles * ranges                                # one CTA per (128 x 256 tile, K range)
    if ranges == 1:
        assert kb == total_kb
        return ranges
    assert K % 256 == 0 and kb % 4 == 0                        # whole spans per range
    assert (ranges - 1) * kb < total_kb <= ranges * kb          # no empty range, full cover
    assert ranges <= 16 and ctas <= SMS                         # one wave of CTAs
    assert ranges * M * N * 4 <= min(ws, CAP)                   # slices fit what the caller gave (and the L2 budget)
    return ranges


def test_known_plans(pkg):
    L = pkg.lib.lib()
    assert _plan(L, Q.Q4_K, 512, 3072, 12288, CAP) == (0, (128, 2, 96, 96))       # 48 tiles x 2 ranges
    assert _plan(L, Q.Q4_K, 64, 3072, 12288, CAP) == (0, (128, 10, 20, 120))      # 12 tiles x 10 ranges
    assert _plan(L, Q.Q5_K, 512, 4096, 4096, CAP) == (0, (128, 2, 32, 128))        # T5 q/k/v/o
    assert _plan(L, Q.Q4_K, 4608, 3072, 3072, CAP)[1][1] == 1                      # plenty of tiles: unsplit
    assert _plan(L, Q.Q4_K, 512, 3072, 12288, 0)[1][1] == 1                        # no workspace: unsplit
    assert _plan(L, Q.Q4_K, 64, 3072, 12288, 3 * 64 * 3072 * 4)[1][1] == 3         # smaller workspace: fewer ranges
    assert _plan(L, Q.Q4_K, 64, 512, 4096 + 64, CAP)[1][1] == 1                    # K not a multiple of 256: unsplit
    assert _plan(L, Q.BF16, 64, 512, 4096, CAP)[0] == -8                           # no fused kernel for dense weights
    assert _plan(L, Q.Q4_K, 64, 512, 4000, CAP)[0] == -4
    assert _plan(L, 99, 64, 512, 4096, CAP)[0] == -1


@settings(max_examples=600, deadline=None)
@given(M=st.integers(9, 1500), n8=st.integers(1, 3000), k64=st.integers(1, 400), ws_slices=st.integers(0, 20))
def test_plan_invariants(pkg, M, n8, k64, ws_slices):
    L = pkg.lib.lib()
    N, K = 8 * n8, 64 * k64
    ws = ws_slices * M * N * 4
    ranges = _check(L, M, N, K, ws)
    # the size the library asks for is exactly what the plan with that size uses
    need = L.ggufb200_linear_workspace(int(Q.Q4_K), M, N, K, 1, pkg.lib.ALGO_FUSED_MMA)
    assert need % (M * N * 4) == 0 and need <= CAP
    if need:
        assert _check(L, M, N, K, need) == need // (M * N * 4) >= 2
    else:
        assert _check(L, M, N, K, CAP) == 1
    assert ranges <= max(1, need // (M * N * 4))


def test_nosplit_flag_disables_every_split(pkg):
    L = pkg.lib.lib()
    for M, N, K in ((64, 512, 4096), (512, 3072, 12288), (1000, 256, 5120)):
        assert _plan(L, Q.Q4_K, M, N, K, CAP, FUSED_MMA | NOSPLIT)[1][1] == 1
        assert _plan(L, Q.Q4_K, M, N, K, CAP, FUSED_TMEM | NOSPLIT)[1][1] == 1
        assert L.ggufb200_linear_workspace(int(Q.Q4_K), M, N, K, 1, FUSED_TMEM | NOSPLIT) == 0


# ---------------------------------------------------------------- FUSED_TMEM kernel (csrc/linear_sm90.cu::tmem_plan)
def _check_tmem(L, M, N, K, ws, flags=0):
    rc, (tokens, ranges, kb, items) = _plan(L, Q.Q4_K, M, N, K, ws, FUSED_TMEM | flags)
    assert rc == 0
    assert tokens in (32, 128, 192, 384) and ranges >= 1 and kb >= 4 and kb % 4 == 0      # whole 256-wide spans
    spans = -(-K // 256)
    per = kb // 4
    assert (ranges - 1) * per < spans <= ranges * per              # no empty K range, exact cover
    tiles = -(-M // tokens) * -(-N // 256)
    assert items == tiles * ranges
    if ranges > 1:
        assert ranges <= 32
        assert ranges * M * N * 4 <= min(ws, CAP)
    if M <= 32:
        assert tokens == 32
    if flags & TILE384 and M > 192:
        assert tokens == 384
    if flags & TILE192 and M > 192:
        assert tokens == 192
    return ranges


def test_known_tmem_plans(pkg):
    L = pkg.lib.lib()
    assert _plan(L, Q.Q4_K, 4608, 12288, 3072, CAP, FUSED_TMEM | TILE192) == (0, (192, 1, 48, 48 * 24))      # Flux mlp.0: 1152 items
    assert _plan(L, Q.Q4_K, 4608, 12288, 3072, CAP, FUSED_TMEM | TILE384) == (0, (384, 1, 48, 48 * 12))
    assert _plan(L, Q.Q4_K, 4608, 12288, 3072, CAP, FUSED_TMEM) == (0, (192, 1, 48, 48 * 24))               # the cost model's pick
    assert _plan(L, Q.Q4_K, 512, 3072, 12288, CAP, FUSED_TMEM) == (0, (192, 3, 64, 108))                     # 36 tiles x 3 K ranges
    assert _plan(L, Q.Q4_K, 1, 18432, 3072, CAP, FUSED_TMEM) == (0, (32, 4, 12, 288))              # modulation GEMV shape: 72 feature tiles x 4 K ranges
    assert _plan(L, Q.Q4_K, 1, 3072, 3072, CAP, FUSED_TMEM) == (0, (32, 4, 12, 48))                # 12 feature tiles x 4 K ranges
    assert _plan(L, Q.Q4_K, 1, 3072, 3072, 0, FUSED_TMEM)[1][1] == 1                               # no workspace: unsplit
    assert _plan(L, Q.Q5_K, 512, 4096, 4096, CAP, FUSED_TMEM) == (0, (128, 1, 64, 64))             # T5 q/k/v/o at 512 tokens
    assert _plan(L, Q.BF16, 64, 512, 4096, CAP, FUSED_TMEM)[0] == -8


@settings(max_examples=400, deadline=None)
@given(M=st.integers(1, 5000), n8=st.integers(1, 3000), k64=st.integers(1, 300), ws_slices=st.integers(0, 40),
       tile=st.sampled_from([0, TILE384, TILE192]))
def test_tmem_plan_invariants(pkg, M, n8, k64, ws_slices, tile):
    L = pkg.lib.lib()
    N, K = 8 * n8, 64 * k64
    flags = tile
    ws = min(ws_slices * M * N * 4, 1 << 40)
    ranges = _check_tmem(L, M, N, K, ws, flags)
    need = L.ggufb200_linear_workspace(int(Q.Q4_K), M, N, K, 1, FUSED_TMEM | flags)
    assert need % (M * N * 4) == 0 and need <= CAP
    if need:
        assert _check_tmem(L, M, N, K, need, flags) == need // (M * N * 4) >= 2
    else:
        assert _check_tmem(L, M, N, K, CAP, flags) == 1
    assert ranges <= max(1, need // (M * N * 4))
