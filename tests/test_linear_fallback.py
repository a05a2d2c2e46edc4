"""CPU tests of the Linear and the row gather of the numpy-fallback types (ggufb200_linear_fallback,
ggufb200_linear_fallback_workspace, ggufb200_dequant_rows_fallback): argument validation before any device is touched, the
supported sets, the header constants and the workspace query's route choice."""
import ctypes
import os
import re

import gguf
import pytest

from fallback_cases import FALLBACK
from linear_fallback_cases import CROSSOVER, auto_fused, plan_problems, splits_of
from util import ALL_QTYPES, Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, E_TYPE, E_DTYPE, E_ALIGN, E_SHAPE, E_NULL, E_UNSUPPORTED = 0, -1, -2, -3, -4, -5, -8


@pytest.fixture()
def bufs():
    """Two 16-byte aligned host addresses (the argument checks never dereference them)."""
    buf = (ctypes.c_uint8 * 8192)()
    p = (ctypes.addressof(buf) + 15) & ~15
    yield p, p + 4096
    del buf


def _linear(L, qt=Q.IQ2_XS, W=None, N=64, K=512, X=None, M=16, ldx=None, act=1, bias=None, bias_dtype=0, Y=None, ldy=None, ws=None,
            ws_bytes=0, algo=0):
    return L.ggufb200_linear_fallback(int(qt), W, N, K, X, M, K if ldx is None else ldx, act, bias, bias_dtype, Y, N if ldy is None else ldy,
                                      ws, ws_bytes, algo, None)


def test_linear_argument_validation(pkg, bufs):
    L, lib = pkg.lib.lib(), pkg.lib
    p, q = bufs
    args = dict(W=p, X=p, Y=q)
    assert _linear(L, qt=Q.Q4_K, **args) == E_TYPE                  # table types keep ggufb200_linear
    assert _linear(L, qt=999, **args) == E_TYPE
    assert _linear(L, qt=Q.BF16, **args) == E_TYPE
    assert _linear(L, act=2, **args) == E_DTYPE                      # fp32 activations
    assert _linear(L, act=7, **args) == E_DTYPE
    assert _linear(L, bias=p, bias_dtype=5, **args) == E_DTYPE
    assert _linear(L, K=384, **args) == E_SHAPE                      # K % 256 != 0
    assert _linear(L, qt=Q.MXFP4, K=36, **args) == E_SHAPE           # K % 8 != 0 (and % 32)
    assert _linear(L, N=60, **args) == E_SHAPE                       # N % 8 != 0
    assert _linear(L, N=0, **args) == E_SHAPE
    assert _linear(L, M=-1, **args) == E_SHAPE
    assert _linear(L, ldx=504, **args) == E_SHAPE
    assert _linear(L, ldy=56, **args) == E_SHAPE
    assert _linear(L, M=0, W=None, X=None, Y=None) == OK             # nothing to do: no pointer checked, no device touched
    assert _linear(L, W=None, X=p, Y=q) == E_NULL
    assert _linear(L, W=p, X=None, Y=q) == E_NULL
    assert _linear(L, W=p, X=p, Y=None) == E_NULL
    assert _linear(L, W=p, X=p + 2, Y=q) == E_ALIGN
    assert _linear(L, W=p, X=p, Y=q + 8) == E_ALIGN
    assert _linear(L, ldx=516, **args) == E_ALIGN
    assert _linear(L, ldy=68, **args) == E_ALIGN
    # a packed base below the type's block alignment needs DEQUANT_MMA's workspace
    assert _linear(L, W=p + 1, X=p, Y=q) == E_ALIGN
    assert _linear(L, W=p + 1, X=p, Y=q, algo=lib.ALGO_FUSED_SYNC) == E_ALIGN
    for algo in (lib.ALGO_GEMV, lib.ALGO_GEMV_FAST, lib.ALGO_FUSED_MMA, lib.ALGO_FUSED_TMEM, 7, 0xFF):
        assert _linear(L, algo=algo, **args) == E_UNSUPPORTED, algo
    for flag in (lib.FLAG_GENERIC, lib.FLAG_TILE384, lib.FLAG_TILE192, lib.FLAG_UNSTAGED, 0x8000):
        assert _linear(L, algo=lib.ALGO_FUSED_SYNC | flag, **args) == E_UNSUPPORTED, flag


def test_rows_argument_validation(pkg, bufs):
    L = pkg.lib.lib()
    p, q = bufs

    def rows(qt=Q.IQ3_S, packed=p, n_table=100, K=512, idx=p, n=4, out=q, out_dtype=1):
        return L.ggufb200_dequant_rows_fallback(int(qt), packed, n_table, K, idx, n, out, out_dtype, None)
    assert rows(qt=Q.Q8_0) == E_TYPE
    assert rows(qt=Q.BF16) == E_TYPE
    assert rows(qt=1000) == E_TYPE
    assert rows(out_dtype=3) == E_DTYPE
    assert rows(out_dtype=-1) == E_DTYPE
    assert rows(K=384) == E_SHAPE
    assert rows(qt=Q.MXFP4, K=40) == E_SHAPE
    assert rows(K=0) == E_SHAPE
    assert rows(n=-1) == E_SHAPE
    assert rows(n_table=-1) == E_SHAPE
    assert rows(n=0, packed=None, idx=None, out=None) == OK
    assert rows(packed=None) == E_NULL
    assert rows(idx=None) == E_NULL
    assert rows(out=None) == E_NULL
    assert rows(out=q + 4) == E_ALIGN


def test_supported_sets(pkg):
    L, lib = pkg.lib.lib(), pkg.lib
    fallback = {int(q) for q in pkg.dequant.FALLBACK_QTYPES}
    assert fallback == {int(q) for q in FALLBACK}
    for op in (lib.OP_LINEAR_FALLBACK, lib.OP_ROWS_FALLBACK):
        assert {int(q) for q in Q if L.ggufb200_supported(int(q), op)} == fallback, op
        for code in (999, -1, 1000):
            assert L.ggufb200_supported(code, op) == 0
    for q in ALL_QTYPES:                  # the table types keep their own entry points
        assert L.ggufb200_supported(int(q), lib.OP_LINEAR_FALLBACK) == 0
        assert L.ggufb200_supported(int(q), lib.OP_ROWS_FALLBACK) == 0


def test_new_defines_match_lib(pkg):
    hdr = open(os.path.join(ROOT, "include", "ggufb200.h")).read()
    defines = {m.group(1): int(m.group(2), 0) for m in re.finditer(r"^#define\s+GGUFB200_(\w+)\s+\(?(-?(?:0x[0-9A-Fa-f]+|\d+))\)?", hdr, re.M)}
    assert defines["OP_LINEAR_FALLBACK"] == pkg.lib.OP_LINEAR_FALLBACK == 7
    assert defines["OP_ROWS_FALLBACK"] == pkg.lib.OP_ROWS_FALLBACK == 8
    assert defines["ALGO_FUSED_SYNC"] == pkg.lib.ALGO_FUSED_SYNC == 6
    algos = [v for k, v in defines.items() if k.startswith("ALGO_") and k != "ALGO_MASK"]
    assert len(algos) == len(set(algos))
    for sym in ("ggufb200_linear_fallback", "ggufb200_linear_fallback_workspace", "ggufb200_linear_fallback_route",
                "ggufb200_dequant_rows_fallback"):
        assert sym in pkg.lib.EXPORTS


@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_workspace_follows_auto(pkg, qt):
    """Up to the crossover, where the kernel splits K, AUTO takes FUSED_SYNC, which needs only its split-K slices; above it, or
    on a grid that runs unsplit, DEQUANT_MMA, N * K * 2."""
    L, lib = pkg.lib.lib(), pkg.lib
    bs = gguf.GGML_QUANT_SIZES[qt][0]
    c = CROSSOVER[qt]
    for N, K in ((2560, 9728), (9728, 2560), (128, 1024), (4096, 256 if bs <= 256 else bs), (16896, 256), (16768, 256)):
        for act in (lib.F16, lib.BF16):
            for M in sorted({1, 9, 64, max(c - 1, 1), c + 1, 512, 5000} | ({c} if c else set())):
                auto = L.ggufb200_linear_fallback_workspace(int(qt), M, N, K, act, lib.ALGO_AUTO)
                fused = L.ggufb200_linear_fallback_workspace(int(qt), M, N, K, act, lib.ALGO_FUSED_SYNC)
                dense = L.ggufb200_linear_fallback_workspace(int(qt), M, N, K, act, lib.ALGO_DEQUANT_MMA)
                assert dense == N * K * 2
                assert not plan_problems(M, N, K, fused), (M, N, K, plan_problems(M, N, K, fused))
                assert auto == (fused if auto_fused(qt, M, fused) else dense), (M, N, K)
                route = L.ggufb200_linear_fallback_route(int(qt), M, N, K, act, lib.ALGO_AUTO)
                assert route == (lib.ALGO_FUSED_SYNC if auto_fused(qt, M, fused) else lib.ALGO_DEQUANT_MMA), (M, N, K)
                for algo in (lib.ALGO_FUSED_SYNC, lib.ALGO_DEQUANT_MMA):
                    assert L.ggufb200_linear_fallback_route(int(qt), M, N, K, act, algo) == algo
                assert L.ggufb200_linear_fallback_workspace(int(qt), M, N, K, act, lib.ALGO_FUSED_SYNC | lib.FLAG_NOSPLIT) == 0
                assert L.ggufb200_linear_fallback_workspace(int(qt), M, N, K, act, lib.ALGO_AUTO | lib.FLAG_W_STABLE | lib.FLAG_EXACT_W) == auto
    # a grid that runs unsplit: DEQUANT_MMA at every M
    assert L.ggufb200_linear_fallback_workspace(int(qt), 16, 9728, 2560, lib.BF16, lib.ALGO_AUTO) == 9728 * 2560 * 2
    # split K engages where the tile grid is short: one feature tile, one token tile
    assert splits_of(L.ggufb200_linear_fallback_workspace(int(qt), 64, 128, 8192, lib.BF16, lib.ALGO_FUSED_SYNC), 64, 128) > 1
    # refused arguments: 0 from the workspace query, the call's error code from the route query
    assert L.ggufb200_linear_fallback_route(int(qt), 64, 128, 8192, lib.BF16, lib.ALGO_FUSED_TMEM) == E_UNSUPPORTED
    assert L.ggufb200_linear_fallback_route(int(qt), 64, 100, 8192, lib.BF16, lib.ALGO_AUTO) == E_SHAPE
    assert L.ggufb200_linear_fallback_route(int(qt), 64, 128, 8192, lib.F32, lib.ALGO_AUTO) == E_DTYPE
    assert L.ggufb200_linear_fallback_route(int(Q.Q4_K), 64, 128, 8192, lib.BF16, lib.ALGO_AUTO) == E_TYPE
    assert L.ggufb200_linear_fallback_workspace(int(qt), 64, 128, 8192, lib.BF16, lib.ALGO_FUSED_TMEM) == 0
    assert L.ggufb200_linear_fallback_workspace(int(qt), 64, 100, 8192, lib.BF16, lib.ALGO_AUTO) == 0
    assert L.ggufb200_linear_fallback_workspace(int(qt), 0, 128, 8192, lib.BF16, lib.ALGO_AUTO) == 0
    assert L.ggufb200_linear_fallback_workspace(int(Q.Q4_K), 64, 128, 8192, lib.BF16, lib.ALGO_AUTO) == 0


def test_split_plan_properties(pkg):
    """FUSED_SYNC's K ranges over a sweep of shapes: checked as properties (plan_problems), not against a copy of the planner."""
    L, lib = pkg.lib.lib(), pkg.lib
    seen = set()
    for N in (8, 128, 136, 1024, 2560, 4224, 8448, 9728, 16896, 32768):
        for K in (256, 512, 1024, 2560, 8192, 32768):
            for M in (1, 9, 64, 65, 128, 200, 1000, 9000):
                ws = L.ggufb200_linear_fallback_workspace(int(Q.IQ2_XS), M, N, K, lib.BF16, lib.ALGO_FUSED_SYNC)
                assert not plan_problems(M, N, K, ws), (M, N, K, plan_problems(M, N, K, ws))
                seen.add(splits_of(ws, M, N))
    assert 1 in seen and max(seen) > 2


def test_empty_batch_queries(pkg):
    """M == 0: the call computes nothing and returns OK, so the route query returns OK and the workspace query 0 for every algo."""
    L, lib = pkg.lib.lib(), pkg.lib
    for qt in FALLBACK:
        for algo in (lib.ALGO_AUTO, lib.ALGO_FUSED_SYNC, lib.ALGO_DEQUANT_MMA, lib.ALGO_AUTO | lib.FLAG_NOSPLIT):
            for act in (lib.F16, lib.BF16):
                assert L.ggufb200_linear_fallback_route(int(qt), 0, 128, 512, act, algo) == OK, (qt, algo)
                assert L.ggufb200_linear_fallback_workspace(int(qt), 0, 128, 512, act, algo) == 0, (qt, algo)
    assert L.ggufb200_linear_fallback_route(int(Q.IQ2_XS), -1, 128, 512, lib.BF16, lib.ALGO_AUTO) == E_SHAPE
