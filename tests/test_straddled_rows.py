"""CPU tests of straddled K-quant weights: the GGUF converter reshapes SD1.5 / SDXL tensors whose last dimension is not a
multiple of 256 to [n / 256, 256] before quantising, so a Linear [N, K] with K % 256 != 0 arrives as a flat stream of
N * K / 256 super-blocks whose rows start inside blocks.  Argument validation, routing, workspace and shadow-copy geometry
need no device; the reference values come from the golden files of tests/golden/make_golden_straddled.py."""
import ctypes
import os

import gguf
import numpy as np
import pytest
import torch

import oracle
from util import Q, bits_to_f32, rel_fro

PITCH = {Q.Q2_K: 112, Q.Q3_K: 112, Q.Q6_K: 240, Q.IQ4_XS: 144}
K_QUANTS = [Q.Q2_K, Q.Q3_K, Q.Q4_K, Q.Q5_K, Q.Q6_K, Q.IQ4_XS]


@pytest.fixture
def p16():
    buf = (ctypes.c_uint8 * 4096)()
    yield (ctypes.addressof(buf) + 15) & ~15
    del buf


def _linear(L, qt, N, K, M, p, algo=0):
    return L.ggufb200_linear(int(qt), p, N, K, p, M, K, 1, 0, None, 0, p, N, None, 0, algo, None)


@pytest.mark.parametrize("qt", K_QUANTS, ids=lambda q: q.name)
def test_straddled_shapes_are_accepted(pkg, qt, p16):
    L = pkg.lib.lib()
    assert _linear(L, qt, 8, 640, 0, p16) == 0           # 8 * 640 = 20 blocks: accepted (M = 0 is a no-op)
    assert _linear(L, qt, 8, 320, 0, p16) == 0
    assert _linear(L, qt, 9, 640, 0, p16) == -4          # 9 * 640 is not a whole number of blocks
    assert _linear(L, qt, 8, 100, 0, p16) == -4          # K not a multiple of 8
    assert _linear(L, qt, 8, 512, 0, p16) == 0           # whole-block rows: unchanged


def test_32_element_formats_keep_whole_block_rows(pkg, p16):
    L = pkg.lib.lib()
    assert _linear(L, Q.Q8_0, 8, 40, 0, p16) == -4       # 8 * 40 = 10 blocks of 32, but rows must stay whole blocks
    assert _linear(L, Q.Q8_0, 8, 320, 0, p16) == 0


def test_row_indexing_routes_refuse_a_straddled_weight(pkg, p16):
    """GEMV, GEMV_FAST and FUSED_MMA index whole rows of blocks: E_UNSUPPORTED before any device work."""
    L, A = pkg.lib.lib(), pkg.lib
    for algo in (A.ALGO_GEMV, A.ALGO_GEMV_FAST, A.ALGO_FUSED_MMA):
        assert _linear(L, Q.Q4_K, 8, 640, 4, p16, algo) == -8, algo
        assert _linear(L, Q.Q6_K, 8, 640, 64, p16, algo) == -8, algo
    # the LoRA entry point still needs FUSED_TMEM
    x = p16
    assert L.ggufb200_linear_lora(int(Q.Q4_K), p16, None, 8, 640, x, 4, 640, 1, None, 0, x, 64, x, x, 8, None, 0, A.ALGO_GEMV, None) == -8


def test_workspace_follows_the_straddled_route(pkg):
    L, A = pkg.lib.lib(), pkg.lib
    wx = L.ggufb200_linear_workspace_ex
    N = K = 640
    q4k, q6k = int(Q.Q4_K), int(Q.Q6_K)
    auto = A.ALGO_AUTO | A.FLAG_EXACT_W
    for M in (16, 300, 4096, 8192):
        # AUTO: dequant + GEMM (measured faster than FUSED_TMEM on these weights, csrc/api.cu pick_route)
        assert wx(q4k, M, N, K, 1, 0, auto) == wx(q6k, M, N, K, 1, 0, auto) == wx(q4k, M, N, K, 1, 0, A.ALGO_AUTO) == N * K * 2
        # FUSED_TMEM when asked for: never split into K ranges -> no workspace
        assert wx(q4k, M, N, K, 1, 0, A.ALGO_FUSED_TMEM) == wx(q6k, M, N, K, 1, 0, A.ALGO_FUSED_TMEM) == 0
    assert wx(q4k, 4, N, K, 1, 0, auto) == N * K * 2                      # M <= 8: dequant + GEMM (the GEMVs index rows)
    assert wx(q4k, 300, N, K, 1, 2, auto) == N * K * 2                    # fp32 math: the reference's sequence
    assert wx(q4k, 300, N, K, 1, 0, A.ALGO_DEQUANT_MMA) == N * K * 2
    assert wx(q4k, 300, N, K, 1, 0, A.ALGO_FUSED_MMA) == 0
    # non-straddled shapes keep their answers (split-K at short M on a whole-block weight)
    assert wx(q4k, 64, 512, 4096, 1, 0, A.ALGO_AUTO) > 0


def test_straddled_plan_never_splits_k(pkg):
    L, A = pkg.lib.lib(), pkg.lib
    out = [ctypes.c_int() for _ in range(4)]
    refs = [ctypes.byref(o) for o in out]
    assert L.ggufb200_linear_plan(int(Q.Q4_K), 64, 640, 640, 1 << 30, A.ALGO_FUSED_TMEM, *refs) == 0
    assert out[1].value == 1
    assert L.ggufb200_linear_plan(int(Q.Q4_K), 64, 640, 768, 1 << 30, A.ALGO_FUSED_TMEM, *refs) == 0
    assert out[1].value > 1                                                # whole-block rows still split at short M


@pytest.mark.parametrize("N,K", [(640, 640), (5120, 640), (320, 320), (8, 320), (264, 640)])
def test_block_major_copy_geometry(pkg, N, K):
    L = pkg.lib.lib()
    for qt, pitch in PITCH.items():
        assert L.ggufb200_repack_bytes(int(qt), N, K) == N * K // 256 * pitch, qt
    for qt in (Q.Q4_K, Q.Q5_K):
        bs, ts = gguf.GGML_QUANT_SIZES[qt]
        assert L.ggufb200_repack_bytes(int(qt), N, K) == N * K // 256 * ts
    assert L.ggufb200_repack_bytes(int(Q.Q6_K), 9, 640) == 0               # not a whole number of blocks
    assert L.ggufb200_repack_bytes(int(Q.Q6_K), 256, 768) == 3 * 256 * 240  # whole-block rows: span-major, unchanged


def test_span_layout_need_matches_the_kernel(pkg):
    """The layer builds the copy exactly for the formats whose blocks are not 16-byte multiples."""
    for K in (320, 640):
        for qt in K_QUANTS:
            assert pkg.ops.needs_span_layout(qt, K) == (qt not in (Q.Q4_K, Q.Q5_K)), (qt, K)
            assert pkg.ops.straddled_rows(qt, K) and not pkg.ops.straddled_rows(qt, 512)
        assert not pkg.ops.straddled_rows(Q.Q8_0, K) and not pkg.ops.straddled_rows(Q.BF16, K)


def _golden(golden_dir, name, act):
    return np.load(os.path.join(golden_dir, f"linear_straddled_{name}_{act}.npz"))


def straddled_reference(packed, qt, N, K, x, bias, act_code):
    """The reference Linear on a straddled weight: the oracle's dequant of the flat block stream, reshaped to [N, K], cast to
    the activation dtype, then x @ W^T + bias in float64, rounded to the activation dtype."""
    w = bits_to_f32(oracle.dequant(packed, int(qt), oracle.DT_F16, oracle.DT_F16), 0).reshape(N, K)
    dt = torch.bfloat16 if act_code == 1 else torch.float16
    w = torch.from_numpy(w).to(dt).double()
    b = torch.from_numpy(np.asarray(bias, dtype=np.float32)).to(dt).double()
    y = torch.from_numpy(np.asarray(x, dtype=np.float32)).double() @ w.t() + b
    return y.to(dt).float().numpy()


@pytest.mark.parametrize("name", ["Q4_K", "Q6_K"])
@pytest.mark.parametrize("act,code", [("bf16", 1), ("f16", 0)])
def test_oracle_straddled_linear_matches_the_reference(pkg, golden_dir, name, act, code):
    g = _golden(golden_dir, name, act)
    qt = Q(int(g["qtype"]))
    N, K, M = int(g["N"]), int(g["K"]), int(g["M"])
    assert K % 256 != 0 and g["packed"].size == N * K // 256 * gguf.GGML_QUANT_SIZES[qt][1]
    x = bits_to_f32(g["x"], code).reshape(M, K)
    got = straddled_reference(g["packed"], qt, N, K, x, g["bias"], code)
    assert rel_fro(got, bits_to_f32(g["y"], code)) <= 1e-3
