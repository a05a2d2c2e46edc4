"""CPU tests: the C-ABI library loads, exports every symbol include/ggufb200.h declares, and validates arguments
before touching the GPU (so these checks run without a device)."""
import ctypes
import os
import re

import gguf
import pytest

from util import ALL_QTYPES, Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_all_exported(pkg):
    header = open(os.path.join(ROOT, "include", "ggufb200.h")).read()
    declared = set(re.findall(r"\b(ggufb200_[a-z_0-9]+)\s*\(", header))
    assert len(declared) >= 10
    L = pkg.lib.lib()
    for sym in sorted(declared):
        assert hasattr(L, sym), f"{sym} declared in include/ggufb200.h but not exported"
    assert declared == set(pkg.lib.EXPORTS)


def test_version_and_strerror(pkg):
    L = pkg.lib.lib()
    assert L.ggufb200_version() == 200
    assert L.ggufb200_strerror(0) == b"ok"
    for rc in range(-9, 0):
        assert len(L.ggufb200_strerror(rc)) > 3


@pytest.mark.parametrize("qt", ALL_QTYPES, ids=lambda q: q.name)
def test_type_info_matches_gguf_py(pkg, qt):
    bs, ts = ctypes.c_int(), ctypes.c_int()
    assert pkg.lib.lib().ggufb200_type_info(int(qt), ctypes.byref(bs), ctypes.byref(ts)) == 0
    assert (bs.value, ts.value) == gguf.GGML_QUANT_SIZES[qt]
    assert pkg.lib.lib().ggufb200_supported(int(qt), pkg.lib.OP_DEQUANT) == 1


def test_supported_set_equals_reference_table(pkg):
    """dequant.py:287-301 lists exactly these 13 types; anything else must be rejected (no numpy fallback)."""
    L = pkg.lib.lib()
    supported = {int(q) for q in Q if L.ggufb200_supported(int(q), 0)}
    assert supported == {int(q) for q in ALL_QTYPES}
    assert set(pkg.dequant.dequantize_functions.keys()) == set(ALL_QTYPES)


def test_argument_validation_without_gpu(pkg):
    L = pkg.lib.lib()
    buf = (ctypes.c_uint8 * 4096)()
    p = ctypes.addressof(buf)
    p16 = (p + 15) & ~15
    assert L.ggufb200_dequant(999, p16, 1, p16, 0, 0, None) == -1          # E_TYPE
    assert L.ggufb200_dequant(int(Q.Q4_K), p16, 1, p16, 7, 0, None) == -2  # E_DTYPE
    assert L.ggufb200_dequant(int(Q.Q4_K), p16, -1, p16, 0, 0, None) == -4  # E_SHAPE
    assert L.ggufb200_dequant(int(Q.Q4_K), p16, 0, None, 0, 0, None) == 0   # empty input is fine
    assert L.ggufb200_dequant(int(Q.Q4_K), None, 1, p16, 0, 0, None) == -5  # E_NULL
    assert L.ggufb200_dequant(int(Q.Q4_K), p16, 1, p16 + 2, 0, 0, None) == -3  # E_ALIGN
    # linear: K must be a multiple of the block size, act dtype must be 16-bit
    assert L.ggufb200_linear(int(Q.Q4_K), p16, 8, 100, p16, 1, 100, 1, 0, None, 0, p16, 8, None, 0, 0, None) == -4
    assert L.ggufb200_linear(int(Q.Q4_K), p16, 8, 256, p16, 1, 256, 2, 0, None, 0, p16, 8, None, 0, 0, None) == -2
    assert L.ggufb200_linear(int(Q.Q4_K), p16, 8, 256, p16, 0, 256, 1, 0, None, 0, p16, 8, None, 0, 0, None) == 0
    assert L.ggufb200_linear_workspace(int(Q.Q4_K), 64, 128, 256, 1, pkg.lib.ALGO_DEQUANT_MMA) == 128 * 256 * 2
    assert L.ggufb200_linear_workspace(int(Q.Q4_K), 1, 128, 256, 1, pkg.lib.ALGO_GEMV) == 0


def test_missing_library_fails_loudly(pkg, monkeypatch):
    monkeypatch.setattr(pkg.lib, "_lib", None)
    monkeypatch.setattr(pkg.lib, "LIB_PATH", "/nonexistent/libggufb200.so")
    with pytest.raises(pkg.lib.GGUFB200Error):
        pkg.lib.lib()


def test_tuning_is_refused_and_gemm_validation_without_gpu(pkg):
    L = pkg.lib.lib()
    # route selection is per call (algo | flags); the process-wide knobs are gone, the two launch knobs of the dequant kernel
    # are benchmark-only and need GGUFB200_ALLOW_TUNING=1 in the environment (not set in the test process)
    for key in (0, 1, 2, 3, 4, 5, 6, 99):
        assert L.ggufb200_set_tuning(key, 1) == -8
    buf = (ctypes.c_uint8 * 4096)()
    p16 = (ctypes.addressof(buf) + 15) & ~15
    # ggufb200_gemm: dtype must be 16-bit, leading dimensions >= K and multiples of 8, pointers aligned
    assert L.ggufb200_gemm(p16, 8, 64, 64, p16, 4, 64, 2, None, 0, p16, 8, None) == -2
    assert L.ggufb200_gemm(p16, 8, 64, 32, p16, 4, 64, 1, None, 0, p16, 8, None) == -4
    assert L.ggufb200_gemm(p16 + 2, 8, 64, 64, p16, 4, 64, 1, None, 0, p16, 8, None) == -3
    assert L.ggufb200_gemm(p16, 8, 64, 64, p16, 0, 64, 1, None, 0, p16, 8, None) == 0   # M == 0 is a no-op
    # ggufb200_linear: an unaligned packed weight needs the dequant+GEMM workspace
    assert L.ggufb200_linear(int(Q.Q4_K), p16 + 2, 8, 256, p16, 4, 256, 1, 0, None, 0, p16, 8, None, 0, 0, None) == -3


def test_workspace_contract_follows_the_route(pkg):
    """Workspace query == what the call with the same (algo | flags, math dtype) will use; no GPU needed."""
    L = pkg.lib.lib()
    A = pkg.lib
    q4k = int(Q.Q4_K)
    ws = L.ggufb200_linear_workspace
    assert ws(q4k, 4608, 3072, 3072, 1, A.ALGO_DEQUANT_MMA) == 3072 * 3072 * 2
    assert ws(q4k, 4608, 3072, 3072, 1, A.ALGO_FUSED_MMA) == 0                        # enough tiles: unsplit
    assert ws(q4k, 64, 512, 4096, 1, A.ALGO_FUSED_MMA) == 16 * 64 * 512 * 4           # split-K: 16 slices
    assert ws(q4k, 64, 512, 4096, 1, A.ALGO_FUSED_MMA | A.FLAG_NOSPLIT) == 0
    assert ws(q4k, 512, 3072, 12288, 1, A.ALGO_FUSED_MMA) == 2 * 512 * 3072 * 4       # 48 tiles of 128x256 -> 2 ranges
    # AUTO: the FUSED_TMEM kernel for every M > 8 (K ranges only when that beats idle
    # SMs by the cost model); EXACT_W only changes its producers, never the route or the workspace
    for flags in (0, A.FLAG_EXACT_W):
        auto = A.ALGO_AUTO | flags
        assert ws(q4k, 4608, 3072, 3072, 1, auto) == 0
        assert ws(q4k, 4, 3072, 3072, 1, auto) == 0                                   # small weight at M <= 8: mma.sync GEMV
        assert ws(q4k, 4, 18432, 3072, 1, auto) == 0                                  # large weight at M <= 8: a GEMV as well
        assert ws(q4k, 64, 512, 4096, 1, auto) == ws(q4k, 64, 512, 4096, 1, A.ALGO_FUSED_TMEM) > 0
        assert ws(q4k, 64, 512, 4096, 1, auto) % (64 * 512 * 4) == 0
        assert ws(q4k, 64, 512, 4096, 1, auto | A.FLAG_NOSPLIT) == 0
    # a non-fp16 math dtype always means the reference's own sequence in that dtype: dequant + GEMM above the GEMV range
    wx = L.ggufb200_linear_workspace_ex
    assert wx(q4k, 4608, 3072, 3072, 1, 1, A.ALGO_AUTO) == 3072 * 3072 * 2
    assert wx(q4k, 64, 512, 4096, 1, 2, A.ALGO_AUTO) == 512 * 4096 * 2
    assert wx(q4k, 4, 3072, 3072, 1, 2, A.ALGO_AUTO) == 0
    assert wx(q4k, 64, 512, 4096, 1, 0, A.ALGO_AUTO) == ws(q4k, 64, 512, 4096, 1, A.ALGO_AUTO)
    # formats / shapes the FUSED_TMEM route cannot read from the canonical rows (no span-major copy at hand) fall back to round 1's routes
    assert ws(int(Q.Q6_K), 4608, 3072, 3072, 1, A.ALGO_AUTO) == 3072 * 3072 * 2       # 210-byte blocks
    assert ws(int(Q.Q8_0), 4608, 7296, 2432, 1, A.ALGO_AUTO) == 7296 * 2432 * 2       # 2584-byte rows
    # row gather: K must be a multiple of the block size
    buf = (ctypes.c_uint8 * 4096)()
    p16 = (ctypes.addressof(buf) + 15) & ~15
    assert L.ggufb200_dequant_rows(int(Q.Q4_K), p16, 4, 100, p16, 1, p16, 0, 0, None) == -4


def test_span_layout_geometry_without_gpu(pkg):
    """ggufb200_repack_bytes = spans * rows padded to 256 * pitch; pitch = span bytes, padded to an odd multiple of 16 when the
    span is not a multiple of 16 bytes (csrc/produce.cuh SpanOf::PITCH)."""
    L = pkg.lib.lib()
    want_pitch = {Q.Q4_0: 144, Q.Q4_1: 160, Q.Q5_0: 176, Q.Q5_1: 192, Q.Q8_0: 272, Q.Q2_K: 112, Q.Q3_K: 112, Q.Q4_K: 144, Q.Q5_K: 176,
                  Q.Q6_K: 240, Q.IQ4_NL: 144, Q.IQ4_XS: 144}
    for qt, pitch in want_pitch.items():
        bs, ts = gguf.GGML_QUANT_SIZES[qt]
        span = 256 // bs * ts
        assert pitch % 16 == 0 and pitch >= span and (pitch == span or (pitch // 16) % 2 == 1)
        assert L.ggufb200_repack_bytes(int(qt), 300, 768) == 3 * 512 * pitch
        assert L.ggufb200_repack_bytes(int(qt), 256, 256) == 256 * pitch
    assert L.ggufb200_repack_bytes(int(Q.Q8_0), 7296, 2432) == 10 * 7424 * 272      # SD3.5 shape: ragged last span
    assert L.ggufb200_repack_bytes(int(Q.BF16), 8, 8) == 0 and L.ggufb200_repack_bytes(999, 8, 256) == 0
    assert L.ggufb200_repack_bytes(int(Q.Q4_K), 8, 100) == 0                          # K not a multiple of the block size
    buf = (ctypes.c_uint8 * 4096)()
    p16 = (ctypes.addressof(buf) + 15) & ~15
    assert L.ggufb200_repack(int(Q.BF16), p16, 8, 8, p16, None) == -1
    assert L.ggufb200_repack(int(Q.Q4_K), None, 8, 256, p16, None) == -5
    assert L.ggufb200_repack(int(Q.Q4_K), p16, 8, 256, p16 + 4, None) == -3
    # the LoRA entry point validates like ggufb200_linear and needs the FUSED_TMEM route
    x = p16
    assert L.ggufb200_linear_lora(int(Q.Q4_K), p16, None, 8, 256, x, 4, 256, 1, None, 0, x, 64, x, x, 8, None, 0,
                                  pkg.lib.ALGO_GEMV, None) == -8
    assert L.ggufb200_linear_lora(int(Q.Q4_K), p16, None, 8, 256, x, 4, 256, 1, None, 0, None, 64, x, x, 8, None, 0,
                                  pkg.lib.ALGO_FUSED_TMEM, None) == -5
    assert L.ggufb200_linear_lora(int(Q.Q4_K), p16, None, 8, 256, x, 4, 256, 1, None, 0, x, 48, x, x, 8, None, 0,
                                  pkg.lib.ALGO_FUSED_TMEM, None) == -3


def test_python_constants_match_the_header(pkg):
    """`_lib.py` mirrors the #define values of include/ggufb200.h by hand: every GGUFB200_ALGO_* / FLAG_* / dtype / op code and
    the stable-source bits must agree (a drifted flag would silently select another route or drop a promise)."""
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ggufb200.h")).read()
    defines = {m.group(1): int(m.group(2), 0) for m in re.finditer(r"^#define\s+GGUFB200_(\w+)\s+\(?(-?(?:0x[0-9A-Fa-f]+|\d+))\)?", hdr, re.M)}
    A = pkg.lib
    pairs = {"ALGO_AUTO": A.ALGO_AUTO, "ALGO_GEMV": A.ALGO_GEMV, "ALGO_FUSED_MMA": A.ALGO_FUSED_MMA, "ALGO_DEQUANT_MMA": A.ALGO_DEQUANT_MMA,
             "ALGO_FUSED_TMEM": A.ALGO_FUSED_TMEM, "ALGO_GEMV_FAST": A.ALGO_GEMV_FAST, "ALGO_MASK": A.ALGO_MASK,
             "FLAG_EXACT_W": A.FLAG_EXACT_W, "FLAG_GENERIC": A.FLAG_GENERIC, "FLAG_TILE384": A.FLAG_TILE384, "FLAG_NOSPLIT": A.FLAG_NOSPLIT,
             "FLAG_UNSTAGED": A.FLAG_UNSTAGED, "FLAG_TILE192": A.FLAG_TILE192, "FLAG_W_STABLE": A.FLAG_W_STABLE,
             "DEQUANT_SRC_STABLE": A.DEQUANT_SRC_STABLE, "F16": A.F16, "BF16": A.BF16, "F32": A.F32,
             "OP_DEQUANT": A.OP_DEQUANT, "OP_LINEAR": A.OP_LINEAR, "OP_ROWS": A.OP_ROWS, "OP_LINEAR_MMA": A.OP_LINEAR_MMA}
    for name, value in pairs.items():
        assert defines.get(name) == value, (name, defines.get(name), value)
    flags = [v for k, v in defines.items() if k.startswith("FLAG_")]
    assert len(set(flags)) == len(flags) and all(f & A.ALGO_MASK == 0 and f & (f - 1) == 0 for f in flags), "flag bits must be distinct single bits above the algo mask"
    assert defines["DEQUANT_SRC_STABLE"] > 2, "the stable-source bit must not collide with a dtype code"
