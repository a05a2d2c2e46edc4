"""CPU tests of the numpy-fallback types (IQ2_XXS ... NVFP4): the decoders of csrc/fallback.cuh against gguf-py bit for bit,
the generated tables, the golden files and the C ABI's argument checks.  No GPU needed.

The decoders are `__host__ __device__`; tests/host_fallback.cu builds the very lines the K1 kernel inlines for the host
(-ffp-contract=off, so no multiply-add is fused, as on the device) and this file compares their output with the reference's
`torch.from_numpy(gguf.quants.dequantize(bytes, qtype)).to(dtype)` (reference dequant.py:24-28)."""
import ctypes
import os
import shutil
import subprocess
import sys

import gguf
import numpy as np
import pytest
import torch

from fallback_cases import FALLBACK, gguf_values, random_blocks, reference_tensor
from util import ALL_QTYPES, Q, canon_nan, torch_bits

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "host_fallback.cu")
OUT = os.path.join(HERE, "_build", "libhostfallback.so")
CSRC = os.path.join(ROOT, "comfyui-gguf_b200", "csrc")
DTYPES = {"f16": 0, "bf16": 1, "f32": 2}
NP_OUT = {0: np.uint16, 1: np.uint16, 2: np.uint32}


@pytest.fixture(scope="module")
def hostfb():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    deps = [SRC] + [os.path.join(CSRC, f) for f in ("fallback.cuh", "fallback_tables.h", "blocks.cuh", "common.cuh")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-o", OUT, SRC], check=True)
    L = ctypes.CDLL(OUT)
    L.hostfb_dequant.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int]
    L.hostfb_geometry.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    return L


def _host_bits(L, blocks, qt, out_code):
    bs, _ts = gguf.GGML_QUANT_SIZES[qt]
    blocks = np.ascontiguousarray(blocks)
    out = np.empty(blocks.shape[0] * bs, dtype=NP_OUT[out_code])
    assert L.hostfb_dequant(int(qt), blocks.ctypes.data, blocks.shape[0], out.ctypes.data, out_code) == 0
    return out


@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_geometry_matches_gguf_py(hostfb, qt):
    bs, ts = ctypes.c_int(), ctypes.c_int()
    assert hostfb.hostfb_geometry(int(qt), ctypes.byref(bs), ctypes.byref(ts)) == 0
    assert (bs.value, ts.value) == gguf.GGML_QUANT_SIZES[qt]


@pytest.mark.parametrize("out", list(DTYPES), ids=str)
@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_decoders_bit_exact_vs_gguf_py(hostfb, qt, out):
    """Raw random blocks (every scale field random: NaN, Inf and subnormal scales occur), plus the edge-case scales of
    fallback_cases (MXFP4 exponents 0, 1, 254, 255; ue4m3 0x00, 0x7F, 0xFF and subnormals; f16 Inf / NaN / subnormals)."""
    code = DTYPES[out]
    bs = gguf.GGML_QUANT_SIZES[qt][0]
    blocks = random_blocks(qt, 4096 // bs * 4, seed=11, specials=True)
    with np.errstate(all="ignore"):
        want = torch_bits(reference_tensor(blocks, qt, code))
    got = _host_bits(hostfb, blocks, qt, code)
    assert np.array_equal(canon_nan(got, code), canon_nan(want, code))


@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_golden_pins_gguf_py(golden_dir, hostfb, qt):
    """The committed golden file still matches the installed gguf-py, and the host decoders reproduce it."""
    g = np.load(os.path.join(golden_dir, f"fallback_{qt.name}.npz"))
    with np.errstate(all="ignore"):
        now = gguf_values(g["blocks"], qt)
    assert np.array_equal(canon_nan(now.view(np.uint32), 2), canon_nan(g["f32"].view(np.uint32), 2))
    assert np.array_equal(canon_nan(_host_bits(hostfb, g["blocks"], qt, 2), 2), canon_nan(g["f32"].view(np.uint32), 2))


def test_tables_regenerate_to_committed_header():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import gen_fallback_tables
    finally:
        sys.path.pop(0)
    with open(gen_fallback_tables.OUT) as f:
        assert f.read() == gen_fallback_tables.render()


def test_supported_fallback_set(pkg):
    L = pkg.lib.lib()
    served = {int(q) for q in Q if L.ggufb200_supported(int(q), pkg.lib.OP_DEQUANT_FALLBACK)}
    assert served == {int(q) for q in pkg.dequant.FALLBACK_QTYPES} == {int(q) for q in FALLBACK}
    for codes in (999, -1, 1000):
        assert L.ggufb200_supported(codes, pkg.lib.OP_DEQUANT_FALLBACK) == 0
    for q in FALLBACK:      # the reference's table stays the table of every other entry point
        for op in (pkg.lib.OP_DEQUANT, pkg.lib.OP_LINEAR, pkg.lib.OP_ROWS, pkg.lib.OP_LINEAR_MMA):
            assert L.ggufb200_supported(int(q), op) == 0
        assert L.ggufb200_type_info(int(q), None, None) == -1
        assert q not in pkg.dequant.dequantize_functions


def test_every_gguf_py_type_is_served(pkg):
    """Every type gguf-py can dequantise, apart from F32 and F16, is in the reference's table or in FALLBACK_QTYPES."""
    for q in Q:
        if q in (Q.F32, Q.F16):
            continue
        try:
            bs, ts = gguf.GGML_QUANT_SIZES[q]
            gguf.quants.dequantize(np.zeros(ts, dtype=np.uint8), q)
        except (NotImplementedError, KeyError, ValueError):
            continue
        assert q in ALL_QTYPES or q in pkg.dequant.FALLBACK_QTYPES, q.name


def test_dequant_fallback_argument_validation_without_gpu(pkg):
    L = pkg.lib.lib()
    buf = (ctypes.c_uint8 * 4096)()
    p16 = (ctypes.addressof(buf) + 15) & ~15
    iq = int(Q.IQ2_XXS)
    assert L.ggufb200_dequant_fallback(int(Q.Q4_K), p16, 1, p16, 0, 0, None) == -1      # E_TYPE: a table type
    assert L.ggufb200_dequant_fallback(999, p16, 1, p16, 0, 0, None) == -1              # E_TYPE
    assert L.ggufb200_dequant_fallback(iq, p16, 1, p16, 3, 0, None) == -2               # E_DTYPE
    assert L.ggufb200_dequant_fallback(iq, p16, 1, p16, -1, 0, None) == -2
    assert L.ggufb200_dequant_fallback(iq, p16, -1, p16, 0, 0, None) == -4              # E_SHAPE
    assert L.ggufb200_dequant_fallback(iq, None, 1, p16, 0, 0, None) == -5              # E_NULL
    assert L.ggufb200_dequant_fallback(iq, p16, 1, None, 0, 0, None) == -5
    assert L.ggufb200_dequant_fallback(iq, p16, 1, p16 + 2, 0, 0, None) == -3           # E_ALIGN (out)
    assert L.ggufb200_dequant_fallback(iq, p16, 1, p16, 0, 0x1, None) == -8             # E_UNSUPPORTED: unknown flag bit
    assert L.ggufb200_dequant_fallback(iq, p16, 0, p16, 0, pkg.lib.DEQUANT_SRC_STABLE, None) == 0   # nothing to do
    # the table entry points keep refusing the fallback types
    assert L.ggufb200_dequant(iq, p16, 1, p16, 0, 0, None) == -1


@pytest.mark.parametrize("qt", FALLBACK, ids=lambda q: q.name)
def test_no_cpu_fallback_for_fallback_types(pkg, qt):
    """Without a CUDA device these types raise NotImplementedError, before any size check (the numpy path is not provided)."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    t = pkg.ops.GGMLTensor(torch.zeros(7, dtype=torch.uint8), tensor_type=qt, tensor_shape=torch.Size((7,)))
    with pytest.raises(NotImplementedError):
        pkg.dequant.dequantize_tensor(t, torch.float16)
    with pytest.raises(NotImplementedError):
        pkg.dequant.dequantize_tensor(t)
