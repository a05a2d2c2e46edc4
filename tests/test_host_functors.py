"""The product's DEVICE functors, executed on the CPU and compared bit for bit with the oracle.

comfyui-gguf_b200/csrc/{blocks.cuh,common.cuh} (per-format unpack, math policies, the 16-element producers of the Linear
kernels) are `__host__ __device__`; tests/host_functors.cu instantiates them for the host.  The same source lines the CUDA
kernels inline are therefore checked here, without a GPU, against oracle/gguf_oracle.c (itself pinned to the unmodified
reference, tests/test_oracle_vs_reference.py and tests/golden/).  Inputs include raw random bytes in every fp16 header
field (NaN / Inf / subnormal scales), which the GPU parity tests avoid."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle
from util import Q

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_functors.cu")
OUT = os.path.join(HERE, "_build", "libhostfunctors.so")
CSRC = os.path.join(os.path.dirname(HERE), "comfyui-gguf_b200", "csrc")
TYPES = [Q.Q4_0, Q.Q4_1, Q.Q5_0, Q.Q5_1, Q.Q8_0, Q.Q2_K, Q.Q3_K, Q.Q4_K, Q.Q5_K, Q.Q6_K, Q.IQ4_NL, Q.IQ4_XS]


@pytest.fixture(scope="module")
def hostf():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    deps = [SRC, os.path.join(CSRC, "blocks.cuh"), os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "produce.cuh")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-o", OUT, SRC], check=True)
    L = ctypes.CDLL(OUT)
    L.hostf_dequant.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    L.hostf_fast16.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int]
    L.hostf_produce.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    L.hostf_k_scale_min.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    L.hostf_iq4_lookup4.restype = ctypes.c_uint32
    L.hostf_iq4_lookup4.argtypes = [ctypes.c_uint32]
    L.hostf_prmt.restype = ctypes.c_uint32
    L.hostf_prmt.argtypes = [ctypes.c_uint32] * 3
    return L


def _aligned_copy(raw):
    """16-byte aligned, contiguous copy (the 16-element producers use 16-byte loads, like the kernels do)."""
    buf = np.empty(raw.size + 16, dtype=np.uint8)
    off = (-buf.ctypes.data) % 16
    view = buf[off:off + raw.size]
    view[:] = raw.reshape(-1)
    return view


def _bits(a):
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _same(a, b):
    """Bit equality, except that any NaN equals any NaN (payload / sign of a NaN is not part of the contract)."""
    a, b = np.asarray(a).reshape(-1), np.asarray(b).reshape(-1)
    if a.dtype == np.float32:
        nan_a, nan_b = np.isnan(a), np.isnan(b)
    else:
        return a, b, np.array_equal(a, b)
    ok = np.array_equal(nan_a, nan_b) and np.array_equal(_bits(a)[~nan_a], _bits(b)[~nan_b])
    return a, b, ok


def _nan16(bits, bf16):
    e, m = (0x7F80, 0x007F) if bf16 else (0x7C00, 0x03FF)
    return ((bits & e) == e) & ((bits & m) != 0)


def _equal_mod_nan(got, want, out_dtype):
    got, want = np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)
    if out_dtype == oracle.DT_F32:
        ng, nw = np.isnan(got), np.isnan(want)
        return np.array_equal(ng, nw) and np.array_equal(got.view(np.uint32)[~ng], want.view(np.uint32)[~nw])
    ng, nw = _nan16(got, out_dtype == oracle.DT_BF16), _nan16(want, out_dtype == oracle.DT_BF16)
    return np.array_equal(ng, nw) and np.array_equal(got[~ng], want[~nw])


@pytest.mark.parametrize("math", [oracle.DT_F16, oracle.DT_BF16, oracle.DT_F32], ids=["math-f16", "math-bf16", "math-f32"])
@pytest.mark.parametrize("out", [oracle.DT_F16, oracle.DT_BF16, oracle.DT_F32], ids=["out-f16", "out-bf16", "out-f32"])
@pytest.mark.parametrize("qt", TYPES, ids=lambda q: q.name)
def test_device_functors_equal_oracle(hostf, qt, out, math):
    n = 257
    raw = _aligned_copy(oracle.random_blocks(int(qt), n, seed=int(qt) * 7 + out * 3 + math, scale=0.02))
    bs, ts = oracle.type_info(int(qt))
    got = np.empty(n * bs, dtype=np.float32 if out == oracle.DT_F32 else np.uint16)
    assert hostf.hostf_dequant(int(qt), raw.ctypes.data, n, got.ctypes.data, out, math) == 0
    want = oracle.dequant(raw.reshape(n, ts), int(qt), out, math)
    assert _equal_mod_nan(got, want, out)


@pytest.mark.parametrize("qt", TYPES, ids=lambda q: q.name)
def test_device_functors_equal_oracle_on_raw_random_bytes(hostf, qt):
    """Header fields left as random bytes: Inf / NaN / subnormal / huge scales go through the same rounding sequence."""
    n = 4096
    bs, ts = oracle.type_info(int(qt))
    raw = _aligned_copy(np.random.default_rng(int(qt)).integers(0, 256, size=n * ts, dtype=np.uint8))
    for out, math in ((oracle.DT_F16, oracle.DT_F16), (oracle.DT_BF16, oracle.DT_F16), (oracle.DT_F32, oracle.DT_F32),
                      (oracle.DT_BF16, oracle.DT_BF16)):
        got = np.empty(n * bs, dtype=np.float32 if out == oracle.DT_F32 else np.uint16)
        assert hostf.hostf_dequant(int(qt), raw.ctypes.data, n, got.ctypes.data, out, math) == 0
        want = oracle.dequant(raw.reshape(n, ts), int(qt), out, math)
        assert _equal_mod_nan(got, want, out), (qt.name, out, math)


@pytest.mark.parametrize("act", [oracle.DT_F16, oracle.DT_BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("qt", [Q.Q4_K, Q.Q8_0], ids=lambda q: q.name)
@pytest.mark.parametrize("wild", [False, True], ids=["trained-like", "raw-bytes"])
def test_fast16_producers_equal_oracle(hostf, qt, act, wild):
    """The hand-scheduled producers of the tensor-core / GEMV Linear kernels: fp16 reference math, cast to the activation
    dtype -- must give exactly the W the reference hands to F.linear (dequant.py:15-28 with dequant_dtype=None)."""
    n = 2048
    bs, ts = oracle.type_info(int(qt))
    if wild:
        raw = np.random.default_rng(5).integers(0, 256, size=n * ts, dtype=np.uint8)
    else:
        raw = oracle.random_blocks(int(qt), n, seed=3, scale=0.02)
    raw = _aligned_copy(raw)
    got = np.empty(n * bs, dtype=np.uint16)
    assert hostf.hostf_fast16(int(qt), raw.ctypes.data, n, got.ctypes.data, act) == 0
    want = oracle.dequant(raw.reshape(n, ts), int(qt), act, oracle.DT_F16)
    assert _equal_mod_nan(got, want, act)


def test_fast16_reports_formats_without_a_producer(hostf):
    out = np.empty(256, dtype=np.uint16)
    raw = _aligned_copy(oracle.random_blocks(int(Q.Q6_K), 1, seed=0))
    assert hostf.hostf_fast16(int(Q.Q6_K), raw.ctypes.data, 1, out.ctypes.data, 0) == -8


def test_k_scale_min_and_value_table(hostf):
    """dequant.py:129-139 (6-bit scale / min packing) and dequant.py:241 (IQ4 value table), exhaustively / by formula."""
    rng = np.random.default_rng(0)
    for _ in range(200):
        s = rng.integers(0, 256, size=12, dtype=np.uint8)
        for j in range(8):
            sc, mn = ctypes.c_int(), ctypes.c_int()
            hostf.hostf_k_scale_min(s.ctypes.data, j, ctypes.byref(sc), ctypes.byref(mn))
            if j < 4:
                want = (s[j] & 63, s[j + 4] & 63)
            else:
                want = ((s[j + 4] & 0xF) | ((s[j - 4] >> 6) << 4), (s[j + 4] >> 4) | ((s[j] >> 6) << 4))
            assert (sc.value, mn.value) == (int(want[0]), int(want[1]))
    kvalues = [-127, -104, -83, -65, -49, -35, -22, -10, 1, 13, 25, 38, 53, 69, 89, 113]
    for a in range(16):
        for b in range(16):
            idx4 = a | (b << 8) | (((a + 5) & 15) << 16) | (((b + 9) & 15) << 24)
            r = hostf.hostf_iq4_lookup4(idx4)
            got = [((r >> (8 * i)) & 0xFF) - 127 for i in range(4)]
            assert got == [kvalues[a], kvalues[b], kvalues[(a + 5) & 15], kvalues[(b + 9) & 15]]
    # the host stand-in of prmt.b32 follows the PTX definition (byte select + sign replicate)
    assert hostf.hostf_prmt(0x33221100, 0x77665544, 0x7531) == 0x77553311
    assert hostf.hostf_prmt(0x80221100, 0x77665544, 0x000B) == 0x000000FF


def test_functors_never_read_past_the_last_block(tmp_path):
    """AddressSanitizer + UBSan over exact-size heap buffers (1, 3, 16 blocks of every format, every dtype pair, both
    16-element producers): a functor that over-reads its block would fault on the GPU at the end of an allocation."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    gxx = shutil.which("g++")
    if not os.path.exists(nvcc) or gxx is None:
        pytest.skip("toolchain not available")
    obj, exe = str(tmp_path / "hf.o"), str(tmp_path / "asan_run")
    san = "-fsanitize=address,-fsanitize=undefined,-fno-sanitize=alignment"   # 2-byte aligned blocks are read with 16-bit loads by design
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-g", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off," + san, "-c", SRC, "-o", obj], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("sanitizer build not available: " + r.stderr[-200:])
    cudart = os.path.join(os.path.dirname(os.path.dirname(nvcc)), "lib64")
    r = subprocess.run([gxx, "-fsanitize=address,undefined", "-g", os.path.join(HERE, "host_functors_asan_main.cpp"), obj,
                        "-L" + cudart, "-lcudart", "-Wl,-rpath," + cudart, "-o", exe], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("sanitizer link not available: " + r.stderr[-200:])
    run = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0 and "asan run ok" in run.stdout, run.stderr[-2000:]


# ---------------------------------------------------------------- produce.cuh: W producers of the fused kernels
EXACT_FAST = {Q.Q8_0, Q.Q4_0, Q.Q6_K}          # hand-written producers whose float step already has a single rounding
FMA_FAST = {Q.Q4_K, Q.Q5_K}                    # one fused multiply-add instead of multiply + subtract


def _spans(qt, n_spans, seed, wild=False, pitch=None):
    """n_spans spans of 256 elements; returns (aligned byte view with row pitch `pitch`, canonical [n_spans, span_bytes])."""
    bs, ts = oracle.type_info(int(qt))
    span = 256 // bs * ts
    if wild:
        raw = np.random.default_rng(seed).integers(0, 256, size=n_spans * span, dtype=np.uint8)
    else:
        raw = oracle.random_blocks(int(qt), n_spans * 256 // bs, seed=seed, scale=0.02).reshape(-1)
    raw = raw.reshape(n_spans, span)
    pitch = pitch or span
    padded = np.zeros((n_spans, pitch), dtype=np.uint8)
    padded[:, :span] = raw
    return _aligned_copy(padded), raw, pitch


@pytest.mark.parametrize("qt", TYPES, ids=lambda q: q.name)
@pytest.mark.parametrize("wild", [False, True], ids=["trained-like", "raw-bytes"])
def test_generic_producer_is_the_reference_fp16_weight(hostf, qt, wild):
    """Producer<Q> (every format): bit-identical to the reference's fp16 dequant (dequant.py, dequant_dtype=None)."""
    n = 600
    bs, ts = oracle.type_info(int(qt))
    span = 256 // bs * ts
    pitch = (span + 15) // 16 * 16                     # rows of the staged layout start on 16-byte boundaries
    buf, raw, pitch = _spans(qt, n, seed=int(qt) + 1, wild=wild, pitch=pitch)
    got = np.empty(n * 256, dtype=np.uint16)
    assert hostf.hostf_produce(int(qt), buf.ctypes.data, n, pitch, got.ctypes.data, 0) == 0
    want = oracle.dequant(raw.reshape(-1, ts), int(qt), oracle.DT_F16, oracle.DT_F16)
    assert _equal_mod_nan(got, want, oracle.DT_F16)


@pytest.mark.parametrize("qt", sorted(EXACT_FAST | FMA_FAST, key=int), ids=lambda q: q.name)
def test_fast_producers(hostf, qt):
    """FastProducer<Q>: the integer unpack is the reference's; formats whose float step is a single multiply stay
    bit-exact; Q4_K / Q5_K replace fp16(fp16(D*q) - M) by one fused multiply-add fp16(D*q - M): the correctly rounded
    value of the float step, which differs from the reference by at most the rounding of its intermediate product
    (half an ulp of D*q) plus the final roundings, and is at least as close to the exact value D*q - M."""
    n = 2000
    bs, ts = oracle.type_info(int(qt))
    span = 256 // bs * ts
    pitch = (span + 15) // 16 * 16
    buf, raw, pitch = _spans(qt, n, seed=int(qt) + 11, pitch=pitch)
    got = np.empty(n * 256, dtype=np.uint16)
    assert hostf.hostf_produce(int(qt), buf.ctypes.data, n, pitch, got.ctypes.data, 1) == 1
    want = oracle.dequant(raw.reshape(-1, ts), int(qt), oracle.DT_F16, oracle.DT_F16)
    if qt in EXACT_FAST:
        assert _equal_mod_nan(got, want, oracle.DT_F16)
        return
    g, w = got.view(np.float16).astype(np.float64), want.view(np.float16).astype(np.float64)
    # exact value of the float step with the reference's sub-block products D = fp16(d*sc), M = fp16(dmin*mn)
    q, sc, mn = oracle.unpack_int(raw.reshape(-1, ts), int(qt))
    blocks = raw.reshape(-1, ts)
    d = blocks[:, 0:2].copy().view(np.float16).astype(np.float32)
    dmin = blocks[:, 2:4].copy().view(np.float16).astype(np.float32)
    D = (d * sc.reshape(len(blocks), -1).astype(np.float32)).astype(np.float16).astype(np.float64)
    Mm = (dmin * mn.reshape(len(blocks), -1).astype(np.float32)).astype(np.float16).astype(np.float64)
    exact = (D * q.reshape(len(blocks), -1) - Mm).reshape(-1)
    assert np.array_equal(got.view(np.float16), exact.astype(np.float16))                 # = one correctly rounded FMA
    assert np.abs(g - exact).sum() <= np.abs(w - exact).sum()
    prod = np.abs(D * q.reshape(len(blocks), -1)).reshape(-1)
    bound = 0.5 * np.spacing(prod.astype(np.float16)).astype(np.float64) + np.spacing(np.maximum(np.abs(g), np.abs(w)).astype(np.float16)).astype(np.float64)
    assert np.all(np.abs(g - w) <= bound)


@pytest.mark.parametrize("qt", sorted(EXACT_FAST | FMA_FAST, key=int), ids=lambda q: q.name)
@pytest.mark.parametrize("wild", [False, True], ids=["trained-like", "raw-bytes"])
def test_hand_written_producers_with_the_reference_sequence_are_bit_exact(hostf, qt, wild):
    """FastProducer<Q, FMA = false> (GGUFB200_FLAG_EXACT_W on the FUSED_TMEM route): the weight is the reference's, bit for bit."""
    n = 1500
    bs, ts = oracle.type_info(int(qt))
    span = 256 // bs * ts
    buf, raw, pitch = _spans(qt, n, seed=int(qt) + 21, wild=wild, pitch=(span + 15) // 16 * 16)
    got = np.empty(n * 256, dtype=np.uint16)
    assert hostf.hostf_produce(int(qt), buf.ctypes.data, n, pitch, got.ctypes.data, 2) == 1
    want = oracle.dequant(raw.reshape(-1, ts), int(qt), oracle.DT_F16, oracle.DT_F16)
    assert _equal_mod_nan(got, want, oracle.DT_F16)


def test_fast_request_falls_back_to_generic_for_other_formats(hostf):
    buf, raw, pitch = _spans(Q.Q3_K, 8, seed=1, pitch=112)
    got = np.empty(8 * 256, dtype=np.uint16)
    assert hostf.hostf_produce(int(Q.Q3_K), buf.ctypes.data, 8, pitch, got.ctypes.data, 1) == 0
    want = oracle.dequant(raw.reshape(-1, 110), int(Q.Q3_K), oracle.DT_F16, oracle.DT_F16)
    assert _equal_mod_nan(got, want, oracle.DT_F16)
