"""Inputs and references shared by the K-quant encoder tests (tests/test_quantize_k.py, tests/test_gpu_quantize_k.py):
  * the plain-C restatement of llama.cpp's K-quant reference quantisers (tests/kquant_oracle.c, built here with gcc and
    -ffp-contract=off) and the product's encoder pieces compiled for the host (tests/host_quantize_k.cu);
  * seeded and adversarial 256-value super-blocks;
  * the layout check: decoded with the existing dequant oracle, every element inside its group's code range lies within half
    a step of its value, whatever the search chose."""
import ctypes
import os
import shutil
import subprocess

import gguf
import numpy as np

Q = gguf.GGMLQuantizationType
K_TYPES = [Q.Q2_K, Q.Q3_K, Q.Q4_K, Q.Q5_K, Q.Q6_K]
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BUILD = os.path.join(HERE, "_build")
CSRC = os.path.join(ROOT, "comfyui-gguf_b200", "csrc")

# (code range of the nearest-code pass, signed): Q2_K / Q4_K / Q5_K codes are l in [0, nmax] with value d*sc*l - dmin*m;
# Q3_K / Q6_K codes are q in [-nmax, nmax - 1] with value d*sc*q
CODE_RANGE = {Q.Q2_K: (3, False), Q.Q3_K: (4, True), Q.Q4_K: (15, False), Q.Q5_K: (31, False), Q.Q6_K: (32, True)}
D_OFFSETS = {Q.Q2_K: (80, 82), Q.Q3_K: (108, None), Q.Q4_K: (0, 2), Q.Q5_K: (0, 2), Q.Q6_K: (208, None)}


def _stale(out, deps):
    return not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps)


def _build(cmd, out):
    os.makedirs(BUILD, exist_ok=True)
    tmp = out + f".{os.getpid()}.tmp"
    subprocess.run(cmd + ["-o", tmp], check=True)
    os.replace(tmp, out)


def oracle_lib():
    """The C restatement, compiled with gcc -O2 -ffp-contract=off -fno-fast-math (None when gcc is missing)."""
    src = os.path.join(HERE, "kquant_oracle.c")
    out = os.path.join(BUILD, "libkquant_oracle.so")
    if _stale(out, [src]):
        cc = shutil.which("gcc") or "/usr/bin/gcc"
        if not os.path.exists(cc):
            return None
        _build([cc, "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-Wall", src, "-lm"], out)
    L = ctypes.CDLL(out)
    L.kqor_quantize.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    L.kqor_counter.argtypes = [ctypes.c_int]
    L.kqor_counter.restype = ctypes.c_longlong
    return L


def host_lib():
    """The product's K-quant pieces compiled for the host by nvcc (None when nvcc is missing)."""
    src = os.path.join(HERE, "host_quantize_k.cu")
    out = os.path.join(BUILD, "libhostquantize_k.so")
    deps = [src] + [os.path.join(CSRC, f) for f in ("quantize.cuh", "blocks.cuh", "common.cuh")]
    if _stale(out, deps):
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        if not os.path.exists(nvcc):
            return None
        _build([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--expt-relaxed-constexpr",
                "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", src], out)
    L = ctypes.CDLL(out)
    L.hostk_quantize.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    return L


def encode(L, x, qtype, fn="kqor_quantize"):
    """Bytes of fp32 values x [..., 256 k] through `fn` of library L, as a flat uint8 array."""
    x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1)
    assert x.size % 256 == 0
    n = x.size // 256
    out = np.zeros(n * gguf.GGML_QUANT_SIZES[qtype][1], dtype=np.uint8)
    assert getattr(L, fn)(int(qtype), x.ctypes.data, n, out.ctypes.data) == 0
    return out


def seeded_blocks(n, seed, heavy=False):
    """n super-blocks [n, 256] fp32 at scales from 1e-3 to 1e2; heavy: Student-t (3 degrees of freedom) values."""
    rng = np.random.default_rng(seed)
    x = rng.standard_t(3, (n, 256)) if heavy else rng.standard_normal((n, 256))
    x = x.astype(np.float32) * np.float32(10.0) ** rng.integers(-3, 3, size=(n, 1)).astype(np.float32)
    return x.astype(np.float32)


def adversarial_blocks():
    """[n, 256] fp32 super-blocks, every value finite and inside the bf16 range."""
    r = np.random.default_rng(23)
    rows = []
    g = lambda s=1.0: (r.standard_normal(256) * s).astype(np.float32)
    rows += [np.zeros(256, np.float32), np.full(256, -0.0, np.float32)]
    for v in (1.0, -3.3, 7e-3, 1e-6, 65504.0):                     # constant blocks
        rows.append(np.full(256, v, np.float32))
    for pos in (0, 17, 130, 255):                                   # one outlier; one nonzero
        b = g(0.01)
        b[pos] = 5.0 if pos % 2 else -5.0
        rows.append(b)
        z = np.zeros(256, np.float32)
        z[pos] = 0.3
        rows.append(z)
    rows += [-np.abs(g()), np.abs(g()), np.abs(g()) + 1.0, -np.abs(g()) - 1.0]   # one-signed blocks (min > 0 clamps to 0)
    b = np.repeat(r.standard_normal(16).astype(np.float32), 16)      # every 16-group constant: max == min
    rows += [b, np.repeat(r.standard_normal(8).astype(np.float32), 32), np.abs(b)]
    for s in (1e-39, 1e-41, 1.4e-45, 2.0 ** -126, 1e-20, 1e-15):   # subnormal and tiny values, below / at GROUP_MAX_EPS
        rows.append(g(s))
        rows.append(np.full(256, s, np.float32))
    for s in (1e5, 3e6, 1e9):                                       # bf16 values beyond the fp16 range
        rows.append(g(s))
    h = g(0.05)
    h[::16] = 0.0
    h[:128] = 0.0                                                   # half the groups zero, half not
    rows.append(h)
    sparse = np.where(r.random(256) < 0.1, g(), 0.0).astype(np.float32)   # mostly zero: groups with one or two nonzero values
    rows.append(sparse)
    rows.append(np.abs(sparse))
    rows += [np.linspace(-1, 1, 256, dtype=np.float32), np.linspace(0, 1, 256, dtype=np.float32),
             np.tile(np.arange(16, dtype=np.float32) - 8, 16), np.tile(np.arange(32, dtype=np.float32), 8) * np.float32(0.5)]
    for k in range(4):                                              # two-level groups: exact grids the fits can hit
        rows.append(np.where(r.random(256) < 0.5, np.float32(0.25 * (k + 1)), np.float32(-0.5)).astype(np.float32))
    mixed = g()
    mixed *= np.float32(10.0) ** r.integers(-8, 3, 256).astype(np.float32)   # magnitudes over ten decades in one block
    rows.append(mixed)
    return np.stack(rows).astype(np.float32)


def to_dtype_values(x, dtype_name):
    """x rounded to fp16 / bf16 (round to nearest even) and widened back to fp32, as the GPU kernels widen their source."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
    if dtype_name == "f16":
        t = t.half()
    elif dtype_name == "bf16":
        t = t.bfloat16()
    return t.float().numpy()


def layout_violations(packed, x, qtype):
    """Elements of fp32 x [n, 256] whose decoded value (the dequant oracle on `packed`, fp32 math) is more than half a step
    (|d*sc| / 2, plus a few ulps) from x although x lies inside its group's code range.  Groups whose decoded scale is 0 are
    not checked.  Returns (indices of violations, number of elements checked)."""
    import oracle
    x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, 256).astype(np.float64)
    n = x.shape[0]
    ts = gguf.GGML_QUANT_SIZES[qtype][1]
    blk = np.ascontiguousarray(packed, dtype=np.uint8).reshape(n, ts)
    y = oracle.dequant(packed, int(qtype), oracle.DT_F32, oracle.DT_F32).reshape(n, 256).astype(np.float64)
    _, sc, mn = oracle.unpack_int(packed, int(qtype))
    sc, mn = sc.reshape(n, 256).astype(np.float64), mn.reshape(n, 256).astype(np.float64)
    o_d, o_m = D_OFFSETS[qtype]
    half = lambda off: blk[:, off:off + 2].copy().view(np.float16)[:, 0].astype(np.float64)[:, None]
    step = half(o_d) * sc
    dm = half(o_m) * mn if o_m is not None else np.zeros_like(step)
    nmax, signed = CODE_RANGE[qtype]
    with np.errstate(all="ignore"):
        t = (x + dm) / step
        inside = (t >= -nmax) & (t <= nmax - 1) if signed else (t >= 0) & (t <= nmax)
        inside &= (step != 0) & np.isfinite(step) & np.isfinite(dm)
        tol = 0.5 * np.abs(step) * (1 + 2.0 ** -18) + 2.0 ** -22 * (np.abs(x) + np.abs(dm) + np.abs(step) * nmax) + 1e-44
        bad = inside & ~(np.abs(y - x) <= tol)
    return np.flatnonzero(bad), int(inside.sum())


def rmse(packed, x, qtype):
    import oracle
    y = oracle.dequant(packed, int(qtype), oracle.DT_F32, oracle.DT_F32).astype(np.float64)
    return float(np.sqrt(np.mean((y - np.asarray(x, np.float64).reshape(-1)) ** 2)))
