#!/usr/bin/env python
"""Generate the committed golden vectors from the UNMODIFIED reference.

Run in the build container only (needs /root/reference, which does not exist on
the GPU box):   python tests/golden/make_golden.py

What is produced (all under tests/golden/):
  dequant_<QTYPE>.npz   seeded packed blocks + the reference's own outputs of
                        `dequant.py::dequantize(...).to(out)` for five
                        (math dtype, out dtype) combinations, as raw bit patterns
  linear_<QTYPE>_<act>.npz   x / packed W / F32 bias and the output of the
                        reference `ops.py::GGMLOps.Linear.forward` (run on CPU
                        through tests/fake_comfy)
  reference_surface.json   public function / class names of the reference's
                        dequant.py and ops.py
  torch_chain.json      the reference's `dequantize(raw, qtype, shape, dtype)` on
                        96 seeded blocks per (qtype, math dtype): dtype, SHA-256 of
                        the result's bytes, and the number of materialising ATen
                        kernels it ran

The reference is imported by path and never copied: dequant.py via importlib,
ops.py through a throw-away package directory of symlinks in $TMPDIR.
"""
import importlib
import importlib.util
import os
import sys
import tempfile

import numpy as np
import torch
import gguf

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "fake_comfy"))

import oracle  # noqa: E402  (only for the seeded block generator)

T = gguf.GGMLQuantizationType
QTYPES = [T.Q4_0, T.Q4_1, T.Q5_0, T.Q5_1, T.Q8_0, T.Q2_K, T.Q3_K, T.Q4_K, T.Q5_K, T.Q6_K, T.IQ4_NL, T.IQ4_XS, T.BF16]
TORCH_DT = {0: torch.float16, 1: torch.bfloat16, 2: torch.float32}
# (math dtype, out dtype): default fp16 math -> fp16 / bf16 / fp32, "target" bf16, explicit fp32
COMBOS = [(0, 0), (0, 1), (0, 2), (1, 1), (2, 2), (2, 0)]


def load_ref_dequant():
    spec = importlib.util.spec_from_file_location("ref_dequant", os.path.join(REF, "dequant.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_ref_ops():
    tmp = tempfile.mkdtemp(prefix="refpkg_")
    pkg = os.path.join(tmp, "refgguf")
    os.mkdir(pkg)
    open(os.path.join(pkg, "__init__.py"), "w").close()
    for f in ("dequant.py", "ops.py"):
        os.symlink(os.path.join(REF, f), os.path.join(pkg, f))
    sys.path.insert(0, tmp)
    return importlib.import_module("refgguf.ops")


def bits(t: torch.Tensor) -> np.ndarray:
    t = t.contiguous()
    if t.dtype == torch.float32:
        return t.numpy().view(np.uint32).copy()
    return t.view(torch.int16).numpy().view(np.uint16).copy()


def edge_blocks(qtype, raw):
    """Overwrite a few leading blocks with corner cases: all-zero / all-one payloads, zero and large scales."""
    bs, ts = gguf.GGML_QUANT_SIZES[qtype]
    if qtype == T.BF16:
        return raw
    offs = oracle._F16_FIELDS[int(qtype)]

    def set_f16(b, vals):
        for off, v in zip(offs, vals):
            raw[b, off:off + 2] = np.array([v], dtype=np.float16).view(np.uint8)

    raw[0, :] = 0
    set_f16(0, [1.0, 1.0])
    raw[1, :] = 0xFF
    set_f16(1, [0.5, -0.25])
    raw[2, :] = 0xAA
    set_f16(2, [0.0, 0.0])
    raw[3, :] = 0x55
    set_f16(3, [-2.0, 6.1e-5])      # smallest normal fp16 as the second field
    raw[4, :] = 0x0F
    set_f16(4, [5.96e-8, 1e-3])     # subnormal scale
    set_f16(5, [48.0, -3.0])        # big-ish scale on random payload (products stay finite in fp16)
    return raw


def make_dequant(ref):
    for qt in QTYPES:
        bs, ts = gguf.GGML_QUANT_SIZES[qt]
        n_blocks = 40 if bs == 256 else (136 if bs == 32 else 4099)
        raw = oracle.random_blocks(int(qt), n_blocks, seed=1000 + int(qt))
        raw = edge_blocks(qt, raw)
        tt = torch.from_numpy(raw.reshape(-1).copy())
        out = {"packed": raw.reshape(-1), "qtype": np.int32(int(qt)), "n_blocks": np.int64(n_blocks)}
        for math, od in COMBOS:
            md = None if math == 0 else TORCH_DT[math]
            with torch.no_grad():
                r = ref.dequantize(tt, qt, (n_blocks * bs,), dtype=md).to(TORCH_DT[od])
            out[f"out_m{math}_o{od}"] = bits(r)
        np.savez_compressed(os.path.join(HERE, f"dequant_{qt.name}.npz"), **out)
        print("wrote dequant", qt.name, n_blocks, "blocks")


def make_linear(refops):
    GGMLTensor, GGMLOps = refops.GGMLTensor, refops.GGMLOps
    cases = [(T.Q4_K, 512, 96), (T.Q8_0, 512, 96), (T.Q5_K, 512, 80), (T.Q6_K, 256, 72), (T.Q4_0, 320, 64), (T.BF16, 192, 40)]
    M = 24
    for qt, K, N in cases:
        bs, ts = gguf.GGML_QUANT_SIZES[qt]
        raw = oracle.random_blocks(int(qt), N * K // bs, seed=2000 + int(qt), scale=0.02).reshape(N, K // bs * ts)
        rng = np.random.default_rng(3000 + int(qt))
        bias = rng.normal(0, 0.02, size=N).astype(np.float32)
        x32 = rng.normal(0, 1, size=(M, K)).astype(np.float32)
        for act, name in ((torch.bfloat16, "bf16"), (torch.float16, "f16"), (torch.float32, "f32")):
            lin = GGMLOps.Linear(K, N)
            sd = {
                "weight": GGMLTensor(torch.from_numpy(raw.copy()), tensor_type=qt, tensor_shape=torch.Size((N, K))),
                "bias": GGMLTensor(torch.from_numpy(bias.copy()), tensor_type=T.F32, tensor_shape=torch.Size((N,))),
            }
            lin.load_state_dict(sd)
            x = torch.from_numpy(x32).to(act)
            with torch.no_grad():
                y = lin(x)
            assert type(y) is torch.Tensor and y.dtype == act and tuple(y.shape) == (M, N)
            np.savez_compressed(
                os.path.join(HERE, f"linear_{qt.name}_{name}.npz"),
                packed=raw.reshape(-1), qtype=np.int32(int(qt)), N=np.int64(N), K=np.int64(K), M=np.int64(M),
                bias=bias, x=bits(x), y=bits(y))
        print("wrote linear", qt.name)


def make_surface():
    import ast
    import json

    def public(path):
        tree = ast.parse(open(path).read())
        return sorted(n.name for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and not n.name.startswith("_"))
    with open(os.path.join(HERE, "reference_surface.json"), "w") as f:
        json.dump({m: public(os.path.join(REF, m)) for m in ("dequant.py", "ops.py")}, f, indent=1)
        f.write("\n")


CHAIN_QTYPES = [T.Q8_0, T.Q4_0, T.Q4_K, T.Q5_K, T.Q6_K, T.BF16]
CHAIN_MATH = {"none": None, "float32": torch.float32, "bfloat16": torch.bfloat16}


def make_torch_chain(ref):
    import hashlib
    import json
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_torch_chain import Count      # the same kernel counter the test applies to oracle/torch_chain.py
    out = {}
    for qt in CHAIN_QTYPES:
        bs, _ts = gguf.GGML_QUANT_SIZES[qt]
        raw = torch.from_numpy(oracle.random_blocks(int(qt), 96, seed=1)).reshape(-1)
        for name, md in CHAIN_MATH.items():
            with Count() as c:
                y = ref.dequantize(raw, qt, (96 * bs,), dtype=md)
            raw_bytes = y.contiguous().view(torch.uint8).numpy()
            out[f"{qt.name}_{name}"] = {"dtype": str(y.dtype), "kernels": c.n, "nbytes": int(raw_bytes.size),
                                        "sha256": hashlib.sha256(raw_bytes.tobytes()).hexdigest()}
    with open(os.path.join(HERE, "torch_chain.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    torch.manual_seed(0)
    make_dequant(load_ref_dequant())
    make_linear(load_ref_ops())
    make_surface()
    make_torch_chain(load_ref_dequant())
    print("total bytes:", sum(os.path.getsize(os.path.join(HERE, f)) for f in os.listdir(HERE) if f.endswith(".npz")))
