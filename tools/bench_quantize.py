"""GPU quantiser (ggufb200_quantize, ggufb200_quantize_k) throughput and a full Flux-shape conversion.

1. Kernel GB/s per type and source dtype over the seven Flux Linear shapes: algorithmic bytes = source bytes read + packed bytes
   written, CUDA events around `--iters` launches that rotate over enough copies of the tensor to spill L2.  The K types
   (Q6_K ... Q2_K, ggufb200_quantize_k) are compute-bound: their rows report the same source-plus-output GB/s and the time.
2. Baseline: gguf-py's numpy `gguf.quants.quantize` on the same tensors (fp32 input; one run per shape, `--numpy-shapes`).
3. A full convert of a random Flux-shape checkpoint (19 double + 38 single blocks, bf16, `--blocks` to shorten) to each
   `--qtype` (a type or a K mixture such as Q4_K_S), the time split into read, quantise (including the copies to and from the
   GPU) and write.
Prints the card name and power limit first; `--json PATH` also writes the rows."""
import argparse
import json
import os
import sys
import tempfile
import time

import gguf
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
from bench_sd_linears import card  # noqa: E402

Q = gguf.GGMLQuantizationType
SHAPES = [(3072, 3072), (9216, 3072), (12288, 3072), (3072, 12288), (18432, 3072), (21504, 3072), (3072, 15360)]
TYPES = [Q.Q8_0, Q.Q5_1, Q.Q5_0, Q.Q4_1, Q.Q4_0, Q.BF16]
K_TYPES = [Q.Q6_K, Q.Q5_K, Q.Q4_K, Q.Q3_K, Q.Q2_K]
SRC = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


def kernel_rows(L, lib, iters, types):
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream(dev).cuda_stream
    rows = []
    for name, dt in SRC.items():
        for qt in types:
            entry = L.ggufb200_quantize_k if qt in K_TYPES else L.ggufb200_quantize
            bs, ts = gguf.GGML_QUANT_SIZES[qt]
            moved = total_s = 0.0
            for N, K in SHAPES:
                n = N * K
                copies = max(2, int(np.ceil(200e6 / (n * torch.finfo(dt).bits // 8))))     # > 50 MB L2, rotated
                xs = [(torch.randn(N, K, device=dev) * 0.02).to(dt) for _ in range(copies)]
                outs = [torch.empty(n // bs * ts, dtype=torch.uint8, device=dev) for _ in range(copies)]
                code = {torch.float16: lib.F16, torch.bfloat16: lib.BF16, torch.float32: lib.F32}[dt]
                launch = lambda i: entry(int(qt), xs[i % copies].data_ptr(), code, n // bs, outs[i % copies].data_ptr(), 0, stream)
                for i in range(copies):
                    assert launch(i) == 0
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for i in range(iters):
                    launch(i)
                b.record()
                torch.cuda.synchronize()
                sec = a.elapsed_time(b) / 1e3 / iters
                nbytes = n * xs[0].element_size() + n // bs * ts
                rows.append({"src": name, "qtype": qt.name, "N": N, "K": K, "us": sec * 1e6, "GB/s": nbytes / sec / 1e9})
                moved += nbytes
                total_s += sec
                del xs, outs
            print(f"{name:>5} {qt.name:>5}: " + " ".join(f"{r['GB/s']:7.0f}" for r in rows[-len(SHAPES):])
                  + f"   all shapes {moved / total_s / 1e9:7.0f} GB/s, {total_s * 1e3:8.2f} ms", flush=True)
    return rows


def numpy_rows(n_shapes):
    rows = []
    for N, K in SHAPES[:n_shapes]:
        x = (np.random.default_rng(0).standard_normal((N, K)) * 0.02).astype(np.float32)
        for qt in TYPES:
            bs, ts = gguf.GGML_QUANT_SIZES[qt]
            t0 = time.perf_counter()
            gguf.quants.quantize(x, qt)
            sec = time.perf_counter() - t0
            rows.append({"qtype": qt.name, "N": N, "K": K, "s": sec, "GB/s": (x.nbytes + N * K // bs * ts) / sec / 1e9})
            print(f"numpy {qt.name:>5} [{N}, {K}]: {sec * 1e3:9.1f} ms  {rows[-1]['GB/s']:6.2f} GB/s", flush=True)
    return rows


def flux_checkpoint(blocks_double, blocks_single):
    g = torch.Generator().manual_seed(0)
    sd = {}

    def add(k, *shape):
        sd["model.diffusion_model." + k] = (torch.randn(*shape, generator=g) * 0.02).bfloat16()
    add("img_in.weight", 3072, 64)
    add("img_in.bias", 3072)
    for i in range(blocks_double):
        for s in ("img", "txt"):
            add(f"double_blocks.{i}.{s}_mod.lin.weight", 18432, 3072)
            add(f"double_blocks.{i}.{s}_attn.qkv.weight", 9216, 3072)
            add(f"double_blocks.{i}.{s}_attn.proj.weight", 3072, 3072)
            add(f"double_blocks.{i}.{s}_mlp.0.weight", 12288, 3072)
            add(f"double_blocks.{i}.{s}_mlp.2.weight", 3072, 12288)
            add(f"double_blocks.{i}.{s}_attn.norm.query_norm.scale", 128)
    for i in range(blocks_single):
        add(f"single_blocks.{i}.modulation.lin.weight", 9216, 3072)
        add(f"single_blocks.{i}.linear1.weight", 21504, 3072)
        add(f"single_blocks.{i}.linear2.weight", 3072, 15360)
        add(f"single_blocks.{i}.linear1.bias", 21504)
    add("final_layer.linear.weight", 64, 3072)
    return sd


def convert_row(qtype, blocks_double, blocks_single, tmp):
    from safetensors.torch import save_file
    conv = ge._sub("convert")
    src = os.path.join(tmp, "flux.safetensors")
    save_file(flux_checkpoint(blocks_double, blocks_single), src)
    res = conv.convert_file(src, os.path.join(tmp, "flux-{ftype}.gguf"), qtype=qtype, overwrite=True)
    size = os.path.getsize(res.path)
    row = {"qtype": qtype, "double_blocks": blocks_double, "single_blocks": blocks_single, "src_bytes": os.path.getsize(src),
           "dst_bytes": size, **{f"{k}_s": v for k, v in res.seconds.items()}}
    print(f"convert {qtype} ({blocks_double} double + {blocks_single} single blocks, {row['src_bytes'] / 1e9:.1f} GB bf16 -> "
          f"{size / 1e9:.2f} GB): " + ", ".join(f"{k} {v:.2f} s" for k, v in res.seconds.items()), flush=True)
    os.remove(src)
    os.remove(res.path)
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--numpy-shapes", type=int, default=2)
    ap.add_argument("--qtype", nargs="+", default=["Q8_0"], help="conversion targets: types or K mixtures")
    ap.add_argument("--types", nargs="+", default=[q.name for q in TYPES + K_TYPES], help="kernel rows for these types")
    ap.add_argument("--blocks", type=int, nargs=2, default=[19, 38], metavar=("DOUBLE", "SINGLE"))
    ap.add_argument("--tmp", default=None, help="directory for the converted checkpoint (default: a temporary directory)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_quantize needs a GPU"
    ge.load_package()
    lib = ge._sub("_lib")
    info = card()
    print(json.dumps(info), flush=True)
    print("kernel GB/s per shape " + " ".join(f"{N}x{K}" for N, K in SHAPES), flush=True)
    types = [Q[t] for t in args.types]
    out = {"card": info, "kernel": kernel_rows(lib.lib(), lib, args.iters, types), "numpy": numpy_rows(args.numpy_shapes)}
    with tempfile.TemporaryDirectory(dir=args.tmp) as tmp:
        out["convert"] = [convert_row(q, args.blocks[0], args.blocks[1], tmp) for q in args.qtype]
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
