#!/usr/bin/env python
"""K1 (ggufb200_dequant_fallback) for the eleven numpy-fallback types on text-encoder weight shapes, with Q4_K K1
(ggufb200_dequant, the reference's default fp16 math) in the same run as the control.

Shapes: T5-xxl [10240, 4096] and [4096, 10240], Qwen3-4B-like [9728, 2560]; bf16 output (the text encoders' activation dtype).
Method: CUDA events around back-to-back launches on --copies distinct packed/output buffer pairs (rotated, > 100 MB in total,
so L2 never holds the next call's bytes), GGUFB200_DEQUANT_SRC_STABLE as the layers pass it; per call the median over
--reps windows of --iters calls.  GB/s counts the algorithmic bytes: TS/BS packed bytes read + 2 output bytes written per
element.  `vs_q4k` is the type's rate over Q4_K's rate at the same shape.  The reference's own path (gguf.quants.dequantize on
the host + the host-to-device copy of its fp32 result, cast to bf16) is timed once, for IQ2_XXS at [9728, 2560].
Prints the card name and power limit first; `--json PATH` also writes the rows."""
import argparse
import json
import os
import sys
import time

import gguf
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402
from bench_sd_linears import card  # noqa: E402
from fallback_cases import FALLBACK, random_blocks  # noqa: E402

Q = gguf.GGMLQuantizationType
SHAPES = [(10240, 4096), (4096, 10240), (9728, 2560)]


def packed_copies(qt, n_elems, copies, dev):
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    n_blocks = n_elems // bs
    if qt == Q.Q4_K:
        seed = torch.from_numpy(oracle.random_blocks(int(qt), 1 << 14, seed=3, scale=0.02))
    else:
        seed = torch.from_numpy(random_blocks(qt, 1 << 14, seed=3, scale=0.01))
    reps = (n_blocks + (1 << 14) - 1) // (1 << 14)
    base = seed.repeat(reps, 1)[:n_blocks].contiguous()
    return [base.to(dev) for _ in range(copies)], n_blocks


def time_k1(L, lib, qt, n_elems, copies, iters, reps, dev):
    packs, n_blocks = packed_copies(qt, n_elems, copies, dev)
    outs = [torch.empty(n_elems, dtype=torch.bfloat16, device=dev) for _ in range(copies)]
    st = torch.cuda.current_stream().cuda_stream
    if qt == Q.Q4_K:
        def call(i):
            return L.ggufb200_dequant(int(qt), packs[i].data_ptr(), n_blocks, outs[i].data_ptr(), lib.BF16, lib.F16 | lib.DEQUANT_SRC_STABLE, st)
    else:
        def call(i):
            return L.ggufb200_dequant_fallback(int(qt), packs[i].data_ptr(), n_blocks, outs[i].data_ptr(), lib.BF16, lib.DEQUANT_SRC_STABLE, st)
    for i in range(copies):
        assert call(i) == 0
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        a.record()
        for i in range(iters):
            call(i % copies)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    total_mb = copies * (packs[0].numel() + outs[0].numel() * 2) / 1e6
    return float(np.median(times)), total_mb


def reference_path(qt, N, K, dev):
    """gguf.quants.dequantize on the host + torch.from_numpy(...).to(device, bf16): the reference's fallback branch."""
    raw = random_blocks(qt, N * K // gguf.GGML_QUANT_SIZES[qt][0], seed=4, scale=0.01)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    host = gguf.quants.dequantize(raw.reshape(-1), qt)
    t1 = time.perf_counter()
    torch.from_numpy(host).to(dev, dtype=torch.bfloat16)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    return (t1 - t0) * 1e3, (t2 - t1) * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--copies", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--types", default=",".join(q.name for q in FALLBACK))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    dev = torch.device("cuda:0")
    lib = ge._sub("_lib")
    L = lib.lib()
    info = card()
    print(json.dumps(info))
    rows = []
    types = [Q.Q4_K] + [Q[t] for t in args.types.split(",")]
    for N, K in SHAPES:
        q4k_rate = None
        for qt in types:
            bs, ts = gguf.GGML_QUANT_SIZES[qt]
            ms, total_mb = time_k1(L, lib, qt, N * K, args.copies, args.iters, args.reps, dev)
            gbs = N * K * (ts / bs + 2) / (ms * 1e-3) / 1e9
            if qt == Q.Q4_K:
                q4k_rate = gbs
            row = {"type": qt.name, "N": N, "K": K, "ms": round(ms, 4), "GB/s": round(gbs, 1), "vs_q4k": round(gbs / q4k_rate, 3),
                   "rotated_MB": round(total_mb, 1)}
            rows.append(row)
            print(json.dumps(row), flush=True)
            torch.cuda.empty_cache()
    host_ms, h2d_ms = reference_path(Q.IQ2_XXS, 9728, 2560, dev)
    ref = {"reference_path": "IQ2_XXS", "N": 9728, "K": 2560, "numpy_dequant_ms": round(host_ms, 1), "h2d_cast_ms": round(h2d_ms, 1)}
    print(json.dumps(ref))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": info, "rows": rows, "reference": ref}, f, indent=1)


if __name__ == "__main__":
    main()
