#!/usr/bin/env python
"""Kernel time of the quantised Linear at SD1.5 / SDXL shapes whose 256-element K-quant blocks straddle rows.

The GGUF converter reshapes SD1.5 / SDXL tensors whose last dimension is not a multiple of 256 to [n / 256, 256] before
quantising, so the K = 320 / 640 Linears of those UNets arrive as flat block streams (csrc/internal.h straddled_rows).  Arms:

    tmem_exact   FUSED_TMEM, reference rounding sequence (FLAG_EXACT_W); Q6_K reads the block-major copy
    tmem_fast    FUSED_TMEM, fused-multiply-add producers (Q4_K; Q6_K has one rounding either way)
    dq_mma       dequant + dense GEMM (GGUFB200_ALGO_DEQUANT_MMA)
    ref_chain    the reference's chain of ATen ops + cuBLAS (oracle/torch_chain.py)

Method: CUDA events over CUDA-graph replays of 8 calls each, weights rotated through `--copies` distinct buffers (ref_chain
builds host tensors per call, which a graph cannot capture: CUDA events around eager calls).  Each arm's
output on copy 0 is compared with tmem_exact's and with x @ W^T in float32 over the dequantised weight.  The card name and
power limit are read in the same run.  `--json PATH` also writes the rows."""
import argparse
import json
import os
import subprocess
import sys

import torch
import gguf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402
from oracle import torch_chain  # noqa: E402

# (model, M, N, K): SDXL at 1024^2 (4096 latent tokens, batch 1 and 2) and SD1.5 at 512^2; (640, 2560) is a whole-block control.
# M = 256 / 1024: shorter activations (smaller images, the 77-token text stream padded to a tile) on the same weights.
SHAPES = ([("sdxl", M, N, K) for M in (256, 1024, 4096, 8192) for N, K in ((640, 640), (5120, 640), (640, 2560))]
          + [("sd15", 4096, N, K) for N, K in ((320, 320), (2560, 320))])
ARMS = ["tmem_exact", "tmem_fast", "dq_mma", "ref_chain"]


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        info["power_limit, max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        info["power_limit, max_sm_clock"] = "unknown"
    return info


def eager_time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def graph_time(fn, iters, per=8):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(per):
            fn()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / (iters * per)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--qtypes", nargs="+", default=["Q4_K", "Q6_K"])
    ap.add_argument("--arms", nargs="+", default=ARMS)
    ap.add_argument("--act", default="bf16", choices=["bf16", "f16"])
    ap.add_argument("--copies", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sd_linears: needs a CUDA device")
    ops, dq, lib = ge._sub("ops"), ge._sub("dequant"), ge._sub("_lib")
    dev = torch.device("cuda:0")
    act = torch.bfloat16 if args.act == "bf16" else torch.float16
    info = card()
    print(json.dumps(info), flush=True)
    rows = []
    for qname in args.qtypes:
        qt = gguf.GGMLQuantizationType[qname]
        bs, ts = gguf.GGML_QUANT_SIZES[qt]
        for model, M, N, K in SHAPES:
            n_blocks = N * K // bs
            ws = []
            for c in range(args.copies):
                raw = torch.from_numpy(oracle.random_blocks(int(qt), n_blocks, seed=c, scale=0.02))
                shape = (n_blocks, ts) if K % bs else (N, K // bs * ts)      # the converter's reshape for a straddled weight
                ws.append(ops.GGMLTensor(raw.reshape(shape).to(dev), tensor_type=qt, tensor_shape=torch.Size((N, K))))
            spans = ops.needs_span_layout(qt, K)
            if spans:
                for w in ws:
                    ops.span_layout(w, w.as_subclass(torch.Tensor))           # built before any graph capture
            x = torch.randn(M, K, device=dev, dtype=act)
            state = {"i": 0}

            def nxt():
                state["i"] = (state["i"] + 1) % len(ws)
                return ws[state["i"]]
            arms = {
                "tmem_exact": lambda w: ops.linear_packed(x, w, None, None, lib.ALGO_FUSED_TMEM | lib.FLAG_EXACT_W, use_spans=spans),
                "tmem_fast": lambda w: ops.linear_packed(x, w, None, None, lib.ALGO_FUSED_TMEM, use_spans=spans),
                "dq_mma": lambda w: ops.linear_packed(x, w, None, None, lib.ALGO_DEQUANT_MMA | lib.FLAG_EXACT_W),
                "ref_chain": lambda w: torch_chain.linear(x, w.as_subclass(torch.Tensor), int(qt), (N, K)),
            }
            w0 = dq.dequantize_tensor(ws[0], act)
            ideal = x.float() @ w0.float().t()
            base = None
            for arm in args.arms:
                timer = eager_time if arm == "ref_chain" else graph_time
                ms = timer(lambda: arms[arm](nxt()), args.iters)
                y = arms[arm](ws[0]).float()
                if base is None:
                    base = y
                row = {"model": model, "qtype": qname, "M": M, "N": N, "K": K, "straddled": K % 256 != 0, "arm": arm, "timing": "eager" if arm == "ref_chain" else "graph", "ms": round(ms, 5),
                       "tflops": round(2.0 * M * N * K / ms / 1e9, 1), "relerr_ideal": float((y - ideal).norm() / ideal.norm()),
                       "relerr_vs_first_arm": float((y - base).norm() / base.norm())}
                rows.append(row)
                print(json.dumps(row), flush=True)
            del ws, w0, ideal, base
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "act": args.act, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
