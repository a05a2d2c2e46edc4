#!/usr/bin/env python
"""Per-shape timing of the quantised Linear at Flux.1 shapes: FUSED_TMEM (tmem, tmem384, tmem_generic), FUSED_MMA with
reference-exact producers (fused), dequant + dense GEMM (dq_mma), K1 dequant + cuBLAS, cuBLAS on a pre-dequantised weight, the reference's
torch chain.  CUDA events, weights rotated through >L2 worth of distinct buffers.  Prints one line per (shape, route): ms,
TFLOP/s and the relative error against fp32-accumulated x @ bf16(W)^T of the SAME weight the timed call used."""
import argparse
import os
import sys

import numpy as np
import torch
import gguf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402
from oracle import torch_chain  # noqa: E402

SHAPES = [(3072, 3072), (9216, 3072), (12288, 3072), (3072, 12288), (18432, 3072), (21504, 3072), (3072, 15360)]


GRAPH = False


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    if GRAPH:   # kernel time without the Python / launch overhead: replay a captured batch of calls
        per = 8
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
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--qtype", default="Q4_K")
    ap.add_argument("--M", type=int, nargs="+", default=[4608])
    ap.add_argument("--shapes", type=int, nargs="*", default=None, help="indices into SHAPES")
    ap.add_argument("--routes", nargs="*", default=["tmem", "tmem384", "fused", "dq_mma", "k1_cublas", "cublas", "ref_chain"])
    ap.add_argument("--act", default="bf16", choices=["bf16", "f16"])
    ap.add_argument("--nk", type=int, nargs="*", default=None, help="explicit N K pairs (flat list) instead of the Flux shapes")
    ap.add_argument("--copies", type=int, default=4)
    ap.add_argument("--graph", action="store_true", help="time CUDA-graph replays (kernel time only)")
    ap.add_argument("--no-splitk", action="store_true")
    args = ap.parse_args()
    global GRAPH
    GRAPH = args.graph
    ops, dq, lib = ge._sub("ops"), ge._sub("dequant"), ge._sub("_lib")
    dev = torch.device("cuda:0")
    nosplit = lib.FLAG_NOSPLIT if args.no_splitk else 0
    act = torch.bfloat16 if args.act == "bf16" else torch.float16
    qt = gguf.GGMLQuantizationType[args.qtype]
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    shapes = SHAPES if not args.shapes else [SHAPES[i] for i in args.shapes]
    if args.nk:
        shapes = list(zip(args.nk[0::2], args.nk[1::2]))
    for (N, K) in shapes:
        ws = []
        for c in range(args.copies):
            chunk = min(N * K // bs, 1 << 15)
            raw = torch.from_numpy(oracle.random_blocks(int(qt), chunk, seed=c, scale=0.02))
            reps = (N * K // bs + chunk - 1) // chunk
            packed = raw.repeat(reps, 1)[: N * K // bs].reshape(N, K // bs * ts).contiguous().to(dev)
            ws.append(ops.GGMLTensor(packed, tensor_type=qt, tensor_shape=torch.Size((N, K))))
        for M in args.M:
            x = torch.randn(M, K, device=dev, dtype=act)
            flops = 2.0 * M * N * K
            state = {"i": 0}

            def nxt():
                state["i"] = (state["i"] + 1) % len(ws)
                return ws[state["i"]]
            dense = [dq.dequantize_tensor(w, act) for w in ws[:2]] if ("cublas" in args.routes or "ours_dense" in args.routes) else []
            routes = {
                "tmem": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | nosplit),
                "tmem384": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | lib.FLAG_TILE384 | nosplit),
                "tmem192": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | lib.FLAG_TILE192 | nosplit),
                "tmem_ns": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | lib.FLAG_NOSPLIT),
                "tmem192_ns": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | lib.FLAG_TILE192 | lib.FLAG_NOSPLIT),
                "tmem384_ns": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | lib.FLAG_TILE384 | lib.FLAG_NOSPLIT),
                "tmem_exact": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | lib.FLAG_EXACT_W | nosplit),
                "tmem384_exact": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | lib.FLAG_EXACT_W | lib.FLAG_TILE384 | nosplit),
                "tmem_spans": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | nosplit, use_spans=True),
                "tmem384_spans": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | lib.FLAG_TILE384 | nosplit, use_spans=True),
                "tmem_generic": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_TMEM | lib.FLAG_GENERIC | nosplit),
                "fused": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_FUSED_MMA | nosplit),
                "auto": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_AUTO),
                "auto_exact": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_AUTO | lib.FLAG_EXACT_W),
                "gemv_fast": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_GEMV_FAST),
                "gemv": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_GEMV),
                "dq_mma": lambda: ops.linear_packed(x, nxt(), None, None, lib.ALGO_DEQUANT_MMA),
                "k1_cublas": lambda: torch.nn.functional.linear(x, dq.dequantize_tensor(nxt(), act)),
                "cublas": lambda: torch.nn.functional.linear(x, dense[state["i"] % 2]),
                "ours_dense": lambda: ops.linear_dense(x, dense[state["i"] % 2]),
                "ref_chain": lambda: torch_chain.linear(x, nxt().as_subclass(torch.Tensor), int(qt), (N, K)),
            }
            pbytes = N * K // bs * ts
            for name in args.routes:
                ms = timeit(routes[name])
                y = routes[name]()
                # the call above advanced the rotation: compare against the weight IT used (cublas / ours_dense: dense[i % 2])
                i = state["i"]
                wref = dense[i % 2] if name in ("cublas", "ours_dense") else dq.dequantize_tensor(ws[i], act)
                ref = (x.float() @ wref.float().t())
                err = float(((y.float() - ref).norm() / ref.norm()).item())
                print(f"{args.qtype} N={N:6d} K={K:6d} M={M:5d} {name:12s} {ms:8.4f} ms  {flops / ms / 1e9:8.1f} TFLOP/s  "
                      f"{pbytes / ms / 1e6:7.1f} GB/s packed  relerr={err:.2e}", flush=True)
                del ref, wref
            del dense


if __name__ == "__main__":
    main()
