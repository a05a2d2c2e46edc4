#!/usr/bin/env python
"""The Linear of the eleven numpy-fallback types on text-encoder shapes: ggufb200_linear_fallback's fused route (FUSED_SYNC, the
weight decoded from the packed bytes in registers) against the two-step route the layer ran before it (ggufb200_dequant_fallback
into an [N, K] activation-dtype weight + ggufb200_gemm), and the Embedding row gather against the whole-table dequant.

Shapes: Qwen3-4B [9728, 2560] [2560, 9728] [4096, 2560], Qwen2.5-VL-7B [18944, 3584] [3584, 18944], Mistral-Small-24B
[32768, 5120] [5120, 32768]; every type, bf16 and fp16, M in 1 8 16 32 64 77 128 256 512.
Method: CUDA events around --iters calls per window, the two routes alternating window by window (--reps windows each, after
--warmup calls); --copies-style rotation of the packed weights and the outputs past L2 (at least 120 MB of packed bytes per
route); the median per call is reported.  Per point: microseconds, packed-byte GB/s (packed bytes / time), TFLOP/s (2 M N K /
time), the bound of the fused route (`bytes`: packed bytes / 3.35 TB/s is the larger lower bound, `flops`: 2 M N K / 989
TFLOP/s is), the speed-up (two-step time / fused time) and the largest ulp difference between the two routes' outputs on the
same seeded inputs (finite elements; both routes use the same weight operand, only the fp32 summation order differs, so the
large counts sit at outputs that cancel to near zero), and that difference over the largest output magnitude.
Embedding: 512 ids from a [151936, 2560] IQ2_XXS table, ggufb200_dequant_rows_fallback against ggufb200_dequant_fallback of the
whole table (fp32, the Embedding's dtype) + the gather.  Prints the card name and power limit first; `--json PATH` also writes
the rows."""
import argparse
import json
import os
import sys

import gguf
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import __graft_entry__ as ge  # noqa: E402
from bench_sd_linears import card  # noqa: E402
from fallback_cases import FALLBACK, random_blocks  # noqa: E402

Q = gguf.GGMLQuantizationType
SHAPES = [(9728, 2560), (2560, 9728), (4096, 2560), (18944, 3584), (3584, 18944), (32768, 5120), (5120, 32768)]
M_LIST = [1, 8, 16, 32, 64, 77, 128, 256, 512]
HBM_BPS, PEAK_FLOPS = 3.35e12, 989e12          # H100 SXM data sheet: HBM3 bandwidth, dense bf16 / fp16 tensor rate


def packed_copies(qt, N, K, dev, min_bytes):
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    n_blocks = N * K // bs
    seed = torch.from_numpy(random_blocks(qt, 1 << 14, seed=3, scale=0.01))
    base = seed.repeat((n_blocks + (1 << 14) - 1) // (1 << 14), 1)[:n_blocks].contiguous().to(dev)
    copies = max(2, min(32, -(-min_bytes // base.numel())))
    return [base] + [base.clone() for _ in range(copies - 1)], n_blocks


def ordered(bits16):
    """fp16 / bf16 bit patterns (int16) -> integers whose difference counts ulps across zero."""
    b = bits16.to(torch.int32)
    return torch.where(b < 0, -(b & 0x7FFF), b)


class Point:
    def __init__(self, L, lib, qt, packs, n_blocks, N, K, M, dt, dev, ws_dense):
        self.L, self.lib, self.qt, self.packs, self.n_blocks, self.N, self.K, self.M, self.dt = L, lib, qt, packs, n_blocks, N, K, M, dt
        self.act = lib.BF16 if dt == torch.bfloat16 else lib.F16
        g = torch.Generator(device=dev).manual_seed(M * 31 + N)
        self.xs = [torch.randn(M, K, generator=g, device=dev).to(dt) for _ in range(len(packs))]
        self.ys = [torch.empty(M, N, dtype=dt, device=dev) for _ in range(len(packs))]
        need = L.ggufb200_linear_fallback_workspace(int(qt), M, N, K, self.act, lib.ALGO_FUSED_SYNC)
        self.ws = torch.empty(max(need, 16), dtype=torch.uint8, device=dev)
        self.need = need
        self.ws_dense = ws_dense
        self.st = torch.cuda.current_stream().cuda_stream

    def fused(self, i):
        p, x, y = self.packs[i], self.xs[i], self.ys[i]
        rc = self.L.ggufb200_linear_fallback(int(self.qt), p.data_ptr(), self.N, self.K, x.data_ptr(), self.M, self.K, self.act, None, 0,
                                             y.data_ptr(), self.N, self.ws.data_ptr(), self.need,
                                             self.lib.ALGO_FUSED_SYNC | self.lib.FLAG_W_STABLE, self.st)
        assert rc == 0, rc

    def two_step(self, i):
        p, x, y, w = self.packs[i], self.xs[i], self.ys[i], self.ws_dense
        rc = self.L.ggufb200_dequant_fallback(int(self.qt), p.data_ptr(), self.n_blocks, w.data_ptr(), self.act, self.lib.DEQUANT_SRC_STABLE,
                                              self.st)
        assert rc == 0, rc
        rc = self.L.ggufb200_gemm(w.data_ptr(), self.N, self.K, self.K, x.data_ptr(), self.M, self.K, self.act, None, 0, y.data_ptr(), self.N,
                                  self.st)
        assert rc == 0, rc


def time_pair(pt, iters, reps, warmup):
    n = len(pt.packs)
    for fn in (pt.fused, pt.two_step):
        for i in range(warmup):
            fn(i % n)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t = {"fused": [], "two_step": []}
    for _ in range(reps):
        for name, fn in (("fused", pt.fused), ("two_step", pt.two_step)):
            a.record()
            for i in range(iters):
                fn(i % n)
            b.record()
            b.synchronize()
            t[name].append(a.elapsed_time(b) * 1e3 / iters)
    return float(np.median(t["fused"])), float(np.median(t["two_step"]))


def max_ulp(pt):
    pt.fused(0)
    y_f = pt.ys[0].clone()
    pt.two_step(0)
    y_d = pt.ys[0].clone()
    fin = torch.isfinite(y_f) & torch.isfinite(y_d)
    assert torch.equal(fin, torch.isfinite(y_f)) and torch.equal(fin, torch.isfinite(y_d)), "the routes disagree on non-finite outputs"
    if not bool(fin.any()):
        return 0, 0.0
    d = (ordered(y_f.view(torch.int16)) - ordered(y_d.view(torch.int16))).abs()
    scale = y_d[fin].float().abs().max()
    rel = float((y_f[fin].float() - y_d[fin].float()).abs().max() / scale) if scale > 0 else 0.0
    return int(d[fin].max()), rel


def embedding_rows(L, lib, dev, iters, reps):
    qt, V, D = Q.IQ2_XXS, 151936, 2560
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    seed = torch.from_numpy(random_blocks(qt, 1 << 14, seed=5, scale=0.01))
    n_blocks = V * D // bs
    table = seed.repeat(n_blocks // (1 << 14) + 1, 1)[:n_blocks].contiguous().to(dev)
    ids = torch.randint(0, V, (512,), device=dev)
    out = torch.empty(512, D, dtype=torch.float32, device=dev)
    full = torch.empty(V, D, dtype=torch.float32, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def gather():
        assert L.ggufb200_dequant_rows_fallback(int(qt), table.data_ptr(), V, D, ids.data_ptr(), 512, out.data_ptr(), lib.F32, st) == 0

    def whole():
        assert L.ggufb200_dequant_fallback(int(qt), table.data_ptr(), n_blocks, full.data_ptr(), lib.F32, lib.DEQUANT_SRC_STABLE, st) == 0
        torch.nn.functional.embedding(ids, full)

    res = {}
    for name, fn in (("rows_us", gather), ("whole_table_us", whole)):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts_ = []
        for _ in range(reps):
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            b.synchronize()
            ts_.append(a.elapsed_time(b) * 1e3 / iters)
        res[name] = round(float(np.median(ts_)), 1)
    gather()
    whole()
    ref = torch.nn.functional.embedding(ids, full)
    res["bit_identical"] = bool(torch.equal(out.view(torch.int32), ref.view(torch.int32)))
    return {"embedding": f"{qt.name} [{V}, {D}], 512 ids, fp32", **res}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--min-rotated-mb", type=int, default=120)
    ap.add_argument("--types", default=",".join(q.name for q in FALLBACK))
    ap.add_argument("--shapes", default=None, help="N:K,N:K,... (default: the seven text-encoder shapes)")
    ap.add_argument("--m", default=",".join(map(str, M_LIST)))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    dev = torch.device("cuda:0")
    lib = ge._sub("_lib")
    L = lib.lib()
    info = card()
    print(json.dumps(info), flush=True)
    shapes = SHAPES if not args.shapes else [tuple(map(int, s.split(":"))) for s in args.shapes.split(",")]
    ms = [int(m) for m in args.m.split(",")]
    rows = []
    for N, K in shapes:
        ws_dense = torch.empty(N * K * 2, dtype=torch.uint8, device=dev)
        for qt in (Q[t] for t in args.types.split(",")):
            bs, ts = gguf.GGML_QUANT_SIZES[qt]
            packs, n_blocks = packed_copies(qt, N, K, dev, args.min_rotated_mb << 20)
            packed_bytes = packs[0].numel()
            for dt in (torch.bfloat16, torch.float16):
                for M in ms:
                    pt = Point(L, lib, qt, packs, n_blocks, N, K, M, dt, dev, ws_dense)
                    fused_us, two_us = time_pair(pt, args.iters, args.reps, args.warmup)
                    flops = 2.0 * M * N * K
                    bound = "bytes" if packed_bytes / HBM_BPS >= flops / PEAK_FLOPS else "flops"
                    row = {"type": qt.name, "N": N, "K": K, "dtype": str(dt).split(".")[-1], "M": M,
                           "fused_us": round(fused_us, 1), "two_step_us": round(two_us, 1), "speedup": round(two_us / fused_us, 3),
                           "fused_packed_GBps": round(packed_bytes / (fused_us * 1e-6) / 1e9, 1),
                           "fused_TFLOPs": round(flops / (fused_us * 1e-6) / 1e12, 2),
                           "two_step_TFLOPs": round(flops / (two_us * 1e-6) / 1e12, 2), "bound": bound,
                           "splits_ws_bytes": pt.need, "rotated_copies": len(packs)}
                    row["max_ulp"], row["max_diff_over_max_abs"] = max_ulp(pt)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                    del pt
            del packs
            torch.cuda.empty_cache()
        del ws_dense
        torch.cuda.empty_cache()
    emb = embedding_rows(L, lib, dev, args.iters * 4, args.reps)
    print(json.dumps(emb), flush=True)
    # per type and M: the smallest and the median speed-up over shapes and dtypes (AUTO's crossover is read from these)
    summary = []
    for t in args.types.split(","):
        for M in ms:
            s = [r["speedup"] for r in rows if r["type"] == t and r["M"] == M]
            if s:
                summary.append({"type": t, "M": M, "min_speedup": min(s), "median_speedup": round(float(np.median(s)), 3)})
    for s in summary:
        print(json.dumps(s))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": info, "rows": rows, "embedding": emb, "summary": summary}, f, indent=1)


if __name__ == "__main__":
    main()
