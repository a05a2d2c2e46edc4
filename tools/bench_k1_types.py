#!/usr/bin/env python
"""Standalone dequant (K1) for every block format x output dtype at [21504,3072] and [3072,3072]: back-to-back GB/s (CUDA-graph
replay over > L2 worth of distinct buffers, GGUFB200_DEQUANT_SRC_STABLE) as a fraction of the measured copy peak."""
import json
import os
import sys

import torch
import gguf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402

lib = ge._sub("_lib")
L = lib.lib()
dev = torch.device("cuda:0")
peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0   # H100 SXM data sheet
side = torch.cuda.Stream()
OUT = ((0, torch.float16, "f16"), (1, torch.bfloat16, "bf16"), (2, torch.float32, "f32"))
names = sys.argv[1:] or ["Q4_0", "Q4_1", "Q5_0", "Q5_1", "Q8_0", "Q2_K", "Q3_K", "Q4_K", "Q5_K", "Q6_K", "IQ4_NL", "IQ4_XS"]
for qname in names:
    qt = gguf.GGMLQuantizationType[qname]
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    seed = torch.from_numpy(oracle.random_blocks(int(qt), 1 << 15, seed=3, scale=0.02))
    for (N, K) in ((21504, 3072), (3072, 3072)):
        n_blocks = N * K // bs
        packed = seed.repeat((n_blocks + (1 << 15) - 1) // (1 << 15), 1)[:n_blocks].contiguous().to(dev)
        for code, tdt, oname in OUT:
            ob = 4 if code == 2 else 2
            copies = max(3, min(16, (600 << 20) // (N * K * ob)))
            ws = [packed.clone() for _ in range(copies)]
            outs = [torch.empty(N * K, dtype=tdt, device=dev) for _ in range(copies)]

            def launch(i, st):
                assert L.ggufb200_dequant(int(qt), ws[i % copies].data_ptr(), n_blocks, outs[i % copies].data_ptr(), code, lib.DEQUANT_SRC_STABLE, st) == 0
            per = 2 * copies
            for i in range(per):
                launch(i, torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                for i in range(per):
                    launch(i, side.cuda_stream)
            g.replay()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            iters = max(3, 300 // per)
            a.record()
            for _ in range(iters):
                g.replay()
            b.record()
            torch.cuda.synchronize()
            us = a.elapsed_time(b) / (iters * per) * 1e3
            by = n_blocks * ts + N * K * ob
            print(f"{qname:7s} [{N},{K}] -> {oname:4s}: {us:8.2f} us/launch  {by / us / 1e3:7.1f} GB/s  ({by / us / 1e3 / peak:.3f} of {peak:.0f})", flush=True)
            del ws, outs
        del packed
        torch.cuda.empty_cache()
