#!/usr/bin/env python
"""K1 launch-overhead probe: back-to-back (CUDA-graph) dequant of Q4_K / Q8_0 tensors of growing size, with and without
GGUFB200_DEQUANT_SRC_STABLE.  If GB/s keeps rising with the tensor size the per-launch ramp / drain, not the steady state, is what
separates the Flux-shape sweep from the copy peak."""
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
for qname in (sys.argv[1:] or ["Q4_K", "Q8_0"]):
    qt = gguf.GGMLQuantizationType[qname]
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    seed = torch.from_numpy(oracle.random_blocks(int(qt), 1 << 15, seed=3, scale=0.02))
    for N in (3072, 9216, 21504, 43008, 86016, 172032):
        K = 3072
        n_blocks = N * K // bs
        copies = max(2, min(12, (1 << 30) // (N * K * 2)))          # > 2 x L2 of distinct outputs per pass
        reps = (n_blocks + (1 << 15) - 1) // (1 << 15)
        packed = seed.repeat(reps, 1)[:n_blocks].contiguous().to(dev)
        ws = [packed.clone() for _ in range(copies)]
        outs = [torch.empty(N * K, dtype=torch.float16, device=dev) for _ in range(copies)]
        torch.cuda.synchronize()
        for label, math in (("plain", 0), ("src_stable", lib.DEQUANT_SRC_STABLE)):
            def launch(i, st):
                rc = L.ggufb200_dequant(int(qt), ws[i % copies].data_ptr(), n_blocks, outs[i % copies].data_ptr(), 0, math, st)
                assert rc == 0, rc
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
            iters = max(3, 400 // per)
            a.record()
            for _ in range(iters):
                g.replay()
            b.record()
            torch.cuda.synchronize()
            us = a.elapsed_time(b) / (iters * per) * 1e3
            by = n_blocks * ts + N * K * 2
            print(f"{qname} [{N},{K}] {label:10s}: {us:8.2f} us/launch  {by / us / 1e3:7.1f} GB/s  ({by / us / 1e3 / peak:.3f} of {peak:.0f})", flush=True)
        del ws, outs, packed
        torch.cuda.empty_cache()
