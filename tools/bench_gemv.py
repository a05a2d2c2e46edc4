#!/usr/bin/env python
"""GPU-side time of the small-M fused Linear (K3): raw C-ABI launches replayed from a CUDA graph (no Python / launch
overhead in the number), weights rotated through > L2 worth of buffers.  Routes: the integer-pattern mma.sync kernel (gemv2.cu, `fast` contract), the
FUSED_TMEM kernel (32-token items, K ranges across SMs) and the reference-exact mma.sync GEMV.  Prints GB/s of packed weight read vs the
measured HBM peak."""
import json
import os
import sys

import torch
import gguf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402

ops, lib = ge._sub("ops"), ge._sub("_lib")
L = lib.lib()
dev = torch.device("cuda:0")
peak = 3350.0      # H100 SXM data sheet, GB/s
try:
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass
CTAS = int(os.environ.get("GEMV2_CTAS", "0"))       # A/B of the CTAs-per-SM choice of gemv2 (needs GGUFB200_ALLOW_TUNING=1)
if CTAS:
    assert L.ggufb200_set_tuning(2, CTAS) == 0, "set GGUFB200_ALLOW_TUNING=1"
ONLY = os.environ.get("GEMV_ROUTES", "").split(",") if os.environ.get("GEMV_ROUTES") else None
ROUTES = (("gemv_fast_ws", lib.ALGO_GEMV_FAST | lib.FLAG_W_STABLE), ("gemv_fast", lib.ALGO_GEMV_FAST), ("tmem", lib.ALGO_FUSED_TMEM), ("tmem_exact", lib.ALGO_FUSED_TMEM | lib.FLAG_EXACT_W), ("gemv_exact", lib.ALGO_GEMV))
side = torch.cuda.Stream()
for qname in (sys.argv[1:] or ["Q4_K", "Q8_0", "Q5_K"]):
    qt = gguf.GGMLQuantizationType[qname]
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    for (N, K) in ((18432, 3072), (9216, 3072), (3072, 3072)):
        copies = 6
        ws = []
        for c in range(copies):
            raw = torch.from_numpy(oracle.random_blocks(int(qt), 1 << 14, seed=c, scale=0.02))
            reps = (N * K // bs + (1 << 14) - 1) // (1 << 14)
            ws.append(raw.repeat(reps, 1)[: N * K // bs].reshape(N, K // bs * ts).contiguous().to(dev))
        spans = [ops.span_layout(ops.GGMLTensor(w, tensor_type=qt, tensor_shape=torch.Size((N, K))), w) for w in ws]
        for M in (1, 4, 8):
            x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
            y = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            for name, algo in ROUTES:
                if name.startswith("gemv_fast") and qname not in ("Q4_K", "Q5_K"):
                    continue
                if ONLY and name not in ONLY:
                    continue
                need = L.ggufb200_linear_workspace(int(qt), M, N, K, 1, algo)
                wsb = torch.empty(max(need, 16), dtype=torch.uint8, device=dev)

                def launch(i, st):
                    if name == "tmem_spans":
                        rc = L.ggufb200_linear_spans(int(qt), ws[i % copies].data_ptr(), spans[i % copies].data_ptr(), N, K, x.data_ptr(), M, K, 1, 0,
                                                     None, 0, y.data_ptr(), N, wsb.data_ptr(), need, algo, st)
                    else:
                        rc = L.ggufb200_linear(int(qt), ws[i % copies].data_ptr(), N, K, x.data_ptr(), M, K, 1, 0, None, 0, y.data_ptr(), N,
                                               wsb.data_ptr(), need, algo, st)
                    assert rc == 0, rc
                st0 = torch.cuda.current_stream().cuda_stream
                for i in range(6):
                    launch(i, st0)
                torch.cuda.synchronize()
                per = 12
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=side):
                    for i in range(per):
                        launch(i, side.cuda_stream)
                g.replay()
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                iters = 10
                a.record()
                for _ in range(iters):
                    g.replay()
                b.record()
                torch.cuda.synchronize()
                us = a.elapsed_time(b) / (iters * per) * 1e3
                gbs = N * K // bs * ts / us / 1e3
                print(f"{qname} N={N} K={K} M={M} {name:12s}: {us:7.1f} us  {gbs:7.1f} GB/s packed read  ({gbs / peak:.3f} of measured HBM peak)", flush=True)
