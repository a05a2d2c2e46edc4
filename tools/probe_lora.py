#!/usr/bin/env python
"""One (M, N, K) Q4_K Linear with a rank-R LoRA patch: in-kernel (extra k-block of FUSED_TMEM) vs side GEMMs -- difference and time.
Run one shape per process under `timeout` so a hang is contained:  python tools/probe_lora.py M N K [rank]"""
import os
import sys
import time

import torch
import gguf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402

M, N, K = (int(v) for v in sys.argv[1:4])
R = int(sys.argv[4]) if len(sys.argv) > 4 else 32
ops = ge._sub("ops")
dev = torch.device("cuda:0")
qt = gguf.GGMLQuantizationType.Q4_K
bs, ts = gguf.GGML_QUANT_SIZES[qt]
raw = torch.from_numpy(oracle.random_blocks(int(qt), 1 << 14, seed=0, scale=0.02))
reps = (N * K // bs + (1 << 14) - 1) // (1 << 14)
w = ops.GGMLTensor(raw.repeat(reps, 1)[: N * K // bs].reshape(N, K // bs * ts).contiguous().to(dev), tensor_type=qt, tensor_shape=torch.Size((N, K)))
lin = ops.GGMLOps.Linear(K, N, bias=False)
lin.load_state_dict({"weight": w})
g = torch.Generator().manual_seed(1)
up = (torch.randn(N, R, generator=g) * 0.02).to(dev, torch.bfloat16)
down = (torch.randn(R, K, generator=g) * 0.02).to(dev, torch.bfloat16)
x = torch.randn(M, K, generator=g).to(dev, torch.bfloat16)
with torch.no_grad():
    y0 = lin(x)
    torch.cuda.synchronize()
    print(f"M={M} N={N} K={K}: unpatched ok", flush=True)
    lin.weight.patches = [([(0.8, ("lora", (up, down, float(R), None, None, None)), 1.0, None, None)], "w")]
    def gpu_us(fn, n=20):
        fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n * 1e3, (time.perf_counter() - t0) / n * 1e6
    res = {}
    for mode in ("side", "in_kernel"):
        ops.GGMLOps.Linear.lora_in_kernel = mode == "in_kernel"
        y = lin(x)
        torch.cuda.synchronize()
        res[mode] = (y, gpu_us(lambda: lin(x)))
    terms = lin._lora_terms(dev)
    down_pad, _u_pad, _tiles = lin._lora_operands(terms, dev, x.dtype)
    t_gemm = gpu_us(lambda: ops.linear_dense(x, down_pad))
    lin.weight.patches = []
    plain = gpu_us(lambda: lin(x))
    d = float(((res["in_kernel"][0].float() - res["side"][0].float()).norm() / res["side"][0].float().norm()).item())
    print(f"  rel diff in-kernel vs side {d:.2e};  (GPU us, wall us) per call: unpatched {plain[0]:.1f} {plain[1]:.1f} | side GEMMs {res['side'][1][0]:.1f} {res['side'][1][1]:.1f} | "
          f"in-kernel {res['in_kernel'][1][0]:.1f} {res['in_kernel'][1][1]:.1f} | T = x * down^T alone {t_gemm[0]:.1f} {t_gemm[1]:.1f}", flush=True)
