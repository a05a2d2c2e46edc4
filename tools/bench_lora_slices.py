#!/usr/bin/env python
"""Diffusers-format (sliced) LoRA on Flux's fused Linears: `qkv` [9216, 3072] (q / k / v bands of 3072 rows) and a single
block's `linear1` [21504, 3072] (q / k / v + proj_mlp bands), Q4_K weights, bf16 activations, one LoRA of rank r per band,
as ComfyUI hands it over (patch entries with offset = (0, start, size)).

Arms, per (shape, M, r):
    unpatched     the layer without patches (AUTO route: the GEMV at M <= 8, else FUSED_TMEM)
    in_kernel     the patched layer: LoRA k-blocks inside FUSED_TMEM with the per-tile k-block table
    no_table      the same call with a NULL table (every tile runs every LoRA k-block)
    two_step      dequantise W, add each band's (strength * alpha / r * up @ down) in fp32 rounded to bf16 the way
                  comfy.lora.calculate_weight does for an offset entry, then F.linear
CUDA events over --iters calls after --warmup calls, layers rotated over --copies weights (more bytes than L2 holds); the arms
are timed in turn, --rounds times, and the median (min - max) ms per call is printed.  The last column is each arm's relative
Frobenius distance to the unrounded result x @ (W + delta)^T (fp32 GEMM on the same dequantised W), so the LoRA's own effect
shows in the unpatched arm's distance.  Prints the GPU name and power limit first."""
import argparse
import os
import subprocess
import sys

import torch
import gguf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402

H = 3072
SHAPES = {"qkv": [(0, H), (H, H), (2 * H, H)], "linear1": [(0, H), (H, H), (2 * H, H), (3 * H, 4 * H)]}


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        q = f"nvidia-smi unavailable ({exc})"
    return f"{name}; power limit, max SM clock: {q}"


def timeit(fn, iters, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="*", default=list(SHAPES))
    ap.add_argument("--M", type=int, nargs="+", default=[1, 512, 4608])
    ap.add_argument("--ranks", type=int, nargs="+", default=[16, 32, 64, 128])
    ap.add_argument("--copies", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    ops, dq = ge._sub("ops"), ge._sub("dequant")
    dev = torch.device("cuda:0")
    act = torch.bfloat16
    qt = gguf.GGMLQuantizationType.Q4_K
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    print(gpu_info(), flush=True)
    g = torch.Generator().manual_seed(0)
    for shape in args.shapes:
        bands = SHAPES[shape]
        N, K = sum(size for _s, size in bands), H
        packed = []
        for c in range(args.copies):
            chunk = 1 << 15
            raw = torch.from_numpy(oracle.random_blocks(int(qt), chunk, seed=c, scale=0.02))
            packed.append(raw.repeat((N * K // bs + chunk - 1) // chunk, 1)[: N * K // bs].reshape(N, K // bs * ts).contiguous().to(dev))

        def layer(p):
            lin = ops.GGMLOps.Linear(K, N, bias=False)
            lin.load_state_dict({"weight": ops.GGMLTensor(p, tensor_type=qt, tensor_shape=torch.Size((N, K)))})
            return lin
        for r in args.ranks:
            patches = [[(1.0, (torch.randn(size, r, generator=g) * 0.05).to(dev, act), (torch.randn(r, K, generator=g) * 0.05).to(dev, act),
                         float(r), (0, start, size)) for start, size in bands] for _c in range(args.copies)]
            plain, tiled, untiled = [], [], []
            for c in range(args.copies):
                plain.append(layer(packed[c]))
                for group in (tiled, untiled):
                    lin = layer(packed[c])
                    lin.weight.patches = [([(s, ("lora", (up, down, alpha, None, None, None)), 1.0, off, None)
                                            for s, up, down, alpha, off in patches[c]], "w")]
                    group.append(lin)
            for M in args.M:
                x = torch.randn(M, K, generator=g).to(dev, act)
                with torch.no_grad():
                    for lin in tiled + untiled:
                        lin(x)                                  # builds and caches the LoRA operands
                    for lin in untiled:                         # same operands, NULL table
                        key, (down_pad, u_pad, _tiles) = lin.__dict__["_gg_lora"]
                        lin.__dict__["_gg_lora"] = (key, (down_pad, u_pad, None))
                    state = {"i": 0}

                    def nxt():
                        state["i"] = (state["i"] + 1) % args.copies
                        return state["i"]

                    def two_step(c=None):
                        c = nxt() if c is None else c
                        W = ops._plain(dq.dequantize_tensor(plain[c].weight, act))
                        for s, up, down, alpha, (dim, start, size) in patches[c]:
                            W.narrow(dim, start, size).add_((s * alpha / r * torch.mm(up.float(), down.float())).to(act))
                        return torch.nn.functional.linear(x, W)
                    arms = {"unpatched": lambda: plain[nxt()](x), "in_kernel": lambda: tiled[nxt()](x),
                            "no_table": lambda: untiled[nxt()](x), "two_step": two_step}
                    W = ops._plain(dq.dequantize_tensor(plain[0].weight, act)).float()
                    for s, up, down, alpha, (dim, start, size) in patches[0]:
                        W.narrow(dim, start, size).add_(s * alpha / r * torch.mm(up.float(), down.float()))
                    ideal = x.float() @ W.t()
                    del W
                    times = {name: [] for name in arms}
                    for _round in range(args.rounds):
                        for name, fn in arms.items():
                            times[name].append(timeit(fn, args.iters, args.warmup))
                    for name in arms:
                        y = {"unpatched": plain, "in_kernel": tiled, "no_table": untiled}[name][0](x) if name != "two_step" else two_step(0)
                        err = float((y.float() - ideal).norm() / ideal.norm())
                        t = sorted(times[name])
                        print(f"{shape:8s} N={N:6d} K={K} M={M:5d} r={r:4d} (sum {r * len(bands):4d}) {name:10s} {t[len(t) // 2]:8.4f} ms "
                              f"({t[0]:.4f} - {t[-1]:.4f})  rel dist to unrounded {err:.2e}", flush=True)


if __name__ == "__main__":
    main()
