#!/usr/bin/env python
"""LoKr and LoHa (LyCORIS) patches on Flux-shape quantised Linears: [3072, 3072], [12288, 3072] and [3072, 12288], bf16
activations, M in {4, 512, 4096}.  Adapters as trainers ship them for Flux: LoKr with factor 16 (w1 [16, 16]) and a full w2, LoKr
factor 16 with w2 decomposed at rank 16, LoHa at dim 8 and 16.

Arms, per (shape, M, adapter):
    two_step    what the reference runs on every forward: dequantise W, comfy.lora.calculate_weight restated (fp32 factors, the
                fp32 kron / Hadamard product at full [N, K] size, scaled, rounded to bf16 and added), then F.linear
    new         the patched layer: LoKr by ggufb200_dequant_kron + ggufb200_gemm; LoHa as a LoRA of rank dim^2 (in-kernel LoRA
                k-blocks up to rank 512)
    unpatched   the layer without patches (timed once per shape and M)
Method: CUDA events over CUDA-graph replays of 8 calls each, layers rotated over --copies weight copies (as
tools/bench_sd_linears.py).  `rel_vs_two_step` is the relative Frobenius distance of the new arm's output to the two-step arm's
on copy 0.  Prints the card name and power limit first; `--json PATH` also writes the rows."""
import argparse
import json
import os
import sys

import torch
import gguf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402
from bench_sd_linears import card, graph_time  # noqa: E402

SHAPES = [(3072, 3072), (12288, 3072), (3072, 12288)]
ADAPTERS = ["lokr_full_w2", "lokr_w2_rank16", "loha_dim8", "loha_dim16"]


def adapter(kind, N, K, g, dev):
    """One patch entry (strength, value, strength_model, offset, function) as ComfyUI builds it."""
    def r(*shape, s=0.05):
        return (torch.randn(*shape, generator=g) * s).to(dev)
    if kind == "lokr_full_w2":
        return (1.0, ("lokr", (r(16, 16, s=1.0), r(N // 16, K // 16, s=0.01), None, None, None, None, None, None, None)), 1.0, None, None)
    if kind == "lokr_w2_rank16":
        return (1.0, ("lokr", (r(16, 16, s=1.0), None, 16.0, None, None, r(N // 16, 16), r(16, K // 16), None, None)), 1.0, None, None)
    dim = int(kind[len("loha_dim"):])
    return (1.0, ("loha", (r(N, dim), r(dim, K), float(dim), r(N, dim), r(dim, K), None, None, None)), 1.0, None, None)


def two_step(ops, dq, x, w, bias, entry):
    """dequantise + calculate_weight (restated for one LoKr / LoHa entry without offset) + F.linear."""
    W = ops._plain(dq.dequantize_tensor(w, x.dtype))
    strength, (kind, v) = entry[0], entry[1]
    if kind == "lokr":
        w1, w2, alpha, w1_a, w1_b, w2_a, w2_b = v[:7]
        dim = None
        if w1 is None:
            dim, w1 = w1_b.shape[0], torch.mm(w1_a.float(), w1_b.float())
        if w2 is None:
            dim, w2 = w2_b.shape[0], torch.mm(w2_a.float(), w2_b.float())
        alpha = alpha / dim if alpha is not None and dim is not None else 1.0
        delta = torch.kron(w1.float(), w2.float())
    else:
        w1a, w1b, alpha, w2a, w2b = v[:5]
        alpha = 1.0 if alpha is None else alpha / w1b.shape[0]
        delta = torch.mm(w1a.float(), w1b.float()) * torch.mm(w2a.float(), w2b.float())
    W += ((strength * alpha) * delta).type(W.dtype)
    return torch.nn.functional.linear(x, W, bias)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--qtype", default="Q4_K")
    ap.add_argument("--M", type=int, nargs="+", default=[4, 512, 4096])
    ap.add_argument("--adapters", nargs="+", default=ADAPTERS)
    ap.add_argument("--copies", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lycoris: needs a CUDA device")
    ops, dq = ge._sub("ops"), ge._sub("dequant")
    dev = torch.device("cuda:0")
    act = torch.bfloat16
    qt = gguf.GGMLQuantizationType[args.qtype]
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    info = card()
    print(json.dumps(info), flush=True)
    rows = []
    for N, K in SHAPES:
        raws = [torch.from_numpy(oracle.random_blocks(int(qt), N * K // bs, seed=c, scale=0.02).reshape(N, K // bs * ts)).to(dev)
                for c in range(args.copies)]
        bias = (torch.randn(N, generator=torch.Generator().manual_seed(N + K)) * 0.02).to(dev, act)

        def layers():
            out = []
            for raw in raws:
                lin = ops.GGMLOps.Linear(K, N)
                lin.load_state_dict({"weight": ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size((N, K))),
                                     "bias": bias.clone()})
                out.append(lin)
            return out
        plain = layers()
        for M in args.M:
            x = torch.randn(M, K, generator=torch.Generator().manual_seed(M), dtype=torch.float32).to(dev, act)
            state = {"i": 0}

            def rotate(seq):
                state["i"] = (state["i"] + 1) % len(seq)
                return seq[state["i"]]
            ms_plain = graph_time(lambda: rotate(plain)(x), args.iters)
            for kind in args.adapters:
                entry = adapter(kind, N, K, torch.Generator().manual_seed(N + K + M), dev)
                patched = layers()
                for lin in patched:
                    lin.weight.patches = [([entry], "diffusion_model.w")]
                ms_new = graph_time(lambda: rotate(patched)(x), args.iters)
                ms_two = graph_time(lambda: two_step(ops, dq, x, rotate(plain).weight, bias, entry), args.iters)
                y_new = patched[0](x).float()
                y_two = two_step(ops, dq, x, plain[0].weight, bias, entry).float()
                row = {"qtype": args.qtype, "N": N, "K": K, "M": M, "adapter": kind, "ms_two_step": round(ms_two, 5),
                       "ms_new": round(ms_new, 5), "ms_unpatched": round(ms_plain, 5), "speedup_vs_two_step": round(ms_two / ms_new, 3),
                       "rel_vs_two_step": float((y_new - y_two).norm() / y_two.norm())}
                rows.append(row)
                print(json.dumps(row), flush=True)
                del patched
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "act": "bf16", "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
