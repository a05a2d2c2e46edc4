#!/usr/bin/env python
"""DoRA (weight-decomposed LoRA) patches on Flux-shape quantised Linears: [3072, 3072], [12288, 3072] and [3072, 12288], bf16
activations, M in {4, 512, 4096}.  The adapter is a rank-16 LoRA (alpha 16) with a DoRA magnitude on the output axis ([N, 1],
LyCORIS wd_on_out) or the input axis ([1, K]) drawn as the weight's own row / column norms times U(0.8, 1.2), at strength 1 and
0.8.

Arms, per (shape, M, axis, strength):
    two_step    what the reference runs on every forward: dequantise W, then comfy.lora.calculate_weight with `weight_decompose`
                restated (fp32 up @ down at full [N, K] size, the norm over the patched weight, the rescale, the blend for
                strength != 1), then F.linear
    new         the patched layer: in-kernel LoRA k-blocks with the feature scale (ggufb200_linear_lora_scaled), the input
                columns scaled first for the input axis
    lora        the same layer with the same LoRA without DoRA (the in-kernel LoRA route), for reference
Method: CUDA events over CUDA-graph replays of 8 calls each, layers rotated over --copies weight copies (as
tools/bench_sd_linears.py); every copy runs once before capture, so the per-patch-set plan is built outside the timed window.
`rel_vs_two_step` is the relative Frobenius distance of the new arm's output to the two-step arm's on copy 0.  Prints the card
name and power limit first; `--json PATH` also writes the rows."""
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
RANK = 16


def adapter(W, axis, strength, g, dev, dora=True):
    """One patch entry (strength, value, strength_model, offset, function) as ComfyUI builds it for a DoRA LoRA on weight W."""
    N, K = W.shape
    up, down = (torch.randn(N, RANK, generator=g) * 0.05).to(dev), (torch.randn(RANK, K, generator=g) * 0.05).to(dev)
    scale = None
    if dora:
        nrm = W.float().norm(dim=1 if axis == "out" else 0, keepdim=True)
        scale = nrm * (torch.rand(*nrm.shape, generator=g) * 0.4 + 0.8).to(dev)
    return (strength, ("lora", (up, down, float(RANK), None, scale, None)), 1.0, None, None)


def two_step(ops, dq, x, w, bias, entry):
    """dequantise + calculate_weight with weight_decompose (restated for one LoRA entry without offset) + F.linear."""
    W = ops._plain(dq.dequantize_tensor(w, x.dtype))
    strength, (_kind, v) = entry[0], entry[1]
    up, down, alpha, _mid, dora_scale = v[:5]
    alpha = alpha / down.shape[0]
    diff = torch.mm(up.float(), down.float())
    dora_scale = dora_scale.float()
    diff *= alpha
    Wc = W + diff.type(W.dtype)
    if dora_scale.shape[0] == W.shape[0]:
        nrm = W.reshape(W.shape[0], -1).norm(dim=1, keepdim=True)
    else:
        nrm = Wc.transpose(0, 1).reshape(W.shape[1], -1).norm(dim=1, keepdim=True).transpose(0, 1)
    nrm = nrm + torch.finfo(W.dtype).eps
    Wc *= (dora_scale / nrm).type(W.dtype)
    if strength != 1.0:
        Wc -= W
        W += strength * Wc
    else:
        W = Wc
    return torch.nn.functional.linear(x, W, bias)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--qtype", default="Q4_K")
    ap.add_argument("--M", type=int, nargs="+", default=[4, 512, 4096])
    ap.add_argument("--axes", nargs="+", default=["out", "in"])
    ap.add_argument("--strengths", type=float, nargs="+", default=[1.0, 0.8])
    ap.add_argument("--copies", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dora: needs a CUDA device")
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

        def layers(entry):
            out = []
            for raw in raws:
                lin = ops.GGMLOps.Linear(K, N)
                lin.load_state_dict({"weight": ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size((N, K))),
                                     "bias": bias.clone()})
                if entry is not None:
                    lin.weight.patches = [([entry], "diffusion_model.w")]
                out.append(lin)
            return out
        plain = layers(None)
        W = ops._plain(dq.dequantize_tensor(plain[0].weight, act))
        for M in args.M:
            x = torch.randn(M, K, generator=torch.Generator().manual_seed(M), dtype=torch.float32).to(dev, act)
            state = {"i": 0}

            def rotate(seq):
                state["i"] = (state["i"] + 1) % len(seq)
                return seq[state["i"]]

            def timed(seq):
                for lin in seq:                              # plans and caches built before capture
                    lin(x)
                return graph_time(lambda: rotate(seq)(x), args.iters)
            for axis in args.axes:
                for st in args.strengths:
                    g = torch.Generator().manual_seed(N + K + M)
                    entry = adapter(W, axis, st, g, dev)
                    g = torch.Generator().manual_seed(N + K + M)
                    lora_entry = adapter(W, axis, st, g, dev, dora=False)
                    patched, lora = layers(entry), layers(lora_entry)
                    ms_new = timed(patched)
                    ms_lora = timed(lora)
                    ms_two = graph_time(lambda: two_step(ops, dq, x, rotate(plain).weight, bias, entry), args.iters)
                    y_new = patched[0](x).float()
                    y_two = two_step(ops, dq, x, plain[0].weight, bias, entry).float()
                    row = {"qtype": args.qtype, "N": N, "K": K, "M": M, "axis": axis, "strength": st, "ms_two_step": round(ms_two, 5),
                           "ms_new": round(ms_new, 5), "ms_lora": round(ms_lora, 5), "new_over_two_step": round(ms_new / ms_two, 3),
                           "rel_vs_two_step": float((y_new - y_two).norm() / y_two.norm())}
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                    del patched, lora
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "act": "bf16", "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
