#!/usr/bin/env python
"""LoRA / LoCon and LoHa patches on quantised SD1.5 / SDXL Conv2d weights, per call.

Shapes (weight, activation at 512 / 1024 px with CFG batch 2): the transformer proj_in / proj_out 1x1 convs at 320, 640 and
1280 channels on [2, 320, 64, 64], [2, 640, 32, 32] and [2, 1280, 32, 32], an SD1.5 ResBlock conv [640, 320, 3, 3] on
[2, 320, 32, 32] (K = 2880: straddled for the K-quants), an SDXL ResBlock conv [1280, 1280, 3, 3] on [2, 1280, 32, 32].
LoRA / LoCon at ranks 16 .. 256 (4-D factors), LoHa at dim 16 and 32.

Arms, per (shape, adapter):
    two_step    what the reference runs on every forward: dequantise W, calculate_weight restated (fp32 torch.mm of the flattened
                factors, scaled, rounded to the activation dtype and added), then the convolution
    new         ggufb200_dequant_lowrank (the patched weight in one launch), then the convolution, whatever the cost model says
    layer       the patched layer as it routes by default (`ops.lowrank_pays`); `kernel_taken` says which route that was
    unpatched   the layer without patches: K1 + the convolution
and the weight alone: `w_two_step` (dequantise + patch), `w_new` (ggufb200_dequant_lowrank), `w_k1` (K1 only).
Method: CUDA events over CUDA-graph replays of 8 calls each, layers rotated over --copies weight copies.  `rel_vs_two_step` is the
relative Frobenius distance of the new arm's output to the two-step arm's on copy 0.  Prints the card name, power limit and
maximum SM clock first; `--json PATH` also writes the rows."""
import argparse
import json
import os
import sys

import gguf
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402
from bench_sd_linears import card, graph_time  # noqa: E402

SHAPES = [((320, 320, 1, 1), (2, 320, 64, 64)), ((640, 640, 1, 1), (2, 640, 32, 32)), ((1280, 1280, 1, 1), (2, 1280, 32, 32)),
          ((640, 320, 3, 3), (2, 320, 32, 32)), ((1280, 1280, 3, 3), (2, 1280, 32, 32))]
ADAPTERS = ["lora16", "lora32", "lora64", "lora128", "lora256", "loha16", "loha32"]


def adapter(kind, shape, g, dev):
    """One patch entry (strength, value, strength_model, offset, function) as ComfyUI builds it."""
    cout, cin, kh, kw = shape

    def r(*s):
        return (torch.randn(*s, generator=g) * 0.05).to(dev)
    if kind.startswith("lora"):
        rank = int(kind[4:])
        return (1.0, ("lora", (r(cout, rank, 1, 1), r(rank, cin, kh, kw), float(rank), None, None, None)), 1.0, None, None)
    dim = int(kind[4:])
    K = cin * kh * kw
    return (1.0, ("loha", (r(cout, dim), r(dim, K), float(dim), r(cout, dim), r(dim, K), None, None, None)), 1.0, None, None)


def two_step_weight(ops, dq, w, dtype, entry):
    """dequantise + calculate_weight restated for one LoRA / LoHa entry without offset."""
    W = ops._plain(dq.dequantize_tensor(w, dtype))
    strength, (kind, v) = entry[0], entry[1]
    if kind == "lora":
        up, down, alpha = v[0].float(), v[1].float(), v[2]
        alpha = 1.0 if alpha is None else alpha / down.shape[0]
        delta = torch.mm(up.flatten(start_dim=1), down.flatten(start_dim=1)).reshape(W.shape)
    else:
        w1a, w1b, alpha, w2a, w2b = v[:5]
        alpha = 1.0 if alpha is None else alpha / w1b.shape[0]
        delta = (torch.mm(w1a.float(), w1b.float()) * torch.mm(w2a.float(), w2b.float())).reshape(W.shape)
    W += ((strength * alpha) * delta).type(W.dtype)
    return W


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--qtypes", nargs="+", default=["Q4_K", "Q8_0"])
    ap.add_argument("--adapters", nargs="+", default=ADAPTERS)
    ap.add_argument("--act", default="f16", choices=["bf16", "f16"])
    ap.add_argument("--copies", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv_patches: needs a CUDA device")
    ops, dq = ge._sub("ops"), ge._sub("dequant")
    dev = torch.device("cuda:0")
    act = torch.bfloat16 if args.act == "bf16" else torch.float16
    info = card()
    print(json.dumps(info), flush=True)
    rows = []
    for qname in args.qtypes:
        qt = gguf.GGMLQuantizationType[qname]
        bs, _ts = gguf.GGML_QUANT_SIZES[qt]
        for shape, xshape in SHAPES:
            numel = shape[0] * shape[1] * shape[2] * shape[3]
            raws = [torch.from_numpy(oracle.random_blocks(int(qt), numel // bs, seed=c, scale=0.02).reshape(-1)).to(dev)
                    for c in range(args.copies)]
            bias = (torch.randn(shape[0], generator=torch.Generator().manual_seed(shape[0])) * 0.02).to(dev)
            x = torch.randn(*xshape, generator=torch.Generator().manual_seed(1)).to(dev, act)

            def layers(entry):
                out = []
                for raw in raws:
                    conv = ops.GGMLOps.Conv2d(shape[1], shape[0], shape[2], padding=shape[2] // 2, device="meta")
                    w = ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size(shape),
                                       patches=[([entry], "diffusion_model.conv.weight")] if entry else [])
                    conv.load_state_dict({"weight": w, "bias": bias.clone()}, assign=True)
                    out.append(conv)
                return out
            state = {"i": 0}

            def rotate(seq):
                state["i"] = (state["i"] + 1) % len(seq)
                return seq[state["i"]]
            plain = layers(None)
            ms_plain = graph_time(lambda: rotate(plain)(x), args.iters)
            ms_w_k1 = graph_time(lambda: dq.dequantize_tensor(rotate(plain).weight, act), args.iters)
            for kind in args.adapters:
                entry = adapter(kind, shape, torch.Generator().manual_seed(numel), dev)
                patched = layers(entry)

                def two_step(conv):
                    W = two_step_weight(ops, dq, conv.weight, act, entry)
                    return conv._conv_forward(x, W, bias.to(act))

                def new_weight(conv):
                    captured = {}
                    conv._conv_forward = lambda inp, w, b: captured.setdefault("w", w)
                    conv(x)
                    del conv._conv_forward
                    return captured["w"]
                N, K = shape[0], numel // shape[0]
                taken = ops.lowrank_pays(N, K, ops.conv_patch_terms([entry]))
                ms_layer = graph_time(lambda: rotate(patched)(x), args.iters)
                pays = ops.lowrank_pays
                ops.lowrank_pays = lambda N, K, terms: True                 # the kernel, whatever the cost model says
                try:
                    ms_new = graph_time(lambda: rotate(patched)(x), args.iters)
                    ms_w_new = graph_time(lambda: new_weight(rotate(patched)), args.iters)
                    y_new = patched[0](x).float()
                finally:
                    ops.lowrank_pays = pays
                ms_two = graph_time(lambda: two_step(rotate(plain)), args.iters)
                ms_w_two = graph_time(lambda: two_step_weight(ops, dq, rotate(plain).weight, act, entry), args.iters)
                y_two = two_step(plain[0]).float()
                row = {"qtype": qname, "shape": list(shape), "x": list(xshape), "adapter": kind, "ms_two_step": round(ms_two, 5),
                       "ms_new": round(ms_new, 5), "ms_layer": round(ms_layer, 5), "kernel_taken": taken, "ms_unpatched": round(ms_plain, 5), "speedup_vs_two_step": round(ms_two / ms_new, 3),
                       "w_two_step": round(ms_w_two, 5), "w_new": round(ms_w_new, 5), "w_k1": round(ms_w_k1, 5),
                       "rel_vs_two_step": float((y_new - y_two).norm() / y_two.norm())}
                rows.append(row)
                print(json.dumps(row), flush=True)
                del patched
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "act": args.act, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
