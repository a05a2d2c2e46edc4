#!/usr/bin/env python
"""DoRA (weight-decomposed LoRA) patches on quantised SD1.5 / SDXL Conv2d weights, per call.

Shapes and method as tools/bench_conv_patches.py: the proj_in / proj_out 1x1 convs at 320, 640 and 1280 channels, the SD1.5 3x3
[640, 320, 3, 3] (K = 2880, straddled for the K-quants) and the SDXL 3x3 [1280, 1280, 3, 3], CFG batch 2.  Adapters: DoRA LoCon
at rank 16 / 32 / 64 on the output (`out`) and input (`in`) axis at strength 1 and 0.8 (`s0.8`), DoRA LoHa dim 16, DoRA LoKr
factor 8 (w2 whole), and a DoRA LoCon 16 followed by a plain LoCon 16.  DoRA magnitudes are the weight's own channel norms times
U(0.8, 1.2), as trainers initialise them.

Arms, per (shape, adapter):
    two_step      dequantise W, calculate_weight with ComfyUI's adapter arithmetic and weight_decompose restated, the convolution
    new           the layer on ggufb200_dequant_patched_dora (the patched weight in one launch, plan cached), the convolution,
                  whatever the cost model says
    layer         the patched layer as it routes by default (`ops.conv_dora_pays`); `route` names the entry point it called
and the weight alone: `w_two_step` / `w_new` for the list, `w_two_step_plain` / `w_new_plain` for the same list without its
dora_scale tensors (the two-step route's LoRA arithmetic and ggufb200_dequant_patched), the difference being what DoRA adds to each.
`plan_ms` is the one-off plan build of a patch set (K1, the replay of weight_decompose, the operands), host clock around a
synchronised build, median of 3.  Method: CUDA events over CUDA-graph replays of 8 calls each, layers rotated over --copies weight
copies.  `rel_new` is the relative Frobenius distance of the new arm's output to the two-step arm's on copy 0.  Prints the card
name, power limit and maximum SM clock first; `--json PATH` also writes the rows."""
import argparse
import json
import os
import statistics
import sys
import time

import gguf
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402
from bench_conv_lycoris import ref_diff  # noqa: E402
from bench_sd_linears import card, graph_time  # noqa: E402

SHAPES = [((320, 320, 1, 1), (2, 320, 64, 64)), ((640, 640, 1, 1), (2, 640, 32, 32)), ((1280, 1280, 1, 1), (2, 1280, 32, 32)),
          ((640, 320, 3, 3), (2, 320, 32, 32)), ((1280, 1280, 3, 3), (2, 1280, 32, 32))]
ADAPTERS = ["dora16-out", "dora32-out", "dora64-out", "dora16-in", "dora32-in", "dora64-in", "dora16-out-s0.8", "dora32-out-s0.8",
            "dora64-out-s0.8", "dora16-in-s0.8", "dora32-in-s0.8", "dora64-in-s0.8", "dloha16-out", "dlokr8-out", "dora16-out+lora16"]
DORA_AT = {"lora": 4, "loha": 7, "lokr": 8}


def weight_decompose(dora_scale, weight, lora_diff, alpha, strength):
    """ComfyUI's weight_decompose (comfy/weight_adapter/base.py), restated."""
    dora_scale = dora_scale.to(device=weight.device, dtype=torch.float32)
    lora_diff *= alpha
    weight_calc = weight + lora_diff.type(weight.dtype)
    if dora_scale.shape[0] == weight_calc.shape[0]:
        weight_norm = weight.reshape(weight.shape[0], -1).norm(dim=1, keepdim=True).reshape(weight.shape[0], *[1] * (weight.dim() - 1))
    else:
        weight_norm = (weight_calc.transpose(0, 1).reshape(weight_calc.shape[1], -1).norm(dim=1, keepdim=True)
                       .reshape(weight_calc.shape[1], *[1] * (weight_calc.dim() - 1)).transpose(0, 1))
    weight_norm = weight_norm + torch.finfo(weight.dtype).eps
    weight_calc *= (dora_scale / weight_norm).type(weight.dtype)
    if strength != 1.0:
        weight_calc -= weight
        weight += strength * weight_calc
    else:
        weight[:] = weight_calc
    return weight


def calculate_weight(patches, weight, key=None, intermediate_dtype=torch.float32, original_weights=None):
    """calculate_weight with ComfyUI's LoRA / LoHa / LoKr arithmetic and weight_decompose (the package's test double knows LoRA
    only)."""
    for strength, (kind, v), *_ in patches:
        alpha, diff = ref_diff(kind, v, weight.shape)
        ds = v[DORA_AT[kind]] if len(v) > DORA_AT[kind] else None
        if ds is not None:
            weight = weight_decompose(ds, weight, diff, alpha, strength)
        else:
            weight += ((strength * alpha) * diff).type(weight.dtype)
    return weight


def entries(name, shape, W, g, dev):
    """Patch entries (strength, value, strength_model, offset, function) as ComfyUI builds them; W: the dequantised weight, for
    the DoRA magnitudes."""
    cout, cin, kh, kw = shape

    def r(*s):
        return (torch.randn(*s, generator=g) * 0.05).to(dev)

    def magnitude(axis):
        if axis == "out":
            n = W.reshape(cout, -1).norm(dim=1).reshape(-1, 1, 1, 1)
        else:
            n = W.transpose(0, 1).reshape(cin, -1).norm(dim=1).reshape(1, -1, 1, 1)
        return n * (0.8 + 0.4 * torch.rand(*n.shape, generator=g).to(dev))
    out = []
    for part in name.split("+"):
        bits = part.split("-")
        strength = float(bits[2][1:]) if len(bits) > 2 else 1.0
        ds = magnitude(bits[1]) if len(bits) > 1 else None
        kind = bits[0].rstrip("0123456789")
        k = int(bits[0][len(kind):])
        if kind == "dlokr":
            payload = ("lokr", (r(k, k) * 20, r(cout // k, cin // k, kh, kw), None, None, None, None, None, None, ds))
        elif kind == "dloha":
            payload = ("loha", (r(cout, k), r(k, cin * kh * kw), float(k), r(cout, k), r(k, cin * kh * kw), None, None, ds))
        else:
            payload = ("lora", (r(cout, k, 1, 1), r(k, cin, kh, kw), float(k), None, ds, None))
        out.append((strength, payload, 1.0, None, None))
    return out


def without_dora(ents):
    return [(s, (kind, v[:DORA_AT[kind]] + (None,) + v[DORA_AT[kind] + 1:]), *rest) for s, (kind, v), *rest in ents]


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
        raise SystemExit("bench_conv_dora: needs a CUDA device")
    ops, dq, lib = ge._sub("ops"), ge._sub("dequant"), ge._sub("_lib")
    ops.comfy_lora.calculate_weight = calculate_weight
    default_pays = ops.conv_dora_pays
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
            N, K = shape[0], numel // shape[0]
            raws = [torch.from_numpy(oracle.random_blocks(int(qt), numel // bs, seed=c, scale=0.02).reshape(-1)).to(dev)
                    for c in range(args.copies)]
            bias = (torch.randn(shape[0], generator=torch.Generator().manual_seed(shape[0])) * 0.02).to(dev)
            bias_act = bias.to(act)
            x = torch.randn(*xshape, generator=torch.Generator().manual_seed(1)).to(dev, act)

            def layers(ents):
                out = []
                for raw in raws:
                    conv = ops.GGMLOps.Conv2d(shape[1], shape[0], shape[2], padding=shape[2] // 2, device="meta")
                    w = ops.GGMLTensor(raw, tensor_type=qt, tensor_shape=torch.Size(shape),
                                       patches=[(ents, "diffusion_model.conv.weight")] if ents else [])
                    conv.load_state_dict({"weight": w, "bias": bias.clone()}, assign=True)
                    out.append(conv)
                return out
            state = {"i": 0}

            def rotate(seq):
                state["i"] = (state["i"] + 1) % len(seq)
                return seq[state["i"]]
            plain = layers(None)
            W0 = ops._plain(dq.dequantize_tensor(plain[0].weight, torch.float32))
            for name in args.adapters:
                ents = entries(name, shape, W0, torch.Generator().manual_seed(numel), dev)
                ents_plain = without_dora(ents)
                patched, patched_plain = layers(ents), layers(ents_plain)

                def w_two(conv, e):
                    return calculate_weight(e, ops._plain(dq.dequantize_tensor(conv.weight, act)))
                # the layer as it routes by default
                route = {}
                real = {n: getattr(lib.lib(), n) for n in ("ggufb200_dequant_patched_dora", "ggufb200_dequant_patched",
                                                            "ggufb200_dequant_lowrank")}
                for n, fn in real.items():
                    setattr(lib.lib(), n, lambda *a, _fn=fn, _n=n: route.setdefault("name", _n) and _fn(*a))
                try:
                    for conv in patched:
                        conv(x)
                finally:
                    for n, fn in real.items():
                        setattr(lib.lib(), n, fn)
                ms_layer = graph_time(lambda: rotate(patched)(x), args.iters)
                # the kernel whatever the cost models say
                ops.conv_dora_pays = lambda *_a: True
                lowrank_pays = ops.lowrank_pays
                ops.lowrank_pays = lambda *_a: True
                try:
                    for conv in patched + patched_plain:
                        conv.__dict__.pop("_gg_conv_dora_" + str(act).split(".")[-1], None)
                        conv(x)
                    ms_new = graph_time(lambda: rotate(patched)(x), args.iters)
                    y_new = patched[0](x).float()
                    plans = [conv._conv_dora_plan(x) for conv in patched]
                    operands = [conv._conv_patch_operands(x) or conv._conv_lycoris_operands(x) for conv in patched_plain]
                    plan_ms = []
                    for _ in range(3):
                        patched[0].__dict__.pop("_gg_conv_dora_" + str(act).split(".")[-1], None)
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        patched[0]._conv_dora_plan(x)
                        torch.cuda.synchronize()
                        plan_ms.append((time.perf_counter() - t0) * 1e3)
                finally:
                    ops.conv_dora_pays, ops.lowrank_pays = default_pays, lowrank_pays
                plain_entry = "ggufb200_dequant_lowrank" if ops.conv_patch_terms(ents_plain) else "ggufb200_dequant_patched"

                def w_new(conv, dora):
                    i = state["i"]
                    W = torch.empty(shape, dtype=act, device=dev)
                    raw = conv.weight.as_subclass(torch.Tensor)
                    if dora:
                        _keep, descs, dd = plans[i]
                        rc = lib.lib().ggufb200_dequant_patched_dora(int(qt), raw.data_ptr(), N, K, W.data_ptr(), dq.dtype_code(act),
                                                                     dq.math_code(None, act), descs, dd, len(ents),
                                                                     torch.cuda.current_stream().cuda_stream)
                    else:
                        _keep, descs = operands[i]
                        rc = getattr(lib.lib(), plain_entry)(int(qt), raw.data_ptr(), N, K, W.data_ptr(), dq.dtype_code(act),
                                                             dq.math_code(None, act), descs, len(ents), torch.cuda.current_stream().cuda_stream)
                    lib.check(rc, "w_new")
                    return W
                ms_two = graph_time(lambda: (lambda c: c._conv_forward(x, w_two(c, ents), bias_act))(rotate(plain)), args.iters)
                y_two = plain[0]._conv_forward(x, w_two(plain[0], ents), bias_act).float()
                row = {"qtype": qname, "shape": list(shape), "x": list(xshape), "adapter": name, "route": route.get("name", "two_step"),
                       "ms_two_step": round(ms_two, 5), "ms_new": round(ms_new, 5), "ms_layer": round(ms_layer, 5),
                       "speedup_new": round(ms_two / ms_new, 3), "plan_ms": round(statistics.median(plan_ms), 3),
                       "rel_new": float((y_new - y_two).norm() / y_two.norm()),
                       "w_two_step": round(graph_time(lambda: w_two(rotate(plain), ents), args.iters), 5),
                       "w_new": round(graph_time(lambda: w_new(rotate(patched), True), args.iters), 5),
                       "w_two_step_plain": round(graph_time(lambda: w_two(rotate(plain), ents_plain), args.iters), 5),
                       "w_new_plain": round(graph_time(lambda: w_new(rotate(patched_plain), False), args.iters), 5)}
                state["i"] = 0
                rows.append(row)
                print(json.dumps(row), flush=True)
                del patched, patched_plain, plans, operands
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "act": args.act, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
