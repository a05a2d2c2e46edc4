#!/usr/bin/env python
"""LoKr, Tucker LoCon and Tucker LoHa patches on quantised SD1.5 / SDXL Conv2d weights, per call.

Shapes and method as tools/bench_conv_patches.py: the proj_in / proj_out 1x1 convs at 320, 640 and 1280 channels, the SD1.5 3x3
[640, 320, 3, 3] (K = 2880, straddled for the K-quants) and the SDXL 3x3 [1280, 1280, 3, 3], CFG batch 2.  Adapters: LoKr factor
4 / 8 / 16 with w2 whole (4-D), decomposed (rank 16) and Tucker (`t2`, rank 16); Tucker LoCon (`mid`) at rank 16 / 32; Tucker
LoHa at dim 8 / 16; LoKr factor 8 + LoRA rank 32.

Arms, per (shape, adapter):
    two_step    dequantise W, calculate_weight restated (ComfyUI's adapter arithmetic), then the convolution
    new         ggufb200_dequant_patched (the patched weight in one launch), then the convolution, whatever the routing says
    kron        ggufb200_dequant_kron + the convolution (LoKr only, block formats)
    layer       the patched layer as it routes by default; `route` names the entry point it called (or "two_step")
    unpatched   the layer without patches: K1 + the convolution
Method: CUDA events over CUDA-graph replays of 8 calls each, layers rotated over --copies weight copies.  `rel_*` is the relative
Frobenius distance of an arm's output to the two-step arm's on copy 0.  A LoKr entry whose reference `torch.kron` raises (ComfyUI
skips it) is reported with `reference_skips`.  Prints the card name, power limit and maximum SM clock first; `--json PATH` also
writes the rows."""
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
ADAPTERS = ["lokr4", "lokr8", "lokr16", "lokr4d", "lokr8d", "lokr16d", "lokr8t", "locon16", "locon32", "loha8", "loha16",
            "lokr8+lora32"]


def entries(name, shape, g, dev):
    """Patch entries (strength, value, strength_model, offset, function) as ComfyUI builds them."""
    cout, cin, kh, kw = shape

    def r(*s):
        return (torch.randn(*s, generator=g) * 0.05).to(dev)
    out = []
    for part in name.split("+"):
        if part.startswith("lokr"):
            form = part[-1] if part[-1] in "dt" else ""
            f = int(part[4:len(part) - len(form)])
            b1, c2 = cout // f, cin // f
            w1 = r(f, f)
            if form == "d":
                payload = (w1, None, 16.0, None, None, r(b1, 16), r(16, c2 * kh * kw), None, None)
            elif form == "t":
                payload = (w1, None, 16.0, None, None, r(16, b1), r(16, c2), r(16, 16, kh, kw), None)
            else:
                payload = (w1, r(b1, c2, kh, kw), None, None, None, None, None, None, None)
            out.append((1.0, ("lokr", payload), 1.0, None, None))
        elif part.startswith("locon"):
            k = int(part[5:])
            out.append((1.0, ("lora", (r(cout, k, 1, 1), r(k, cin, 1, 1), float(k), r(k, k, kh, kw), None, None)), 1.0, None, None))
        elif part.startswith("loha"):
            k = int(part[4:])
            out.append((1.0, ("loha", (r(k, cout), r(k, cin), float(k), r(k, cout), r(k, cin), r(k, k, kh, kw), r(k, k, kh, kw), None)),
                        1.0, None, None))
        else:
            k = int(part[4:])
            out.append((1.0, ("lora", (r(cout, k, 1, 1), r(k, cin, kh, kw), float(k), None, None, None)), 1.0, None, None))
    return out


def ref_diff(kind, v, shape):
    """(alpha, fp32 diff or None when ComfyUI skips the entry) of one payload, as ComfyUI's adapters form it."""
    f = [t.float() if torch.is_tensor(t) else t for t in v]
    if kind == "lora":
        up, down, alpha, mid = f[:4]
        alpha = 1.0 if alpha is None else alpha / down.shape[0]
        if mid is not None:
            final_shape = [down.shape[1], down.shape[0], mid.shape[2], mid.shape[3]]
            down = torch.mm(down.transpose(0, 1).flatten(start_dim=1), mid.transpose(0, 1).flatten(start_dim=1)).reshape(final_shape).transpose(0, 1)
        return alpha, torch.mm(up.flatten(start_dim=1), down.flatten(start_dim=1)).reshape(shape)
    if kind == "loha":
        w1a, w1b, alpha, w2a, w2b, t1, t2 = f[:7]
        alpha = 1.0 if alpha is None else alpha / w1b.shape[0]
        if t1 is not None:
            m1 = torch.einsum("i j k l, j r, i p -> p r k l", t1, w1b, w1a)
            m2 = torch.einsum("i j k l, j r, i p -> p r k l", t2, w2b, w2a)
        else:
            m1, m2 = torch.mm(w1a, w1b), torch.mm(w2a, w2b)
        return alpha, (m1 * m2).reshape(shape)
    w1, w2, alpha, w1_a, w1_b, w2_a, w2_b, t2 = f[:8]
    dim = None
    if w1 is None:
        dim, w1 = w1_b.shape[0], torch.mm(w1_a, w1_b)
    if w2 is None:
        dim = w2_b.shape[0]
        w2 = torch.mm(w2_a, w2_b) if t2 is None else torch.einsum("i j k l, j r, i p -> p r k l", t2, w2_b, w2_a)
    if w2.dim() == 4:
        w1 = w1.unsqueeze(2).unsqueeze(2)
    alpha = alpha / dim if (alpha is not None and dim is not None) else 1.0
    try:
        return alpha, torch.kron(w1, w2).reshape(shape)
    except RuntimeError:
        return alpha, None


def two_step_weight(ops, dq, w, dtype, ents):
    W = ops._plain(dq.dequantize_tensor(w, dtype))
    for strength, (kind, v), *_ in ents:
        alpha, diff = ref_diff(kind, v, W.shape)
        if diff is not None:
            W += ((strength * alpha) * diff).type(W.dtype)
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
        raise SystemExit("bench_conv_lycoris: needs a CUDA device")
    ops, dq, lib = ge._sub("ops"), ge._sub("dequant"), ge._sub("_lib")

    def calculate_weight(patches, weight, key, intermediate_dtype=torch.float32, original_weights=None):
        """The layer's two-step route with ComfyUI's adapter arithmetic (the package's test double knows LoRA only)."""
        for strength, (kind, v), *_ in patches:
            alpha, diff = ref_diff(kind, v, weight.shape)
            if diff is not None:
                weight += ((strength * alpha) * diff).type(weight.dtype)
        return weight
    ops.comfy_lora.calculate_weight = calculate_weight
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
            ms_plain = graph_time(lambda: rotate(plain)(x), args.iters)
            for name in args.adapters:
                ents = entries(name, shape, torch.Generator().manual_seed(numel), dev)
                patched = layers(ents)
                terms = ops.conv_lycoris_terms(ents)
                skips = any(kind == "lokr" and ops.conv_lokr_operands(f, dev) is None for kind, _s, f, _src in terms)
                bias_act = bias.to(act)

                def two_step(conv):
                    return conv._conv_forward(x, two_step_weight(ops, dq, conv.weight, act, ents), bias_act)
                route = {}
                real = {n: getattr(lib.lib(), n) for n in ("ggufb200_dequant_patched", "ggufb200_dequant_kron")}
                for n, fn in real.items():
                    setattr(lib.lib(), n, lambda *a, _fn=fn, _n=n: route.setdefault("name", _n) and _fn(*a))
                try:
                    patched[0](x)
                finally:
                    for n, fn in real.items():
                        setattr(lib.lib(), n, fn)
                ms_layer = graph_time(lambda: rotate(patched)(x), args.iters)
                y_layer = patched[0](x).float()
                ms_two = graph_time(lambda: two_step(rotate(plain)), args.iters)
                y_two = two_step(plain[0]).float()
                row = {"qtype": qname, "shape": list(shape), "x": list(xshape), "adapter": name, "route": route.get("name", "two_step"),
                       "reference_skips": skips, "ms_two_step": round(ms_two, 5), "ms_layer": round(ms_layer, 5),
                       "ms_unpatched": round(ms_plain, 5), "rel_layer": float((y_layer - y_two).norm() / y_two.norm())}
                if not skips:
                    keeps = [ops.conv_lycoris_operands(terms, dev) for _ in raws]
                    pure = all(kind == "lokr" for kind, *_t in terms)
                    kron = ([(ops.conv_lokr_operands(f, dev), s) for _k, s, f, _src in terms] if pure else None)

                    def run(conv, entry_point):
                        i = state["i"]
                        W = torch.empty(shape, dtype=act, device=dev)
                        raw = conv.weight.as_subclass(torch.Tensor)
                        if entry_point == "patched":
                            _keep, descs = keeps[i]
                            rc = lib.lib().ggufb200_dequant_patched(int(qt), raw.data_ptr(), N, K, W.data_ptr(), dq.dtype_code(act),
                                                                    dq.math_code(None, act), descs, len(terms),
                                                                    torch.cuda.current_stream().cuda_stream)
                        else:
                            descs = (lib.KronPatch * len(kron))(*[lib.KronPatch(A.data_ptr(), B.data_ptr(), A.shape[0], A.shape[1],
                                                                                B.shape[0], B.shape[1], -1, s, 0, 0)
                                                                  for (A, B), s in kron])
                            rc = lib.lib().ggufb200_dequant_kron(int(qt), raw.data_ptr(), N, K, W.data_ptr(), dq.dtype_code(act),
                                                                 dq.math_code(None, act) | lib.DEQUANT_SRC_STABLE, descs, len(kron),
                                                                 torch.cuda.current_stream().cuda_stream)
                        lib.check(rc, entry_point)
                        return conv._conv_forward(x, W, bias_act)
                    ms_new = graph_time(lambda: run(rotate(patched), "patched"), args.iters)
                    state["i"] = 0
                    row.update(ms_new=round(ms_new, 5), speedup_new=round(ms_two / ms_new, 3),
                               rel_new=float((run(patched[0], "patched").float() - y_two).norm() / y_two.norm()))
                    if pure:
                        ms_kron = graph_time(lambda: run(rotate(patched), "kron"), args.iters)
                        state["i"] = 0
                        row.update(ms_kron=round(ms_kron, 5), speedup_kron=round(ms_two / ms_kron, 3),
                                   rel_kron=float((run(patched[0], "kron").float() - y_two).norm() / y_two.norm()))
                rows.append(row)
                print(json.dumps(row), flush=True)
                del patched
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "act": args.act, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
