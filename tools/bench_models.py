#!/usr/bin/env python
"""BASELINE configs[3]: SD3.5-large-SHAPE MMDiT (hidden 2432, 38 joint blocks, Q8_0) one denoise step and T5-v1.1-xxl-SHAPE
encoder (24 layers, d_model 4096, d_ff 10240, Q5_K, 512 tokens, quantised Embedding through the row-gather kernel),
this repo's ops vs the reference's torch chain on the same packed weights.  Prints one JSON object per model."""
import json
import os
import sys

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
import flux_harness as fh  # noqa: E402
from bench_flux import time_steps  # noqa: E402


class T5Layer(nn.Module):
    def __init__(self, ops, d=4096, ff=10240, heads=64):
        super().__init__()
        self.heads = heads
        self.q, self.k, self.v, self.o = (ops.Linear(d, d, bias=False) for _ in range(4))
        self.wi_0, self.wi_1, self.wo = ops.Linear(d, ff, bias=False), ops.Linear(d, ff, bias=False), ops.Linear(ff, d, bias=False)
        self.register_buffer("n1", torch.ones(d), persistent=False)
        self.register_buffer("n2", torch.ones(d), persistent=False)

    def forward(self, x):
        B, L, D = x.shape
        h = F.rms_norm(x, (D,), self.n1.to(x.dtype), 1e-6)
        q, k, v = (m(h).view(B, L, self.heads, -1).transpose(1, 2) for m in (self.q, self.k, self.v))
        x = x + self.o(F.scaled_dot_product_attention(q, k, v).transpose(1, 2).flatten(2))
        h = F.rms_norm(x, (D,), self.n2.to(x.dtype), 1e-6)
        return x + self.wo(F.gelu(self.wi_0(h), approximate="tanh") * self.wi_1(h))


class T5ShapeEncoder(nn.Module):
    def __init__(self, ops, layers=24, vocab=32128, d=4096):
        super().__init__()
        self.ops_has_embedding = hasattr(ops, "Embedding")
        self.vocab, self.d = vocab, d
        self.shared = ops.Embedding(vocab, d, device="meta") if self.ops_has_embedding else None
        self.layers = nn.ModuleList([T5Layer(ops, d) for _ in range(layers)])

    def forward(self, ids, table=None):
        if self.shared is not None and table is None:
            x = self.shared(ids, out_dtype=torch.bfloat16)
        else:   # reference arm: dequantise the WHOLE table, then gather (ops.py:251-259)
            from oracle import torch_chain
            w = torch_chain.dequantize_tensor(table.as_subclass(torch.Tensor), int(table.tensor_type), tuple(table.tensor_shape), torch.bfloat16)
            x = F.embedding(ids, w)
        for layer in self.layers:
            x = layer(x)
        return x


def build_sd(model, GGMLTensor, dev, qt, bias, seed=0, scale=2e-4):
    gen = torch.Generator(device=dev).manual_seed(seed)
    sd = {}
    for name, mod in model.named_modules():
        if hasattr(mod, "in_features"):
            N, K = mod.out_features, mod.in_features
            sd[f"{name}.weight"] = GGMLTensor(fh.random_packed(qt, N, K, dev, gen, scale=scale), tensor_type=qt, tensor_shape=torch.Size((N, K)))
            if bias:
                sd[f"{name}.bias"] = GGMLTensor(torch.randn(N, device=dev, generator=gen) * 0.02, tensor_type=fh.Q.F32, tensor_shape=torch.Size((N,)))
    return sd


def attach(model, sd):
    for name, mod in model.named_modules():
        if hasattr(mod, "in_features"):
            mod.weight = nn.Parameter(sd[f"{name}.weight"], requires_grad=False)
            mod.bias = nn.Parameter(sd[f"{name}.bias"], requires_grad=False) if f"{name}.bias" in sd else None
    return model


def run_t5(steps=6, ref_steps=2, layers=24, tokens=512):
    ops_mod = ge._sub("ops")
    dev = torch.device("cuda:0")
    with torch.no_grad():
        ours, ref = T5ShapeEncoder(ops_mod.GGMLOps, layers), T5ShapeEncoder(fh.RefChainOps, layers)
        sd = build_sd(ours, ops_mod.GGMLTensor, dev, fh.Q.Q5_K, bias=False, scale=5e-5)   # keeps the residual stream finite
        gen = torch.Generator(device=dev).manual_seed(5)
        table = ops_mod.GGMLTensor(fh.random_packed(fh.Q.Q5_K, 32128, 4096, dev, gen, scale=1e-3), tensor_type=fh.Q.Q5_K, tensor_shape=torch.Size((32128, 4096)))
        ours.shared.weight = nn.Parameter(table, requires_grad=False)
        attach(ours, sd).to(dev)
        attach(ref, sd).to(dev)
        ids = torch.randint(0, 32128, (1, tokens), device=dev)
        a, b = ours(ids), ref(ids, table)
        rel = float(((a.float() - b.float()).norm() / b.float().norm()).item())
        print("t5 out stats: |b|max", float(b.float().abs().max()), "max|a-b|", float((a.float() - b.float()).abs().max()), "finite", bool(torch.isfinite(a).all()), file=sys.stderr)
        ms, _ = time_steps(lambda: ours(ids), steps, 2)
        ms_ref, _ = time_steps(lambda: ref(ids, table), ref_steps, 1)
    return {"workload": f"T5-v1.1-xxl-shape encoder, {layers} layers, Q5_K Linears + Q5_K embedding table [32128,4096], {tokens} tokens, bf16",
            "ms_per_encode": ms, "reference_chain_ms": ms_ref, "speedup_vs_reference_chain": ms_ref / ms, "output_rel_err_vs_reference_chain": rel}


def run_sd35(steps=6, ref_steps=2, depth=38, img_tokens=4096, txt_tokens=333):
    ops_mod = ge._sub("ops")
    dev = torch.device("cuda:0")
    with torch.no_grad():
        kw = dict(hidden=2432, heads=38, depth=depth, depth_single=0, ctx=4096, vec=2048)
        ours, ref = fh.FluxShapeDiT(ops_mod.GGMLOps, **kw), fh.FluxShapeDiT(fh.RefChainOps, **kw)
        sd = fh.build_state_dict(ours, ops_mod.GGMLTensor, dev, block_qtype=fh.Q.Q8_0)
        fh.load_shared(ours, sd).to(dev)
        fh.load_shared(ref, sd).to(dev)
        inp = fh.make_inputs(dev, torch.bfloat16, img_tokens=img_tokens, txt_tokens=txt_tokens)
        inp["y"] = torch.randn(1, 2048, device=dev).to(torch.bfloat16)
        a, b = ours(**inp), ref(**inp)
        rel = float(((a.float() - b.float()).norm() / b.float().norm()).item())
        ms, _ = time_steps(lambda: ours(**inp), steps, 2)
        ms_ref, _ = time_steps(lambda: ref(**inp), ref_steps, 1)
    return {"workload": f"SD3.5-large-shape MMDiT ({depth} joint blocks, hidden 2432, 38 heads x 64), block Linears Q8_0, {img_tokens}+{txt_tokens} tokens, bf16",
            "ms_per_step": ms, "reference_chain_ms": ms_ref, "speedup_vs_reference_chain": ms_ref / ms, "output_rel_err_vs_reference_chain": rel}


def parity(which, numerics):
    """Per-Linear parity (tools/flux_harness.py::LinearParity) of a full-size model under one numerics contract."""
    ops_mod, dq = ge._sub("ops"), ge._sub("dequant")
    ops_mod.GGMLOps.Linear.linear_numerics = numerics
    dev = torch.device("cuda:0")
    with torch.no_grad():
        if which == "flux":
            model = fh.FluxShapeDiT(ops_mod.GGMLOps)
            fh.load_shared(model, fh.build_state_dict(model, ops_mod.GGMLTensor, dev)).to(dev)
            inp = fh.make_inputs(dev, torch.bfloat16)
            call = lambda: model(**inp)
        elif which == "sd35":
            kw = dict(hidden=2432, heads=38, depth=38, depth_single=0, ctx=4096, vec=2048)
            model = fh.FluxShapeDiT(ops_mod.GGMLOps, **kw)
            fh.load_shared(model, fh.build_state_dict(model, ops_mod.GGMLTensor, dev, block_qtype=fh.Q.Q8_0)).to(dev)
            inp = fh.make_inputs(dev, torch.bfloat16, img_tokens=4096, txt_tokens=333)
            inp["y"] = torch.randn(1, 2048, device=dev).to(torch.bfloat16)
            call = lambda: model(**inp)
        else:
            model = T5ShapeEncoder(ops_mod.GGMLOps, 24)
            sd = build_sd(model, ops_mod.GGMLTensor, dev, fh.Q.Q5_K, bias=False, scale=5e-5)
            gen = torch.Generator(device=dev).manual_seed(5)
            table = ops_mod.GGMLTensor(fh.random_packed(fh.Q.Q5_K, 32128, 4096, dev, gen, scale=1e-3), tensor_type=fh.Q.Q5_K, tensor_shape=torch.Size((32128, 4096)))
            model.shared.weight = nn.Parameter(table, requires_grad=False)
            attach(model, sd).to(dev)
            ids = torch.randint(0, 32128, (1, 512), device=dev)
            call = lambda: model(ids)
        with fh.LinearParity(model, dq) as lp:
            call()
        out = lp.summary()
    out.update(model=which, numerics=numerics, activation="bf16",
               budget="1e-3 (exact: weight operand bit-identical to the reference's)" if numerics == "exact" else
                      "8e-3 (fast, bf16 = 1e-3 in fp16 ulps)")
    del model
    torch.cuda.empty_cache()
    return out


if __name__ == "__main__":
    which = sys.argv[1:] or ["t5", "sd35"]
    if which[0] == "parity":
        for m in (which[1:] or ["flux", "sd35", "t5"]):
            for numerics in ("exact", "fast"):
                print(json.dumps(parity(m, numerics)), flush=True)
        sys.exit(0)
    if "t5" in which:
        print(json.dumps(run_t5()), flush=True)
    if "sd35" in which:
        print(json.dumps(run_sd35()), flush=True)
