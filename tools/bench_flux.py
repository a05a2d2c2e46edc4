#!/usr/bin/env python
"""Flux.1-dev-shape Q4_K_S denoise step (1024x1024: 4096 img + 512 txt tokens, bf16, batch 1): this repo's GGMLOps vs the
reference's torch-GPU chain (restated in oracle/torch_chain.py) on the same packed weights, same process, CUDA events.
Prints one JSON object."""
import argparse
import json
import os
import sys

import numpy as np
import torch

if os.environ.get("GGUFB200_DEBUG_HANG"):           # diagnostics: dump every thread's Python stack after N seconds
    import faulthandler
    faulthandler.dump_traceback_later(int(os.environ["GGUFB200_DEBUG_HANG"]), exit=False)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
import flux_harness as fh  # noqa: E402


def time_steps(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


class LinearTimer:
    """CUDA-event pairs around every quantised GGMLOps.Linear forward of one step: GPU time spent inside the Linear layers
    (kernels + the launch gaps between a layer's own kernels) -- `linear_ms`; the rest of the step is `other_ms`."""

    def __init__(self, ops_mod):
        self.cls = ops_mod.GGMLOps.Linear
        self.pairs = []

    def __enter__(self):
        orig = self.cls.forward_ggml_cast_weights
        pairs = self.pairs

        def timed(mod, x):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            y = orig(mod, x)
            b.record()
            pairs.append((a, b))
            return y
        self.orig = orig
        self.cls.forward_ggml_cast_weights = timed
        return self

    def __exit__(self, *exc):
        self.cls.forward_ggml_cast_weights = self.orig

    def total_ms(self):
        torch.cuda.synchronize()
        return float(sum(a.elapsed_time(b) for a, b in self.pairs)), len(self.pairs)


ROUTE_NAMES = {"exact": "fused dequant -> shared memory -> wgmma (gemm4), reference-sequence producers: weight operand bit-identical to the reference's",
               "fast": "fused dequant -> shared memory -> wgmma (gemm4), fused-multiply-add producers; M <= 8: integer-pattern mma.sync kernel (gemv2)"}


def run(depth=19, depth_single=38, steps=10, warmup=3, ref_steps=3, txt_tokens=512, img_tokens=4096, device="cuda:0", numerics="exact",
        block_qtype="Q4_K", batch=1, lora_rank=0, lora_in_kernel=False):
    ops_mod, lib = ge._sub("ops"), ge._sub("_lib")
    ops_mod.GGMLOps.Linear.linear_numerics = numerics
    dev = torch.device(device)
    qt = fh.Q[block_qtype]
    with torch.no_grad():
        ours = fh.FluxShapeDiT(ops_mod.GGMLOps, depth=depth, depth_single=depth_single)
        ref = fh.FluxShapeDiT(fh.RefChainOps, depth=depth, depth_single=depth_single)
        sd = fh.build_state_dict(ours, ops_mod.GGMLTensor, dev, block_qtype=qt)
        fh.load_shared(ours, sd)
        fh.load_shared(ref, sd)
        ours.to(dev)
        ref.to(dev)
        inp = fh.make_inputs(dev, torch.bfloat16, batch=batch, img_tokens=img_tokens, txt_tokens=txt_tokens)
        packed_bytes = sum(v.numel() * v.element_size() for k, v in sd.items() if k.endswith("weight"))
        y_ours = ours(**inp)
        y_ref = ref(**inp)
        torch.cuda.synchronize()
        rel = float(((y_ours.float() - y_ref.float()).norm() / y_ref.float().norm()).item())
        finite = bool(torch.isfinite(y_ours).all().item())
        ms_ours, min_ours = time_steps(lambda: ours(**inp), steps, warmup)
        ms_ref, min_ref = time_steps(lambda: ref(**inp), ref_steps, 1) if ref_steps > 0 else (None, None)
        with LinearTimer(ops_mod) as lt:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            ours(**inp)
            b.record()
            linear_ms, n_linear = lt.total_ms()
            timed_step_ms = a.elapsed_time(b)
        lora = None
        if lora_rank > 0:
            # a rank-R LoRA patch on every quantised Linear (the patch-list format of ops.py:171-190 / nodes.py:43-47): timed through the same
            # GGMLOps.Linear forward, in-kernel (one extra k-block of the fused kernel) -- `in_kernel` -- and as two side GEMMs -- `side_gemms`
            g = torch.Generator().manual_seed(7)
            n_patched = 0
            for mod in ours.modules():
                if isinstance(mod, ops_mod.GGMLOps.Linear) and ops_mod.is_quantized(mod.weight):
                    N, K = mod.weight.tensor_shape
                    up = (torch.randn(N, lora_rank, generator=g) * 0.02).to(dev, torch.bfloat16)
                    down = (torch.randn(lora_rank, K, generator=g) * 0.02).to(dev, torch.bfloat16)
                    mod.weight.patches = [([(0.8, ("lora", (up, down, float(lora_rank), None, None, None)), 1.0, None, None)], "w")]
                    n_patched += 1
            print(f"lora: {n_patched} Linears patched", file=sys.stderr, flush=True)
            # fallback route first: the unpatched fused kernel + two side GEMMs of rank R (GGMLOps.Linear.lora_in_kernel = False)
            ops_mod.GGMLOps.Linear.lora_in_kernel = False
            y_s = ours(**inp)
            ms_side, _ = time_steps(lambda: ours(**inp), steps, warmup)
            print("lora: side-GEMM timing done", file=sys.stderr, flush=True)
            lora = {"rank": lora_rank, "patched_linears": n_patched, "ms_per_step_side_gemms": ms_side, "side_gemms_over_unpatched": ms_side / ms_ours,
                    "output_rel_diff_vs_unpatched": float(((y_s.float() - y_ours.float()).norm() / y_ours.float().norm()).item())}
            if lora_in_kernel:
                # default route (one extra k-block of the fused kernel); GGUFB200_LORA_NOSYNC=1 queues the forwards without a synchronise
                ops_mod.GGMLOps.Linear.lora_in_kernel = True
                nosync = bool(os.environ.get("GGUFB200_LORA_NOSYNC"))             # diagnostics of the intermittent hang
                if os.environ.get("GGUFB200_LORA_T_TORCH"):                        # diagnostics: T = x * down^T by the library GEMM
                    ops_mod.linear_dense = lambda x, w, b=None: torch.nn.functional.linear(x, w.to(x.dtype), None if b is None else b.to(x.dtype))
                try:
                    def fwd_sync():
                        y = ours(**inp)
                        if not nosync:
                            torch.cuda.synchronize()
                        return y
                    y_l = fwd_sync()
                    ms_in, _ = time_steps(fwd_sync, steps, warmup)
                finally:
                    pass
                lora.update({"ms_per_step_in_kernel": ms_in, "in_kernel_over_unpatched": ms_in / ms_ours,
                             "output_rel_diff_in_kernel_vs_side_gemms": float(((y_l.float() - y_s.float()).norm() / y_s.float().norm()).item())})
            ops_mod.GGMLOps.Linear.lora_in_kernel = True
            for mod in ours.modules():
                if isinstance(mod, ops_mod.GGMLOps.Linear) and ops_mod.is_quantized(mod.weight):
                    mod.weight.patches = []
    flops = fh.linear_flops(ours, img_tokens, txt_tokens, batch)
    return {
        "workload": f"Flux.1-dev-shape DiT ({depth} double + {depth_single} single blocks), block Linears {block_qtype}, others BF16, "
                    f"{img_tokens} img + {txt_tokens} txt tokens, bf16 activations, batch {batch}, random-init",
        "ms_per_step": ms_ours, "min_ms": min_ours, "steps": steps,
        "reference_chain_ms_per_step": ms_ref, "reference_chain_min_ms": min_ref,
        "speedup_vs_reference_chain": (ms_ref / ms_ours) if ms_ref else None,
        "linear_tflops_per_step": flops / 1e12, "linear_tflops_rate": flops / (ms_ours * 1e-3) / 1e12,
        "packed_weight_gb": packed_bytes / 1e9, "output_rel_err_vs_reference_chain": rel, "output_finite": finite,
        "linear_ms": linear_ms, "other_ms": timed_step_ms - linear_ms, "instrumented_step_ms": timed_step_ms, "quantised_linear_calls": n_linear,
        "linear_tflops_rate_inside_linears": flops / (linear_ms * 1e-3) / 1e12,
        "numerics": numerics, "large_m_route": ROUTE_NAMES[numerics], "lora": lora,
    }


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=19)
    ap.add_argument("--depth-single", type=int, default=38)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--ref-steps", type=int, default=3)
    ap.add_argument("--txt", type=int, default=512)
    ap.add_argument("--numerics", default="exact", choices=["fast", "exact"])
    ap.add_argument("--qtype", default="Q4_K")
    ap.add_argument("--lora", type=int, default=0, help="also time the step with a rank-R LoRA on every quantised Linear")
    ap.add_argument("--lora-in-kernel", action="store_true", help="also time the opt-in in-kernel LoRA route (synchronised forwards)")
    a = ap.parse_args()
    print(json.dumps(run(a.depth, a.depth_single, a.steps, 3, a.ref_steps, a.txt, numerics=a.numerics, block_qtype=a.qtype, lora_rank=a.lora, lora_in_kernel=a.lora_in_kernel)))
