#!/usr/bin/env python
"""Generate the golden vectors of a STRADDLED Linear weight from the UNMODIFIED reference.

Run in the build container only (needs /root/reference, which does not exist on
the GPU box):   python tests/golden/make_golden_straddled.py

For SD1.5 / SDXL the GGUF converter reshapes every tensor whose last dimension is not a
multiple of 256 to [n / 256, 256] before quantising, and records the logical shape in
`comfy.gguf.orig_shape.<key>`.  A K-quant Linear [N, K] with K % 256 != 0 is then a flat
stream of N * K / 256 super-blocks, and its rows start inside blocks.  The reference loader
builds a GGMLTensor of those bytes ([N * K / 256, type_size]) with tensor_shape = (N, K);
this script runs the reference's `GGMLOps.Linear.forward` on exactly that (CPU, through
tests/fake_comfy) and writes

  linear_straddled_<QTYPE>_<act>.npz   x / packed stream / F32 bias / y, act = bf16 or f16

The golden files of make_golden.py are not touched.
"""
import os
import sys

import numpy as np
import torch
import gguf

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (reference loader, bit helper, seeded block generator)

T = gguf.GGMLQuantizationType


def make_linear_straddled(refops):
    GGMLTensor, GGMLOps = refops.GGMLTensor, refops.GGMLOps
    N, K, M = 200, 640, 24                      # K of SDXL's 640-wide projections; odd rows start mid-block
    for qt in (T.Q4_K, T.Q6_K):
        bs, ts = gguf.GGML_QUANT_SIZES[qt]
        assert K % bs != 0 and N * K % bs == 0
        raw = make_golden.oracle.random_blocks(int(qt), N * K // bs, seed=4000 + int(qt), scale=0.02)   # [N*K/256, ts]
        rng = np.random.default_rng(5000 + int(qt))
        bias = rng.normal(0, 0.02, size=N).astype(np.float32)
        x32 = rng.normal(0, 1, size=(M, K)).astype(np.float32)
        for act, name in ((torch.bfloat16, "bf16"), (torch.float16, "f16")):
            lin = GGMLOps.Linear(K, N)
            sd = {
                "weight": GGMLTensor(torch.from_numpy(raw.copy()), tensor_type=qt, tensor_shape=torch.Size((N, K))),
                "bias": GGMLTensor(torch.from_numpy(bias.copy()), tensor_type=T.F32, tensor_shape=torch.Size((N,))),
            }
            lin.load_state_dict(sd)
            x = torch.from_numpy(x32).to(act)
            with torch.no_grad():
                y = lin(x)
            assert type(y) is torch.Tensor and y.dtype == act and tuple(y.shape) == (M, N)
            np.savez_compressed(
                os.path.join(HERE, f"linear_straddled_{qt.name}_{name}.npz"),
                packed=raw.reshape(-1), qtype=np.int32(int(qt)), N=np.int64(N), K=np.int64(K), M=np.int64(M),
                bias=bias, x=make_golden.bits(x), y=make_golden.bits(y))
        print("wrote straddled linear", qt.name)


if __name__ == "__main__":
    torch.manual_seed(0)
    make_linear_straddled(make_golden.load_ref_ops())
