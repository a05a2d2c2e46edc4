"""CPU test: oracle/torch_chain.py reproduces the reference's torch path bit-for-bit and with the same number of
materialising ATen kernels, so that timing it on a GPU is a fair stand-in for the reference.  What the unmodified reference
computed (the SHA-256 of its bytes, and how many kernels it ran) is stored in tests/golden/torch_chain.json
(tests/golden/make_golden.py)."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch
import gguf
from torch.utils._python_dispatch import TorchDispatchMode

import oracle
from oracle import torch_chain

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "torch_chain.json")
Q = gguf.GGMLQuantizationType
MATH_NAMES = {None: "none", torch.float32: "float32", torch.bfloat16: "bfloat16"}


class Count(TorchDispatchMode):
    VIEWS = ("view", "reshape", "split", "unsqueeze", "expand", "_unsafe_view", "alias", "detach", "select", "slice", "squeeze",
             "permute", "transpose", "t.default", "split_with_sizes", "_reshape_alias", "lift_fresh")

    def __init__(self):
        super().__init__()
        self.n = 0

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        name = str(func)
        if not any(v in name for v in self.VIEWS):
            self.n += 1
        return func(*args, **(kwargs or {}))


@pytest.mark.parametrize("qt", [Q.Q8_0, Q.Q4_0, Q.Q4_K, Q.Q5_K, Q.Q6_K, Q.BF16], ids=lambda q: q.name)
@pytest.mark.parametrize("md", [None, torch.float32, torch.bfloat16])
def test_chain_equals_reference(qt, md):
    want = json.load(open(GOLDEN))[f"{qt.name}_{MATH_NAMES[md]}"]
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    raw = torch.from_numpy(oracle.random_blocks(int(qt), 96, seed=1)).reshape(-1)
    shape = (96 * bs,)
    with Count() as c_mine:
        b = torch_chain.dequantize(raw, qt, shape, dtype=md)
    got = b.contiguous().view(torch.uint8).numpy()
    assert str(b.dtype) == want["dtype"] and got.size == want["nbytes"]
    assert hashlib.sha256(got.tobytes()).hexdigest() == want["sha256"]
    assert want["kernels"] == c_mine.n, (want["kernels"], c_mine.n)
