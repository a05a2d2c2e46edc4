"""CPU tests of the packed Linear's backward surface: the ggufb200_linear_grad_input prototypes and constants, its argument
validation (all of it runs before a device is touched), the set of types it serves and the layer's grad predicate."""
import os
import re

import gguf
import pytest
import torch

from fallback_cases import FALLBACK
from util import ALL_QTYPES, Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "ggufb200.h")).read()


def test_header_prototypes_and_constants(pkg):
    flat = " ".join(HEADER.split())
    assert ("size_t ggufb200_linear_grad_input_workspace(int ggml_type, int64_t N, int64_t K, int act_dtype);" in flat)
    assert ("int ggufb200_linear_grad_input(int ggml_type, const void *W_packed, int64_t N, int64_t K, const void *dY, int64_t M, "
            "int64_t ldy, int act_dtype, int math_dtype, void *dX, int64_t ldx, void *workspace, size_t workspace_bytes, int flags, "
            "void *stream);") in flat
    op = re.search(r"^#define GGUFB200_OP_LINEAR_GRAD (\d+)", HEADER, re.M)
    assert op and int(op.group(1)) == pkg.lib.OP_LINEAR_GRAD
    ops = [int(v) for v in re.findall(r"^#define GGUFB200_OP_\w+ (\d+)", HEADER, re.M)]
    assert len(ops) == len(set(ops))
    assert {"ggufb200_linear_grad_input", "ggufb200_linear_grad_input_workspace"} <= set(pkg.lib.EXPORTS)


def test_supported_types(pkg):
    L = pkg.lib.lib()
    served = {int(q) for q in Q if L.ggufb200_supported(int(q), pkg.lib.OP_LINEAR_GRAD)}
    assert served == {int(q) for q in ALL_QTYPES} | {int(q) for q in FALLBACK}


def test_workspace_query(pkg):
    L = pkg.lib.lib()
    assert L.ggufb200_linear_grad_input_workspace(int(Q.Q4_K), 3072, 12288, 1) == 3072 * 12288 * 2
    assert L.ggufb200_linear_grad_input_workspace(int(Q.IQ2_XS), 256, 512, 0) == 256 * 512 * 2
    assert L.ggufb200_linear_grad_input_workspace(int(Q.BF16), 256, 512, 1) == 0         # the bytes are the operand
    assert L.ggufb200_linear_grad_input_workspace(int(Q.BF16), 256, 512, 0) == 256 * 512 * 2
    assert L.ggufb200_linear_grad_input_workspace(int(Q.F16), 256, 512, 0) == 0
    assert L.ggufb200_linear_grad_input_workspace(int(Q.Q4_K), 0, 512, 0) == 0


def _call(L, qt=Q.Q4_K, W=16, N=256, K=512, dY=4096, M=4, ldy=256, act=0, math=0, dX=8192, ldx=512, ws=1 << 20, ws_bytes=256 * 512 * 2,
          flags=0):
    return L.ggufb200_linear_grad_input(int(qt), W, N, K, dY, M, ldy, act, math, dX, ldx, ws, ws_bytes, flags, None)


def test_argument_validation_without_gpu(pkg):
    L = pkg.lib.lib()
    assert _call(L, qt=Q.F16) == -1 and _call(L, qt=99) == -1
    assert _call(L, act=2) == -2 and _call(L, math=3) == -2
    assert _call(L, flags=pkg.lib.FLAG_EXACT_W) == -8 and _call(L, flags=pkg.lib.FLAG_NOSPLIT) == -8
    assert _call(L, K=500, ldx=512) == -4                     # K % 8
    assert _call(L, K=320, ldx=320, N=257) == -4              # Q4_K rows of 320 elements that are not a straddled stream
    assert _call(L, ldy=255) == -4 and _call(L, ldx=511) == -4 and _call(L, M=-1) == -4 and _call(L, N=0) == -4
    assert _call(L, qt=Q.IQ2_XS, N=3, K=8, ldy=8, ldx=8) == -4   # N * K not a whole number of 256-element blocks
    assert _call(L, M=0, W=None, dY=None, dX=None) == 0       # nothing to do
    assert _call(L, W=None) == -5 and _call(L, dY=None) == -5 and _call(L, dX=None) == -5
    assert _call(L, dY=4098) == -3 and _call(L, dX=8200) == -3 and _call(L, ldy=260) == -3 and _call(L, ldx=516) == -3
    assert _call(L, ws=None) == -7 and _call(L, ws_bytes=256 * 512 * 2 - 16) == -7
    assert _call(L, ws=(1 << 20) + 8) == -3
    assert _call(L, qt=Q.BF16, act=1, W=18, ws=None, ws_bytes=0) == -3    # BF16 read in place: 16-byte aligned rows


def test_grad_predicate(pkg):
    ops = pkg.ops
    x = torch.randn(2, 8)
    w = ops.GGMLTensor(torch.zeros(8, dtype=torch.uint8), tensor_type=Q.Q8_0, tensor_shape=torch.Size((8, 8)))
    assert not ops.grad_needed(x, w)
    assert ops.grad_needed(x.clone().requires_grad_(True), w)
    with torch.no_grad():
        assert not ops.grad_needed(x.clone().requires_grad_(True), w)
    up, down = torch.randn(8, 2), torch.randn(2, 8)
    w.patches = [([(1.0, ("lora", (up, down, None)), 1.0, None, None)], "k")]
    assert not ops.grad_needed(x, w)
    up.requires_grad_(True)
    assert ops.grad_needed(x, w)

    class LoRAAdapter:
        def __init__(self, weights):
            self.weights = weights
    w.patches = [([(1.0, LoRAAdapter((torch.randn(8, 2), torch.randn(2, 8).requires_grad_(True), None)), 1.0, None, None)], "k")]
    assert ops.grad_needed(x, w)
    with torch.no_grad():
        assert not ops.grad_needed(x, w)
