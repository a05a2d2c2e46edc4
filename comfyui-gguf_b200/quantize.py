"""Dense tensor -> packed GGUF blocks on the GPU: the inverse of dequant.py, used by convert.py to write GGUF files.

`quantize_tensor(t, qtype)` is ONE launch of csrc/quantize.cu through the C ABI (`ggufb200_quantize`).  Its bytes are
bit-identical to gguf-py's `gguf.quants.quantize(t.float().numpy(), qtype)` for every finite input, for the types gguf-py can
quantise itself: Q8_0, Q5_1, Q5_0, Q4_1, Q4_0 and BF16.  Nothing is computed on the CPU: without a CUDA tensor it raises
NotImplementedError, as dequant.py does for a type it has no kernel for.

`quantize_k_tensor(t, qtype)` is the same for the K types Q2_K ... Q6_K, through `ggufb200_quantize_k`.  Its encoders restate
llama.cpp's reference quantisers at tag b3962 without an importance matrix (what `llama-quantize` runs without --imatrix); the
bytes equal a plain-C restatement of that code bit for bit.  Parity with a llama-quantize binary is not verified: see DESIGN.md.
"""
from __future__ import annotations

import gguf
import torch

from . import _lib
from .dequant import _stream_ptr, dtype_code

_Q = gguf.GGMLQuantizationType
QUANTIZE_QTYPES = (_Q.BF16, _Q.Q8_0, _Q.Q5_1, _Q.Q5_0, _Q.Q4_1, _Q.Q4_0)
KQUANT_QTYPES = (_Q.Q6_K, _Q.Q5_K, _Q.Q4_K, _Q.Q3_K, _Q.Q2_K)


def quantize_tensor(t: torch.Tensor, qtype) -> torch.Tensor:
    """t [..., K] (fp32 / fp16 / bf16, on a CUDA device) -> uint8 [..., K / block_size * type_size] on t's device: the GGUF
    bytes of `qtype`, row by row.  K must be a multiple of the block size, as gguf-py requires: 32 for the Q types, any K for
    BF16 (ValueError otherwise).  The Q types refuse non-finite input (ValueError); BF16 converts it as gguf-py does."""
    qtype = _Q(qtype)
    if qtype not in QUANTIZE_QTYPES:
        raise NotImplementedError(f"ggufb200: no quantiser for qtype {qtype.name!r} (only {', '.join(q.name for q in QUANTIZE_QTYPES)})")
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise NotImplementedError("ggufb200: quantize_tensor needs a CUDA tensor; this package has no CPU quantiser")
    src_code = dtype_code(t.dtype)
    block_size, type_size = gguf.GGML_QUANT_SIZES[qtype]
    if t.dim() == 0 or t.shape[-1] % block_size != 0:
        raise ValueError(f"quantize_tensor: the last dimension of shape {tuple(t.shape)} must be a multiple of {block_size} for {qtype.name}")
    if qtype != _Q.BF16 and not bool(torch.isfinite(t).all()):
        raise ValueError(f"quantize_tensor: {qtype.name} input must be finite (the tensor holds NaN or Inf)")
    src = t.contiguous()
    n_blocks = src.numel() // block_size
    out = torch.empty(*src.shape[:-1], src.shape[-1] // block_size * type_size, dtype=torch.uint8, device=src.device)
    if n_blocks == 0:
        return out
    with torch.cuda.device(src.device):
        rc = _lib.lib().ggufb200_quantize(int(qtype), src.data_ptr(), src_code, n_blocks, out.data_ptr(), 0, _stream_ptr(src.device))
    _lib.check(rc, f"ggufb200_quantize({qtype.name})")
    return out


def quantize_k_tensor(t: torch.Tensor, qtype) -> torch.Tensor:
    """t [..., K] (fp32 / fp16 / bf16, on a CUDA device) -> uint8 [..., K / 256 * type_size] on t's device: the K-quant bytes of
    `qtype` (one of KQUANT_QTYPES), row by row, in one launch.  K must be a multiple of 256 (ValueError otherwise) and the input
    finite (ValueError otherwise)."""
    qtype = _Q(qtype)
    if qtype not in KQUANT_QTYPES:
        raise NotImplementedError(f"ggufb200: no K-quant encoder for qtype {qtype.name!r} (only {', '.join(q.name for q in KQUANT_QTYPES)})")
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise NotImplementedError("ggufb200: quantize_k_tensor needs a CUDA tensor; this package has no CPU quantiser")
    src_code = dtype_code(t.dtype)
    block_size, type_size = gguf.GGML_QUANT_SIZES[qtype]
    if t.dim() == 0 or t.shape[-1] % block_size != 0:
        raise ValueError(f"quantize_k_tensor: the last dimension of shape {tuple(t.shape)} must be a multiple of {block_size} for {qtype.name}")
    if not bool(torch.isfinite(t).all()):
        raise ValueError(f"quantize_k_tensor: {qtype.name} input must be finite (the tensor holds NaN or Inf)")
    src = t.contiguous()
    n_blocks = src.numel() // block_size
    out = torch.empty(*src.shape[:-1], src.shape[-1] // block_size * type_size, dtype=torch.uint8, device=src.device)
    if n_blocks == 0:
        return out
    with torch.cuda.device(src.device):
        rc = _lib.lib().ggufb200_quantize_k(int(qtype), src.data_ptr(), src_code, n_blocks, out.data_ptr(), 0, _stream_ptr(src.device))
    _lib.check(rc, f"ggufb200_quantize_k({qtype.name})")
    return out
