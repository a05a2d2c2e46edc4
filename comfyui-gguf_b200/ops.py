"""Drop-in for the reference's ops.py -- the ComfyUI custom-operations surface, H100 kernels inside.

Mirrored surface (reference file:line):
    GGMLTensor      ops.py:44-91     tensor subclass carrying packed bytes + tensor_type/tensor_shape/patches
    GGMLLayer       ops.py:93-225    state-dict hooks, get_weight, cast_bias_weight, forward dispatch
    GGMLOps         ops.py:227-271   Linear / Conv2d / Embedding / LayerNorm / GroupNorm
    move_patch_to_device  ops.py:273-281

What changes underneath:
    * Linear.forward_ggml_cast_weights (ops.py:242-244) no longer materialises W through ~17 ATen kernels and
      then calls F.linear: it hands the PACKED weight to ggufb200_linear (fused dequant + GEMV / warpgroup-MMA GEMM).
      LoRA-patched weights, fp32 activations and CPU inputs take the two-step route (one dequant launch,
      then comfy.lora.calculate_weight / F.linear) so their semantics stay those of the reference.
    * get_weight (ops.py:166-191) dequantises with ONE kernel launch (dequant.py of this package).
    * Embedding (ops.py:251-259) gathers only the indexed rows instead of dequantising the whole table.
    * The packed-weight Linear is differentiable in its input like the reference's F.linear (`grad_needed`,
      PackedLinearFunction): the backward dequantises W again from the packed bytes (ggufb200_linear_grad_input) instead of
      keeping a dense W per layer between forward and backward; patch lists other than plain / banded LoRA, and patched
      Conv2d weights, take the two-step route while gradients are needed.
"""
from __future__ import annotations

import logging
import math

import gguf
import torch

from . import _lib
from ._host import comfy_lora, comfy_mm, comfy_ops
from .dequant import (FALLBACK_QTYPES, SUPPORTED_QTYPES, dequantize, dequantize_fallback, dequantize_rows, dequantize_tensor, dtype_code,
                      is_quantized, math_code)

_Q = gguf.GGMLQuantizationType
_FUSED_ACT = (torch.float16, torch.bfloat16)
GEMV_MAX_M = 8   # csrc/gemv.cu kGemvMaxM


def torch_compiler_disable(*_args, **_kwargs):
    """ops.py:21-42: on torch >= 2.8 the reference lets torch.compile trace through; the kernels here are
    reached through ctypes, which dynamo treats as an opaque call, so the guard is an identity decorator."""
    def wrap(fn):
        return fn
    return wrap


class GGMLTensor(torch.Tensor):
    """Packed GGUF payload as a tensor (ops.py:44-91).  `.shape` is the LOGICAL shape; `.size()` the byte shape."""

    def __new__(cls, data, *args, tensor_type, tensor_shape, patches=(), **kwargs):
        return torch.Tensor._make_subclass(cls, data, False)

    def __init__(self, data, *args, tensor_type, tensor_shape, patches=(), **kwargs):
        self.tensor_type = tensor_type
        self.tensor_shape = tensor_shape
        self.patches = list(patches)

    def _meta_onto(self, other):
        other.tensor_type = getattr(self, "tensor_type", None)
        other.tensor_shape = getattr(self, "tensor_shape", other.data.shape)
        other.patches = list(getattr(self, "patches", []))
        return other

    def to(self, *args, **kwargs):
        return self._meta_onto(super().to(*args, **kwargs))

    def clone(self, *args, **kwargs):
        return self  # nn.Parameter(GGMLTensor) must stay the same object (ops.py:64-68, 124)

    def detach(self, *args, **kwargs):
        return self

    def copy_(self, *args, **kwargs):
        try:
            return super().copy_(*args, **kwargs)
        except Exception as exc:  # ops.py:70-75: CLIP text models call weight.copy_ with logical shapes
            logging.warning(f"ignoring 'copy_' on tensor: {exc}")

    def new_empty(self, size, *args, **kwargs):
        fresh = super().new_empty(size, *args, **kwargs)
        return GGMLTensor(fresh, tensor_type=getattr(self, "tensor_type", None), tensor_shape=size,
                          patches=list(getattr(self, "patches", [])))

    @property
    def shape(self):
        if not hasattr(self, "tensor_shape"):
            self.tensor_shape = self.size()
        return self.tensor_shape


def move_patch_to_device(item, device):
    """ops.py:273-281."""
    if isinstance(item, torch.Tensor):
        return item.to(device, non_blocking=True)
    if isinstance(item, tuple):
        return tuple(move_patch_to_device(x, device) for x in item)
    if isinstance(item, list):
        return [move_patch_to_device(x, device) for x in item]
    return item


def _plain(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, GGMLTensor) else t


# Raw-handle accessors: `torch.cuda.current_stream()` builds a Stream object through three layers of Python (~5 us per
# call, more than the kernel launch it precedes); the private C entry points return the same values directly.
_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
_raw_device = getattr(torch._C, "_cuda_getDevice", None)


def _current_stream_ptr(index):
    if _raw_stream is not None:
        return _raw_stream(index)
    return torch.cuda.current_stream(index).cuda_stream


def _is_current_device(index):
    return index == (_raw_device() if _raw_device is not None else torch.cuda.current_device())


_F16_CODE = _lib.F16


def needs_span_layout(qtype, K):
    """True when the canonical GGUF rows cannot be staged by a 2-D tensor map (a row's 256-wide K-span or the row stride is
    not a multiple of 16 bytes): Q2_K / Q3_K / Q6_K / IQ4_XS always, the others for some K (Q8_0 at K = 2432).
    The answer holds for a straddled weight too (SD1.5 / SDXL K-quants at K % 256 != 0, whose 256-element blocks straddle
    rows): the kernel reads Q4_K / Q5_K from the canonical block stream and the other four from a block-major copy."""
    bs, ts = gguf.GGML_QUANT_SIZES[qtype]
    return bs > 1 and (((256 // bs) * ts) % 16 != 0 or ((K // bs) * ts) % 16 != 0)


def straddled_rows(qtype, K):
    """True for a weight whose 256-element blocks straddle rows (csrc/internal.h): K % 256 != 0 with a K-quant, the flat block
    stream the GGUF converter writes for SD1.5 / SDXL tensors.  The library serves it by dequant + GEMM unless a route is asked
    for (FUSED_TMEM, which the in-kernel LoRA takes)."""
    return gguf.GGML_QUANT_SIZES[qtype][0] == 256 and K % 256 != 0


def span_layout(weight, wraw):
    """The re-packed span-major copy of a device-resident packed weight (csrc/repack.cu, SURVEY 8f rank 3; block-major for a
    straddled weight), built once and
    cached ON the GGMLTensor object: `.to()` / reload create new tensor objects, so the cache can never outlive its bytes.
    The canonical bytes are untouched (state_dict / offload semantics stay the reference's)."""
    key = (wraw.data_ptr(), wraw._version)
    cached = weight.__dict__.get("_gg_spans")
    if cached is not None and cached[0] == key:
        return cached[1]
    qcode = int(weight.tensor_type)
    N, K = tuple(weight.tensor_shape)
    L = _lib.lib()
    nbytes = L.ggufb200_repack_bytes(qcode, N, K)
    out = torch.empty(nbytes, dtype=torch.uint8, device=wraw.device)
    with torch.cuda.device(wraw.device):
        _lib.check(L.ggufb200_repack(qcode, wraw.data_ptr(), N, K, out.data_ptr(), _current_stream_ptr(wraw.device.index)),
                   f"ggufb200_repack({weight.tensor_type.name}, N={N}, K={K})")
    weight.__dict__["_gg_spans"] = (key, out)
    return out


LORA_MAX_RANK = 64     # width of one LoRA k-block of the FUSED_TMEM kernel
LORA_KERNEL_MAX_RANK = 8 * LORA_MAX_RANK     # at most 8 LoRA k-blocks: a larger total rank takes the side GEMMs (`_add_lora`)
KRON_MAX_PATCHES = 8   # LoKr patches one ggufb200_dequant_kron call applies (csrc/internal.h kKronMaxPatches); more -> two-step route
# weight types and activation dtypes ggufb200_dequant_lowrank serves (every block format and numpy-fallback type but BF16)
_LOWRANK_QTYPES = tuple(q for q in SUPPORTED_QTYPES if q != _Q.BF16) + FALLBACK_QTYPES
_LOWRANK_ACT = (torch.float16, torch.bfloat16, torch.float32)
# `lowrank_pays` terms of the conv LyCORIS entries (microseconds, tools/bench_conv_lycoris.py): the kernel's Kronecker pass per
# tile wave; the two-step route's kron + scale + cast + add per LoKr entry (fixed + per million weight elements); the Tucker
# composition (LoCon mid's mm and transposed copy, LoHa's two einsums) the two-step route adds per Tucker entry
KRON_KERNEL_US, KRON_TWO_STEP_US, TUCKER_TWO_STEP_US = 1.5, (8.0, 10.0), 6.0
# `conv_dora_pays`: what weight_decompose's passes add to the two-step route per DoRA entry, net of the kernel's DoRA step (fixed,
# per million weight elements; microseconds, the lower envelope over both axes and strengths in tools/bench_conv_dora.py)
DORA_TWO_STEP_US = (9.0, 3.9)


def _launch_linear(x, wraw, qtype, N, K, bias, math, algo, spans=None, lora=None, scale=None):
    """The call itself.  x: CUDA fp16/bf16 [..., K]; wraw: PLAIN uint8 tensor holding the packed rows on x.device;
    bias: PLAIN tensor on x.device or None; scale (LoRA only): fp32 [N] feature scale of ggufb200_linear_lora_scaled.  Kept free of tensor-subclass traffic (every attribute read on a GGMLTensor
    goes through __torch_function__) and of per-call object construction: for short activations the host side of this
    function, not the GPU, bounds the layer."""
    x2 = x if x.dim() == 2 else x.reshape(-1, K)
    if x2.stride(-1) != 1 or (x2.stride(0) & 7) or (x2.data_ptr() & 15):
        x2 = x2.contiguous()
    M = x2.shape[0]
    device = x.device
    y = torch.empty((M, N), dtype=x.dtype, device=device)
    if not wraw.is_contiguous():
        wraw = wraw.contiguous()
    act = dtype_code(x.dtype)
    bias_ptr, bias_code = None, 0
    if bias is not None:
        if not bias.is_contiguous():
            bias = bias.contiguous()
        bias_ptr, bias_code = bias.data_ptr(), dtype_code(bias.dtype)
    w_ptr = wraw.data_ptr()
    if w_ptr & 15:
        algo = _lib.ALGO_DEQUANT_MMA | (algo & ~_lib.ALGO_MASK)   # byte-offset view: only the standalone dequant stages any alignment
    L = _lib.lib()
    qcode = int(qtype)
    ws, ws_ptr = None, None
    need = L.ggufb200_linear_workspace_ex(qcode, M, N, K, act, math, algo)     # same routing function as the call below
    if need:
        ws = torch.empty(need, dtype=torch.uint8, device=device)
        ws_ptr = ws.data_ptr()
    index = device.index
    if lora is not None:
        # T = x * down^T [M, 64 J] act dtype, U = scale * up [N, 64 J] fp16 (zero padded), per-tile k-block ranges or None
        t_pad, u_pad, tiles = lora
        J = u_pad.shape[1] // LORA_MAX_RANK
        if scale is not None:
            def call():
                return L.ggufb200_linear_lora_scaled(qcode, w_ptr, None if spans is None else spans.data_ptr(), N, K, x2.data_ptr(), M,
                                                     x2.stride(0), act, bias_ptr, bias_code, t_pad.data_ptr(), t_pad.stride(0), u_pad.data_ptr(),
                                                     u_pad.stride(0), J, None if tiles is None else tiles.data_ptr(), scale.data_ptr(),
                                                     y.data_ptr(), N, ws_ptr, need, algo, _current_stream_ptr(index))
        elif J == 1 and tiles is None:
            def call():
                return L.ggufb200_linear_lora(qcode, w_ptr, None if spans is None else spans.data_ptr(), N, K, x2.data_ptr(), M, x2.stride(0), act,
                                              bias_ptr, bias_code, t_pad.data_ptr(), t_pad.stride(0), u_pad.data_ptr(), y.data_ptr(), N, ws_ptr,
                                              need, algo, _current_stream_ptr(index))
        else:
            def call():
                return L.ggufb200_linear_lora_ex(qcode, w_ptr, None if spans is None else spans.data_ptr(), N, K, x2.data_ptr(), M, x2.stride(0),
                                                 act, bias_ptr, bias_code, t_pad.data_ptr(), t_pad.stride(0), u_pad.data_ptr(), u_pad.stride(0), J,
                                                 None if tiles is None else tiles.data_ptr(), y.data_ptr(), N, ws_ptr, need, algo,
                                                 _current_stream_ptr(index))
    elif spans is not None:
        def call():
            return L.ggufb200_linear_spans(qcode, w_ptr, spans.data_ptr(), N, K, x2.data_ptr(), M, x2.stride(0), act, math, bias_ptr, bias_code,
                                           y.data_ptr(), N, ws_ptr, need, algo, _current_stream_ptr(index))
    else:
        def call():
            return L.ggufb200_linear(qcode, w_ptr, N, K, x2.data_ptr(), M, x2.stride(0), act, math, bias_ptr, bias_code, y.data_ptr(), N,
                                     ws_ptr, need, algo, _current_stream_ptr(index))
    if _is_current_device(index):                     # the common case: no device-guard round trip
        rc = call()
    else:
        with torch.cuda.device(device):
            rc = call()
    if rc:
        _lib.check(rc, f"ggufb200_linear({getattr(qtype, 'name', qtype)}, M={M}, N={N}, K={K})")
    return y if x.dim() == 2 else y.reshape(*x.shape[:-1], N)


def linear_fallback(x, wraw, qtype, N, K, bias, algo=_lib.ALGO_AUTO | _lib.FLAG_W_STABLE):
    """y = x @ W.T + bias for a weight in one of FALLBACK_QTYPES (ggufb200_linear_fallback): W is gguf-py's fp32 value rounded
    once to x.dtype, decoded from the packed rows `wraw` (plain uint8 on x.device) inside the kernel, or dequantised into a
    workspace above AUTO's crossover M.  x: CUDA fp16/bf16 [..., K]; bias: PLAIN tensor on x.device or None.  W_STABLE: the
    packed weight is a parameter (or its host-to-device copy), never written by a kernel in flight."""
    x2 = x if x.dim() == 2 else x.reshape(-1, K)
    if x2.stride(-1) != 1 or (x2.stride(0) & 7) or (x2.data_ptr() & 15):
        x2 = x2.contiguous()
    M = x2.shape[0]
    device = x.device
    y = torch.empty((M, N), dtype=x.dtype, device=device)
    if not wraw.is_contiguous():
        wraw = wraw.contiguous()
    bias_ptr, bias_code = None, 0
    if bias is not None:
        if not bias.is_contiguous():
            bias = bias.contiguous()
        bias_ptr, bias_code = bias.data_ptr(), dtype_code(bias.dtype)
    L = _lib.lib()
    qcode, act = int(qtype), dtype_code(x.dtype)
    # the workspace query assumes a base aligned to the type's blocks (gcd(type_size, 16), fallback.cuh A_BLK); a byte-offset view
    # below that is read by the standalone dequant only, which the call then takes whatever `algo` says: ask for that route's size
    query_algo = algo
    if wraw.data_ptr() % math.gcd(gguf.GGML_QUANT_SIZES[qtype][1], 16):
        query_algo = _lib.ALGO_DEQUANT_MMA | (algo & ~_lib.ALGO_MASK)
    need = L.ggufb200_linear_fallback_workspace(qcode, M, N, K, act, query_algo)      # same routing function as the call below
    ws = torch.empty(need, dtype=torch.uint8, device=device) if need else None
    with torch.cuda.device(device):
        rc = L.ggufb200_linear_fallback(qcode, wraw.data_ptr(), N, K, x2.data_ptr(), M, x2.stride(0), act, bias_ptr, bias_code, y.data_ptr(), N,
                                        None if ws is None else ws.data_ptr(), need, algo, _current_stream_ptr(device.index))
    _lib.check(rc, f"ggufb200_linear_fallback({getattr(qtype, 'name', qtype)}, M={M}, N={N}, K={K})")
    return y if x.dim() == 2 else y.reshape(*x.shape[:-1], N)


def linear_packed(x, weight, bias, dequant_dtype=None, algo=_lib.ALGO_AUTO, use_spans=False):
    """y = x @ dequant(weight).T + bias through the C ABI, weight still packed.  `algo` = _lib.ALGO_* | _lib.FLAG_*.
    use_spans: hand the re-packed span-major copy of the weight (built once, cached on the tensor) to the FUSED_TMEM kernel.

    x: CUDA fp16/bf16 [..., K]; weight: CUDA GGMLTensor (quantised type); bias: None or a CUDA tensor
    (fp32 / fp16 / bf16, rounded to x.dtype inside the kernel exactly like ops.py:205-207 does)."""
    N, K = tuple(weight.tensor_shape)
    if x.shape[-1] != K:
        raise ValueError(f"linear_packed: input features {x.shape[-1]} != weight in_features {K}")
    wraw = _plain(weight)
    spans = span_layout(weight, wraw) if use_spans else None
    return _launch_linear(x, wraw, weight.tensor_type, N, K, None if bias is None else _plain(bias),
                          math_code(dequant_dtype, x.dtype), algo, spans)


def linear_dense(x, weight, bias=None, feature_scale=None):
    """y = x @ weight.T + bias on the tensor-core GEMM with an already dense fp16/bf16 weight (ggufb200_gemm).
    feature_scale: None, or a CUDA fp32 [N] tensor: y = feature_scale * (x @ weight.T) + bias (ggufb200_gemm_scaled)."""
    N, K = weight.shape
    x2 = x.reshape(-1, K)
    if x2.stride(-1) != 1 or (x2.stride(0) % 8) != 0 or (x2.data_ptr() % 16) != 0:
        x2 = x2.contiguous()
    weight = _plain(weight)
    if weight.dtype != x.dtype or weight.stride(-1) != 1 or (weight.stride(0) % 8) != 0:
        weight = weight.to(x.dtype).contiguous()
    M = x2.shape[0]
    y = torch.empty(M, N, dtype=x.dtype, device=x.device)
    bias_ptr, bias_code = None, 0
    if bias is not None:
        bias = _plain(bias).contiguous()
        bias_ptr, bias_code = bias.data_ptr(), dtype_code(bias.dtype)
    with torch.cuda.device(x.device):
        if feature_scale is None:
            rc = _lib.lib().ggufb200_gemm(weight.data_ptr(), N, K, weight.stride(0), x2.data_ptr(), M, x2.stride(0), dtype_code(x.dtype),
                                          bias_ptr, bias_code, y.data_ptr(), N, torch.cuda.current_stream(x.device).cuda_stream)
        else:
            rc = _lib.lib().ggufb200_gemm_scaled(weight.data_ptr(), N, K, weight.stride(0), x2.data_ptr(), M, x2.stride(0), dtype_code(x.dtype),
                                                 bias_ptr, bias_code, feature_scale.data_ptr(), y.data_ptr(), N,
                                                 torch.cuda.current_stream(x.device).cuda_stream)
    _lib.check(rc, f"ggufb200_gemm(M={M}, N={N}, K={K})")
    return y.reshape(*x.shape[:-1], N)


def linear_grad_input(dy, wraw, qtype, N, K, math):
    """dX = dY @ W for a CUDA fp16/bf16 dY [..., N] and the packed rows `wraw` (plain uint8 on dy.device) of an [N, K] weight
    (ggufb200_linear_grad_input): W is dequantised with the math dtype code `math` into a workspace, never kept."""
    dy2 = dy.reshape(-1, N)
    # rows that overlap (a stride below N: autograd hands broadcast gradients such as that of y.sum(0) with row stride 0), are
    # not contiguous, or do not start on 16-byte boundaries are copied
    if dy2.stride(-1) != 1 or dy2.stride(0) < N or (dy2.stride(0) % 8) != 0 or (dy2.data_ptr() % 16) != 0:
        pad = -N % 8                                     # rows of dY must start on 16-byte boundaries: pad them to 8 elements
        dy2 = torch.nn.functional.pad(dy2, (0, pad)) if pad else dy2.contiguous()
    if not wraw.is_contiguous() or (qtype == _Q.BF16 and wraw.data_ptr() & 15):      # BF16 rows are read in place: 16-byte aligned
        wraw = wraw.clone(memory_format=torch.contiguous_format)
    M = dy2.shape[0]
    dx = torch.empty(M, K, dtype=dy.dtype, device=dy.device)
    L = _lib.lib()
    qcode, act = int(qtype), dtype_code(dy.dtype)
    need = L.ggufb200_linear_grad_input_workspace(qcode, N, K, act)
    ws = torch.empty(need, dtype=torch.uint8, device=dy.device) if need else None
    with torch.cuda.device(dy.device):
        rc = L.ggufb200_linear_grad_input(qcode, wraw.data_ptr(), N, K, dy2.data_ptr(), M, dy2.stride(0), act, math, dx.data_ptr(), K,
                                          None if ws is None else ws.data_ptr(), need, _lib.FLAG_W_STABLE,
                                          _current_stream_ptr(dy.device.index))
    _lib.check(rc, f"ggufb200_linear_grad_input({getattr(qtype, 'name', qtype)}, M={M}, N={N}, K={K})")
    return dx.reshape(*dy.shape[:-1], K)


class PackedLinearFunction(torch.autograd.Function):
    """y = run(), the packed-weight Linear's forward as it runs without gradients (bit-identical output), differentiable in x.

    Saves only the packed rows `wraw` and the (qtype, N, K, math) metadata, never a dense W: the backward dequantises again
    from the packed bytes (`linear_grad_input`).  The weight and bias are frozen (no gradient).  The backward always uses the
    exact weight, also after a `fast`-contract forward.  Once differentiable: double backward raises."""

    @staticmethod
    def forward(ctx, x, wraw, run, qtype, N, K, math):
        ctx.save_for_backward(wraw)
        ctx.meta = (qtype, N, K, math)
        return run()

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        (wraw,) = ctx.saved_tensors
        dx = linear_grad_input(dy, wraw, *ctx.meta) if ctx.needs_input_grad[0] else None
        return dx, None, None, None, None, None, None


def _requires_grad(item):
    """True when a tensor inside a patch structure (entries, payload tuples, adapter objects' `.weights`) requires grad."""
    if torch.is_tensor(item):
        return item.requires_grad
    if isinstance(item, (tuple, list)):
        return any(_requires_grad(x) for x in item)
    weights = getattr(item, "weights", None)
    return weights is not None and _requires_grad(weights)


def grad_needed(input, weight):
    """The one predicate of the differentiable routes: gradients are being recorded and the input or a factor of the weight's
    patches requires grad.  False keeps every route, launch and output bit exactly as without autograd."""
    return torch.is_grad_enabled() and (input.requires_grad or _requires_grad(getattr(weight, "patches", ())))


def lora_side_sum(y, x, terms):
    """y + sum of the LoRA side terms scale * (x_band down^T) up^T of `lora_band_terms`, in differentiable torch ops (gradients
    reach x, up and down with calculate_weight's scale strength * alpha / r); a row band adds into its output columns only."""
    N = y.shape[-1]
    for scale, up, down, band in terms:
        xs = x[..., band[1]:band[1] + band[2]] if band is not None and band[0] == 1 else x
        u = (up.to(device=x.device, dtype=torch.float32) * scale).to(x.dtype)
        t = torch.nn.functional.linear(torch.nn.functional.linear(xs, down.to(device=x.device, dtype=x.dtype)), u)
        if band is not None and band[0] == 0:
            t = torch.nn.functional.pad(t, (band[1], N - band[1] - band[2]))
        y = y + t
    return y


def scale_columns(x, col_scale):
    """act(fp32(x) * col_scale) for a CUDA fp16/bf16 x [..., K] and fp32 col_scale [K] (ggufb200_scale_columns), bit-identical to
    `(x.float() * col_scale).to(x.dtype)`."""
    K = x.shape[-1]
    x2 = x.reshape(-1, K)
    if x2.stride(-1) != 1 or (x2.stride(0) % 8) != 0 or (x2.data_ptr() % 16) != 0:
        x2 = x2.contiguous()
    y = torch.empty(x2.shape, dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        rc = _lib.lib().ggufb200_scale_columns(x2.data_ptr(), x2.shape[0], K, x2.stride(0), dtype_code(x.dtype), col_scale.data_ptr(),
                                               y.data_ptr(), K, torch.cuda.current_stream(x.device).cuda_stream)
    _lib.check(rc, f"ggufb200_scale_columns(M={x2.shape[0]}, K={K})")
    return y.reshape(x.shape)


_BIG_EMBEDDING_ROWS = 64 * 1024     # loader threshold above which Embedding always takes the GGML load path (ops.py:116-117)
_META = torch.device("meta")


def _collect_patches(tensor):
    """Flatten `tensor.patches` ([(patch_list, key), ...]) onto the tensor's device; returns (patches, last key)."""
    gathered, key = [], None
    for entries, key in getattr(tensor, "patches", []):
        gathered.extend(move_patch_to_device(entries, tensor.device))
    return gathered, key


def _patch_entries(tensor):
    """`tensor.patches` ([(patch_list, key), ...]) flattened into one list of entries, where they are."""
    return [entry for patch_list, _key in tensor.patches for entry in patch_list]


_ADAPTER_KINDS = {"LoRAAdapter": "lora", "LoHaAdapter": "loha", "LoKrAdapter": "lokr"}


def _entry_tensors(entry):
    """The tensors of a patch entry's payload ((kind, payload) or an adapter's `.weights`)."""
    value = entry[1] if len(entry) > 1 else None
    payload = getattr(value, "weights", None)
    if payload is None and isinstance(value, (tuple, list)) and len(value) == 2:
        payload = value[1]
    return [t for t in (payload or ()) if torch.is_tensor(t)] if isinstance(payload, (tuple, list)) else []


def _mat(t):
    return torch.is_tensor(t) and t.dim() == 2


def _decode_patch(entry, kinds=("lora", "loha", "lokr")):
    """One comfy.lora patch entry `(strength_patch, value, strength_model[, offset, function])` of one of `kinds` as the record
    (kind, strength, a, factors, band, dora_scale), or None when it needs the general `calculate_weight` machinery or is of
    another kind.

    The value is `(kind, payload)` or an adapter object carrying the payload in `.weights`, matched by its class name
    (LoRAAdapter / LoHaAdapter / LoKrAdapter), not by type:
        "lora"  (up, down, alpha, mid, dora_scale, reshape)               factors (up, down),  a = alpha / down.shape[0]
        "loha"  (w1a, w1b, alpha, w2a, w2b, t1, t2, dora_scale)          factors (w1a, w1b, w2a, w2b),  a = alpha / w1b.shape[0]
        "lokr"  (w1, w2, alpha, w1_a, w1_b, w2_a, w2_b, t2, dora_scale)  factors (w1, w2, w1_a, w1_b, w2_a, w2_b), w1 or (w1_a, w1_b)
                given, likewise w2;  a = alpha / dim with dim = w1_b.shape[0] when w1 is decomposed, w2_b.shape[0] when w2 is
                (that one wins), 1.0 when neither is
    and a = 1.0 when alpha is None: comfy.lora.calculate_weight scales the delta by strength * a.  strength = float(strength_patch);
    band = the offset (dim, start, size), dim 0 for output rows and 1 for input features, or None for the whole weight;
    dora_scale = the entry's DoRA tensor or None.  None for strength_model != 1, a function hook, any other offset, LoCon mid,
    reshape, Tucker factors (t1 / t2), a dora_scale that is not a tensor, and factors that are not 2-D or do not chain."""
    if len(entry) < 3 or entry[2] != 1.0 or (len(entry) > 4 and entry[4] is not None):
        return None
    offset = entry[3] if len(entry) > 3 else None
    band = None
    if offset is not None:
        if not isinstance(offset, (tuple, list)) or len(offset) != 3 or offset[0] not in (0, 1):
            return None
        band = (int(offset[0]), int(offset[1]), int(offset[2]))
        if band[1] < 0 or band[2] <= 0:
            return None
    value = entry[1]
    kind = _ADAPTER_KINDS.get(type(value).__name__)
    if kind in kinds and hasattr(value, "weights"):
        payload = tuple(value.weights)
    elif isinstance(value, (tuple, list)) and len(value) == 2 and value[0] in kinds:
        kind, payload = value[0], tuple(value[1])
    else:
        return None
    if kind == "lora":
        if len(payload) < 2:
            return None
        up, down, alpha, mid, dora_scale, reshape = (payload + (None,) * 4)[:6]
        if mid is not None or reshape is not None or not (_mat(up) and _mat(down)) or up.shape[1] != down.shape[0]:
            return None
        factors, dim = (up, down), down.shape[0]
    elif kind == "loha":
        if len(payload) < 5:
            return None
        w1a, w1b, alpha, w2a, w2b, t1, t2, dora_scale = (payload + (None,) * 3)[:8]
        if t1 is not None or t2 is not None or not all(_mat(t) for t in (w1a, w1b, w2a, w2b)) or w1a.shape[1] != w1b.shape[0] \
                or w2a.shape[1] != w2b.shape[0] or w1a.shape[0] != w2a.shape[0] or w1b.shape[1] != w2b.shape[1]:
            return None
        factors, dim = (w1a, w1b, w2a, w2b), w1b.shape[0]
    else:
        if len(payload) < 7:
            return None
        w1, w2, alpha, w1_a, w1_b, w2_a, w2_b, t2, dora_scale = (payload + (None,) * 2)[:9]
        if t2 is not None:
            return None
        dim = None
        for whole, a, b in ((w1, w1_a, w1_b), (w2, w2_a, w2_b)):
            if whole is not None:
                if not _mat(whole):
                    return None
            elif _mat(a) and _mat(b) and a.shape[1] == b.shape[0]:
                dim = b.shape[0]
            else:
                return None
        factors = (w1, w2, w1_a, w1_b, w2_a, w2_b)
    if dora_scale is not None and not torch.is_tensor(dora_scale):
        return None
    a = 1.0 if alpha is None or dim is None else float(alpha) / dim
    return kind, float(entry[0]), a, factors, band, dora_scale


def lora_side_terms(patches):
    """Recognise a patch list of plain whole-weight LoRA deltas (SURVEY 8f rank 1): [(scale, up[N, r], down[r, K]), ...] with
    scale = strength_patch * alpha / r, or None when any entry is anything else (`lora_band_terms` without offsets)."""
    terms = lora_band_terms(patches)
    if terms is None or any(band is not None for _s, _u, _d, band in terms):
        return None
    return [(scale, up, down) for scale, up, down, _band in terms]


def lora_band_terms(patches):
    """Recognise a patch list of plain LoRA entries, each on the whole weight or on a band (`_decode_patch`): ComfyUI gives
    diffusers-format LoRAs an `offset = (dim, start, size)`, one entry per q / k / v / mlp slice of a fused Flux or SD3 weight,
    and the LoRA then patches rows (dim 0) or input features (dim 1) `start .. start + size` only.  Returns [(scale, up, down,
    band), ...] with scale = strength_patch * a, or None when any entry is not a plain LoRA (`lycoris_terms` of LoRA only)."""
    terms = []
    for entry in patches:
        record = _decode_patch(entry, ("lora",))
        if record is None or record[5] is not None:                            # not a plain LoRA
            return None
        _kind, strength, a, (up, down), band, _dora_scale = record
        terms.append((strength * a, up, down, band))
    return terms


def lycoris_terms(patches):
    """Recognise a patch list of LoRA, LoHa and LoKr (LyCORIS) entries without DoRA, in any mix (`_decode_patch`).  Returns
    [(kind, scale, factors, band), ...] in list order with scale = strength_patch * a, or None when any entry needs
    `calculate_weight`."""
    terms = []
    for entry in patches:
        record = _decode_patch(entry)
        if record is None:
            return None
        kind, strength, a, factors, band, dora_scale = record
        if dora_scale is not None:
            return None
        terms.append((kind, strength * a, factors, band))
    return terms


def _flat_lora_entry(entry):
    """(entry', sources): `entry` with the up / down factors of a LoRA / LoCon payload flattened to 2-D as calculate_weight
    multiplies them (`flatten(start_dim=1)`: up [Cout, r, 1, 1] -> [Cout, r], down [r, Cin, kh, kw] -> [r, Cin kh kw]) and the
    two 4-D tensors it flattened; (entry, None) for any other entry.  LoHa factors are not flattened: the reference multiplies
    them with torch.mm as they come."""
    value = entry[1] if len(entry) > 1 else None
    if _ADAPTER_KINDS.get(type(value).__name__) == "lora" and hasattr(value, "weights"):
        payload = tuple(value.weights)
    elif isinstance(value, (tuple, list)) and len(value) == 2 and value[0] == "lora":
        payload = tuple(value[1])
    else:
        return entry, None
    if len(payload) < 2 or not all(torch.is_tensor(t) and t.dim() == 4 for t in payload[:2]):
        return entry, None
    flat = (entry[0], ("lora", tuple(t.flatten(start_dim=1) for t in payload[:2]) + payload[2:])) + tuple(entry[2:])
    return flat, payload[:2]


def conv_patch_terms(patches):
    """Recognise a Conv2d patch list of whole-weight LoRA / LoCon and LoHa entries (`_decode_patch`, LoRA factors flattened by
    `_flat_lora_entry`).  Returns [(kind, scale, factors, sources), ...] in list order with scale = strength_patch * a, factors
    the 2-D matrices of the delta ((up, down) or (w1a, w1b, w2a, w2b)) and sources the entry's own tensors (cache keys), or None
    when any entry is LoKr, has an offset, carries DoRA or needs `calculate_weight` (strength_model != 1, a hook, Tucker / mid,
    reshape).  The Linear recognisers are separate and keep refusing 4-D factors."""
    terms = []
    for entry in patches:
        flat, sources = _flat_lora_entry(entry)
        record = _decode_patch(flat, ("lora", "loha"))
        if record is None or record[4] is not None or record[5] is not None:
            return None
        kind, strength, a, factors, _band, _dora_scale = record
        terms.append((kind, strength * a, factors, factors if sources is None else sources))
    return terms


def lowrank_pays(N, K, terms):
    """True when ggufb200_dequant_lowrank (or ggufb200_dequant_patched) is expected to form the patched [N, K] weight faster than
    the two-step route (K1 + calculate_weight).  Cost model in microseconds, fitted to tools/bench_conv_patches.py and
    tools/bench_conv_lycoris.py on an NVIDIA H100 80GB HBM3 at 700 W (Q4_K, fp16, SD1.5 / SDXL conv shapes, LoRA ranks 16-256,
    LoHa 16 / 32, LoKr factors 4-16; DESIGN.md section 9), with E = N K / 1e6:
        kernel     6 + 2.6 E + 0.11 L R + KRON_KERNEL_US L per LoKr entry
                   R = rank sums per element (LoRA r, LoHa r1 + r2), L = max(1, 64 x 128 tiles / 132 SMs)
        two-step   per LoRA entry 8 + 9 E + 0.041 E r, per LoHa entry 16 + 15.4 E + 0.041 E (r1 + r2),
                   per LoKr entry KRON_TWO_STEP_US[0] + KRON_TWO_STEP_US[1] E
    The kernel's rank loop costs more per rank than cuBLAS's product, so high ranks on small weights keep the two-step route
    (LoRA above about rank 40 on a 320-channel 1x1 conv, about 120 on the SDXL 1280-channel 3x3).  LoCon `mid` and Tucker LoHa
    entries are priced as the LoRA / LoHa they become, plus TUCKER_TWO_STEP_US on the two-step side for the Tucker products."""
    kernel, two_step = _lowrank_costs(N, K, terms)
    return kernel <= two_step


def _lowrank_costs(N, K, terms):
    """(kernel, two-step) microseconds of `lowrank_pays`'s cost model."""
    E = N * K / 1e6
    L = max(1.0, -(-N // 64) * -(-K // 128) / 132)
    kernel, two_step = 6 + 2.6 * E, 0.0
    for kind, _scale, factors, _sources in terms:
        if kind == "lokr":
            kernel += KRON_KERNEL_US * L
            two_step += KRON_TWO_STEP_US[0] + KRON_TWO_STEP_US[1] * E
            continue
        R = sum(conv_term_ranks(kind, factors))
        kernel += 0.11 * L * R
        two_step += (16 + 15.4 * E if kind in ("loha", "loha_tucker") else 8 + 9 * E) + 0.041 * E * R
        if kind in ("locon_mid", "loha_tucker"):
            two_step += TUCKER_TWO_STEP_US
    return kernel, two_step


def conv_dora_pays(N, K, terms):
    """True when ggufb200_dequant_patched_dora is expected to form the patched [N, K] weight of recognised `conv_dora_terms`
    faster than the two-step route: `lowrank_pays`'s model of the deltas, plus on the two-step side weight_decompose's passes
    per DoRA entry (alpha scale, cast, add, norm, division, factor scale and, at strength != 1, the blend), net of the kernel's
    DoRA step: DORA_TWO_STEP_US fixed + per million weight elements.  Measured on an NVIDIA H100 80GB HBM3 at 700 W (Q4_K / Q8_0,
    fp16, SD1.5 / SDXL conv shapes, DoRA LoCon ranks 16-64, LoHa 16, LoKr factor 8; DESIGN.md section 9) the kernel won in every
    row, including rank 64 on the 320-channel 1x1 conv, where the plain LoRA keeps the two-step route."""
    kernel, two_step = _lowrank_costs(N, K, [(kind, st * a, factors, sources) for kind, st, a, factors, sources, _ds, _axis in terms])
    for *_t, ds, _axis in terms:
        if ds is not None:
            two_step += DORA_TWO_STEP_US[0] + DORA_TWO_STEP_US[1] * N * K / 1e6
    return kernel <= two_step


def conv_patch_operands(terms, device):
    """The fp32 factors of recognised `conv_patch_terms` on `device` and their ggufb200_lowrank_patch array (the tensors stay
    referenced by the returned list for as long as the array is used)."""
    ops = [(kind, scale, tuple(t.to(device=device, dtype=torch.float32).contiguous() for t in factors))
           for kind, scale, factors, _sources in terms]

    def desc(kind, scale, f):
        loha = kind == "loha"
        return _lib.LowrankPatch(f[0].data_ptr(), f[1].data_ptr(), f[2].data_ptr() if loha else None, f[3].data_ptr() if loha else None,
                                 f[0].shape[1], f[2].shape[1] if loha else 0, scale)
    return ops, (_lib.LowrankPatch * max(1, len(ops)))(*[desc(*op) for op in ops])


def _conv_lycoris_entry(entry):
    """One whole-weight Conv2d patch entry of a form only `conv_lycoris_terms` serves, as (kind, scale, factors, sources), or None:
        "locon_mid"    LoCon with a Tucker `mid`: factors (up, down, mid), a = alpha / down.shape[0]
        "loha_tucker"  LoHa with both `t1` and `t2`: factors (w1a, w1b, t1, w2a, w2b, t2), a = alpha / w1b.shape[0]
        "lokr"         LoKr, w1 whole 2-D or decomposed, w2 whole 2-D / 4-D, decomposed or Tucker (`t2`): factors (w1, w2, w1_a,
                       w1_b, w2_a, w2_b, t2) with t2 None unless w2 is Tucker-decomposed, a = alpha / dim as `_decode_patch`
    with scale = strength_patch * a and sources the entry's own tensors (cache keys).  None for an offset, DoRA, reshape,
    strength_model != 1, a hook, only one of t1 / t2, a 4-D w1, factors that do not chain, and every plain LoRA / LoHa entry."""
    if len(entry) < 3 or entry[2] != 1.0 or (len(entry) > 3 and entry[3] is not None) or (len(entry) > 4 and entry[4] is not None):
        return None
    value = entry[1]
    kind = _ADAPTER_KINDS.get(type(value).__name__)
    if kind is not None and hasattr(value, "weights"):
        payload = tuple(value.weights)
    elif isinstance(value, (tuple, list)) and len(value) == 2 and value[0] in ("lora", "loha", "lokr"):
        kind, payload = value[0], tuple(value[1])
    else:
        return None

    def dims(t, *n):
        return torch.is_tensor(t) and t.dim() in n

    def column(t):                                     # [r, c] or [r, c, 1, 1]: flatten(start_dim=1) keeps it a column factor
        return dims(t, 2) or (dims(t, 4) and tuple(t.shape[2:]) == (1, 1))
    if kind == "lora":
        if len(payload) < 4:
            return None
        up, down, alpha, mid, dora_scale, reshape = (payload + (None,) * 2)[:6]
        if mid is None or dora_scale is not None or reshape is not None or not (column(up) and column(down) and dims(mid, 4)):
            return None
        r = down.shape[0]
        if up.shape[1] != r or tuple(mid.shape[:2]) != (r, r):
            return None
        factors, dim = (up, down, mid), r
    elif kind == "loha":
        if len(payload) < 7:
            return None
        w1a, w1b, alpha, w2a, w2b, t1, t2, dora_scale = (payload + (None,))[:8]
        if t1 is None or t2 is None or dora_scale is not None or not all(dims(t, 2) for t in (w1a, w1b, w2a, w2b)) \
                or not (dims(t1, 4) and dims(t2, 4)):
            return None
        if t1.shape[0] != w1a.shape[0] or t1.shape[1] != w1b.shape[0] or t2.shape[0] != w2a.shape[0] or t2.shape[1] != w2b.shape[0] \
                or w1a.shape[1] != w2a.shape[1] or w1b.shape[1] != w2b.shape[1] or t1.shape[2:] != t2.shape[2:]:
            return None
        factors, dim = (w1a, w1b, t1, w2a, w2b, t2), w1b.shape[0]
    else:
        if len(payload) < 7:
            return None
        w1, w2, alpha, w1_a, w1_b, w2_a, w2_b, t2, dora_scale = (payload + (None,) * 2)[:9]
        if dora_scale is not None:
            return None
        dim = None
        if w1 is not None:
            if not dims(w1, 2):
                return None
        elif dims(w1_a, 2) and dims(w1_b, 2) and w1_a.shape[1] == w1_b.shape[0]:
            dim = w1_b.shape[0]
        else:
            return None
        if w2 is not None:
            if not dims(w2, 2, 4):
                return None
            t2 = None                                  # the reference reads t2 only for a decomposed w2
        elif not (dims(w2_a, 2) and dims(w2_b, 2)):
            return None
        elif t2 is None:
            if w2_a.shape[1] != w2_b.shape[0]:
                return None
            dim = w2_b.shape[0]
        elif dims(t2, 4) and t2.shape[0] == w2_a.shape[0] and t2.shape[1] == w2_b.shape[0]:
            dim = w2_b.shape[0]
        else:
            return None
        factors = (w1, w2, w1_a, w1_b, w2_a, w2_b, t2)
    a = 1.0 if alpha is None or dim is None else float(alpha) / dim
    sources = tuple(t for t in factors if t is not None)
    return {"lora": "locon_mid", "loha": "loha_tucker", "lokr": "lokr"}[kind], float(entry[0]) * a, factors, sources


def conv_lycoris_terms(patches):
    """Recognise a Conv2d patch list of whole-weight entries of which at least one is LoKr, LoCon with `mid` or Tucker LoHa
    (`_conv_lycoris_entry`), mixed in any order with plain LoRA / LoCon and LoHa entries (`conv_patch_terms`).  Returns
    [(kind, scale, factors, sources), ...] in list order, or None when the list has none of these entries (`conv_patch_terms`
    serves it) or any entry needs `calculate_weight`."""
    terms, lycoris = [], False
    for entry in patches:
        term = _conv_lycoris_entry(entry)
        if term is None:
            plain = conv_patch_terms([entry])
            if not plain:
                return None
            term = plain[0]
        else:
            lycoris = True
        terms.append(term)
    return terms if lycoris else None


def conv_lokr_shapes(factors):
    """(a1, a2), (b1, b2) of a "lokr" conv term: A = w1 or w1_a @ w1_b, B = w2 (or its product / Tucker einsum) as [b1, b2]."""
    w1, w2, w1_a, w1_b, w2_a, w2_b, t2 = factors
    a = tuple(w1.shape) if w1 is not None else (w1_a.shape[0], w1_b.shape[1])
    if w2 is not None:
        b = (w2.shape[0], w2.numel() // w2.shape[0])
    elif t2 is None:
        b = (w2_a.shape[0], w2_b.shape[1])
    else:
        b = (w2_a.shape[1], w2_b.shape[1] * t2.shape[2] * t2.shape[3])
    return a, b


def conv_term_shape(kind, factors):
    """(rows, cols) of the [N, K] delta of a `conv_lycoris_terms` term."""
    if kind == "lokr":
        (a1, a2), (b1, b2) = conv_lokr_shapes(factors)
        return a1 * b1, a2 * b2
    if kind == "locon_mid":
        up, down, mid = factors
        return up.shape[0], down.shape[1] * mid.shape[2] * mid.shape[3]
    if kind == "loha_tucker":
        w1a, w1b, t1 = factors[:3]
        return w1a.shape[1], w1b.shape[1] * t1.shape[2] * t1.shape[3]
    return factors[0].shape[0], factors[-1].shape[1]


def conv_term_ranks(kind, factors):
    """The ranks of a `conv_lycoris_terms` term's factor pairs (one for LoRA, two for LoHa, none for LoKr)."""
    if kind == "lokr":
        return ()
    if kind == "locon_mid":
        return (factors[1].shape[0],)
    if kind == "loha_tucker":
        return factors[2].shape[0], factors[5].shape[0]
    return tuple(f.shape[0] for f in factors[1::2])


def _reference_kron_raises(w1, w2):
    """True when comfy.lora's `torch.kron(w1, w2)` (w1 unsqueezed to 4-D for a 4-D w2) raises for factors of these shapes and
    strides: torch.kron views its product, which fails for some non-contiguous factors (a Tucker w2 straight out of
    torch.einsum), and ComfyUI then logs the error and skips the entry.  Checked on meta tensors: no data is touched."""
    m1 = torch.empty_strided(w1.shape, w1.stride(), device=_META)
    m2 = torch.empty_strided(w2.shape, w2.stride(), device=_META)
    if m2.dim() == 4:
        m1 = m1.unsqueeze(2).unsqueeze(2)
    try:
        torch.kron(m1, m2)
    except RuntimeError:
        return True
    return False


def conv_lokr_operands(factors, device):
    """fp32 A [a1, a2] and B [b1, K / a2] of a "lokr" conv term on `device`, each formed by comfy.lora's own expressions: a
    decomposed factor is torch.mm of its halves, a Tucker w2 torch.einsum('i j k l, j r, i p -> p r k l', t2, w2_b, w2_a).  B's
    2-D view makes torch.kron(w1, w2).reshape(Cout, -1) the 2-D Kronecker product of A and B.  None when the reference's
    torch.kron raises for these factors (`_reference_kron_raises`): the entry is then the two-step route's to skip."""
    w1, w2, w1_a, w1_b, w2_a, w2_b, t2 = factors

    def f32(t):
        return t.to(device=device, dtype=torch.float32)
    A = f32(w1) if w1 is not None else torch.mm(f32(w1_a), f32(w1_b))
    if w2 is not None:
        B = f32(w2)
    elif t2 is None:
        B = torch.mm(f32(w2_a), f32(w2_b))
    else:
        B = torch.einsum("i j k l, j r, i p -> p r k l", f32(t2), f32(w2_b), f32(w2_a))
    if _reference_kron_raises(A, B):
        return None
    return A.contiguous(), B.reshape(B.shape[0], -1).contiguous()


def locon_mid_down(down, mid, device):
    """LoCon's Tucker-composed down [r, Cin kh kw] in fp32 on `device`, by comfy.lora's expression (mm of the transposed down and
    mid, reshaped and transposed back), flattened as calculate_weight multiplies it."""
    down, mid = down.to(device=device, dtype=torch.float32), mid.to(device=device, dtype=torch.float32)
    final_shape = [down.shape[1], down.shape[0], mid.shape[2], mid.shape[3]]
    down = torch.mm(down.transpose(0, 1).flatten(start_dim=1), mid.transpose(0, 1).flatten(start_dim=1)).reshape(final_shape).transpose(0, 1)
    return down.flatten(start_dim=1).contiguous()


def loha_tucker_half(wa, wb, t, device):
    """One Tucker LoHa half einsum('i j k l, j r, i p -> p r k l', t, wb, wa) as a rank-r product a @ b in fp32 on `device`:
    a = wa^T [Cout, r], b = einsum('i j k l, j r -> i r k l', t, wb).reshape(r, Cin kh kw)."""
    wa, wb, t = (x.to(device=device, dtype=torch.float32) for x in (wa, wb, t))
    b = torch.einsum("i j k l, j r -> i r k l", t, wb)
    return wa.t().contiguous(), b.reshape(b.shape[0], -1).contiguous()


def conv_lycoris_operands(terms, device):
    """The fp32 operands of recognised `conv_lycoris_terms` on `device` and their ggufb200_weight_patch array (the tensors stay
    referenced by the returned list for as long as the array is used): LoRA / LoHa factors as they are, LoCon `mid` as a LoRA
    with `locon_mid_down`, Tucker LoHa as a LoHa of `loha_tucker_half` pairs, LoKr as a Kronecker patch (`conv_lokr_operands`).
    None when a LoKr entry is one the reference skips."""
    keep, descs = [], []
    for kind, scale, factors, _sources in terms:
        if kind == "lokr":
            AB = conv_lokr_operands(factors, device)
            if AB is None:
                return None
            A, B = AB
            keep.append(AB)
            kron = _lib.KronPatch(A.data_ptr(), B.data_ptr(), A.shape[0], A.shape[1], B.shape[0], B.shape[1], -1, scale, 0, 0)
            descs.append(_lib.WeightPatch(_lib.PATCH_KRON, _lib.LowrankPatch(), kron))
            continue
        if kind == "locon_mid":
            f = (factors[0].to(device=device, dtype=torch.float32).flatten(start_dim=1).contiguous(), locon_mid_down(*factors[1:], device))
        elif kind == "loha_tucker":
            f = loha_tucker_half(*factors[:3], device) + loha_tucker_half(*factors[3:], device)
        else:
            f = tuple(t.to(device=device, dtype=torch.float32).contiguous() for t in factors)
        keep.append(f)
        loha = len(f) == 4
        lowrank = _lib.LowrankPatch(f[0].data_ptr(), f[1].data_ptr(), f[2].data_ptr() if loha else None, f[3].data_ptr() if loha else None,
                                    f[0].shape[1], f[2].shape[1] if loha else 0, scale)
        descs.append(_lib.WeightPatch(_lib.PATCH_LOWRANK, lowrank, _lib.KronPatch()))
    return keep, (_lib.WeightPatch * max(1, len(descs)))(*descs)


_DORA_AT = {"lora": 4, "loha": 7, "lokr": 8}      # index of dora_scale in a LoRA / LoHa / LoKr payload


def _split_dora(entry):
    """(entry', dora_scale) of a LoRA / LoHa / LoKr patch entry: entry' is the entry at strength 1 with its value as a (kind,
    payload) pair whose dora_scale is None, dora_scale the entry's own (None when it has none).  (None, None) for another value."""
    value = entry[1] if len(entry) > 1 else None
    kind = _ADAPTER_KINDS.get(type(value).__name__)
    if kind is not None and hasattr(value, "weights"):
        payload = tuple(value.weights)
    elif isinstance(value, (tuple, list)) and len(value) == 2 and value[0] in _DORA_AT:
        kind, payload = value[0], tuple(value[1])
    else:
        return None, None
    at = _DORA_AT[kind]
    dora_scale = payload[at] if len(payload) > at else None
    if dora_scale is not None:
        payload = payload[:at] + (None,) + payload[at + 1:]
    return (1.0, (kind, payload)) + tuple(entry[2:]), dora_scale


def conv_dora_axis(dora_scale, shape):
    """weight_decompose's axis for a Conv2d weight of `shape` [Cout, Cin, kh, kw]: 0 for dora_scale [Cout, 1, 1, 1] (one norm per
    output channel), 1 for [1, Cin, 1, 1] (one per input channel), None for any other shape.  The reference normalises the output
    axis when dora_scale.shape[0] == Cout."""
    cout, cin = shape[0], shape[1]
    ds = tuple(dora_scale.shape)
    if ds == (cout, 1, 1, 1):
        return 0
    if ds == (1, cin, 1, 1) and cout != 1:
        return 1
    return None


def conv_dora_terms(patches, shape):
    """Recognise a Conv2d patch list of whole-weight entries of which at least one carries DoRA (`dora_scale`), for a weight of
    `shape` [Cout, Cin, kh, kw].  Every entry, its dora_scale set aside (`_split_dora`), is one `conv_patch_terms` or
    `conv_lycoris_terms` serve: LoRA / LoCon (with or without `mid`), LoHa (plain or Tucker) and LoKr, in any order.  Returns
    [(kind, strength, a, factors, sources, dora_scale, axis), ...] in list order (a = alpha / rank, kept apart from the strength;
    sources the entry's tensors, dora_scale included, as cache keys; dora_scale and axis None for a plain entry), or None when
    the list has no DoRA entry (the other recognisers serve it), has more than LOWRANK_MAX_PATCHES entries, or any entry needs
    `calculate_weight` (strength_model != 1, a hook, an offset, reshape), does not fit [Cout, Cin kh kw], exceeds the rank limit,
    has a dora_scale that is not a tensor of a `conv_dora_axis` shape, or a strength != 1 that rounds to 1 in fp32."""
    if len(patches) > _lib.LOWRANK_MAX_PATCHES:
        return None
    N, K = shape[0], shape[1] * shape[2] * shape[3]
    terms = []
    for entry in patches:
        unit, dora_scale = _split_dora(entry)
        if unit is None:
            return None
        term = _conv_lycoris_entry(unit)
        if term is None:
            plain = conv_patch_terms([unit])
            if not plain:
                return None
            term = plain[0]
        kind, a, factors, sources = term
        if conv_term_shape(kind, factors) != (N, K) or max(conv_term_ranks(kind, factors), default=0) > _lib.LOWRANK_MAX_RANK:
            return None
        strength, axis = float(entry[0]), None
        if dora_scale is not None:
            if not torch.is_tensor(dora_scale):
                return None
            axis = conv_dora_axis(dora_scale, shape)
            if axis is None or (strength != 1.0 and float(torch.tensor(strength, dtype=torch.float32)) == 1.0):
                return None
            sources = tuple(sources) + (dora_scale,)
        terms.append((kind, strength, a, factors, tuple(sources), dora_scale, axis))
    return terms if any(t[5] is not None for t in terms) else None


def conv_term_delta(kind, factors, device):
    """The fp32 [N, K] delta of a `conv_dora_terms` term as ComfyUI's adapters form it (`calculate_weight`, before scaling):
    LoRA torch.mm of the flattened factors (LoCon `mid`: of the composed down, `locon_mid_down`), LoHa the product of two torch.mm
    (Tucker: of two einsum('i j k l, j r, i p -> p r k l', t, wb, wa)), LoKr the Kronecker product (`conv_lokr_operands`; None
    when the reference skips the entry)."""
    def f32(t):
        return t.to(device=device, dtype=torch.float32)
    if kind == "lokr":
        AB = conv_lokr_operands(factors, device)
        return None if AB is None else torch.kron(*AB)
    if kind == "locon_mid":
        return torch.mm(f32(factors[0]).flatten(start_dim=1), locon_mid_down(*factors[1:], device))
    if kind == "loha_tucker":
        w1a, w1b, t1, w2a, w2b, t2 = (f32(t) for t in factors)
        m1 = torch.einsum("i j k l, j r, i p -> p r k l", t1, w1b, w1a)
        m2 = torch.einsum("i j k l, j r, i p -> p r k l", t2, w2b, w2a)
        return (m1 * m2).reshape(m1.shape[0], -1)
    return _dora_delta(kind, factors, device)


def build_conv_dora_plan(W, terms):
    """The cached operands of ggufb200_dequant_patched_dora for recognised `conv_dora_terms` on the dequantised weight W
    ([Cout, Cin, kh, kw] in the activation dtype, on the device of the forward): (tensors to keep, ggufb200_weight_patch array,
    ggufb200_dora_patch array).  The factors s are the reference's own, `dora_replay` of the entries on W; the deltas' operands
    are `conv_lycoris_operands`' with scale alpha for a DoRA entry (the kernel applies its strength in the DoRA step) and
    strength * alpha for a plain one.  None when an entry is a LoKr entry the reference skips."""
    if any(kind == "lokr" and conv_lokr_operands(f, W.device) is None for kind, _st, _a, f, *_rest in terms):
        return None
    factors, _patched = dora_replay(W, [(kind, st, a, f, ds) for kind, st, a, f, _src, ds, _axis in terms], conv_term_delta)
    operands = conv_lycoris_operands([(kind, a if ds is not None else st * a, f, src) for kind, st, a, f, src, ds, _axis in terms], W.device)
    if operands is None:
        return None
    keep, descs = operands
    group = W.shape[2] * W.shape[3]
    s32 = [None if s is None else s.float().contiguous() for s in factors]
    dora = (_lib.DoraPatch * max(1, len(terms)))(*[
        _lib.DoraPatch() if s is None else _lib.DoraPatch(s.data_ptr(), axis, group, st)
        for (_kind, st, _a, _f, _src, _ds, axis), s in zip(terms, s32)])
    return (keep, s32), descs, dora


def lokr_factor_shapes(factors):
    """(a1, a2), (b1, b2) of a recognised LoKr term's A = w1 (or w1_a @ w1_b) and B = w2 (or w2_a @ w2_b)."""
    w1, w2, w1_a, w1_b, w2_a, w2_b = factors
    a = tuple(w1.shape) if w1 is not None else (w1_a.shape[0], w1_b.shape[1])
    b = tuple(w2.shape) if w2 is not None else (w2_a.shape[0], w2_b.shape[1])
    return a, b


def loha_as_lora(w1a, w1b, w2a, w2b, device):
    """LoHa's (w1a @ w1b) * (w2a @ w2b) as one LoRA of rank r1 r2, in fp32: up[:, i r2 + j] = w1a[:, i] * w2a[:, j] and
    down[i r2 + j, :] = w1b[i, :] * w2b[j, :]."""
    f = [t.to(device=device, dtype=torch.float32) for t in (w1a, w1b, w2a, w2b)]
    up = (f[0][:, :, None] * f[2][:, None, :]).reshape(f[0].shape[0], -1)
    down = (f[1][:, None, :] * f[3][None, :, :]).reshape(-1, f[1].shape[1])
    return up, down


def lokr_operands(factors, device):
    """A, B of a LoKr term as comfy.lora.calculate_weight forms them: fp32 factors, a decomposed one as the fp32 torch.mm of its
    halves on `device`."""
    w1, w2, w1_a, w1_b, w2_a, w2_b = factors

    def f32(t):
        return t.to(device=device, dtype=torch.float32)
    A = f32(w1) if w1 is not None else torch.mm(f32(w1_a), f32(w1_b))
    B = f32(w2) if w2 is not None else torch.mm(f32(w2_a), f32(w2_b))
    return A.contiguous(), B.contiguous()


def lycoris_operands(terms, device):
    """(LoRA terms, LoKr patches) of recognised `lycoris_terms` (shapes checked): LoRA entries as they are and LoHa entries as
    LoRA terms of rank r1 r2 (`loha_as_lora`), all (scale, up, down, band); the LoKr entries as ((scale, A, B, band), ...) with
    fp32 A / B on `device` (`lokr_operands`) and their ggufb200_kron_patch array, or None when there are none."""
    lora, kron = [], []
    for kind, scale, factors, band in terms:
        if kind == "lora":
            lora.append((scale, factors[0], factors[1], band))
        elif kind == "loha":
            lora.append((scale, *loha_as_lora(*factors, device), band))
        else:
            kron.append((scale, *lokr_operands(factors, device), band))
    descs = (_lib.KronPatch * max(1, len(kron)))(*[
        _lib.KronPatch(A.data_ptr(), B.data_ptr(), A.shape[0], A.shape[1], B.shape[0], B.shape[1], -1 if band is None else band[0],
                       scale, 0 if band is None else band[1], 0 if band is None else band[2])
        for scale, A, B, band in kron])
    return lora, ((kron, descs) if kron else None)


def lora_kernel_operands(terms, N, K, dtype, device):
    """Pack recognised LoRA terms ([(scale, up, down, band), ...], shapes checked) into the operands of
    ggufb200_linear_lora_ex: down_pad [64 J, K] in `dtype`, U [N, 64 J] fp16 = scale * up, and the per-tile k-block table
    (int32 [ceil(N / 128), 2] of (first, count), or None when no term has a band).  A term takes the next r columns; its up
    rows land on its output band (zero elsewhere), its down columns on its input band.  Terms are ordered by output band, so
    the columns a 128-feature tile needs are contiguous and few: with disjoint q / k / v bands a tile runs only the k-blocks
    of the bands it overlaps."""
    def rows(band):
        return (band[1], band[1] + band[2]) if band is not None and band[0] == 0 else (0, N)

    order = sorted(terms, key=lambda t: rows(t[3]))
    R = sum(down.shape[0] for _s, _u, down, _b in order)
    J = max(1, -(-R // LORA_MAX_RANK))
    down_pad = torch.zeros(J * LORA_MAX_RANK, K, device=device, dtype=dtype)
    u_pad = torch.zeros(N, J * LORA_MAX_RANK, device=device, dtype=torch.float16)
    n_tiles = -(-N // 128)
    lo, hi = [None] * n_tiles, [None] * n_tiles            # column range per 128-feature tile
    r0 = 0
    for scale, up, down, band in order:
        r = down.shape[0]
        n0, n1 = rows(band)
        k0, k1 = (band[1], band[1] + band[2]) if band is not None and band[0] == 1 else (0, K)
        down_pad[r0:r0 + r, k0:k1] = down.to(device=device, dtype=dtype)
        u_pad[n0:n1, r0:r0 + r] = (up.to(device=device, dtype=torch.float32) * scale).to(torch.float16)
        if r:
            for tile in range(n0 // 128, -(-n1 // 128)):
                lo[tile] = r0 if lo[tile] is None else min(lo[tile], r0)
                hi[tile] = r0 + r if hi[tile] is None else max(hi[tile], r0 + r)
        r0 += r
    tiles = None
    if any(band is not None for *_t, band in terms):
        pairs = [(0, 0) if lo[i] is None else (lo[i] // LORA_MAX_RANK, (hi[i] - 1) // LORA_MAX_RANK - lo[i] // LORA_MAX_RANK + 1)
                 for i in range(n_tiles)]
        tiles = torch.tensor(pairs, dtype=torch.int32).to(device)
    return down_pad, u_pad, tiles


def dora_terms(patches):
    """Recognise a patch list of whole-weight LoRA and LoHa entries of which at least one carries DoRA (`dora_scale`).  Returns
    [(kind, strength, a, factors, dora_scale), ...] in list order (`_decode_patch`: a is kept apart from the strength, dora_scale
    is None for a plain entry).  None when the list has no DoRA entry (the other recognisers serve it) or when any entry needs
    `calculate_weight`, has an offset or is LoKr.  The dora_scale's axis is checked against the weight by `dora_axis`."""
    terms = []
    for entry in patches:
        record = _decode_patch(entry, ("lora", "loha"))
        if record is None or record[4] is not None:                            # banded DoRA is not served
            return None
        kind, strength, a, factors, _band, dora_scale = record
        terms.append((kind, strength, a, factors, dora_scale))
    return terms if any(dora_scale is not None for *_t, dora_scale in terms) else None


def dora_axis(dora_scale, N, K):
    """0 when `weight_decompose` normalises an [N, K] weight along the output axis (dora_scale [N, 1]: one norm per row, LyCORIS
    wd_on_out), 1 along the input axis (dora_scale [1, K] or [K]: one norm per column), None for a shape whose reference
    broadcast is not one factor per row or per column.  The reference picks the output axis when dora_scale.shape[0] == N."""
    shape = tuple(dora_scale.shape)
    if shape == (N, 1):
        return 0
    if shape in ((1, K), (K,)) and shape[0] != N:
        return 1
    return None


def _fits_weight(kind, factors, band, N, K):
    """True when a recognised term's delta has the shape of its band of an [N, K] weight (the whole weight for band None) and
    the band lies inside the weight: LoRA / LoHa rows from factors[0] and columns from factors[-1], LoKr a1 b1 x a2 b2."""
    rows, cols = N, K
    if band is not None:
        dim, start, size = band
        if start + size > (N, K)[dim]:
            return False
        rows, cols = (size, K) if dim == 0 else (N, size)
    if kind == "lokr":
        (a1, a2), (b1, b2) = lokr_factor_shapes(factors)
        return a1 * b1 == rows and a2 * b2 == cols
    return factors[0].shape[0] == rows and factors[-1].shape[1] == cols


def _tensor_key(t):
    """Identity, storage, version and shape of a patch factor (None for an absent one): a factor that was swapped for another
    one (even at a recycled id()) or modified in place changes the key of every plan built from it."""
    return None if t is None else (id(t), t.data_ptr(), t._version, tuple(t.shape))


def _cached(owner, slot, key, build):
    """`owner.__dict__[slot]` holds (key, value): the value when its key equals `key`, else `build()`, stored with `key`."""
    cached = owner.__dict__.get(slot)
    if cached is not None and cached[0] == key:
        return cached[1]
    value = build()
    owner.__dict__[slot] = (key, value)
    return value


def _dora_delta(kind, factors, device):
    """The entry's fp32 delta as calculate_weight forms it: up @ down, or (w1a @ w1b) * (w2a @ w2b) for LoHa."""
    f = [t.to(device=device, dtype=torch.float32) for t in factors]
    if kind == "lora":
        return torch.mm(f[0], f[1])
    return torch.mm(f[0], f[1]) * torch.mm(f[2], f[3])


def dora_replay(W, terms, delta_of=_dora_delta):
    """The reference's calculate_weight over recognised `dora_terms` on W ([N, K] in the activation dtype, the dequantised weight,
    or a Conv2d's [Cout, Cin, kh, kw]; not modified), in the same ops, dtype and device.  Returns each entry's DoRA factor s (W's
    dtype, [N] / [Cout] for the output axis, [K] / [Cin] for the input axis; None for an entry without DoRA) and the patched
    weight.  Per entry with strength st and alpha a, delta = delta_of(kind, factors, device) as calculate_weight forms it:
        plain   W += ((st * a) * delta).to(W.dtype)
        DoRA    Wc = W + (delta * a).to(W.dtype)
                nrm = norms of W's rows W.reshape(N, -1) (output axis: the weight BEFORE this patch) or of Wc's input slices
                      Wc.transpose(0, 1).reshape(W.shape[1], -1) (input axis), + eps(W.dtype)
                s = (fp32(dora_scale) / nrm).to(W.dtype);  Wc *= s
                W = Wc if st == 1 else W + st * (Wc - W)"""
    W = W.clone()
    N = W.shape[0]
    ones = [1] * (W.dim() - 1)
    eps = torch.finfo(W.dtype).eps
    factors = []
    for kind, strength, alpha, fac, dora_scale in terms:
        delta = delta_of(kind, fac, W.device).reshape(W.shape)
        if dora_scale is None:
            W += ((strength * alpha) * delta).to(W.dtype)
            factors.append(None)
            continue
        delta *= alpha
        Wc = W + delta.to(W.dtype)
        if dora_scale.shape[0] == N:
            nrm = W.reshape(N, -1).norm(dim=1, keepdim=True).reshape(N, *ones)
        else:
            C = W.shape[1]
            nrm = Wc.transpose(0, 1).reshape(C, -1).norm(dim=1, keepdim=True).reshape(C, *ones).transpose(0, 1)
        nrm = nrm + eps
        s = (dora_scale.to(device=W.device, dtype=torch.float32) / nrm).to(W.dtype)
        Wc *= s
        if strength != 1.0:
            Wc -= W
            W += strength * Wc
        else:
            W = Wc
        factors.append(s.reshape(-1))
    return factors, W


def dora_compact(terms, factors, N, K):
    """The patched weight of `dora_replay` in the compact form
        W_final = diag(r) W0 diag(c) + sum_j diag(rho_j) (a_j st_j up_j down_j) diag(gamma_j)
    with the reference's factors s: a plain entry appends a term with rho = gamma = 1; an output-axis DoRA entry multiplies r
    and every earlier rho_j by (1 - st + st s) and appends its term with rho = s; an input-axis entry does the same to c and
    the gamma_j.  Returns r [N], c [K], [(a_j st_j, rho_j [N] or None, gamma_j [K] or None)] in float64 (None = ones)."""
    dev = next(s.device for s in factors if s is not None)
    r = torch.ones(N, dtype=torch.float64, device=dev)
    c = torch.ones(K, dtype=torch.float64, device=dev)
    rho, gamma, coef = [], [], []
    for (_kind, strength, alpha, _fac, dora_scale), s in zip(terms, factors):
        coef.append(strength * alpha)
        if s is None:
            rho.append(None)
            gamma.append(None)
            continue
        s = s.double()
        f = 1.0 - strength + strength * s
        if dora_scale.shape[0] == N:
            r *= f
            rho = [f if p is None else p * f for p in rho] + [s]
            gamma.append(None)
        else:
            c *= f
            gamma = [f if g is None else g * f for g in gamma] + [s]
            rho.append(None)
    return r, c, list(zip(coef, rho, gamma))


class DoraPlan:
    """What a DoRA patch set costs per forward, built once (`build_dora_plan`):
        r       fp32 [N] output feature scale (ggufb200_*_scaled)
        c       fp32 [K] input feature scale (ggufb200_scale_columns) or None when no entry normalises the input axis
        down    [R, K] activation dtype: the down'_j = down_j diag(gamma_j), stacked
        up      [N, R] activation dtype: a_j st_j diag(rho_j) up_j, the side GEMMs' up-projection
        kernel  (down_pad, u_pad) of ggufb200_linear_lora_scaled with U_j = a_j st_j diag(rho_j / r) up_j in fp16, or None when
                R > LORA_KERNEL_MAX_RANK, some r_n == 0 or some rho_j / r is not finite in fp16 (then the side form serves)."""

    def __init__(self, r, c, down, up, kernel):
        self.r, self.c, self.down, self.up, self.kernel = r, c, down, up, kernel


def build_dora_plan(W, terms, dtype):
    """DoraPlan of recognised `dora_terms` (shapes checked) for the dequantised weight W ([N, K], `dtype`, on the device of the
    forward)."""
    N, K = W.shape
    dev = W.device
    factors, _patched = dora_replay(W, terms)
    r, c, compact = dora_compact(terms, factors, N, K)
    ups, downs = [], []
    for (kind, _st, _a, fac, _ds), (coef, rho, gamma) in zip(terms, compact):
        up, down = (fac[0].to(device=dev, dtype=torch.float32), fac[1].to(device=dev, dtype=torch.float32)) if kind == "lora" \
            else loha_as_lora(*fac, dev)
        ups.append(up.double() * (coef if rho is None else coef * rho[:, None]))
        downs.append(down.double() if gamma is None else down.double() * gamma[None, :])
    up = torch.cat(ups, 1)
    down = torch.cat(downs, 0).to(dtype)
    kernel = None
    if down.shape[0] <= LORA_KERNEL_MAX_RANK and bool((r != 0).all()):
        down_pad, u_pad, _tiles = lora_kernel_operands([(1.0, (up / r[:, None]).float(), down, None)], N, K, dtype, dev)
        if bool(torch.isfinite(u_pad).all()):
            kernel = (down_pad, u_pad)
    has_c = any(g is not None for _coef, _rho, g in compact)            # some entry normalises the input axis
    return DoraPlan(r.float(), c.float() if has_c else None, down, up.to(dtype), kernel)


class GGMLLayer(torch.nn.Module):
    """Base of every GGUF-aware op: state-dict plumbing for packed tensors and on-the-fly weight materialisation.

    Mirrors the reference class of the same name (ops.py:93-225): same attributes (`comfy_cast_weights`, `dequant_dtype`,
    `patch_dtype`, `largest_layer`) and the same method names, because ComfyUI and the loader nodes address them by name."""
    comfy_cast_weights = True
    dequant_dtype = None
    patch_dtype = None
    largest_layer = False
    torch_compatible_tensor_types = {None, _Q.F32, _Q.F16}

    # ------------------------------------------------------------------ predicates
    def is_ggml_quantized(self, *, weight=None, bias=None):
        w = self.weight if weight is None else weight
        b = self.bias if bias is None else bias
        return is_quantized(w) or is_quantized(b)

    def _takes_ggml_load_path(self, weight, bias):
        if isinstance(self, torch.nn.Linear):            # Linear never allocates, so it always loads by assignment
            return True
        if self.is_ggml_quantized(weight=weight, bias=bias):
            return True
        return isinstance(self, torch.nn.Embedding) and self.weight.shape[0] >= _BIG_EMBEDDING_ROWS

    # ------------------------------------------------------------------ load: adopt the tensors of the state dict as they are
    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        if self._takes_ggml_load_path(state_dict.get(prefix + "weight"), state_dict.get(prefix + "bias")):
            return self.ggml_load_from_state_dict(state_dict, prefix, *args, **kwargs)
        return super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def ggml_load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        cut = len(prefix)
        for full_key, tensor in state_dict.items():
            leaf = full_key[cut:]
            if leaf == "weight" or (leaf == "bias" and tensor is not None):
                # nn.Parameter(GGMLTensor) is the very same object: detach()/clone() return self
                setattr(self, leaf, torch.nn.Parameter(tensor, requires_grad=False))
            else:
                unexpected_keys.append(full_key)
        if isinstance(self, torch.nn.Linear) and self.weight is None:
            placeholder = torch.zeros(self.in_features, self.out_features)      # shape quirk kept from ops.py:131-134
            self.weight = torch.nn.Parameter(placeholder, requires_grad=False)
            missing_keys.append(prefix + "weight")
        self.largest_layer = self.largest_layer or bool(getattr(self.weight, "is_largest_weight", False))

    # ------------------------------------------------------------------ save: meta stand-ins for the host's VRAM estimate
    def _save_to_state_dict(self, *args, **kwargs):
        if not self.is_ggml_quantized():
            return super()._save_to_state_dict(*args, **kwargs)
        return self.ggml_save_to_state_dict(*args, **kwargs)

    def ggml_save_to_state_dict(self, destination, prefix, keep_vars):
        for leaf in ("weight", "bias"):
            tensor = getattr(self, leaf)
            if tensor is not None:
                destination[prefix + leaf] = torch.zeros_like(tensor, device=_META)
        if self.largest_layer:
            # room for the largest dequantised weight (the two-step route's scratch), reported like the reference does
            logical = getattr(self.weight, "tensor_shape", self.weight.shape)
            explicit = self.dequant_dtype not in (None, "target")
            destination[prefix + "temp.weight"] = torch.empty(*logical, device=_META,
                                                              dtype=self.dequant_dtype if explicit else torch.float16)

    # ------------------------------------------------------------------ weight materialisation (two-step route)
    def get_weight(self, tensor, dtype):
        """Dequantise `tensor` (ONE kernel launch) and apply attached LoRA patches; returns a plain torch.Tensor."""
        if tensor is None:
            return None
        patches, key = _collect_patches(tensor)          # patches start moving to the device before the dequant launch
        dense = _plain(dequantize_tensor(tensor, dtype, self.dequant_dtype))
        if not patches:
            return dense
        if self.patch_dtype is None:
            return comfy_lora.calculate_weight(patches, dense, key)
        return comfy_lora.calculate_weight(patches, dense, key, dtype if self.patch_dtype == "target" else self.patch_dtype)

    @torch_compiler_disable()
    def cast_bias_weight(s, input=None, dtype=None, device=None, bias_dtype=None):
        if input is not None:                            # unspecified targets follow the activation
            dtype = getattr(input, "dtype", torch.float32) if dtype is None else dtype
            bias_dtype = dtype if bias_dtype is None else bias_dtype
            device = input.device if device is None else device
        async_ok = comfy_mm.device_supports_non_blocking(device)

        def materialise(param, want):
            dense = s.get_weight(param.to(device), dtype)
            return comfy_ops.cast_to(dense, want, device, non_blocking=async_ok, copy=False)

        bias = materialise(s.bias, bias_dtype) if s.bias is not None else None      # bias first, as in ops.py:205-207
        return materialise(s.weight, dtype), bias

    # ------------------------------------------------------------------ forward dispatch
    def forward_comfy_cast_weights(self, input, *args, **kwargs):
        route = self.forward_ggml_cast_weights if self.is_ggml_quantized() else super().forward_comfy_cast_weights
        return _plain(route(input, *args, **kwargs))      # never leak the tensor subclass to the host

    def forward_ggml_cast_weights(self, input):
        raise NotImplementedError


class GGMLOps(comfy_ops.manual_cast):
    """`custom_operations` object handed to comfy.sd loaders (ops.py:227-271)."""

    class Linear(GGMLLayer, comfy_ops.manual_cast.Linear):
        def __init__(self, in_features, out_features, bias=True, device=None, dtype=None):
            torch.nn.Module.__init__(self)   # allocates nothing (ops.py:232-240)
            self.in_features = in_features
            self.out_features = out_features
            self.weight = None
            self.bias = None

        # LoRA on a packed weight as rank-r side GEMMs on top of the packed-weight Linear (SURVEY 8f rank 1):
        #   y = x W^T + b + sum_i scale_i (x down_i^T) up_i^T
        # instead of dequantise + calculate_weight + F.linear on every forward (ops.py:171-190).  W + delta is then never
        # rounded to the activation dtype, so the result differs from the reference by that one rounding (parity budget in
        # tests/test_gpu_linear.py); set to False to get the reference's two-step arithmetic back.
        lora_side_gemm = True

        # Numerics contract of the packed-weight Linear (DESIGN.md section 3, include/ggufb200.h GGUFB200_FLAG_EXACT_W):
        #   "exact"  (default) the weight operand of every route is bit-identical to the reference's
        #            `dequantize_tensor(...).to(dtype)`; only the fp32 summation order differs (<= 1e-3, measured <= 3e-4)
        #   "fast"   the FUSED_TMEM kernel runs its fused-multiply-add producers (Q4_K / Q5_K: one rounding instead of two per
        #            element; 1e-3 for fp16 activations, 8e-3 for bf16) -- only pays off where the producers, not the tensor
        #            pipe, bound the kernel (small M)
        linear_numerics = "exact"
        # Weights whose canonical rows the TMA engine cannot stage (Q2_K / Q3_K / Q6_K / IQ4_XS, Q8_0 at K = 2432 ...) get a
        # re-packed span-major shadow copy on first use (one extra copy of the packed bytes in HBM, csrc/repack.cu) so that
        # they too run on the FUSED_TMEM kernel; False keeps them on the round-1 routes (smem-fed fused / dequant + dense GEMM).
        # Straddled weights (`straddled_rows`) get no copy: dequant + dense GEMM was the faster route for them at every M measured.
        repack_spans = True

        def _fused_ok(self, input):
            w = self.weight
            return (input.is_cuda and input.dtype in _FUSED_ACT and is_quantized(w)
                    and not is_quantized(self.bias) and len(getattr(w, "tensor_shape", ())) == 2
                    and not getattr(self.bias, "patches", None))

        def _lora_terms(self, dev):
            """[] for an unpatched weight, the side-GEMM terms for a LoRA-only patch list, None -> two-step route."""
            w = self.weight
            if not getattr(w, "patches", None):
                return []
            if not self.lora_side_gemm or self.patch_dtype not in (None, "target"):
                return None
            terms = lora_band_terms(_patch_entries(w))
            N, K = tuple(w.tensor_shape)
            if terms is None or not all(_fits_weight("lora", (up, down), band, N, K) for _s, up, down, band in terms):
                return None
            return terms

        # LoRA inside the fused kernel (GGUFB200_ALGO_FUSED_TMEM, csrc/linear_sm90.cu: J <= 8 extra k-blocks, SURVEY 8f rank 1):
        # U = scale * up (fp16 [N, 64 J]), down (act dtype [64 J, K]) and, for row-band patches, the per-tile k-block table are
        # cached per patch set (`lora_kernel_operands`); per forward only T = x * down^T ([M, 64 J], this package's dense
        # tensor-core GEMM) is computed before the fused call.
        # False -> the unpatched fused kernel plus library GEMMs of rank sum(r) (`_add_lora`), as for sum(r) > 512.
        lora_in_kernel = True

        def _lora_operands(self, terms, dev, dtype):
            """`lora_kernel_operands` of `_lora_terms`, cached per patch set, device and activation dtype; None when U = scale * up
            does not fit fp16 (or down the activation dtype): the side GEMMs, whose U is in the activation dtype, serve those."""
            key = tuple((float(scale), band, _tensor_key(up), _tensor_key(down)) for scale, up, down, band in terms) + (str(dev), dtype)

            def build():
                down_pad, u_pad, tiles = lora_kernel_operands(terms, *self.weight.tensor_shape, dtype, dev)
                return (down_pad, u_pad, tiles) if bool(torch.isfinite(u_pad).all()) and bool(torch.isfinite(down_pad).all()) else None
            return _cached(self, "_gg_lora", key, build)

        def _patches_finite(self, dev, dtype, terms):
            """False when a tensor of the weight's patch entries holds NaN / Inf, or a LoRA-form term's scale * up or down (the
            side GEMMs' operands) does not fit the activation dtype.  Such a patch set takes the two-step route: a factorised
            evaluation sums the rank terms before an infinity meets them (an Inf in up is NaN in the reference's x W'^T, +-Inf in
            t u^T; a NaN in a banded term's factor would reach the rows of its tile outside the band), so only the reference's
            own arithmetic gives its NaN / Inf pattern.  Cached per patch set, device and activation dtype."""
            tensors = [t for entry in _patch_entries(self.weight) for t in _entry_tensors(entry)]
            key = tuple(map(_tensor_key, tensors)) + tuple(float(s) for s, *_r in terms or ()) + (str(dev), dtype)

            def build():
                if not all(bool(torch.isfinite(t).all()) for t in tensors):
                    return False
                return all(bool(torch.isfinite((up.to(device=dev, dtype=torch.float32) * scale).to(dtype)).all())
                           and bool(torch.isfinite(down.to(device=dev, dtype=dtype)).all()) for scale, up, down, _band in terms or ())
            return _cached(self, "_gg_finite", key, build)

        def _lycoris_terms(self, dev):
            """For a patch list with LoHa / LoKr entries (`lycoris_terms`, any mix with LoRA): `lycoris_operands` on `dev`, cached
            per patch set.  None -> two-step route (also for patch_dtype other than None: the reference then forms the delta in
            another dtype)."""
            w = self.weight
            if not self.lora_side_gemm or self.patch_dtype is not None:
                return None
            terms = lycoris_terms(_patch_entries(w))
            N, K = tuple(w.tensor_shape)
            if terms is None or not all(_fits_weight(kind, factors, band, N, K) for kind, _s, factors, band in terms):
                return None
            key = tuple((kind, float(scale), band) + tuple(map(_tensor_key, factors)) for kind, scale, factors, band in terms) + (str(dev),)
            return _cached(self, "_gg_lycoris", key, lambda: lycoris_operands(terms, dev))

        def _kron_linear(self, input, wraw, qtype, N, K, bias, kron):
            """ggufb200_dequant_kron (the patched weight, bit-identical to the reference's) into an [N, K] workspace, then
            ggufb200_gemm with the bias."""
            patches, descs = kron
            dev = input.device
            if not wraw.is_contiguous():
                wraw = wraw.contiguous()
            W = torch.empty(N, K, dtype=input.dtype, device=dev)
            # the packed weight is a parameter (or its host-to-device copy): never written by a kernel in flight
            math = math_code(self.dequant_dtype, input.dtype) | _lib.DEQUANT_SRC_STABLE
            with torch.cuda.device(dev):
                rc = _lib.lib().ggufb200_dequant_kron(int(qtype), wraw.data_ptr(), N, K, W.data_ptr(), dtype_code(input.dtype), math, descs,
                                                      len(patches), _current_stream_ptr(dev.index))
            _lib.check(rc, f"ggufb200_dequant_kron({getattr(qtype, 'name', qtype)}, N={N}, K={K})")
            return linear_dense(input, W, bias)

        def _add_lora(self, y, input, terms):
            x2 = input.reshape(-1, input.shape[-1])
            y2 = y.view(-1, y.shape[-1])
            if any(band is not None for *_t, band in terms):     # one pair of GEMMs per term, on its bands of x and y
                for scale, up, down, band in terms:
                    xs = x2[:, band[1]:band[1] + band[2]] if band is not None and band[0] == 1 else x2
                    ys = y2[:, band[1]:band[1] + band[2]] if band is not None and band[0] == 0 else y2
                    t = xs @ down.to(device=x2.device, dtype=x2.dtype, non_blocking=True).t()
                    ys.addmm_(t, (up.to(device=x2.device, dtype=torch.float32, non_blocking=True) * scale).to(x2.dtype).t())
                return y
            if len(terms) == 1:
                scale, up, down, _band = terms[0]
                down_all = down.to(device=x2.device, dtype=x2.dtype, non_blocking=True)
                up_all = up.to(device=x2.device, dtype=torch.float32, non_blocking=True) * scale
            else:                                                   # one pair of GEMMs for any number of LoRAs
                down_all = torch.cat([d.to(device=x2.device, dtype=x2.dtype, non_blocking=True) for _s, _u, d, _b in terms], 0)
                up_all = torch.cat([u.to(device=x2.device, dtype=torch.float32, non_blocking=True) * s for s, u, _d, _b in terms], 1)
            t = x2 @ down_all.t()                                   # [M, R]   library GEMMs: R is tens, not thousands
            y2.addmm_(t, up_all.to(x2.dtype).t())
            return y

        # DoRA (weight-decomposed LoRA, `dora_terms`): a list of whole-weight LoRA / LoHa entries with DoRA factors keeps the form
        #   W_final = diag(r) W0 diag(c) + sum_j diag(rho_j) (a_j st_j up_j down_j) diag(gamma_j)
        # (`dora_compact`; the factors are the reference's own, replayed once per patch set on the dequantised weight), so
        #   y = r * ((x diag(c)) W0^T) + sum_j (x down'_j^T) (a_j st_j diag(rho_j) up_j)^T + b,   down'_j = down_j diag(gamma_j).
        # In-kernel (`_takes_lora_kblocks`): ggufb200_linear_lora_scaled with feature scale r and U_j = a_j st_j diag(rho_j / r)
        # up_j.  Side form (everything else): the dequantised weight, ggufb200_gemm_scaled with r, plus the side GEMMs.
        def _dora_terms(self):
            """`dora_terms` of the weight's patch list with every factor and dora_scale shape checked against [N, K]; None -> two-step
            route (also for lora_side_gemm = False and a patch_dtype other than None)."""
            w = self.weight
            if not self.lora_side_gemm or self.patch_dtype is not None:
                return None
            terms = dora_terms(_patch_entries(w))
            N, K = tuple(w.tensor_shape)
            if terms is None or not all(_fits_weight(kind, factors, None, N, K) and (ds is None or dora_axis(ds, N, K) is not None)
                                        for kind, _st, _a, factors, ds in terms):
                return None
            return terms

        def _dense_weight(self, wraw, qtype, N, K, dtype):
            """dequantize_tensor(weight, dtype, self.dequant_dtype) of the packed bytes `wraw` (on the forward's device): [N, K] in dtype."""
            if qtype in FALLBACK_QTYPES:
                return dequantize_fallback(wraw, qtype, (N, K), dtype)
            if qtype == _Q.BF16 and dtype == torch.bfloat16:
                return wraw.view(torch.bfloat16).view(N, K)
            return dequantize(wraw, qtype, (N, K), dtype=dtype if self.dequant_dtype == "target" else self.dequant_dtype, out_dtype=dtype)

        def _dora_plan(self, terms, src, wraw, qtype, N, K, dev, dtype):
            """`build_dora_plan`, cached per patch set: identity + storage + version of every factor and dora_scale, the strengths,
            the weight's storage, the device, the activation dtype and dequant_dtype (the factors s depend on all of them)."""
            key = tuple((kind, st, a) + tuple(map(_tensor_key, factors + (ds,))) for kind, st, a, factors, ds in terms) \
                + (id(self.weight), src.data_ptr(), src._version, str(dev), dtype, self.dequant_dtype)
            return _cached(self, "_gg_dora", key, lambda: build_dora_plan(self._dense_weight(wraw, qtype, N, K, dtype), terms, dtype))

        def _dora_linear(self, input, terms, src, wraw, resident, bias, M):
            """y for a DoRA patch list (`_dora_terms`) on a weight with N and K multiples of 8; the other arguments as
            `forward_ggml_cast_weights` prepares them."""
            w = self.weight
            qtype, (N, K) = w.tensor_type, w.tensor_shape
            dev, dtype = input.device, input.dtype
            if not wraw.is_contiguous():
                wraw = wraw.contiguous()
            plan = self._dora_plan(terms, src, wraw, qtype, N, K, dev, dtype)
            x2 = input.reshape(-1, K)
            xs = x2 if plan.c is None else scale_columns(x2, plan.c)
            math = math_code(self.dequant_dtype, dtype)
            exact = (_lib.FLAG_EXACT_W if self.linear_numerics != "fast" else 0) | _lib.FLAG_W_STABLE
            spans = span_layout(w, wraw) if self._takes_span_copy(qtype, N, K, M, math, resident) else None
            if plan.kernel is not None and self._takes_lora_kblocks(qtype, N, K, math, spans):
                down_pad, u_pad = plan.kernel
                t = linear_dense(x2, down_pad)                                     # T = x * down'^T, [M, 64 J]
                y = _launch_linear(xs, wraw, qtype, N, K, bias, math, _lib.ALGO_FUSED_TMEM | exact, spans, (t, u_pad, None), plan.r)
            else:
                y = linear_dense(xs, self._dense_weight(wraw, qtype, N, K, dtype), bias, plan.r)
                y.addmm_(x2 @ plan.down.t(), plan.up.t())
            return y.reshape(*input.shape[:-1], N)

        def _takes_span_copy(self, qtype, N, K, M, math, resident):
            """True when the FUSED_TMEM kernel reads the re-packed span-major copy of the weight (`span_layout`): the canonical
            rows cannot be staged by TMA and the copy is allowed, resident, and worth it at this M."""
            return (self.repack_spans and resident and M > GEMV_MAX_M and math == _F16_CODE and N % 8 == 0 and qtype != _Q.BF16
                    and needs_span_layout(qtype, K) and qtype not in FALLBACK_QTYPES and not straddled_rows(qtype, K))

        def _takes_lora_kblocks(self, qtype, N, K, math, spans):
            """True when the FUSED_TMEM kernel may run LoRA k-blocks on this weight (`lora_in_kernel`); the caller adds its rank
            limit.  `spans`: the span copy the forward reads, or None."""
            return (self.lora_in_kernel and math == _F16_CODE and N % 8 == 0 and qtype != _Q.BF16 and qtype not in FALLBACK_QTYPES
                    and (spans is not None or not needs_span_layout(qtype, K)))

        # Autograd (`grad_needed`): an unpatched weight keeps the route it takes without gradients, wrapped in
        # PackedLinearFunction (same output bits; the backward is ggufb200_linear_grad_input on the packed bytes, no dense W is
        # saved); a plain or banded LoRA list takes that base plus its side terms in torch ops (`lora_side_sum`, gradients for x,
        # up and down); every other patch list takes the two-step route, the reference's own differentiable arithmetic.
        def forward_ggml_cast_weights(self, input):
            y = None
            if self._fused_ok(input):
                dev = input.device
                grad = grad_needed(input, self.weight)
                terms, kron, dora = self._lora_terms(dev), None, None
                if terms is None and self.weight.tensor_type not in FALLBACK_QTYPES and not grad:
                    lycoris = self._lycoris_terms(dev)                 # LoHa / LoKr entries: LoRA terms + LoKr patches
                    if lycoris is not None:
                        terms, kron = lycoris
                if terms is None and not grad:
                    dora = self._dora_terms()                          # tried after the LoRA and LyCORIS recognisers declined
                if (terms or kron is not None or dora is not None) and not self._patches_finite(dev, input.dtype, terms):
                    terms, kron, dora = None, None, None                # non-finite factors: the two-step route
                if terms is not None or dora is not None:
                    w = self.weight
                    qtype, (N, K) = w.tensor_type, w.tensor_shape      # plain Python attributes: no subclass dispatch
                    src = w.as_subclass(torch.Tensor)
                    resident = src.device == dev
                    wraw = src if resident else src.to(dev)            # offloaded module: packed bytes H2D
                    b = self.bias
                    if b is not None:
                        b = _plain(b)
                        if b.device != dev:
                            b = b.to(dev)
                    M = input.numel() // K if input.shape[-1] == K else -1
                    run = None                                         # the unpatched forward, where a kernel route serves it
                    if M < 0:
                        pass                                           # feature mismatch: let F.linear raise the usual error
                    elif dora is not None:
                        if N % 8 == 0 and K % 8 == 0:
                            y = self._dora_linear(input, dora, src, wraw, resident, b, M)
                    elif qtype in FALLBACK_QTYPES:
                        # numpy-fallback types (csrc/fallback.cuh): above M = 8, whole-block rows run on ggufb200_linear_fallback
                        # where its AUTO decodes the weight from the packed bytes (FUSED_SYNC); everywhere else (AUTO's
                        # DEQUANT_MMA, M <= 8, rows that straddle blocks) K1 into an [N, K] activation-dtype weight (the
                        # reference's fp32 -> dtype rounding) + the dense GEMM; other shapes: two-step route.
                        # Where AUTO would take DEQUANT_MMA the layer keeps issuing the two library calls itself instead of
                        # one ggufb200_linear_fallback: the work and the bits are the same, and callers that trace the layer
                        # by the entry points it calls (tests/test_gpu_linear_grad.py::test_no_grad_path_unchanged watches
                        # ggufb200_dequant_fallback and ggufb200_gemm at M = 300) keep seeing the route they saw before.
                        # Do not fold this back into one AUTO call.
                        if (M > GEMV_MAX_M and N % 8 == 0 and K % 8 == 0 and K % gguf.GGML_QUANT_SIZES[qtype][0] == 0
                                and _lib.lib().ggufb200_linear_fallback_route(int(qtype), M, N, K, dtype_code(input.dtype),
                                                                              _lib.ALGO_AUTO) == _lib.ALGO_FUSED_SYNC):
                            def run():
                                return linear_fallback(input, wraw, qtype, N, K, b)
                        elif N % 8 == 0 and K % 8 == 0:
                            def run():
                                return linear_dense(input, dequantize_fallback(wraw, qtype, (N, K), input.dtype), b)
                    elif kron is not None:
                        # LoKr: the patched weight in one K1 launch + the dense GEMM at every M; LoRA / LoHa terms as side GEMMs
                        if qtype != _Q.BF16 and N % 8 == 0 and K % 8 == 0 and len(kron[0]) <= KRON_MAX_PATCHES:
                            y = self._kron_linear(input, wraw, qtype, N, K, b, kron)
                    elif qtype == _Q.BF16 and M > GEMV_MAX_M:
                        if input.dtype == torch.bfloat16 and K % 8 == 0 and N % 8 == 0:   # already dense: straight to the tensor-core GEMM
                            def run():
                                return linear_dense(input, wraw.view(torch.bfloat16).view(N, K), b)
                    elif M <= GEMV_MAX_M or N % 8 == 0:                # (the M <= 8 kernel stores per element: any N)
                        math = math_code(self.dequant_dtype, input.dtype)
                        # W_STABLE: the packed weight is a parameter (or its host-to-device copy just above): never written by a
                        # kernel in flight
                        exact = (_lib.FLAG_EXACT_W if self.linear_numerics != "fast" else 0) | _lib.FLAG_W_STABLE
                        algo, spans = _lib.ALGO_AUTO | exact, None
                        if self._takes_span_copy(qtype, N, K, M, math, resident):
                            spans = span_layout(w, wraw)               # cached on the tensor after the first forward
                            algo = _lib.ALGO_FUSED_TMEM | exact
                        if (terms and not grad and self._takes_lora_kblocks(qtype, N, K, math, spans)
                                and sum(d.shape[0] for _s, _u, d, _b in terms) <= LORA_KERNEL_MAX_RANK):
                            operands = self._lora_operands(terms, dev, input.dtype)
                            if operands is not None:
                                down_pad, u_pad, tiles = operands
                                lora = (linear_dense(input.reshape(-1, K), down_pad), u_pad, tiles)       # T = x * down^T, [M, 64 J]
                                return _launch_linear(input, wraw, qtype, N, K, b, math, _lib.ALGO_FUSED_TMEM | exact, spans, lora)

                        def run():
                            return _launch_linear(input, wraw, qtype, N, K, b, math, algo, spans)
                    if run is not None:
                        if not grad:
                            y = run()
                        else:
                            math = math_code(self.dequant_dtype, input.dtype)
                            y = PackedLinearFunction.apply(input, wraw, run, qtype, N, K, math)
                            return lora_side_sum(y, input, terms) if terms else y
                    if y is not None and terms:
                        y = self._add_lora(y, input, terms)
            if y is not None:
                return y
            weight, bias = self.cast_bias_weight(input)
            return torch.nn.functional.linear(input, weight, bias)

    class Conv2d(GGMLLayer, comfy_ops.manual_cast.Conv2d):
        # LoRA / LoCon and LoHa patches (`conv_patch_terms`) on a packed weight: the patched weight [Cout, Cin, kh, kw] in one
        # launch of ggufb200_dequant_lowrank, which forms each element's rank sums from staged factor tiles instead of
        # dequantise + calculate_weight's fp32 [Cout, Cin kh kw] delta, scale, cast and add.  Same per-element rounding sequence;
        # only the order of the rank sums differs from torch.mm.  Taken where its cost model says it wins (`lowrank_pays`: high
        # ranks on small weights keep the two-step route).
        # Lists with LoKr, LoCon `mid` or Tucker LoHa entries (`conv_lycoris_terms`) take ggufb200_dequant_patched the same way,
        # LoKr as a Kronecker patch (bit-identical to the reference's), the Tucker factors composed once per patch set.  (K1 with
        # the Kronecker patch, ggufb200_dequant_kron, measured slower for LoKr factors 4 and 8 and within 4 % at 16.)
        # Lists with DoRA entries (`conv_dora_terms`) take ggufb200_dequant_patched_dora: the factors s of weight_decompose are
        # replayed once per patch set on the dequantised weight (`build_conv_dora_plan`), and the kernel applies each entry's
        # delta, factor and strength blend per element, in the reference's rounding sequence.
        # False -> the reference's two-step arithmetic everywhere.
        conv_patches_in_kernel = True

        def _conv_kernel_shape(self, input):
            """(qtype, N, K) of a patched packed weight the patch kernels can serve for this input, or None."""
            w = self.weight
            if not (self.conv_patches_in_kernel and input.is_cuda and input.dtype in _LOWRANK_ACT and is_quantized(w)
                    and self.patch_dtype is None and not is_quantized(self.bias) and getattr(w, "patches", None)):
                return None
            qtype, shape = w.tensor_type, tuple(getattr(w, "tensor_shape", ()))
            if qtype not in _LOWRANK_QTYPES or len(shape) != 4:
                return None
            N, K = shape[0], shape[1] * shape[2] * shape[3]
            if K % 32 != 0 or (N * K) % gguf.GGML_QUANT_SIZES[qtype][0] != 0:
                return None
            return qtype, N, K

        def _conv_patch_operands(self, input):
            """`conv_patch_operands` of the weight's patch list, cached per patch set and device; None -> not served."""
            geometry = self._conv_kernel_shape(input)
            if geometry is None:
                return None
            _qtype, N, K = geometry
            terms = conv_patch_terms(_patch_entries(self.weight))
            if not terms or len(terms) > _lib.LOWRANK_MAX_PATCHES or not all(
                    _fits_weight(kind, factors, None, N, K) and max(f.shape[0] for f in factors[1::2]) <= _lib.LOWRANK_MAX_RANK
                    for kind, _s, factors, _src in terms) or not lowrank_pays(N, K, terms):
                return None
            dev = input.device
            key = tuple((kind, float(scale)) + tuple(map(_tensor_key, sources)) for kind, scale, _f, sources in terms) + (str(dev),)
            return _cached(self, "_gg_conv", key, lambda: conv_patch_operands(terms, dev))

        def _conv_lycoris_operands(self, input):
            """`conv_lycoris_operands` of a list with LoKr / LoCon mid / Tucker LoHa entries (`conv_lycoris_terms`), cached per
            patch set and device, where `lowrank_pays` expects ggufb200_dequant_patched to win; None -> two-step route."""
            geometry = self._conv_kernel_shape(input)
            if geometry is None:
                return None
            _qtype, N, K = geometry
            terms = conv_lycoris_terms(_patch_entries(self.weight))
            if not terms or len(terms) > _lib.LOWRANK_MAX_PATCHES or not all(
                    conv_term_shape(kind, factors) == (N, K) and max(conv_term_ranks(kind, factors), default=0) <= _lib.LOWRANK_MAX_RANK
                    for kind, _s, factors, _src in terms) or not lowrank_pays(N, K, terms):
                return None
            dev = input.device
            key = tuple((kind, float(scale)) + tuple(map(_tensor_key, sources)) for kind, scale, _f, sources in terms) + (str(dev),)
            # None (a LoKr entry the reference skips) is cached too
            return _cached(self, "_gg_conv_lycoris", key, lambda: conv_lycoris_operands(terms, dev))

        def _conv_dora_plan(self, input):
            """`build_conv_dora_plan` of a list with DoRA entries (`conv_dora_terms`), cached per patch set and activation dtype
            (one slot per dtype), where `conv_dora_pays` expects ggufb200_dequant_patched_dora to win; None -> two-step route.
            The key holds every factor and dora_scale (identity, storage, version), the strengths, the packed weight (identity,
            storage, version), the device and dequant_dtype: the factors s depend on all of them."""
            geometry = self._conv_kernel_shape(input)
            if geometry is None:
                return None
            _qtype, N, K = geometry
            w = self.weight
            shape = tuple(w.tensor_shape)
            terms = conv_dora_terms(_patch_entries(w), shape)
            if terms is None or not conv_dora_pays(N, K, terms):
                return None
            dev, dtype = input.device, input.dtype
            src = w.as_subclass(torch.Tensor)
            key = tuple((kind, st, a) + tuple(map(_tensor_key, sources)) for kind, st, a, _f, sources, _ds, _axis in terms) \
                + (id(w), src.data_ptr(), src._version, str(dev), self.dequant_dtype)

            def build():
                W = _plain(dequantize_tensor(w if src.device == dev else w.to(dev), dtype, self.dequant_dtype))
                return build_conv_dora_plan(W, terms)
            # None (a LoKr entry the reference skips) is cached too
            return _cached(self, "_gg_conv_dora_" + str(dtype).split(".")[-1], key, build)

        def forward_ggml_cast_weights(self, input):
            if grad_needed(input, self.weight):                       # the patch kernels' weight carries no gradient
                weight, bias = self.cast_bias_weight(input)
                return self._conv_forward(input, weight, bias)
            entry, operands = "ggufb200_dequant_lowrank", self._conv_patch_operands(input)
            if operands is None:
                entry, operands = "ggufb200_dequant_patched", self._conv_lycoris_operands(input)
            dora = None
            if operands is None:
                plan = self._conv_dora_plan(input)
                if plan is not None:
                    entry, (keep, _s), descs, dora = "ggufb200_dequant_patched_dora", *plan
                    operands = keep, descs
            if operands is None:
                weight, bias = self.cast_bias_weight(input)
                return self._conv_forward(input, weight, bias)
            keep, descs = operands
            dev, dtype = input.device, input.dtype
            bias = None
            if self.bias is not None:                                  # as cast_bias_weight brings it in, before the weight
                async_ok = comfy_mm.device_supports_non_blocking(dev)
                bias = comfy_ops.cast_to(self.get_weight(self.bias.to(dev), dtype), dtype, dev, non_blocking=async_ok, copy=False)
            w = self.weight
            qtype, shape = w.tensor_type, tuple(w.tensor_shape)
            src = w.as_subclass(torch.Tensor)
            wraw = src if src.device == dev else src.to(dev)           # offloaded module: packed bytes H2D for this call
            if not wraw.is_contiguous():
                wraw = wraw.contiguous()
            W = torch.empty(shape, dtype=dtype, device=dev)
            N, K = shape[0], W.numel() // shape[0]
            args = (descs, len(keep)) if dora is None else (descs, dora, len(keep))
            with torch.cuda.device(dev):
                rc = getattr(_lib.lib(), entry)(int(qtype), wraw.data_ptr(), N, K, W.data_ptr(), dtype_code(dtype),
                                                math_code(self.dequant_dtype, dtype), *args, _current_stream_ptr(dev.index))
            _lib.check(rc, f"{entry}({getattr(qtype, 'name', qtype)}, N={N}, K={K})")
            return self._conv_forward(input, W, bias)

    class Embedding(GGMLLayer, comfy_ops.manual_cast.Embedding):
        def forward_ggml_cast_weights(self, input, out_dtype=None):
            want = out_dtype
            if self.weight.dtype in (torch.float16, torch.bfloat16):
                out_dtype = None
            w = self.weight
            qtype = getattr(w, "tensor_type", None)
            shape = tuple(getattr(w, "tensor_shape", ()))
            # the row gather needs whole blocks and K % 8 == 0 for every type (a BF16 table can be any width); any other table
            # takes the whole-table dequant below
            plain_case = (self.max_norm is None and not getattr(w, "patches", None) and input.is_cuda and len(shape) == 2
                          and shape[1] % 8 == 0 and shape[1] % gguf.GGML_QUANT_SIZES[qtype][0] == 0)
            if plain_case:
                w = w if w.device == input.device else w.to(input.device)
                # the reference passes the module itself as `input` to cast_bias_weight (ops.py:256), so a missing
                # out_dtype resolves to float32 there
                row_dtype = torch.float32 if out_dtype is None else out_dtype
                rows = dequantize_rows(w, input, row_dtype, self.dequant_dtype)
                if self.padding_idx is not None:
                    pass  # padding_idx only affects gradients in F.embedding
                return rows.to(dtype=want)
            weight, _bias = self.cast_bias_weight(self, device=input.device, dtype=out_dtype)
            return torch.nn.functional.embedding(input, weight, self.padding_idx, self.max_norm, self.norm_type,
                                                 self.scale_grad_by_freq, self.sparse).to(dtype=want)

    class LayerNorm(GGMLLayer, comfy_ops.manual_cast.LayerNorm):
        def forward_ggml_cast_weights(self, input):
            if self.weight is None:
                return super().forward_comfy_cast_weights(input)
            weight, bias = self.cast_bias_weight(input)
            return torch.nn.functional.layer_norm(input, self.normalized_shape, weight, bias, self.eps)

    class GroupNorm(GGMLLayer, comfy_ops.manual_cast.GroupNorm):
        def forward_ggml_cast_weights(self, input):
            weight, bias = self.cast_bias_weight(input)
            return torch.nn.functional.group_norm(input, self.num_groups, weight, bias, self.eps)
