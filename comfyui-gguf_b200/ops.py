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
"""
from __future__ import annotations

import logging

import gguf
import torch

from . import _lib
from ._host import comfy_lora, comfy_mm, comfy_ops
from .dequant import FALLBACK_QTYPES, dequantize_fallback, dequantize_rows, dequantize_tensor, dtype_code, is_quantized, math_code

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


def _launch_linear(x, wraw, qtype, N, K, bias, math, algo, spans=None, lora=None):
    """The call itself.  x: CUDA fp16/bf16 [..., K]; wraw: PLAIN uint8 tensor holding the packed rows on x.device;
    bias: PLAIN tensor on x.device or None.  Kept free of tensor-subclass traffic (every attribute read on a GGMLTensor
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
        if J == 1 and tiles is None:
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


def linear_dense(x, weight, bias=None):
    """y = x @ weight.T + bias on the tensor-core GEMM with an already dense fp16/bf16 weight (ggufb200_gemm)."""
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
        rc = _lib.lib().ggufb200_gemm(weight.data_ptr(), N, K, weight.stride(0), x2.data_ptr(), M, x2.stride(0), dtype_code(x.dtype),
                                      bias_ptr, bias_code, y.data_ptr(), N, torch.cuda.current_stream(x.device).cuda_stream)
    _lib.check(rc, f"ggufb200_gemm(M={M}, N={N}, K={K})")
    return y.reshape(*x.shape[:-1], N)


_BIG_EMBEDDING_ROWS = 64 * 1024     # loader threshold above which Embedding always takes the GGML load path (ops.py:116-117)
_META = torch.device("meta")


def _collect_patches(tensor):
    """Flatten `tensor.patches` ([(patch_list, key), ...]) onto the tensor's device; returns (patches, last key)."""
    gathered, key = [], None
    for entries, key in getattr(tensor, "patches", []):
        gathered.extend(move_patch_to_device(entries, tensor.device))
    return gathered, key


def lora_side_terms(patches):
    """Recognise a patch list that consists of plain LoRA deltas only (SURVEY 8f rank 1).

    `patches` is the flat list `_collect_patches` returns; entries follow comfy.lora's layout
    `(strength_patch, value, strength_model[, offset, function])` with value `("lora", (up, down, alpha, mid, dora_scale,
    reshape))` or a LoRAAdapter object carrying the same tuple in `.weights`.  Returns [(scale, up[N, r], down[r, K]), ...]
    with scale = strength_patch * alpha / r, or None when any entry needs the general `calculate_weight` machinery
    (strength_model != 1, offset / function hooks, LoCon mid weights, DoRA, reshape, diff / loha / lokr ... patches)."""
    terms = lora_band_terms(patches)
    if terms is None or any(band is not None for _s, _u, _d, band in terms):
        return None
    return [(scale, up, down) for scale, up, down, _band in terms]


def lora_band_terms(patches):
    """`lora_side_terms` that also accepts an `offset = (dim, start, size)`: the LoRA patches the band `start .. start + size`
    of the output rows (dim 0) or of the input features (dim 1) only.  ComfyUI gives diffusers-format LoRAs such offsets, one
    entry per q / k / v / mlp slice of a fused Flux or SD3 weight.  Returns [(scale, up, down, band), ...] with band None
    (the whole weight) or (dim, start, size), or None when any entry needs `calculate_weight` (as `lora_side_terms`)."""
    terms = []
    for entry in patches:
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
        if type(value).__name__ == "LoRAAdapter" and hasattr(value, "weights"):
            payload = value.weights
        elif isinstance(value, (tuple, list)) and len(value) == 2 and value[0] == "lora":
            payload = value[1]
        else:
            return None
        up, down = payload[0], payload[1]
        alpha = payload[2] if len(payload) > 2 else None
        if any(extra is not None for extra in payload[3:6]):
            return None
        if not (torch.is_tensor(up) and torch.is_tensor(down)) or up.dim() != 2 or down.dim() != 2 or up.shape[1] != down.shape[0]:
            return None
        scale = float(entry[0]) * (1.0 if alpha is None else float(alpha) / down.shape[0])
        terms.append((scale, up, down, band))
    return terms


def lycoris_terms(patches):
    """Recognise a patch list of LoRA, LoHa and LoKr (LyCORIS) entries, in any mix.

    Entries follow comfy.lora's layout (see `lora_side_terms`); a LoHa value is `("loha", (w1a, w1b, alpha, w2a, w2b, t1, t2,
    dora_scale))` or a LoHaAdapter carrying that tuple in `.weights`, a LoKr value `("lokr", (w1, w2, alpha, w1_a, w1_b, w2_a, w2_b,
    t2, dora_scale))` or a LoKrAdapter.  Returns [(kind, scale, factors, band), ...] in list order:
        "lora"  factors (up, down)                          scale as `lora_band_terms`
        "loha"  factors (w1a, w1b, w2a, w2b)                scale = strength * alpha / w1b.shape[0] (strength when alpha is None)
        "lokr"  factors (w1, w2, w1_a, w1_b, w2_a, w2_b),   w1 or (w1_a, w1_b) given, likewise w2;  scale = strength * alpha / dim
                with dim = w1_b.shape[0] when w1 is decomposed, w2_b.shape[0] when w2 is (that one wins), strength when alpha is
                None or neither is decomposed
    which is how comfy.lora.calculate_weight scales them.  band as `lora_band_terms`.  None when any entry needs the general
    machinery: strength_model != 1, a function hook, another offset, Tucker factors (t1 / t2), DoRA, factors that are not 2-D
    or do not chain, any other patch kind."""
    def mat(t):
        return torch.is_tensor(t) and t.dim() == 2

    terms = []
    for entry in patches:
        lora = lora_band_terms([entry])
        if lora is not None:
            scale, up, down, band = lora[0]
            terms.append(("lora", scale, (up, down), band))
            continue
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
        kind = {"LoHaAdapter": "loha", "LoKrAdapter": "lokr"}.get(type(value).__name__)
        if kind is not None and hasattr(value, "weights"):
            payload = value.weights
        elif isinstance(value, (tuple, list)) and len(value) == 2 and value[0] in ("loha", "lokr"):
            kind, payload = value
        else:
            return None
        strength = float(entry[0])
        if kind == "loha":
            if len(payload) < 5 or any(extra is not None for extra in payload[5:8]):
                return None
            w1a, w1b, alpha, w2a, w2b = payload[:5]
            if not all(mat(t) for t in (w1a, w1b, w2a, w2b)) or w1a.shape[1] != w1b.shape[0] or w2a.shape[1] != w2b.shape[0] \
                    or w1a.shape[0] != w2a.shape[0] or w1b.shape[1] != w2b.shape[1]:
                return None
            terms.append(("loha", strength * (1.0 if alpha is None else float(alpha) / w1b.shape[0]), (w1a, w1b, w2a, w2b), band))
            continue
        if len(payload) < 7 or any(extra is not None for extra in payload[7:9]):
            return None
        w1, w2, alpha, w1_a, w1_b, w2_a, w2_b = payload[:7]
        dim = None
        for whole, a, b in ((w1, w1_a, w1_b), (w2, w2_a, w2_b)):
            if whole is not None:
                if not mat(whole):
                    return None
            elif mat(a) and mat(b) and a.shape[1] == b.shape[0]:
                dim = b.shape[0]
            else:
                return None
        scale = strength * (float(alpha) / dim if alpha is not None and dim is not None else 1.0)
        terms.append(("lokr", scale, (w1, w2, w1_a, w1_b, w2_a, w2_b), band))
    return terms


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
            entries = []
            for patch_list, _key in w.patches:
                entries.extend(patch_list)
            terms = lora_band_terms(entries)
            if terms is None:
                return None
            N, K = tuple(w.tensor_shape)
            for _s, up, down, band in terms:
                rows, cols = N, K
                if band is not None:
                    dim, start, size = band
                    if start + size > (N, K)[dim]:
                        return None
                    rows, cols = (size, K) if dim == 0 else (N, size)
                if tuple(up.shape) != (rows, down.shape[0]) or down.shape[1] != cols:
                    return None
            return terms

        # LoRA inside the fused kernel (GGUFB200_ALGO_FUSED_TMEM, csrc/linear_sm90.cu: J <= 8 extra k-blocks, SURVEY 8f rank 1):
        # U = scale * up (fp16 [N, 64 J]), down (act dtype [64 J, K]) and, for row-band patches, the per-tile k-block table are
        # cached per patch set (`lora_kernel_operands`); per forward only T = x * down^T ([M, 64 J], this package's dense
        # tensor-core GEMM) is computed before the fused call.
        # False -> the unpatched fused kernel plus library GEMMs of rank sum(r) (`_add_lora`), as for sum(r) > 512.
        lora_in_kernel = True

        def _lora_operands(self, terms, dev, dtype):
            # identity + storage + version of every factor: a patch set that was swapped for another one (even at a recycled
            # id()) or modified in place rebuilds the operands
            key = tuple((id(up), up.data_ptr(), up._version, tuple(up.shape), id(down), down.data_ptr(), down._version, float(scale), band)
                        for scale, up, down, band in terms) + (str(dev), dtype)
            cached = self.__dict__.get("_gg_lora")
            if cached is not None and cached[0] == key:
                return cached[1]
            N, K = tuple(self.weight.tensor_shape)
            operands = lora_kernel_operands(terms, N, K, dtype, dev)
            self.__dict__["_gg_lora"] = (key, operands)
            return operands

        def _lycoris_terms(self, dev):
            """For a patch list with LoHa / LoKr entries (`lycoris_terms`, any mix with LoRA): (LoRA terms, LoKr patches) with the
            LoHa entries as LoRA terms of rank r1 r2 and each LoKr entry as (scale, A, B, band), fp32 A / B on `dev`; both built
            once per patch set.  None -> two-step route (also for patch_dtype other than None: the reference then forms the
            delta in another dtype)."""
            w = self.weight
            if not self.lora_side_gemm or self.patch_dtype is not None:
                return None
            entries = []
            for patch_list, _key in w.patches:
                entries.extend(patch_list)
            terms = lycoris_terms(entries)
            if terms is None:
                return None
            N, K = tuple(w.tensor_shape)
            for kind, _s, factors, band in terms:
                rows, cols = N, K
                if band is not None:
                    dim, start, size = band
                    if start + size > (N, K)[dim]:
                        return None
                    rows, cols = (size, K) if dim == 0 else (N, size)
                if kind == "lokr":
                    (a1, a2), (b1, b2) = lokr_factor_shapes(factors)
                    if a1 * b1 != rows or a2 * b2 != cols:
                        return None
                else:
                    up, down = factors[0], factors[-1]      # LoRA (up, down); LoHa: w1a and w2b carry the shape
                    if up.shape[0] != rows or down.shape[1] != cols:
                        return None
            # identity + storage + version of every factor, as for `_lora_operands`
            key = tuple((kind, float(scale), band) + tuple((id(t), t.data_ptr(), t._version, tuple(t.shape)) if t is not None else None
                                                            for t in factors) for kind, scale, factors, band in terms) + (str(dev),)
            cached = self.__dict__.get("_gg_lycoris")
            if cached is not None and cached[0] == key:
                return cached[1]
            lora, kron = [], []
            for kind, scale, factors, band in terms:
                if kind == "lora":
                    lora.append((scale, factors[0], factors[1], band))
                elif kind == "loha":
                    lora.append((scale, *loha_as_lora(*factors, dev), band))
                else:
                    kron.append((scale, *lokr_operands(factors, dev), band))
            descs = (_lib.KronPatch * max(1, len(kron)))(*[
                _lib.KronPatch(A.data_ptr(), B.data_ptr(), A.shape[0], A.shape[1], B.shape[0], B.shape[1], -1 if band is None else band[0],
                               scale, 0 if band is None else band[1], 0 if band is None else band[2])
                for scale, A, B, band in kron])
            operands = (lora, (kron, descs) if kron else None)
            self.__dict__["_gg_lycoris"] = (key, operands)
            return operands

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

        def forward_ggml_cast_weights(self, input):
            fused = self._fused_ok(input)
            terms = self._lora_terms(input.device) if fused else None
            kron = None
            if terms is None and fused and getattr(self.weight, "patches", None) and self.weight.tensor_type not in FALLBACK_QTYPES:
                lycoris = self._lycoris_terms(input.device)           # LoHa / LoKr entries: LoRA terms + LoKr patches
                if lycoris is not None:
                    terms, kron = lycoris
            if terms is not None:
                dev = input.device
                w = self.weight
                qtype, (N, K) = w.tensor_type, w.tensor_shape          # plain Python attributes: no subclass dispatch
                wraw = w.as_subclass(torch.Tensor)
                resident = wraw.device == dev
                if not resident:
                    wraw = wraw.to(dev)                                # offloaded module: packed bytes H2D
                b = self.bias
                if b is not None:
                    b = _plain(b)
                    if b.device != dev:
                        b = b.to(dev)
                M = input.numel() // K if input.shape[-1] == K else -1
                y = None
                if M < 0:
                    pass                                               # feature mismatch: let F.linear raise the usual error
                elif qtype in FALLBACK_QTYPES:
                    # numpy-fallback types (csrc/fallback.cuh): no fused kernel reads them, so K1 into an [N, K] activation-dtype
                    # weight (the reference's fp32 -> dtype rounding) + the dense GEMM at every M; other shapes: two-step route
                    if N % 8 == 0 and K % 8 == 0:
                        W = dequantize_fallback(wraw, qtype, (N, K), input.dtype)
                        y = linear_dense(input, W, b)
                elif kron is not None:
                    # LoKr: the patched weight in one K1 launch + the dense GEMM at every M; LoRA / LoHa terms as side GEMMs
                    if qtype != _Q.BF16 and N % 8 == 0 and K % 8 == 0 and len(kron[0]) <= KRON_MAX_PATCHES:
                        y = self._kron_linear(input, wraw, qtype, N, K, b, kron)
                elif qtype == _Q.BF16 and M > GEMV_MAX_M:
                    if input.dtype == torch.bfloat16 and K % 8 == 0 and N % 8 == 0:   # already dense: straight to the tensor-core GEMM
                        y = linear_dense(input, wraw.view(torch.bfloat16).view(N, K), b)
                elif M <= GEMV_MAX_M or N % 8 == 0:                    # (the M <= 8 kernel stores per element: any N)
                    math = math_code(self.dequant_dtype, input.dtype)
                    algo, spans = _lib.ALGO_AUTO, None
                    # W_STABLE: the packed weight is a parameter (or its host-to-device copy just above): never written by a kernel in flight
                    exact = (_lib.FLAG_EXACT_W if self.linear_numerics != "fast" else 0) | _lib.FLAG_W_STABLE
                    algo |= exact
                    if (self.repack_spans and resident and math == _F16_CODE and N % 8 == 0 and qtype != _Q.BF16
                            and needs_span_layout(qtype, K) and M > GEMV_MAX_M and not straddled_rows(qtype, K)):
                        spans = span_layout(w, wraw)                   # cached on the tensor after the first forward
                        algo = _lib.ALGO_FUSED_TMEM | exact
                    lora = None
                    if (terms and self.lora_in_kernel and math == _F16_CODE and N % 8 == 0
                            and qtype != _Q.BF16 and sum(d.shape[0] for _s, _u, d, _b in terms) <= LORA_KERNEL_MAX_RANK
                            and (spans is not None or not needs_span_layout(qtype, K))):
                        down_pad, u_pad, tiles = self._lora_operands(terms, dev, input.dtype)
                        lora = (linear_dense(input.reshape(-1, K), down_pad), u_pad, tiles)       # T = x * down^T, [M, 64 J]
                        algo = _lib.ALGO_FUSED_TMEM | exact
                    y = _launch_linear(input, wraw, qtype, N, K, b, math, algo, spans, lora)
                    if lora is not None:
                        return y
                if y is not None:
                    return self._add_lora(y, input, terms) if terms else y
            weight, bias = self.cast_bias_weight(input)
            return torch.nn.functional.linear(input, weight, bias)

    class Conv2d(GGMLLayer, comfy_ops.manual_cast.Conv2d):
        def forward_ggml_cast_weights(self, input):
            weight, bias = self.cast_bias_weight(input)
            return self._conv_forward(input, weight, bias)

    class Embedding(GGMLLayer, comfy_ops.manual_cast.Embedding):
        def forward_ggml_cast_weights(self, input, out_dtype=None):
            want = out_dtype
            if self.weight.dtype in (torch.float16, torch.bfloat16):
                out_dtype = None
            w = self.weight
            plain_case = (self.max_norm is None and not getattr(w, "patches", None) and input.is_cuda
                          and len(getattr(w, "tensor_shape", ())) == 2 and getattr(w, "tensor_type", None) not in FALLBACK_QTYPES)
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
