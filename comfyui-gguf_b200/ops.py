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
from .dequant import dequantize_rows, dequantize_tensor, dtype_code, is_quantized, math_code

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
    not a multiple of 16 bytes): Q2_K / Q3_K / Q6_K / IQ4_XS always, the others for some K (Q8_0 at K = 2432)."""
    bs, ts = gguf.GGML_QUANT_SIZES[qtype]
    return bs > 1 and (((256 // bs) * ts) % 16 != 0 or ((K // bs) * ts) % 16 != 0)


def span_layout(weight, wraw):
    """The re-packed span-major copy of a device-resident packed weight (csrc/repack.cu, SURVEY 8f rank 3), built once and
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


LORA_MAX_RANK = 64     # the LoRA k-block of the FUSED_TMEM kernel is one 64-wide k-block


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
        t_pad, u_pad = lora           # T = x * down^T [M, 64] act dtype, U = scale * up [N, 64] fp16 (zero padded)

        def call():
            return L.ggufb200_linear_lora(qcode, w_ptr, None if spans is None else spans.data_ptr(), N, K, x2.data_ptr(), M, x2.stride(0), act,
                                          bias_ptr, bias_code, t_pad.data_ptr(), t_pad.stride(0), u_pad.data_ptr(), y.data_ptr(), N, ws_ptr, need,
                                          algo, _current_stream_ptr(index))
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
    terms = []
    for entry in patches:
        if len(entry) < 3 or entry[2] != 1.0 or any(extra is not None for extra in entry[3:5]):
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
        terms.append((scale, up, down))
    return terms


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
            terms = lora_side_terms(entries)
            if terms is None:
                return None
            N, K = tuple(w.tensor_shape)
            if any(tuple(up.shape) != (N, down.shape[0]) or down.shape[1] != K for _s, up, down in terms):
                return None
            return terms

        # LoRA inside the fused kernel (csrc/gemm4.cu: one extra k-block, SURVEY 8f rank 1): U = scale * up (fp16 [N, 64]) and
        # down (act dtype [64, K]), zero padded to rank 64 and cached per patch set; per forward only T = x * down^T
        # ([M, 64], this package's dense tensor-core GEMM) is computed before the fused call.
        # False -> the unpatched fused kernel plus two library GEMMs of rank sum(r) (`_add_lora`).
        lora_in_kernel = True

        def _lora_operands(self, terms, dev, dtype):
            # identity + storage + version of every factor: a patch set that was swapped for another one (even at a recycled
            # id()) or modified in place rebuilds the operands
            key = tuple((id(up), up.data_ptr(), up._version, tuple(up.shape), id(down), down.data_ptr(), down._version, float(scale))
                        for scale, up, down in terms) + (str(dev), dtype)
            cached = self.__dict__.get("_gg_lora")
            if cached is not None and cached[0] == key:
                return cached[1], cached[2]
            N, K = tuple(self.weight.tensor_shape)
            down_pad = torch.zeros(LORA_MAX_RANK, K, device=dev, dtype=dtype)
            u_pad = torch.zeros(N, LORA_MAX_RANK, device=dev, dtype=torch.float16)
            r0 = 0
            for scale, up, down in terms:
                r = down.shape[0]
                down_pad[r0:r0 + r] = down.to(device=dev, dtype=dtype)
                u_pad[:, r0:r0 + r] = (up.to(device=dev, dtype=torch.float32) * scale).to(torch.float16)
                r0 += r
            self.__dict__["_gg_lora"] = (key, down_pad, u_pad)
            return down_pad, u_pad

        def _add_lora(self, y, input, terms):
            x2 = input.reshape(-1, input.shape[-1])
            y2 = y.view(-1, y.shape[-1])
            if len(terms) == 1:
                scale, up, down = terms[0]
                down_all = down.to(device=x2.device, dtype=x2.dtype, non_blocking=True)
                up_all = up.to(device=x2.device, dtype=torch.float32, non_blocking=True) * scale
            else:                                                   # one pair of GEMMs for any number of LoRAs
                down_all = torch.cat([d.to(device=x2.device, dtype=x2.dtype, non_blocking=True) for _s, _u, d in terms], 0)
                up_all = torch.cat([u.to(device=x2.device, dtype=torch.float32, non_blocking=True) * s for s, u, _d in terms], 1)
            t = x2 @ down_all.t()                                   # [M, R]   library GEMMs: R is tens, not thousands
            y2.addmm_(t, up_all.to(x2.dtype).t())
            return y

        def forward_ggml_cast_weights(self, input):
            terms = self._lora_terms(input.device) if self._fused_ok(input) else None
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
                            and needs_span_layout(qtype, K) and M > GEMV_MAX_M):
                        spans = span_layout(w, wraw)                   # cached on the tensor after the first forward
                        algo = _lib.ALGO_FUSED_TMEM | exact
                    lora = None
                    if (terms and self.lora_in_kernel and math == _F16_CODE and N % 8 == 0
                            and qtype != _Q.BF16 and sum(d.shape[0] for _s, _u, d in terms) <= LORA_MAX_RANK
                            and (spans is not None or not needs_span_layout(qtype, K))):
                        down_pad, u_pad = self._lora_operands(terms, dev, input.dtype)
                        lora = (linear_dense(input.reshape(-1, K), down_pad), u_pad)       # T = x * down^T, [M, 64]
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
                          and len(getattr(w, "tensor_shape", ())) == 2)
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
