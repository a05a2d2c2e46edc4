"""Diffusion-model checkpoint -> GGUF file, optionally quantised on the GPU (the reference's tools/convert.py plus the
quantisation step it leaves to a patched llama.cpp, tools/lcpp.patch).

One table, ARCHES, describes the eleven image architectures: how each is recognised from its tensor names, which key sets
are refused (the diffusers layout of the same model), which tensors keep full precision, which are skipped, whether SD1 /
SDXL tensors get the `comfy.gguf.orig_shape` reshape, and which tensors stay unquantised.  The loader uses the same table to
recognise stable-diffusion.cpp files that carry no architecture field.

convert_file() writes in one pass what the reference's two steps write:
  stage 1 (the F16 / BF16 file of tools/convert.py): bf16 tensors -> BF16, everything else -> F16 (fp8 through fp16); fp32 /
      bf16 tensors that are 1-D, have <= 1024 elements or match a high-precision key -> F32; SD1 / SDXL tensors whose last
      dimension is not a multiple of 256 -> [n / 256, 256] plus an INT32 `comfy.gguf.orig_shape.<key>` array; tensors with
      more than four dimensions -> F32 directly (what tools/fix_5d_tensors.py adds afterwards).
  stage 2 (`qtype`, llama-quantize with the image-model patch): a tensor is quantised when stage 1 made it F16 or BF16, it is
      2-D as llama.cpp counts dimensions (leading size-1 dimensions dropped: [1, K] is 1-D, [1, A, B] is 2-D), its name ends in
      "weight" but not "_norm.weight" (llama.cpp's rule for every model), it is not on its architecture's keep-list, and, for
      the Q types, its rows are a multiple of 32 long (F16 / BF16 take any row); ffn_down-type tensors go from Q4_0 to Q4_1 and from
      Q5_0 to Q5_1.  The quantiser reads the value the stage-1 file holds (fp32 rounded to fp16, bf16 exact), so the bytes
      are those of the two-step pipeline.  Quantisation runs on the GPU (quantize.py); tensors come back one at a time.
  K mixtures (`qtype` one of KQUANT_MIXTURES' names: Q2_K, Q3_K_S / M / L, Q4_K_S / M, Q5_K_S / M, Q6_K, llama-quantize's file
      types): the same tensors are quantised, each to the type the patch's img_tensor_get_type picks: the mixture's default
      K type, raised for attention-value, fused-qkv and ffn_down tensors as the table says (the attention-value rule of Q3_K_M
      and Q4_K_S depends on how many attention-value tensors came before, in file order); a tensor whose rows are not a
      multiple of 256 then becomes F16, even when stage 1 holds BF16.  The K bytes come from quantize_k_tensor.
Tensors are written in input order with their full shapes.
"""
from __future__ import annotations

import logging
import os
import time
from dataclasses import dataclass, field

import gguf
import numpy as np
import torch

_Q = gguf.GGMLQuantizationType

QUANTIZATION_THRESHOLD = 1024     # fp32 / bf16 tensors with at most this many elements stay F32
REARRANGE_THRESHOLD = 512         # SD1 / SDXL: smallest tensor that gets the [n / 256, 256] reshape
MAX_TENSOR_NAME_LENGTH = 127
MAX_TENSOR_DIMS = 4


@dataclass(frozen=True)
class Arch:
    """One image architecture.  `keep` / `keep_names`: tensors that stay unquantised when their name contains one of `keep`
    or equals one of `keep_names` (the per-architecture lists of the reference's llama.cpp patch)."""
    name: str
    detect: tuple = ()            # tuples of keys; the first tuple whose keys are all present identifies the architecture
    banned: tuple = ()            # any of these present as well: the diffusers layout, which is refused
    hiprec: tuple = ()            # substrings: fp32 / bf16 tensors kept in F32
    ignore: tuple = ()            # substrings: tensors left out of the file
    shape_fix: bool = False       # SD1 / SDXL reshape to [n / 256, 256]
    keep: tuple = ()
    keep_names: tuple = ()


_FLUX_KEEP = ("txt_in.", "img_in.", "time_in.", "vector_in.", "guidance_in.", "final_layer.")
_UNET_KEEP = ("class_embedding.", "time_embedding.", "add_embedding.", "time_embed.", "label_emb.", "conv_in.", "conv_out.")

ARCHES = (
    Arch("flux", detect=(("transformer_blocks.0.attn.norm_added_k.weight",), ("double_blocks.0.img_attn.proj.weight",)),
         banned=("transformer_blocks.0.attn.norm_added_k.weight",), keep=_FLUX_KEEP),
    Arch("sd3", detect=(("transformer_blocks.0.attn.add_q_proj.weight",), ("joint_blocks.0.x_block.attn.qkv.weight",)),
         banned=("transformer_blocks.0.attn.add_q_proj.weight",),
         keep=("final_layer.", "time_text_embed.", "context_embedder.", "t_embedder.", "y_embedder.", "x_embedder."),
         keep_names=("proj_out.weight", "pos_embed")),
    Arch("aura", detect=(("double_layers.3.modX.1.weight",), ("joint_transformer_blocks.3.ff_context.out_projection.weight",)),
         banned=("joint_transformer_blocks.3.ff_context.out_projection.weight",), keep=("t_embedder.", "init_x_linear."),
         keep_names=("modF.1.weight", "cond_seq_linear.weight", "final_linear.weight", "positional_encoding", "register_tokens")),
    Arch("hidream", detect=(("caption_projection.0.linear.weight", "double_stream_blocks.0.block.ff_i.shared_experts.w3.weight"),),
         hiprec=(".ff_i.gate.weight", "img_emb.emb_pos"),
         keep=("p_embedder.", "t_embedder.", "x_embedder.", "final_layer.", ".ff_i.gate.weight", "caption_projection.")),
    Arch("cosmos", detect=(("blocks.0.mlp.layer1.weight", "blocks.0.adaln_modulation_cross_attn.1.weight"),),
         hiprec=("pos_embedder",), ignore=("_extra_state", "accum_"),
         keep=("p_embedder.", "t_embedder.", "t_embedding_norm.", "x_embedder.", "pos_embedder.", "final_layer.")),
    Arch("ltxv", detect=(("adaln_single.emb.timestep_embedder.linear_2.weight", "transformer_blocks.27.scale_shift_table",
                          "caption_projection.linear_2.weight"),),
         hiprec=("scale_shift_table",),
         keep=("adaln_single.", "caption_projection.", "patchify_proj.", "proj_out.", "scale_shift_table")),
    Arch("hyvid", detect=(("double_blocks.0.img_attn_proj.weight", "txt_in.individual_token_refiner.blocks.1.self_attn_qkv.weight"),),
         keep=_FLUX_KEEP),
    Arch("wan", detect=(("blocks.0.self_attn.norm_q.weight", "text_embedding.2.weight", "head.modulation"),),
         hiprec=(".modulation",),
         keep=("modulation.", "patch_embedding.", "text_embedding.", "time_projection.", "time_embedding.", "img_emb.", "head.")),
    Arch("sdxl", shape_fix=True,
         detect=(("down_blocks.0.downsamplers.0.conv.weight", "add_embedding.linear_1.weight"),
                 ("input_blocks.3.0.op.weight", "input_blocks.6.0.op.weight", "output_blocks.2.2.conv.weight",
                  "output_blocks.5.2.conv.weight"),
                 ("label_emb.0.0.weight",)),
         keep=_UNET_KEEP, keep_names=("input_blocks.0.0.weight", "out.2.weight")),
    Arch("sd1", shape_fix=True,
         detect=(("down_blocks.0.downsamplers.0.conv.weight",),
                 ("input_blocks.3.0.op.weight", "input_blocks.6.0.op.weight", "input_blocks.9.0.op.weight",
                  "output_blocks.2.1.conv.weight", "output_blocks.5.2.conv.weight", "output_blocks.8.2.conv.weight")),
         keep=_UNET_KEEP, keep_names=("input_blocks.0.0.weight", "out.2.weight")),
    Arch("lumina2", detect=(("cap_embedder.1.weight", "context_refiner.0.attention.qkv.weight"),),
         keep=("t_embedder.", "x_embedder.", "final_layer.", "cap_embedder.", "context_refiner.", "noise_refiner.")),
)
ARCH_BY_NAME = {a.name: a for a in ARCHES}


def detect_arch(keys) -> Arch:
    """The architecture of a (prefix-stripped) key set, in table order.  ValueError for a banned (diffusers-layout) or an
    unknown key set."""
    keys = set(keys)
    for arch in ARCHES:
        for match in arch.detect:
            if all(k in keys for k in match):
                if any(k in keys for k in arch.banned):
                    raise ValueError("Model architecture not allowed for conversion! (i.e. reference VS diffusers format)")
                return arch
    raise ValueError("Unknown model architecture!")


def strip_prefix(state_dict: dict) -> dict:
    """Drop `model.diffusion_model.` or `model.` (when any key has it; keys without it are dropped) or a `net.` that every key
    carries."""
    prefix = next((p for p in ("model.diffusion_model.", "model.") if any(k.startswith(p) for k in state_dict)), None)
    if prefix is None and state_dict and all(k.startswith("net.") for k in state_dict):
        prefix = "net."
    if prefix is None:
        return state_dict
    logging.info(f"State dict prefix found: '{prefix}'")
    return {k.replace(prefix, ""): v for k, v in state_dict.items() if prefix in k}


def load_state_dict(path: str) -> dict:
    """A checkpoint's tensors with the prefix stripped: .ckpt / .pt / .pth / .bin through torch.load(weights_only=True)
    (unwrapping a `model` or `module` entry), anything else as safetensors."""
    if path.endswith((".ckpt", ".pt", ".bin", ".pth")):
        sd = torch.load(path, map_location="cpu", weights_only=True)
        for sub in ("model", "module"):
            if sub in sd:
                sd = sd[sub]
                break
        if len(sd) < 20:
            raise RuntimeError(f"pt subkey load failed: {sd.keys()}")
    else:
        from safetensors.torch import load_file
        sd = load_file(path)
    return strip_prefix(sd)


# ------------------------------------------------------------------ type policy
QTYPES = {"F16": _Q.F16, "BF16": _Q.BF16, "Q8_0": _Q.Q8_0, "Q5_1": _Q.Q5_1, "Q5_0": _Q.Q5_0, "Q4_1": _Q.Q4_1, "Q4_0": _Q.Q4_0}
FILE_TYPES = {_Q.F16: gguf.LlamaFileType.MOSTLY_F16, _Q.BF16: gguf.LlamaFileType.MOSTLY_BF16, _Q.Q8_0: gguf.LlamaFileType.MOSTLY_Q8_0,
              _Q.Q5_1: gguf.LlamaFileType.MOSTLY_Q5_1, _Q.Q5_0: gguf.LlamaFileType.MOSTLY_Q5_0, _Q.Q4_1: gguf.LlamaFileType.MOSTLY_Q4_1,
              _Q.Q4_0: gguf.LlamaFileType.MOSTLY_Q4_0}
_FP8 = tuple(getattr(torch, n) for n in ("float8_e4m3fn", "float8_e5m2") if hasattr(torch, n))

# the patch's name rules, checked in its order: a name caught by the attention-value or fused-qkv rule is never an ffn_down
_ATTN_V = ("attn_v.weight", ".to_v.weight", ".v.weight", ".attn.w1v.weight", ".attn.w2v.weight", "_attn.v_proj.weight")
_ATTN_QKV = ("attn_qkv.weight", "attn.qkv.weight", "attention.qkv.weight")
_FFN_DOWN = ("ffn_down", ".ffn.2.weight", ".ff.net.2.weight", ".mlp.layer2.weight", ".adaln_modulation_mlp.2.weight",
             ".feed_forward.w2.weight")
_FFN_UPGRADE = {_Q.Q4_0: _Q.Q4_1, _Q.Q5_0: _Q.Q5_1}


# llama-quantize's K mixtures (the patch's img_tensor_get_type): default type, general.file_type, and the raised types of the
# attention-value tensors ((n, type) pairs: the i-th attention-value tensor gets the type of the first pair with i < n, else the
# default), of the fused-qkv tensors and of the ffn_down tensors (None: the default)
@dataclass(frozen=True)
class KMixture:
    name: str
    default: _Q
    file_type: gguf.LlamaFileType
    attn_v: tuple = ()
    qkv: _Q | None = None
    ffn_down: _Q | None = None


_ALL = 1 << 62
_FT = gguf.LlamaFileType
KQUANT_MIXTURES = {m.name: m for m in (
    KMixture("Q2_K", _Q.Q2_K, _FT.MOSTLY_Q2_K, attn_v=((_ALL, _Q.Q3_K),)),
    KMixture("Q3_K_S", _Q.Q3_K, _FT.MOSTLY_Q3_K_S),
    KMixture("Q3_K_M", _Q.Q3_K, _FT.MOSTLY_Q3_K_M, attn_v=((2, _Q.Q5_K), (_ALL, _Q.Q4_K)), qkv=_Q.Q4_K, ffn_down=_Q.Q4_K),
    KMixture("Q3_K_L", _Q.Q3_K, _FT.MOSTLY_Q3_K_L, attn_v=((_ALL, _Q.Q5_K),), qkv=_Q.Q4_K, ffn_down=_Q.Q5_K),
    KMixture("Q4_K_S", _Q.Q4_K, _FT.MOSTLY_Q4_K_S, attn_v=((4, _Q.Q5_K),), ffn_down=_Q.Q5_K),
    KMixture("Q4_K_M", _Q.Q4_K, _FT.MOSTLY_Q4_K_M, attn_v=((_ALL, _Q.Q6_K),), qkv=_Q.Q5_K, ffn_down=_Q.Q6_K),
    KMixture("Q5_K_S", _Q.Q5_K, _FT.MOSTLY_Q5_K_S),
    KMixture("Q5_K_M", _Q.Q5_K, _FT.MOSTLY_Q5_K_M, attn_v=((_ALL, _Q.Q6_K),), qkv=_Q.Q6_K, ffn_down=_Q.Q6_K),
    KMixture("Q6_K", _Q.Q6_K, _FT.MOSTLY_Q6_K),
)}
KQUANT_TYPES = (_Q.Q2_K, _Q.Q3_K, _Q.Q4_K, _Q.Q5_K, _Q.Q6_K)


def is_attn_v(name: str) -> bool:
    return any(p in name for p in _ATTN_V)


def is_attn_qkv(name: str) -> bool:
    return not is_attn_v(name) and any(p in name for p in _ATTN_QKV)


def is_ffn_down(name: str) -> bool:
    if any(p in name for p in _ATTN_V + _ATTN_QKV):
        return False
    return any(p in name for p in _FFN_DOWN) or ("experts." in name and ".w2.weight" in name)


def stage1_type(key: str, dtype: torch.dtype, shape, arch: Arch):
    """(type of the F16 / BF16 file, whether the SD1 / SDXL [n / 256, 256] reshape applies) for one source tensor."""
    shape = tuple(shape)
    n = int(np.prod(shape, dtype=np.int64)) if shape else 1
    if len(shape) > MAX_TENSOR_DIMS:
        return _Q.F32, False
    qtype = _Q.BF16 if dtype == torch.bfloat16 else _Q.F16
    if dtype in (torch.float32, torch.bfloat16):
        if len(shape) == 1 or n <= QUANTIZATION_THRESHOLD or any(h in key for h in arch.hiprec):
            qtype = _Q.F32
    reshape = (arch.shape_fix and len(shape) > 1 and n >= REARRANGE_THRESHOLD and n % 256 == 0 and shape[-1] % 256 != 0)
    return qtype, reshape


def ggml_n_dims(shape) -> int:
    """llama.cpp's ggml_n_dims of a tensor with this (torch-order) shape: leading size-1 dimensions do not count, so [1, K] is
    1-D and [1, A, B] is 2-D there.  The file keeps the full shape; this only decides whether llama-quantize quantises it."""
    shape = tuple(shape)
    lead = 0
    while lead < len(shape) - 1 and shape[lead] == 1:
        lead += 1
    return max(len(shape) - lead, 1)


def quantisable(key: str, stage1: _Q, stored_shape, arch: Arch) -> bool:
    """Whether llama-quantize with the image-model patch quantises `key` at all (the row-length check aside)."""
    if stage1 not in (_Q.F16, _Q.BF16) or ggml_n_dims(stored_shape) != 2:
        return False
    if not key.endswith("weight") or "_norm.weight" in key:
        return False
    return not (any(k in key for k in arch.keep) or key in arch.keep_names)


def stage2_type(key: str, stage1: _Q, stored_shape, arch: Arch, qtype) -> _Q:
    """The type `key` is written in when the file is quantised to `qtype` (None: stage 1 only).  `stored_shape` is the shape
    stage 1 writes (after the SD1 / SDXL reshape)."""
    if qtype is None or not quantisable(key, stage1, stored_shape, arch):
        return stage1
    if qtype not in (_Q.F16, _Q.BF16) and stored_shape[-1] % 32 != 0:     # F16 / BF16 have 1-element blocks
        return stage1
    if qtype in _FFN_UPGRADE and is_ffn_down(key):
        return _FFN_UPGRADE[qtype]
    return qtype


def kquant_type(key: str, stored_shape, mix: KMixture, n_attn_v: int) -> _Q:
    """The type of a quantisable tensor in K mixture `mix`, `n_attn_v` attention-value tensors having come before it."""
    qtype = mix.default
    if is_attn_v(key):
        qtype = next((t for n, t in mix.attn_v if n_attn_v < n), mix.default)
    elif is_attn_qkv(key):
        qtype = mix.qkv or mix.default
    elif is_ffn_down(key):
        qtype = mix.ffn_down or mix.default
    return qtype if stored_shape[-1] % 256 == 0 else _Q.F16


@dataclass
class TensorPlan:
    key: str
    shape: tuple            # shape written to the file (after the SD1 / SDXL reshape)
    orig_shape: tuple | None
    stage1: _Q
    qtype: _Q               # final type


def plan_tensors(state_dict: dict, arch: Arch, qtype=None) -> list:
    """Every written tensor's plan, in input order; ignored keys are left out.  `qtype`: None, a type, or a KMixture."""
    plans = []
    n_attn_v = 0
    for key, t in state_dict.items():
        if any(x in key for x in arch.ignore):
            logging.info(f"Filtering ignored key: '{key}'")
            continue
        stage1, reshape = stage1_type(key, t.dtype, t.shape, arch)
        shape = tuple(int(d) for d in t.shape)
        orig = None
        if reshape:
            orig, shape = shape, (t.numel() // 256, 256)
        if isinstance(qtype, KMixture):
            final = stage1
            if quantisable(key, stage1, shape, arch):
                final = kquant_type(key, shape, qtype, n_attn_v)
                n_attn_v += is_attn_v(key)        # counted before the row check, as the patch does
        else:
            final = stage2_type(key, stage1, shape, arch, qtype)
        plans.append(TensorPlan(key, shape, orig, stage1, final))
    return plans


def _stage1_values(t: torch.Tensor, stage1: _Q) -> torch.Tensor:
    """The values the stage-1 file holds, as a tensor of the stage-1 dtype (fp8 goes through fp16 as in the reference)."""
    if stage1 == _Q.F32:
        return t.to(torch.float32)
    if stage1 == _Q.BF16:
        return t
    return t.to(torch.float16)


def _host_bytes(v: torch.Tensor, qtype: _Q) -> np.ndarray:
    """F32 / F16 / BF16 bytes of stage-1 values without the GPU quantiser (BF16 from bf16 values: the bits, NaNs quietened as
    gguf-py's BF16 rounding does)."""
    v = v.detach().cpu().contiguous()
    if qtype == _Q.F32:
        return v.to(torch.float32).numpy().view(np.uint8)
    if qtype == _Q.F16:
        return v.to(torch.float16).numpy().view(np.uint8)
    assert v.dtype == torch.bfloat16
    bits = v.view(torch.int16).numpy().view(np.uint16).copy()
    nan = (bits & 0x7FFF) > 0x7F80
    bits[nan] |= 0x0040
    return bits.view(np.uint8)


def needs_quantiser(plan: TensorPlan) -> bool:
    """Whether `plan` runs on the GPU quantiser: the Q types, and BF16 from F16 values."""
    return plan.qtype != plan.stage1 and plan.qtype not in (_Q.F16, _Q.F32)


def tensor_bytes(t: torch.Tensor, plan: TensorPlan, device=None) -> np.ndarray:
    """The bytes `plan` writes for source tensor `t`."""
    v = _stage1_values(t, plan.stage1).reshape(plan.shape)
    if not needs_quantiser(plan):
        return _host_bytes(v, plan.qtype).reshape(-1)
    from .quantize import quantize_k_tensor, quantize_tensor
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    encode = quantize_k_tensor if plan.qtype in KQUANT_TYPES else quantize_tensor
    packed = encode(v.to(device, non_blocking=False), plan.qtype)
    return packed.cpu().numpy().reshape(-1)


@dataclass
class ConvertResult:
    path: str
    arch: Arch
    plans: list
    seconds: dict = field(default_factory=dict)   # read / quantise / write


def convert_state_dict(state_dict: dict, dst_path: str, qtype=None, arch: Arch | None = None, device=None) -> ConvertResult:
    """Write the GGUF file of a prefix-stripped state dict (see the module docstring).  `qtype`: None (the F16 / BF16 file),
    one of QTYPES' names or values, or one of KQUANT_MIXTURES' names (or a KMixture)."""
    if isinstance(qtype, str):
        if qtype.upper() in KQUANT_MIXTURES:
            qtype = KQUANT_MIXTURES[qtype.upper()]
        elif qtype.upper() not in QTYPES:
            raise ValueError(f"unsupported qtype {qtype!r}: one of {', '.join(list(QTYPES) + list(KQUANT_MIXTURES))}")
        else:
            qtype = QTYPES[qtype.upper()]
    elif qtype is not None and not isinstance(qtype, KMixture):
        qtype = _Q(qtype)
        if qtype not in FILE_TYPES:
            raise ValueError(f"unsupported qtype {qtype.name}: one of {', '.join(QTYPES)}")
    arch = arch or detect_arch(state_dict.keys())
    too_long = [k for k in state_dict if len(k) > MAX_TENSOR_NAME_LENGTH]
    if too_long:
        raise ValueError(f"Can only handle tensor names up to {MAX_TENSOR_NAME_LENGTH} characters. Tensors exceeding the limit: "
                         + ", ".join(f"{k!r} ({len(k)})" for k in too_long))
    if qtype is None:
        dtypes = [t.dtype for t in state_dict.values()]
        main = max(set(dtypes), key=dtypes.count) if dtypes else torch.float16
        file_type = gguf.LlamaFileType.MOSTLY_BF16 if main == torch.bfloat16 else gguf.LlamaFileType.MOSTLY_F16
    elif isinstance(qtype, KMixture):
        file_type = qtype.file_type
    else:
        file_type = FILE_TYPES[qtype]
    plans = plan_tensors(state_dict, arch, qtype)
    if any(needs_quantiser(p) for p in plans) and device is None and not torch.cuda.is_available():
        raise NotImplementedError(f"quantising to {qtype.name} runs on the GPU and no CUDA device is visible")

    writer = gguf.GGUFWriter(path=None, arch=arch.name)
    writer.add_quantization_version(gguf.GGML_QUANT_VERSION)
    writer.add_file_type(file_type)
    for p in plans:
        if p.orig_shape is not None:
            writer.add_array(f"comfy.gguf.orig_shape.{p.key}", [int(d) for d in p.orig_shape])
    for p in plans:
        byte_shape = gguf.quant_shape_to_byte_shape(p.shape, p.qtype)
        writer.add_tensor_info(p.key, byte_shape, np.dtype(np.uint8), int(np.prod(byte_shape, dtype=np.int64)), raw_dtype=p.qtype)
    t_quant = t_write = 0.0
    writer.write_header_to_file(path=dst_path)
    writer.write_kv_data_to_file()
    writer.write_ti_data_to_file()
    for p in plans:
        t0 = time.perf_counter()
        data = tensor_bytes(state_dict[p.key], p, device)
        t1 = time.perf_counter()
        writer.write_tensor_data(data)
        t_write += time.perf_counter() - t1
        t_quant += t1 - t0
        logging.info(f"{p.key:<{MAX_TENSOR_NAME_LENGTH}} {state_dict[p.key].dtype} --> {p.qtype.name}, shape = {p.shape}")
    writer.close()
    return ConvertResult(dst_path, arch, plans, {"quantise": t_quant, "write": t_write})


def convert_file(src_path: str, dst_path: str | None = None, qtype=None, overwrite: bool = False, device=None) -> ConvertResult:
    """Convert the checkpoint at `src_path`.  dst_path: default `<src without extension>-<type>.gguf`; a `{ftype}` in it is
    replaced by the type name.  An existing destination is refused unless `overwrite`."""
    t0 = time.perf_counter()
    sd = load_state_dict(src_path)
    read = time.perf_counter() - t0
    arch = detect_arch(sd.keys())
    logging.info(f"* Architecture detected from input: {arch.name}")
    if qtype is not None:
        name = qtype.upper() if isinstance(qtype, str) else qtype.name if isinstance(qtype, KMixture) else _Q(qtype).name
    else:
        dtypes = [t.dtype for t in sd.values()]
        name = "BF16" if dtypes and max(set(dtypes), key=dtypes.count) == torch.bfloat16 else "F16"
    if dst_path is None:
        dst_path = f"{os.path.splitext(src_path)[0]}-{name}.gguf"
    elif "{ftype}" in dst_path:
        dst_path = dst_path.replace("{ftype}", name)
    if os.path.exists(dst_path) and not overwrite:
        raise FileExistsError(f"{dst_path} exists (pass overwrite=True / --overwrite to replace it)")
    result = convert_state_dict(sd, dst_path, qtype, arch, device)
    result.seconds["read"] = read
    return result
