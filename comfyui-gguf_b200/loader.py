"""GGUF file -> state dict of GGMLTensor (drop-in for the reference's loader.py).

Mirrored (reference file:line): gguf_sd_loader loader.py:51-141 (mmap read, prefix strip, architecture check,
`comfy.gguf.orig_shape.*` metadata loader.py:16-24, F32/F16 reshaped views vs raw uint8 payloads loader.py:118-120,
1-D BF16 -> F32 loader.py:122-124, qtype histogram log loader.py:130-131, largest-weight mark loader.py:133-137)
and gguf_clip_loader loader.py:377-406 with what it needs for the UMT5, Mistral and Qwen2.5-VL encoders:
the GGUF field readers loader.py:26-49, the sentencepiece rebuild gguf_tokenizer_loader loader.py:286-332, the tekken
rebuild gguf_tekken_tokenizer_loader loader.py:334-375, and the sibling mmproj vision tower strip_quant_suffix /
gguf_mmproj_loader loader.py:213-284.  Everything here runs once at load time; the tensors it dequantises go through
dequantize_tensor (the GPU kernels), and everything it leaves packed runs on the packed-Linear routes.

Image-model files without `general.architecture`, or with the old `pig` / `cow` tags (stable-diffusion.cpp and early
converters), load in the reference's compatibility mode (loader.py:77-94, 111-115): the architecture is recognised from the
tensor names by convert.py's table, and sd.cpp SDXL files get their `proj_in` / `proj_out` shapes fixed.
"""
from __future__ import annotations

import base64
import json
import logging
import os
import re
import warnings

import gguf
import torch

from .convert import detect_arch
from .dequant import dequantize_tensor, is_quantized
from .ops import GGMLTensor

IMG_ARCH_LIST = {"flux", "sd1", "sdxl", "sd3", "aura", "hidream", "cosmos", "ltxv", "hyvid", "wan", "lumina2", "qwen_image"}
TXT_ARCH_LIST = {"t5", "t5encoder", "llama", "qwen2vl", "qwen3", "qwen3vl"}
VIS_TYPE_LIST = {"clip-vision", "mmproj"}
_Q = gguf.GGMLQuantizationType

# token_embd shapes that identify the encoders whose tokenizer is rebuilt from the GGUF metadata
UMT5_EMBED_SHAPE = (256384, 4096)      # UMT5-XXL (Wan 2.x): sentencepiece model -> sd["spiece_model"]
MISTRAL_EMBED_SHAPE = (131072, 5120)   # Mistral: tekken JSON -> sd["tekken_model"]


def _string_field(reader, name):
    field = reader.get_field(name)
    if field is None:
        return None
    if len(field.types) != 1 or field.types[0] != gguf.GGUFValueType.STRING:
        raise TypeError(f"Bad type for GGUF {name} key: expected string, got {field.types!r}")
    return str(field.parts[field.data[-1]], encoding="utf-8")


def _scalar_field(reader, name, kind):
    """A bool / int / str metadata value, or None when the key is absent."""
    if kind is str:
        return _string_field(reader, name)
    if kind not in (bool, int, float):
        raise TypeError(f"Unknown field type {kind}")
    field = reader.get_field(name)
    if field is None:
        return None
    return kind(field.parts[field.data[-1]][0])


def _list_field(reader, name, kind):
    """An array metadata value (tokenizer.ggml.tokens / .scores / .token_type) as a tuple, or None when absent."""
    field = reader.get_field(name)
    if field is None:
        return None
    if kind is str:
        return tuple(str(field.parts[i], encoding="utf-8") for i in field.data)
    if kind not in (bool, int, float):
        raise TypeError(f"Unknown field type {kind}")
    return tuple(kind(field.parts[i][0]) for i in field.data)


def get_orig_shape(reader, tensor_name):
    """Logical shape stored by the converter for tensors it had to reshape (loader.py:16-24)."""
    key = f"comfy.gguf.orig_shape.{tensor_name}"
    field = reader.get_field(key)
    if field is None:
        return None
    if len(field.types) != 2 or field.types[0] != gguf.GGUFValueType.ARRAY or field.types[1] != gguf.GGUFValueType.INT32:
        raise TypeError(f"Bad original shape metadata for {key}: Expected ARRAY of INT32, got {field.types}")
    return torch.Size(int(field.parts[i][0]) for i in field.data)


def _check_arch(arch, kind, is_text_model, path, keys):
    """(architecture, compatibility mode or None).  Image models without an architecture field, or tagged `pig` / `cow`, are
    recognised from their (prefix-stripped) tensor names: compatibility mode "sd.cpp" or the tag."""
    if arch in (None, "pig", "cow"):
        if is_text_model:
            raise ValueError(f"This gguf file is incompatible with llama.cpp!\nConsider using safetensors or a compatible gguf file\n({path})")
        compat = "sd.cpp" if arch is None else arch
        try:
            arch = detect_arch(keys).name
        except ValueError as e:
            raise ValueError(f"This model is not currently supported - ({e})") from None
        logging.warning(f"Warning: This gguf model file is loaded in compatibility mode '{compat}' [arch:{arch}]")
        return arch, compat
    if is_text_model:
        if arch not in TXT_ARCH_LIST and kind not in VIS_TYPE_LIST:
            raise ValueError(f"Unexpected text model architecture type in GGUF file: {arch!r}")
    elif arch not in IMG_ARCH_LIST:
        raise ValueError(f"Unexpected architecture type in GGUF file: {arch!r}")
    return arch, None


def gguf_sd_loader(path, handle_prefix="model.diffusion_model.", return_arch=False, is_text_model=False):
    """Read a GGUF file into {key: GGMLTensor}; quantised payloads stay packed uint8 views of the mmap."""
    reader = gguf.GGUFReader(path)

    entries = [(t.name, t) for t in reader.tensors]
    if handle_prefix is not None and any(name.startswith(handle_prefix) for name, _ in entries):
        cut = len(handle_prefix)
        entries = [(name[cut:], t) for name, t in entries if name.startswith(handle_prefix)]

    arch = _string_field(reader, "general.architecture")
    arch, compat = _check_arch(arch, _string_field(reader, "general.type"), is_text_model, path, [name for name, _ in entries])

    state_dict, histogram = {}, {}
    for key, t in entries:
        with warnings.catch_warnings():
            warnings.filterwarnings("ignore", message="The given NumPy array is not writable")
            payload = torch.from_numpy(t.data)  # zero-copy view of the mmap
        shape = get_orig_shape(reader, t.name)
        if shape is None:
            shape = torch.Size(int(v) for v in reversed(t.shape))
            if compat == "sd.cpp" and arch == "sdxl" and t.name.endswith((".proj_in.weight", ".proj_out.weight")):
                # sd.cpp writes SDXL's 1x1 projections with their conv shape: drop the trailing size-1 dimensions
                while len(shape) > 2 and shape[-1] == 1:
                    shape = shape[:-1]
        if t.tensor_type in (_Q.F32, _Q.F16):
            payload = payload.view(*shape)
        item = GGMLTensor(payload, tensor_type=t.tensor_type, tensor_shape=shape)
        if len(shape) <= 1 and t.tensor_type == _Q.BF16:
            # 1-D tensors are never meant to be quantised: plain widening cast bf16 -> fp32 at load time
            item = payload.view(torch.bfloat16).to(torch.float32).reshape(shape)
        state_dict[key] = item
        tname = getattr(t.tensor_type, "name", repr(t.tensor_type))
        histogram[tname] = histogram.get(tname, 0) + 1

    logging.info("gguf qtypes: " + ", ".join(f"{k} ({v})" for k, v in histogram.items()))

    quantised = [k for k, v in state_dict.items() if is_quantized(v)]
    if quantised:
        biggest = max(quantised, key=lambda k: state_dict[k].numel())
        state_dict[biggest].is_largest_weight = True   # read by GGMLLayer for VRAM estimation

    return (state_dict, arch) if return_arch else state_dict


# llama.cpp tensor names -> original checkpoint names (order matters: longer patterns first where they overlap)
T5_SD_MAP = (
    ("enc.", "encoder."), (".blk.", ".block."), ("token_embd", "shared"), ("output_norm", "final_layer_norm"),
    ("attn_q", "layer.0.SelfAttention.q"), ("attn_k", "layer.0.SelfAttention.k"), ("attn_v", "layer.0.SelfAttention.v"),
    ("attn_o", "layer.0.SelfAttention.o"), ("attn_norm", "layer.0.layer_norm"),
    ("attn_rel_b", "layer.0.SelfAttention.relative_attention_bias"),
    ("ffn_up", "layer.1.DenseReluDense.wi_1"), ("ffn_down", "layer.1.DenseReluDense.wo"),
    ("ffn_gate", "layer.1.DenseReluDense.wi_0"), ("ffn_norm", "layer.1.layer_norm"),
)
LLAMA_SD_MAP = (
    ("blk.", "model.layers."), ("attn_norm", "input_layernorm"), ("attn_q_norm.", "self_attn.q_norm."),
    ("attn_k_norm.", "self_attn.k_norm."), ("attn_v_norm.", "self_attn.v_norm."), ("attn_q", "self_attn.q_proj"),
    ("attn_k", "self_attn.k_proj"), ("attn_v", "self_attn.v_proj"), ("attn_output", "self_attn.o_proj"),
    ("ffn_up", "mlp.up_proj"), ("ffn_down", "mlp.down_proj"), ("ffn_gate", "mlp.gate_proj"),
    ("ffn_norm", "post_attention_layernorm"), ("token_embd", "model.embed_tokens"), ("output_norm", "model.norm"),
    ("output.weight", "lm_head.weight"),
)
# llama.cpp's Qwen2-VL mmproj names -> the vision tower's checkpoint names
CLIP_VISION_SD_MAP = (
    ("mm.", "visual.merger.mlp."), ("v.post_ln.", "visual.merger.ln_q."), ("v.patch_embd", "visual.patch_embed.proj"),
    ("v.blk.", "visual.blocks."), ("ffn_up", "mlp.up_proj"), ("ffn_down", "mlp.down_proj"), ("ffn_gate", "mlp.gate_proj"),
    ("attn_out.", "attn.proj."), ("ln1.", "norm1."), ("ln2.", "norm2."),
)


def sd_map_replace(raw_sd, key_map):
    pairs = key_map.items() if isinstance(key_map, dict) else key_map
    pairs = list(pairs)
    out = {}
    for key, value in raw_sd.items():
        for old, new in pairs:
            key = key.replace(old, new)
        out[key] = value
    return out


def llama_permute(raw_sd, n_head, n_head_kv):
    """Undo llama.cpp's rotary-friendly q/k row permutation (loader.py:205-216); acts on the packed rows."""
    def unpermute(x, heads):
        return x.reshape(heads, x.shape[0] // heads // 2, 2, *x.shape[1:]).swapaxes(1, 2).reshape(x.shape)
    for key, value in raw_sd.items():
        if key.endswith(("q_proj.weight", "q_proj.bias")):
            value.data = unpermute(value.data, n_head)
        elif key.endswith(("k_proj.weight", "k_proj.bias")):
            value.data = unpermute(value.data, n_head_kv)
    return raw_sd


_QUANT_SUFFIX = re.compile(r"[-_]?(?:ud-)?i?q[0-9]_[a-z0-9_-]{1,8}$", re.IGNORECASE)


def strip_quant_suffix(name):
    """'qwen2.5-vl-7b-instruct-q4_k_m' -> 'qwen2.5-vl-7b-instruct' (also IQ* and Unsloth 'UD-' suffixes)."""
    match = _QUANT_SUFFIX.search(name)
    return name[:match.start()] if match else name


def gguf_mmproj_loader(path):
    """The Qwen2.5-VL vision tower from the mmproj GGUF beside the text encoder at `path`, with checkpoint key names.

    The sibling is the first `.gguf` in the directory (listdir order) whose lower-cased name contains "mmproj" and the
    encoder's lower-cased file name without its quant suffix.  Without one the text encoder still loads: an error is
    logged and {} returned.  The two patch-embedding halves become one 5-D fp32 weight, and each block's split q / k / v
    weight and bias are also fused into attn.qkv (bf16 when quantised, fp16 otherwise); the split keys stay."""
    logging.info("Attempting to find mmproj file for text encoder...")
    tenc_fname = os.path.basename(path)
    tenc = strip_quant_suffix(os.path.splitext(tenc_fname)[0].lower())
    root = os.path.dirname(path)
    target = []
    for fname in os.listdir(root):
        name, ext = os.path.splitext(fname)
        if ext.lower() == ".gguf" and "mmproj" in name.lower() and tenc in name.lower():
            target.append(fname)
    if not target:
        logging.error(f"Error: Can't find mmproj file for '{tenc_fname}' (matching:'{tenc}')! Qwen-Image-Edit will be broken!")
        return {}
    if len(target) > 1:
        logging.error(f"Ambiguous mmproj for text encoder '{tenc_fname}', will use first match.")
    logging.info(f"Using mmproj '{target[0]}' for text encoder '{tenc_fname}'.")
    vsd = gguf_sd_loader(os.path.join(root, target[0]), is_text_model=True)

    if "v.patch_embd.weight.1" in vsd:
        halves = [dequantize_tensor(vsd.pop(k), dtype=torch.float32) for k in ("v.patch_embd.weight", "v.patch_embd.weight.1")]
        vsd["v.patch_embd.weight"] = torch.stack(halves, dim=2)

    vsd = sd_map_replace(vsd, CLIP_VISION_SD_MAP)

    if "visual.blocks.0.attn_q.weight" in vsd:
        fused = {}     # "visual.blocks.<i>.attn.qkv.<weight|bias>" -> {"q.weight": tensor, ...}
        for key, value in vsd.items():
            if "attn_q" in key or "attn_k" in key or "attn_v" in key:
                block, part = key.rsplit(".attn_", 1)
                dtype = torch.bfloat16 if is_quantized(value) else torch.float16
                fused.setdefault(f"{block}.attn.qkv.{part.split('.')[-1]}", {})[part] = dequantize_tensor(value, dtype=dtype)
        for key, parts in fused.items():
            suffix = key.split(".")[-1]
            vsd[key] = torch.cat([parts[f"{p}.{suffix}"] for p in "qkv"], dim=0)
    return vsd


def gguf_tokenizer_loader(path, temb_shape):
    """The UMT5 sentencepiece model rebuilt from the GGUF's tokenizer metadata, serialised into a uint8 tensor."""
    logging.info("Attempting to recreate sentencepiece tokenizer from GGUF file metadata...")
    try:
        from sentencepiece import sentencepiece_model_pb2 as model
    except ImportError:
        raise ImportError("Please make sure sentencepiece and protobuf are installed.\npip install sentencepiece protobuf")
    reader = gguf.GGUFReader(path)
    if _string_field(reader, "tokenizer.ggml.model") != "t5" or tuple(temb_shape) != UMT5_EMBED_SHAPE:
        raise NotImplementedError("Unknown model, can't set tokenizer!")

    spm = model.ModelProto()   # trainer_spec.model_type keeps its default, UNIGRAM
    spm.normalizer_spec.add_dummy_prefix = _scalar_field(reader, "tokenizer.ggml.add_space_prefix", bool)
    spm.normalizer_spec.remove_extra_whitespaces = _scalar_field(reader, "tokenizer.ggml.remove_extra_whitespaces", bool)
    tokens = _list_field(reader, "tokenizer.ggml.tokens", str)
    scores = _list_field(reader, "tokenizer.ggml.scores", float)
    types = _list_field(reader, "tokenizer.ggml.token_type", int)
    for token, score, kind in zip(tokens, scores, types):
        piece = spm.SentencePiece()
        piece.piece, piece.score, piece.type = token, score, kind
        spm.pieces.append(piece)
    spm.trainer_spec.byte_fallback = True
    spm.trainer_spec.vocab_size = len(tokens)
    spm.trainer_spec.max_sentence_length = 4096
    spm.trainer_spec.eos_id = _scalar_field(reader, "tokenizer.ggml.eos_token_id", int)
    spm.trainer_spec.pad_id = _scalar_field(reader, "tokenizer.ggml.padding_token_id", int)
    logging.info(f"Created tokenizer with vocab size of {len(spm.pieces)}")
    return torch.ByteTensor(list(spm.SerializeToString()))


def _gpt2_byte_decoder():
    """GPT-2 byte-level BPE alphabet, inverted: the printable character that stands for each byte -> the byte.
    Printable Latin-1 bytes stand for themselves; the other 68 bytes map, in order, to U+0100 onwards."""
    printable = [*range(ord("!"), ord("~") + 1), *range(ord("¡"), ord("¬") + 1), *range(ord("®"), ord("ÿ") + 1)]
    others = [b for b in range(256) if b not in printable]
    decoder = {chr(b): b for b in printable}
    decoder.update({chr(256 + i): b for i, b in enumerate(others)})
    return decoder


def gguf_tekken_tokenizer_loader(path, temb_shape):
    """The Mistral tekken tokenizer JSON rebuilt from the GGUF's byte-level BPE token list, as a uint8 tensor."""
    logging.info("Attempting to recreate tekken tokenizer from GGUF file metadata...")
    reader = gguf.GGUFReader(path)
    if _string_field(reader, "tokenizer.ggml.model") != "gpt2" or tuple(temb_shape) != MISTRAL_EMBED_SHAPE:
        raise NotImplementedError("Unknown model, can't set tokenizer!")

    data = {"config": {"num_vocab_tokens": 150000, "default_vocab_size": 131072}, "vocab": [], "special_tokens": []}
    tokens = _list_field(reader, "tokenizer.ggml.tokens", str)
    types = _list_field(reader, "tokenizer.ggml.token_type", int)
    decoder = _gpt2_byte_decoder()
    for idx, (token, kind) in enumerate(zip(tokens, types)):
        if kind == 3:    # CONTROL: kept by its position in the file
            data["special_tokens"].append({"rank": idx, "token_str": token, "is_control": True})
        else:
            raw = bytes(decoder[ch] for ch in token)
            data["vocab"].append({"rank": len(data["vocab"]), "token_bytes": base64.b64encode(raw).decode("ascii"),
                                  "token_str": raw.decode("utf-8", errors="replace")})
    logging.info(f"Created tekken tokenizer with vocab size of {len(data['vocab'])} (+{len(data['special_tokens'])})")
    return torch.ByteTensor(list(json.dumps(data).encode("utf-8")))


def gguf_clip_loader(path):
    """Text-encoder GGUF -> state dict with original key names (loader.py:377-406).  UMT5 files gain sd["spiece_model"],
    Mistral files sd["tekken_model"], and Qwen2.5-VL (qwen2vl) files the vision tower of their sibling mmproj GGUF."""
    sd, arch = gguf_sd_loader(path, return_arch=True, is_text_model=True)
    temb = "token_embd.weight"
    temb_shape = tuple(sd[temb].shape) if temb in sd else None
    if arch in {"t5", "t5encoder"}:
        if temb_shape == UMT5_EMBED_SHAPE:
            sd["spiece_model"] = gguf_tokenizer_loader(path, temb_shape)
            logging.warning(f"Dequantizing {temb} to prevent runtime OOM.")
            sd[temb] = dequantize_tensor(sd[temb], dtype=torch.float16)
        return sd_map_replace(sd, T5_SD_MAP)
    if arch in {"llama", "qwen2vl", "qwen3", "qwen3vl"}:
        is_mistral = arch == "llama" and temb_shape == MISTRAL_EMBED_SHAPE
        if is_mistral:
            sd["tekken_model"] = gguf_tekken_tokenizer_loader(path, temb_shape)
        # a Mistral table (131072 rows) is always above the 64K-row bound; naming it keeps that so for a smaller constant
        if temb_shape is not None and (temb_shape[0] >= 64 * 1024 or is_mistral):
            # the reference pre-dequantises huge embedding tables to dodge its whole-table dequant per call
            # (loader.py:391-397); the row-gather kernel makes that unnecessary, but the host model may index
            # the table directly, so keep the reference behaviour
            logging.warning(f"Dequantizing {temb} to prevent runtime OOM.")
            sd[temb] = dequantize_tensor(sd[temb], dtype=torch.float16)
        sd = sd_map_replace(sd, LLAMA_SD_MAP)
        if arch == "llama":
            sd = llama_permute(sd, 32, 8)
        if arch == "qwen2vl":
            sd.update(gguf_mmproj_loader(path))
        return sd
    return sd
