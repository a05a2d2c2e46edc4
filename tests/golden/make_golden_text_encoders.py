#!/usr/bin/env python
"""Generate the text-encoder GGUF fixtures and what the UNMODIFIED reference loads from them.

Run where the reference package and `transformers` (which the reference's tekken loader imports) are installed:

    python tests/golden/make_golden_text_encoders.py

Writes under tests/golden/ (names in tests/text_encoder_cases.py):
  umt5-tiny-Q8_0.gguf, mistral-tiny-Q4_K_M.gguf, Qwen2.5-VL-tiny-Q4_K_M.gguf, Qwen2.5-VL-tiny-mmproj-F16.gguf
      synthetic GGUFs written by gguf.GGUFWriter: metadata and seeded tensors only
  text_encoders.json / text_encoders.npz
      the reference's state dict for each encoder file, key by key (format in tests/text_encoder_cases.py)

The reference is imported by path through a throw-away package of symlinks and never copied.  Its gguf_clip_loader
recognises UMT5 and Mistral only by the full-size token table, so for those two files this script runs the steps of its
t5 / llama branch itself, with the reference's own functions: gguf_sd_loader, gguf_tokenizer_loader or
gguf_tekken_tokenizer_loader called with the full-size shape, dequantize_tensor of the table to fp16, sd_map_replace and
llama_permute.  The qwen2vl file goes through the reference's gguf_clip_loader unchanged (the vision tower included).
"""
import importlib
import json
import os
import sys
import tempfile

import gguf
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "fake_comfy"))

import oracle  # noqa: E402  (seeded block generator of the block formats)
import text_encoder_cases as tc  # noqa: E402
from fallback_cases import random_blocks as fallback_blocks  # noqa: E402

Q = gguf.GGMLQuantizationType
FALLBACK = {Q.IQ2_XXS}


def load_ref_loader():
    tmp = tempfile.mkdtemp(prefix="refpkg_")
    pkg = os.path.join(tmp, "refgguf_te")
    os.mkdir(pkg)
    open(os.path.join(pkg, "__init__.py"), "w").close()
    for f in ("dequant.py", "ops.py", "loader.py"):
        os.symlink(os.path.join(REF, f), os.path.join(pkg, f))
    sys.path.insert(0, tmp)
    return importlib.import_module("refgguf_te.loader")


def _tensor(qt, shape, seed):
    """Seeded numpy payload of a GGUF tensor of logical `shape`: float values for F32 / F16, packed rows otherwise."""
    rng = np.random.default_rng(seed)
    if qt == Q.F32:
        return rng.normal(0.0, 0.5, size=shape).astype(np.float32)
    if qt == Q.F16:
        return rng.normal(0.0, 0.05, size=shape).astype(np.float16)
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    n_blocks = int(np.prod(shape)) // bs
    raw = fallback_blocks(qt, n_blocks, seed=seed, scale=0.002) if qt in FALLBACK else oracle.random_blocks(int(qt), n_blocks, seed=seed, scale=0.02)
    return raw.reshape(*shape[:-1], shape[-1] // bs * ts)


def _write(path, arch, tensors, meta=None, seed=0):
    w = gguf.GGUFWriter(path, arch)
    if meta is not None:
        meta(w)
    for i, (name, (qt, shape)) in enumerate(tensors.items()):
        data = _tensor(qt, shape, seed + i)
        w.add_tensor(name, data, raw_dtype=None if qt in (Q.F32, Q.F16) else qt)
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    print("wrote", path)


def _mistral_tokenizer(w):
    from transformers.convert_slow_tokenizer import bytes_to_unicode
    enc = bytes_to_unicode()

    def bpe(text_bytes):
        return "".join(enc[b] for b in text_bytes)
    specials = ["<unk>", "<s>", "</s>", "[INST]", "[/INST]", "[IMG]"]
    words = [" the", " a", "\n\n", " Hello", " world", "’", " über", " 日本", "ing", "  "]
    tokens = specials[:3] + [bpe(bytes([b])) for b in range(256)] + specials[3:]
    tokens += [bpe(s.encode("utf-8")) for s in words]
    tokens += [bpe("日".encode("utf-8")[:2]), bpe(b"\xff\xfe")]          # byte strings that are not valid UTF-8
    types = [3 if t in specials else 1 for t in tokens]
    w.add_tokenizer_model("gpt2")
    w.add_token_list(tokens)
    w.add_token_types(types)
    w.add_bos_token_id(1)
    w.add_eos_token_id(2)


def _mmproj_meta(w):
    w.add_type("mmproj")


UMT5 = {
    "token_embd.weight": (Q.Q8_0, tc.UMT5_TABLE),
    "enc.blk.0.attn_q.weight": (Q.Q8_0, (64, 64)),
    "enc.blk.0.attn_rel_b.weight": (Q.F16, (32, 8)),
    "enc.blk.0.attn_norm.weight": (Q.F32, (64,)),
    "enc.blk.0.ffn_up.weight": (Q.Q4_0, (64, 64)),
    "enc.output_norm.weight": (Q.F32, (64,)),
}
MISTRAL = {
    "token_embd.weight": (Q.Q4_K, tc.MISTRAL_TABLE),
    "blk.0.attn_q.weight": (Q.Q4_K, (64, 256)),
    "blk.0.attn_k.weight": (Q.Q8_0, (16, 256)),
    "blk.0.attn_norm.weight": (Q.F32, (256,)),
    "output_norm.weight": (Q.F32, (256,)),
}
QWEN = {
    "token_embd.weight": (Q.Q8_0, (32, 256)),
    "blk.0.attn_q.weight": (Q.Q4_K, (16, 256)),
    "blk.0.attn_q.bias": (Q.F32, (16,)),
    "blk.0.ffn_down.weight": (Q.IQ2_XXS, (16, 256)),
    "blk.0.attn_norm.weight": (Q.F32, (256,)),
    "output_norm.weight": (Q.F32, (256,)),
}
MMPROJ = {
    "v.patch_embd.weight": (Q.F16, (64, 3, 4, 4)),
    "v.patch_embd.weight.1": (Q.F16, (64, 3, 4, 4)),
    "v.blk.0.attn_q.weight": (Q.Q4_K, (16, 256)),
    "v.blk.0.attn_k.weight": (Q.Q8_0, (16, 256)),
    "v.blk.0.attn_v.weight": (Q.IQ2_XXS, (16, 256)),
    "v.blk.1.attn_q.weight": (Q.F16, (16, 256)),
    "v.blk.1.attn_k.weight": (Q.F16, (16, 256)),
    "v.blk.1.attn_v.weight": (Q.F16, (16, 256)),
    **{f"v.blk.{i}.attn_{p}.bias": (Q.F32, (16,)) for i in (0, 1) for p in "qkv"},
    **{f"v.blk.{i}.attn_out.weight": (Q.Q8_0, (32, 96)) for i in (0, 1)},
    **{f"v.blk.{i}.ln{j}.{p}": (Q.F32, (256,)) for i in (0, 1) for j in (1, 2) for p in ("weight", "bias")},
    "v.blk.0.ffn_gate.weight": (Q.Q4_K, (16, 256)),
    "v.blk.0.ffn_up.weight": (Q.Q8_0, (16, 256)),
    "v.blk.0.ffn_down.weight": (Q.IQ2_XXS, (16, 256)),
    "v.blk.1.ffn_up.weight": (Q.F16, (16, 64)),
    "mm.0.weight": (Q.Q8_0, (256, 32)),
    "mm.0.bias": (Q.F32, (256,)),
    "mm.2.weight": (Q.Q4_K, (32, 256)),
    "v.post_ln.weight": (Q.F32, (256,)),
    "v.post_ln.bias": (Q.F32, (256,)),
}


def main():
    ref = load_ref_loader()
    paths = {name: os.path.join(HERE, name) for name in (tc.UMT5_FILE, tc.MISTRAL_FILE, tc.QWEN_FILE, tc.MMPROJ_FILE)}
    _write(paths[tc.UMT5_FILE], "t5encoder", UMT5, tc.add_t5_tokenizer, seed=100)
    _write(paths[tc.MISTRAL_FILE], "llama", MISTRAL, _mistral_tokenizer, seed=200)
    _write(paths[tc.QWEN_FILE], "qwen2vl", QWEN, seed=300)
    _write(paths[tc.MMPROJ_FILE], "clip", MMPROJ, _mmproj_meta, seed=400)

    temb = "token_embd.weight"
    sds = {}
    sd = ref.gguf_sd_loader(paths[tc.UMT5_FILE], is_text_model=True)
    sd["spiece_model"] = ref.gguf_tokenizer_loader(paths[tc.UMT5_FILE], (256384, 4096))
    sd[temb] = ref.dequantize_tensor(sd[temb], dtype=torch.float16)
    sds[tc.UMT5_FILE] = ref.sd_map_replace(sd, ref.T5_SD_MAP)
    sd = ref.gguf_sd_loader(paths[tc.MISTRAL_FILE], is_text_model=True)
    sd["tekken_model"] = ref.gguf_tekken_tokenizer_loader(paths[tc.MISTRAL_FILE], (131072, 5120))
    sd[temb] = ref.dequantize_tensor(sd[temb], dtype=torch.float16)
    sds[tc.MISTRAL_FILE] = ref.llama_permute(ref.sd_map_replace(sd, ref.LLAMA_SD_MAP), 32, 8)
    sds[tc.QWEN_FILE] = ref.gguf_clip_loader(paths[tc.QWEN_FILE])

    table, arrays = {}, {}
    for fname, sd in sds.items():
        entries = table[fname] = {}
        for key, v in sd.items():
            tag = f"{fname}|{key}"
            if ref.is_quantized(v):
                entries[key] = {"packed": True, "type": v.tensor_type.name, "shape": list(v.tensor_shape)}
                arrays[tag] = tc.tensor_bits(v)
                arrays[tag + "|f32"] = tc.tensor_bits(ref.dequantize_tensor(v, dtype=torch.float32))
            else:
                entries[key] = {"packed": False, "dtype": str(v.dtype).removeprefix("torch."), "shape": list(v.shape)}
                arrays[tag] = tc.tensor_bits(v)
    with open(os.path.join(HERE, tc.GOLDEN_JSON), "w") as f:
        json.dump(table, f, indent=1)
    np.savez_compressed(os.path.join(HERE, tc.GOLDEN_NPZ), **arrays)
    print("wrote", tc.GOLDEN_JSON, tc.GOLDEN_NPZ, f"({len(arrays)} arrays)")


if __name__ == "__main__":
    main()
