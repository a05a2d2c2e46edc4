"""The small text-encoder GGUFs under tests/golden/ (written by tests/golden/make_golden_text_encoders.py) and what the
tests need to know about them.

Four files stand in for the three encoder kinds whose loading needs more than key renaming:
    UMT5_FILE      arch t5encoder, a `t5` sentencepiece tokenizer in the metadata, a UMT5_TABLE token table
    MISTRAL_FILE   arch llama, a `gpt2` byte-level tokenizer, a MISTRAL_TABLE token table
    QWEN_FILE      arch qwen2vl, and beside it MMPROJ_FILE: arch clip, general.type mmproj, a two-block vision tower
The tables are far smaller than the real UMT5 / Mistral ones; tests set loader.UMT5_EMBED_SHAPE /
MISTRAL_EMBED_SHAPE to them.

GOLDEN_JSON maps each file to the reference's state dict, key by key: {"packed": true, "type", "shape"} for a tensor left
packed, else {"packed": false, "dtype", "shape"} (or {"bytes": n} for a tokenizer).  GOLDEN_NPZ holds "<file>|<key>":
the raw bytes of a packed tensor ("<file>|<key>|f32" its fp32 dequantisation), the bit pattern of any other tensor.
"""
import json
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")

UMT5_FILE = "umt5-tiny-Q8_0.gguf"
MISTRAL_FILE = "mistral-tiny-Q4_K_M.gguf"
QWEN_FILE = "Qwen2.5-VL-tiny-Q4_K_M.gguf"
MMPROJ_FILE = "Qwen2.5-VL-tiny-mmproj-F16.gguf"
GOLDEN_JSON = "text_encoders.json"
GOLDEN_NPZ = "text_encoders.npz"

UMT5_TABLE = (160, 64)
MISTRAL_TABLE = (64, 256)

# sentencepiece piece types (sentencepiece_model.proto): NORMAL, UNKNOWN, CONTROL, USER_DEFINED, UNUSED, BYTE
NORMAL, UNKNOWN, CONTROL, USER_DEFINED, UNUSED, BYTE = 1, 2, 3, 4, 5, 6
T5_WORDS = ["▁", "▁the", "▁a", "▁of", "▁and", "▁to", "▁in", "▁is", "▁that", "▁for", "▁it", "▁with", "▁as", "▁was", "▁on",
            "▁be", "▁at", "▁by", "▁this", "▁from", "▁Hello", "▁world", "▁cat", "▁sat", "▁mat", "ing", "ed", "er", "ly",
            "▁über", "▁日本", "語", "▁день", "é", "."] + list("abcdefghijklmnopqrstuvwxyzHW")


def t5_tokenizer():
    """(tokens, scores, types) of a UMT5-like unigram vocabulary: pad / eos / unk first, the 256 byte pieces, words,
    two user-defined pieces and one unused piece."""
    tokens = ["<pad>", "</s>", "<unk>"]
    types = [CONTROL, CONTROL, UNKNOWN]
    scores = [0.0, 0.0, 0.0]
    for b in range(256):
        tokens.append(f"<0x{b:02X}>")
        types.append(BYTE)
        scores.append(0.0)
    for i, w in enumerate(T5_WORDS):
        tokens.append(w)
        types.append(NORMAL)
        scores.append(-1.0 - 0.25 * i)
    tokens += ["<extra_id_1>", "<extra_id_0>", "<unused_0>"]
    types += [USER_DEFINED, USER_DEFINED, UNUSED]
    scores += [0.0, 0.0, 0.0]
    return tokens, scores, types


def add_t5_tokenizer(writer):
    tokens, scores, types = t5_tokenizer()
    writer.add_tokenizer_model("t5")
    writer.add_token_list(tokens)
    writer.add_token_scores(scores)
    writer.add_token_types(types)
    writer.add_add_space_prefix(True)
    writer.add_remove_extra_whitespaces(True)
    writer.add_eos_token_id(1)
    writer.add_pad_token_id(0)


def golden():
    with open(os.path.join(GOLDEN, GOLDEN_JSON)) as f:
        return json.load(f), np.load(os.path.join(GOLDEN, GOLDEN_NPZ))


_BITS = {torch.float16: np.uint16, torch.bfloat16: np.uint16, torch.float32: np.uint32, torch.uint8: np.uint8}


def tensor_bits(t):
    """The bit pattern of a plain tensor (any subclass dropped), on the host, flat."""
    t = t.as_subclass(torch.Tensor).detach().cpu().contiguous()
    width = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()]
    return t.view(width).numpy().view(_BITS[t.dtype]).reshape(-1)
