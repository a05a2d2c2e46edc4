"""CPU tests of the UMT5, Mistral and Qwen2.5-VL text-encoder loading in loader.py (reference loader.py:213-406): the rebuilt
sentencepiece and tekken tokenizers, the mmproj sibling search, and gguf_clip_loader's state dict for each fixture under
tests/golden/, against what the reference loads from the same files (tests/golden/make_golden_text_encoders.py).

Without a GPU the quantised tensors the loader dequantises cannot be formed, so these tests replace dequantize_tensor by
a stand-in of the right shape and dtype; tests/test_gpu_text_encoder_loaders.py checks their values."""
import base64
import json
import logging
import os
import shutil

import gguf
import numpy as np
import pytest
import torch

import text_encoder_cases as tc

Q = gguf.GGMLQuantizationType


@pytest.fixture(scope="module")
def gold():
    return tc.golden()


def _path(name):
    return os.path.join(tc.GOLDEN, name)


@pytest.fixture
def small_tables(pkg, monkeypatch):
    monkeypatch.setattr(pkg.loader, "UMT5_EMBED_SHAPE", tc.UMT5_TABLE)
    monkeypatch.setattr(pkg.loader, "MISTRAL_EMBED_SHAPE", tc.MISTRAL_TABLE)


@pytest.fixture
def host_dequant(pkg, monkeypatch):
    """dequantize_tensor without a GPU: F32 / F16 as the real one, quantised tensors as zeros of the result's shape."""
    real = pkg.loader.dequantize_tensor

    def stand_in(t, dtype=None, dequant_dtype=None):
        if not pkg.dequant.is_quantized(t):
            return real(t, dtype, dequant_dtype)
        return torch.zeros(tuple(t.tensor_shape), dtype=dtype or torch.float32)
    monkeypatch.setattr(pkg.loader, "dequantize_tensor", stand_in)


def test_fixtures_cover_every_dequantised_kind(gold):
    """What the reference dequantises while loading the fixtures: fp16 token tables, the 5-D fp32 patch embedding, the
    fused q/k/v in bf16 (quantised halves) or fp16."""
    table, _arrays = gold
    assert table[tc.UMT5_FILE]["shared.weight"] == {"packed": False, "dtype": "float16", "shape": list(tc.UMT5_TABLE)}
    assert table[tc.MISTRAL_FILE]["model.embed_tokens.weight"] == {"packed": False, "dtype": "float16", "shape": list(tc.MISTRAL_TABLE)}
    qwen = table[tc.QWEN_FILE]
    assert qwen["visual.patch_embed.proj.weight"] == {"packed": False, "dtype": "float32", "shape": [64, 3, 2, 4, 4]}
    assert qwen["visual.blocks.0.attn.qkv.weight"] == {"packed": False, "dtype": "bfloat16", "shape": [48, 256]}
    assert qwen["visual.blocks.1.attn.qkv.weight"] == {"packed": False, "dtype": "float16", "shape": [48, 256]}
    assert qwen["visual.blocks.0.attn.qkv.bias"] == {"packed": False, "dtype": "float16", "shape": [48]}
    assert {qwen[f"visual.blocks.0.attn_{p}.weight"]["type"] for p in "qkv"} == {"Q4_K", "Q8_0", "IQ2_XXS"}


def _bytes(t):
    return bytes(t.numpy().tobytes())


def test_spiece_model_equals_the_reference(pkg, gold):
    table, arrays = gold
    got = pkg.loader.gguf_tokenizer_loader(_path(tc.UMT5_FILE), (256384, 4096))
    assert got.dtype == torch.uint8 and got.dim() == 1
    assert np.array_equal(got.numpy(), arrays[f"{tc.UMT5_FILE}|spiece_model"])


def test_spiece_model_tokenizes(pkg):
    import sentencepiece
    from sentencepiece import sentencepiece_model_pb2
    blob = _bytes(pkg.loader.gguf_tokenizer_loader(_path(tc.UMT5_FILE), (256384, 4096)))
    proto = sentencepiece_model_pb2.ModelProto.FromString(blob)
    tokens, scores, types = tc.t5_tokenizer()
    assert [p.piece for p in proto.pieces] == tokens and [p.type for p in proto.pieces] == types
    assert np.array_equal([p.score for p in proto.pieces], np.float32(scores))
    assert proto.trainer_spec.model_type == sentencepiece_model_pb2.TrainerSpec.UNIGRAM and not proto.trainer_spec.HasField("model_type")
    assert (proto.trainer_spec.vocab_size, proto.trainer_spec.eos_id, proto.trainer_spec.pad_id) == (len(tokens), 1, 0)
    assert proto.trainer_spec.byte_fallback and proto.normalizer_spec.add_dummy_prefix

    sp = sentencepiece.SentencePieceProcessor(model_proto=blob)
    assert sp.vocab_size() == len(tokens) and sp.eos_id() == 1 and sp.pad_id() == 0
    for text in ("Hello world", "the cat sat on the mat", "über 日本語 день", "  extra   spaces  ", "emoji 🙂 and ¿?"):
        ids = sp.encode(text)
        assert sp.decode(ids) == " ".join(text.split()), text
    assert sp.encode("the cat", out_type=str) == ["▁the", "▁cat"]
    assert "<0xF0>" in sp.encode("🙂", out_type=str)          # byte fallback for a character with no piece


def test_tekken_model_equals_the_reference(pkg, gold):
    table, arrays = gold
    got = pkg.loader.gguf_tekken_tokenizer_loader(_path(tc.MISTRAL_FILE), (131072, 5120))
    assert got.dtype == torch.uint8
    assert np.array_equal(got.numpy(), arrays[f"{tc.MISTRAL_FILE}|tekken_model"])
    data = json.loads(_bytes(got))
    assert data["config"] == {"num_vocab_tokens": 150000, "default_vocab_size": 131072}
    assert [s["rank"] for s in data["special_tokens"]] == [0, 1, 2, 259, 260, 261]
    assert [v["rank"] for v in data["vocab"]] == list(range(len(data["vocab"])))
    by_bytes = {base64.b64decode(v["token_bytes"]): v["token_str"] for v in data["vocab"]}
    assert by_bytes[b" the"] == " the" and by_bytes["’".encode()] == "’" and by_bytes[b"\xe6\x97"] == "\ufffd"
    assert len(by_bytes) == len(data["vocab"]) and all(bytes([b]) in by_bytes for b in range(256))


def test_gpt2_byte_map_is_a_bijection(pkg):
    decoder = pkg.loader._gpt2_byte_decoder()
    assert sorted(decoder.values()) == list(range(256)) and len(decoder) == 256
    assert decoder["Ġ"] == 0x20 and decoder["Ċ"] == 0x0A and decoder["!"] == 0x21 and decoder["ÿ"] == 0xFF and decoder["Ā"] == 0


@pytest.mark.parametrize("loader, path, good", [("gguf_tokenizer_loader", tc.UMT5_FILE, (256384, 4096)),
                                                ("gguf_tekken_tokenizer_loader", tc.MISTRAL_FILE, (131072, 5120))])
def test_unknown_tokenizer_raises(pkg, loader, path, good):
    fn = getattr(pkg.loader, loader)
    other = tc.MISTRAL_FILE if path == tc.UMT5_FILE else tc.UMT5_FILE
    for p, shape in ((path, (good[0] - 1, good[1])), (path, (good[0], good[1] * 2)), (other, good), (tc.QWEN_FILE, good)):
        with pytest.raises(NotImplementedError, match="Unknown model, can't set tokenizer!"):
            fn(_path(p), shape)


@pytest.mark.parametrize("name, stem", [
    ("qwen2.5-vl-7b-instruct-q4_k_m", "qwen2.5-vl-7b-instruct"),
    ("Qwen2.5-VL-7B-Instruct-Q4_K_M", "Qwen2.5-VL-7B-Instruct"),
    ("qwen2.5-vl-7b-instruct-iq2_xxs", "qwen2.5-vl-7b-instruct"),
    ("Qwen2.5-VL-7B-Instruct-UD-Q5_K_XL", "Qwen2.5-VL-7B-Instruct"),
    ("qwen2.5-vl-7b-instruct_q8_0", "qwen2.5-vl-7b-instruct"),
    ("qwen2.5-vl-7b-instruct", "qwen2.5-vl-7b-instruct"),
    ("qwen2.5-vl-7b-instruct-f16", "qwen2.5-vl-7b-instruct-f16"),
    ("model-q4_k_m_extra_long_tail", "model-q4_k_m_extra_long_tail"),
])
def test_strip_quant_suffix(pkg, name, stem):
    assert pkg.loader.strip_quant_suffix(name) == stem


def _tiny_mmproj(path, tensor_name):
    w = gguf.GGUFWriter(path, "clip")
    w.add_type("mmproj")
    w.add_tensor(tensor_name, np.ones(8, dtype=np.float32))
    w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()


def test_mmproj_missing_logs_and_returns_nothing(pkg, tmp_path, caplog):
    enc = tmp_path / "Qwen2.5-VL-7B-Instruct-Q4_K_M.gguf"
    _tiny_mmproj(str(tmp_path / "other-model-mmproj-F16.gguf"), "v.post_ln.weight")
    (tmp_path / "Qwen2.5-VL-7B-Instruct-mmproj.txt").write_text("not a gguf")
    with caplog.at_level(logging.ERROR):
        assert pkg.loader.gguf_mmproj_loader(str(enc)) == {}
    assert any(r.levelno == logging.ERROR and "Can't find mmproj" in r.getMessage() for r in caplog.records)


def test_mmproj_ambiguous_takes_the_first_listed(pkg, tmp_path, caplog):
    enc = tmp_path / "Qwen2.5-VL-7B-Instruct-Q4_K_M.gguf"
    names = {"Qwen2.5-VL-7B-Instruct-mmproj-F16.gguf": "v.post_ln.weight", "mmproj-qwen2.5-vl-7b-instruct-BF16.GGUF": "mm.0.bias"}
    for name, tensor in names.items():
        _tiny_mmproj(str(tmp_path / name), tensor)
    first = next(f for f in os.listdir(tmp_path) if f in names)
    want = pkg.loader.sd_map_replace({names[first]: None}, pkg.loader.CLIP_VISION_SD_MAP)
    with caplog.at_level(logging.ERROR):
        got = pkg.loader.gguf_mmproj_loader(str(enc))
    assert set(got) == set(want)
    assert any(r.levelno == logging.ERROR and "Ambiguous mmproj" in r.getMessage() for r in caplog.records)


@pytest.mark.parametrize("fname", [tc.UMT5_FILE, tc.MISTRAL_FILE, tc.QWEN_FILE])
def test_clip_loader_matches_the_reference(pkg, gold, small_tables, host_dequant, fname):
    table, arrays = gold
    sd = pkg.loader.gguf_clip_loader(_path(fname))
    assert set(sd) == set(table[fname])
    for key, e in table[fname].items():
        if e["packed"]:       # left packed: same type, logical shape and bytes (llama_permute included)
            v = sd[key]
            assert pkg.dequant.is_quantized(v), key
            assert v.tensor_type.name == e["type"] and list(v.tensor_shape) == e["shape"], key
            assert np.array_equal(tc.tensor_bits(v), arrays[f"{fname}|{key}"]), key
    for key in ("spiece_model", "tekken_model"):
        if key in sd:
            assert np.array_equal(sd[key].numpy(), arrays[f"{fname}|{key}"])


def test_clip_loader_without_the_shape_constants(pkg, gold, host_dequant):
    """At the real UMT5 / Mistral shapes the small fixture tables are ordinary encoders: no tokenizer, table left packed."""
    table, _arrays = gold
    t5 = pkg.loader.gguf_clip_loader(_path(tc.UMT5_FILE))
    assert "spiece_model" not in t5 and t5["shared.weight"].tensor_type == Q.Q8_0
    mistral = pkg.loader.gguf_clip_loader(_path(tc.MISTRAL_FILE))
    assert "tekken_model" not in mistral and mistral["model.embed_tokens.weight"].tensor_type == Q.Q4_K
    assert set(mistral) == set(table[tc.MISTRAL_FILE]) - {"tekken_model"}


def test_qwen2vl_without_mmproj_still_loads_the_text_model(pkg, gold, tmp_path, caplog):
    table, _arrays = gold
    shutil.copy(_path(tc.QWEN_FILE), tmp_path / tc.QWEN_FILE)
    with caplog.at_level(logging.ERROR):
        sd = pkg.loader.gguf_clip_loader(str(tmp_path / tc.QWEN_FILE))
    assert set(sd) == {k for k in table[tc.QWEN_FILE] if not k.startswith("visual.")}
    assert any("Can't find mmproj" in r.getMessage() for r in caplog.records)
