"""GPU tests of the UMT5, Mistral and Qwen2.5-VL text-encoder loading (loader.py): the tensors gguf_clip_loader dequantises
(token tables, the 5-D patch embedding, the fused vision q/k/v) are bit-identical to what the reference loads from the
fixtures under tests/golden/, and every tensor it leaves packed runs on the packed-Linear / Embedding kernels within 1e-3
of the float64 product of the reference's dequantised weight.  One test loads a token table at the full UMT5 size."""
import os

import gguf
import numpy as np
import pytest
import torch

import text_encoder_cases as tc
from fallback_cases import gguf_values, random_blocks
from util import rel_fro

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
Q = gguf.GGMLQuantizationType
FILES = [tc.UMT5_FILE, tc.MISTRAL_FILE, tc.QWEN_FILE]


@pytest.fixture(scope="module")
def gold():
    return tc.golden()


@pytest.fixture
def small_tables(pkg, monkeypatch):
    monkeypatch.setattr(pkg.loader, "UMT5_EMBED_SHAPE", tc.UMT5_TABLE)
    monkeypatch.setattr(pkg.loader, "MISTRAL_EMBED_SHAPE", tc.MISTRAL_TABLE)


def _path(name):
    return os.path.join(tc.GOLDEN, name)


def _dtype_name(t):
    return str(t.dtype).removeprefix("torch.")


def _check_unpacked(sd, entries, arrays, fname):
    """Every tensor the reference does not leave packed: same dtype, shape and bits."""
    for key, e in entries.items():
        if e["packed"]:
            continue
        v = sd[key]
        assert _dtype_name(v) == e["dtype"] and list(v.shape) == e["shape"], key
        assert np.array_equal(tc.tensor_bits(v), arrays[f"{fname}|{key}"]), key


@pytest.mark.parametrize("fname", FILES)
def test_loaded_tensors_are_the_reference_bits(pkg, gold, small_tables, fname):
    table, arrays = gold
    sd = pkg.loader.gguf_clip_loader(_path(fname))
    assert set(sd) == set(table[fname])
    _check_unpacked(sd, table[fname], arrays, fname)
    for key, e in table[fname].items():
        if e["packed"]:
            assert sd[key].tensor_type.name == e["type"] and list(sd[key].tensor_shape) == e["shape"], key
            assert np.array_equal(tc.tensor_bits(sd[key]), arrays[f"{fname}|{key}"]), key


def _rel(y, ref):
    return rel_fro(y.float().cpu().numpy(), ref.float().cpu().numpy())


@pytest.mark.parametrize("fname", FILES)
def test_packed_tensors_run_on_the_kernels(pkg, gold, small_tables, fname):
    table, arrays = gold
    sd = pkg.loader.gguf_clip_loader(_path(fname))
    g = torch.Generator().manual_seed(11)
    ran = 0
    for key, e in table[fname].items():
        if not e["packed"]:
            continue
        N, K = e["shape"]
        w32 = torch.from_numpy(arrays[f"{fname}|{key}|f32"].view(np.float32).reshape(N, K)).to(DEV)
        if key.endswith("embed_tokens.weight"):
            emb = pkg.ops.GGMLOps.Embedding(N, K, device="meta")
            emb.load_state_dict({"weight": sd[key]}, assign=True)
            ids = torch.randint(0, N, (2, 9), generator=g).to(DEV)
            assert torch.equal(emb(ids), torch.nn.functional.embedding(ids, w32)), key
        else:
            lin = pkg.ops.GGMLOps.Linear(K, N)
            lin.load_state_dict({"weight": sd[key]})
            for M, dt in ((5, torch.bfloat16), (77, torch.float16)):
                x = torch.randn(M, K, generator=g).to(DEV).to(dt)
                want = (x.double() @ w32.to(dt).double().t()).to(dt)
                y = lin(x)
                assert y.dtype == dt and tuple(y.shape) == (M, N)
                assert _rel(y, want) <= 1e-3, (key, M)
        ran += 1
    assert ran == sum(e["packed"] for e in table[fname].values()) > 0


def test_clip_loader_node_returns_the_merged_dict(pkg, gold):
    import importlib
    import __graft_entry__ as ge
    nodes = importlib.import_module(f"{ge.PKG_NAME}.nodes")
    table, arrays = gold
    (sd,) = nodes.CLIPLoaderGGUF().load_data([_path(tc.QWEN_FILE)])
    assert set(sd) == set(table[tc.QWEN_FILE])
    assert any(k.startswith("visual.") for k in sd) and any(k.startswith("model.") for k in sd)
    _check_unpacked(sd, table[tc.QWEN_FILE], arrays, tc.QWEN_FILE)


def test_full_size_umt5_table(pkg, gold, tmp_path):
    """A t5encoder GGUF with a (256384, 4096) TQ1_0 token table (about 220 MB) at the real UMT5_EMBED_SHAPE: the tokenizer
    is rebuilt and the table dequantised to fp16 on the GPU, equal to gguf-py's values rounded to fp16."""
    _table, arrays = gold
    V, D = pkg.loader.UMT5_EMBED_SHAPE
    assert (V, D) == (256384, 4096)
    qt = Q.TQ1_0
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    per_row = D // bs
    raw = random_blocks(qt, V * per_row, seed=17, scale=0.01)
    path = str(tmp_path / "umt5-xxl-encoder-TQ1_0.gguf")
    w = gguf.GGUFWriter(path, "t5encoder")
    tc.add_t5_tokenizer(w)
    w.add_tensor("token_embd.weight", raw.reshape(V, per_row * ts), raw_dtype=qt)
    w.add_tensor("enc.output_norm.weight", np.ones(D, dtype=np.float32))
    w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()

    sd = pkg.loader.gguf_clip_loader(path)
    assert set(sd) == {"shared.weight", "encoder.final_layer_norm.weight", "spiece_model"}
    assert np.array_equal(sd["spiece_model"].numpy(), arrays[f"{tc.UMT5_FILE}|spiece_model"])
    table = sd["shared.weight"]
    assert table.dtype == torch.float16 and tuple(table.shape) == (V, D)
    rows = [0, 1, 4095, 4096, 65535, 131072, 200003, V - 2, V - 1]
    rows += np.random.default_rng(3).integers(0, V, size=23).tolist()
    for r in rows:
        want = torch.from_numpy(gguf_values(raw[r * per_row:(r + 1) * per_row], qt)).to(torch.float16)
        assert torch.equal(table[r].view(torch.int16), want.view(torch.int16)), r
