"""CPU tests of the K-quant encoders (Q2_K ... Q6_K) and the converter's K mixtures:
  * restatement parity: the product's encoder pieces (comfyui-gguf_b200/csrc/quantize.cuh, compiled for the host by
    tests/host_quantize_k.cu) equal the plain-C restatement of llama.cpp's reference quantisers (tests/kquant_oracle.c) bit for
    bit, on seeded, heavy-tailed and adversarial super-blocks, for values from fp32, fp16 and bf16 sources;
  * the layout, independent of the restatement: decoded by the existing dequant oracle, every element inside its group's code
    range lies within half a step of its value;
  * quality: round-trip RMSE orders Q2_K > Q3_K > Q4_K > Q5_K > Q6_K, and Q4_K / Q5_K beat Q4_0 / Q5_0;
  * the converter's nine K mixtures: per-tensor types, the attention-value counter, the F16 fallback, general.file_type;
  * the ABI constants of ggufb200_quantize_k."""
import os
import re

import gguf
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
import kquant_cases as kc
import quantize_cases as qc

Q = gguf.GGMLQuantizationType
DTYPES = ["f32", "f16", "bf16"]


@pytest.fixture(scope="module")
def oracle_k():
    L = kc.oracle_lib()
    if L is None:
        pytest.skip("gcc not available")
    return L


@pytest.fixture(scope="module")
def host_k():
    L = kc.host_lib()
    if L is None:
        pytest.skip("nvcc not available")
    return L


def _datasets(dt):
    return {
        "seeded": kc.to_dtype_values(kc.seeded_blocks(512, seed=1), dt),
        "heavy": kc.to_dtype_values(kc.seeded_blocks(512, seed=2, heavy=True), dt),
        "adversarial": kc.to_dtype_values(kc.adversarial_blocks(), dt),
    }


def _finite_rows(x):
    return x[np.isfinite(x).all(1)]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("qt", kc.K_TYPES, ids=lambda q: q.name)
def test_functors_equal_the_c_restatement(oracle_k, host_k, qt, dt):
    ts = gguf.GGML_QUANT_SIZES[qt][1]
    for name, x in _datasets(dt).items():
        x = _finite_rows(x)                                         # fp16 turns the largest adversarial rows into Inf
        want = kc.encode(oracle_k, x, qt).reshape(-1, ts)
        got = kc.encode(host_k, x, qt, "hostk_quantize").reshape(-1, ts)
        bad = np.flatnonzero((want != got).any(1))
        assert bad.size == 0, (qt.name, dt, name, bad[:5])


def test_adversarial_blocks_reach_the_edge_cases(oracle_k):
    """The adversarial set exercises what it claims: D <= 0 and this_min > 0 in make_qkx2_quants, its max == min exit, the early
    exit of make_q3_quants' refinement, Q6_K's all-zero block, groups below GROUP_MAX_EPS next to groups above it, and bf16
    values beyond the fp16 range."""
    x = kc.adversarial_blocks()
    assert np.isfinite(x).all()
    assert (np.abs(x) > 65504).any() and np.isfinite(x.astype(np.float32)).all()
    counts = {}
    for qt in kc.K_TYPES:
        oracle_k.kqor_reset_counters()
        kc.encode(oracle_k, x, qt)
        counts[qt] = [oracle_k.kqor_counter(i) for i in range(4)]
    assert counts[Q.Q2_K][0] > 0 and counts[Q.Q4_K][0] + counts[Q.Q5_K][0] > 0, counts      # D <= 0
    assert counts[Q.Q2_K][1] > 0 and counts[Q.Q4_K][1] > 0 and counts[Q.Q5_K][1] > 0, counts  # this_min > 0
    assert counts[Q.Q3_K][2] > 0, counts                                                   # refinement converged early
    assert counts[Q.Q2_K][3] > 0 and counts[Q.Q4_K][3] > 0, counts                         # max == min
    q6 = kc.encode(oracle_k, x, Q.Q6_K).reshape(len(x), -1)
    zero_rows = np.flatnonzero(~(q6.any(1)))
    assert zero_rows.size >= 3                                    # zeros, -0 and the sub-epsilon blocks
    assert (np.abs(x[zero_rows]).max(1) > 0).any()                # the early exit, not only all-zero input


@pytest.mark.parametrize("qt", kc.K_TYPES, ids=lambda q: q.name)
def test_all_zero_blocks_encode_to_zero_bytes(oracle_k, host_k, qt):
    x = np.zeros((3, 256), np.float32)
    x[1] = -0.0
    assert not kc.encode(oracle_k, x, qt).any()
    assert not kc.encode(host_k, x, qt, "hostk_quantize").any()


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("qt", kc.K_TYPES, ids=lambda q: q.name)
def test_layout_decodes_within_half_a_step(oracle_k, qt, dt):
    """Independent of the restatement: through the existing dequant oracle, an element whose scaled value lies inside its
    group's code range decodes within half a step of its value.  A mispacked scale, min, high bit or code fails this whatever
    the search chose."""
    checked = 0
    for name, x in _datasets(dt).items():
        x = _finite_rows(x)
        bad, n = kc.layout_violations(kc.encode(oracle_k, x, qt), x, qt)
        assert bad.size == 0, (qt.name, dt, name, bad[:5])
        checked += n
    assert checked > 0.8 * 1024 * 256


def test_rmse_orders_the_types(oracle_k, host_k):
    """On seeded Gaussian data: Q2_K > Q3_K > Q4_K > Q5_K > Q6_K, and the K types beat the legacy types of the same bits per
    weight.  Checked on the C restatement first, then on the product's pieces."""
    x = np.random.default_rng(7).standard_normal((256, 256)).astype(np.float32) * np.float32(0.02)
    for L, fn in ((oracle_k, "kqor_quantize"), (host_k, "hostk_quantize")):
        e = {qt: kc.rmse(kc.encode(L, x, qt, fn), x, qt) for qt in kc.K_TYPES}
        assert e[Q.Q2_K] > e[Q.Q3_K] > e[Q.Q4_K] > e[Q.Q5_K] > e[Q.Q6_K], e
        legacy = {qt: float(np.sqrt(np.mean((gguf.quants.dequantize(qc.gguf_bytes(x.reshape(-1, 32), qt), qt).reshape(-1)
                                              - x.reshape(-1).astype(np.float64)) ** 2))) for qt in (Q.Q4_0, Q.Q5_0)}
        assert e[Q.Q4_K] < legacy[Q.Q4_0] and e[Q.Q5_K] < legacy[Q.Q5_0], (e, legacy)


# ---------------------------------------------------------------- converter: K mixtures
@pytest.fixture(scope="module")
def conv():
    return ge._sub("convert")


def _meta(*shape, dtype=torch.bfloat16):
    return torch.empty(shape, dtype=dtype, device="meta")


KEYSETS = {
    "flux": {
        "img_in.weight": _meta(3072, 64),
        "double_blocks.0.img_attn.qkv.weight": _meta(9216, 3072),
        "double_blocks.0.img_attn.proj.weight": _meta(3072, 3072),
        "double_blocks.0.img_attn.norm.key_norm.scale": _meta(128),
        "double_blocks.0.img_mlp.0.weight": _meta(12288, 3072),
        "double_blocks.0.img_mlp.2.weight": _meta(3072, 12288),
        "double_blocks.0.odd.weight": _meta(3072, 48),                       # BF16 stage 1, rows not a multiple of 256
        "double_blocks.0.odd16.weight": _meta(3072, 320, dtype=torch.float16),  # F16 stage 1, the same
        "single_blocks.0.linear1.weight": _meta(21504, 3072),
        "single_blocks.0.linear2.weight": _meta(3072, 15360),
        "final_layer.linear.weight": _meta(64, 3072),
    },
    "sd3": {
        "joint_blocks.0.x_block.attn.qkv.weight": _meta(4608, 1536, dtype=torch.float16),
        "joint_blocks.0.x_block.mlp.fc2.weight": _meta(1536, 6144, dtype=torch.float16),
        "joint_blocks.0.context_block.attn.qkv.weight": _meta(4608, 1536, dtype=torch.float16),
        "pos_embed": _meta(1, 36864, 1536, dtype=torch.float16),
        "proj_out.weight": _meta(64, 1536, dtype=torch.float16),
    },
    "wan": {
        "blocks.0.self_attn.norm_q.weight": _meta(5120),
        "blocks.0.self_attn.q.weight": _meta(5120, 5120),
        "blocks.0.self_attn.v.weight": _meta(5120, 100),                      # counted, then F16
        "blocks.0.cross_attn.v.weight": _meta(5120, 5120),
        "blocks.0.ffn.0.weight": _meta(13824, 5120),
        "blocks.0.ffn.2.weight": _meta(5120, 13824),
        "blocks.1.self_attn.v.weight": _meta(5120, 5120),
        "blocks.1.cross_attn.v.weight": _meta(5120, 5120),
        "blocks.1.ffn.2.weight": _meta(5120, 13800),                          # ffn_down, then F16
        "blocks.2.self_attn.v.weight": _meta(5120, 5120),
        "blocks.2.cross_attn.v.weight": _meta(5120, 5120),
        "text_embedding.2.weight": _meta(5120, 5120),
        "head.modulation": _meta(1, 2, 5120, dtype=torch.float32),
    },
    "hidream": {
        "caption_projection.0.linear.weight": _meta(2560, 4096),
        "double_stream_blocks.0.block.attn1.to_v.weight": _meta(2560, 2560),
        "double_stream_blocks.0.block.attn1.to_v_t.weight": _meta(2560, 2560),
        "double_stream_blocks.0.block.ff_i.shared_experts.w3.weight": _meta(3584, 2560),
        "double_stream_blocks.0.block.ff_i.shared_experts.w2.weight": _meta(2560, 3584),
        "double_stream_blocks.0.block.ff_i.experts.0.w2.weight": _meta(2560, 3584),
        "double_stream_blocks.0.block.ff_i.gate.weight": _meta(4, 2560),
    },
    "sdxl": {
        "input_blocks.1.0.in_layers.2.weight": _meta(320, 320, 3, 3, dtype=torch.float16),       # reshaped: rows of 256
        "input_blocks.4.1.proj_in.weight": _meta(640, 640, dtype=torch.float16),                  # reshaped
        "input_blocks.4.1.transformer_blocks.0.attn1.to_v.weight": _meta(640, 640, dtype=torch.float16),
        "input_blocks.4.1.transformer_blocks.0.attn2.to_v.weight": _meta(640, 2048, dtype=torch.float16),
        "input_blocks.4.1.transformer_blocks.0.ff.net.2.weight": _meta(640, 2560, dtype=torch.float16),
        "middle_block.1.proj_in.weight": _meta(1280, 1280, dtype=torch.float16),
        "middle_block.1.transformer_blocks.0.attn1.to_v.weight": _meta(1280, 1280, dtype=torch.float16),
        "middle_block.1.transformer_blocks.0.attn2.to_v.weight": _meta(1280, 2048, dtype=torch.float16),
        "output_blocks.0.0.x.weight": _meta(3, 5, 7, 11, dtype=torch.float16),                   # 4-D, not reshaped: kept
        "time_embed.0.weight": _meta(1280, 320, dtype=torch.float16),
        "input_blocks.0.0.weight": _meta(320, 4, 3, 3, dtype=torch.float16),
    },
}


def _reference_types(sd, arch, name):
    """img_tensor_get_type restated for a whole file: the i-th attention-value tensor, counted over every tensor that reaches the
    function (2-D weights, not norms, not kept), its row check afterwards."""
    default = {"Q2_K": Q.Q2_K, "Q3_K_S": Q.Q3_K, "Q3_K_M": Q.Q3_K, "Q3_K_L": Q.Q3_K, "Q4_K_S": Q.Q4_K, "Q4_K_M": Q.Q4_K,
               "Q5_K_S": Q.Q5_K, "Q5_K_M": Q.Q5_K, "Q6_K": Q.Q6_K}[name]
    V = ("attn_v.weight", ".to_v.weight", ".v.weight", ".attn.w1v.weight", ".attn.w2v.weight", "_attn.v_proj.weight")
    QKV = ("attn_qkv.weight", "attn.qkv.weight", "attention.qkv.weight")
    FFN = ("ffn_down", ".ffn.2.weight", ".ff.net.2.weight", ".mlp.layer2.weight", ".adaln_modulation_mlp.2.weight",
           ".feed_forward.w2.weight")
    i_v = 0
    out = {}
    conv = ge._sub("convert")
    for key, t in sd.items():
        stage1, reshape = conv.stage1_type(key, t.dtype, t.shape, arch)
        shape = (t.numel() // 256, 256) if reshape else tuple(t.shape)
        lead = next((i for i, d in enumerate(shape) if d != 1), len(shape) - 1)
        reaches = (stage1 in (Q.F16, Q.BF16) and len(shape) - lead == 2 and key.endswith("weight") and "_norm.weight" not in key
                   and not any(k in key for k in arch.keep) and key not in arch.keep_names)
        if not reaches:
            out[key] = stage1
            continue
        new = default
        if any(p in key for p in V):
            new = {"Q2_K": Q.Q3_K, "Q3_K_M": Q.Q5_K if i_v < 2 else Q.Q4_K, "Q3_K_L": Q.Q5_K, "Q4_K_M": Q.Q6_K,
                   "Q5_K_M": Q.Q6_K}.get(name, new)
            if name == "Q4_K_S" and i_v < 4:
                new = Q.Q5_K
            i_v += 1
        elif any(p in key for p in QKV):
            new = {"Q3_K_M": Q.Q4_K, "Q3_K_L": Q.Q4_K, "Q4_K_M": Q.Q5_K, "Q5_K_M": Q.Q6_K}.get(name, new)
        elif any(p in key for p in FFN) or ("experts." in key and ".w2.weight" in key):
            new = {"Q3_K_M": Q.Q4_K, "Q3_K_L": Q.Q5_K, "Q4_K_S": Q.Q5_K, "Q4_K_M": Q.Q6_K, "Q5_K_M": Q.Q6_K}.get(name, new)
        out[key] = new if shape[-1] % 256 == 0 else Q.F16
    return out


MIXTURES = ["Q2_K", "Q3_K_S", "Q3_K_M", "Q3_K_L", "Q4_K_S", "Q4_K_M", "Q5_K_S", "Q5_K_M", "Q6_K"]


def test_the_mixture_table(conv):
    assert list(conv.KQUANT_MIXTURES) == MIXTURES
    for name, mix in conv.KQUANT_MIXTURES.items():
        assert mix.file_type == getattr(gguf.LlamaFileType, f"MOSTLY_{name}")
    # the legacy names and file types are unchanged
    assert list(conv.QTYPES) == ["F16", "BF16", "Q8_0", "Q5_1", "Q5_0", "Q4_1", "Q4_0"]
    assert set(conv.FILE_TYPES) == {Q.F16, Q.BF16, Q.Q8_0, Q.Q5_1, Q.Q5_0, Q.Q4_1, Q.Q4_0}


@pytest.mark.parametrize("name", MIXTURES)
@pytest.mark.parametrize("arch_name", sorted(KEYSETS))
def test_mixture_policy(conv, arch_name, name):
    sd = KEYSETS[arch_name]
    arch = conv.ARCH_BY_NAME[arch_name]
    plans = conv.plan_tensors(sd, arch, conv.KQUANT_MIXTURES[name])
    assert [p.key for p in plans] == list(sd)
    want = _reference_types(sd, arch, name)
    assert {p.key: p.qtype for p in plans} == want
    # every quantised tensor has rows of 256; the rest keep their stage-1 type or fell back to F16
    for p in plans:
        if p.qtype in conv.KQUANT_TYPES:
            assert p.shape[-1] % 256 == 0 and len(p.shape) - next(i for i, d in enumerate(p.shape) if d != 1) == 2


def test_attention_value_counter(conv):
    """Q3_K_M: the first two attention-value tensors Q5_K, later ones Q4_K; Q4_K_S: the first four Q5_K.  The counter includes
    the attention-value tensor that falls back to F16 for its rows, and skips one that never reaches the rule."""
    arch = conv.ARCH_BY_NAME["wan"]
    sd = dict(KEYSETS["wan"])
    sd = {"blocks.9.self_attn.v.weight": _meta(5120), **sd}                 # 1-D: never reaches the rule, not counted
    v_keys = [k for k in sd if k.endswith(".v.weight") and sd[k].dim() == 2]
    types = lambda name: [p.qtype for p in conv.plan_tensors(sd, arch, conv.KQUANT_MIXTURES[name]) if p.key in v_keys]
    assert types("Q3_K_M") == [Q.F16, Q.Q5_K, Q.Q4_K, Q.Q4_K, Q.Q4_K, Q.Q4_K]
    assert types("Q4_K_S") == [Q.F16, Q.Q5_K, Q.Q5_K, Q.Q5_K, Q.Q4_K, Q.Q4_K]
    assert types("Q2_K") == [Q.F16] + [Q.Q3_K] * 5
    assert types("Q5_K_S") == [Q.F16] + [Q.Q5_K] * 5


def test_f16_fallback_and_sdxl_reshape(conv):
    flux = {p.key: p for p in conv.plan_tensors(KEYSETS["flux"], conv.ARCH_BY_NAME["flux"], conv.KQUANT_MIXTURES["Q4_K_S"])}
    assert flux["double_blocks.0.odd.weight"].stage1 == Q.BF16 and flux["double_blocks.0.odd.weight"].qtype == Q.F16
    assert flux["double_blocks.0.odd16.weight"].qtype == Q.F16
    assert flux["double_blocks.0.img_attn.qkv.weight"].qtype == Q.Q4_K
    assert flux["img_in.weight"].qtype == Q.BF16 and flux["final_layer.linear.weight"].qtype == Q.BF16
    sdxl = {p.key: p for p in conv.plan_tensors(KEYSETS["sdxl"], conv.ARCH_BY_NAME["sdxl"], conv.KQUANT_MIXTURES["Q6_K"])}
    assert sdxl["input_blocks.4.1.proj_in.weight"].shape == (1600, 256) and sdxl["input_blocks.4.1.proj_in.weight"].qtype == Q.Q6_K
    assert sdxl["input_blocks.1.0.in_layers.2.weight"].shape == (3600, 256)
    assert sdxl["input_blocks.1.0.in_layers.2.weight"].qtype == Q.Q6_K
    assert sdxl["time_embed.0.weight"].qtype == Q.F16 and sdxl["output_blocks.0.0.x.weight"].qtype == Q.F16


def test_legacy_plans_are_unchanged(conv):
    """The K mixtures share plan_tensors with the legacy types; a legacy plan still ignores the attention-value rule."""
    plans = conv.plan_tensors(KEYSETS["wan"], conv.ARCH_BY_NAME["wan"], Q.Q4_0)
    assert {p.key: p.qtype for p in plans}["blocks.2.self_attn.v.weight"] == Q.Q4_0
    assert {p.key: p.qtype for p in plans}["blocks.0.ffn.2.weight"] == Q.Q4_1
    assert {p.key: p.qtype for p in plans}["blocks.0.self_attn.v.weight"] == Q.BF16


def test_convert_refuses_unknown_names_and_needs_cuda(conv, tmp_path, monkeypatch):
    sd = {"double_blocks.0.img_attn.proj.weight": torch.zeros(256, 256, dtype=torch.bfloat16), "img_in.weight": torch.zeros(4, 4)}
    with pytest.raises(ValueError, match="Q4_K_S"):
        conv.convert_state_dict(sd, str(tmp_path / "x.gguf"), "Q4_K_X")
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(NotImplementedError, match="Q4_K_S"):
        conv.convert_state_dict(sd, str(tmp_path / "y.gguf"), "q4_k_s")


def test_convert_writes_the_file_type_without_a_quantised_tensor(conv, tmp_path):
    """A file whose tensors all stay unquantised needs no GPU: general.file_type is the mixture's all the same."""
    sd = {"double_blocks.0.img_attn.proj.weight": torch.zeros(256, 48, dtype=torch.bfloat16), "img_in.weight": torch.ones(64, 32)}
    res = conv.convert_state_dict(sd, str(tmp_path / "z.gguf"), "Q3_K_M", conv.ARCH_BY_NAME["flux"])
    r = gguf.GGUFReader(res.path)
    ft = r.get_field("general.file_type")
    assert int(ft.parts[ft.data[-1]][0]) == gguf.LlamaFileType.MOSTLY_Q3_K_M
    assert [t.tensor_type for t in r.tensors] == [Q.F16, Q.F16]
    want = torch.zeros(256, 48, dtype=torch.bfloat16).half().numpy()
    assert np.array_equal(np.asarray(r.tensors[0].data).view(np.float16).reshape(256, 48), want)


# ---------------------------------------------------------------- ABI
def test_abi_constants_match_the_header(pkg):
    text = open(os.path.join(kc.ROOT, "include", "ggufb200.h")).read()
    assert int(re.search(r"#define GGUFB200_OP_QUANTIZE_K (\d+)", text).group(1)) == pkg.lib.OP_QUANTIZE_K == 9
    assert re.search(r"int ggufb200_quantize_k\(int ggml_type, const void \*src, int src_dtype, int64_t n_blocks, void \*packed, "
                     r"int flags, void \*stream\);", text)
    assert "ggufb200_quantize_k" in pkg.lib.EXPORTS and len(pkg.lib.lib().ggufb200_quantize_k.argtypes) == 7
    assert set(ge._sub("quantize").KQUANT_QTYPES) == set(kc.K_TYPES)
    L = pkg.lib.lib()
    for t in range(64):
        assert L.ggufb200_supported(t, pkg.lib.OP_QUANTIZE_K) == (t in {int(q) for q in kc.K_TYPES})
    assert L.ggufb200_quantize_k(int(Q.Q4_0), None, 2, 1, None, 0, None) == -1     # E_TYPE before anything else


def test_quantize_k_tensor_refuses_without_cuda():
    quantize = ge._sub("quantize")
    with pytest.raises(NotImplementedError):
        quantize.quantize_k_tensor(torch.zeros(4, 256), Q.Q4_K)
    with pytest.raises(NotImplementedError):
        quantize.quantize_k_tensor(torch.zeros(4, 256), Q.Q4_0)
