"""CPU tests of the GGUF quantiser and converter:
  * the quantiser's block functors (comfyui-gguf_b200/csrc/quantize.cuh, compiled for the host by tests/host_quantize.cu)
    against gguf-py's `gguf.quants.quantize`, bit for bit, on seeded and adversarial blocks;
  * convert.py's architecture table (detect_arch) and its stage-1 / stage-2 type policy;
  * the new C ABI constants;
  * the loader's compatibility mode for GGUFs without an architecture field or with the `pig` tag."""
import ctypes
import logging
import os
import re
import shutil
import subprocess

import gguf
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
import quantize_cases as qc

Q = gguf.GGMLQuantizationType
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "host_quantize.cu")
OUT = os.path.join(HERE, "_build", "libhostquantize.so")
CSRC = os.path.join(ROOT, "comfyui-gguf_b200", "csrc")


@pytest.fixture(scope="module")
def hostq():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    deps = [SRC] + [os.path.join(CSRC, f) for f in ("quantize.cuh", "blocks.cuh", "common.cuh")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        tmp = OUT + f".{os.getpid()}.tmp"
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-o", tmp, SRC], check=True)
        os.replace(tmp, OUT)
    L = ctypes.CDLL(OUT)
    L.hostq_quantize.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    return L


def _host_quantize(L, x, qtype):
    x = np.ascontiguousarray(x, dtype=np.float32)
    bs, ts = gguf.GGML_QUANT_SIZES[qtype]
    n = x.size // bs
    out = np.zeros(n * ts, dtype=np.uint8)
    assert L.hostq_quantize(int(qtype), x.ctypes.data, n, out.ctypes.data) == 0
    return out


@pytest.mark.parametrize("qt", qc.QUANT_TYPES, ids=lambda q: q.name)
def test_functors_equal_gguf_py_on_seeded_blocks(hostq, qt):
    x = qc.seeded_blocks(4096, seed=int(qt))
    assert np.array_equal(_host_quantize(hostq, x, qt), qc.gguf_bytes(x, qt).reshape(-1))


@pytest.mark.parametrize("qt", qc.QUANT_TYPES, ids=lambda q: q.name)
def test_functors_equal_gguf_py_on_adversarial_blocks(hostq, qt):
    x = qc.adversarial_blocks()
    got = _host_quantize(hostq, x, qt).reshape(len(x), -1)
    with np.errstate(all="ignore"):
        want = qc.gguf_bytes(x, qt).reshape(len(x), -1)
    bad = [i for i in range(len(x)) if not np.array_equal(got[i], want[i])]
    assert not bad, (qt.name, bad[:5], x[bad[0]], got[bad[0]], want[bad[0]])


def test_adversarial_blocks_reach_the_edge_cases():
    """The adversarial set does exercise what it claims: codes 16 / 32 before the clip, an fp16-overflowing scale, a
    negative-zero scale and an overflowing reciprocal."""
    x = qc.adversarial_blocks()
    assert np.isfinite(x).all()
    with np.errstate(all="ignore"):
        d = qc.gguf_bytes(x, Q.Q4_0).reshape(len(x), -1)[:, :2].copy().view(np.float16)[:, 0]
        raw4 = np.trunc(x * (1 / (x[np.arange(len(x)), np.abs(x).argmax(1)] / -8))[:, None] + np.float32(8.5))
        raw5 = np.trunc(x * (1 / (x[np.arange(len(x)), np.abs(x).argmax(1)] / -16))[:, None] + np.float32(16.5))
    assert (raw4 == 16).any() and (raw5 == 32).any()
    assert np.isinf(d).any()
    assert (np.signbit(d) & (d == 0)).any()
    with np.errstate(all="ignore"):
        assert np.isinf(np.float32(1) / (np.abs(x).max(1) / np.float32(127))).any()


def test_bf16_functor_is_exact_for_non_finite_input(hostq):
    bits = np.array([0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0xFFBFFFFF, 0x7FFFFFFF, 0x00000001, 0x80000000,
                     0x3F808000, 0x3F818000, 0x7F7FFFFF, 0x3F7FFFFF], dtype=np.uint32)
    x = np.concatenate([bits.view(np.float32), np.random.default_rng(0).integers(0, 2 ** 32, 4096, dtype=np.uint32).view(np.float32)])
    with np.errstate(all="ignore"):
        assert np.array_equal(_host_quantize(hostq, x, Q.BF16), qc.gguf_bytes(x, Q.BF16).reshape(-1))


# ---------------------------------------------------------------- ABI
def test_abi_constants_match_the_header(pkg):
    text = open(os.path.join(ROOT, "include", "ggufb200.h")).read()
    assert int(re.search(r"#define GGUFB200_OP_QUANTIZE (\d+)", text).group(1)) == pkg.lib.OP_QUANTIZE == 5
    assert re.search(r"int ggufb200_quantize\(int ggml_type, const void \*src, int src_dtype, int64_t n_blocks, void \*packed, "
                     r"int flags, void \*stream\);", text)
    assert "ggufb200_quantize" in pkg.lib.EXPORTS
    quantize = ge._sub("quantize")
    assert set(quantize.QUANTIZE_QTYPES) == set(qc.QUANT_TYPES)


def test_quantize_tensor_refuses_without_cuda():
    quantize = ge._sub("quantize")
    with pytest.raises(NotImplementedError):
        quantize.quantize_tensor(torch.zeros(4, 64), Q.Q8_0)
    with pytest.raises(NotImplementedError):
        quantize.quantize_tensor(torch.zeros(4, 64), Q.Q4_K)


# ---------------------------------------------------------------- convert.py: architecture table
@pytest.fixture(scope="module")
def conv():
    return ge._sub("convert")


def test_the_table_has_the_eleven_architectures(conv):
    assert [a.name for a in conv.ARCHES] == ["flux", "sd3", "aura", "hidream", "cosmos", "ltxv", "hyvid", "wan", "sdxl", "sd1", "lumina2"]
    assert set(qc.ARCH_KEYS) == set(conv.ARCH_BY_NAME)


@pytest.mark.parametrize("name", sorted(qc.ARCH_KEYS))
def test_detect_arch(conv, name):
    keys = qc.ARCH_KEYS[name] + ["some.other.weight", "bias"]
    assert conv.detect_arch(keys).name == name
    assert conv.detect_arch(set(keys)).name == name


def test_detect_arch_other_sdxl_and_sd1_key_sets(conv):
    assert conv.detect_arch(["down_blocks.0.downsamplers.0.conv.weight", "add_embedding.linear_1.weight"]).name == "sdxl"
    assert conv.detect_arch(["label_emb.0.0.weight"]).name == "sdxl"
    assert conv.detect_arch(["down_blocks.0.downsamplers.0.conv.weight"]).name == "sd1"


@pytest.mark.parametrize("keys", [
    ["transformer_blocks.0.attn.norm_added_k.weight"],                                   # diffusers Flux
    ["transformer_blocks.0.attn.add_q_proj.weight"],                                     # diffusers SD3
    ["joint_transformer_blocks.3.ff_context.out_projection.weight"],                     # diffusers AuraFlow
    ["double_blocks.0.img_attn.proj.weight", "transformer_blocks.0.attn.norm_added_k.weight"],
])
def test_detect_arch_refuses_diffusers_layouts(conv, keys):
    with pytest.raises(ValueError, match="not allowed for conversion"):
        conv.detect_arch(keys)


@pytest.mark.parametrize("keys", [[], ["a.weight", "b.bias"], ["blocks.0.mlp.layer1.weight"], qc.ARCH_KEYS["wan"][:2]])
def test_detect_arch_refuses_unknown_key_sets(conv, keys):
    with pytest.raises(ValueError, match="Unknown model architecture"):
        conv.detect_arch(keys)


def test_strip_prefix(conv):
    t = torch.zeros(1)
    assert list(conv.strip_prefix({"model.diffusion_model.a": t, "first_stage_model.b": t})) == ["a"]
    assert list(conv.strip_prefix({"model.a": t, "cond.b": t})) == ["a"]
    assert list(conv.strip_prefix({"net.a": t, "net.b": t})) == ["a", "b"]
    assert list(conv.strip_prefix({"net.a": t, "b": t})) == ["net.a", "b"]


# ---------------------------------------------------------------- convert.py: type policy
F32, F16, BF16 = Q.F32, Q.F16, Q.BF16
f32, f16, bf16 = torch.float32, torch.float16, torch.bfloat16

# (arch, key, source dtype, source shape) -> (stage-1 type, reshaped?, Q4_0 file type, Q8_0 file type, BF16 file type)
POLICY = [
    ("flux", "double_blocks.0.img_attn.proj.weight", bf16, (3072, 3072), BF16, False, Q.Q4_0, Q.Q8_0, BF16),
    ("flux", "double_blocks.0.img_attn.proj.weight", f32, (3072, 3072), F16, False, Q.Q4_0, Q.Q8_0, BF16),
    ("flux", "double_blocks.0.img_attn.proj.weight", f16, (3072, 3072), F16, False, Q.Q4_0, Q.Q8_0, BF16),
    ("flux", "double_blocks.0.img_attn.proj.bias", bf16, (3072,), F32, False, F32, F32, F32),
    ("flux", "double_blocks.0.img_attn.proj.bias", f16, (3072,), F16, False, F16, F16, F16),         # 1-D fp16: F16, never quantised
    ("flux", "double_blocks.0.img_attn.norm.key_norm.scale", bf16, (128,), F32, False, F32, F32, F32),
    ("flux", "small.weight", f32, (32, 32), F32, False, F32, F32, F32),                              # <= 1024 elements
    ("flux", "small.weight", f16, (32, 32), F16, False, Q.Q4_0, Q.Q8_0, BF16),
    ("flux", "img_in.weight", bf16, (3072, 64), BF16, False, BF16, BF16, BF16),                       # keep-list
    ("flux", "final_layer.linear.weight", bf16, (64, 3072), BF16, False, BF16, BF16, BF16),
    ("flux", "double_blocks.0.img_mlp.2.weight", bf16, (3072, 12288), BF16, False, Q.Q4_0, Q.Q8_0, BF16),
    ("flux", "double_blocks.0.img_attn.proj.weight", bf16, (3072, 48), BF16, False, BF16, BF16, BF16),  # rows not a multiple of 32
    ("flux", "double_blocks.0.img_attn.proj.weight", f16, (3072, 48), F16, False, F16, F16, BF16),    # BF16 takes any row
    ("flux", "double_blocks.0.x.weight", bf16, (8, 3072, 16), BF16, False, BF16, BF16, BF16),       # 3-D: not quantised
    ("flux", "double_blocks.0.x.weight", f16, (1, 3072), F16, False, F16, F16, F16),                 # 1-D to llama.cpp
    ("flux", "double_blocks.0.x.weight", bf16, (1, 64, 3072), BF16, False, Q.Q4_0, Q.Q8_0, BF16),   # 2-D to llama.cpp
    ("flux", "double_blocks.0.x.scale", bf16, (3072, 3072), BF16, False, BF16, BF16, BF16),         # not a `weight`
    ("flux", "double_blocks.0.attn_norm.weight", f16, (64, 64), F16, False, F16, F16, F16),         # `_norm.weight`
    ("wan", "blocks.0.ffn.2.weight", bf16, (5120, 13824), BF16, False, Q.Q4_1, Q.Q8_0, BF16),       # ffn_down upgrade
    ("wan", "blocks.0.ffn.0.weight", bf16, (13824, 5120), BF16, False, Q.Q4_0, Q.Q8_0, BF16),
    ("wan", "blocks.0.modulation", f32, (1, 6, 5120), F32, False, F32, F32, F32),                   # high precision
    ("wan", "head.head.weight", bf16, (64, 5120), BF16, False, BF16, BF16, BF16),
    ("wan", "patch_embedding.weight", bf16, (5120, 16, 1, 2, 2), F32, False, F32, F32, F32),        # 5-D -> F32
    ("sd3", "proj_out.weight", f16, (64, 1536), F16, False, F16, F16, F16),                          # exact-name keep
    ("sd3", "joint_blocks.0.x_block.mlp.fc2.weight", f16, (1536, 6144), F16, False, Q.Q4_0, Q.Q8_0, BF16),
    ("cosmos", "blocks.0.mlp.layer2.weight", bf16, (2048, 8192), BF16, False, Q.Q4_1, Q.Q8_0, BF16),
    ("hidream", "double_stream_blocks.0.block.ff_i.experts.0.w2.weight", bf16, (2560, 6912), BF16, False, Q.Q4_1, Q.Q8_0, BF16),
    ("hidream", "double_stream_blocks.0.block.ff_i.gate.weight", bf16, (4, 2560), F32, False, F32, F32, F32),
    ("lumina2", "layers.0.feed_forward.w2.weight", bf16, (2304, 6144), BF16, False, Q.Q4_1, Q.Q8_0, BF16),
    ("ltxv", "transformer_blocks.0.ff.net.2.weight", bf16, (2048, 8192), BF16, False, Q.Q4_1, Q.Q8_0, BF16),
    ("ltxv", "transformer_blocks.0.attn1.to_v.weight", bf16, (2048, 2048), BF16, False, Q.Q4_0, Q.Q8_0, BF16),
    ("sdxl", "input_blocks.1.0.in_layers.2.weight", f16, (320, 320, 3, 3), F16, True, Q.Q4_0, Q.Q8_0, BF16),
    ("sdxl", "input_blocks.4.1.proj_in.weight", f16, (640, 640), F16, True, Q.Q4_0, Q.Q8_0, BF16),  # 640 % 256 != 0
    ("sdxl", "output_blocks.0.0.skip_connection.weight", f16, (1280, 2560, 1, 1), F16, True, Q.Q4_0, Q.Q8_0, BF16),
    ("sdxl", "output_blocks.0.0.x.weight", f16, (3, 5, 7, 11), F16, False, F16, F16, F16),        # 4-D, n % 256 != 0: kept
    ("sdxl", "middle_block.1.proj_in.weight", f16, (1280, 1280), F16, False, Q.Q4_0, Q.Q8_0, BF16),
    ("sdxl", "input_blocks.0.0.weight", f16, (320, 4, 3, 3), F16, True, F16, F16, F16),             # exact-name keep
    ("sdxl", "time_embed.0.weight", f16, (1280, 320), F16, True, F16, F16, F16),
    ("sdxl", "label_emb.0.0.weight", f32, (1280, 2816), F16, False, F16, F16, F16),
    ("sd1", "input_blocks.1.1.norm.weight", f32, (320,), F32, False, F32, F32, F32),
    ("sd1", "out.0.weight", f16, (100, 3), F16, False, F16, F16, BF16),                             # < 512 elements: no reshape
]


@pytest.mark.parametrize("case", POLICY, ids=lambda c: f"{c[0]}:{c[1]}:{str(c[2])[6:]}:{'x'.join(map(str, c[3]))}")
def test_type_policy(conv, case):
    arch_name, key, dtype, shape, want1, want_reshape, want_q4, want_q8, want_bf16 = case
    arch = conv.ARCH_BY_NAME[arch_name]
    stage1, reshape = conv.stage1_type(key, dtype, shape, arch)
    assert (stage1, reshape) == (want1, want_reshape)
    n = int(np.prod(shape))
    stored = (n // 256, 256) if reshape else shape
    assert conv.stage2_type(key, stage1, stored, arch, None) == stage1
    assert conv.stage2_type(key, stage1, stored, arch, Q.Q4_0) == want_q4
    assert conv.stage2_type(key, stage1, stored, arch, Q.Q8_0) == want_q8
    assert conv.stage2_type(key, stage1, stored, arch, Q.BF16) == want_bf16
    q5 = conv.stage2_type(key, stage1, stored, arch, Q.Q5_0)
    assert q5 == {Q.Q4_0: Q.Q5_0, Q.Q4_1: Q.Q5_1}.get(want_q4, want_q4)
    # an F16 file converts every tensor the Q types quantise, and also those whose rows are not a multiple of 32
    rows_not_32 = len(stored) == 2 and stored[-1] % 32 != 0 and key.endswith("proj.weight") and arch_name == "flux"
    want_f16 = F16 if want_q8 == Q.Q8_0 or rows_not_32 else stage1
    assert conv.stage2_type(key, stage1, stored, arch, Q.F16) == want_f16


def test_ggml_n_dims(conv):
    assert [conv.ggml_n_dims(s) for s in ((7,), (1,), (1, 1), (1, 64), (64, 1), (1, 6, 64), (1, 1, 6, 64), (2, 1, 64), (320, 4, 3, 3))] == \
        [1, 1, 1, 1, 2, 2, 2, 3, 4]


def test_ffn_down_names(conv):
    for name in ("blk.0.ffn_down.weight", "layers.0.experts.3.w2.weight", "blocks.0.ffn.2.weight", "t.0.ff.net.2.weight",
                 "blocks.0.mlp.layer2.weight", "blocks.0.adaln_modulation_mlp.2.weight", "layers.0.feed_forward.w2.weight"):
        assert conv.is_ffn_down(name), name
    for name in ("blocks.0.ffn.0.weight", "w2.weight", "blocks.0.attn.qkv.weight", "blocks.0.ffn_down.v.weight"):
        assert not conv.is_ffn_down(name), name


def test_plan_keeps_input_order_and_drops_ignored_keys(conv):
    arch = conv.ARCH_BY_NAME["cosmos"]
    sd = {"b.weight": torch.zeros(64, 64, dtype=bf16), "a._extra_state": torch.zeros(4), "blocks.0.accum_x": torch.zeros(4),
          "a.weight": torch.zeros(64, 64, dtype=bf16)}
    plans = conv.plan_tensors(sd, arch, Q.Q8_0)
    assert [p.key for p in plans] == ["b.weight", "a.weight"]
    assert [p.qtype for p in plans] == [Q.Q8_0, Q.Q8_0]


# ---------------------------------------------------------------- loader compatibility mode
def _write(path, arch, tensors, orig_shapes=()):
    w = gguf.GGUFWriter(path, arch or "flux")
    if arch is None:
        w.kv_data[0].pop(gguf.Keys.General.ARCHITECTURE)
    for key, shape in orig_shapes:
        w.add_array(f"comfy.gguf.orig_shape.{key}", list(shape))
    for name, arr in tensors.items():
        w.add_tensor(name, arr)
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    return path


def _f16(*shape):
    return np.random.default_rng(sum(shape)).standard_normal(shape).astype(np.float16)


def test_loader_compat_mode_without_architecture(pkg, tmp_path, caplog):
    tensors = {"model.diffusion_model.double_blocks.0.img_attn.proj.weight": _f16(64, 64),
               "model.diffusion_model.img_in.weight": _f16(64, 32),
               "model.diffusion_model.img_in.bias": np.zeros(64, np.float32)}
    path = _write(str(tmp_path / "flux-sdcpp.gguf"), None, tensors)
    with caplog.at_level(logging.WARNING):
        sd, arch = pkg.loader.gguf_sd_loader(path, return_arch=True)
    assert arch == "flux"
    assert "compatibility mode 'sd.cpp' [arch:flux]" in caplog.text
    assert list(sd) == ["double_blocks.0.img_attn.proj.weight", "img_in.weight", "img_in.bias"]
    assert tuple(sd["img_in.weight"].shape) == (64, 32)
    assert np.array_equal(sd["img_in.weight"].as_subclass(torch.Tensor).numpy(), tensors["model.diffusion_model.img_in.weight"])


def test_loader_compat_mode_pig(pkg, tmp_path, caplog):
    tensors = {k: _f16(32, 32) for k in qc.ARCH_KEYS["wan"]}
    path = _write(str(tmp_path / "wan-pig.gguf"), "pig", tensors)
    with caplog.at_level(logging.WARNING):
        sd, arch = pkg.loader.gguf_sd_loader(path, return_arch=True)
    assert arch == "wan"
    assert "compatibility mode 'pig' [arch:wan]" in caplog.text
    assert sorted(sd) == sorted(qc.ARCH_KEYS["wan"])


def test_loader_compat_mode_sdxl_strips_projection_dims(pkg, tmp_path):
    tensors = {k: _f16(8, 4, 3, 3) for k in qc.ARCH_KEYS["sdxl"]}
    tensors["input_blocks.4.1.proj_in.weight"] = _f16(640, 640, 1, 1)
    tensors["input_blocks.4.1.proj_out.weight"] = _f16(640, 640, 1, 1)
    tensors["input_blocks.4.0.skip_connection.weight"] = _f16(640, 320, 1, 1)
    path = _write(str(tmp_path / "sdxl-sdcpp.gguf"), None, tensors)
    sd = pkg.loader.gguf_sd_loader(path)
    assert tuple(sd["input_blocks.4.1.proj_in.weight"].shape) == (640, 640)
    assert tuple(sd["input_blocks.4.1.proj_out.weight"].shape) == (640, 640)
    assert tuple(sd["input_blocks.4.0.skip_connection.weight"].shape) == (640, 320, 1, 1)
    # only sd.cpp files get the fix: the same tensors tagged `cow` keep their shape
    sd = pkg.loader.gguf_sd_loader(_write(str(tmp_path / "sdxl-cow.gguf"), "cow", tensors))
    assert tuple(sd["input_blocks.4.1.proj_in.weight"].shape) == (640, 640, 1, 1)


def test_loader_compat_mode_refuses_unrecognised_files(pkg, tmp_path):
    path = _write(str(tmp_path / "unknown.gguf"), None, {"a.weight": _f16(32, 32)})
    with pytest.raises(ValueError, match=r"This model is not currently supported - \(Unknown model architecture!\)"):
        pkg.loader.gguf_sd_loader(path)
    path = _write(str(tmp_path / "diffusers.gguf"), "pig", {"transformer_blocks.0.attn.norm_added_k.weight": _f16(32, 32)})
    with pytest.raises(ValueError, match="This model is not currently supported - .*not allowed for conversion"):
        pkg.loader.gguf_sd_loader(path)


def test_text_models_without_architecture_keep_their_refusal(pkg, tmp_path):
    path = _write(str(tmp_path / "te.gguf"), None, {k: _f16(32, 32) for k in qc.ARCH_KEYS["flux"]})
    with pytest.raises(ValueError, match="incompatible with llama.cpp"):
        pkg.loader.gguf_sd_loader(path, is_text_model=True)
