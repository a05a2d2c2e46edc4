"""CPU tests of the GGUF-input converter (convert.convert_gguf_file, llama-quantize's step):
  * plan_gguf on a stage-1 file equals plan_tensors on the checkpoint it came from, for every architecture and target;
  * the source's fields keep their order, types and values; general.file_type and general.quantization_version are set;
  * tensors whose type stays are copied byte for byte (F32, F16, BF16 keep-listed tensors and packed tensors alike);
  * the requantisation refusal, the missing-5-D refusal and the --fix-5d placement on the reference's wan stage-1 fixture;
  * a stable-diffusion.cpp file (no architecture field) is planned for the architecture its names show and gains no field;
  * NotImplementedError without a CUDA device only where a tensor needs the GPU; tools/convert.py's GGUF options."""
import os

import gguf
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
import convert_gguf_cases as cc
import quantize_cases as qc

Q = gguf.GGMLQuantizationType
TARGETS = ["F16", "BF16", "Q8_0", "Q5_1", "Q5_0", "Q4_1", "Q4_0",
           "Q2_K", "Q3_K_S", "Q3_K_M", "Q3_K_L", "Q4_K_S", "Q4_K_M", "Q5_K_S", "Q5_K_M", "Q6_K"]


@pytest.fixture(scope="module")
def conv():
    return ge._sub("convert")


@pytest.fixture
def no_cuda(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)


def _tensors(path):
    r = gguf.GGUFReader(path)
    return {t.name: (t.tensor_type, tuple(int(d) for d in t.shape), np.asarray(t.data).view(np.uint8).reshape(-1).copy())
            for t in r.tensors}


def _fields(path):
    r = gguf.GGUFReader(path)
    return [(k, list(f.types), f.contents()) for k, f in r.fields.items() if not k.startswith("GGUF.")]


def _field(path, key):
    f = gguf.GGUFReader(path).get_field(key)
    return None if f is None else f.contents()


def _add(w, name, data, shape, qtype):
    """Add a tensor of `shape` (torch order) and type `qtype` whose bytes are `data`."""
    w.add_tensor(name, np.ascontiguousarray(data).view(np.uint8).reshape(gguf.quant_shape_to_byte_shape(shape, qtype)),
                 raw_dtype=qtype)


def _add_torch(w, name, t):
    if t.dtype == torch.bfloat16:
        _add(w, name, t.view(torch.int16).numpy(), tuple(t.shape), Q.BF16)
    else:
        w.add_tensor(name, t.numpy())


def _arch_state_dict(name):
    """ARCH_KEYS' names of `name` as bf16 matrices, plus the tensor kinds the rules tell apart."""
    g = torch.Generator().manual_seed(len(name))
    r = lambda *s, dt=torch.bfloat16: (torch.randn(*s, generator=g) * 0.02).to(dt)
    sd = {k: r(64, 256) for k in qc.ARCH_KEYS[name]}
    sd.update({
        "extra.0.attn.qkv.weight": r(96, 256),
        "extra.0.self_attn.v.weight": r(64, 256),
        "extra.0.to_v.weight": r(64, 512),
        "extra.0.ffn.2.weight": r(64, 512),
        "extra.0.f16.weight": r(64, 256, dt=torch.float16),
        "extra.0.f32.weight": r(64, 256, dt=torch.float32),
        "extra.0.small.weight": r(16, 16, dt=torch.float32),
        "extra.0.odd.weight": r(64, 96),
        "extra.0.odd2.weight": r(32, 48),
        "extra.0.conv.weight": r(32, 32, 3, 3, dt=torch.float16),
        "extra.0.norm.bias": r(64),
        "extra.0.nd.weight": r(4, 4, 1, 2, 2),
    })
    return sd


# ---------------------------------------------------------------- planning
@pytest.mark.parametrize("name", [a.name for a in ge._sub("convert").ARCHES])
def test_plans_from_a_stage1_file_equal_the_checkpoint_plans(conv, tmp_path, name):
    arch = conv.ARCH_BY_NAME[name]
    sd = _arch_state_dict(name)
    path = conv.convert_state_dict(sd, str(tmp_path / "stage1.gguf"), None, arch).path
    src = conv.open_gguf_source(path)
    assert src.arch is arch and src.arch_field == name
    for target in TARGETS:
        qtype = conv._parse_qtype(target)
        assert conv.plan_gguf(src, qtype) == conv.plan_tensors(sd, arch, qtype), (name, target)


def test_packed_sources_are_ruled_on_as_f16(conv):
    """A packed source tensor gets the type its F16 original would get, and keeps its own where the rules leave it alone."""
    arch = conv.ARCH_BY_NAME["flux"]
    sd = cc.checkpoint("flux", torch.bfloat16)
    plans = {p.key: p for p in conv.plan_tensors(sd, arch, None)}

    class T:                                       # a reader tensor of the packed source file
        def __init__(self, key):
            self.name, p = key, plans[key]
            self.tensor_type = Q.Q8_0 if conv.quantisable(key, p.stage1, p.shape, arch) else p.stage1
            self.shape = np.array(list(reversed(p.shape)), np.uint64)

    class R:
        tensors = [T(k) for k in plans]
        fields = {}
    src = conv.GGUFSource("x.gguf", R, arch, "flux", [k for k in plans])
    for target in TARGETS:
        qtype = conv._parse_qtype(target)
        direct = {p.key: p.qtype for p in conv.plan_tensors(sd, arch, qtype)}
        for p in conv.plan_gguf(src, qtype):
            if p.stage1 == Q.Q8_0:
                want = direct[p.key] if direct[p.key] != plans[p.key].stage1 else Q.F16
                if target == "BF16" and plans[p.key].stage1 == Q.BF16:
                    want = Q.BF16
                assert p.qtype == want, (target, p.key)
            else:
                assert p.qtype == direct[p.key], (target, p.key)


# ---------------------------------------------------------------- fields and bytes
def test_fields_keep_their_order_and_values(conv, tmp_path):
    path = str(tmp_path / "src.gguf")
    w = gguf.GGUFWriter(path, "flux")
    w.add_string("general.name", "tiny flux")
    w.add_uint32(gguf.Keys.General.FILE_TYPE, int(gguf.LlamaFileType.MOSTLY_BF16))
    w.add_uint8("test.u8", 7)
    w.add_float32("test.f32", 0.25)
    w.add_bool("test.flag", True)
    w.add_array("test.ints", [3, 1, 2])
    w.add_array("test.names", ["a", "bc"])
    w.add_array("comfy.gguf.orig_shape.double_blocks.0.img_attn.proj.weight", [64, 256])
    sd = cc.checkpoint("flux", torch.bfloat16)
    for k, t in sd.items():
        _add_torch(w, k, t if t.dtype == torch.bfloat16 else t.float())
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    out = conv.convert_gguf_file(path, str(tmp_path / "out-{ftype}.gguf"), "F16").path
    assert out.endswith("out-F16.gguf")
    src, got = _fields(path), _fields(out)
    # quantization_version was absent: appended; file_type set in place
    assert [k for k, _, _ in got] == [k for k, _, _ in src] + [gguf.Keys.General.QUANTIZATION_VERSION]
    for (k, types, val), (k2, types2, val2) in zip(src, got):
        assert types == types2, k
        assert val2 == (int(gguf.LlamaFileType.MOSTLY_F16) if k == gguf.Keys.General.FILE_TYPE else val), k
    assert got[-1][1:] == ([gguf.GGUFValueType.UINT32], gguf.GGML_QUANT_VERSION)


@pytest.mark.parametrize("arch", sorted(cc.FIXTURES))
def test_unchanged_tensors_are_copied_byte_for_byte(conv, tmp_path, no_cuda, arch):
    """F16 from the reference's stage 1: BF16 -> F16 is a host cast; every F32, F16 and keep-listed tensor is the source's bytes."""
    src = cc.fixture_path(arch)
    res = conv.convert_gguf_file(src, str(tmp_path / "out.gguf"), "F16", fix_5d=cc.FIX_5D if arch == "wan" else None)
    before, after = _tensors(src), _tensors(res.path)
    kept = [p for p in res.plans if p.qtype == p.stage1 and p.key in before]
    assert {before[p.key][0] for p in kept} >= {Q.F32, Q.F16} - ({Q.F16} if cc.FIXTURES[arch] == torch.bfloat16 else set())
    for p in kept:
        assert after[p.key][0] == before[p.key][0] and np.array_equal(after[p.key][2], before[p.key][2]), p.key
    cast = [p for p in res.plans if p.qtype != p.stage1]
    for p in cast:
        assert (p.stage1, p.qtype) == (Q.BF16, Q.F16)
        want = torch.from_numpy(before[p.key][2].copy()).view(torch.bfloat16).half().view(torch.uint8).numpy()
        assert np.array_equal(after[p.key][2], want), p.key
    assert len(cast) >= (3 if cc.FIXTURES[arch] == torch.bfloat16 else 0)
    assert _field(res.path, gguf.Keys.General.FILE_TYPE) == int(gguf.LlamaFileType.MOSTLY_F16)


def _q8_0_file(conv, tmp_path, name="q8.gguf"):
    """The flux checkpoint's stage 1 with every tensor Q8_0 quantises as Q8_0 (gguf-py's bytes), the rest as stage 1 wrote them."""
    sd = cc.checkpoint("flux", torch.bfloat16)
    stage1 = conv.convert_state_dict(sd, str(tmp_path / "s1.gguf"), None).path
    q8 = {p.key: p.qtype for p in conv.plan_tensors(sd, conv.ARCH_BY_NAME["flux"], Q.Q8_0)}
    r = gguf.GGUFReader(stage1)
    path = str(tmp_path / name)
    w = gguf.GGUFWriter(path, "flux")
    w.add_quantization_version(gguf.GGML_QUANT_VERSION)
    w.add_file_type(gguf.LlamaFileType.MOSTLY_Q8_0)
    for t in r.tensors:
        shape = tuple(int(d) for d in reversed(t.shape.tolist()))
        if q8[t.name] == Q.Q8_0:
            vals = sd[t.name].float().numpy()
            _add(w, t.name, gguf.quants.quantize(vals, Q.Q8_0), shape, Q.Q8_0)
        else:
            _add(w, t.name, np.asarray(t.data), shape, t.tensor_type)
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    return path


def test_requantisation_is_refused_by_default(conv, tmp_path):
    path = _q8_0_file(conv, tmp_path)
    with pytest.raises(ValueError, match=r"requantizing from type Q8_0 is disabled .*--allow-requantize"):
        conv.convert_gguf_file(path, str(tmp_path / "a.gguf"), "Q4_K_S")
    with pytest.raises(ValueError, match=r"requantizing from type Q8_0 is disabled"):
        conv.convert_gguf_file(path, str(tmp_path / "b.gguf"), "Q4_0")
    assert not os.path.exists(tmp_path / "a.gguf") and not os.path.exists(tmp_path / "b.gguf")


def test_already_that_type_is_copied(conv, tmp_path, no_cuda):
    """Q8_0 -> Q8_0 quantises nothing: no GPU, every tensor's bytes and the fields as they were."""
    path = _q8_0_file(conv, tmp_path)
    res = conv.convert_gguf_file(path, str(tmp_path / "same.gguf"), "Q8_0")
    assert not any(conv.needs_gpu(p) for p in res.plans)
    assert open(res.path, "rb").read() == open(path, "rb").read()


def test_requantisation_needs_the_gpu(conv, tmp_path, no_cuda):
    path = _q8_0_file(conv, tmp_path)
    with pytest.raises(NotImplementedError, match="Q4_K_S runs on the GPU"):
        conv.convert_gguf_file(path, str(tmp_path / "c.gguf"), "Q4_K_S", allow_requantize=True)
    # F16 from Q8_0 is still a GPU decode
    with pytest.raises(NotImplementedError, match="F16 runs on the GPU"):
        conv.convert_gguf_file(path, str(tmp_path / "d.gguf"), "F16", allow_requantize=True)


def test_requant_types_are_the_gpu_decoders(conv, pkg):
    assert set(conv.REQUANT_TYPES) == (set(pkg.dequant.SUPPORTED_QTYPES) - {Q.BF16}) | set(pkg.dequant.FALLBACK_QTYPES)
    assert len(conv.REQUANT_TYPES) == 23


# ---------------------------------------------------------------- wan's 5-D tensor
def test_missing_5d_weight_is_refused(conv, tmp_path):
    with pytest.raises(ValueError, match=r"lacks 'patch_embedding.weight'.*fix_5d=PATH \(--fix-5d PATH\)"):
        conv.convert_gguf_file(cc.fixture_path("wan"), str(tmp_path / "w.gguf"), "Q4_K_S")
    assert conv.missing_nd_weights(conv.open_gguf_source(cc.fixture_path("flux"))) == []


def test_fix_5d_placement(conv, tmp_path, no_cuda):
    """The 5-D tensor goes in as F32 right after its `.bias`, as fix_5d_tensors.py places it; an unmatched one goes last."""
    from safetensors.torch import load_file, save_file
    side = load_file(cc.FIX_5D)
    assert list(side) == ["patch_embedding.weight"] and side["patch_embedding.weight"].dim() == 5
    names = [t.name for t in gguf.GGUFReader(cc.fixture_path("wan")).tensors]
    want = []
    for n in names:
        want.append(n)
        if n == "patch_embedding.bias":
            want.append("patch_embedding.weight")
    res = conv.convert_gguf_file(cc.fixture_path("wan"), str(tmp_path / "w.gguf"), "F16", fix_5d=cc.FIX_5D)
    r = gguf.GGUFReader(res.path)
    assert [t.name for t in r.tensors] == want
    t = r.tensors[want.index("patch_embedding.weight")]
    assert t.tensor_type == Q.F32 and tuple(int(d) for d in reversed(t.shape.tolist())) == tuple(side["patch_embedding.weight"].shape)
    assert np.array_equal(np.asarray(t.data).reshape(-1), side["patch_embedding.weight"].float().numpy().reshape(-1))
    # a side tensor without a matching .bias is appended
    extra = dict(side)
    extra["blocks.7.extra.weight"] = torch.ones(2, 2, 1, 1, 2)
    save_file(extra, str(tmp_path / "fix.safetensors"))
    res = conv.convert_gguf_file(cc.fixture_path("wan"), str(tmp_path / "w2.gguf"), "F16", fix_5d=str(tmp_path / "fix.safetensors"))
    assert [p.key for p in res.plans] == want + ["blocks.7.extra.weight"]
    # a side tensor the file already holds is refused
    save_file({"head.head.weight": torch.ones(2, 2, 1, 1, 2)}, str(tmp_path / "dup.safetensors"))
    with pytest.raises(ValueError, match="already holds head.head.weight"):
        conv.convert_gguf_file(cc.fixture_path("wan"), str(tmp_path / "w3.gguf"), "F16", fix_5d=str(tmp_path / "dup.safetensors"))


# ---------------------------------------------------------------- stable-diffusion.cpp files
def _sdcpp_file(path, sd):
    w = gguf.GGUFWriter(path, "flux")
    w.kv_data[0].pop(gguf.Keys.General.ARCHITECTURE)
    w.add_string("general.name", "sd.cpp flux")
    w.add_uint32("test.value", 11)
    for k, t in sd.items():
        _add_torch(w, k, t)
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    return path


def test_sdcpp_file_is_planned_for_its_architecture_and_gains_no_field(conv, pkg, tmp_path, no_cuda):
    ckpt = cc.checkpoint("flux", torch.bfloat16)
    sd = {"model.diffusion_model." + k: (t.half() if t.dtype == torch.float32 and t.dim() > 1 else t) for k, t in ckpt.items()}
    sd["first_stage_model.decoder.conv_out.weight"] = torch.zeros(64, 256, dtype=torch.bfloat16)   # outside the diffusion model
    path = _sdcpp_file(str(tmp_path / "flux-sdcpp.gguf"), sd)
    src = conv.open_gguf_source(path)
    assert src.arch.name == "flux" and src.arch_field is None
    assert src.rule_names[-1] is None and src.rule_names[0] == "img_in.weight"
    plans = {p.key: p for p in conv.plan_gguf(src, conv.KQUANT_MIXTURES["Q4_K_S"])}
    assert plans["model.diffusion_model.double_blocks.0.img_attn.qkv.weight"].qtype == Q.Q4_K
    assert plans["model.diffusion_model.img_in.weight"].qtype == Q.BF16                 # on flux's keep-list
    assert plans["model.diffusion_model.final_layer.linear.weight"].qtype == Q.BF16
    assert plans["first_stage_model.decoder.conv_out.weight"].qtype == Q.BF16          # copied as it is

    res = conv.convert_gguf_file(path, str(tmp_path / "out.gguf"), "F16")
    assert _fields(res.path) == _fields(path)                                         # no architecture, no new field
    assert [t.name for t in gguf.GGUFReader(res.path).tensors] == list(sd)
    types = {k: v[0] for k, v in _tensors(res.path).items()}
    assert types["model.diffusion_model.double_blocks.0.img_attn.qkv.weight"] == Q.F16
    assert types["first_stage_model.decoder.conv_out.weight"] == Q.BF16
    state, arch = pkg.loader.gguf_sd_loader(res.path, return_arch=True)
    assert arch == "flux" and list(state) == list(ckpt)


def test_unknown_architectures_are_refused(conv, tmp_path):
    path = str(tmp_path / "t5.gguf")
    w = gguf.GGUFWriter(path, "t5")
    w.add_tensor("enc.blk.0.attn_q.weight", np.zeros((64, 64), np.float16))
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    with pytest.raises(ValueError, match="unsupported architecture 't5'"):
        conv.convert_gguf_file(path, str(tmp_path / "o.gguf"), "Q8_0")


# ---------------------------------------------------------------- the GPU only where needed; the interface
def test_gpu_needed_only_where_a_tensor_is_quantised(conv, tmp_path, no_cuda):
    with pytest.raises(NotImplementedError, match="Q8_0 runs on the GPU and no CUDA device is visible"):
        conv.convert_gguf_file(cc.fixture_path("flux"), str(tmp_path / "a.gguf"), "Q8_0")
    assert not os.path.exists(tmp_path / "a.gguf")
    conv.convert_gguf_file(cc.fixture_path("flux"), str(tmp_path / "b.gguf"), "F16")
    # nothing quantisable: rows of 48 never take a Q type
    sd = {"double_blocks.0.img_attn.proj.weight": torch.zeros(64, 48, dtype=torch.bfloat16), "img_in.weight": torch.ones(64, 32)}
    s1 = conv.convert_state_dict(sd, str(tmp_path / "s1.gguf"), None, conv.ARCH_BY_NAME["flux"]).path
    res = conv.convert_gguf_file(s1, str(tmp_path / "c.gguf"), "Q4_0")
    assert [p.qtype for p in res.plans] == [Q.BF16, Q.F16]


def test_qtype_and_destination(conv, tmp_path):
    src = str(tmp_path / "model-BF16.gguf")
    with open(cc.fixture_path("flux"), "rb") as f, open(src, "wb") as g:
        g.write(f.read())
    with pytest.raises(ValueError, match="needs a qtype"):
        conv.convert_gguf_file(src)
    with pytest.raises(ValueError, match="unsupported qtype 'Q4_K_X'"):
        conv.convert_gguf_file(src, qtype="Q4_K_X")
    res = conv.convert_gguf_file(src, qtype="f16")
    assert res.path == str(tmp_path / "model-BF16-F16.gguf") and set(res.seconds) == {"read", "quantise", "write"}
    with pytest.raises(FileExistsError):
        conv.convert_gguf_file(src, qtype="F16")
    conv.convert_gguf_file(src, qtype="F16", overwrite=True)


def test_cli_dispatches_gguf_sources(tmp_path, capsys):
    import sys
    sys.path.insert(0, os.path.join(cc.HERE, "..", "tools"))
    import convert as cli
    out = str(tmp_path / "w-{ftype}.gguf")
    cli.main(["--src", cc.fixture_path("wan"), "--qtype", "F16", "--dst", out, "--fix-5d", cc.FIX_5D])
    assert "wrote " + str(tmp_path / "w-F16.gguf") in capsys.readouterr().out
    with pytest.raises(SystemExit):
        cli.main(["--src", cc.fixture_path("wan"), "--dst", out])                     # a GGUF input needs --qtype
    with pytest.raises(SystemExit):
        cli.main(["--src", cc.FIX_5D, "--qtype", "Q8_0", "--allow-requantize"])       # GGUF-only options
