"""GPU tests of the GGUF-input converter (convert.convert_gguf_file).

* Byte identity: checkpoint -> stage-1 GGUF (BF16 or F16 main dtype) -> X is the very file checkpoint -> X, for flux, sd3, sdxl
  (with `comfy.gguf.orig_shape`) and wan (5-D), every legacy type and all nine K mixtures.
* The reference's stage-1 fixtures (tests/golden/stage1_*.gguf, wan with its fix_5d side file) convert to the tensors (names,
  types, shapes, bytes) and fields of the direct conversion of the same seeded checkpoint.
* Requantisation from Q8_0, Q4_K, Q6_K, IQ4_XS and TQ2_0: legacy and BF16 / F16 targets equal gguf-py's quantiser (or cast) on
  gguf-py's dequantised values, K targets equal tests/kquant_oracle.c on those values; a requantised file loads through
  gguf_sd_loader and its packed Linears run."""
import os

import gguf
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
import convert_gguf_cases as cc
import fallback_cases as fc
import kquant_cases as kc
import oracle
from test_convert_gguf import TARGETS, _add, _fields, _tensors
from util import rel_fro

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Q = gguf.GGMLQuantizationType
DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16}


@pytest.fixture(scope="module")
def conv():
    return ge._sub("convert")


@pytest.fixture(scope="module")
def ok():
    L = kc.oracle_lib()
    if L is None:
        pytest.skip("gcc not available")
    return L


@pytest.fixture(scope="module")
def stage1(conv, tmp_path_factory):
    """(checkpoint path, stage-1 GGUF path) per (architecture, dtype name), written once."""
    from safetensors.torch import save_file
    tmp = tmp_path_factory.mktemp("stage1")
    cache = {}

    def get(arch, dt):
        if (arch, dt) not in cache:
            src = str(tmp / f"{arch}-{dt}.safetensors")
            save_file(cc.checkpoint(arch, DTYPES[dt]), src)
            cache[arch, dt] = src, conv.convert_file(src, str(tmp / f"{arch}-{dt}-stage1.gguf")).path
        return cache[arch, dt]
    return get


@pytest.mark.parametrize("target", TARGETS)
@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("arch", cc.ARCHES)
def test_stage1_then_target_is_the_direct_file(conv, stage1, tmp_path, arch, dt, target):
    src, s1 = stage1(arch, dt)
    assert gguf.GGUFReader(s1).get_field(gguf.Keys.General.FILE_TYPE).contents() in (
        gguf.LlamaFileType.MOSTLY_BF16, gguf.LlamaFileType.MOSTLY_F16)
    direct = conv.convert_file(src, str(tmp_path / "direct.gguf"), target)
    two = conv.convert_gguf_file(s1, str(tmp_path / "two.gguf"), target)
    assert two.plans == direct.plans
    assert open(two.path, "rb").read() == open(direct.path, "rb").read(), (arch, dt, target)
    if target not in ("F16", "BF16"):
        assert any(conv.needs_quantiser(p) for p in two.plans)
    if arch == "sdxl" and target != dt.upper():                # F16 from an F16 stage 1 (BF16 from BF16) changes nothing
        assert any(p.orig_shape is not None and p.qtype != p.stage1 for p in two.plans)
    if arch == "wan":
        assert any(len(p.shape) == 5 for p in two.plans)


@pytest.mark.parametrize("target", TARGETS)
@pytest.mark.parametrize("arch", sorted(cc.FIXTURES))
def test_reference_stage1_fixtures(conv, tmp_path, arch, target):
    from safetensors.torch import save_file
    src = str(tmp_path / f"{arch}.safetensors")
    save_file(cc.checkpoint(arch, cc.FIXTURES[arch]), src)
    direct = conv.convert_file(src, str(tmp_path / "direct.gguf"), target)
    got = conv.convert_gguf_file(cc.fixture_path(arch), str(tmp_path / "got.gguf"), target,
                                 fix_5d=cc.FIX_5D if arch == "wan" else None)
    a, b = _tensors(got.path), _tensors(direct.path)
    assert sorted(a) == sorted(b)
    for name in b:
        assert a[name][:2] == b[name][:2] and np.array_equal(a[name][2], b[name][2]), (arch, target, name)
    assert sorted(_fields(got.path), key=str) == sorted(_fields(direct.path), key=str)


# ---------------------------------------------------------------- requantisation
SOURCES = [Q.Q8_0, Q.Q4_K, Q.Q6_K, Q.IQ4_XS, Q.TQ2_0]
REQUANT_TARGETS = ["Q8_0", "Q5_1", "Q4_0", "BF16", "F16", "Q4_K_S", "Q3_K_M", "Q6_K"]


def _packed_file(conv, path, qt):
    """The flux checkpoint's stage 1 with each tensor the rules quantise, and whose rows fit `qt`'s blocks, replaced by seeded
    `qt` blocks of about the checkpoint's scale."""
    sd = cc.checkpoint("flux", torch.bfloat16)
    arch = conv.ARCH_BY_NAME["flux"]
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    w = gguf.GGUFWriter(path, "flux")
    w.add_quantization_version(gguf.GGML_QUANT_VERSION)
    w.add_file_type(gguf.LlamaFileType.MOSTLY_Q8_0)
    for i, p in enumerate(conv.plan_tensors(sd, arch, None)):
        n = int(np.prod(p.shape))
        if conv.quantisable(p.key, p.stage1, p.shape, arch) and p.shape[-1] % bs == 0:
            if qt in fc.FALLBACK:
                blocks = fc.random_blocks(qt, n // bs, seed=i, scale=1e-3)
            else:
                blocks = oracle.random_blocks(int(qt), n // bs, seed=i, scale=1e-3)
            _add(w, p.key, blocks, p.shape, qt)
        else:
            vals = conv._host_bytes(conv._stage1_values(sd[p.key], p.stage1), p.stage1)
            _add(w, p.key, vals, p.shape, p.stage1)
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    return path


def _requantised(ok, values, qt):
    """gguf-py's bytes (legacy types, BF16), the fp16 cast (F16) or the C restatement's bytes (K types) of fp32 values."""
    if qt == Q.F16:
        return values.astype(np.float16).view(np.uint8).reshape(-1)
    if qt in kc.K_TYPES:
        return kc.encode(ok, values, qt)
    return gguf.quants.quantize(np.ascontiguousarray(values), qt).reshape(-1)


@pytest.mark.parametrize("target", REQUANT_TARGETS)
@pytest.mark.parametrize("qt", SOURCES, ids=lambda q: q.name)
def test_requantisation(conv, ok, tmp_path, qt, target):
    path = _packed_file(conv, str(tmp_path / f"src-{qt.name}.gguf"), qt)
    src = _tensors(path)
    res = conv.convert_gguf_file(path, str(tmp_path / "out.gguf"), target, allow_requantize=True)
    out = _tensors(res.path)
    assert [p.key for p in res.plans] == list(src)
    n_packed = n_requant = 0
    for p in res.plans:
        n_packed += p.stage1 == qt
        assert out[p.key][0] == p.qtype
        if p.qtype == p.stage1:
            assert np.array_equal(out[p.key][2], src[p.key][2]), p.key
        elif p.stage1 == qt:
            values = gguf.quants.dequantize(src[p.key][2], qt).reshape(p.shape).astype(np.float32)
            assert np.array_equal(out[p.key][2], _requantised(ok, values, p.qtype)), (p.key, p.qtype.name)
            n_requant += 1
    assert n_packed >= 5
    already = conv._parse_qtype(target)
    already = already.default if isinstance(already, conv.KMixture) else already
    if already != qt:                           # otherwise llama-quantize's "already that type" rule copies most of them
        assert n_requant >= 3, n_requant


def test_requantised_file_loads_and_runs(conv, pkg, tmp_path):
    path = _packed_file(conv, str(tmp_path / "src-Q8_0.gguf"), Q.Q8_0)
    res = conv.convert_gguf_file(path, str(tmp_path / "out-{ftype}.gguf"), "Q4_K_S", allow_requantize=True)
    reader = gguf.GGUFReader(res.path)
    sd = pkg.loader.gguf_sd_loader(res.path)
    assert list(sd) == [p.key for p in res.plans]
    g = torch.Generator().manual_seed(3)
    ran = 0
    for i, p in enumerate(res.plans):
        if p.qtype not in conv.KQUANT_TYPES or len(p.shape) != 2:
            continue
        N, K = p.shape
        lin = pkg.ops.GGMLOps.Linear(K, N)
        lin.load_state_dict({"weight": sd[p.key].to(DEV)})
        ref_w = gguf.quants.dequantize(np.asarray(reader.tensors[i].data), p.qtype).reshape(N, K)
        for M, dt in ((3, torch.float16), (300, torch.bfloat16)):
            x = torch.randn(M, K, generator=g).to(dt)
            y = lin(x.to(DEV))
            want = (x.double() @ torch.from_numpy(ref_w).to(dt).double().t()).to(dt)
            assert rel_fro(y.float().cpu().numpy(), want.float().numpy()) <= (1e-3 if dt == torch.float16 else 8e-3), (p.key, M)
        ran += 1
    assert ran >= 3
    assert os.path.basename(res.path) == "out-Q4_K_S.gguf"
