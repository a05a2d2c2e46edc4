"""GPU tests of the K-quant encoders (ggufb200_quantize_k / quantize.quantize_k_tensor) and the converter's K mixtures.

The kernel equals the plain-C restatement of llama.cpp's reference quantisers (tests/kquant_oracle.c) bit for bit for the five
K types and three source dtypes, on Flux-size tensors, the adversarial super-blocks of tests/kquant_cases.py, block counts off
the tile, offset views and back-to-back launches.  The converter's K files carry the planned types and the restated bytes, load
with gguf_sd_loader, and their packed Linears match F.linear on the dequantised weight within the packed Linear's budget."""
import gguf
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
import kquant_cases as kc
import quantize_cases as qc
from test_quantize_k import _reference_types
from util import rel_fro

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Q = gguf.GGMLQuantizationType
SRC_DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["f32", "f16", "bf16"]


@pytest.fixture(scope="module")
def qz():
    return ge._sub("quantize")


@pytest.fixture(scope="module")
def ok():
    L = kc.oracle_lib()
    if L is None:
        pytest.skip("gcc not available")
    return L


def _want(ok, x, qt):
    """The C restatement's bytes for the values of x (any float dtype), flat."""
    return kc.encode(ok, x.float().cpu().numpy(), qt)


def _got(qz, x, qt):
    return qz.quantize_k_tensor(x.to(DEV), qt).cpu().numpy()


@pytest.mark.parametrize("src", SRC_DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("qt", kc.K_TYPES, ids=lambda q: q.name)
def test_bit_exact_on_flux_shapes(qz, ok, qt, src):
    g = torch.Generator().manual_seed(int(qt) * 3 + SRC_DTYPES.index(src))
    x = (torch.randn(3072, 3072, generator=g) * 0.02).to(src)
    got = _got(qz, x, qt)
    assert got.shape == (3072, 3072 // 256 * gguf.GGML_QUANT_SIZES[qt][1])
    assert np.array_equal(got.reshape(-1), _want(ok, x, qt)), (qt.name, src)


@pytest.mark.parametrize("src", SRC_DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("qt", kc.K_TYPES, ids=lambda q: q.name)
def test_bit_exact_on_adversarial_and_heavy_tailed_blocks(qz, ok, qt, src):
    for x in (kc.adversarial_blocks(), kc.seeded_blocks(2000, seed=int(qt), heavy=True)):
        x = torch.from_numpy(x).to(src)
        x = x[torch.isfinite(x).all(1)]             # fp16 turns the largest rows into Inf: refused
        got = _got(qz, x, qt).reshape(len(x), -1)
        want = _want(ok, x, qt).reshape(len(x), -1)
        bad = np.flatnonzero((got != want).any(1))
        assert bad.size == 0, (qt.name, src, bad[:5])


@pytest.mark.parametrize("qt", kc.K_TYPES, ids=lambda q: q.name)
def test_block_counts_off_the_tile(qz, ok, qt):
    """8 (Q2_K, Q3_K, Q6_K) or 16 (Q4_K, Q5_K) super-blocks per CTA: partial tiles of every size class."""
    for n_blocks in (1, 7, 8, 9, 15, 16, 17, 255, 1001):
        x = torch.from_numpy(kc.seeded_blocks(n_blocks, seed=n_blocks)).reshape(1, -1)
        for src in SRC_DTYPES:
            xs = x.to(src)
            assert np.array_equal(_got(qz, xs, qt).reshape(-1), _want(ok, xs, qt)), (qt.name, n_blocks, src)


@pytest.mark.parametrize("qt", kc.K_TYPES, ids=lambda q: q.name)
def test_offset_views_and_back_to_back_launches(pkg, ok, qt):
    """The C entry point on source / output pointers at small offsets (no 16-byte alignment), several launches queued on one
    stream before a single synchronisation; nothing is written outside the output."""
    L = pkg.lib.lib()
    ts = gguf.GGML_QUANT_SIZES[qt][1]
    n_blocks = 77
    stream = torch.cuda.current_stream(DEV)
    jobs = []
    for k, src in enumerate(SRC_DTYPES):
        base = torch.from_numpy(kc.seeded_blocks(n_blocks + 1, seed=k)).reshape(-1).to(src).to(DEV)
        for off in (0, 1, 5):
            for ooff in (0, 7):
                view = base[off:off + n_blocks * 256]
                out = torch.full((n_blocks * ts + 16,), 0xA5, dtype=torch.uint8, device=DEV)
                rc = L.ggufb200_quantize_k(int(qt), view.data_ptr(), pkg.dequant.dtype_code(src), n_blocks, out.data_ptr() + ooff, 0,
                                           stream.cuda_stream)
                assert rc == 0
                jobs.append((view, out, ooff))
    torch.cuda.synchronize()
    for view, out, ooff in jobs:
        o = out.cpu().numpy()
        assert np.array_equal(o[ooff:ooff + n_blocks * ts], _want(ok, view, qt))
        assert (o[:ooff] == 0xA5).all() and (o[ooff + n_blocks * ts:] == 0xA5).all()


@pytest.mark.parametrize("qt", kc.K_TYPES, ids=lambda q: q.name)
def test_packed_bytes_are_complete_for_a_stable_source_consumer(pkg, qz, qt):
    """The encoder lets the next kernel launch only after its last store: a dequant launched right behind it with the
    stable-source promise sees every byte."""
    x = torch.randn(3072, 3072, device=DEV) * 0.02
    shape = torch.Size(x.shape)
    outs = []
    for _ in range(2):
        x.mul_(1.5)
        packed = qz.quantize_k_tensor(x, qt)
        w = pkg.ops.GGMLTensor(packed, tensor_type=qt, tensor_shape=shape)
        got = pkg.dequant.dequantize_tensor(w, dtype=torch.float16)
        torch.cuda.synchronize()
        want = pkg.dequant.dequantize_tensor(w, dtype=torch.float16)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), qt.name
        outs.append(packed)
    assert not torch.equal(outs[0], outs[1])


def test_abi_refusals(pkg):
    L = pkg.lib.lib()
    x = torch.zeros(512, device=DEV)
    out = torch.empty(512, dtype=torch.uint8, device=DEV)
    s = torch.cuda.current_stream(DEV).cuda_stream
    assert L.ggufb200_quantize_k(int(Q.Q4_0), x.data_ptr(), 2, 1, out.data_ptr(), 0, s) == -1       # E_TYPE
    assert L.ggufb200_quantize_k(int(Q.BF16), x.data_ptr(), 2, 1, out.data_ptr(), 0, s) == -1
    assert L.ggufb200_quantize_k(int(Q.Q4_K), x.data_ptr(), 3, 1, out.data_ptr(), 0, s) == -2       # E_DTYPE
    assert L.ggufb200_quantize_k(int(Q.Q4_K), None, 2, 1, out.data_ptr(), 0, s) == -5               # E_NULL
    assert L.ggufb200_quantize_k(int(Q.Q4_K), x.data_ptr(), 2, 1, out.data_ptr(), 0x100, s) == -8   # E_UNSUPPORTED
    assert L.ggufb200_quantize_k(int(Q.Q4_K), x.data_ptr(), 2, -1, out.data_ptr(), 0, s) == -4      # E_SHAPE
    assert L.ggufb200_quantize_k(int(Q.Q4_K), x.data_ptr() + 2, 2, 1, out.data_ptr(), 0, s) == -3  # E_ALIGN
    assert L.ggufb200_quantize_k(int(Q.Q4_K), None, 2, 0, None, 0, s) == 0
    # the legacy entry point keeps refusing the K types
    assert L.ggufb200_quantize(int(Q.Q4_K), x.data_ptr(), 2, 2, out.data_ptr(), 0, s) == -1


def test_python_entry_point_refusals(qz, ok):
    with pytest.raises(ValueError, match="multiple of 256"):
        qz.quantize_k_tensor(torch.zeros(4, 320, device=DEV), Q.Q4_K)
    for bad in (float("inf"), float("nan")):
        x = torch.zeros(4, 256, device=DEV)
        x[2, 7] = bad
        for qt in kc.K_TYPES:
            with pytest.raises(ValueError, match="finite"):
                qz.quantize_k_tensor(x, qt)
    with pytest.raises(NotImplementedError):
        qz.quantize_k_tensor(torch.zeros(4, 256, device=DEV), Q.Q4_0)
    y = qz.quantize_k_tensor(torch.randn(5, 2, 512, device=DEV), Q.Q6_K)
    assert y.shape == (5, 2, 420) and y.dtype == torch.uint8 and y.device.type == "cuda"
    xt = torch.randn(512, 6, device=DEV).t()                          # a non-contiguous source is quantised row by row
    assert np.array_equal(qz.quantize_k_tensor(xt, Q.Q3_K).cpu().numpy().reshape(-1), _want(ok, xt, Q.Q3_K))


@pytest.mark.parametrize("qt", kc.K_TYPES, ids=lambda q: q.name)
def test_packed_linear_on_encoded_weights(pkg, qz, qt):
    """One GGMLOps.Linear per K type on weights this encoder wrote matches F.linear on the dequantised weight."""
    g = torch.Generator().manual_seed(int(qt))
    w = torch.randn(768, 1024, generator=g) * 0.02
    packed = qz.quantize_k_tensor(w.to(DEV), qt)
    wt = pkg.ops.GGMLTensor(packed, tensor_type=qt, tensor_shape=torch.Size(w.shape))
    ref_w = gguf.quants.dequantize(packed.cpu().numpy(), qt).reshape(768, 1024)
    lin = pkg.ops.GGMLOps.Linear(1024, 768)
    lin.load_state_dict({"weight": wt})
    for M, dt in ((3, torch.float16), (300, torch.bfloat16)):
        x = torch.randn(M, 1024, generator=g).to(dt)
        y = lin(x.to(DEV))
        want = (x.double() @ torch.from_numpy(ref_w).to(dt).double().t()).to(dt)
        bound = 1e-3 if dt == torch.float16 else 8e-3
        assert rel_fro(y.float().cpu().numpy(), want.float().numpy()) <= bound, (qt.name, M, dt)


# ---------------------------------------------------------------- converter, end to end
def _flux_checkpoint():
    g = torch.Generator().manual_seed(5)
    r = lambda *s: torch.randn(*s, generator=g) * 0.02
    return {
        "model.diffusion_model.img_in.weight": r(256, 64).bfloat16(),
        "model.diffusion_model.double_blocks.0.img_attn.proj.weight": r(256, 256).bfloat16(),
        "model.diffusion_model.double_blocks.0.img_attn.proj.bias": r(256).bfloat16(),
        "model.diffusion_model.double_blocks.0.img_attn.qkv.weight": r(768, 256).bfloat16(),
        "model.diffusion_model.double_blocks.0.img_mlp.0.weight": r(1024, 256).bfloat16(),
        "model.diffusion_model.double_blocks.0.img_mlp.2.weight": r(256, 1024).bfloat16(),
        "model.diffusion_model.single_blocks.0.linear2.weight": r(256, 512),              # fp32 -> F16 stage 1
        "model.diffusion_model.double_blocks.0.odd.weight": r(256, 96).bfloat16(),          # rows not a multiple of 256: F16
        "model.diffusion_model.final_layer.linear.weight": r(64, 256).bfloat16(),
    }


def _sdxl_checkpoint():
    g = torch.Generator().manual_seed(6)
    r = lambda *s: (torch.randn(*s, generator=g) * 0.02).half()
    sd = {f"model.diffusion_model.{k}": r(64, 4, 1, 1) for k in qc.ARCH_KEYS["sdxl"]}
    sd.update({
        "model.diffusion_model.input_blocks.0.0.weight": r(320, 4, 3, 3),
        "model.diffusion_model.input_blocks.4.1.proj_in.weight": r(640, 640),                            # reshaped: straddled rows
        "model.diffusion_model.input_blocks.4.1.transformer_blocks.0.attn1.to_v.weight": r(512, 512),
        "model.diffusion_model.input_blocks.4.1.transformer_blocks.0.attn2.to_v.weight": r(512, 768),
        "model.diffusion_model.input_blocks.4.1.transformer_blocks.0.ff.net.2.weight": r(512, 1024),
        "model.diffusion_model.input_blocks.4.1.transformer_blocks.0.attn1.to_q.weight": r(512, 512),
        "model.diffusion_model.time_embed.0.weight": (torch.randn(1280, 320, generator=g) * 0.02),
    })
    return sd


@pytest.mark.parametrize("mix", ["Q4_K_S", "Q3_K_M", "Q6_K"])
@pytest.mark.parametrize("which", ["flux", "sdxl"])
def test_convert_end_to_end(pkg, ok, tmp_path, which, mix):
    from safetensors.torch import save_file
    conv = ge._sub("convert")
    ckpt = _flux_checkpoint() if which == "flux" else _sdxl_checkpoint()
    src = str(tmp_path / f"{which}.safetensors")
    save_file(ckpt, src)
    res = conv.convert_file(src, str(tmp_path / f"{which}-{{ftype}}.gguf"), qtype=mix)
    assert res.path.endswith(f"{which}-{mix}.gguf")
    arch = conv.ARCH_BY_NAME[which]
    reader = gguf.GGUFReader(res.path)
    ftype = reader.get_field("general.file_type")
    assert int(ftype.parts[ftype.data[-1]][0]) == getattr(gguf.LlamaFileType, f"MOSTLY_{mix}")
    sd_src = conv.load_state_dict(src)
    want_types = _reference_types(sd_src, arch, mix)
    plans = {p.key: p for p in res.plans}
    quantised = []
    for t in reader.tensors:
        assert t.tensor_type == want_types[t.name], t.name
        p = plans[t.name]
        data = np.asarray(t.data).view(np.uint8).reshape(-1)
        if p.qtype in conv.KQUANT_TYPES:
            vals = sd_src[t.name].reshape(p.shape)
            vals = vals if p.stage1 == Q.BF16 else vals.to(torch.float16)
            assert np.array_equal(data, _want(ok, vals, p.qtype)), t.name
            quantised.append(t.name)
        elif p.qtype == Q.F16 and p.stage1 == Q.BF16:
            assert np.array_equal(data.view(np.float16), sd_src[t.name].to(torch.float16).reshape(-1).numpy()), t.name
    assert len(quantised) >= 3

    sd = pkg.loader.gguf_sd_loader(res.path)
    assert list(sd) == list(sd_src)
    g = torch.Generator().manual_seed(1)
    for key in quantised:
        w = sd[key]
        if sd_src[key].dim() != 2:
            continue
        N, K = sd_src[key].shape
        assert tuple(w.tensor_shape) == (N, K)
        lin = pkg.ops.GGMLOps.Linear(K, N)
        lin.load_state_dict({"weight": w.to(DEV)})
        ref_w = gguf.quants.dequantize(np.asarray(reader.get_tensor(list(sd_src).index(key)).data), w.tensor_type).reshape(N, K)
        for M, dt in ((3, torch.float16), (300, torch.bfloat16)):
            x = torch.randn(M, K, generator=g).to(dt)
            y = lin(x.to(DEV))
            want = (x.double() @ torch.from_numpy(ref_w).to(dt).double().t()).to(dt)
            bound = 1e-3 if dt == torch.float16 else 8e-3
            assert rel_fro(y.float().cpu().numpy(), want.float().numpy()) <= bound, (key, M, dt)
