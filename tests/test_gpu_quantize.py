"""GPU tests of the quantiser (ggufb200_quantize / quantize.quantize_tensor) and the converter (convert.py).

The quantiser is bit-exact against gguf-py's `gguf.quants.quantize` for its six types and three source dtypes, on Flux-size
tensors and on the adversarial blocks of tests/quantize_cases.py, for any block count, offset views and back-to-back launches.
The converter's file is restated tensor by tensor from gguf.quants.quantize, loads with gguf_sd_loader, and its quantised
Linears match F.linear on gguf-py's dequantised weight within the packed Linear's budget (1e-3 relative Frobenius for fp16
activations, 8e-3 = the same bound in bf16 ulps for bf16: the layer's weight is the reference's fp16-math dequant, not
gguf-py's fp32 one, so single-ulp differences of the rounded outputs are expected)."""
import gguf
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
import quantize_cases as qc
from util import rel_fro

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Q = gguf.GGMLQuantizationType
SRC_DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["f32", "f16", "bf16"]


@pytest.fixture(scope="module")
def qz():
    return ge._sub("quantize")


def _want(x, qt):
    """gguf-py's bytes for the values of x (any float dtype), as [n_rows, bytes]."""
    with np.errstate(all="ignore"):
        return qc.gguf_bytes(x.float().cpu().numpy(), qt)


def _got(qz, x, qt):
    return qz.quantize_tensor(x.to(DEV), qt).cpu().numpy()


@pytest.mark.parametrize("src", SRC_DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("qt", qc.QUANT_TYPES, ids=lambda q: q.name)
def test_bit_exact_on_flux_shapes(qz, qt, src):
    g = torch.Generator().manual_seed(int(qt) * 3 + SRC_DTYPES.index(src))
    shapes = [(3072, 3072)]
    if SRC_DTYPES.index(src) == int(qt) % 3:       # one 12288 x 3072 (Flux MLP) run per type, the source dtype rotating
        shapes.append((12288, 3072))
    for shape in shapes:
        x = (torch.randn(shape, generator=g) * 0.02).to(src)
        got = _got(qz, x, qt)
        assert got.shape == (shape[0], shape[1] // gguf.GGML_QUANT_SIZES[qt][0] * gguf.GGML_QUANT_SIZES[qt][1])
        assert np.array_equal(got, _want(x, qt)), (qt.name, src, shape)


@pytest.mark.parametrize("src", SRC_DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("qt", qc.QUANT_TYPES, ids=lambda q: q.name)
def test_bit_exact_on_adversarial_blocks(qz, qt, src):
    x = torch.from_numpy(qc.adversarial_blocks()).to(src)
    x = x[torch.isfinite(x).all(1)]                 # fp16 turns the largest rows into Inf: Q types refuse those
    assert np.array_equal(_got(qz, x, qt), _want(x, qt)), (qt.name, src)


def test_bf16_is_exact_for_non_finite_input(qz):
    bits = torch.from_numpy(np.random.default_rng(3).integers(0, 2 ** 32, 8192, dtype=np.uint32).view(np.int32))
    x = bits.view(torch.float32)
    x[:4] = torch.tensor([float("inf"), -float("inf"), float("nan"), -float("nan")])
    assert np.array_equal(_got(qz, x.reshape(256, 32), Q.BF16), _want(x.reshape(256, 32), Q.BF16))


@pytest.mark.parametrize("qt", qc.QUANT_TYPES, ids=lambda q: q.name)
def test_block_counts_off_the_tile(qz, qt):
    """256 blocks per CTA tile (BF16: 2048 elements per CTA): partial tiles of every size class."""
    for n_blocks in (1, 7, 255, 257, 511, 1000, 2049):
        x = torch.from_numpy(qc.seeded_blocks(n_blocks, seed=n_blocks)).reshape(1, -1)
        for src in SRC_DTYPES:
            xs = x.to(src)
            assert np.array_equal(_got(qz, xs, qt), _want(xs, qt)), (qt.name, n_blocks, src)


@pytest.mark.parametrize("qt", qc.QUANT_TYPES, ids=lambda q: q.name)
def test_offset_views_and_back_to_back_launches(pkg, qt):
    """The C entry point on source / output pointers at every small offset (no 16-byte alignment), several launches queued on
    one stream before a single synchronisation."""
    L = pkg.lib.lib()
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    n_blocks = 700 if bs == 32 else 700 * 32
    stream = torch.cuda.current_stream(DEV)
    jobs = []
    for k, src in enumerate(SRC_DTYPES):
        base = torch.from_numpy(qc.seeded_blocks(n_blocks * bs // 32 + 1, seed=k)).reshape(-1).to(src).to(DEV)
        for off in (0, 1, 3, 5):                    # off = 0: a 16-byte aligned source
            for ooff in (0, 7, 10):                 # every pairing of aligned / unaligned source and output
                view = base[off:off + n_blocks * bs]
                out = torch.full((n_blocks * ts + 16,), 0xA5, dtype=torch.uint8, device=DEV)
                rc = L.ggufb200_quantize(int(qt), view.data_ptr(), pkg.dequant.dtype_code(src), n_blocks, out.data_ptr() + ooff, 0,
                                         stream.cuda_stream)
                assert rc == 0
                jobs.append((view, out, ooff))
    torch.cuda.synchronize()
    for view, out, ooff in jobs:
        o = out.cpu().numpy()
        assert np.array_equal(o[ooff:ooff + n_blocks * ts], _want(view.reshape(-1, 32), qt).reshape(-1))
        assert (o[:ooff] == 0xA5).all() and (o[ooff + n_blocks * ts:] == 0xA5).all()     # nothing written outside


@pytest.mark.parametrize("qt", qc.QUANT_TYPES, ids=lambda q: q.name)
def test_packed_bytes_are_complete_for_a_stable_source_consumer(pkg, qz, qt):
    """The quantiser lets the next kernel launch only after its last store: a dequant launched right behind it on the same
    stream with the stable-source promise (which reads the packed bytes before waiting for its predecessor) sees every byte.
    A Flux linear1-size weight keeps the quantiser running long after the dependent grid could have started."""
    x = (torch.randn(21504, 3072, device=DEV) * 0.02)
    shape = torch.Size(x.shape)
    outs = []
    for _ in range(2):
        x.mul_(1.5)                                  # a new source each round: stale bytes of the previous round would show
        packed = qz.quantize_tensor(x, qt)           # no synchronisation between the two launches
        w = pkg.ops.GGMLTensor(packed, tensor_type=qt, tensor_shape=shape)
        got = pkg.dequant.dequantize_tensor(w, dtype=torch.float16)
        torch.cuda.synchronize()
        want = pkg.dequant.dequantize_tensor(w, dtype=torch.float16)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), qt.name
        outs.append(packed)
    assert not torch.equal(outs[0], outs[1])


def test_abi_refusals(pkg):
    L = pkg.lib.lib()
    x = torch.zeros(64, device=DEV)
    out = torch.empty(64, dtype=torch.uint8, device=DEV)
    s = torch.cuda.current_stream(DEV).cuda_stream
    assert L.ggufb200_quantize(int(Q.Q4_K), x.data_ptr(), 2, 2, out.data_ptr(), 0, s) == -1        # E_TYPE
    assert L.ggufb200_quantize(int(Q.Q4_0), x.data_ptr(), 3, 2, out.data_ptr(), 0, s) == -2        # E_DTYPE
    assert L.ggufb200_quantize(int(Q.Q4_0), None, 2, 2, out.data_ptr(), 0, s) == -5                # E_NULL
    assert L.ggufb200_quantize(int(Q.Q4_0), x.data_ptr(), 2, 2, out.data_ptr(), 0x100, s) == -8    # E_UNSUPPORTED
    assert L.ggufb200_quantize(int(Q.Q4_0), x.data_ptr(), 2, -1, out.data_ptr(), 0, s) == -4       # E_SHAPE
    assert L.ggufb200_quantize(int(Q.Q4_0), x.data_ptr() + 2, 2, 2, out.data_ptr(), 0, s) == -3   # E_ALIGN: fp32 at 2 bytes
    assert L.ggufb200_quantize(int(Q.Q4_0), None, 2, 0, None, 0, s) == 0
    for t in range(64):
        assert L.ggufb200_supported(t, pkg.lib.OP_QUANTIZE) == (t in {int(q) for q in qc.QUANT_TYPES})


def test_python_entry_point_refusals(qz):
    with pytest.raises(ValueError, match="multiple of 32"):
        qz.quantize_tensor(torch.zeros(4, 48, device=DEV), Q.Q8_0)
    xb = torch.randn(4, 47, device=DEV)                               # BF16 has 1-element blocks: any row length
    assert np.array_equal(qz.quantize_tensor(xb, Q.BF16).cpu().numpy(), _want(xb.cpu(), Q.BF16))
    for bad in (float("inf"), float("nan")):
        x = torch.zeros(4, 64, device=DEV)
        x[2, 7] = bad
        for qt in (Q.Q4_0, Q.Q4_1, Q.Q5_0, Q.Q5_1, Q.Q8_0):
            with pytest.raises(ValueError, match="finite"):
                qz.quantize_tensor(x, qt)
        qz.quantize_tensor(x, Q.BF16)
    with pytest.raises(NotImplementedError):
        qz.quantize_tensor(torch.zeros(4, 64, device=DEV), Q.Q4_K)
    y = qz.quantize_tensor(torch.randn(5, 2, 64, device=DEV), Q.Q8_0)
    assert y.shape == (5, 2, 68) and y.dtype == torch.uint8 and y.device.type == "cuda"
    xt = torch.randn(64, 6, device=DEV).t()                           # a non-contiguous source is quantised row by row
    assert np.array_equal(qz.quantize_tensor(xt, Q.Q4_0).cpu().numpy(), _want(xt.cpu(), Q.Q4_0))


@pytest.mark.parametrize("qt", qc.QUANT_TYPES, ids=lambda q: q.name)
def test_quantise_then_dequantise(pkg, qz, qt):
    """Our bytes through the package's dequant (fp32 math) equal gguf-py's dequantised value of gguf-py's bytes."""
    x = torch.randn(256, 1024, generator=torch.Generator().manual_seed(int(qt))) * 0.05
    packed = qz.quantize_tensor(x.to(DEV), qt)
    w = pkg.ops.GGMLTensor(packed, tensor_type=qt, tensor_shape=torch.Size(x.shape))
    got = pkg.dequant.dequantize_tensor(w, dtype=torch.float32, dequant_dtype=torch.float32).cpu().numpy()
    want = gguf.quants.dequantize(_want(x, qt), qt)
    assert np.array_equal(got.view(np.uint32), want.astype(np.float32).view(np.uint32))


# ---------------------------------------------------------------- converter, end to end
def _flux_checkpoint():
    g = torch.Generator().manual_seed(5)
    r = lambda *s: torch.randn(*s, generator=g) * 0.02
    return {
        "model.diffusion_model.img_in.weight": r(256, 64).bfloat16(),
        "model.diffusion_model.img_in.bias": r(256).bfloat16(),
        "model.diffusion_model.double_blocks.0.img_attn.proj.weight": r(256, 256).bfloat16(),
        "model.diffusion_model.double_blocks.0.img_attn.proj.bias": r(256).bfloat16(),
        "model.diffusion_model.double_blocks.0.img_attn.norm.query_norm.scale": r(128).bfloat16(),
        "model.diffusion_model.double_blocks.0.img_mlp.0.weight": r(1024, 256).bfloat16(),
        "model.diffusion_model.double_blocks.0.img_mlp.2.weight": r(256, 1024).bfloat16(),
        "model.diffusion_model.single_blocks.0.linear2.weight": r(256, 512),            # fp32 -> F16 stage 1
        "model.diffusion_model.single_blocks.0.modulation.lin.weight": r(768, 256).half(),
        "model.diffusion_model.guidance_in.in_layer.weight": r(256, 256),
        "model.diffusion_model.final_layer.linear.weight": r(64, 256).bfloat16(),
        "model.diffusion_model.double_blocks.0.odd.weight": r(256, 48).bfloat16(),        # rows not a multiple of 32
        "model.diffusion_model.double_blocks.0.odd32.weight": r(256, 48),                 # the same from fp32: F16, BF16 file: BF16
        "model.diffusion_model.double_blocks.0.row.weight": r(1, 3072).half(),            # 1-D to llama.cpp: never quantised
        "model.diffusion_model.double_blocks.0.rows3d.weight": r(1, 64, 512).half(),      # 2-D to llama.cpp: quantised
        "first_stage_model.decoder.conv_in.weight": r(16, 16),                            # dropped with the prefix
    }


def _sdxl_checkpoint():
    g = torch.Generator().manual_seed(6)
    r = lambda *s: (torch.randn(*s, generator=g) * 0.02).half()
    sd = {f"model.diffusion_model.{k}": r(64, 4, 1, 1) for k in qc.ARCH_KEYS["sdxl"]}
    sd.update({
        "model.diffusion_model.input_blocks.0.0.weight": r(320, 4, 3, 3),
        "model.diffusion_model.input_blocks.1.0.in_layers.2.weight": r(320, 320, 3, 3),
        "model.diffusion_model.input_blocks.4.1.proj_in.weight": r(640, 640),
        "model.diffusion_model.input_blocks.4.1.transformer_blocks.0.ff.net.2.weight": r(640, 2560),
        "model.diffusion_model.input_blocks.4.1.transformer_blocks.0.attn1.to_q.weight": r(640, 640),
        "model.diffusion_model.time_embed.0.weight": (torch.randn(1280, 320, generator=g) * 0.02),
        "model.diffusion_model.input_blocks.4.1.norm.weight": torch.ones(640),
    })
    return sd


def _restate(key, t, arch, qtype):
    """(type, stored shape, bytes) of one tensor, restated from the converter's rules with gguf.quants.quantize."""
    shape = tuple(t.shape)
    n = t.numel()
    f32src = t.dtype in (torch.float32, torch.bfloat16)
    stage1 = Q.BF16 if t.dtype == torch.bfloat16 else Q.F16
    if len(shape) > 4 or (f32src and (len(shape) == 1 or n <= 1024 or any(h in key for h in arch.hiprec))):
        stage1 = Q.F32
    if arch.shape_fix and len(shape) > 1 and n >= 512 and n % 256 == 0 and shape[-1] % 256 != 0:
        shape = (n // 256, 256)
    vals = t.float().numpy().reshape(shape)
    if stage1 == Q.F16:
        vals = vals.astype(np.float16).astype(np.float32)
    final = stage1
    ggml_dims = len(shape) - next((i for i, d in enumerate(shape) if d != 1), len(shape) - 1)
    if (qtype is not None and stage1 in (Q.F16, Q.BF16) and ggml_dims == 2 and key.endswith("weight") and "_norm.weight" not in key
            and not any(k in key for k in arch.keep) and key not in arch.keep_names
            and (shape[-1] % 32 == 0 or qtype in (Q.F16, Q.BF16))):
        final = {Q.Q4_0: Q.Q4_1, Q.Q5_0: Q.Q5_1}.get(qtype, qtype) if ".ff.net.2.weight" in key else qtype
    data = gguf.quants.quantize(vals, final)
    return final, shape, np.ascontiguousarray(data).view(np.uint8).reshape(-1)


@pytest.mark.parametrize("qtype", [None, Q.Q8_0, Q.Q5_1, Q.Q5_0, Q.Q4_1, Q.Q4_0, Q.BF16, Q.F16], ids=lambda q: q.name if q else "stage1")
@pytest.mark.parametrize("which", ["flux", "sdxl"])
def test_convert_end_to_end(pkg, tmp_path, which, qtype):
    from safetensors.torch import save_file
    conv = ge._sub("convert")
    ckpt = _flux_checkpoint() if which == "flux" else _sdxl_checkpoint()
    src = str(tmp_path / f"{which}.safetensors")
    save_file(ckpt, src)
    res = conv.convert_file(src, str(tmp_path / f"{which}-{{ftype}}.gguf"), qtype=qtype.name if qtype else None)
    arch = conv.ARCH_BY_NAME[which]
    assert res.arch is arch

    reader = gguf.GGUFReader(res.path)
    field = reader.get_field("general.architecture")
    assert str(field.parts[field.data[-1]], encoding="utf-8") == which
    ftype = reader.get_field("general.file_type")
    want_ftype = conv.FILE_TYPES[qtype] if qtype else (gguf.LlamaFileType.MOSTLY_BF16 if which == "flux" else gguf.LlamaFileType.MOSTLY_F16)
    assert int(ftype.parts[ftype.data[-1]][0]) == want_ftype
    sd_src = conv.load_state_dict(src)                  # input order: the order the checkpoint file lists its tensors in
    assert sd_src.keys() == conv.strip_prefix(ckpt).keys()
    assert [t.name for t in reader.tensors] == list(sd_src)
    quantised = []
    for t in reader.tensors:
        final, shape, data = _restate(t.name, sd_src[t.name], arch, qtype)
        assert t.tensor_type == final, t.name
        assert tuple(int(v) for v in reversed(t.shape)) == shape, t.name
        assert np.array_equal(np.asarray(t.data).view(np.uint8).reshape(-1), data), t.name
        if final not in (Q.F32, Q.F16, Q.BF16):
            quantised.append(t.name)
        orig = reader.get_field(f"comfy.gguf.orig_shape.{t.name}")
        assert (orig is not None) == (shape != tuple(sd_src[t.name].shape)), t.name
    if qtype not in (None, Q.F16, Q.BF16):
        assert len(quantised) >= 3

    sd = pkg.loader.gguf_sd_loader(res.path)
    assert list(sd) == list(sd_src)
    g = torch.Generator().manual_seed(1)
    for key in quantised:
        w = sd[key]
        N, K = sd_src[key].shape[:2]
        if sd_src[key].dim() != 2:
            continue
        assert tuple(w.tensor_shape) == (N, K)
        lin = pkg.ops.GGMLOps.Linear(K, N)
        lin.load_state_dict({"weight": w.to(DEV)})
        ref_w = gguf.quants.dequantize(np.asarray(reader.get_tensor(list(sd_src).index(key)).data), w.tensor_type).reshape(N, K)
        for M, dt in ((3, torch.float16), (300, torch.bfloat16)):
            x = (torch.randn(M, K, generator=g)).to(dt)
            y = lin(x.to(DEV))
            want = (x.double() @ torch.from_numpy(ref_w).to(dt).double().t()).to(dt)
            bound = 1e-3 if dt == torch.float16 else 8e-3          # the packed Linear's budget: 1e-3, the same in bf16 ulps
            assert rel_fro(y.float().cpu().numpy(), want.float().numpy()) <= bound, (key, M, dt)
