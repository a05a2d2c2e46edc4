"""GPU tests of the Embedding row gather (csrc/rows.cu), bit for bit.

* Every case of tests/rows_cases.py through ggufb200_dequant_rows / ggufb200_dequant_rows_fallback: the golden values of the
  unmodified reference where the golden stream is the table, else the C oracle (gguf-py for the fallback types) on the
  gathered rows' bytes; NaN payloads aside.  The output sits 16-byte aligned inside a larger buffer: filled with a NaN pattern
  the kernel cannot produce (so every element must be written) and with sentinel guard bytes before and after it (untouched).
* Large: a full-size Qwen3-4B Q4_K token table, a Q8_0 table of more than 2^31 bytes read at its tail rows, and 70 000 ids
  into an fp32 output of more than 2^31 bytes.
* The standalone dequant at math bf16 / out fp32 for all 13 types.
* GGMLOps.Embedding against the reference's semantics, restated here, for every out_dtype x dequant_dtype, id layout and an
  offloaded table; one row-gather call per forward; BF16 tables whose width is not a multiple of 8."""
import os

import gguf
import numpy as np
import pytest
import torch

import oracle
import rows_cases as rc
from fallback_cases import FALLBACK, gguf_values
from util import ALL_QTYPES, Q, TORCH_DT, torch_bits

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GUARD = 64          # sentinel bytes before and after every output
SENTINEL = 0x5A
_INT = {0: torch.int16, 1: torch.int16, 2: torch.int32}
_ESIZE = {0: 2, 1: 2, 2: 4}


@pytest.fixture(scope="module", autouse=True)
def peak_memory():
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    print(f"\ntest_gpu_rows: peak device memory allocated {torch.cuda.max_memory_allocated(DEV) / 2**30:.2f} GiB")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _device_table(table, offset=0):
    """The table's bytes at `offset` from the start of an allocation: (buffer, pointer)."""
    flat = torch.from_numpy(np.ascontiguousarray(table).reshape(-1))
    buf = torch.zeros(flat.numel() + offset + 16, dtype=torch.uint8, device=DEV)
    buf[offset:offset + flat.numel()].copy_(flat)
    return buf, buf.data_ptr() + offset


def _output(n, K, out):
    """(buffer, pointer, bytes): n * K elements of the out dtype filled with rc.FILL, at byte GUARD of a buffer whose GUARD bytes
    before and after hold SENTINEL."""
    nbytes = n * K * _ESIZE[out]
    buf = torch.full((GUARD + nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device=DEV)
    if nbytes:
        buf[GUARD:GUARD + nbytes].view(_INT[out]).fill_(rc.FILL[out])
    ptr = buf.data_ptr() + GUARD
    assert ptr % 16 == 0
    return buf, ptr, nbytes


def _gather(pkg, qt, tptr, V, K, ids, optr, out, math):
    L = pkg.lib.lib()
    if qt in FALLBACK:
        return L.ggufb200_dequant_rows_fallback(int(qt), tptr, V, K, ids.data_ptr(), ids.numel(), optr, out, _stream())
    return L.ggufb200_dequant_rows(int(qt), tptr, V, K, ids.data_ptr(), ids.numel(), optr, out, math, _stream())


def _guards_untouched(buf, nbytes):
    return bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[GUARD + nbytes:] == SENTINEL).all())


# ---------------------------------------------------------------- the C ABI, every case
@pytest.mark.parametrize("case", rc.CASES, ids=lambda c: c.id)
def test_gather_bit_exact(pkg, case):
    table = rc.table_bytes(case)
    ids = rc.make_ids(case.ids, case.V, case.seed)
    _tbuf, tptr = _device_table(table, case.offset)
    d_ids = torch.from_numpy(ids).to(DEV)
    obuf, optr, nbytes = _output(ids.size, case.K, case.out)
    assert _gather(pkg, case.qt, tptr, case.V, case.K, d_ids, optr, case.out, case.math) == 0
    host = obuf.cpu().numpy()
    assert _guards_untouched(obuf, nbytes), f"{case.id}: a guard byte was written"
    got = host[GUARD:GUARD + nbytes].view(rc.BITS[case.out]).reshape(ids.size, case.K)
    msg = rc.mismatch(got, rc.expected(case, table, ids), case.out)
    assert msg is None, f"{case.id}: {msg}"


# ---------------------------------------------------------------- large tables and outputs
def test_full_size_qwen3_4b_token_table(pkg):
    """[151936, 2560] Q4_K (219 MB): ids up to the last row, checked against the oracle on those rows."""
    qt, V, K = Q.Q4_K, 151936, 2560
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    raw = oracle.random_blocks(int(qt), V * K // bs, seed=40).reshape(V, K // bs * ts)
    table = torch.from_numpy(raw).to(DEV)
    ids = np.concatenate([[V - 1, 0, V - 2, V // 2, V - 1], np.random.default_rng(1).integers(0, V, 507)]).astype(np.int64)
    d_ids = torch.from_numpy(ids).to(DEV)
    for math, out in ((0, 2), (1, 1)):
        obuf, optr, nbytes = _output(ids.size, K, out)
        assert _gather(pkg, qt, table.data_ptr(), V, K, d_ids, optr, out, math) == 0
        got = obuf[GUARD:GUARD + nbytes].cpu().numpy().view(rc.BITS[out])
        want = oracle.dequant(raw[ids], int(qt), out, math)
        assert rc.mismatch(got, want.view(rc.BITS[out]), out) is None and _guards_untouched(obuf, nbytes)
        del obuf
    del table
    torch.cuda.empty_cache()


def test_table_beyond_2_gib_read_at_its_tail(pkg):
    """[600000, 4096] Q8_0: 2.61e9 packed bytes; the tail rows start past 2^31 bytes, so a 32-bit row offset would show."""
    qt, V, K = Q.Q8_0, 600000, 4096
    rb = K // 32 * 34
    assert (V - 1) * rb > 2**31
    g = torch.Generator(device=DEV).manual_seed(41)
    table = torch.randint(0, 256, (V, rb), dtype=torch.uint8, device=DEV, generator=g)
    ids = np.array([V - 1, V - 2, 2**31 // rb + 1, 2**31 // rb, 0, V - 1, 555555, -1, V], dtype=np.int64)
    d_ids = torch.from_numpy(ids).to(DEV)
    inside = (ids >= 0) & (ids < V)
    rows = table[torch.from_numpy(ids[inside]).to(DEV)].cpu().numpy()
    for math, out in ((0, 0), (2, 2)):
        obuf, optr, nbytes = _output(ids.size, K, out)
        assert _gather(pkg, qt, table.data_ptr(), V, K, d_ids, optr, out, math) == 0
        got = obuf[GUARD:GUARD + nbytes].cpu().numpy().view(rc.BITS[out]).reshape(ids.size, K)
        want = np.zeros((ids.size, K), dtype=rc.BITS[out])
        want[inside] = oracle.dequant(rows, int(qt), out, math).view(rc.BITS[out]).reshape(-1, K)
        assert rc.mismatch(got, want, out) is None and _guards_untouched(obuf, nbytes)
        del obuf
    del table
    torch.cuda.empty_cache()


def test_70000_ids_into_an_fp32_output_beyond_2_gib(pkg):
    """70 000 ids x 8192 fp32 = 2.29e9 output bytes over two grid-y slices; compared on the device, slice by slice."""
    qt, V, K = Q.Q5_0, 64, 8192
    raw = oracle.random_blocks(int(qt), V * K // 32, seed=42).reshape(V, -1)
    table = torch.from_numpy(raw).to(DEV)
    ids = rc.make_ids("many", V, seed=43)
    d_ids = torch.from_numpy(ids).to(DEV)
    obuf, optr, nbytes = _output(ids.size, K, 2)
    assert nbytes > 2**31
    assert _gather(pkg, qt, table.data_ptr(), V, K, d_ids, optr, 2, 1) == 0
    values = torch.from_numpy(oracle.dequant(raw, int(qt), 2, 1).reshape(V, K).view(np.int32)).to(DEV)
    got = obuf[GUARD:GUARD + nbytes].view(torch.int32).view(ids.size, K)
    inside = (d_ids >= 0) & (d_ids < V)
    for s in range(0, ids.size, 8192):
        want = torch.where(inside[s:s + 8192, None], values[d_ids[s:s + 8192].clamp(0, V - 1)], 0)
        assert torch.equal(got[s:s + 8192], want), f"ids {s} .. {s + 8192}"
    assert _guards_untouched(obuf, nbytes)
    del obuf, got
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- the standalone dequant at math bf16, out fp32
@pytest.mark.parametrize("qt", ALL_QTYPES, ids=lambda q: q.name)
def test_dequant_bf16_math_into_fp32(pkg, qt):
    """Pair (1, 2): equal to the oracle, and to the exact widening of the (1, 1) output (which needs no oracle)."""
    bs = gguf.GGML_QUANT_SIZES[qt][0]
    K = {1: 4104, 32: 2080, 256: 2304}[bs]
    case = rc.RowsCase(qt, 37, K, "edges", 2, 1, specials=True)
    raw = rc.table_bytes(case)
    packed = torch.from_numpy(raw.reshape(-1)).to(DEV)
    n = 37 * K
    f32 = pkg.dequant.dequantize(packed, qt, (n,), dtype=torch.bfloat16, out_dtype=torch.float32)
    b16 = pkg.dequant.dequantize(packed, qt, (n,), dtype=torch.bfloat16, out_dtype=torch.bfloat16)
    assert f32.dtype == torch.float32
    got = torch_bits(f32)
    want = oracle.dequant(raw, int(qt), 2, 1).view(np.uint32)
    assert np.array_equal(rc.canon(got, 2), rc.canon(want, 2)), qt.name
    widened = torch_bits(b16).astype(np.uint32) << 16
    assert np.array_equal(rc.canon(got, 2), rc.canon(widened, 2)), qt.name
    assert not np.isfinite(got.view(np.float32)).all(), "the special blocks reach the output"


# ---------------------------------------------------------------- the layer
def _spy(pkg, monkeypatch):
    names = {"ggufb200_dequant_rows", "ggufb200_dequant_rows_fallback", "ggufb200_dequant", "ggufb200_dequant_fallback"}
    calls = []
    real = pkg.lib.lib()

    class Spy:
        def __getattr__(self, name):
            fn = getattr(real, name)
            if name in names:
                def wrapped(*a):
                    calls.append(name)
                    return fn(*a)
                return wrapped
            return fn
    monkeypatch.setattr(pkg.lib, "lib", lambda: Spy())
    return calls


def _raw_table(qt, V, K, seed):
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    if qt in FALLBACK:
        from fallback_cases import random_blocks
        return random_blocks(qt, V * K // bs, seed=seed, scale=0.01).reshape(V, -1)
    return oracle.random_blocks(int(qt), V * K // bs, seed=seed).reshape(V, -1)


def _embedding(pkg, qt, raw, V, K, device=DEV, dequant_dtype=None):
    emb = pkg.ops.GGMLOps.Embedding(V, K, device="meta")
    w = pkg.ops.GGMLTensor(torch.from_numpy(np.ascontiguousarray(raw)).to(device), tensor_type=qt, tensor_shape=torch.Size((V, K)))
    emb.load_state_dict({"weight": w}, assign=True)
    emb.dequant_dtype = dequant_dtype
    return emb


_CODE = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}


def reference(raw, qt, V, K, ids, out_dtype, dequant_dtype):
    """The reference's Embedding (ops.py Embedding + dequant.py), restated on the CPU:
        row  = fp32 if out_dtype is None else out_dtype       (cast_bias_weight with the module as `input`)
        math = row if dequant_dtype == "target" else dequant_dtype
        F.embedding(ids, dequantize(raw, math).to(row)).to(out_dtype)
    dequantize: the oracle's chain in math (None = fp16); BF16 always widens to fp32; the fallback types take gguf-py's fp32
    values (dequant_dtype ignored)."""
    row = torch.float32 if out_dtype is None else out_dtype
    math = row if dequant_dtype == "target" else dequant_dtype
    flat = np.ascontiguousarray(raw).reshape(-1)
    if qt in FALLBACK:
        W = torch.from_numpy(gguf_values(flat, qt))
    elif qt == Q.BF16:
        W = torch.from_numpy((flat.view(np.uint16).astype(np.uint32) << 16).view(np.float32))
    else:
        code = 0 if math is None else _CODE[math]
        bits = oracle.dequant(flat, int(qt), code, code)
        W = torch.from_numpy(bits) if code == 2 else torch.from_numpy(bits.view(np.int16)).view(TORCH_DT[code])
    W = W.to(row).reshape(V, K)
    return torch.nn.functional.embedding(ids.cpu().long(), W).to(dtype=out_dtype)


def _same(got, want):
    assert got.dtype == want.dtype and tuple(got.shape) == tuple(want.shape), (got.dtype, want.dtype, got.shape, want.shape)
    assert np.array_equal(torch_bits(got), torch_bits(want))


LAYER_TYPES = [Q.Q4_0, Q.Q8_0, Q.Q3_K, Q.Q6_K, Q.IQ4_XS, Q.BF16, Q.IQ2_XS]
OUT_DTYPES = [None, torch.float16, torch.bfloat16, torch.float32]
DEQUANT_DTYPES = [None, torch.float16, torch.bfloat16, torch.float32, "target"]
_ROWS_ENTRY = lambda qt: "ggufb200_dequant_rows_fallback" if qt in FALLBACK else "ggufb200_dequant_rows"  # noqa: E731


def _forward(emb, ids, out_dtype):
    return emb(ids) if out_dtype is None else emb(ids, out_dtype=out_dtype)


@pytest.mark.parametrize("dequant_dtype", DEQUANT_DTYPES, ids=str)
@pytest.mark.parametrize("out_dtype", OUT_DTYPES, ids=str)
@pytest.mark.parametrize("qt", LAYER_TYPES, ids=lambda q: q.name)
def test_layer_equals_the_reference(pkg, monkeypatch, qt, out_dtype, dequant_dtype):
    V, K = 300, 768
    raw = _raw_table(qt, V, K, seed=50)
    emb = _embedding(pkg, qt, raw, V, K, dequant_dtype=dequant_dtype)
    ids = torch.tensor([[0, V - 1, 5, 5], [17, 299, 1, 0]], device=DEV)
    calls = _spy(pkg, monkeypatch)
    got = _forward(emb, ids, out_dtype)
    monkeypatch.undo()
    assert calls == [_ROWS_ENTRY(qt)], calls
    _same(got.cpu(), reference(raw, qt, V, K, ids, out_dtype, dequant_dtype))


@pytest.mark.parametrize("qt", [Q.Q6_K, Q.BF16, Q.IQ2_XS], ids=lambda q: q.name)
def test_layer_id_layouts(pkg, monkeypatch, qt):
    """1-D, 2-D and 3-D ids, int32 ids, non-contiguous ids and empty ids: one gather per forward, the reference's rows."""
    V, K = 257, 1280
    raw = _raw_table(qt, V, K, seed=51)
    emb = _embedding(pkg, qt, raw, V, K)
    base = torch.randint(0, V, (4, 6, 5), device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    base[0, 0, 0], base[-1, -1, -1] = 0, V - 1
    layouts = [base[0, 0], base[0], base, base.to(torch.int32), base[:, ::2, 1:], base.transpose(0, 2),
               torch.zeros(0, dtype=torch.int64, device=DEV), torch.zeros(2, 0, dtype=torch.int64, device=DEV)]
    for ids in layouts:
        for out_dtype in (None, torch.bfloat16):
            calls = _spy(pkg, monkeypatch)
            got = _forward(emb, ids, out_dtype)
            monkeypatch.undo()
            assert calls == [_ROWS_ENTRY(qt)], (tuple(ids.shape), calls)
            _same(got.cpu(), reference(raw, qt, V, K, ids, out_dtype, None))


@pytest.mark.parametrize("qt", [Q.Q4_0, Q.BF16, Q.IQ2_XS], ids=lambda q: q.name)
def test_layer_offloaded_table(pkg, monkeypatch, qt):
    """A table kept on the CPU, ids on the GPU: the rows are gathered on the GPU from the moved table."""
    V, K = 120, 2560
    raw = _raw_table(qt, V, K, seed=52)
    emb = _embedding(pkg, qt, raw, V, K, device="cpu", dequant_dtype="target")
    ids = torch.tensor([[3, 119, 0, 3]], device=DEV)
    calls = _spy(pkg, monkeypatch)
    got = _forward(emb, ids, torch.float16)
    monkeypatch.undo()
    assert calls == [_ROWS_ENTRY(qt)] and got.device.type == "cuda"
    _same(got.cpu(), reference(raw, qt, V, K, ids, torch.float16, "target"))


@pytest.mark.parametrize("dequant_dtype", [None, "target"], ids=str)
@pytest.mark.parametrize("out_dtype", OUT_DTYPES, ids=str)
@pytest.mark.parametrize("V,K", rc.BF16_ODD_WIDTHS, ids=lambda v: str(v))
def test_layer_bf16_table_at_a_width_not_a_multiple_of_8(pkg, monkeypatch, golden_dir, V, K, out_dtype, dequant_dtype):
    """The row gather needs K % 8 == 0; a BF16 table of any other width takes the whole-table dequant, which gives the
    reference's rows.  The 4099-element shapes are the golden stream, checked against its reference values too."""
    if V * K == 4099:
        g = np.load(os.path.join(golden_dir, "dequant_BF16.npz"))
        raw = g["packed"].reshape(V, 2 * K)
        assert np.array_equal(g["out_m0_o2"], (raw.reshape(-1).view(np.uint16).astype(np.uint32) << 16))
    else:
        raw = oracle.random_blocks(int(Q.BF16), V * K, seed=53).reshape(V, 2 * K)
    emb = _embedding(pkg, Q.BF16, raw, V, K, dequant_dtype=dequant_dtype)
    ids = torch.tensor([0, V - 1, V // 2, 0], device=DEV)
    calls = _spy(pkg, monkeypatch)
    got = _forward(emb, ids, out_dtype)
    monkeypatch.undo()
    assert calls == ["ggufb200_dequant"], calls
    _same(got.cpu(), reference(raw, Q.BF16, V, K, ids, out_dtype, dequant_dtype))
