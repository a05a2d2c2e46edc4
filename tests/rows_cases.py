"""Cases, restated geometry and a numpy model of the Embedding row gather (csrc/rows.cu: ggufb200_dequant_rows for the 13
table types, ggufb200_dequant_rows_fallback for the numpy-fallback types).

The geometry is restated from rows.cu and is used only to check that the case list reaches every branch of the kernel:
  * one CTA per (gathered row, chunk); a chunk is chunk_elems(qt) elements (2048 for the table types, 8192 for the fallback
    types), i.e. chunk_blocks = chunk_elems / block_size blocks; chunk c covers blocks b0 = c * chunk_blocks .. b0 + nb of the
    row, nb = min(chunk_blocks, row_blocks - b0), so the last chunk of a row may be partial;
  * a chunk's packed bytes are staged into shared memory as 32-bit words when src % 4 == 0 and len % 4 == 0, byte by byte
    otherwise (src = table + (r * row_blocks + b0) * type_size, len = nb * type_size);
  * the ids are cut into grid-y slices of at most 65535, slice y0 writing output rows y0 ..;
  * BF16 has its own kernel: 1024 elements per CTA, read in place from the table (no staging).

The model (`gather_model`) is the gather built on the C oracle (`oracle.dequant` of the gathered rows' bytes) for the table
types, on gguf-py (`fallback_cases.gguf_values`, rounded once) for the fallback types, and on the plain widening for BF16.  It
takes a `fault` switch that simulates one way the kernel could be subtly wrong; tests/test_rows.py shows that the listed cases
reject each fault."""
import dataclasses
import os
import zlib

import gguf
import numpy as np
import torch

import oracle
from fallback_cases import FALLBACK, random_blocks as fallback_blocks
from util import ALL_QTYPES, COMBOS, Q, canon_nan

TABLE = [q for q in ALL_QTYPES if q != Q.BF16]        # the 12 block formats of ggufb200_dequant_rows
PAIRS = [(m, o) for m in (0, 1, 2) for o in (0, 1, 2)]  # (math dtype, out dtype) codes
SHAPES = ("below", "one", "tail", "whole")              # K < one chunk, exactly one, several with a partial last, several whole
WORD, BYTE, INPLACE = "word", "byte", "inplace"         # staging branches (BF16: read in place)
GRID_Y = 65535

# unwritten output elements keep these bits: signalling NaNs (fp16 / bf16) or a NaN with low payload bits (fp32) that no
# conversion or arithmetic of the kernel can produce, so "still the fill" means "never written"
FILL = {0: 0x7D11, 1: 0x7F91, 2: 0x7FA11111}
BITS = {0: np.uint16, 1: np.uint16, 2: np.uint32}


def geom(qt):
    return gguf.GGML_QUANT_SIZES[qt]


def chunk_elems(qt):
    if qt == Q.BF16:
        return 1024                 # rows_bf16_kernel: 256 threads x 4 elements per CTA column
    return 8192 if qt in FALLBACK else 2048


def chunk_blocks(qt):
    return chunk_elems(qt) // geom(qt)[0]


def n_chunks(qt, K):
    return -(-K // chunk_elems(qt))


def last_chunk_blocks(qt, K):
    row_blocks = K // geom(qt)[0]
    return row_blocks - (n_chunks(qt, K) - 1) * chunk_blocks(qt)


def chunk_shape(qt, K):
    c = chunk_elems(qt)
    if K < c:
        return "below"
    if K == c:
        return "one"
    return "tail" if K % c else "whole"


def row_bytes(qt, K):
    bs, ts = geom(qt)
    return K // bs * ts


def staging(qt, K, offset, rows):
    """The staging branch of every (row, chunk) CTA for the in-range `rows` of a table at byte `offset` from a 4-byte aligned
    base: the set of branches taken."""
    if qt == Q.BF16:
        return {INPLACE} if len(rows) else set()
    bs, ts = geom(qt)
    rows = np.unique(np.asarray(rows, dtype=np.int64))
    rb, cb = K // bs, chunk_blocks(qt)
    taken = set()
    for c in range(n_chunks(qt, K)):
        b0 = c * cb
        nb = min(cb, rb - b0)
        src = offset + (rows * rb + b0) * ts
        ok = (src % 4 == 0) & ((nb * ts) % 4 == 0)
        if ok.any():
            taken.add(WORD)
        if (~ok).any():
            taken.add(BYTE)
    return taken


def grid_y_slices(n):
    return [(y0, min(GRID_Y, n - y0)) for y0 in range(0, n, GRID_Y)]


# ---------------------------------------------------------------- the cases
@dataclasses.dataclass(frozen=True)
class RowsCase:
    qt: object
    V: int
    K: int
    ids: str            # "edges", "empty" or "many" (see make_ids)
    out: int            # dtype code of the output
    math: int           # dtype code of the dequant math (fallback types: 2, their fp32 decoder; BF16: ignored)
    offset: int = 0     # byte offset of the table from an aligned base
    specials: bool = False
    golden: bool = False  # the table is the golden stream of tests/golden/dequant_<T>.npz reshaped to [V, K]

    @property
    def pair(self):
        return (self.math, self.out)

    @property
    def id(self):
        return (f"{self.qt.name}-V{self.V}-K{self.K}-m{self.math}o{self.out}-{self.ids}-off{self.offset}"
                f"{'-sp' if self.specials else ''}{'-golden' if self.golden else ''}")

    @property
    def seed(self):
        return zlib.crc32(self.id.encode())


def make_ids(spec, V, seed=0):
    """int64 ids.  edges: 0 and V - 1, repeats, both parities of row, -1, V and 10^9; empty; many: 70 000 ids in -3 .. V + 2 with
    the edges at both ends and around the grid-y split."""
    if spec == "empty":
        return np.zeros(0, dtype=np.int64)
    edges = [0, V - 1, 1, 2, 2, -1, V - 1, V, 0, 3, 10**9, 5]
    edges = [i if i in (-1, V, 10**9) or i < V else i % V for i in edges]
    if spec == "edges":
        return np.array(edges, dtype=np.int64)
    assert spec == "many"
    ids = np.random.default_rng(seed).integers(-3, V + 3, size=70000, dtype=np.int64)
    ids[:len(edges)] = edges
    ids[-len(edges):] = edges
    ids[GRID_Y - 6:GRID_Y + 6] = edges
    return ids


K_CANDIDATES = {   # per family and chunk shape; real widths (CLIP-L / CLIP-G / Qwen3-4B / Qwen2.5-VL-7B / Mistral-24B) and 32 * odd
    32: {"below": [768, 1312, 1280], "one": [2048], "tail": [2080, 2560, 3584, 5120], "whole": [4096]},
    256: {"below": [768, 1280, 512, 1024], "one": [2048], "tail": [2560, 3584, 5120, 2304], "whole": [4096]},
    "fallback": {"below": [768, 2560], "one": [8192], "tail": [8192 + 256], "whole": [16384]},
    "bf16": {"below": [520, 768], "one": [1024], "tail": [2056, 3080], "whole": [2048, 4096]},
}
OFFSETS = (2, 1, 6, 3)          # byte-offset views: data_ptr % 4 == 2 and odd


def _family(qt):
    if qt == Q.BF16:
        return "bf16"
    if qt in FALLBACK:
        return "fallback"
    return geom(qt)[0]


def pairs_of(qt):
    return [(2, o) for o in (0, 1, 2)] if qt in FALLBACK else PAIRS


def _in_range(spec, V):
    ids = make_ids(spec, V, 0)
    return ids[(ids >= 0) & (ids < V)]


def _grid_cases(qt, V=9):
    """Every (pair, chunk shape) of the type, each staging branch reached: offset-0 tables whose rows take the word branch (and
    the byte branch where the row or chunk bytes are not a multiple of 4), plus a byte-offset view where they never do."""
    cases = []
    rows = _in_range("edges", V)
    cands = K_CANDIDATES[_family(qt)]
    for pi, (m, o) in enumerate(pairs_of(qt)):
        for si, shape in enumerate(SHAPES):
            ks = cands[shape][pi % len(cands[shape]):] + cands[shape][:pi % len(cands[shape])]
            specials = (pi + si) % 2 == 1
            mk = lambda K, off: RowsCase(qt, V, K, "edges", o, m, off, specials)  # noqa: E731
            cases.append(mk(ks[0], 0))
            reached = staging(qt, ks[0], 0, rows)
            if qt == Q.BF16:
                if pi % 3 == 0:
                    cases.append(mk(ks[0], 2))          # 2-byte aligned: the kernel reads uint16
                continue
            if WORD not in reached:
                k_word = next(k for k in ks[1:] + [2048 if qt not in FALLBACK else 8192] if WORD in staging(qt, k, 0, rows))
                cases.append(mk(k_word, 0))
            if BYTE not in reached:
                cases.append(mk(ks[0], OFFSETS[(pi + si) % len(OFFSETS)]))
    return cases


def _golden_cases():
    """The golden streams (40 blocks of 256, 136 blocks of 32) as [4, 2560] / [5, 2048] and [2, 2176] / [17, 256] tables, at the
    (math, out) pairs the golden files hold."""
    cases = []
    for qt in TABLE:
        shapes = [(4, 2560), (5, 2048)] if geom(qt)[0] == 256 else [(2, 2176), (17, 256)]
        for i, (m, o) in enumerate(COMBOS):
            V, K = shapes[i % 2]
            cases.append(RowsCase(qt, V, K, "edges", o, m, golden=True))
    return cases


def _edge_cases():
    cases = []
    for i, qt in enumerate(TABLE + [Q.BF16] + FALLBACK):
        m, o = pairs_of(qt)[i % len(pairs_of(qt))]
        cases.append(RowsCase(qt, 9, 768 if qt != Q.BF16 else 520, "empty", o, m))
    cases += [RowsCase(Q.Q4_K, 64, 256, "many", 1, 0), RowsCase(Q.Q3_K, 64, 768, "many", 0, 2, specials=True),
              RowsCase(Q.Q5_0, 64, 2080, "many", 0, 1, offset=2), RowsCase(Q.BF16, 64, 8, "many", 2, 0),
              RowsCase(Q.IQ2_XXS, 64, 256, "many", 1, 2)]
    return cases


CASES = [c for qt in TABLE + [Q.BF16] + FALLBACK for c in _grid_cases(qt)] + _golden_cases() + _edge_cases()

# BF16 tables whose width is not a multiple of 8 (the ABI refuses them; the Embedding layer must still give the reference's
# rows): (V, K), the first two the golden stream of 4099 elements
BF16_ODD_WIDTHS = [(4099, 1), (1, 4099), (50, 100), (7, 4), (33, 1030)]


# ---------------------------------------------------------------- tables
_SPECIAL_F16 = (0x7C00, 0x7E00, 0xFC00)     # +Inf, NaN, -Inf block scales


def table_bytes(case):
    """[V, row_bytes] uint8: random blocks with finite scales; with `specials`, gathered rows carry blocks with +Inf, NaN and
    -Inf scales, an all-0x00 block and an all-0xFF block."""
    qt, V, K = case.qt, case.V, case.K
    bs, ts = geom(qt)
    if case.golden:
        g = np.load(_golden_path(qt))
        return g["packed"].reshape(V, row_bytes(qt, K))
    n = V * K // bs
    if qt in FALLBACK:
        blocks = fallback_blocks(qt, n, seed=case.seed, scale=0.01, specials=case.specials)
    else:
        blocks = oracle.random_blocks(int(qt), n, seed=case.seed, scale=0.01).reshape(n, ts).copy()
    if case.specials:
        rb = K // bs
        at = [(1 * rb) % n, (2 * rb - 1) % n, ((V - 1) * rb + rb // 2) % n, (2 * rb) % n, (rb - 1) % n]
        if qt == Q.BF16:
            flat = blocks.reshape(-1).view(np.uint16)
            for j, bits in zip(at, (0x7F80, 0x7FC1, 0xFF80, 0x0000, 0xFFFF)):
                flat[j] = bits
        else:
            if qt not in FALLBACK:
                off = oracle._F16_FIELDS[int(qt)][0]
                for j, bits in zip(at[:3], _SPECIAL_F16):
                    blocks[j, off:off + 2] = np.array([bits], dtype=np.uint16).view(np.uint8)
            blocks[at[3]] = 0x00
            blocks[at[4]] = 0xFF
    return blocks.reshape(V, row_bytes(qt, K))


def _golden_path(qt):
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"dequant_{qt.name}.npz")


def golden_values(case):
    """The reference's values of the golden table, [V, K] bits of the case's out dtype."""
    g = np.load(_golden_path(case.qt))
    return g[f"out_m{case.math}_o{case.out}"].reshape(case.V, case.K)


# ---------------------------------------------------------------- the model
def _round(f32, out):
    """fp32 values rounded once (to nearest even) to out, as bits."""
    t = torch.from_numpy(np.ascontiguousarray(f32, dtype=np.float32))
    if out == 2:
        return t.numpy().view(np.uint32).copy()
    return t.to({0: torch.float16, 1: torch.bfloat16}[out]).view(torch.int16).numpy().view(np.uint16).copy()


def dequant_rows_bytes(qt, raw, K, out, math):
    """Bits [n, K] of the dequantised rows `raw` ([n, row_bytes] uint8): the oracle, gguf-py or the bf16 widening."""
    n = raw.shape[0]
    if n == 0:
        return np.zeros((0, K), dtype=BITS[out])
    flat = np.ascontiguousarray(raw).reshape(-1)
    if qt == Q.BF16:
        f32 = (flat.view(np.uint16).astype(np.uint32) << 16).view(np.float32)
        return _round(f32, out).reshape(n, K)
    if qt in FALLBACK:
        from fallback_cases import gguf_values
        return _round(gguf_values(flat, qt), out).reshape(n, K)
    bits = oracle.dequant(flat, int(qt), out, math)
    return (bits.view(np.uint32) if out == 2 else bits).reshape(n, K)


FAULTS = ("drop_tail", "b0_shift", "math_ignored", "clamp_oob", "negative_zero", "grid_y_at_0")


def gather_model(case, table, ids, fault=None):
    """Bits [len(ids), K] the gather writes into an output filled with FILL, with `fault` simulated:
      drop_tail      the last partial chunk of every row is never written (chunk count rounded down);
      b0_shift       chunks after the first read from one block past their b0 (row bytes continue into the next row);
      math_ignored   the fp16 chain is run whatever the math dtype;
      clamp_oob      an out-of-range id gathers the nearest row instead of zeros;
      negative_zero  an out-of-range id gives -0 instead of +0;
      grid_y_at_0    the second grid-y slice is written at output row 0 instead of row 65535."""
    qt, V, K, out = case.qt, case.V, case.K, case.out
    ids = np.asarray(ids, dtype=np.int64)
    n = ids.size
    res = np.full((n, K), FILL[out], dtype=BITS[out])
    inside = (ids >= 0) & (ids < V)
    math = 0 if fault == "math_ignored" else case.math
    uniq, inv = np.unique(ids[inside], return_inverse=True)
    res[inside] = dequant_rows_bytes(qt, table[uniq], K, out, math)[inv]
    if fault == "clamp_oob":
        res[~inside] = dequant_rows_bytes(qt, table[np.clip(ids[~inside], 0, V - 1)], K, out, math)
    else:
        res[~inside] = (0x8000 if out < 2 else 0x80000000) if fault == "negative_zero" else 0
    c = chunk_elems(qt)
    if fault == "drop_tail" and K % c:
        res[:, K // c * c:] = FILL[out]
    if fault == "b0_shift" and n_chunks(qt, K) > 1 and qt != Q.BF16:
        bs, ts = geom(qt)
        rb, cb = K // bs, chunk_blocks(qt)
        stream = np.concatenate([table.reshape(-1), np.zeros(ts, dtype=np.uint8)])
        for i in np.flatnonzero(inside):
            for ch in range(1, n_chunks(qt, K)):
                b0, nb = ch * cb, min(cb, rb - ch * cb)
                s = (ids[i] * rb + b0 + 1) * ts
                res[i, b0 * bs:(b0 + nb) * bs] = dequant_rows_bytes(qt, stream[s:s + nb * ts].reshape(1, -1), nb * bs, out, math)[0]
    if fault == "grid_y_at_0" and n > GRID_Y:
        moved = res.copy()
        for y0, ny in grid_y_slices(n)[1:]:
            moved[0:ny] = res[y0:y0 + ny]
            moved[y0:y0 + ny] = FILL[out]
        res = moved
    return res


def canon(bits, out):
    """NaN payloads canonicalised (not part of the contract), every other bit pattern kept."""
    return canon_nan(np.ascontiguousarray(bits).reshape(-1).view(BITS[out]), out)


def mismatch(got, want, out):
    """None when `got` (bits) is what the gather must write for `want`: equal up to NaN payloads, and no element left at the
    fill pattern.  Otherwise a short description."""
    got = np.ascontiguousarray(got).reshape(-1).view(BITS[out])
    unwritten = int(np.count_nonzero(got == FILL[out]))
    if unwritten:
        return f"{unwritten} elements never written"
    bad = canon(got, out) != canon(want, out)
    if bad.any():
        return f"{int(bad.sum())} of {bad.size} elements differ, first at flat index {int(np.flatnonzero(bad)[0])}"
    return None


def expected(case, table, ids):
    """What ggufb200_dequant_rows(_fallback) must write: the golden values for golden tables, else the model without a fault."""
    if case.golden:
        g = golden_values(case)
        ids = np.asarray(ids)
        inside = (ids >= 0) & (ids < case.V)
        res = np.zeros((ids.size, case.K), dtype=BITS[case.out])
        res[inside] = g[ids[inside]]
        return res
    return gather_model(case, table, ids)
