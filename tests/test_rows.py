"""CPU checks of the Embedding row gather's test cases (tests/rows_cases.py) and of the C ABI's refusals.

* Coverage: the case list reaches, per table type, every (math, out) pair at every chunk shape on both staging branches of
  csrc/rows.cu, computed from the restated geometry rather than counted by hand; likewise the fallback types (out dtypes) and
  BF16 (its own in-place kernel); plus the id edges and the grid-y split.
* The model: the gather built on the C oracle reproduces the reference's golden values, and some listed case rejects each
  simulated fault (a dropped partial chunk, a chunk's b0 off by one block, the math dtype ignored, an out-of-range id clamped
  or zeroed as -0, the second grid-y slice written at row 0).  Where a fault is invisible on a case, that is shown too.
* ggufb200_dequant_rows and ggufb200_unpack_int refuse bad arguments before any device is touched."""
import ctypes

import numpy as np
import pytest

import rows_cases as rc
from fallback_cases import FALLBACK
from util import COMBOS, Q

OK, E_TYPE, E_DTYPE, E_ALIGN, E_SHAPE, E_NULL = 0, -1, -2, -3, -4, -5
REAL_WIDTHS = (768, 1280, 2560, 3584, 4096, 5120)


def _rows_of(case):
    ids = rc.make_ids(case.ids, case.V, case.seed)
    return ids[(ids >= 0) & (ids < case.V)]


def _cells(qt):
    got = set()
    for c in rc.CASES:
        if c.qt == qt:
            for branch in rc.staging(qt, c.K, c.offset, _rows_of(c)):
                got.add((c.pair, rc.chunk_shape(qt, c.K), branch))
    return got


# ---------------------------------------------------------------- coverage
@pytest.mark.parametrize("qt", rc.TABLE + FALLBACK, ids=lambda q: q.name)
def test_every_pair_chunk_shape_and_staging_branch_is_reached(qt):
    want = {(p, s, b) for p in rc.pairs_of(qt) for s in rc.SHAPES for b in (rc.WORD, rc.BYTE)}
    missing = want - _cells(qt)
    assert not missing, f"{qt.name}: no case reaches {sorted(missing)}"


def test_bf16_every_pair_and_chunk_shape_in_place():
    want = {(p, s, rc.INPLACE) for p in rc.PAIRS for s in rc.SHAPES}
    assert not want - _cells(Q.BF16)
    assert any(c.qt == Q.BF16 and c.offset % 4 == 2 for c in rc.CASES), "a 2-byte aligned BF16 view"
    assert all(c.offset % 2 == 0 for c in rc.CASES if c.qt == Q.BF16), "the BF16 kernel reads uint16: never an odd view"
    assert all(K % 8 for _V, K in rc.BF16_ODD_WIDTHS) and (4099, 1) in rc.BF16_ODD_WIDTHS and (1, 4099) in rc.BF16_ODD_WIDTHS


@pytest.mark.parametrize("qt", rc.TABLE, ids=lambda q: q.name)
def test_real_widths_odd_block_counts_and_goldens(qt):
    ks = {c.K for c in rc.CASES if c.qt == qt}
    assert set(REAL_WIDTHS) <= ks
    bs = rc.geom(qt)[0]
    if bs == 32:
        assert any(k // 32 % 2 == 1 and rc.chunk_shape(qt, k) == "tail" for k in ks), "32 * odd with a partial last chunk"
    golden = {(c.pair, c.V, c.K) for c in rc.CASES if c.qt == qt and c.golden}
    assert {p for p, _V, _K in golden} == set(COMBOS)
    assert {(V, K) for _p, V, K in golden} == ({(4, 2560), (5, 2048)} if bs == 256 else {(2, 2176), (17, 256)})


def test_the_formats_whose_rows_are_whole_words_reach_bytes_only_through_a_view():
    """Q4_1, Q5_1, Q2_K, Q4_K, Q5_K and IQ4_XS rows are a multiple of 4 bytes at every K: only an offset view stages bytes.
    The 18-, 22- and 34-byte formats take the byte branch at an odd block count per row, Q3_K and Q6_K at K = 768 and 1280."""
    for qt in (Q.Q4_1, Q.Q5_1, Q.Q2_K, Q.Q4_K, Q.Q5_K, Q.IQ4_XS):
        for c in rc.CASES:
            if c.qt == qt and c.offset == 0 and c.ids != "empty":
                assert rc.staging(qt, c.K, 0, _rows_of(c)) == {rc.WORD}, c.id
        assert any(c.qt == qt and c.offset % 4 == 2 and rc.BYTE in rc.staging(qt, c.K, c.offset, _rows_of(c)) for c in rc.CASES)
    rows = np.arange(9)
    for qt in (Q.Q4_0, Q.Q5_0, Q.Q8_0, Q.IQ4_NL):
        assert rc.staging(qt, 2080, 0, rows) == {rc.WORD, rc.BYTE} and rc.staging(qt, 2048, 0, rows) == {rc.WORD}
    for qt in (Q.Q3_K, Q.Q6_K):
        assert rc.staging(qt, 768, 0, rows) == {rc.BYTE} and rc.staging(qt, 1280, 0, rows) == {rc.BYTE}
        assert rc.staging(qt, 512, 0, rows) == {rc.WORD}


def test_id_edges_specials_empty_and_the_grid_y_split():
    for qt in rc.TABLE + [Q.BF16] + FALLBACK:
        mine = [c for c in rc.CASES if c.qt == qt]
        assert any(c.specials for c in mine), qt.name
        assert any(c.ids == "empty" for c in mine), qt.name
        edges = [c for c in mine if c.ids == "edges"]
        assert edges and all({0, c.V - 1, -1, c.V, 10**9} <= set(rc.make_ids("edges", c.V).tolist()) for c in edges)
        ids = rc.make_ids("edges", 9)
        assert len(set(ids[(ids >= 0) & (ids < 9)].tolist())) < np.count_nonzero((ids >= 0) & (ids < 9)), "repeated ids"
    many = [c for c in rc.CASES if c.ids == "many"]
    assert {Q.BF16} < {c.qt for c in many} and any(c.qt in FALLBACK for c in many) and any(c.qt in rc.TABLE for c in many)
    for c in many:
        n = rc.make_ids("many", c.V, c.seed).size
        assert n == 70000 and len(rc.grid_y_slices(n)) == 2 and rc.grid_y_slices(n)[1] == (65535, 70000 - 65535)
    assert rc.make_ids("empty", 9).size == 0


def test_geometry_restatement():
    assert rc.chunk_elems(Q.Q4_K) == rc.chunk_elems(Q.Q8_0) == 2048 and rc.chunk_elems(Q.IQ2_XXS) == 8192
    assert rc.chunk_blocks(Q.Q4_0) == 64 and rc.chunk_blocks(Q.Q6_K) == 8 and rc.chunk_blocks(Q.MXFP4) == 256
    assert (rc.n_chunks(Q.Q4_0, 2080), rc.last_chunk_blocks(Q.Q4_0, 2080)) == (2, 1)
    assert (rc.n_chunks(Q.Q4_K, 5120), rc.last_chunk_blocks(Q.Q4_K, 5120)) == (3, 4)
    assert (rc.n_chunks(Q.IQ3_S, 8448), rc.last_chunk_blocks(Q.IQ3_S, 8448)) == (2, 1)
    assert [rc.chunk_shape(Q.Q4_K, k) for k in (768, 2048, 2560, 4096)] == ["below", "one", "tail", "whole"]
    assert rc.grid_y_slices(0) == [] and rc.grid_y_slices(65535) == [(0, 65535)]


# ---------------------------------------------------------------- the model
GOLDEN = [c for c in rc.CASES if c.golden]


@pytest.mark.parametrize("case", GOLDEN, ids=lambda c: c.id)
def test_the_model_reproduces_the_golden_values(case):
    table = rc.table_bytes(case)
    ids = rc.make_ids(case.ids, case.V, case.seed)
    assert rc.mismatch(rc.gather_model(case, table, ids), rc.expected(case, table, ids), case.out) is None


def _rejects(case, fault, ids=None):
    table = rc.table_bytes(case)
    ids = rc.make_ids(case.ids, case.V, case.seed) if ids is None else ids
    want = rc.gather_model(case, table, ids)
    return rc.mismatch(rc.gather_model(case, table, ids, fault), want, case.out) is not None


def _first_rejecting(fault, pool):
    for c in pool:
        if _rejects(c, fault):
            return c
    return None


SMALL = [c for c in rc.CASES if c.ids == "edges"]


@pytest.mark.parametrize("fault", rc.FAULTS)
def test_each_simulated_fault_is_rejected_by_a_listed_case(fault):
    # the cases on which the fault can show at all (test_where_each_fault_is_invisible shows the others)
    pool = {"grid_y_at_0": [c for c in rc.CASES if c.ids == "many"],
            "drop_tail": [c for c in SMALL if c.K % rc.chunk_elems(c.qt)],
            "b0_shift": [c for c in SMALL if rc.n_chunks(c.qt, c.K) > 1],
            "math_ignored": [c for c in SMALL if c.math != 0 and c.qt in rc.TABLE]}.get(fault, SMALL)
    assert _first_rejecting(fault, pool) is not None, f"no listed case rejects {fault}"
    # each fault but the grid-y one is seen on every table type
    if fault != "grid_y_at_0":
        for qt in rc.TABLE:
            assert _first_rejecting(fault, [c for c in pool if c.qt == qt]) is not None, (fault, qt.name)


def test_where_each_fault_is_invisible():
    """A fault shows only on the cases that exercise its branch; the list has those, and these would not do alone."""
    one = next(c for c in SMALL if c.qt == Q.Q4_K and c.K == 2048 and c.pair == (1, 1))
    whole = next(c for c in SMALL if c.qt == Q.Q4_0 and c.K == 4096 and c.pair == (2, 0))
    tail = next(c for c in SMALL if c.qt == Q.Q4_0 and c.K == 2080)
    # a dropped partial chunk: invisible when K is a whole number of chunks
    assert not _rejects(one, "drop_tail") and not _rejects(whole, "drop_tail") and _rejects(tail, "drop_tail")
    # b0 off by one block: invisible with one chunk per row
    assert not _rejects(one, "b0_shift") and _rejects(whole, "b0_shift") and _rejects(tail, "b0_shift")
    # the math dtype ignored: invisible at fp16 math, and at fp32 math for Q8_0 into fp16 (d * q is exact in fp32)
    fp16_math = next(c for c in SMALL if c.qt == Q.Q4_K and c.math == 0)
    q8 = next(c for c in SMALL if c.qt == Q.Q8_0 and c.pair == (2, 0) and not c.specials)
    assert not _rejects(fp16_math, "math_ignored") and not _rejects(q8, "math_ignored") and _rejects(one, "math_ignored")
    # out-of-range ids clamped or zeroed as -0: invisible when every id is in range
    inside = np.array([0, 3, 8, 8, 1], dtype=np.int64)
    for fault in ("clamp_oob", "negative_zero"):
        assert not _rejects(one, fault, inside) and _rejects(one, fault)
    # the second grid-y slice written at row 0: invisible below 65536 ids
    assert not _rejects(tail, "grid_y_at_0")


def test_the_model_marks_unwritten_elements():
    case = SMALL[0]
    table = rc.table_bytes(case)
    ids = rc.make_ids(case.ids, case.V)
    want = rc.gather_model(case, table, ids)
    got = want.copy()
    got[3, 5] = rc.FILL[case.out]
    assert "never written" in rc.mismatch(got, want, case.out)


# ---------------------------------------------------------------- ABI refusals
@pytest.fixture
def ptrs():
    buf = (ctypes.c_uint8 * 8192)()
    p16 = (ctypes.addressof(buf) + 15) & ~15
    yield p16, p16 + 4096
    del buf


def test_dequant_rows_refusals(pkg, ptrs):
    L = pkg.lib.lib()
    p, q = ptrs

    def rows(qt=Q.Q4_K, packed=p, n_table=100, K=512, idx=p, n=4, out=q, out_dtype=1, math=0):
        return L.ggufb200_dequant_rows(int(qt), packed, n_table, K, idx, n, out, out_dtype, math, None)
    for qt in (999, -1, Q.IQ2_XXS, Q.MXFP4, Q.F16, Q.F32):
        assert rows(qt=qt) == E_TYPE, qt
    for od, md in ((3, 0), (-1, 0), (0, 3), (0, -1)):
        assert rows(out_dtype=od, math=md) == E_DTYPE
    assert rows(K=128) == E_SHAPE                               # K % 256
    assert rows(qt=Q.Q4_0, K=48) == E_SHAPE                     # K % 32
    assert rows(qt=Q.BF16, K=4) == E_SHAPE and rows(qt=Q.BF16, K=1030) == E_SHAPE   # K % 8
    assert rows(K=0) == E_SHAPE and rows(K=-256) == E_SHAPE
    assert rows(n=-1) == E_SHAPE and rows(n_table=-1) == E_SHAPE
    assert rows(n=0, packed=None, idx=None, out=None) == OK     # zero ids: nothing to read or write
    assert rows(n=0, K=100) == E_SHAPE                          # the shape is still checked
    assert rows(packed=None) == E_NULL and rows(idx=None) == E_NULL and rows(out=None) == E_NULL
    assert rows(out=q + 4) == E_ALIGN and rows(out=q + 8) == E_ALIGN
    assert rows(qt=Q.BF16, K=8, out=q + 2) == E_ALIGN


def test_unpack_int_refusals(pkg, ptrs):
    L = pkg.lib.lib()
    p, q = ptrs

    def unpack(qt=Q.Q4_K, packed=p, n=2, outs=(q, q, q)):
        return L.ggufb200_unpack_int(int(qt), packed, n, *outs, None)
    assert unpack(qt=Q.BF16) == E_TYPE and unpack(qt=999) == E_TYPE
    for qt in FALLBACK:
        assert unpack(qt=qt) == E_TYPE, qt.name
    assert unpack(n=-1) == E_SHAPE
    assert unpack(n=0) == OK and unpack(n=0, packed=None, outs=(None, None, None)) == OK
    assert unpack(packed=None) == E_NULL
