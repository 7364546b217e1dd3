"""tg_topn (csrc/topn.cu) against the exact order of oracle/topn.py, row by row.

Every table carries a permuted unique `id` column.  For every call the test asserts the row count, that the ORDER BY
key sequence equals the reference's, that each output row is the input row with its id bit for bit in every column
(NULL flags, the sign of zero, NaN payloads and fsp bits included: only the comparison normalises), that no id
appears twice, and that every key group wholly inside the output holds exactly the reference's rows.  Ties in a group
cut by the window are unordered in the reference (a heap), so only their keys are compared."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column, MutChunk

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import topn as OT   # noqa: E402

gpu = pytest.mark.gpu
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
TYPES = {"int": (abi.TYPE_LONGLONG, 0), "uint": (abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED), "real": (abi.TYPE_DOUBLE, 0),
         "date": (abi.TYPE_DATE, 0), "datetime": (abi.TYPE_DATETIME, 0), "timestamp": (abi.TYPE_TIMESTAMP, 0),
         "duration": (abi.TYPE_DURATION, 0)}
KIND = {"int": "int", "uint": "uint", "real": "real", "date": "time", "datetime": "time", "timestamp": "time", "duration": "int"}
F64 = lambda bits: np.array([bits], np.uint64).view(np.float64)[0]
REAL_SPECIAL = [0.0, -0.0, np.inf, -np.inf, np.nan, F64(0xFFF8000000000000), F64(0x7FF0000000000001), F64(0xFFF00000DEADBEEF),
                5e-324, -5e-324, 2.2250738585072009e-308, 1.7976931348623157e308, -1.7976931348623157e308, 1.0, -1.0]
INT_SPECIAL = [INT64_MIN, INT64_MIN + 1, INT64_MAX, INT64_MAX - 1, 0, 1, -1, 1 << 32, -(1 << 32)]
UINT_SPECIAL = [0, 1, INT64_MIN, INT64_MAX, -1, -2]          # words: 2^63, 2^63 - 1, 2^64 - 1, 2^64 - 2


def _times(rng, n, tp):
    y = rng.choice([0, 1, 1970, 1999, 2000, 2024, 2038, 9999], n)
    mo, d = rng.integers(1, 13, n), rng.integers(1, 29, n)
    if tp == "date":
        h = mi = s = us = np.zeros(n, np.int64)
    else:
        h, mi, s = rng.integers(0, 24, n), rng.integers(0, 60, n), rng.integers(0, 60, n)
        us = rng.choice([0, 1, 500000, 999999], n) if tp == "datetime" else rng.integers(0, 1_000_000, n)
    fsp = rng.integers(0, 16, n)                                # fsp / type bits vary under equal calendar values
    w = np.zeros(n, np.uint64)
    for (_, off, _w), v in zip(OT.TIME_FIELDS, (y, mo, d, h, mi, s, us)):
        w |= np.asarray(v, np.uint64) << np.uint64(off)
    return (w | fsp.astype(np.uint64)).view(np.int64)


def gen_column(rng, tp, n, card):
    """8-byte words of a column of type tp: `card` distinct values (None: mostly distinct), specials always included"""
    m = n if card is None else card
    if tp == "int":
        pool = np.concatenate([np.array(INT_SPECIAL, np.int64), rng.integers(INT64_MIN, INT64_MAX, m, endpoint=True, dtype=np.int64)])
    elif tp == "uint":
        pool = np.concatenate([np.array(UINT_SPECIAL, np.int64), rng.integers(INT64_MIN, INT64_MAX, m, endpoint=True, dtype=np.int64)])
    elif tp == "real":
        pool = np.concatenate([np.array(REAL_SPECIAL), np.round(rng.normal(0, 1e6, m), 2)]).view(np.int64)
    elif tp == "duration":
        pool = np.concatenate([np.array([0, 1, -1, 838 * 3600 * 10**9, -838 * 3600 * 10**9], np.int64),
                               rng.integers(-838 * 3600 * 10**9, 838 * 3600 * 10**9, m)])
    else:
        pool = _times(rng, m + 8, tp)
    if card is not None:
        pool = pool[:card]
    return pool[rng.integers(0, len(pool), n)]


# the 15 data columns of every table (type, distinct values or None) and the id column at index 15
SCHEMA = [("int", 5), ("uint", 6), ("real", 8), ("date", 4), ("datetime", 6), ("timestamp", 5), ("duration", 4),
          ("int", None), ("uint", None), ("real", None), ("datetime", None), ("int", 300), ("real", 200), ("timestamp", 300),
          ("uint", 300)]
ID = len(SCHEMA)
ALL_NULL = 14          # column 14 is all NULL in every table with more than one row


def make_table(rng, n):
    vals, nulls = [], []
    for c, (tp, card) in enumerate(SCHEMA):
        vals.append(gen_column(rng, tp, n, card))
        nl = rng.random(n) < (0.1 if c % 3 else 0.0)           # every third column has no NULLs (and no bitmap)
        if c == ALL_NULL and n > 1:
            nl[:] = True
        nulls.append(nl)
    vals.append(rng.permutation(n).astype(np.int64))
    nulls.append(np.zeros(n, bool))
    types = [t for t, _ in SCHEMA] + ["int"]
    return vals, nulls, types


ITEM_SETS = [
    [(0, False)],
    [(2, True), (4, False)],
    [(3, False), (1, True), (5, False)],
    [(ALL_NULL, False), (6, True), (12, False), (0, True), (8, False)],
    [(2, False), (1, False), (5, True), (0, True), (3, False), (6, False), (11, True), (9, False)],
]


def _columns(vals, nulls, on_device=False):
    cols, keep = [], []
    for v, nl in zip(vals, nulls):
        col = Column(v, nl if nl.any() else None)
        cols.append(col)
    chk = Chunk(cols)
    if not on_device:
        return chk, chk.to_struct(), keep
    import torch
    s = chk.to_struct()
    for i, col in enumerate(cols):
        d = torch.from_numpy(col.data.view(np.int64).copy()).cuda()
        keep.append(d)
        s.cols[i].data = d.data_ptr()
        if col.null_bitmap is not None:
            b = torch.from_numpy(col.null_bitmap.copy()).cuda()
            keep.append(b)
            s.cols[i].null_bitmap = b.data_ptr()
    return chk, s, keep


def run_topn(vals, nulls, types, items, offset, count, cap=None, on_device=False, out=None):
    """-> (status, rows, [(values, NULL flags)] of the output)"""
    lib = abi.load_lib()
    chk, cs, keep = _columns(vals, nulls, on_device)
    n = len(vals[0])
    if out is None:
        out = MutChunk([8] * len(vals), cap if cap is not None else max(min(count, max(n - offset, 0)), 1), [np.int64] * len(vals))
    its = (abi.TgSortItem * max(len(items), 1))(*[abi.TgSortItem(c, int(d)) for c, d in items])
    tps = (C.c_int32 * len(types))(*[TYPES[t][0] for t in types])
    fls = (C.c_uint32 * len(types))(*[TYPES[t][1] for t in types])
    nr = C.c_int64(-1)
    rc = lib.tg_topn(0, int(on_device), C.byref(cs), tps, fls, its, len(items), C.c_int64(offset), C.c_int64(count),
                     C.byref(out.struct), C.byref(nr), None)
    if on_device:
        import torch
        torch.cuda.synchronize()
    return rc, nr.value, (out.columns(nr.value) if rc == 0 else None)


class Ref:
    """the reference order of one table under one ORDER BY, computed once and sliced per offset / count.  The table's
    last column is its id: a permutation of 0..n-1."""

    def __init__(self, vals, nulls, types, items):
        self.cols = list(zip(vals, nulls))
        self.kinds = [KIND[t] for t in types]
        self.items = items
        self.id = len(vals) - 1
        self.order = OT.topn_order(self.cols, self.kinds, items, 0, len(vals[0]))
        self.row_of_id = np.empty(len(vals[0]), np.int64)
        self.row_of_id[vals[self.id]] = np.arange(len(vals[0]))

    def check(self, rc, nrows, got, offset, count):
        assert rc == 0, abi.load_lib().tg_last_error()
        exp = self.order[offset:offset + count] if offset < len(self.order) else self.order[:0]
        assert nrows == len(exp)
        ids, id_nulls = got[self.id]
        assert not id_nulls.any() and len(np.unique(ids)) == nrows
        src = self.row_of_id[ids]
        for c, (v, nl) in enumerate(got):                        # each row is its input row, bit for bit
            iv, inl = self.cols[c][0][src], self.cols[c][1][src]
            assert np.array_equal(nl, inl), f"column {c}: NULL flags"
            assert np.array_equal(v[~nl].view(np.int64), iv[~inl].view(np.int64)), f"column {c}: values"
        gk = OT.item_keys(self.cols, self.kinds, self.items, src)
        ek = OT.item_keys(self.cols, self.kinds, self.items, exp)
        bad = np.flatnonzero((gk != ek).any(axis=1))
        assert len(bad) == 0, f"ORDER BY keys differ first at output row {bad[0]}: got row {src[bad[0]]}, expected row {exp[bad[0]]}"
        if nrows:
            # key groups wholly inside the window hold the same rows; the last group (and the first one, when the
            # window starts past row 0) may be cut by the window, and its rows are any of the tied ones
            inner = ~(ek == ek[-1]).all(axis=1)
            if offset > 0:
                inner &= ~(ek == ek[0]).all(axis=1)
            assert set(ids[inner].tolist()) == set(self.cols[self.id][0][exp[inner]].tolist())


def _run_check(vals, nulls, types, items, cases, ref=None):
    ref = ref or Ref(vals, nulls, types, items)
    for offset, count, cap in cases:
        rc, nr, got = run_topn(vals, nulls, types, items, offset, count, cap)
        ref.check(rc, nr, got, offset, count)
    return ref


def _cases(n):
    # (offset, count, output capacity or None = the rows the call can return)
    return [(0, 1, None), (0, n, None), (0, n + 10, None), (3, n + 10, None), (n, 5, 8), (n + 7, 5, 8), (5, INT64_MAX, n)]


@gpu
@pytest.mark.parametrize("n", [1, 255, 256, 257, 1_000_003])
def test_topn_shapes_types_and_limits(n):
    rng = np.random.default_rng(n)
    vals, nulls, types = make_table(rng, n)
    item_sets = ITEM_SETS if n < 1_000_000 else [ITEM_SETS[1], ITEM_SETS[4]]
    for items in item_sets:
        cases = _cases(n) if n < 1_000_000 else [(0, 1, None), (0, n, None), (5, INT64_MAX, n), (n, 5, 8), (1000, 777, None)]
        _run_check(vals, nulls, types, items, cases)


@gpu
@pytest.mark.parametrize("desc", [False, True])
def test_topn_signed_zero_is_one_value(desc):
    # ORDER BY x, y LIMIT 1 over (-0.0, 2), (+0.0, 1): the zeros tie, so y decides -> (+0.0, 1); DESC the same with the
    # zeros swapped.  A rank that separates the zeros leaves one of them out of the candidates.
    z0, z1 = (-0.0, 0.0) if not desc else (0.0, -0.0)
    x = np.array([z0, z1, -1.0, -2.0] if desc else [z0, z1, 1.0, 2.0])
    vals = [x.view(np.int64), np.array([2, 1, 3, 4], np.int64), np.arange(4, dtype=np.int64)]
    nulls = [np.zeros(4, bool)] * 3
    types = ["real", "int", "int"]
    rc, nr, got = run_topn(vals, nulls, types, [(0, desc), (1, False)], 0, 1)
    assert rc == 0 and nr == 1
    assert got[1][0].tolist() == [1] and got[0][0].view(np.uint64).tolist() == [np.float64(z1).view(np.uint64)]
    # the same at scale: many rows on each zero, ties broken by a unique second item
    rng = np.random.default_rng(3)
    n = 100_000
    x = rng.choice([-0.0, 0.0, 1.0, -1.0], n)
    vals = [x.view(np.int64), rng.permutation(n).astype(np.int64)]
    vals.append(vals[1].copy())
    nulls = [np.zeros(n, bool)] * 3
    for items in ([(0, desc), (1, False)], [(0, desc), (1, True)]):
        _run_check(vals, nulls, types, items, [(0, 10, None), (20_000, 30_000, None), (n - 5, 10, None)])


@gpu
def test_topn_time_compares_calendar_value_not_fsp_bits():
    # equal datetimes whose fsp / type bits differ are one value: the next item decides
    t = OT.pack_time(2024, 2, 29, 23, 59, 58, 999999)
    for tp in ("date", "datetime", "timestamp"):
        base = OT.pack_time(2024, 2, 29) if tp == "date" else t
        words = np.array([base | 0xF, base | 0x1, base | 0x6, base + (1 << 4)], np.uint64).view(np.int64)
        vals = [words, np.array([1, 3, 2, 0], np.int64), np.arange(4, dtype=np.int64)]
        nulls = [np.zeros(4, bool)] * 3
        for desc in (False, True):
            rc, nr, got = run_topn(vals, nulls, [tp, "int", "int"], [(0, desc), (1, False)], 0, 2)
            assert rc == 0 and nr == 2
            exp_ids = [0, 2] if not desc else [3, 0]
            assert got[2][0].tolist() == exp_ids, (tp, desc)
            assert got[0][0].tolist() == words[exp_ids].tolist()      # output keeps the fsp bits of its row
    # at scale, with the fsp bits random under a few calendar values
    rng = np.random.default_rng(11)
    n = 50_000
    vals = [_times(rng, 40, "datetime")[rng.integers(0, 40, n)], rng.integers(0, 1000, n).astype(np.int64), rng.permutation(n).astype(np.int64)]
    vals[0] = (vals[0] & ~np.int64(0xF)) | rng.integers(0, 16, n).astype(np.int64)
    nulls = [rng.random(n) < 0.05, np.zeros(n, bool), np.zeros(n, bool)]
    for items in ([(0, False), (1, True)], [(0, True), (1, False)]):
        _run_check(vals, nulls, ["datetime", "int", "int"], items, [(0, 100, None), (4000, 3000, None)])


@gpu
def test_topn_count_int64_max_with_offset():
    # offset + count overflows int64: the call returns every row past the offset into an output sized to the input
    rng = np.random.default_rng(8)
    n = 1000
    vals, nulls, types = make_table(rng, n)
    _run_check(vals, nulls, types, [(0, False), (7, True)], [(5, INT64_MAX, n), (0, INT64_MAX, n), (n - 1, INT64_MAX, 1),
                                                             (INT64_MAX, INT64_MAX, 1), (5, INT64_MAX - 4, n)])


@gpu
def test_topn_tie_group_larger_than_first_collect():
    # 2 M rows, 3 distinct first-item values: the boundary group has ~700 K rows, far past the first collect's
    # want + 65536 slots, so the candidates are collected a second time
    rng = np.random.default_rng(21)
    n = 2_000_000
    a = rng.choice(np.array([-5, 0, 7], np.int64), n, p=[0.35, 0.35, 0.3])
    b = rng.integers(INT64_MIN, INT64_MAX, n, dtype=np.int64)
    x = rng.normal(0, 1, n)
    vals = [a, b, x.view(np.int64), rng.permutation(n).astype(np.int64)]
    nulls = [rng.random(n) < 0.01, np.zeros(n, bool), rng.random(n) < 0.2, np.zeros(n, bool)]
    types = ["int", "int", "real", "int"]
    for items in ([(0, False), (1, False)], [(0, True), (2, False), (1, True)]):
        _run_check(vals, nulls, types, items, [(0, 10, None), (750_000, 100, None)])


@gpu
def test_topn_on_device_columns():
    rng = np.random.default_rng(5)
    n = 300_001
    vals, nulls, types = make_table(rng, n)
    for items in (ITEM_SETS[2], ITEM_SETS[4]):
        ref = Ref(vals, nulls, types, items)
        for offset, count in ((0, 100), (n - 50, 100), (5, INT64_MAX)):
            rc, nr, got = run_topn(vals, nulls, types, items, offset, count, on_device=True)
            ref.check(rc, nr, got, offset, count)


@gpu
def test_topn_output_capacity_and_null_bitmap_errors():
    rng = np.random.default_rng(6)
    vals, nulls, types = make_table(rng, 500)
    rc, _, _ = run_topn(vals, nulls, types, [(0, False)], 10, 100, cap=99)
    assert rc == abi.TG_ERR_CAPACITY
    # a column whose output rows are NULL needs a bitmap
    out = MutChunk([8] * len(vals), 500, [np.int64] * len(vals))
    out._cols[ALL_NULL].null_bitmap = None
    rc, _, _ = run_topn(vals, nulls, types, [(0, False)], 0, 50, out=out)
    assert rc == abi.TG_ERR_INVALID
    # ... and one with no NULLs does not
    out = MutChunk([8] * len(vals), 500, [np.int64] * len(vals))
    out._cols[ID].null_bitmap = None
    rc, nr, _ = run_topn(vals, nulls, types, [(0, False)], 0, 50, out=out)
    assert rc == 0 and nr == 50


def test_topn_gate_errors():
    # argument checks run before tg_topn looks for a device, so they hold on a machine without one
    lib = abi.load_lib()
    n = 16
    vals = [np.arange(n, dtype=np.int64), np.arange(n, dtype=np.float64).view(np.int64)]
    types = ["int", "real"]

    def call(chk, items, offset=0, count=5, tps=None):
        cs = chk.to_struct()
        out = MutChunk([8] * chk.num_cols(), n, [np.int64] * chk.num_cols())
        its = (abi.TgSortItem * max(len(items), 1))(*[abi.TgSortItem(c, d) for c, d in items])
        tps = tps or [TYPES[t][0] for t in types]
        ta = (C.c_int32 * len(tps))(*tps)
        fa = (C.c_uint32 * len(tps))(*([0] * len(tps)))
        nr = C.c_int64(0)
        return lib.tg_topn(0, 0, C.byref(cs), ta, fa, its, len(items), C.c_int64(offset), C.c_int64(count), C.byref(out.struct), C.byref(nr), None)

    chk = Chunk([Column(v) for v in vals])
    assert call(chk, []) == abi.TG_ERR_UNSUPPORTED
    assert call(chk, [(0, 0)] * 9) == abi.TG_ERR_UNSUPPORTED
    assert call(Chunk(chk.columns, np.arange(0, n, 2)), [(0, 0)]) == abi.TG_ERR_UNSUPPORTED
    assert call(Chunk([Column(vals[0]), Column(np.arange(n, dtype=np.float32))]), [(0, 0)]) == abi.TG_ERR_UNSUPPORTED
    assert call(chk, [(1, 0)], tps=[abi.TYPE_LONGLONG, abi.TYPE_VARSTRING]) == abi.TG_ERR_UNSUPPORTED
    assert call(chk, [(1, 0)], tps=[abi.TYPE_LONGLONG, abi.TYPE_NEWDECIMAL]) == abi.TG_ERR_UNSUPPORTED
    assert call(chk, [(0, 0)], offset=-1) == abi.TG_ERR_INVALID
    assert call(chk, [(0, 0)], count=-1) == abi.TG_ERR_INVALID
    assert call(chk, [(2, 0)]) == abi.TG_ERR_INVALID
