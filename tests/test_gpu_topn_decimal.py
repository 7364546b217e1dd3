"""tg_topn over DECIMAL columns (40-byte MyDecimal cells) against the exact order of tests/topn_decimal.py (oracle/topn.py
extended with DECIMAL cells), row by row.

Checked as tests/test_gpu_topn_exact.py checks 8-byte columns: the row count, the ORDER BY key sequence, every output row
equal to its input row bit for bit in every column (whole 40-byte cells: header, resultFrac and unused words included),
no id twice, and whole tie groups exact.  The DECIMAL columns hold values of several (p, s) up to (65, 30) in stored forms
that differ for equal values (digitsInt, padded fraction digits, resultFrac, garbage in the unused words, negative zeros),
with NULLs carrying garbage cells."""
import ctypes as C
import struct

import numpy as np
import pytest

import mydecimal_args as A
import test_gpu_topn_exact as T
import topn_decimal as TD
from tidb_b200 import abi
from tidb_b200.chunk import DECIMAL_DTYPE, Chunk, Column, MutChunk

pytestmark = pytest.mark.gpu
INT64_MAX = T.INT64_MAX


def dec_pool(rng, m, p, s):
    """2 * m stored cells of DECIMAL(p, s): m values (specials first), each in two random stored forms"""
    lim = 10 ** p - 1
    vals = [0, 1, -1, lim, -lim, 10 ** s, -(10 ** s)]
    for _ in range(m):
        k = int(rng.integers(0, max(p - 8, 1)))
        vals.append(int(rng.integers(-(10 ** 9), 10 ** 9)) * 10 ** k + int(rng.integers(0, 10 ** min(k, 18))))
    vals = [max(-lim, min(lim, v)) for v in vals][:max(m, 1)]
    out = []
    for v in vals:
        for _ in range(2):
            extra = int(rng.integers(0, 3)) if s + 2 <= 30 else 0       # padded fraction digits: 1.5 as 1.50
            sc = s + extra
            wf = (sc + 8) // 9
            need = len(str(abs(v) // 10 ** s)) if abs(v) >= 10 ** s else 0
            di = int(rng.choice([need, max(p - s, need), 9 * (9 - wf)]))
            c = bytearray(A.cell(v * 10 ** extra, max(di, need) + sc, sc, di, int(rng.integers(0, 31)),
                                 neg_zero=v == 0 and rng.random() < 0.5))
            for j in range((di + 8) // 9 + wf, 9):                      # words after the used ones are not looked at
                struct.pack_into("<I", c, 4 + 4 * j, int(rng.integers(0, 1 << 32)))
            out.append(bytes(c))
    return np.frombuffer(b"".join(out), np.uint8).reshape(len(out), 40)


# (name, (p, s) or None, distinct values or None = mostly distinct); the id column is appended
SCHEMA = [("dec", (15, 2), 6), ("int", None, 5), ("dec", (65, 30), None), ("real", None, 8), ("dec", (18, 0), 300),
          ("datetime", None, None), ("dec", (38, 10), 50), ("dec", (20, 5), 40), ("uint", None, None), ("dec", (9, 9), 1000)]
ALL_NULL = 7
ID = len(SCHEMA)
ITEM_SETS = [
    [(0, False)],
    [(0, True), (1, False)],
    [(1, False), (2, True)],
    [(2, False), (3, True)],
    [(4, True), (6, False), (9, True)],
    [(ALL_NULL, False), (0, True), (5, False)],
    [(3, False), (9, False), (4, True), (0, False)],
    [(6, True), (8, False), (2, False)],
]


def make_table(rng, n):
    vals, nulls, kinds, tps = [], [], [], []
    for c, (tp, ps, card) in enumerate(SCHEMA):
        if tp == "dec":
            pool = dec_pool(rng, min(card or n, 20_000), *ps)
            vals.append(pool[rng.integers(0, len(pool), n)])
            kinds.append("decimal")
            tps.append((abi.TYPE_NEWDECIMAL, 0))
        else:
            vals.append(T.gen_column(rng, tp, n, card))
            kinds.append(T.KIND[tp])
            tps.append(T.TYPES[tp])
        nl = rng.random(n) < (0.1 if c % 3 else 0.0)
        if c == ALL_NULL and n > 1:
            nl[:] = True
        if vals[-1].ndim == 2:
            vals[-1][nl] = rng.integers(0, 256, (int(nl.sum()), 40), dtype=np.uint8)   # garbage under NULL
        nulls.append(nl)
    vals.append(rng.permutation(n).astype(np.int64))
    nulls.append(np.zeros(n, bool))
    kinds.append("int")
    tps.append(T.TYPES["int"])
    return vals, nulls, kinds, tps


def run_topn(vals, nulls, tps, items, offset, count, cap=None, on_device=False, out=None):
    lib = abi.load_lib()
    cols = [Column(v, nl if nl.any() else None) for v, nl in zip(vals, nulls)]
    cs = Chunk(cols).to_struct()
    keep = []
    if on_device:
        import torch
        for i, col in enumerate(cols):
            d = torch.from_numpy(col.data.copy()).cuda()
            keep.append(d)
            cs.cols[i].data = d.data_ptr()
            if col.null_bitmap is not None:
                b = torch.from_numpy(col.null_bitmap.copy()).cuda()
                keep.append(b)
                cs.cols[i].null_bitmap = b.data_ptr()
    n = len(vals[0])
    if out is None:
        el = [c.elem_len for c in cols]
        out = MutChunk(el, cap if cap is not None else max(min(count, max(n - offset, 0)), 1), [DECIMAL_DTYPE if e == 40 else np.int64 for e in el])
    its = (abi.TgSortItem * len(items))(*[abi.TgSortItem(c, int(d)) for c, d in items])
    ta = (C.c_int32 * len(tps))(*[t for t, _ in tps])
    fa = (C.c_uint32 * len(tps))(*[f for _, f in tps])
    nr = C.c_int64(-1)
    rc = lib.tg_topn(0, int(on_device), C.byref(cs), ta, fa, its, len(items), C.c_int64(offset), C.c_int64(count),
                     C.byref(out.struct), C.byref(nr), None)
    if on_device:
        import torch
        torch.cuda.synchronize()
    return rc, nr.value, (out.columns(nr.value) if rc == 0 else None)


class Ref:
    """the reference order of one table under one ORDER BY, and its keys for every row (DECIMAL keys are dense ranks over
    the whole column, so they are computed once).  The last column is the id: a permutation of 0..n-1."""

    def __init__(self, vals, nulls, kinds, items):
        n = len(vals[0])
        self.cols = list(zip(vals, nulls))
        self.items = items
        self.id = len(vals) - 1
        self.order = TD.topn_order(self.cols, kinds, items, 0, n)
        self.keys = TD.item_keys(self.cols, kinds, items, np.arange(n))
        self.row_of_id = np.empty(n, np.int64)
        self.row_of_id[vals[self.id]] = np.arange(n)

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
            bits = (lambda x: x) if v.ndim == 2 else (lambda x: x.view(np.int64))   # DOUBLE: the bits, NaN payloads included
            assert np.array_equal(bits(v[~nl]), bits(iv[~inl])), f"column {c}: values"
            if v.ndim == 2:
                assert not v[nl].any(), f"column {c}: a NULL cell is 40 zero bytes"
        gk, ek = self.keys[src], self.keys[exp]
        bad = np.flatnonzero((gk != ek).any(axis=1))
        assert len(bad) == 0, f"ORDER BY keys differ first at output row {bad[0]}: got row {src[bad[0]]}, expected row {exp[bad[0]]}"
        if nrows:
            inner = ~(ek == ek[-1]).all(axis=1)
            if offset > 0:
                inner &= ~(ek == ek[0]).all(axis=1)
            assert set(ids[inner].tolist()) == set(self.cols[self.id][0][exp[inner]].tolist())


@pytest.mark.parametrize("n", [1, 255, 257, 1_000_003])
def test_topn_decimal_shapes_and_limits(n):
    rng = np.random.default_rng(100 + n)
    vals, nulls, kinds, tps = make_table(rng, n)
    big = n >= 1_000_000
    for k, items in enumerate(ITEM_SETS if not big else [ITEM_SETS[1], ITEM_SETS[4], ITEM_SETS[7]]):
        ref = Ref(vals, nulls, kinds, items)
        cases = T._cases(n) if not big else [(0, 1, None), (0, n, None), (5, INT64_MAX, n), (n, 5, 8), (1000, 777, None)]
        for offset, count, cap in cases:
            ref.check(*run_topn(vals, nulls, tps, items, offset, count, cap), offset, count)
        # the same calls on device-resident columns
        for offset, count, cap in (cases[:2] if not big else cases[:1] + cases[-1:]) if k % 2 == 0 else ():
            ref.check(*run_topn(vals, nulls, tps, items, offset, count, cap, on_device=True), offset, count)


def test_topn_decimal_rank_ties_past_16_digits():
    # 2 M rows of DECIMAL(30, 10) whose values share their first 20 significant digits (positive and negative): the rank
    # ties on each sign, the candidates overflow the first collect and are collected a second time, and the host
    # comparator orders them
    rng = np.random.default_rng(31)
    n = 2_000_000
    r = rng.integers(0, 10 ** 10, n)
    neg = rng.random(n) < 0.5
    w = np.zeros((n, 10), np.int64)
    w[:, 0] = 27 | (10 << 8) | (neg.astype(np.int64) << 24)            # digitsInt 27: 3 integer words, 2 fraction words
    w[:, 1], w[:, 2], w[:, 3] = 12, 345678901, 234567890              # integer part 12345678901234567890
    fr = r * 10 ** 8                                                   # 10 fraction digits, left-aligned in 2 words
    w[:, 4], w[:, 5] = fr // 10 ** 9, fr % 10 ** 9
    cells = w.astype(np.int32).view(np.uint8).reshape(n, 40)
    second = rng.integers(-5, 5, n).astype(np.int64)
    vals = [cells, second, rng.permutation(n).astype(np.int64)]
    nulls = [rng.random(n) < 0.01, np.zeros(n, bool), np.zeros(n, bool)]
    kinds = ["decimal", "int", "int"]
    tps = [(abi.TYPE_NEWDECIMAL, 0), T.TYPES["int"], T.TYPES["int"]]
    for items in ([(0, False), (1, True)], [(0, True), (1, False)]):
        ref = Ref(vals, nulls, kinds, items)
        for offset, count in ((0, 10), (999_000, 2_000)):
            ref.check(*run_topn(vals, nulls, tps, items, offset, count), offset, count)


def test_topn_decimal_malformed_cells():
    rng = np.random.default_rng(41)
    n = 5000
    vals, nulls, kinds, tps = make_table(rng, n)
    good = Ref(vals, nulls, kinds, [(0, False), (4, True)])
    bad_cells = {"digitsInt < 0": struct.pack("<bbbB9i", -1, 2, 2, 0, *([0] * 9)),
                 "digitsFrac < 0": struct.pack("<bbbB9i", 9, -3, 0, 0, *([1] + [0] * 8)),
                 "10 words": struct.pack("<bbbB9i", 54, 36, 0, 0, *([1] * 9)),
                 "word >= 10^9": struct.pack("<bbbB9I", 18, 0, 0, 0, *([5, 1_000_000_000] + [0] * 7)),
                 "negative word": struct.pack("<bbbB9i", 9, 9, 0, 1, *([7, -4] + [0] * 7))}
    row = int(np.flatnonzero(~nulls[4])[-1])
    for col, items in ((0, [(0, False), (4, True)]), (4, [(0, False), (4, True)]), (4, [(1, False), (2, False), (4, True)])):
        for why, cell in bad_cells.items():
            v = [x.copy() for x in vals]
            r = row if col == 4 else int(np.flatnonzero(~nulls[col])[0])
            v[col][r] = np.frombuffer(cell, np.uint8)
            for offset, count in ((0, 10), (n, 5), (0, 0)):
                out = MutChunk([x.shape[1] if x.ndim == 2 else 8 for x in v], 10, [DECIMAL_DTYPE if x.ndim == 2 else np.int64 for x in v])
                rc, nr, _ = run_topn(v, nulls, tps, items, offset, count, out=out)
                assert rc == abi.TG_ERR_INVALID and nr == 0, (col, why, offset, count)
                assert not any(d.any() for d in out.data), "the output is not written"
    # a malformed cell in a payload column, or under NULL, is never interpreted
    v = [x.copy() for x in vals]
    v[2][0] = np.frombuffer(bad_cells["10 words"], np.uint8)
    v[4][np.flatnonzero(nulls[4])[0]] = np.frombuffer(bad_cells["word >= 10^9"], np.uint8)
    good.cols[2] = (v[2], nulls[2])
    good.check(*run_topn(v, nulls, tps, [(0, False), (4, True)], 0, 100), 0, 100)


def test_topn_decimal_output_column_width():
    rng = np.random.default_rng(42)
    vals, nulls, kinds, tps = make_table(rng, 300)
    el = [x.shape[1] if x.ndim == 2 else 8 for x in vals]
    el[6] = 8
    out = MutChunk(el, 300, [DECIMAL_DTYPE if e == 40 else np.int64 for e in el])
    rc, nr, _ = run_topn(vals, nulls, tps, [(1, False)], 0, 20, out=out)
    assert rc == abi.TG_ERR_INVALID and nr == 0


def test_topn_exec_decimal_schema():
    from tidb_b200.executor import MockDataSource, TopNExec, drain
    from tidb_b200.plan import FieldType
    rng = np.random.default_rng(43)
    n = 20_000
    vals, nulls, kinds, tps = make_table(rng, n)
    schema = [FieldType(t, f) for t, f in tps]
    items = [(2, True), (0, False), (1, False)]
    chunks = Chunk([Column(v, nl if nl.any() else None) for v, nl in zip(vals, nulls)]).split(1024)
    ref = Ref(vals, nulls, kinds, items)
    for offset, count in ((0, 50), (19_990, 100), (7, 3000)):
        out = drain(TopNExec(MockDataSource(schema, chunks), items, offset, count), 1024)
        got = [(np.concatenate([c.columns[k].data for c in out]), np.concatenate([c.columns[k].nulls() for c in out])) for k in range(len(schema))]
        ref.check(0, len(got[0][0]), got, offset, count)
