"""The Python chunk layer over var-length columns (tidb_b200/chunk.py): Column.take, Column.slice and concat_columns with
offsets that do not start at 0, NULL rows that own bytes and empty columns, and MutChunk.column of var-length outputs,
each against plain lists of bytes.  Then one end-to-end SelectionExec -> HashAggExec over strings on the GPU."""
import numpy as np
import pytest

from tidb_b200 import abi
from tidb_b200.chunk import VARLEN, Chunk, Column, MutChunk, concat_columns


def view_column(rows, nulls, lead=0, tail=0):
    """rows (bytes; NULL rows keep theirs) in a buffer with `lead` junk bytes ahead and `tail` after: offsets[0] == lead"""
    offs = np.full(len(rows) + 1, lead, np.int64)
    np.cumsum([len(r) for r in rows], out=offs[1:])
    offs[1:] += lead
    data = np.frombuffer(b"J" * lead + b"".join(rows) + b"T" * tail, np.uint8).copy()
    return Column(data, np.asarray(nulls, bool) if any(nulls) else None, offs)


def listed(c):
    """(row bytes, null) per row, read straight from offsets and data"""
    nl = c.nulls()
    return [(c.data[c.offsets[i]:c.offsets[i + 1]].tobytes(), bool(nl[i])) for i in range(c.length)]


ROWS = [b"", b"abc", "é".encode(), b"\xff\x00", b"   ", b"x" * 40, b"", b"owned", b"z"]
NULLS = [False, False, True, False, False, True, True, True, False]   # NULL rows 2, 5 and 7 own bytes


@pytest.mark.parametrize("lead", [0, 1, 13])
def test_take(lead):
    c = view_column(ROWS, NULLS, lead, tail=5)
    expect = list(zip(ROWS, NULLS))
    assert listed(c) == expect and c.values() == [None if z else r for r, z in expect]
    for idx in ([], [0], [8, 0, 8], [2, 5, 7], list(range(9))[::-1], [3, 3, 3, 6]):
        t = c.take(np.array(idx, np.int64))
        assert t.offsets[0] == 0 and t.length == len(idx)
        assert listed(t) == [expect[i] for i in idx]
        assert t.data.size == sum(len(ROWS[i]) for i in idx)   # a NULL row keeps its bytes through take


@pytest.mark.parametrize("lead", [0, 7])
def test_slice(lead):
    c = view_column(ROWS, NULLS, lead, tail=3)
    expect = list(zip(ROWS, NULLS))
    for lo, hi in ((0, 9), (0, 0), (4, 4), (2, 6), (8, 9), (1, 2), (6, 8)):
        s = c.slice(lo, hi)
        assert s.offsets[0] == 0 and s.length == hi - lo
        assert listed(s) == expect[lo:hi]
        assert s.data.size == sum(len(r) for r in ROWS[lo:hi])


def test_concat_columns():
    a = view_column(ROWS[:4], NULLS[:4], lead=3, tail=2)
    b = view_column(ROWS[4:], NULLS[4:], lead=11)
    e = view_column([], [], lead=5)
    no_nulls = view_column([b"p", b"", b"q"], [False] * 3, lead=2)
    assert e.length == 0 and listed(e) == []
    for parts in ([a, b], [e, a, e, b, e], [b, no_nulls, a], [e], [e, e], [no_nulls]):
        got = concat_columns(parts)
        want = [x for p in parts for x in listed(p)]
        assert got.offsets[0] == 0 and listed(got) == want
        assert (got.null_bitmap is None) == (not any(z for _, z in want))


def test_mut_chunk_varlen_column():
    m = MutChunk([VARLEN, 8], 6, [np.uint8, np.int64], data_cap=32)
    rows = [b"ab", b"", b"cde", b"zz", b"", b"q"]
    nulls = [False, True, False, True, False, False]
    o = np.zeros(7, np.int64)
    np.cumsum([len(r) for r in rows], out=o[1:])
    m.offsets[0][:7] = o
    m.data[0][:o[-1]] = np.frombuffer(b"".join(rows), np.uint8)
    m.data[0][o[-1]:] = 0xEE
    m.bitmaps[0][:] = np.packbits(~np.array(nulls + [False, False]), bitorder="little")
    m.data[1][:6] = np.arange(6)
    for n in (0, 1, 4, 6):
        c = m.column(0, n)
        assert c.is_varlen and c.elem_len == VARLEN and c.length == n and c.data.size == o[n]
        assert c.values() == [None if z else r for r, z in zip(rows[:n], nulls[:n])]
        assert listed(c) == list(zip(rows[:n], nulls[:n]))
        f = m.column(1, n)
        assert not f.is_varlen and f.data.tolist() == list(range(n))
    vals = m.columns(6)[0][0]
    assert list(vals) == [None if z else r for r, z in zip(rows, nulls)]


@pytest.mark.gpu
@pytest.mark.parametrize("required_rows", [1, 7, 1024])
def test_selection_then_string_group_by(required_rows):
    from tidb_b200.executor import HashAggExec, MockDataSource, SelectionExec, drain
    from tidb_b200.plan import AggFunc, AggPlan, FieldType, FilterItem
    rng = np.random.default_rng(required_rows)
    n = 20_000
    pool = [b"AIR", b"AIR ", b"MAIL", b"MAIL  ", "é".encode(), "é ".encode(), b"", b" ", b"special requests", b"x\xff"]
    s = [pool[i] for i in rng.integers(0, len(pool), n)]
    sn = rng.random(n) < 0.05
    v = rng.integers(0, 100, n).astype(np.int64)
    col = view_column(s, sn, lead=0)
    chunks = []
    for lo in range(0, n, 1000):
        hi = min(n, lo + 1000)
        part = Chunk([col.slice(lo, hi), Column(v[lo:hi])])
        sel = np.sort(rng.choice(hi - lo, (hi - lo) * 2 // 3, replace=False)).astype(np.int64)
        chunks.append(Chunk(part.columns, sel))
    schema = [FieldType(abi.TYPE_VARCHAR, 0, collation=46), FieldType(abi.TYPE_LONGLONG, 0)]
    items = [FilterItem(abi.CMP_EQ, 0, is_string=True, str_kind=abi.STR_NOT_LIKE, const_bytes=b"%special%", collation=46),
             FilterItem(abi.CMP_LT, 1, const_i64=80)]
    plan = AggPlan(schema, [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_MAX, 1)])
    out = drain(HashAggExec(plan, SelectionExec(MockDataSource(schema, chunks), items)), required_rows)
    assert all(c.num_rows() <= required_rows for c in out)
    got = {}
    for c in out:
        for f, cnt, mx in zip(c.columns[0].values(), c.columns[1].data.tolist(), c.columns[2].data.tolist()):
            k = None if f is None else f.rstrip(b" ")
            assert k not in got
            got[k] = (f, cnt, mx)
    # pure Python: the rows each chunk's sel keeps, in order, then the filter, then the groups
    want = {}
    for lo, ch in zip(range(0, n, 1000), chunks):
        for r in ch.sel:
            i = lo + int(r)
            if sn[i] or b"special" in s[i] or v[i] >= 80:
                continue
            k = s[i].rstrip(b" ")
            f, cnt, mx = want.get(k, (s[i], 0, -1))
            want[k] = (f, cnt + 1, max(mx, int(v[i])))
    assert got == want
