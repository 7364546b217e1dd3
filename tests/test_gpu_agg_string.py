"""GROUP BY over string columns on the GPU, against the exact reference of agg_string_reference.py: the six offloaded
collations, every update path, FIRSTROW's earliest row, host and device pushes, dictionary growth, long rows, mixed
plans, rejected pushes and the var-length result calls.  Where a test names a path, tg_agg_stats.paths proves it ran."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

import agg_string_reference as S
import mydecimal as D
from tidb_b200 import abi
from tidb_b200.chunk import VARLEN, Chunk, Column, MutChunk, unpack_nulls
from tidb_b200.executor import HashAggExec, MockDataSource, SelectionExec, drain
from tidb_b200.plan import AggFunc, AggPlan, FieldType, FilterItem

pytestmark = pytest.mark.gpu

INT = FieldType(abi.TYPE_LONGLONG, 0)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
COLLATIONS = (63, 46, 83, 65, 47, 309)
MIXED = [b"", b" ", b"a", b"a ", b"a\t", None, b"\xff\xfe", b"a\xc3", "é".encode(), "é ".encode(), "中文".encode(), b"\xf0\x9f\x98\x80",
         b"a  ", b"  ", b"b", None]


def st(coll=46, flag=0):
    return FieldType(abi.TYPE_VARCHAR, flag, collation=coll)


def fr(c):
    return AggFunc(abi.AGG_FIRSTROW, c)


@pytest.fixture(scope="module")
def lib():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return abi.load_lib()


def rows_of(chunks):
    out = []
    for ch in chunks:
        cols = []
        for c in ch.columns:
            if c.is_varlen:
                cols.append(c.values())
            else:
                nl = c.nulls()
                cols.append([None if nl[i] else c.data[i].item() if c.data.ndim == 1 else bytes(c.data[i]) for i in range(c.length)])
        out.extend(zip(*cols))
    return out


def drain_keep(e, required=1024):
    """drain() without close, so stats can still be read; the caller closes"""
    e.open()
    out = []
    while True:
        c = e.next(required)
        if c.num_rows() == 0:
            return out
        out.append(c)


def stats_run(plan, chunks, required=1024):
    e = HashAggExec(plan, MockDataSource(plan.col_types, chunks))
    try:
        got = rows_of(drain_keep(e, required))
        return got, e.stats(), e.string_stats()
    finally:
        e.close()


def rand_strings(rng, n, pool):
    idx = rng.integers(0, len(pool), n)
    return [pool[i] for i in idx]


# ---- collations, update paths ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("coll", COLLATIONS)
def test_collations(lib, coll):
    rng = np.random.default_rng(coll)
    n = 20000
    vals = rand_strings(rng, n, MIXED)
    x = np.floor(rng.random(n) * 100)
    plan = AggPlan([st(coll), DBL], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_COUNT, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE)])
    chunks = Chunk([Column.strings(vals), Column(x)]).split(1024)
    got, stats, ss = stats_run(plan, chunks)
    groups = S.check(plan, chunks, got)
    distinct = {S.collation_key(v, coll) for v in MIXED}
    assert groups == len(distinct)
    assert stats.paths & abi.AGG_PATH_STRING_KEY and ss.dict_entries == len(distinct - {None})


@pytest.mark.parametrize("variant,env,bit", [("v2_global", {"TG_AGG_LOCAL": "0"}, abi.AGG_PATH_V2_GLOBAL),
                                             ("v2_local", {"TG_AGG_LOCAL": "2"}, abi.AGG_PATH_V2_LOCAL),
                                             ("v1", {"TG_AGG_V1": "1"}, abi.AGG_PATH_V1_GLOBAL | abi.AGG_PATH_V1_LOCAL)])
def test_update_paths(lib, monkeypatch, variant, env, bit):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(7)
    n = 200000
    pool = [f"key-{i:05d}".encode() + b" " * (i % 3) for i in range(3000)] + [None]
    vals = rand_strings(rng, n, pool)
    x = np.floor(rng.random(n) * 1000)
    plan = AggPlan([st(46), DBL], [0], [fr(0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 0)])
    chunks = Chunk([Column.strings(vals), Column(x)]).split(1024)
    got, stats, _ = stats_run(plan, chunks)
    S.check(plan, chunks, got)
    assert stats.paths & bit and stats.paths & abi.AGG_PATH_STRING_KEY, (variant, stats.paths)


@pytest.mark.parametrize("shape", ["s_i", "i_s_d", "s_s_i_d"])
def test_multi_key(lib, shape):
    rng = np.random.default_rng(len(shape))
    n = 100000
    pool = [b"AIR", b"AIR ", b"MAIL", b"MAIL  ", b"SHIP", b"TRUCK", b"RAIL", b"FOB", b"REG AIR", b"", b" ", None]
    mk = {"s": lambda i: (st((46, 309, 83, 63)[i % 4]), Column.strings(rand_strings(rng, n, pool))),
          "i": lambda i: (INT, Column(rng.integers(0, 7, n).astype(np.int64), rng.random(n) < 0.05)),
          "d": lambda i: (DBL, Column(rng.integers(-2, 3, n).astype(np.float64) * 0.5))}
    parts = [mk[k](i) for i, k in enumerate(shape.split("_"))]
    types = [t for t, _ in parts] + [DBL]
    cols = [c for _, c in parts] + [Column(np.floor(rng.random(n) * 10))]
    g = list(range(len(parts)))
    plan = AggPlan(types, g, [fr(i) for i in g] + [AggFunc(abi.AGG_SUM, len(parts), abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, -1)])
    chunks = Chunk(cols).split(1024)
    got, stats, _ = stats_run(plan, chunks)
    S.check(plan, chunks, got)
    assert stats.paths & abi.AGG_PATH_MULTI_KEY and stats.paths & abi.AGG_PATH_STRING_KEY


# ---- FIRSTROW's earliest row -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("coll", (46, 83, 65, 47))
def test_firstrow_earliest(lib, coll):
    plan = AggPlan([st(coll), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)])
    # chunk 1: the earliest variant of "k" is physically last but first in sel order
    vals1 = [b"k", b"k ", b"z", b"k  "] * 300 + [b"k   "]
    sel1 = np.array([len(vals1) - 1] + list(range(len(vals1) - 1)), dtype=np.int64)
    c1 = Chunk([Column.strings(vals1), Column(np.arange(len(vals1), dtype=np.int64))], sel=sel1)
    # chunk 2 brings other variants of "k" and the first "q "; chunk 3 an earlier-pushed-wins case for "q"
    c2 = Chunk([Column.strings([b"k", b"q ", b"k "]), Column(np.zeros(3, dtype=np.int64))])
    c3 = Chunk([Column.strings([b"q", b"q  "] * 2000), Column(np.zeros(4000, dtype=np.int64))])
    got, _, _ = stats_run(plan, [c1, c2, c3])
    S.check(plan, [c1, c2, c3], got)
    d = {r[0].rstrip(b" "): r for r in got}
    assert d[b"k"][0] == b"k   " and d[b"q"][0] == b"q "


@pytest.mark.parametrize("coll", (46, 83, 65, 47))
def test_firstrow_earliest_per_group_multi_key(lib, coll):
    # under a PAD collation the earliest variant of one key differs between the groups it is part of: group (k, 1)
    # starts with "k  " (first in sel order of the first chunk), group (k, 2) with "k", group (k, 3) with "k " from the
    # second push, and a later push's variants never win
    plan = AggPlan([st(coll), INT, st(coll)], [0, 1, 2], [fr(0), fr(1), AggFunc(abi.AGG_COUNT, -1), fr(2)])
    vals1 = [b"k", b"k ", b"k  "] * 500 + [b"k  "]
    g1 = [2, 1, 2] * 500 + [1]
    t1 = [b"x", b"x ", b"y"] * 500 + [b"x  "]
    sel1 = np.array([len(vals1) - 1] + list(range(len(vals1) - 1)), dtype=np.int64)
    c1 = Chunk([Column.strings(vals1), Column(np.array(g1, np.int64)), Column.strings(t1)], sel=sel1)
    c2 = Chunk([Column.strings([b"k ", b"k", b"k   "] * 700), Column(np.array([3, 1, 2] * 700, np.int64)),
                Column.strings([b"y ", b"x", b"x"] * 700)])
    got, stats, _ = stats_run(plan, [c1, c2])
    S.check(plan, [c1, c2], got)
    assert stats.paths & abi.AGG_PATH_MULTI_KEY
    d = {(r[0].rstrip(b" "), r[1], r[3].rstrip(b" ")): (r[0], r[3]) for r in got}
    assert d[(b"k", 1, b"x")] == (b"k  ", b"x  ") and d[(b"k", 2, b"x")] == (b"k", b"x") and d[(b"k", 3, b"y")] == (b"k ", b"y ")
    # the same through device pushes, with offsets that do not start at 0 and a dictionary that grows
    import torch
    from tidb_b200.device import DeviceAgg
    rng = np.random.default_rng(coll)
    dplan = AggPlan([st(coll), INT], [0, 1], [fr(0), fr(1), AggFunc(abi.AGG_COUNT, -1)], expected_groups=1)
    dev = DeviceAgg(dplan)
    chunks = []
    for k in range(3):
        n = 40000
        ids = rng.integers(0, 3000, n)
        vals = [b"key%d" % i + b" " * int(j) for i, j in zip(ids, rng.integers(0, 4, n))]
        gv = rng.integers(0, 5, n).astype(np.int64)
        (offs, data), c = _dev_string(vals, pad=3 + k)
        dev.push([(offs, data), torch.from_numpy(gv).cuda()])
        chunks.append(Chunk([c, Column(gv)]))
    rows, cols, nulls = dev.finish()
    S.check(dplan, chunks, fetch_result(dev, dplan, rows, cols, nulls))
    assert dev.string_stats().dict_grows > 0
    dev.close()


# ---- push routes -----------------------------------------------------------------------------------------------------
def test_host_pushes_across_staging_flushes(lib):
    # about 4.7 M rows in chunks of up to 1536 rows, most with sel vectors: more than one staging batch (4 M rows)
    rng = np.random.default_rng(11)
    pool = [f"s{i}".encode() + b" " * (i % 2) for i in range(500)] + [None, b""]
    base = rand_strings(rng, 1536, pool)
    col = Column.strings(base)
    chunks = []
    for k in range(3500):
        sel = np.sort(rng.choice(1536, 1536 - (k % 7) * 100, replace=False)).astype(np.int64) if k % 3 else None
        chunks.append(Chunk([col, Column(np.full(1536, k % 5, dtype=np.int64))], sel=sel))
    plan = AggPlan([st(46), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_MAX, 1)])
    got, stats, _ = stats_run(plan, chunks)
    S.check(plan, chunks, got)
    assert stats.input_rows > 4 << 20


def _dev_string(vals, pad=0):
    """(offsets, bytes) CUDA tensors of a string column, its offsets starting at `pad` (junk bytes before row 0)"""
    import torch
    c = Column.strings(vals)
    data = np.concatenate([np.full(pad, 0x58, np.uint8), c.data, np.zeros(1, np.uint8)])
    return (torch.from_numpy(c.offsets + pad).cuda(), torch.from_numpy(data).cuda()), c


def _dev_nulls(c):
    import torch
    return torch.from_numpy(c.null_bitmap.copy()).cuda() if c.null_bitmap is not None else None


def fetch_result(dev, plan, rows, cols, nulls):
    from tidb_b200.device import fetch_device
    out = []
    for k, (p, nb) in enumerate(zip(cols, nulls)):
        nl = unpack_nulls(fetch_device(nb, (rows + 7) // 8), rows) if nb else np.zeros(rows, bool)
        if dev.offsets[k]:
            o = fetch_device(dev.offsets[k], (rows + 1) * 8).view(np.int64)
            assert o[0] == 0 and np.all(np.diff(o) >= 0)
            b = fetch_device(p, int(o[-1]))
            out.append([None if nl[r] else b[o[r]:o[r + 1]].tobytes() for r in range(rows)])
        else:
            v = fetch_device(p, rows * 8).view(np.float64 if plan.funcs[k].name == abi.AGG_SUM else np.int64)
            out.append([None if nl[r] else v[r].item() for r in range(rows)])
    return list(zip(*out))


def test_device_pushes(lib):
    import torch
    from tidb_b200.device import DeviceAgg
    rng = np.random.default_rng(3)
    plan = AggPlan([st(63), INT, DBL], [0, 1], [fr(0), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE), fr(1)])
    dev = DeviceAgg(plan)
    chunks = []
    for k in range(4):
        n = 50000 + k
        vals = rand_strings(rng, n, MIXED)
        (offs, data), c = _dev_string(vals, pad=5 + k)
        iv = rng.integers(0, 3, n).astype(np.int64)
        x = np.floor(rng.random(n) * 10)
        dev.push([(offs, data), torch.from_numpy(iv).cuda(), torch.from_numpy(x).cuda()], [_dev_nulls(c), None, None])
        chunks.append(Chunk([c, Column(iv), Column(x)]))
    rows, cols, nulls = dev.finish()
    got = fetch_result(dev, plan, rows, cols, nulls)
    S.check(plan, chunks, got)
    assert dev.stats().paths & abi.AGG_PATH_STRING_KEY
    # a plan with a string result refuses tg_agg_result_dev
    r = C.c_int64(-7)
    assert lib.tg_agg_result_dev(dev.h, C.byref(r), None, None) == abi.TG_ERR_INVALID and r.value == -7
    dev.close()


# ---- growth, long rows, contention ----------------------------------------------------------------------------------
def test_growth_over_pushes(lib):
    import torch
    from tidb_b200.device import DeviceAgg
    rng = np.random.default_rng(5)
    # expected_groups = 1: the first dictionary and group table have 1024 slots, and each push brings 4x the keys of
    # the one before, some of them seen in earlier pushes
    plan = AggPlan([st(46), DBL], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE)], expected_groups=1)
    dev = DeviceAgg(plan)
    chunks = []
    for k in range(6):
        n = 500 * 4 ** k
        keys = [b"grow-%d" % i + b" " * (i % 3) for i in rng.integers(0, n, n)]
        (offs, data), c = _dev_string(keys, pad=k)
        x = np.ones(n)
        dev.push([(offs, data), torch.from_numpy(x).cuda()])
        chunks.append(Chunk([c, Column(x)]))
    rows, cols, nulls = dev.finish()
    got = fetch_result(dev, plan, rows, cols, nulls)
    S.check(plan, chunks, got)
    ss = dev.string_stats()
    assert ss.dict_grows > 0 and ss.dict_entries == rows and dev.stats().table_slots > 2048
    dev.close()


def test_growth_device_millions(lib):
    import torch
    from tidb_b200.device import DeviceAgg
    rng = np.random.default_rng(9)
    plan = AggPlan([st(309), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_MAX, 1)])
    dev = DeviceAgg(plan)
    want = {}
    for k in range(3):   # 3 pushes, up to 1.5 M distinct keys of 20 bytes
        n = 10000 if k == 0 else 1_000_000
        ids = rng.integers(0, 1_500_000, n)
        keys = [b"Customer#%011d" % i for i in ids]
        (offs, data), c = _dev_string(keys)
        v = rng.integers(0, 1 << 40, n).astype(np.int64)
        dev.push([(offs, data), torch.from_numpy(v).cuda()])
        for i, x in zip(ids.tolist(), v.tolist()):
            cnt, mx = want.get(i, (0, -1))
            want[i] = (cnt + 1, max(mx, x))
    rows, cols, nulls = dev.finish()
    got = fetch_result(dev, plan, rows, cols, nulls)
    ss = dev.string_stats()
    assert ss.dict_grows > 0 and ss.dict_entries == len(want) == rows
    for key, cnt, mx in got:
        assert want[int(key[9:])] == (cnt, mx)
    dev.close()


def test_long_rows_and_contention(lib):
    import torch
    from tidb_b200.device import DeviceAgg
    rng = np.random.default_rng(13)
    # rows longer than 2 KiB, a few variants each
    longs = [bytes([65 + j]) * (2048 + 700 * j) + b" " * (j % 2) for j in range(5)]
    vals = rand_strings(rng, 5000, longs + [None, b"short"])
    plan = AggPlan([st(46), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)])
    got, _, _ = stats_run(plan, [Chunk([Column.strings(vals), Column(np.zeros(5000, np.int64))])])
    S.check(plan, [Chunk([Column.strings(vals), Column(np.zeros(5000, np.int64))])], got)
    # 3 groups over 4 M rows, one device push
    n = 4 << 20
    pick = rng.integers(0, 3, n)
    lens = np.array([1, 2, 1])[pick]
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    table = [b"R", b"N ", b"A"]
    data = np.frombuffer(b"".join(table[i] for i in range(3)), np.uint8)
    starts = np.array([0, 1, 3])[pick]
    byts = np.empty(int(offs[-1]), np.uint8)
    pos = np.repeat(starts - offs[:-1], lens) + np.arange(int(offs[-1]))
    byts[:] = data[pos]
    dev = DeviceAgg(AggPlan([st(46), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)]))
    dev.push([(torch.from_numpy(offs).cuda(), torch.from_numpy(byts).cuda()), torch.zeros(n, dtype=torch.int64, device="cuda")])
    rows, cols, nulls = dev.finish()
    res = dict(fetch_result(dev, dev.plan, rows, cols, nulls))
    assert res == {b"R": int((pick == 0).sum()), b"N ": int((pick == 1).sum()), b"A": int((pick == 2).sum())}
    dev.close()


# ---- mixed plans -----------------------------------------------------------------------------------------------------
def test_q16_shape_count_distinct(lib):
    rng = np.random.default_rng(16)
    n = 300000
    brands = [b"Brand#%d%d" % (a, b) for a in range(1, 6) for b in range(1, 6)]
    types = [(t1 + b" " + t2 + b" " + t3).ljust(25) for t1 in (b"STANDARD", b"SMALL", b"MEDIUM") for t2 in (b"ANODIZED", b"BURNISHED")
             for t3 in (b"TIN", b"NICKEL", b"BRASS", b"STEEL")]
    plan = AggPlan([st(46), st(46), INT, INT], [0, 1, 2],
                   [fr(0), fr(1), fr(2), AggFunc(abi.AGG_COUNT, 3, distinct=True)])
    cols = [Column.strings(rand_strings(rng, n, brands)), Column.strings(rand_strings(rng, n, types)),
            Column(rng.choice([1, 9, 14, 23, 45], n).astype(np.int64)), Column(rng.integers(0, 2000, n).astype(np.int64))]
    chunks = Chunk(cols).split(1024)
    e = HashAggExec(plan, MockDataSource(plan.col_types, chunks))
    try:
        got = rows_of(drain_keep(e))
        assert e.distinct_stats().pairs > 0
    finally:
        e.close()
    import agg_distinct_reference  # noqa: F401  (same rule: distinct values per group)
    exp = {}
    v = [c.values() if c.is_varlen else c.data.tolist() for c in cols]
    for i in range(n):
        exp.setdefault((v[0][i], v[1][i], v[2][i]), set()).add(v[3][i])
    assert {(a, b, c): d for a, b, c, d in got} == {k: len(s) for k, s in exp.items()}


def test_q1_shape_through_selection(lib):
    rng = np.random.default_rng(1)
    n = 200000
    flag = rand_strings(rng, n, [b"A", b"N", b"R", b"A ", b"R "])   # CHAR(1) under utf8mb4_bin, with PAD variants
    status = rand_strings(rng, n, [b"F", b"O", b"O "])
    qty = rng.integers(100, 5000, n)                      # DECIMAL(15, 2) quantities
    ship = rng.integers(0, 2500, n).astype(np.int64)
    DEC = FieldType(abi.TYPE_NEWDECIMAL, abi.FLAG_NOT_NULL, 15, 2)
    cells = np.frombuffer(b"".join(D.encode(Fraction(int(q), 100), 2) for q in qty), np.uint8).reshape(n, 40)
    types = [st(46), st(46), DEC, INT]
    plan = AggPlan(types, [0, 1], [fr(0), fr(1), AggFunc(abi.AGG_SUM, 2, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=2),
                                   AggFunc(abi.AGG_AVG, 2, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=6), AggFunc(abi.AGG_COUNT, -1)])
    chunks = Chunk([Column.strings(flag), Column.strings(status), Column(cells), Column(ship)]).split(1024)
    sel = SelectionExec(MockDataSource(types, chunks), [FilterItem(abi.CMP_LE, 3, const_i64=2000)])
    e = HashAggExec(plan, sel)
    got = rows_of(drain(e))
    keep = ship <= 2000
    assert len(got) == 6
    fk = np.array([a.rstrip(b" ") for a in flag], dtype=object)
    sk = np.array([b.rstrip(b" ") for b in status], dtype=object)
    for f, s_, sm, av, cnt in got:
        m = keep & (fk == f.rstrip(b" ")) & (sk == s_.rstrip(b" "))
        first = int(np.flatnonzero(m)[0])   # FIRSTROW: the raw bytes of the group's earliest selected row
        assert (f, s_) == (flag[first], status[first])
        tot = int(qty[m].sum())
        assert cnt == int(m.sum()) and D.value(sm) == Fraction(tot, 100)
        assert abs(D.value(av) - Fraction(tot, 100 * cnt)) <= Fraction(1, 10 ** 6)


# ---- rejected pushes, result calls ---------------------------------------------------------------------------------
def _open(lib, plan):
    d, keep = plan.to_struct_ex3()
    h = C.c_void_p()
    abi.check(lib.tg_agg_open_ex3(C.byref(d), C.byref(h)))
    return h, keep


def _next_ex(lib, h, ncols, str_cols, cap_rows, data_cap):
    els = [VARLEN if k in str_cols else 8 for k in range(ncols)]
    mc = MutChunk(els, cap_rows, [np.uint8 if k in str_cols else np.int64 for k in range(ncols)], data_cap)
    n = C.c_int64(-1)
    rc = lib.tg_agg_next_ex(h, C.byref(mc.struct), mc.varlen, C.c_int64(cap_rows), C.byref(n))
    return rc, n.value, mc


def test_empty_result_and_device_data_checks(lib):
    import torch
    from tidb_b200.device import DeviceAgg, dev_chunk
    plan = AggPlan([st(46), INT], [0, 1], [fr(0), fr(1), AggFunc(abi.AGG_COUNT, -1)])
    dev = DeviceAgg(plan)
    # a device string column with rows of bytes but no data pointer: TG_ERR_INVALID, nothing aggregated
    offs = torch.tensor([0, 2, 3], dtype=torch.int64, device="cuda")
    ck = dev_chunk([(offs, torch.zeros(0, dtype=torch.uint8, device="cuda")), torch.zeros(2, dtype=torch.int64, device="cuda")])
    assert lib.tg_agg_push_dev(dev.h, C.byref(ck)) == abi.TG_ERR_INVALID
    # all rows empty with no data pointer is a valid column; an empty push adds nothing
    empty = dev_chunk([(torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(0, dtype=torch.uint8, device="cuda")),
                       torch.zeros(0, dtype=torch.int64, device="cuda")])
    abi.check(lib.tg_agg_push_dev(dev.h, C.byref(empty)))
    rows, cols, nulls = dev.finish()
    from tidb_b200.device import fetch_device
    assert rows == 0 and dev.offsets[0] and fetch_device(dev.offsets[0], 8).view(np.int64)[0] == 0 and not dev.offsets[1]
    dev.close()
    got, _, _ = stats_run(plan, [])
    assert got == []


def test_rejected_pushes_and_result_calls(lib):
    import torch
    plan = AggPlan([st(46), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)])
    h, keep = _open(lib, plan)
    good = Chunk([Column.strings([b"aa", b"b ", b"aa ", b"dd", b"cccc"]), Column(np.zeros(5, np.int64))])
    cs = good.to_struct()
    abi.check(lib.tg_agg_push(h, C.byref(cs)))
    # host push with a row whose offsets run backwards
    bad = Chunk([Column(np.frombuffer(b"xyzw", np.uint8).copy(), None, np.array([0, 3, 1, 4], np.int64)), Column(np.zeros(3, np.int64))])
    bs = bad.to_struct()
    assert lib.tg_agg_push(h, C.byref(bs)) == abi.TG_ERR_INVALID
    # device push with an offset past offsets[length]
    from tidb_b200.device import dev_chunk
    offs = torch.tensor([0, 2, 9, 4], dtype=torch.int64, device="cuda")
    data = torch.zeros(8, dtype=torch.uint8, device="cuda")
    dc = dev_chunk([(offs, data), torch.zeros(3, dtype=torch.int64, device="cuda")])
    assert lib.tg_agg_push_dev(h, C.byref(dc)) == abi.TG_ERR_INVALID
    abi.check(lib.tg_agg_finish(h))
    # tg_agg_next and tg_agg_result_dev refuse the plan and write nothing
    mc = MutChunk([8, 8], 8)
    n = C.c_int64(-3)
    assert lib.tg_agg_next(h, C.byref(mc.struct), C.c_int64(8), C.byref(n)) == abi.TG_ERR_INVALID and n.value == -3
    # a data_cap too small for the next row: TG_ERR_CAPACITY, nothing written, the cursor unmoved
    rc, nn, mc = _next_ex(lib, h, 2, {0}, 8, 1)
    assert rc == abi.TG_ERR_CAPACITY and not mc.offsets[0].any() and not mc.data[1].any()
    rows, cap = [], 2
    while True:   # small caps serve prefixes; a cap the next row does not fit fails and moves nothing
        rc, nn, mc = _next_ex(lib, h, 2, {0}, 8, cap)
        if rc == abi.TG_ERR_CAPACITY:
            cap += 1
            continue
        abi.check(rc)
        if nn == 0:
            break
        assert 0 < mc.offsets[0][nn] <= cap
        vals = mc.columns(nn)
        rows += list(zip(vals[0][0], vals[1][0]))
    assert sorted(rows) == [(b"aa", 2), (b"b ", 1), (b"cccc", 1), (b"dd", 1)]
    lib.tg_agg_close(h)
