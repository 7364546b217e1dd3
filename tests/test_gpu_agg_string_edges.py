"""String GROUP BY (csrc/str_dict.cu, encode_strings in csrc/agg.cu) at the edges of the dictionary's warp election,
its earliest-row bookkeeping across CTAs and retry rounds, arena moves, and the var-length result download, against a
plain Python dictionary keyed by the collation key.

Every case is read back twice, through tg_agg_result_dev_ex (device offsets and bytes) and through tg_agg_next_ex
(host pages), and the two must agree row for row.  FIRSTROW of a string GROUP BY column is the raw bytes of the group's
earliest row in push order (sel order within a chunk); under the PAD collations (46, 83, 65, 47) rows of one key may
differ in their trailing spaces, which is the only place a wrong earliest row shows."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

import mydecimal as D
from tidb_b200 import abi
from tidb_b200.chunk import VARLEN, Chunk, Column, MutChunk, unpack_nulls
from tidb_b200.executor import HashAggExec, np_dtype_of
from tidb_b200.plan import AggFunc, AggPlan, FieldType

pytestmark = pytest.mark.gpu

INT = FieldType(abi.TYPE_LONGLONG, 0)
DEC = FieldType(abi.TYPE_NEWDECIMAL, 0, 15, 2)
COLLS = (46, 63, 309)
PAD = (46, 83, 65, 47)


def st(coll):
    return FieldType(abi.TYPE_VARCHAR, 0, collation=coll)


def fr(c):
    return AggFunc(abi.AGG_FIRSTROW, c)


@pytest.fixture(scope="module")
def lib():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return abi.load_lib()


# ---- reference ------------------------------------------------------------------------------------------------------
def logical_rows(plan, chunks):
    """the input rows in push order (sel order within a chunk), one tuple per row: bytes / int / Fraction / None"""
    out = []
    for ch in chunks:
        cols = []
        for c, t in enumerate(plan.col_types):
            col = ch.columns[c]
            nl = col.nulls()
            if col.is_varlen:
                v = [None if nl[i] else col.get_bytes(i) for i in range(col.length)]
            elif t.tp == abi.TYPE_NEWDECIMAL:
                v = [None if nl[i] else D.value(bytes(col.data[i])) for i in range(col.length)]
            else:
                v = [None if nl[i] else int(col.data[i]) for i in range(col.length)]
            cols.append(v if ch.sel is None else [v[i] for i in ch.sel])
        out.extend(zip(*cols))
    return out


def key_of(t, v):
    if v is None or t.tp not in abi.STRING_TYPES:
        return v
    return v.rstrip(b" ") if t.collation in PAD else v


def reference(plan, chunks):
    """group key -> the expected result row (FIRSTROW, COUNT, COUNT(DISTINCT), SUM over DECIMAL as a Fraction)"""
    groups = {}
    for r in logical_rows(plan, chunks):
        k = tuple(key_of(plan.col_types[g], r[g]) for g in plan.group_by)
        groups.setdefault(k, []).append(r)
    out = {}
    for k, rows in groups.items():
        vals = []
        for f in plan.funcs:
            col = [r[f.arg_col] for r in rows] if f.arg_col >= 0 else None
            if f.name == abi.AGG_FIRSTROW:
                vals.append(col[0])
            elif f.name == abi.AGG_COUNT:
                vals.append(len(rows) if col is None else len({x for x in col if x is not None}) if f.distinct
                            else sum(x is not None for x in col))
            elif f.name == abi.AGG_SUM:
                xs = [x for x in col if x is not None]
                vals.append(sum(xs, Fraction(0)) if xs else None)
            else:
                raise ValueError(f.name)
        out[k] = tuple(vals)
    return out


def result_key(plan, row):
    pos = {f.arg_col: i for i, f in reversed(list(enumerate(plan.funcs))) if f.name == abi.AGG_FIRSTROW}
    return tuple(key_of(plan.col_types[g], row[pos[g]]) for g in plan.group_by)


def check(plan, chunks, got):
    exp = reference(plan, chunks)
    seen = {}
    for r in got:
        k = result_key(plan, r)
        assert k not in seen, f"group {k!r:.80} twice"
        seen[k] = r
    assert set(seen) == set(exp), sorted(map(repr, set(seen) ^ set(exp)))[:5]
    for k, e in exp.items():
        g = tuple(D.value(v) if isinstance(v, bytes) and f.name == abi.AGG_SUM else v for v, f in zip(seen[k], plan.funcs))
        assert g == e, (repr(k)[:80], repr(g)[:200], repr(e)[:200])
    return exp


# ---- one handle, pushed from the host or the device, read back both ways ---------------------------------------------
def out_schema(plan):
    return HashAggExec(plan, None).schema


def read_dev(lib, h, plan):
    from tidb_b200.device import fetch_device
    nf = len(plan.funcs)
    rows = C.c_int64(-1)
    cols, nulls, offs = (C.c_void_p * nf)(), (C.c_void_p * nf)(), (C.c_void_p * nf)()
    abi.check(lib.tg_agg_result_dev_ex(h, C.byref(rows), cols, nulls, offs))
    n = rows.value
    out = []
    for k, t in enumerate(out_schema(plan)):
        nl = unpack_nulls(fetch_device(nulls[k], (n + 7) // 8), n) if nulls[k] else np.zeros(n, bool)
        if offs[k]:
            o = fetch_device(offs[k], (n + 1) * 8).view(np.int64)
            assert o[0] == 0 and np.all(np.diff(o) >= 0)
            b = fetch_device(cols[k], int(o[-1]))
            out.append([None if nl[r] else b[o[r]:o[r + 1]].tobytes() for r in range(n)])
            continue
        dt = np.dtype(np_dtype_of(t))
        raw = fetch_device(cols[k], n * dt.itemsize)
        if t.tp == abi.TYPE_NEWDECIMAL:
            out.append([None if nl[r] else raw[40 * r:40 * r + 40].tobytes() for r in range(n)])
        else:
            v = raw.view(dt)
            out.append([None if nl[r] else v[r].item() for r in range(n)])
    return list(zip(*out)) if out else []


def next_page(lib, h, plan, cap_rows, data_cap):
    schema, strs = out_schema(plan), plan.string_results()
    els = [VARLEN if s else np.dtype(np_dtype_of(t)).itemsize for s, t in zip(strs, schema)]
    mc = MutChunk(els, cap_rows, [np.uint8 if s else np_dtype_of(t) for s, t in zip(strs, schema)], data_cap)
    for k, s in enumerate(strs):
        if s:
            mc.data[k][:] = 0xEE
            mc.offsets[k][:] = -5
    n = C.c_int64(-1)
    rc = lib.tg_agg_next_ex(h, C.byref(mc.struct), mc.varlen, C.c_int64(cap_rows), C.byref(n))
    return rc, n.value, mc


def page_rows(plan, mc, n):
    out = []
    for k, (v, nl) in enumerate(mc.columns(n)):
        if v.ndim == 2:
            out.append([None if nl[r] else v[r].tobytes() for r in range(n)])
        else:
            out.append([None if nl[r] else (v[r] if isinstance(v[r], bytes) else v[r].item()) for r in range(n)])
    return list(zip(*out))


def read_next(lib, h, plan, cap_rows=1024, data_cap=1 << 20):
    """every result row through tg_agg_next_ex pages; a row that does not fit data_cap gets a 16x bigger one"""
    rows = []
    while True:
        rc, n, mc = next_page(lib, h, plan, cap_rows, data_cap)
        if rc == abi.TG_ERR_CAPACITY:
            data_cap *= 16
            continue
        abi.check(rc)
        if n == 0:
            return rows
        rows += page_rows(plan, mc, n)


def open_handle(lib, plan):
    d, keep = plan.to_struct_ex3()
    h = C.c_void_p()
    abi.check(lib.tg_agg_open_ex3(C.byref(d), C.byref(h)))
    return h, keep


def dev_cols(plan, ch, pad):
    import torch
    cols, nulls = [], []
    for c, t in enumerate(plan.col_types):
        col = ch.columns[c]
        if col.is_varlen:
            data = np.concatenate([np.full(pad, 0x58, np.uint8), col.data, np.zeros(1, np.uint8)])
            cols.append((torch.from_numpy(col.offsets + pad).cuda(), torch.from_numpy(data).cuda()))
        else:
            cols.append(torch.from_numpy(np.ascontiguousarray(col.data)).cuda())
        nulls.append(torch.from_numpy(col.null_bitmap.copy()).cuda() if col.null_bitmap is not None else None)
    return cols, nulls


def push_all(lib, h, plan, chunks, device):
    from tidb_b200.device import dev_chunk
    for i, ch in enumerate(chunks):
        if device:
            assert ch.sel is None
            cols, nulls = dev_cols(plan, ch, pad=i % 13)
            abi.check(lib.tg_agg_push_dev(h, C.byref(dev_chunk(cols, nulls))))
        else:
            cs = ch.to_struct()
            abi.check(lib.tg_agg_push(h, C.byref(cs)))


def run(lib, plan, chunks, device=False, stats=False):
    """push, finish, read back through both calls (they must agree); -> result rows (and the stats)"""
    h, keep = open_handle(lib, plan)
    try:
        push_all(lib, h, plan, chunks, device)
        abi.check(lib.tg_agg_finish(h))
        dev = read_dev(lib, h, plan)
        nxt = read_next(lib, h, plan)
        assert dev == nxt, "tg_agg_result_dev_ex and tg_agg_next_ex disagree"
        if not stats:
            return dev
        s, ss = abi.TgAggStats(), abi.TgAggStringStats()
        abi.check(lib.tg_agg_get_stats(h, C.byref(s)))
        abi.check(lib.tg_agg_get_string_stats(h, C.byref(ss)))
        return dev, s, ss
    finally:
        lib.tg_agg_close(h)


def both(lib, plan, chunks):
    """host pushes (as given, sel vectors kept) and device pushes (sel applied) give the reference"""
    check(plan, chunks, run(lib, plan, chunks))
    dense = [Chunk([c.take(ch.sel) for c in ch.columns]) if ch.sel is not None else ch for ch in chunks]
    check(plan, dense, run(lib, plan, dense, device=True))


# ---- warp election --------------------------------------------------------------------------------------------------
def election_rows(rng):
    sp = lambda k: b" " * int(k)
    rows = []
    rows += [b"same" + sp(j % 4) for j in range(32)]                 # one warp, one key (PAD: four raw forms)
    rows += [b"d%02d" % j for j in range(32)]                        # one warp, 32 keys
    rows += [b"p%02d" % (j % 16) + sp(j // 16) for j in range(32)]   # 16 pairs, lanes j and j + 16
    rows += [b"q%02d" % (j // 2) + sp(1 - j % 2) for j in range(32)]  # 16 pairs, adjacent lanes
    # PAD-equal keys spread over warps and CTAs: each appears first in its earliest form at a random row
    n = 60_000
    ks = rng.integers(0, 400, n)
    rows += [b"w%03d" % k + sp(t) for k, t in zip(ks, rng.integers(0, 5, n))]
    return rows


@pytest.mark.parametrize("coll", COLLS)
def test_warp_election_and_earliest_row(lib, coll):
    rng = np.random.default_rng(coll)
    rows = election_rows(rng)
    n = len(rows)
    plan = AggPlan([st(coll), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_COUNT, 0)])
    chunks = [Chunk([Column.strings(rows), Column(np.arange(n, dtype=np.int64))])]
    both(lib, plan, chunks)
    # the same rows in 1024-row chunks, each with a sel vector that reverses it
    parts = Chunk([Column.strings(rows), Column(np.arange(n, dtype=np.int64))]).split(1024)
    both(lib, plan, [Chunk(p.columns, np.arange(p.num_rows() - 1, -1, -1, dtype=np.int64)) for p in parts])


@pytest.mark.parametrize("coll", PAD)
def test_earliest_row_that_arrives_last(lib, coll):
    # row 0's key has a million trailing spaces, so its warp is still cutting them when warps of later rows of the
    # same key insert the entry: the entry's earliest ordinal must still come down to row 0
    rng = np.random.default_rng(coll)
    n = 40_000
    rows = [b"K" + b" " * (1 << 20)] + [b"K" + b" " * int(t) if k == 0 else b"o%d" % k for k, t in
                                         zip(rng.integers(0, 50, n - 1), rng.integers(0, 3, n - 1))]
    plan = AggPlan([st(coll), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)])
    chunks = [Chunk([Column.strings(rows), Column(np.zeros(n, np.int64))])]
    exp = check(plan, chunks, run(lib, plan, chunks))
    assert exp[(b"K",)][0] == rows[0]
    check(plan, chunks, run(lib, plan, chunks, device=True))


# ---- forced deferral --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("coll", COLLS)
def test_forced_deferral_in_one_push(lib, coll):
    # expected_groups = 1: the dictionary starts at 1024 slots and 1024 ids, and one batch brings 300 k keys, so rows
    # are deferred both for a full id array and for a long probe while the table and the arrays grow
    rng = np.random.default_rng(100 + coll)
    nk = 300_000
    keys = rng.permutation(nk)
    order = np.concatenate([keys, rng.permutation(nk)[: nk // 2], keys[::-3]])
    rows = [b"key-%06d" % k + b" " * int((k * 7 + j) % 4) for j, k in enumerate(order)]
    n = len(rows)
    plan = AggPlan([st(coll), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)], expected_groups=1)
    for device in (False, True):
        chunks = [Chunk([Column.strings(rows), Column(np.zeros(n, np.int64))])]
        got, s, ss = run(lib, plan, chunks, device=device, stats=True)
        exp = check(plan, chunks, got)
        assert ss.dict_grows > 0 and ss.dict_entries == len(exp) >= nk
        assert s.paths & abi.AGG_PATH_STRING_KEY


# ---- arena moves ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_arena_moves_over_many_pushes(lib, device):
    rng = np.random.default_rng(int(device))
    plan = AggPlan([st(46), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)], expected_groups=1)
    chunks, made = [], 0
    for p in range(56):
        new = [bytes([65 + (made + j) % 26]) * int(rng.integers(100, 3001)) + b"#%d" % (made + j) +
               b" " * int(rng.integers(0, 3)) for j in range(int(rng.integers(5, 40)))]
        made += len(new)
        old = [chunks[int(i)].columns[0].get_bytes(0) for i in rng.integers(0, len(chunks), 5)] if chunks else []
        vals = new + old
        chunks.append(Chunk([Column.strings(vals), Column(np.zeros(len(vals), np.int64))]))
    h, keep = open_handle(lib, plan)
    try:
        push_all(lib, h, plan, chunks, device)
        abi.check(lib.tg_agg_finish(h))
        dev = read_dev(lib, h, plan)
        assert dev == read_next(lib, h, plan, cap_rows=7, data_cap=20_000)
        ss = abi.TgAggStringStats()
        abi.check(lib.tg_agg_get_string_stats(h, C.byref(ss)))
    finally:
        lib.tg_agg_close(h)
    check(plan, chunks, dev)
    assert ss.dict_entries == made
    if device:
        assert ss.launches > 3 * 56   # every push ran its own encode pass, claim and copy


# ---- NULL and empty -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("coll", (63, 46, 83, 65, 47, 309))
def test_null_empty_and_spaces(lib, coll):
    rng = np.random.default_rng(coll)
    pool = [None, b"", b"   ", b" ", b"x", b"x ", None]
    vals = [pool[i] for i in rng.integers(0, len(pool), 5000)]
    plan = AggPlan([st(coll), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, 0), AggFunc(abi.AGG_COUNT, -1)])
    chunks = Chunk([Column.strings(vals), Column(np.zeros(5000, np.int64))]).split(1024)
    exp = reference(plan, chunks)
    assert exp[(None,)][1] == 0 and exp[(None,)][2] == sum(v is None for v in vals)
    assert (b"",) in exp and exp[(b"",)][1] > 0
    assert len(exp) == (3 if coll in PAD else 6)   # PAD: NULL, '' (with ' ' and '   '), 'x' (with 'x ')
    both(lib, plan, chunks)


# ---- multi-key ----------------------------------------------------------------------------------------------------------
PATHS = [("v1", {"TG_AGG_V1": "1"}, abi.AGG_PATH_V1_GLOBAL | abi.AGG_PATH_V1_LOCAL),
         ("v2_global", {"TG_AGG_LOCAL": "0"}, abi.AGG_PATH_V2_GLOBAL),
         ("v2_local", {"TG_AGG_LOCAL": "2"}, abi.AGG_PATH_V2_LOCAL)]


def multi_key_table(rng, shape, coll, n=30_000):
    words = [b"AIR", b"MAIL", b"SHIP", b"zz" * 20, b"a", b"", b"TRUCK"]
    sp = lambda: b" " * int(rng.integers(0, 3)) if coll in PAD else b""
    a_i = rng.integers(0, len(words), n)
    if shape == "swapped":
        b_i = (a_i + 1 + rng.integers(0, 2, n)) % len(words)
        swap = rng.random(n) < 0.5
        a_i, b_i = np.where(swap, b_i, a_i), np.where(swap, a_i, b_i)
        c0 = [words[i] + sp() for i in a_i]
        c1 = [words[i] + sp() for i in b_i]
        types = [st(coll), st(coll)]
    elif shape == "identical":
        c0 = [words[i] + sp() for i in a_i]
        c1 = list(c0)
        types = [st(coll), st(coll)]
    else:   # (string, BIGINT) whose integers are the ids the strings get (first seen first)
        c0 = [words[i] + sp() for i in a_i]
        c1 = rng.integers(0, len(words), n).astype(np.int64)
        types = [st(coll), INT]
    # the earliest row of key "a" in group ("a", x) has more trailing spaces than the key's first row overall
    if coll in PAD:
        c0[0], c0[1] = b"a", b"a   "
        if shape == "int":
            c1[0], c1[1] = 0, 1
        else:
            c1[0], c1[1] = b"AIR", b"MAIL"
    cnul = rng.random(n) < 0.03
    cnul[:2] = False
    dv = rng.integers(-99999, 99999, n)
    cells = np.frombuffer(b"".join(D.encode(Fraction(int(v), 100), 2) for v in dv), np.uint8).reshape(n, 40).copy()
    iv = rng.integers(0, 50, n).astype(np.int64)
    col1 = Column.strings(c1) if shape != "int" else Column(c1)
    cols = [Column.strings([None if z else v for v, z in zip(c0, cnul)]), col1, Column(iv), Column(cells)]
    return types + [INT, DEC], cols


@pytest.mark.parametrize("shape", ["swapped", "identical", "int"])
def test_multi_key_with_distinct_and_decimal_sum(lib, shape):
    # several GROUP BY columns run through the one multi-key update (k_agg_update_mk)
    for coll in (46, 309):
        rng = np.random.default_rng(["swapped", "identical", "int"].index(shape) * 1000 + coll)
        types, cols = multi_key_table(rng, shape, coll)
        plan = AggPlan(types, [0, 1], [fr(0), fr(1), AggFunc(abi.AGG_COUNT, 2, distinct=True),
                                       AggFunc(abi.AGG_SUM, 3, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=2), AggFunc(abi.AGG_COUNT, -1)])
        chunks = Chunk(cols).split(1024)
        for device in (False, True):
            got, s, _ = run(lib, plan, chunks, device=device, stats=True)
            exp = check(plan, chunks, got)
            assert s.paths & abi.AGG_PATH_STRING_KEY and s.paths & abi.AGG_PATH_MULTI_KEY, s.paths
            if coll in PAD:
                second = (b"a", 1 if shape == "int" else b"MAIL")
                assert exp[second][0] == b"a   "


@pytest.mark.parametrize("variant,env,bit", PATHS, ids=[p[0] for p in PATHS])
def test_string_key_update_paths_with_distinct_and_decimal_sum(lib, monkeypatch, variant, env, bit):
    # one string GROUP BY column: its id column takes each forced single-key update path.  The CTA-local level holds at
    # most 4 state words per group, so DISTINCT and the DECIMAL SUM also run in plans of their own, which it takes.
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    distinct, dec_sum = AggFunc(abi.AGG_COUNT, 2, distinct=True), AggFunc(abi.AGG_SUM, 3, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=2)
    funcs = [[distinct, AggFunc(abi.AGG_COUNT, 0)], [dec_sum]]
    if variant != "v2_local":
        funcs.append([distinct, dec_sum, AggFunc(abi.AGG_COUNT, 0)])
    for coll in (46, 309):
        rng = np.random.default_rng(coll)
        types, cols = multi_key_table(rng, "int", coll)
        chunks = Chunk(cols).split(1024)
        for fs in funcs:
            plan = AggPlan(types, [0], [fr(0)] + fs)
            for device in (False, True):
                got, s, _ = run(lib, plan, chunks, device=device, stats=True)
                check(plan, chunks, got)
                assert s.paths & bit and s.paths & abi.AGG_PATH_STRING_KEY, (variant, len(fs), s.paths)


# ---- result download ------------------------------------------------------------------------------------------------
def _finished(lib, plan, chunks):
    h, keep = open_handle(lib, plan)
    push_all(lib, h, plan, chunks, False)
    abi.check(lib.tg_agg_finish(h))
    return h, keep


def test_download_page_sizes(lib):
    rng = np.random.default_rng(2)
    vals = [b"r%05d" % i + b"x" * int(rng.integers(0, 40)) for i in range(5000)]
    plan = AggPlan([st(63), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)])
    chunks = Chunk([Column.strings(vals), Column(np.zeros(5000, np.int64))]).split(1024)
    h, keep = _finished(lib, plan, chunks)
    try:
        want = read_dev(lib, h, plan)
        page, got = 100, []
        while len(got) < len(want):
            rows = want[len(got):len(got) + page]
            exact = sum(len(r[0]) for r in rows)
            # one byte short: one row fewer
            rc, n, mc = next_page(lib, h, plan, page, exact - 1)
            if len(rows) == 1:
                assert rc == abi.TG_ERR_CAPACITY and n == 0
                continue
            assert rc == 0 and n == len(rows) - 1, (n, len(rows))
            assert page_rows(plan, mc, n) == rows[:n]
            assert mc.offsets[0][0] == 0 and mc.offsets[0][n] <= exact - 1
            got += rows[:n]
            rows = want[len(got):len(got) + page]
            exact = sum(len(r[0]) for r in rows)
            rc, n, mc = next_page(lib, h, plan, page, exact)   # exactly the bytes of a page
            assert rc == 0 and n == len(rows) and mc.offsets[0][n] == exact
            assert page_rows(plan, mc, n) == rows
            got += rows
        rc, n, mc = next_page(lib, h, plan, page, 10)
        assert rc == 0 and n == 0
        assert got == want
        check(plan, chunks, got)
    finally:
        lib.tg_agg_close(h)


def test_download_row_larger_than_cap(lib):
    big = b"B" * 70_000
    vals = [b"a", b"bb", big, b"c", big + b" ", b"d"]
    plan = AggPlan([st(309), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)])
    chunks = [Chunk([Column.strings(vals), Column(np.zeros(len(vals), np.int64))])]
    h, keep = _finished(lib, plan, chunks)
    try:
        want = read_dev(lib, h, plan)
        got, cap = [], 1000
        while True:
            rc, n, mc = next_page(lib, h, plan, 16, cap)
            if rc == abi.TG_ERR_CAPACITY:
                # nothing written: the caller's bytes and offsets keep their fill, and the next call resumes at this row
                assert n == 0 and (mc.data[0] == 0xEE).all() and (mc.offsets[0] == -5).all()
                assert len(want[len(got)][0]) > cap
                cap = 100_000
                continue
            abi.check(rc)
            if n == 0:
                break
            got += page_rows(plan, mc, n)
            cap = 1000
        assert got == want
        check(plan, chunks, got)
    finally:
        lib.tg_agg_close(h)


def test_download_offsets_across_scan_blocks(lib):
    # 300 k result rows: the offsets scan runs in 1024-row blocks, and the block sums of more than 256 blocks are
    # carried across passes of k_scan_carry
    rng = np.random.default_rng(3)
    nk = 300_000
    vals = [b"g%d" % i + b"." * int(i % 7) for i in rng.permutation(nk)]
    plan = AggPlan([st(63), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)])
    chunks = [Chunk([Column.strings(vals), Column(np.zeros(nk, np.int64))])]
    for device in (False, True):
        got = run(lib, plan, chunks, device=device)
        check(plan, chunks, got)


def test_download_empty_input(lib):
    from tidb_b200.device import fetch_device
    plan = AggPlan([st(46), INT], [0], [fr(0), AggFunc(abi.AGG_COUNT, -1)])
    h, keep = open_handle(lib, plan)
    try:
        abi.check(lib.tg_agg_finish(h))
        rows = C.c_int64(-1)
        cols, nulls, offs = (C.c_void_p * 2)(), (C.c_void_p * 2)(), (C.c_void_p * 2)()
        abi.check(lib.tg_agg_result_dev_ex(h, C.byref(rows), cols, nulls, offs))
        assert rows.value == 0 and offs[0] and not offs[1]
        assert fetch_device(offs[0], 8).view(np.int64).tolist() == [0]
        rc, n, mc = next_page(lib, h, plan, 8, 64)
        assert rc == 0 and n == 0
    finally:
        lib.tg_agg_close(h)


# ---- trailing-space count overflow --------------------------------------------------------------------------------------
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_tail_overflow_breaks_the_handle(lib, device):
    # two GROUP BY columns, FIRSTROW of a PAD string column: a row with 2^23 trailing spaces is refused, and the handle
    # refuses every later push and finish (the dictionary has already taken the batch's keys)
    plan = AggPlan([st(46), INT], [0, 1], [fr(0), fr(1), AggFunc(abi.AGG_COUNT, -1)])
    ok = Chunk([Column.strings([b"a", b"b "]), Column(np.array([1, 2], np.int64))])
    bad = Chunk([Column.strings([b"c", b"k" + b" " * (1 << 23)]), Column(np.array([1, 2], np.int64))])
    short = Chunk([Column.strings([b"k" + b" " * ((1 << 23) - 1)]), Column(np.array([3], np.int64))])
    from tidb_b200.device import dev_chunk
    h, keep = open_handle(lib, plan)
    try:
        if device:
            push_all(lib, h, plan, [ok, short], True)   # one space fewer is accepted
            cols, nulls = dev_cols(plan, bad, 3)
            assert lib.tg_agg_push_dev(h, C.byref(dev_chunk(cols, nulls))) == abi.TG_ERR_UNSUPPORTED
        else:
            push_all(lib, h, plan, [ok, short, bad], False)   # staged: the batch runs at finish
            assert lib.tg_agg_finish(h) == abi.TG_ERR_UNSUPPORTED
        cs = ok.to_struct()
        assert lib.tg_agg_push(h, C.byref(cs)) == abi.TG_ERR_STATE
        cols, nulls = dev_cols(plan, ok, 0)
        assert lib.tg_agg_push_dev(h, C.byref(dev_chunk(cols, nulls))) == abi.TG_ERR_STATE
        assert lib.tg_agg_finish(h) == abi.TG_ERR_STATE
    finally:
        lib.tg_agg_close(h)
    # without the too-wide row the same plan keeps the 2^23 - 1 spaces of its FIRSTROW
    check(plan, [ok, short], run(lib, plan, [ok, short]))
