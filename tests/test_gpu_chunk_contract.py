"""The chunk contract at every operator boundary (csrc/chunk_io.cu): how pushed chunks are read and how a caller's output
chunk is filled, for the join, the aggregation, TopN and the VecEval calls.

One generator cuts the same logical rows into many physical layouts: chunk lengths 0 (data NULL), 1, 5, 7, 9, 1023, 1025
and primes; sel vectors absent, identity, reversed, a sorted random subset over garbage rows, and empty (nsel = 0 over
physical rows); NULL bitmaps absent, all-valid, first brought after 5 + 7 + 9 rows, dropped and brought back, and with
stray 1 bits past `length`.  Every result is compared twice:
  (a) with an exact reference of the logical rows (join_reference, an exact numpy aggregation, vec_reference), and
  (b) bit for bit with the same operator's result on the canonical layout: one dense chunk, no sel, and a bitmap only
      where a NULL exists.
DOUBLE values are multiples of 1/4 far below 2^53, so every SUM is exact in any order and (b) is bitwise too.

Output windows visit every read cursor mod 8 and check that the bits past the rows returned are zero.  A rejected output
call (nullable column without a bitmap, elem_len mismatch, TopN capacity, malformed DECIMAL) must write nothing: the
sentinel in `out` survives, *nrows is 0, and the cursor and d2h_bytes do not move.  Every rejection here is a host-side
argument check that returns before any kernel runs."""
import ctypes as C

import numpy as np
import pytest

import mydecimal_args as A
import vec_reference as V
from join_reference import assert_same_rows, join_reference
from tidb_b200 import abi
from tidb_b200.chunk import DECIMAL_DTYPE, Chunk, Column, MutChunk, unpack_nulls
from tidb_b200.executor import np_dtype_of
from tidb_b200.plan import AggFunc, AggPlan, FieldType, FilterItem, JoinPlan

pytestmark = pytest.mark.gpu

INT, INT_NN = FieldType(abi.TYPE_LONGLONG, 0), FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
DBL, FLT = FieldType(abi.TYPE_DOUBLE, 0), FieldType(abi.TYPE_FLOAT, 0)
DEC, DEC_NN = FieldType(abi.TYPE_NEWDECIMAL, 0, 15, 2), FieldType(abi.TYPE_NEWDECIMAL, abi.FLAG_NOT_NULL, 15, 2)
SWITCHES = ("TG_AGG_LOCAL", "TG_AGG_LOCAL_SLOTS", "TG_AGG_V1", "TG_PROBE_PARTITION", "TG_PROBE_PARTS", "TG_PROBE_PART_MIN_MB",
            "TG_PROBE_PART_MIN_ROWS", "TG_PROBE_UQ", "TG_PROBE_INPLACE")
LENGTHS = (5, 7, 9, 0, 1, 1023, 1025, 13, 0, 2039, 1, 131, 7, 4099, 9, 1021)
SEL_MODES = ("none", "identity", "reversed", "subset")
BM_MODES = ("absent", "all_valid", "late", "dropped", "stray")
STAGE_ROWS = 4 << 20          # kStageBatchRows: the host staging of pushed chunks is flushed at this many rows
DIRECT_ROWS = 128 << 10       # kDirectPushRows: probe chunks this big (without sel) go straight to the device


@pytest.fixture(autouse=True)
def _default_switches(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)


# ---- the layout generator --------------------------------------------------------------------------------------------
def null_plan(rng, lengths, mode, rate=0.25):
    """per chunk: (logical NULL flags, whether the chunk carries a bitmap, whether its last byte gets stray bits)"""
    out, row = [], 0
    for i, n in enumerate(lengths):
        nl = np.zeros(n, dtype=bool)
        if mode == "absent":
            bm = False
        elif mode == "all_valid":
            bm = True
        elif mode == "late":                 # no NULL in the first 5 + 7 + 9 rows, a bitmap only on chunks with a NULL
            nl = (rng.random(n) < rate) & (row + np.arange(n) >= 21)
            bm = bool(nl.any())
        elif mode == "dropped":              # chunks 0-2 bring one, 3-5 do not, 6-8 do, ...
            bm = (i // 3) % 2 == 0
            nl = (rng.random(n) < rate) if bm else nl
        else:                                # "stray"
            bm, nl = True, rng.random(n) < rate
        out.append((nl, bm, mode == "stray"))
        row += n
    return out


def logical(rng, lengths, values, mode, nullable):
    """(values, nulls, per-chunk null plan or None) of one column: NOT NULL columns have no plan"""
    if not nullable:
        return values, np.zeros(len(values), dtype=bool), None
    plan = null_plan(rng, lengths, mode)
    nl = np.concatenate([p[0] for p in plan]) if plan else np.zeros(0, dtype=bool)
    return values, nl, plan


def _garbage(rng, shape, dtype):
    return rng.integers(0, 256, (int(np.prod(shape)) * np.dtype(dtype).itemsize,), dtype=np.uint8).view(dtype).reshape(shape)


def cut(rng, cols, lengths, sel_mode):
    """chunks holding the logical rows of `cols` [(values, nulls, null plan)], chunk i with lengths[i] logical rows laid
    out by sel_mode; rows no sel points at hold garbage (random bytes and random NULL bits).  Every fourth chunk of a
    sel mode is preceded by a chunk with physical rows and an empty sel."""
    chunks, lo = [], 0
    for i, n in enumerate(lengths):
        if sel_mode != "none" and i % 4 == 3:
            phys = [Column(_garbage(rng, (11,) + v.shape[1:], v.dtype), rng.random(11) < 0.5 if plan else None) for v, _, plan in cols]
            empty = Chunk(phys, np.zeros(0, dtype=np.int64))
            assert empty.sel.ctypes.data     # nsel = 0 with a non-NULL sel pointer: no logical row at all
            chunks.append(empty)
        if sel_mode == "none" or sel_mode == "identity":
            p, pos = n, np.arange(n)
        elif sel_mode == "reversed":
            p, pos = n, np.arange(n)[::-1].copy()
        else:
            p = 2 * n + 3
            pos = np.sort(rng.choice(p, n, replace=False))
        out = []
        for v, nl, plan in cols:
            data = _garbage(rng, (p,) + v.shape[1:], v.dtype) if p != n else np.empty((p,) + v.shape[1:], dtype=v.dtype)
            data[pos] = v[lo:lo + n]
            col = Column(data)
            if plan is not None and plan[i][1]:
                pn = rng.random(p) < 0.5
                pn[pos] = nl[lo:lo + n]
                bm = np.packbits(~pn, bitorder="little")
                if plan[i][2] and p & 7:
                    bm[-1] |= np.uint8((0xFF << (p & 7)) & 0xFF)
                col.null_bitmap = bm
            else:
                assert not nl[lo:lo + n].any()
            out.append(col)
        chunks.append(Chunk(out, None if sel_mode == "none" else pos.astype(np.int64)))
        lo += n
    return chunks


def canonical(cols):
    """the canonical layout of the same logical rows: one dense chunk, a bitmap only where a NULL exists"""
    return [Chunk([Column(v, nl if nl.any() else None) for v, nl, _ in cols])]


def quarters(rng, n, lim=1 << 20):
    return rng.integers(-lim, lim, n).astype(np.float64) / 4


def dec_cells(scaled):
    """DECIMAL(15, 2) cells in FromBin's stored form"""
    n = len(scaled)
    return A.cells_np(scaled, 15, 2, np.full(n, 13), np.zeros(n, dtype=np.int64), scaled < 0)


# ---- driving the ABI -----------------------------------------------------------------------------------------------
def push(fn, h, chunks):
    for ch in chunks:
        cs = ch.to_struct()
        abi.check(fn(h, C.byref(cs)))


def out_dtypes(schema):
    return [np_dtype_of(t) for t in schema]


def drain(next_fn, h, dts, windows, cap=None):
    """every result row through next_fn with max_rows cycling through `windows`; checks that the bits past the rows
    returned are zero -> ([(values, nulls)], the set of read cursors mod 8 the calls started at)"""
    cap = cap or max(windows)
    out = MutChunk([np.dtype(d).itemsize for d in dts], cap, dts)
    vals, nls, starts, lo, k = [[] for _ in dts], [[] for _ in dts], set(), 0, 0
    while True:
        w = windows[k % len(windows)]
        k += 1
        for b in out.bitmaps:
            b[:] = 0xA5
        n = C.c_int64(-1)
        abi.check(next_fn(h, C.byref(out.struct), C.c_int64(w), C.byref(n)))
        m = n.value
        if m == 0:
            break
        assert 0 < m <= min(w, cap)
        starts.add(lo % 8)
        lo += m
        for c in range(len(dts)):
            if m & 7:
                assert out.bitmaps[c][m >> 3] >> (m & 7) == 0, f"column {c}: bits past the {m} rows returned are set"
            vals[c].append(out.data[c][:m].copy())
            nls[c].append(unpack_nulls(out.bitmaps[c], m))
    res = []
    for c, d in enumerate(dts):
        dt = np.dtype(d)
        res.append((np.concatenate(vals[c]) if vals[c] else np.zeros((0,) + dt.shape, dtype=dt.base),
                    np.concatenate(nls[c]) if nls[c] else np.zeros(0, dtype=bool)))
    return res, starts


class Join:
    def __init__(self, plan):
        self.lib, self.plan = abi.load_lib(), plan
        d, self._keep = plan.to_struct()
        self.h = C.c_void_p()
        abi.check(self.lib.tg_join_open(C.byref(d), C.byref(self.h)))

    def build(self, chunks):
        push(self.lib.tg_join_build_push, self.h, chunks)
        abi.check(self.lib.tg_join_build_finish(self.h))

    def probe(self, chunks):
        push(self.lib.tg_join_probe_push, self.h, chunks)
        abi.check(self.lib.tg_join_probe_finish(self.h))

    def drain(self, windows=(4096,), cap=None):
        return drain(self.lib.tg_join_next, self.h, out_dtypes(self.plan.out_schema()), windows, cap)

    def stats(self):
        s = abi.TgJoinStats()
        abi.check(self.lib.tg_join_get_stats(self.h, C.byref(s)))
        return s

    def close(self):
        self.lib.tg_join_close(self.h)


def run_join(plan, build, probe, windows=(4096,), cap=None):
    j = Join(plan)
    try:
        j.build(build)
        j.probe(probe)
        cols, _ = j.drain(windows, cap)
        return cols, j.stats()
    finally:
        j.close()


class Agg:
    def __init__(self, plan):
        self.lib, self.plan = abi.load_lib(), plan
        d, self._keep = plan.to_struct_ex2()
        self.h = C.c_void_p()
        abi.check(self.lib.tg_agg_open_ex2(C.byref(d), C.byref(self.h)))

    def push(self, chunks):
        push(self.lib.tg_agg_push, self.h, chunks)

    def finish(self):
        abi.check(self.lib.tg_agg_finish(self.h))

    def dtypes(self):
        return [DECIMAL_DTYPE if f.ret_type == abi.TYPE_NEWDECIMAL else (np.float64 if f.name in (abi.AGG_SUM, abi.AGG_AVG) else np.int64)
                for f in self.plan.funcs]

    def drain(self, windows=(4096,), cap=None):
        return drain(self.lib.tg_agg_next, self.h, self.dtypes(), windows, cap)

    def stats(self):
        s = abi.TgAggStats()
        abi.check(self.lib.tg_agg_get_stats(self.h, C.byref(s)))
        return s

    def close(self):
        self.lib.tg_agg_close(self.h)


def run_agg(plan, chunks, windows=(4096,), cap=None):
    a = Agg(plan)
    try:
        a.push(chunks)
        a.finish()
        cols, _ = a.drain(windows, cap)
        return cols, a.stats()
    finally:
        a.close()


def assert_bitwise(want, got, what=""):
    """same rows in the same order, values compared by their bits (zero under NULL is not required of `want`)"""
    assert len(want) == len(got)
    for c, ((wv, wn), (gv, gn)) in enumerate(zip(want, got)):
        assert np.array_equal(wn, gn), f"{what} column {c}: NULL flags differ"
        wb = np.ascontiguousarray(wv).reshape(len(wv), -1).view(np.uint8)
        gb = np.ascontiguousarray(gv).reshape(len(gv), -1).view(np.uint8)
        assert np.array_equal(wb[~wn], gb[~gn]), f"{what} column {c}: values differ"


# ---- join: every layout of both sides -------------------------------------------------------------------------------
# probe (left): 0 key INT | 1 x DOUBLE | 2 f FLOAT (4 bytes) | 3 d DECIMAL      build (right): 0 key INT | 1 INT | 2 DECIMAL
LTYPES, RTYPES = [INT, DBL, FLT, DEC], [INT, INT, DEC]


def join_side_cols(rng, lengths, mode, probe):
    n = sum(lengths)
    if probe:
        vals = [rng.integers(0, 3000, n).astype(np.int64), quarters(rng, n), (rng.integers(-1000, 1000, n) / 8).astype(np.float32),
                rng.integers(0, 256, (n, 40), dtype=np.uint8)]
    else:   # duplicate build keys: the general probe
        vals = [rng.integers(0, 4000, n).astype(np.int64), rng.integers(-10**12, 10**12, n), rng.integers(0, 256, (n, 40), dtype=np.uint8)]
    return [logical(rng, lengths, v, mode, True) for v in vals]


@pytest.mark.parametrize("sel_mode", SEL_MODES)
@pytest.mark.parametrize("bm_mode", BM_MODES)
def test_join_layouts(sel_mode, bm_mode):
    rng = np.random.default_rng(100 + SEL_MODES.index(sel_mode) * 10 + BM_MODES.index(bm_mode))
    plengths, blengths = LENGTHS, LENGTHS[::-1][:9]
    pcols, bcols = join_side_cols(rng, plengths, bm_mode, True), join_side_cols(rng, blengths, bm_mode, False)
    probe, build = cut(rng, pcols, plengths, sel_mode), cut(rng, bcols, blengths, sel_mode)
    for jt in (abi.JOIN_INNER, abi.JOIN_LEFT_OUTER):
        plan = JoinPlan(jt, LTYPES, RTYPES, [0], [0], lused=[3, 0, 2, 1], rused=[2, 1])
        want = join_reference(plan, [(v, nl) for v, nl, _ in pcols], [(v, nl) for v, nl, _ in bcols], flat=True)
        got, _ = run_join(plan, build, probe)
        assert_same_rows(want, got, f"{sel_mode}/{bm_mode} join type {jt} vs reference")
        canon, _ = run_join(plan, canonical(bcols), canonical(pcols))
        assert_same_rows(canon, got, f"{sel_mode}/{bm_mode} join type {jt} vs canonical layout")


# ---- join: staged chunks between direct pushes, and the paths they reach ----------------------------------------------
def unique_probe(rng, nb, npr, bitmaps):
    """build: unique keys with two INT payloads and a DECIMAL one; probe: key, row id, DECIMAL (all-valid bitmaps on
    every probe column when `bitmaps`)"""
    bkey = rng.permutation(nb).astype(np.int64) * 3 + 1
    pkey = np.where(rng.random(npr) < 0.7, bkey[rng.integers(0, nb, npr)], -5).astype(np.int64)
    b = [(bkey, np.zeros(nb, bool), None), (bkey * 5, np.zeros(nb, bool), None), (rng.integers(0, 256, (nb, 40), dtype=np.uint8), np.zeros(nb, bool), None)]
    p = [pkey, np.arange(npr, dtype=np.int64), rng.integers(0, 256, (npr, 40), dtype=np.uint8)]
    return b, p


def interleaved(rng, pvals, bitmaps):
    """probe chunks alternating between runs of 1023-row staged chunks with sel and >= 128 K-row direct pushes"""
    n = len(pvals[0])
    chunks, lo, k = [], 0, 0
    while lo < n:
        if k % 2 == 0:
            m = min(n - lo, 1023 * 40)
            lens = [1023] * (m // 1023) + ([m % 1023] if m % 1023 else [])
            cols = [(v[lo:lo + m], np.zeros(m, bool), [(np.zeros(x, bool), bitmaps, False) for x in lens]) for v in pvals]
            chunks += cut(rng, cols, lens, "subset")
        else:
            m = min(n - lo, DIRECT_ROWS + 4099)
            cols = [Column(v[lo:lo + m].copy()) for v in pvals]
            if bitmaps:
                for c in cols:
                    c.null_bitmap = np.full((m + 7) // 8, 0xFF, dtype=np.uint8)
            chunks.append(Chunk(cols))
        lo += m
        k += 1
    return chunks


@pytest.mark.parametrize("shape", ["uq", "direct", "general"])
def test_join_staged_and_direct_pushes_reach_each_path(shape):
    rng = np.random.default_rng(300 + ["uq", "direct", "general"].index(shape))
    nb, npr = 40_000, 3 * DIRECT_ROWS + 60_000
    bcols, pvals = unique_probe(rng, nb, npr, False)
    lt, rt = [INT_NN, INT_NN, DEC_NN], [INT_NN, INT_NN, DEC_NN]
    if shape == "uq":          # two 8-byte build payloads and a probe filter: k_probe_inner_uq
        plan = JoinPlan(abi.JOIN_INNER, lt, rt, [0], [0], lused=[0, 1], rused=[1, 0], probe_filter=[FilterItem(abi.CMP_GE, 1, const_i64=100)])
        path = abi.JOIN_PATH_PROBE_UQ
    elif shape == "direct":    # the DECIMAL cell is the only build payload: the fused warp probe over a U1 table
        plan, path = JoinPlan(abi.JOIN_INNER, lt, rt, [0], [0], lused=[0, 2, 1], rused=[2]), abi.JOIN_PATH_PROBE_DIRECT
    else:                      # left outer: count -> scan -> write
        plan, path = JoinPlan(abi.JOIN_LEFT_OUTER, [INT, INT, DEC], rt, [0], [0], lused=[2, 1], rused=[1, 2]), abi.JOIN_PATH_PROBE_GENERAL
    want = join_reference(plan, [(v, np.zeros(npr, bool)) for v in pvals], [(v, nl) for v, nl, _ in bcols], flat=True)
    build = cut(rng, bcols, [1023] * (nb // 1023) + [nb % 1023], "reversed")
    runs = {}
    for bitmaps in (False, True):
        probe = interleaved(rng, pvals, bitmaps)
        assert any(ch.sel is None and ch.num_rows() >= DIRECT_ROWS for ch in probe)
        got, st = run_join(plan, build, probe, windows=(1 << 17, 4096, 7))
        assert_same_rows(want, got, f"{shape}, all-valid bitmaps {bitmaps}")
        runs[bitmaps] = (got, st.paths)
    # the same rows with all-valid bitmaps and with none give the same result, whatever path each took
    assert_same_rows(runs[False][0], runs[True][0], f"{shape}: all-valid bitmaps vs none")
    assert runs[False][1] & path, hex(runs[False][1])
    if shape == "uq":          # a probe bitmap takes the UQ kernel out of play
        assert not runs[True][1] & abi.JOIN_PATH_PROBE_UQ, hex(runs[True][1])
    if shape == "general":
        assert runs[True][1] & path, hex(runs[True][1])


# ---- aggregation --------------------------------------------------------------------------------------------------
# columns: 0 g INT | 1 h INT (a few values) | 2 x DOUBLE (quarters) | 3 i INT | 4 d DECIMAL(15, 2)
ATYPES = [INT, INT, DBL, INT, DEC]
COMMON = [AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_COUNT, 2, abi.TYPE_DOUBLE), AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE),
          AggFunc(abi.AGG_MIN, 3), AggFunc(abi.AGG_MAX, 3),
          AggFunc(abi.AGG_SUM, 4, abi.TYPE_NEWDECIMAL, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=2),
          AggFunc(abi.AGG_MAX, 4, abi.TYPE_NEWDECIMAL, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=2)]


def agg_plan(kind):
    gb = {"nogroup": [], "v2": [0], "multi": [0, 1]}[kind]
    return AggPlan(ATYPES, gb, [AggFunc(abi.AGG_FIRSTROW, g) for g in gb] + COMMON, expected_groups=0)


def agg_values(rng, n, ngroups=500):
    return [rng.integers(0, ngroups, n).astype(np.int64), rng.integers(0, 3, n).astype(np.int64), quarters(rng, n),
            rng.integers(-10**12, 10**12, n), rng.integers(-10**9, 10**9, n)]


def agg_expected(plan, cols):
    """exact results per group key (None = NULL key): [count(*), count(x), sum(x), min(i), max(i), sum(d), max(d)], with
    the DECIMAL results as the cells the library must write"""
    (x, xn), (i, inn), (d, dn) = cols[2], cols[3], cols[4]
    n = len(x)
    if plan.group_by:
        km = np.stack([np.where(cols[g][1], 0, cols[g][0]) for g in plan.group_by] + [cols[g][1].astype(np.int64) for g in plan.group_by], axis=1)
        keys, inv = np.unique(km, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
    else:
        keys, inv = np.zeros((1, 0), dtype=np.int64), np.zeros(n, dtype=np.int64)
    ng = len(keys)
    cnt = np.bincount(inv, minlength=ng)
    cx = np.bincount(inv, weights=~xn, minlength=ng).astype(np.int64)
    sx = np.bincount(inv, weights=np.where(xn, 0.0, x), minlength=ng)
    mn, mx = np.full(ng, np.iinfo(np.int64).max), np.full(ng, np.iinfo(np.int64).min)
    np.minimum.at(mn, inv[~inn], i[~inn]); np.maximum.at(mx, inv[~inn], i[~inn])
    ci = np.bincount(inv[~inn], minlength=ng)
    sd, md = np.zeros(ng, dtype=np.int64), np.full(ng, np.iinfo(np.int64).min)
    np.add.at(sd, inv[~dn], d[~dn]); np.maximum.at(md, inv[~dn], d[~dn])
    cd = np.bincount(inv[~dn], minlength=ng)
    ngb = len(plan.group_by)
    out = {}
    for r in range(ng):
        key = tuple(None if keys[r, ngb + q] else int(keys[r, q]) for q in range(ngb))
        out[key] = [int(cnt[r]), int(cx[r]), float(sx[r]) if cx[r] else None, int(mn[r]) if ci[r] else None,
                    int(mx[r]) if ci[r] else None, A.sum_result(int(sd[r]), 2) if cd[r] else None, A.sum_result(int(md[r]), 2) if cd[r] else None]
    if not plan.group_by and n == 0:
        out = {(): [0, 0, None, None, None, None, None]}
    return out


def agg_rows(plan, got):
    ngb = len(plan.group_by)
    rows = {}
    for r in range(len(got[0][0])):
        vals = [None if nl[r] else (v[r].tobytes() if v.ndim == 2 else v[r].item()) for v, nl in got]
        key = tuple(vals[:ngb])
        assert key not in rows, f"group {key} emitted twice"
        rows[key] = vals[ngb:]
    return rows


def assert_agg(plan, cols, got, what):
    want, rows = agg_expected(plan, cols), agg_rows(plan, got)
    assert set(want) == set(rows), f"{what}: {len(rows)} groups, expected {len(want)}"
    for k, w in want.items():
        assert rows[k] == w, f"{what}: group {k}: got {rows[k]}, want {w}"


def sort_by_key(plan, got):
    ngb = len(plan.group_by)
    if not ngb or not len(got[0][0]):
        return got
    order = np.lexsort([np.where(got[q][1], np.iinfo(np.int64).min, got[q][0]) for q in reversed(range(ngb))] +
                       [got[q][1] for q in reversed(range(ngb))])
    return [(v[order], nl[order]) for v, nl in got]


def agg_cols(rng, lengths, mode, vals):
    cols = [logical(rng, lengths, v, mode, True) for v in vals]
    cols[4] = (dec_cells(cols[4][0]), cols[4][1], cols[4][2])
    return cols


def scaled(cols):
    """the reference's view: DECIMAL column 4 as its scaled integers"""
    return [(v, nl) for v, nl, _ in cols[:4]] + [(cols[4][3], cols[4][1])]


@pytest.mark.parametrize("sel_mode", SEL_MODES)
@pytest.mark.parametrize("bm_mode", BM_MODES)
def test_agg_layouts(sel_mode, bm_mode):
    rng = np.random.default_rng(400 + SEL_MODES.index(sel_mode) * 10 + BM_MODES.index(bm_mode))
    vals = agg_values(rng, sum(LENGTHS))
    cols = agg_cols(rng, LENGTHS, bm_mode, vals)
    ref = [(v, nl) for v, nl, _ in cols[:4]] + [(vals[4], cols[4][1])]
    chunks = cut(rng, cols, LENGTHS, sel_mode)
    plan = agg_plan("v2")
    got, st = run_agg(plan, chunks)
    assert st.paths & (abi.AGG_PATH_V2_GLOBAL | abi.AGG_PATH_V2_LOCAL), hex(st.paths)
    assert_agg(plan, ref, got, f"{sel_mode}/{bm_mode}")
    canon, _ = run_agg(plan, canonical(cols))
    assert_bitwise(sort_by_key(plan, canon), sort_by_key(plan, got), f"{sel_mode}/{bm_mode} vs canonical layout")


@pytest.mark.parametrize("kind", ["nogroup", "multi"])
def test_agg_staging_flush_at_odd_row_count_then_first_bitmaps(kind):
    # 1023-row chunks with (reversed) sel: staging crosses kStageBatchRows at 4101 * 1023 rows (= 3 mod 8) and is flushed;
    # columns h and x bring their first bitmap in the chunk right after the flush, g, i and d in the one after that
    # (staging row 1023: the lazy back-fill and a carry into a byte)
    rng = np.random.default_rng(500 + len(kind))
    k_flush = -(-STAGE_ROWS // 1023)
    assert (k_flush * 1023) % 8
    lengths = [1023] * (k_flush + 40)
    n = sum(lengths)
    vals = agg_values(rng, n, 700)
    cols = []
    for c, v in enumerate(vals):
        first = k_flush + (0 if c in (1, 2) else 1)
        nplan = [((rng.random(m) < 0.2) if q >= first else np.zeros(m, bool), q >= first, q % 5 == 0) for q, m in enumerate(lengths)]
        cols.append((v, np.concatenate([p[0] for p in nplan]), nplan))
    cols[4] = (dec_cells(vals[4]), cols[4][1], cols[4][2], vals[4])
    chunks = cut(rng, [c[:3] for c in cols], lengths, "reversed")
    plan = agg_plan(kind)
    got, st = run_agg(plan, chunks)
    del chunks
    assert st.paths & (abi.AGG_PATH_NOGROUP if kind == "nogroup" else abi.AGG_PATH_MULTI_KEY), hex(st.paths)
    assert st.input_rows == n
    assert_agg(plan, scaled(cols), got, kind)
    canon, _ = run_agg(plan, canonical([c[:3] for c in cols]))
    assert_bitwise(sort_by_key(plan, canon), sort_by_key(plan, got), f"{kind} vs canonical layout")


# ---- VecEval: filter through sel, compare / arith over every bitmap layout ------------------------------------------
@pytest.mark.parametrize("sel_mode", SEL_MODES)
@pytest.mark.parametrize("bm_mode", BM_MODES)
def test_vec_filter_layouts(sel_mode, bm_mode):
    rng = np.random.default_rng(600 + SEL_MODES.index(sel_mode) * 10 + BM_MODES.index(bm_mode))
    n = sum(LENGTHS)
    cols = [logical(rng, LENGTHS, rng.integers(-50, 50, n).astype(np.int64), bm_mode, True),
            logical(rng, LENGTHS, quarters(rng, n, 400), bm_mode, True), logical(rng, LENGTHS, rng.integers(-50, 50, n).astype(np.int64), bm_mode, True)]
    items = [FilterItem(abi.CMP_LE, 0, 2), FilterItem(abi.CMP_GT, 1, is_real=True, const_f64=-20.25)]
    want = V.filter_rows([(v.view(np.int64), nl) for v, nl, _ in cols], items)
    arr = (abi.TgFilterItem * 2)(*[it.to_struct() for it in items])
    lib, lo = abi.load_lib(), 0
    for ch in cut(rng, cols, LENGTHS, sel_mode):
        phys, m = ch.columns[0].length, ch.num_rows()
        selected = np.full(max(phys, 1), 0x5A, dtype=np.uint8)
        cnt = C.c_int64(-1)
        cs = ch.to_struct()
        abi.check(lib.tg_vec_filter(0, 0, C.byref(cs), arr, 2, C.c_void_p(selected.ctypes.data), C.byref(cnt), None))
        exp = np.zeros(phys, dtype=bool)
        idx = ch.sel if ch.sel is not None else np.arange(phys)
        exp[idx] = want[lo:lo + m]
        assert np.array_equal(selected[:phys].astype(bool), exp) and set(np.unique(selected[:phys])) <= {0, 1}
        assert cnt.value == int(exp.sum())
        lo += m
    assert lo == n


@pytest.mark.parametrize("bm_mode", BM_MODES)
@pytest.mark.parametrize("length", [1, 5, 7, 9, 1023, 1025, 4099])
def test_vec_compare_and_arith_bitmap_layouts(bm_mode, length):
    rng = np.random.default_rng(700 + length + BM_MODES.index(bm_mode))
    lib = abi.load_lib()
    mk = lambda v: logical(rng, [length], v, bm_mode, True)
    a, b = mk(rng.integers(-1000, 1000, length).astype(np.int64)), mk(rng.integers(-1000, 1000, length).astype(np.int64))
    x, y = mk(quarters(rng, length, 4000)), mk(quarters(rng, length, 4000))

    def col(c, canon):
        ch = canonical([c])[0] if canon else cut(rng, [c], [length], "none")[0]
        return ch.columns[0].to_struct(), ch

    def call(fn, p, q, real, op, kind):
        res = np.zeros(length, dtype=np.float64 if real and kind == "arith" else np.int64)
        nb = np.zeros((length + 7) // 8, dtype=np.uint8)
        args = (0, 0, op) + (() if real else (0, 0)) + (C.byref(p), C.byref(q), C.c_double(0) if real else C.c_int64(0),
                                                       C.c_void_p(res.ctypes.data), C.c_void_p(nb.ctypes.data), None)
        abi.check(fn(*args))
        return res, unpack_nulls(nb, length)

    for fn, (p, q), real, op, kind in ((lib.tg_vec_compare_int, (a, b), False, abi.CMP_LT, "cmp"), (lib.tg_vec_arith_int, (a, b), False, abi.ARITH_MINUS, "arith"),
                                       (lib.tg_vec_compare_real, (x, y), True, abi.CMP_GE, "cmp"), (lib.tg_vec_arith_real, (x, y), True, abi.ARITH_PLUS, "arith")):
        (sp, kp), (sq, kq) = col(p, False), col(q, False)
        got = call(fn, sp, sq, real, op, kind)
        (cp, kcp), (cq, kcq) = col(p, True), col(q, True)
        canon = call(fn, cp, cq, real, op, kind)
        if kind == "cmp":
            want = V.compare_real_col(op, p[0], p[1], q[0], q[1]) if real else V.compare_int_col(op, p[0], p[1], q[0], q[1])
        else:
            want = V.arith_real_vec(op, p[0], p[1], q[0], q[1])[1:3] if real else V.arith_int_vec(op, p[0], p[1], q[0], q[1])[1:3]
        wv, wn = np.asarray(want[0]), np.asarray(want[1], dtype=bool)
        assert np.array_equal(got[1], wn), f"{fn.__name__}: NULL flags"
        assert np.array_equal(got[0][~wn].view(np.int64), wv.astype(got[0].dtype)[~wn].view(np.int64)), f"{fn.__name__}: values"
        assert np.array_equal(canon[1], got[1]) and np.array_equal(canon[0][~wn].view(np.int64), got[0][~wn].view(np.int64))


# ---- device-resident inputs ------------------------------------------------------------------------------------------
def _bits(nl):
    import torch
    return torch.from_numpy(np.packbits(~nl, bitorder="little")).cuda()


def test_join_build_push_dev_bitmaps_on_byte_boundaries():
    import torch
    from tidb_b200.device import dev_chunk
    rng = np.random.default_rng(800)
    lengths = [16, 8, 13]                       # bitmaps start at rows 0, 16 and 24; the last is 29 rows in
    nb = sum(lengths)
    bkey = rng.permutation(nb).astype(np.int64)
    bpay, bnl = rng.integers(-99, 99, nb).astype(np.int64), rng.random(nb) < 0.3
    bnl[16:24] = False                          # the middle push brings no bitmap
    pkey = rng.integers(0, nb + 5, 3000).astype(np.int64)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT], [0], [0], lused=[1], rused=[1, 0])
    probe = [Chunk([Column(pkey), Column(np.arange(3000, dtype=np.int64))])]
    want = join_reference(plan, probe, [Chunk([Column(bkey), Column(bpay, bnl)])])
    j = Join(plan)
    lib = j.lib
    try:
        lo, keep = 0, []
        for q, m in enumerate(lengths):
            k, p = torch.from_numpy(bkey[lo:lo + m]).cuda(), torch.from_numpy(bpay[lo:lo + m]).cuda()
            nbits = _bits(bnl[lo:lo + m]) if q != 1 else None       # the middle push has no bitmap
            dc = dev_chunk([k, p], [None, nbits])
            keep.append(dc)
            torch.cuda.synchronize()
            abi.check(lib.tg_join_build_push_dev(j.h, C.byref(dc)))
            lo += m
        # a bitmap at row 37 (not a multiple of 8) is declined; the handle goes on as if it was never pushed
        extra = dev_chunk([torch.arange(10**6, 10**6 + 9, device="cuda"), torch.zeros(9, dtype=torch.int64, device="cuda")],
                          [None, _bits(np.zeros(9, bool))])
        assert lib.tg_join_build_push_dev(j.h, C.byref(extra)) == abi.TG_ERR_UNSUPPORTED
        # sel on a device entry point is declined too
        dc = dev_chunk([torch.arange(8, device="cuda"), torch.zeros(8, dtype=torch.int64, device="cuda")])
        sel = np.arange(4, dtype=np.int64)
        dc.sel, dc.nsel = sel.ctypes.data, 4
        assert lib.tg_join_build_push_dev(j.h, C.byref(dc)) == abi.TG_ERR_UNSUPPORTED
        abi.check(lib.tg_join_build_finish(j.h))
        j.probe(probe)
        got, _ = j.drain((1000, 3))
        assert j.stats().build_rows == nb
    finally:
        j.close()
    assert_same_rows(want, got, "device build pushes")


def test_agg_push_dev_odd_lengths_between_host_pushes():
    import torch
    from tidb_b200.device import dev_chunk
    rng = np.random.default_rng(810)
    lengths = [13, 1021, 5, 2039, 9, 7, 1025]
    vals = agg_values(rng, sum(lengths), 40)
    cols = agg_cols(rng, lengths, "stray", vals)
    ref = [(v, nl) for v, nl, _ in cols[:4]] + [(vals[4], cols[4][1])]
    plan = agg_plan("v2")
    a = Agg(plan)
    lib = a.lib
    try:
        lo, keep = 0, []
        host = [ch for ch in cut(rng, cols, lengths, "subset") if len(ch.sel)]    # without the empty-sel chunks
        for q, m in enumerate(lengths):
            if q % 2 == 0:                     # host pushes stay staged until the next device push flushes them
                a.push([host[q]])
            else:
                t = [torch.from_numpy(np.ascontiguousarray(v[lo:lo + m])).cuda() for v, _, _ in cols]
                nb = [_bits(nl[lo:lo + m]) for _, nl, _ in cols]
                dc = dev_chunk(t, nb)
                keep.append(dc)
                torch.cuda.synchronize()
                abi.check(lib.tg_agg_push_dev(a.h, C.byref(dc)))
            lo += m
        dc = dev_chunk([torch.zeros(8, dtype=torch.int64, device="cuda")] * 4 + [torch.zeros((8, 40), dtype=torch.uint8, device="cuda")])
        sel = np.arange(4, dtype=np.int64)
        dc.sel, dc.nsel = sel.ctypes.data, 4
        assert lib.tg_agg_push_dev(a.h, C.byref(dc)) == abi.TG_ERR_UNSUPPORTED
        a.finish()
        got, _ = a.drain()
    finally:
        a.close()
    assert_agg(plan, ref, got, "device and host pushes")


def test_device_entry_points_decline_sel():
    import torch
    from tidb_b200.device import dev_chunk
    lib = abi.load_lib()
    sel = np.arange(3, dtype=np.int64)
    t = torch.arange(8, dtype=torch.int64, device="cuda")
    dc = dev_chunk([t, t])
    dc.sel, dc.nsel = sel.ctypes.data, 3
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    j = Join(plan)
    try:
        j.build([Chunk([Column(np.arange(8, dtype=np.int64)), Column(np.arange(8, dtype=np.int64))])])
        rows = C.c_int64(0)
        ocols, onulls = (C.c_void_p * 4)(), (C.c_void_p * 4)()
        assert j.lib.tg_join_probe_dev(j.h, C.byref(dc), C.byref(rows), ocols, onulls) == abi.TG_ERR_UNSUPPORTED
    finally:
        j.close()
    # tg_topn takes no sel vector, on host or device columns
    hc = Chunk([Column(np.arange(8, dtype=np.int64))], np.arange(3, dtype=np.int64))
    out = MutChunk([8], 8, [np.int64])
    n = C.c_int64(0)
    cs = hc.to_struct()
    assert lib.tg_topn(0, 0, C.byref(cs), (C.c_int32 * 1)(abi.TYPE_LONGLONG), (C.c_uint32 * 1)(0), (abi.TgSortItem * 1)(abi.TgSortItem(0, 0)), 1,
                       C.c_int64(0), C.c_int64(3), C.byref(out.struct), C.byref(n), None) == abi.TG_ERR_UNSUPPORTED


# ---- output windows --------------------------------------------------------------------------------------------------
WINDOWS = [((3,), None), ((5, 1, 13), None), ((1 << 20,), 5), ((2,), 1), ((1 << 17, 11), None)]


@pytest.mark.parametrize("shape", ["general", "uq", "direct"])
def test_join_next_windows(shape):
    rng = np.random.default_rng(900 + len(shape))
    nb, npr = 3000, 9000
    bcols, pvals = unique_probe(rng, nb, npr, False)
    lt, rt = [INT_NN, INT_NN, DEC_NN], [INT_NN, INT_NN, DEC_NN]
    if shape == "general":     # nullable cells and NULL padding
        pn = rng.random(npr) < 0.2
        pcols = [(pvals[0], np.zeros(npr, bool)), (pvals[1], pn), (pvals[2], pn)]
        plan = JoinPlan(abi.JOIN_LEFT_OUTER, [INT, INT, DEC], rt, [0], [0], lused=[2, 1], rused=[2, 1, 0])
    else:
        pcols = [(v, np.zeros(npr, bool)) for v in pvals]
        plan = JoinPlan(abi.JOIN_INNER, lt, rt, [0], [0], lused=[0, 1], rused=[1, 0]) if shape == "uq" else \
            JoinPlan(abi.JOIN_INNER, lt, rt, [0], [0], lused=[2, 1], rused=[2])
    want = join_reference(plan, pcols, [(v, nl) for v, nl, _ in bcols], flat=True)
    probe = [Chunk([Column(v, nl if nl.any() else None) for v, nl in pcols])]
    build = canonical(bcols)
    for windows, cap in WINDOWS:
        j = Join(plan)
        try:
            j.build(build)
            j.probe(probe)
            got, starts = j.drain(windows, cap)
        finally:
            j.close()
        assert_same_rows(want, got, f"{shape} windows {windows} capacity {cap}")
        if cap is None and max(windows) < 64:
            assert starts == set(range(8)), starts


@pytest.mark.parametrize("kind", ["v2", "nogroup_empty", "nogroup"])
def test_agg_next_windows(kind):
    rng = np.random.default_rng(950 + len(kind))
    n = 0 if kind == "nogroup_empty" else 12_000
    vals = agg_values(rng, n, 3000)
    cols = agg_cols(rng, [n], "stray", vals)
    ref = [(v, nl) for v, nl, _ in cols[:4]] + [(vals[4], cols[4][1])]
    plan = agg_plan("v2" if kind == "v2" else "nogroup")
    chunks = canonical(cols)
    for windows, cap in WINDOWS:
        a = Agg(plan)
        try:
            a.push(chunks)
            a.finish()
            got, starts = a.drain(windows, cap)
        finally:
            a.close()
        assert_agg(plan, ref, got, f"{kind} windows {windows} capacity {cap}")
        if kind == "v2" and cap is None and max(windows) < 64:
            assert starts == set(range(8)), starts


# ---- failure atomicity of rejected output calls ----------------------------------------------------------------------
SENTINEL = 0x5C


def sentinel_out(elems, dts, cap, drop_bitmap=None):
    out = MutChunk(elems, cap, dts)
    for d in out.data:
        d.view(np.uint8)[...] = SENTINEL
    for b in out.bitmaps:
        b[:] = SENTINEL
    if drop_bitmap is not None:
        out._cols[drop_bitmap].null_bitmap = None
    return out


def assert_untouched(out):
    for c, d in enumerate(out.data):
        assert (d.view(np.uint8) == SENTINEL).all(), f"column {c}: data written by a rejected call"
    for c, b in enumerate(out.bitmaps):
        assert (b == SENTINEL).all(), f"column {c}: bitmap written by a rejected call"


def bad_outputs(dts, nullable_col):
    """(name, elem_lens, dtypes, column without a bitmap) of every malformed output chunk: a nullable column without a
    bitmap, and an elem_len mismatch on each column (8 <-> 40, 8 -> 4), the last one included"""
    elems = [np.dtype(d).itemsize for d in dts]
    yield "nullable without bitmap", elems, dts, nullable_col
    for c in range(len(dts)):
        e, d = list(elems), list(dts)
        e[c], d[c] = (8, np.int64) if elems[c] == 40 else (40, DECIMAL_DTYPE)
        yield f"elem_len {e[c]} on column {c}", e, d, None
        if elems[c] == 8:
            e[c], d[c] = 4, np.float32
            yield f"elem_len 4 on column {c}", e, d, None


def check_rejections(next_fn, h, dts, nullable_col, stats, fresh_rows):
    """every malformed output rejected with nothing written, then the next valid call returns what a fresh handle gives"""
    lib = abi.load_lib()
    for window in (1000, 70_000):
        for name, elems, d, drop in bad_outputs(dts, nullable_col):
            out = sentinel_out(elems, d, 2 * window, drop)    # room for window rows of 8 bytes where 4 are declared
            before = stats()
            n = C.c_int64(-1)
            rc = next_fn(h, C.byref(out.struct), C.c_int64(window), C.byref(n))
            abi.check(lib.tg_device_synchronize(0))
            assert rc == abi.TG_ERR_INVALID, f"{name}, window {window}: rc {rc}"
            assert n.value == 0, name
            assert_untouched(out)
            assert stats().d2h_bytes == before.d2h_bytes, f"{name}: d2h_bytes moved"
    got, _ = drain(next_fn, h, dts, (1000, 70_000))
    assert_same_rows(fresh_rows, got, "after rejected calls")


def test_join_rejected_next_writes_nothing():
    rng = np.random.default_rng(1000)
    nb, npr = 50_000, 150_000
    bcols, pvals = unique_probe(rng, nb, npr, False)
    pn = rng.random(npr) < 0.1
    plan = JoinPlan(abi.JOIN_LEFT_OUTER, [INT, INT, DEC], [INT_NN, INT_NN, DEC_NN], [0], [0], lused=[1, 2], rused=[1, 2])
    probe = [Chunk([Column(pvals[0]), Column(pvals[1], pn), Column(pvals[2], pn)])]
    build = canonical(bcols)
    dts = out_dtypes(plan.out_schema())
    ordered = []
    for _ in range(2):     # the same pushes give the same batches: a fresh handle's rows, in its order
        j = Join(plan)
        try:
            j.build(build)
            j.probe(probe)
            if not ordered:
                ordered, _ = j.drain((1000, 70_000))
                continue
            check_rejections(j.lib.tg_join_next, j.h, dts, 0, j.stats, ordered)
        finally:
            j.close()


def test_agg_rejected_next_writes_nothing():
    rng = np.random.default_rng(1010)
    n = 400_000
    vals = agg_values(rng, n, 150_000)
    cols = agg_cols(rng, [n], "stray", vals)
    plan = agg_plan("v2")
    a = Agg(plan)
    dts = a.dtypes()
    try:
        a.push(canonical(cols))
        a.finish()
        fresh, _ = a.drain((1000, 70_000))
    finally:
        a.close()
    a = Agg(plan)
    try:
        a.push(canonical(cols))
        a.finish()
        check_rejections(a.lib.tg_agg_next, a.h, dts, 3, a.stats, fresh)
    finally:
        a.close()


def test_agg_next_rejects_any_elem_len_mismatch():
    # an 8-byte result passed as 4 bytes would get twice its buffer; passed as 40 it would get packed 8-byte values
    rng = np.random.default_rng(1020)
    vals = agg_values(rng, 5000, 100)
    plan = AggPlan(ATYPES, [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE)])
    a = Agg(plan)
    try:
        a.push([Chunk([Column(v) for v in vals[:4]] + [Column(dec_cells(vals[4]))])])
        a.finish()
        for c in range(3):
            for el, dt in ((4, np.float32), (40, DECIMAL_DTYPE)):
                elems, dts = [8, 8, 8], [np.int64, np.int64, np.float64]
                elems[c], dts[c] = el, dt
                out = sentinel_out(elems, dts, 32)    # max_rows 16: room for 16 rows of 8 bytes where 4 are declared
                n = C.c_int64(-1)
                assert a.lib.tg_agg_next(a.h, C.byref(out.struct), C.c_int64(16), C.byref(n)) == abi.TG_ERR_INVALID, (c, el)
                assert n.value == 0
                assert_untouched(out)
        got, _ = a.drain((16,))
        assert len(got[0][0]) == 100
    finally:
        a.close()


def test_topn_rejected_call_writes_nothing():
    rng = np.random.default_rng(1030)
    n = 5000
    key = rng.permutation(n).astype(np.int64) * 7 - 1000
    pay, pn = rng.integers(-99, 99, n).astype(np.int64), rng.random(n) < 0.5
    dec = dec_cells(rng.integers(-10**6, 10**6, n))
    bad_dec = dec.copy()
    bad_dec[77, 4:8] = np.frombuffer(np.int32(10**9).tobytes(), dtype=np.uint8)   # a word >= 10^9
    lib = abi.load_lib()
    types = (C.c_int32 * 3)(abi.TYPE_LONGLONG, abi.TYPE_LONGLONG, abi.TYPE_NEWDECIMAL)
    flags = (C.c_uint32 * 3)(0, 0, 0)
    dts = [np.int64, np.int64, DECIMAL_DTYPE]

    def call(dcol, items, count, elems, d, cap, drop=None):
        chk = Chunk([Column(key), Column(pay, pn), Column(dcol)])
        cs = chk.to_struct()
        out = sentinel_out(elems, d, cap, drop)
        nr = C.c_int64(-1)
        it = (abi.TgSortItem * len(items))(*[abi.TgSortItem(c, 0) for c in items])
        rc = lib.tg_topn(0, 0, C.byref(cs), types, flags, it, len(items), C.c_int64(10), C.c_int64(count), C.byref(out.struct), C.byref(nr), None)
        return rc, nr.value, out

    cases = [("capacity below count", dec, [0], 100, [8, 8, 40], dts, 99, None, abi.TG_ERR_CAPACITY),
             ("malformed DECIMAL item", bad_dec, [2, 0], 100, [8, 8, 40], dts, 100, None, abi.TG_ERR_INVALID),
             ("NULL payload without bitmap", dec, [0], 100, [8, 8, 40], dts, 100, 1, abi.TG_ERR_INVALID),
             ("elem_len 8 on the last (DECIMAL) column", dec, [0], 100, [8, 8, 8], [np.int64] * 3, 100, None, abi.TG_ERR_INVALID),
             ("elem_len 40 on the middle column", dec, [0], 100, [8, 40, 40], [np.int64, DECIMAL_DTYPE, DECIMAL_DTYPE], 100, None, abi.TG_ERR_INVALID)]
    for name, dcol, items, count, elems, d, cap, drop, code in cases:
        rc, nr, out = call(dcol, items, count, elems, d, cap, drop)
        abi.check(lib.tg_device_synchronize(0))
        assert rc == code, f"{name}: rc {rc}"
        assert nr == 0, name
        assert_untouched(out)
    # the valid call: rows 10 .. 109 in key order
    rc, nr, out = call(dec, [0], 100, [8, 8, 40], dts, 100)
    assert rc == 0 and nr == 100
    order = np.argsort(key, kind="stable")[10:110]
    assert np.array_equal(out.data[0][:100], key[order])
    assert np.array_equal(unpack_nulls(out.bitmaps[1], 100), pn[order])
    assert np.array_equal(out.data[1][:100][~pn[order]], pay[order][~pn[order]])
    assert np.array_equal(out.data[2][:100], dec[order])
