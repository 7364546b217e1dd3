"""SUM / AVG / MIN / MAX / COUNT over DECIMAL(p <= 18, s) columns on every update path of the CUDA hash aggregation,
compared exactly.

Each case forces one path through the TG_AGG_* switches, proves from tg_agg_stats.paths / local_rows that it ran, and
compares every group's 40-byte MyDecimal cell byte for byte with the exact answer of tests/mydecimal_args.py.  Input cells
come in the stored form and its variants (digitsInt 0, leading zero integer words, negative zeros, any resultFrac), with
garbage bytes under NULL.  The data holds groups of +-(10^p - 1) whose sums pass 2^64, groups that cancel to 0, all-NULL
groups, and the DECIMAL functions mixed with DOUBLE SUM, COUNT, an integer DECIMAL SUM and integer MIN / MAX (those are
checked with tests/agg_reference.py)."""
import ctypes as C
import functools
from fractions import Fraction

import numpy as np
import pytest

import agg_reference as R
import mydecimal as D
import mydecimal_args as A
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column, MutChunk, unpack_nulls
from tidb_b200.executor import HashAggExec, MockDataSource
from tidb_b200.plan import AggFunc, AggPlan, FieldType

pytestmark = pytest.mark.gpu

P = abi
DEC = abi.TYPE_NEWDECIMAL
INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
SWITCHES = ("TG_AGG_LOCAL", "TG_AGG_LOCAL_SLOTS", "TG_AGG_V1")
K_MAX, K_MIN, K_CANCEL, K_ALLNULL = (7_000_000_000_000 + j for j in range(4))
SCALES = [(18, 0), (18, 2), (18, 9), (18, 18), (15, 2)]


@pytest.fixture(autouse=True)
def _default_switches(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)


# ---- data --------------------------------------------------------------------------------------------------------
# columns: 0 g BIGINT key (nullable) | 1 a DECIMAL(p, s) (nullable, garbage under NULL) | 2 b DECIMAL(p, s) NOT NULL
#          3 i BIGINT (nullable, full range) | 4 d DOUBLE (nullable)
def types_of(p, s):
    return [INT, FieldType(DEC, 0, p, s), FieldType(DEC, abi.FLAG_NOT_NULL, p, s), INT, DBL]


def dec_values(rng, n, p, s):
    lim = 10 ** p - 1
    v = rng.integers(-lim, lim, n, endpoint=True, dtype=np.int64)
    small = rng.random(n) < 0.2                      # below 1: digitsInt may be 0
    v[small] = rng.integers(-(10 ** s) + 1, 10 ** s, int(small.sum())) if s else 0
    v[rng.random(n) < 0.02] = 0
    return v


def encode(rng, v, p, s, nulls=None):
    """stored cells with random header variants: digitsInt = the digits needed (0 for a value below 1), FromBin's p - s, or
    every integer word there is (leading zero words); any resultFrac; a negative zero on half of the zeros"""
    n = len(v)
    ip = np.abs(v) // 10 ** s
    need = np.where(ip > 0, np.char.str_len(ip.astype(str)), 0)
    choice = rng.integers(0, 3, n)
    di = np.where(choice == 0, need, np.where(choice == 1, p - s, 9 * (9 - (s + 8) // 9)))
    di = np.maximum(di, need)
    neg = (v < 0) | ((v == 0) & (rng.random(n) < 0.5))
    cells = A.cells_np(v, p, s, di, rng.integers(0, 31, n), neg)
    if nulls is not None:
        cells[nulls] = rng.integers(0, 256, (int(nulls.sum()), 40), dtype=np.uint8)   # garbage under NULL
    return cells


def make_rows(rng, n, ngroups, p, s):
    """-> (Chunk, {column: (int64 values * 10^s or integers, nulls)}) with the special groups"""
    lim = 10 ** p - 1
    g = (rng.integers(0, ngroups, n) * 2654435761 % (1 << 40) - (1 << 39)).astype(np.int64)
    sp = rng.random(n) < 0.04
    g[sp] = rng.choice(np.array([K_MAX, K_MIN, K_CANCEL, K_ALLNULL], dtype=np.int64), int(sp.sum()))
    gn = rng.random(n) < 0.01
    g[gn] = 0
    a, b = dec_values(rng, n, p, s), dec_values(rng, n, p, s)
    for k, val in ((K_MAX, lim), (K_MIN, -lim)):    # >= 19 rows of 10^18 - 1: the sum passes 2^64
        a[(g == k) & ~gn] = val; b[(g == k) & ~gn] = val
    idx = np.flatnonzero((g == K_CANCEL) & ~gn)      # x / -x pairs: the group's sum is exactly 0
    for col in (a, b):
        col[idx[1::2]] = -col[idx[0:len(idx) // 2 * 2:2]]
        if len(idx) % 2:
            col[idx[-1]] = 0
    an = (rng.random(n) < 0.05) | ((g == K_ALLNULL) & ~gn)
    i = rng.integers(-(1 << 63), (1 << 63) - 1, n, endpoint=True, dtype=np.int64)
    inl = rng.random(n) < 0.05
    d = rng.standard_normal(n) * 1e3
    dn = rng.random(n) < 0.05
    chunk = Chunk([Column(g, gn), Column(encode(rng, a, p, s, an), an), Column(encode(rng, b, p, s)), Column(i, inl), Column(d, dn)])
    return chunk, {0: (g, gn), 1: (a, an), 2: (b, np.zeros(n, dtype=bool)), 3: (i, inl), 4: (d, dn)}


@functools.lru_cache(maxsize=None)
def dataset(p, s, n=120_000, ngroups=5000, seed=0):
    return make_rows(np.random.default_rng(seed + 31 * p + s), n, ngroups, p, s)


def fracs(s):
    """the AVG scales every test covers: s + 4, 30, and a multiple of 9 (the truncation case)"""
    return min(s + 4, 30), 30, max(9, 9 * ((s + 8) // 9))


def dsum(c, s):
    return AggFunc(P.AGG_SUM, c, DEC, ret_type=DEC, ret_frac=s)


def davg(c, f):
    return AggFunc(P.AGG_AVG, c, DEC, ret_type=DEC, ret_frac=f)


def dmin(c, s):
    return AggFunc(P.AGG_MIN, c, DEC, ret_type=DEC, ret_frac=s)


def dmax(c, s):
    return AggFunc(P.AGG_MAX, c, DEC, ret_type=DEC, ret_frac=s)


def plans(p, s, group_by=(0,), expected_groups=0, local=True):
    """lists of at most 4 device states (the CTA-local level takes no more), and with local=False one plan mixing the
    DECIMAL functions with DOUBLE SUM, COUNT, an integer DECIMAL SUM and integer MIN / MAX"""
    f1, f2, f3 = fracs(s)
    fr = [AggFunc(P.AGG_FIRSTROW, g) for g in group_by]
    lists = [[dsum(1, s)], [dsum(2, s), davg(2, f1)], [davg(1, f2)], [dmin(1, s), dmax(2, s), AggFunc(P.AGG_COUNT, 1)],
             [davg(1, f3)], [dmax(1, s), davg(2, f2)], [dmin(2, s)]]
    if not local:
        lists.append([dsum(1, s), davg(1, f1), dmin(2, s), dmax(1, s), AggFunc(P.AGG_COUNT, 1), AggFunc(P.AGG_SUM, 4, P.TYPE_DOUBLE),
                      AggFunc(P.AGG_SUM, 3, ret_type=DEC), AggFunc(P.AGG_MIN, 3), AggFunc(P.AGG_MAX, 3), AggFunc(P.AGG_COUNT, -1),
                      davg(2, f3)])
    cols = types_of(p, s)
    return [AggPlan(cols, list(group_by), fr + fs, expected_groups=expected_groups) for fs in lists]


# ---- exact reference ---------------------------------------------------------------------------------------------
def _group_ids(plan, vals):
    n = len(vals[1][0])
    if not plan.group_by:
        return np.zeros(n, dtype=np.int64), [()]
    k = np.stack([a for g in plan.group_by for a in (vals[g][1].astype(np.int64), np.where(vals[g][1], 0, vals[g][0]))], axis=1)
    uk, inv = np.unique(k, axis=0, return_inverse=True)
    return inv.ravel(), [tuple(None if r[2 * j] else int(r[2 * j + 1]) for j in range(len(plan.group_by))) for r in uk]


def dec_expected(plan, vals):
    """group key tuple -> {function index: expected cell or None} for every function with a DECIMAL result.  Sums are exact:
    the 32-bit halves are summed per group as float64, exact while a group has fewer than 2^21 rows"""
    inv, tuples = _group_ids(plan, vals)
    ng = len(tuples)
    assert len(inv) < (1 << 21)
    out = {t: {} for t in tuples}
    for k, f in enumerate(plan.funcs):
        if f.ret_type != DEC:
            continue
        t = plan.col_types[f.arg_col]
        s = t.decimal if t.tp == DEC else 0
        v, nl = vals[f.arg_col]
        keep = ~nl
        cnt = np.bincount(inv[keep], minlength=ng)
        if f.name in (P.AGG_SUM, P.AGG_AVG):
            lo = np.bincount(inv[keep], weights=(v[keep] & 0xFFFFFFFF).astype(np.float64), minlength=ng)
            hi = np.bincount(inv[keep], weights=(v[keep] >> 32).astype(np.float64), minlength=ng)
            agg = [(int(hi[j]) << 32) + int(lo[j]) for j in range(ng)]
        else:
            big = np.full(ng, np.iinfo(np.int64).max if f.name == P.AGG_MIN else np.iinfo(np.int64).min, dtype=np.int64)
            (np.minimum if f.name == P.AGG_MIN else np.maximum).at(big, inv[keep], v[keep])
            agg = big.tolist()
        for j, tup in enumerate(tuples):
            if cnt[j] == 0:
                out[tup][k] = None
            elif f.name == P.AGG_AVG:
                out[tup][k] = A.avg_result(agg[j], int(cnt[j]), s, f.ret_frac)
            else:
                out[tup][k] = A.sum_result(agg[j], s)
    return out


def check(plan, vals, got_rows):
    """every group's DECIMAL cells equal the exact answer's; the other functions through tests/agg_reference.py"""
    exp = dec_expected(plan, vals)
    got = {}
    for r in got_rows:
        k = R.result_key(plan, r) if plan.group_by else ()
        assert k not in got, f"group {k} emitted twice"
        got[k] = r
    assert set(got) == set(exp), sorted(set(map(repr, exp)) ^ set(map(repr, got)))[:10]
    for key, want in exp.items():
        for k, cell in want.items():
            g = got[key][k]
            if cell is None or g is None:
                assert cell is None and g is None, (key, k, g if g is None else D.to_string(g))
                continue
            assert g == cell, f"group {key!r} aggregate {k}: got {D.to_string(g)} {D.decode(g)}, want {D.to_string(cell)} {D.decode(cell)}"
    others = [k for k, f in enumerate(plan.funcs) if f.ret_type != DEC]
    if any(plan.funcs[k].name != P.AGG_FIRSTROW for k in others):
        # the reference reads only the nulls of a DECIMAL column (COUNT): hand it int64 stand-ins
        cols = [Column(np.zeros(len(v), dtype=np.int64) if plan.col_types[c].tp == DEC else v, nl) for c, (v, nl) in sorted(vals.items())]
        sub = AggPlan(plan.col_types, plan.group_by, [plan.funcs[k] for k in others])
        R.check(sub, [Chunk(cols)], [tuple(r[k] for k in others) for r in got_rows])
    return len(exp)


def rows_of(chunk):
    cols = []
    for col in chunk.columns:
        nl = col.nulls()
        if col.data.ndim == 2:
            cols.append([None if nl[r] else bytes(col.data[r]) for r in range(col.length)])
        else:
            cols.append([None if x else v for v, x in zip(col.data.tolist(), nl.tolist())])
    return list(zip(*cols))


# ---- running ---------------------------------------------------------------------------------------------------
def run_host(plan, chunks, page=1 << 20):
    e = HashAggExec(plan, MockDataSource(plan.col_types, chunks))
    e.open()
    try:
        rows = []
        while True:
            c = e.next(page)
            if c.num_rows() == 0:
                break
            rows.extend(rows_of(c))
        return rows, e.stats()
    finally:
        e.close()


def dev_columns(chunk, misalign=False):
    """device copies of the chunk's columns; misalign=True puts DECIMAL columns at 8 bytes past a 16-byte boundary"""
    import torch
    keep, cs = [], (abi.TgColumn * len(chunk.columns))()
    for c, col in enumerate(chunk.columns):
        raw = np.ascontiguousarray(col.data).view(np.uint8).ravel()
        if col.data.ndim == 2 and misalign:
            buf = torch.zeros(raw.size + 8, dtype=torch.uint8, device="cuda")
            buf[8:] = torch.from_numpy(raw).cuda()
            ptr = buf.data_ptr() + 8
            assert ptr % 16 == 8
        else:
            buf = torch.from_numpy(raw).cuda()
            ptr = buf.data_ptr()
        keep.append(buf)
        cs[c].length, cs[c].data, cs[c].elem_len = col.length, ptr, col.elem_len
        if col.null_bitmap is not None:
            nb = torch.from_numpy(np.ascontiguousarray(col.null_bitmap)).cuda(); keep.append(nb)
            cs[c].null_bitmap = nb.data_ptr()
    chk = abi.TgChunk(); chk.ncols = len(chunk.columns); chk.cols = C.cast(cs, C.POINTER(abi.TgColumn))
    torch.cuda.synchronize()
    return chk, (keep, cs)


def run_dev(plan, batches, misalign=False):
    e = HashAggExec(plan, MockDataSource(plan.col_types, []))
    e.open()
    try:
        lib = abi.load_lib()
        for b in batches:
            chk, keep = dev_columns(b, misalign)
            abi.check(lib.tg_agg_push_dev(e._h, C.byref(chk)))
        rows = []
        while True:
            c = e.next(1 << 20)
            if c.num_rows() == 0:
                break
            rows.extend(rows_of(c))
        return rows, e.stats()
    finally:
        e.close()


def check_all(plan_list, chunks, vals, want, dont=0, local=None):
    st = None
    for plan in plan_list:
        rows, st = run_host(plan, chunks)
        check(plan, vals, rows)
        assert st.paths & want == want, (hex(st.paths), hex(want))
        assert st.paths & dont == 0, (hex(st.paths), hex(dont))
        if local is not None:
            assert (st.local_rows > 0) == local, st.local_rows
    return st


# ---- paths -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p,s", SCALES)
def test_no_group_by(p, s):
    chunk, vals = dataset(p, s)
    check_all(plans(p, s, group_by=(), local=False), chunk.split(1 << 15), vals, want=P.AGG_PATH_NOGROUP, dont=~P.AGG_PATH_NOGROUP)


@pytest.mark.parametrize("p,s", SCALES)
def test_v2_global(p, s, monkeypatch):
    monkeypatch.setenv("TG_AGG_LOCAL", "0")
    chunk, vals = dataset(p, s)
    check_all(plans(p, s, local=False), chunk.split(1 << 15), vals, want=P.AGG_PATH_V2_GLOBAL,
              dont=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE, local=False)


@pytest.mark.parametrize("p,s", SCALES)
def test_v2_cta_local(p, s):
    rng = np.random.default_rng(40 + s)
    chunk, vals = make_rows(rng, 150_000, 60, p, s)
    check_all(plans(p, s), chunk.split(1 << 15), vals, want=P.AGG_PATH_V2_LOCAL, local=True)


@pytest.mark.parametrize("p,s", [(18, 2), (15, 2)])
def test_v2_local_spills_and_merges(p, s, monkeypatch):
    monkeypatch.setenv("TG_AGG_LOCAL", "2")
    chunk, vals = dataset(p, s)
    st = check_all(plans(p, s, expected_groups=64), chunk.split(1 << 16), vals, want=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE, local=True)
    assert st.table_slots > 1024


@pytest.mark.parametrize("p,s", SCALES)
def test_multi_key(p, s):
    rng = np.random.default_rng(50 + s)
    chunk, vals = make_rows(rng, 150_000, 50, p, s)
    n = chunk.num_rows()
    k2 = rng.integers(-3, 4, n).astype(np.int64)
    chunk = Chunk([chunk.columns[0], Column(k2)] + chunk.columns[1:])
    vals = {0: vals[0], 1: (k2, np.zeros(n, dtype=bool)), **{c + 1: vals[c] for c in range(1, 5)}}
    pl = []
    for plan in plans(p, s, local=False):
        shift = [f if f.arg_col < 0 else AggFunc(f.name, f.arg_col + (f.arg_col >= 1), f.arg_type, f.arg_flag, f.mode, ret_type=f.ret_type,
                                                     ret_frac=f.ret_frac) for f in plan.funcs[1:]]
        shift = [f for f in shift if not (f.name == P.AGG_COUNT and f.arg_col < 0)]   # two FIRSTROWs: at most 12 functions
        pl.append(AggPlan([INT, INT_NN] + types_of(p, s)[1:], [0, 1], [AggFunc(P.AGG_FIRSTROW, 0), AggFunc(P.AGG_FIRSTROW, 1)] + shift,
                          expected_groups=16))
    check_all(pl, chunk.split(1 << 15), vals, want=P.AGG_PATH_MULTI_KEY, dont=~P.AGG_PATH_MULTI_KEY)


@pytest.mark.parametrize("ngroups,hint,want", [(60, 0, P.AGG_PATH_V1_LOCAL | P.AGG_PATH_MERGE),
                                               (60_000, 60_000, P.AGG_PATH_V1_GLOBAL)])
@pytest.mark.parametrize("p,s", [(18, 9), (15, 2)])
def test_v1_paths(ngroups, hint, want, p, s, monkeypatch):
    monkeypatch.setenv("TG_AGG_V1", "1")
    monkeypatch.setenv("TG_AGG_LOCAL_SLOTS", "512")
    rng = np.random.default_rng(60 + ngroups + s)
    chunk, vals = make_rows(rng, 150_000, ngroups, p, s)
    v2 = P.AGG_PATH_V2_LOCAL | P.AGG_PATH_V2_GLOBAL
    check_all(plans(p, s, expected_groups=hint), chunk.split(1 << 15), vals, want=want, dont=v2, local=False)


# ---- input routes ------------------------------------------------------------------------------------------------
def _concat(parts):
    return {c: (np.concatenate([v[c][0] for v in parts]), np.concatenate([v[c][1] for v in parts])) for c in parts[0]}


@pytest.mark.parametrize("misalign", [False, True])
def test_device_pushes(misalign):
    p, s = 15, 2
    rng = np.random.default_rng(70 + misalign)
    parts = [make_rows(rng, n, g, p, s) for n, g in ((50_001, 30), (100_000, 3000), (99_999, 30_000))]
    vals = _concat([v for _, v in parts])
    for plan in plans(p, s, expected_groups=16, local=False)[::2]:
        rows, st = run_dev(plan, [c for c, _ in parts], misalign)
        check(plan, vals, rows)
        assert st.table_slots > 1024
    plan = plans(p, s, group_by=(), local=False)[-1]
    rows, _ = run_dev(plan, [c for c, _ in parts], misalign)
    check(plan, vals, rows)


def test_host_pushes_with_sel_skip_unselected_cells():
    # the rows a sel vector leaves out hold cells in no valid form: they must never reach the decoder
    p, s = 18, 9
    rng = np.random.default_rng(80)
    chunk, vals = make_rows(rng, 120_000, 500, p, s)
    n = chunk.num_rows()
    phys = 2 * n
    cols = []
    for c, col in enumerate(chunk.columns):
        if col.data.ndim == 2:
            data = rng.integers(0, 256, (phys, 40), dtype=np.uint8)
            data[:, 1] = 77                              # digitsFrac != s
        else:
            data = rng.integers(-5, 5, phys).astype(col.data.dtype)
        data[0::2] = col.data
        nl = np.zeros(phys, dtype=bool)
        nl[0::2] = col.nulls()
        cols.append(Column(data, nl))
    big = Chunk(cols)
    chunks = []
    for lo in range(0, phys, 1 << 14):
        part = Chunk([c.slice(lo, min(phys, lo + (1 << 14))) for c in big.columns])
        chunks.append(Chunk(part.columns, np.arange(0, part.num_rows(), 2)))
    check_all(plans(p, s), chunks, vals, want=P.AGG_PATH_V2_LOCAL)
    check_all(plans(p, s, local=False)[-1:], chunks, vals, want=P.AGG_PATH_V2_GLOBAL)


def test_paging_and_result_dev():
    p, s = 18, 2
    chunk, vals = dataset(p, s)
    chunks = chunk.split(1 << 15)
    plan = AggPlan(types_of(p, s), [0], [AggFunc(P.AGG_FIRSTROW, 0), dsum(1, s), AggFunc(P.AGG_COUNT, -1), davg(2, 6), dmin(1, s)],
                   expected_groups=5000)
    rows, _ = run_host(plan, chunks, page=37)          # 37-row pages: cells and bitmaps start inside a byte
    assert check(plan, vals, rows) > 5000
    lib = abi.load_lib()
    e = HashAggExec(plan, MockDataSource(plan.col_types, chunks))
    e.open()
    try:
        e.next(8)
        # every DECIMAL result column needs 40-byte cells: an 8-byte one is refused
        bad = MutChunk([8, 40, 8, 40, 8], 16, [np.int64, np.dtype((np.uint8, 40)), np.int64, np.dtype((np.uint8, 40)), np.int64])
        n = C.c_int64(0)
        assert lib.tg_agg_next(e._h, C.byref(bad.struct), C.c_int64(16), C.byref(n)) == abi.TG_ERR_INVALID
        assert b"elem_len 40" in lib.tg_last_error()
        nrows = C.c_int64(0)
        cols = (C.c_void_p * 5)(); nulls = (C.c_void_p * 5)()
        abi.check(lib.tg_agg_result_dev(e._h, C.byref(nrows), cols, nulls))
        m = nrows.value
        keys = np.zeros(m, dtype=np.int64)
        abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(keys.ctypes.data), C.c_void_p(cols[0]), C.c_size_t(m * 8)))
        knb = np.zeros((m + 7) // 8, dtype=np.uint8)
        abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(knb.ctypes.data), C.c_void_p(nulls[0]), C.c_size_t(len(knb))))
        kn = unpack_nulls(knb, m)
        exp = dec_expected(plan, vals)
        for k in (1, 3, 4):
            host = np.zeros((m, 40), dtype=np.uint8)
            abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(host.ctypes.data), C.c_void_p(cols[k]), C.c_size_t(m * 40)))
            nb = np.zeros((m + 7) // 8, dtype=np.uint8)
            abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(nb.ctypes.data), C.c_void_p(nulls[k]), C.c_size_t(len(nb))))
            sn = unpack_nulls(nb, m)
            for r in range(m):
                key = (None if kn[r] else int(keys[r]),)
                assert (None if sn[r] else bytes(host[r])) == exp[key][k], (key, k)
    finally:
        e.close()


# ---- known answers and AVG rounding on the device ------------------------------------------------------------------
def test_known_answers():
    # NewDecFromInt(0..4) then a second partial {2, 3, 4} (func_sum_test.go:30, func_avg_test.go:29, func_max_min_test.go:113,
    # :125); max(b) of DECIMAL(15,2) (aggregate.result:1085); sum of DECIMAL(10,4) 0, -0.9871, -0.9871 twice (:1168)
    g = np.array([0] * 5 + [1] * 3 + [2] * 8 + [3, 4] + [5] * 6, dtype=np.int64)
    x = [0, 1, 2, 3, 4] + [2, 3, 4] + [0, 1, 2, 3, 4, 2, 3, 4] + [771.64, 378.49] + [0, -0.9871, -0.9871] * 2
    t = FieldType(DEC, abi.FLAG_NOT_NULL, 15, 4)
    scaled = np.array([round(v * 10 ** 4) for v in x], dtype=np.int64)
    chk = Chunk([Column(g), Column(A.cells_np(scaled, 15, 4, np.full(len(x), 11), np.zeros(len(x), dtype=np.int64), scaled < 0))])
    plan = AggPlan([INT_NN, t], [0], [AggFunc(P.AGG_FIRSTROW, 0), dsum(1, 4), davg(1, 8), dmax(1, 4), dmin(1, 4)])
    rows, _ = run_host(plan, [chk])
    got = {r[0]: tuple(D.to_string(c) for c in r[1:]) for r in rows}
    assert got[0] == ("10.0000", "2.00000000", "4.0000", "0.0000")
    assert got[1] == ("9.0000", "3.00000000", "4.0000", "2.0000")
    assert got[2] == ("19.0000", "2.37500000", "4.0000", "0.0000")
    assert got[3][2] == "771.6400" and got[4][2] == "378.4900"
    assert got[5][0] == "-3.9484"


AVG_CASES = [(1, 2), (-1, 2), (3, 2), (-3, 2), (1, 8), (-1, 8), (1, 32), (-1, 32), (5, 16), (-5, 16), (2, 3), (-2, 3), (-1, 3),
             (7, 7), (0, 5), (1, 64), (-1, 64), (99999, 100000), (-99999, 100000)]


@pytest.mark.parametrize("p,s", SCALES)
@pytest.mark.parametrize("local", ["0", "2"])
def test_avg_ties_and_signs(p, s, local, monkeypatch):
    # one group per (sum, count): a row with the sum and count - 1 zero rows.  1/32 = 0.03125 puts a tie on digit s + 5, the
    # first digit after f = s + 4; results that round or truncate to zero keep no sign; +-(10^p - 1) / 2 carries
    monkeypatch.setenv("TG_AGG_LOCAL", local)
    lim = 10 ** p - 1
    cases = AVG_CASES + [(lim, 2), (-lim, 2), (lim, 1), (-lim, 3)]
    g, x = [], []
    for j, (sm, n) in enumerate(cases):
        g += [j] * n
        x += [sm] + [0] * (n - 1)
    rng = np.random.default_rng(90 + s)
    perm = rng.permutation(len(g))
    x = np.array(x, dtype=np.int64)[perm]
    chk = Chunk([Column(np.array(g, dtype=np.int64)[perm]), Column(encode(rng, x, p, s))])
    t = FieldType(DEC, abi.FLAG_NOT_NULL, p, s)
    f1, f2, f3 = fracs(s)
    assert any((Fraction(abs(sm), n * 10 ** s) * 10 ** (f1 + 1)) % 10 == 5 for sm, n in cases)   # an exact tie at digit f1 + 1
    plan = AggPlan([INT_NN, t], [0], [AggFunc(P.AGG_FIRSTROW, 0), davg(1, f1), davg(1, f2), davg(1, f3)])
    rows, _ = run_host(plan, chk.split(1 << 15))
    vals = {0: (np.array(g, dtype=np.int64)[perm], np.zeros(len(g), dtype=bool)), 1: (x, np.zeros(len(g), dtype=bool))}
    assert check(plan, vals, rows) == len(cases)
    for r in rows:
        for cell in r[1:]:
            assert not (D.decode(cell).negative and D.value(cell) == 0), D.to_string(cell)


# ---- bad cells -----------------------------------------------------------------------------------------------------
def _bad_cells():
    """(description, cell) for DECIMAL(15, 2): each breaks the column's stored form"""
    good = A.cell(12345, 15, 2)
    wrong_frac = bytearray(good); wrong_frac[1] = 3                       # digitsFrac 3 != 2
    wrong_frac4 = bytearray(A.cell(12345, 15, 2)); wrong_frac4[1] = 0     # digitsFrac 0
    too_many = A.cell(10 ** 15, 16, 2, digits_int=14)                     # 16 significant digits
    past_scale = bytearray(A.cell(12345, 15, 2)); past_scale[12:16] = (450_000_001).to_bytes(4, "little")   # a digit after the scale
    big_word = bytearray(good); big_word[4:8] = (10 ** 9).to_bytes(4, "little")
    return [("digitsFrac != s", bytes(wrong_frac)), ("digitsFrac 0", bytes(wrong_frac4)), ("too many digits", too_many),
            ("digits past the scale", bytes(past_scale)), ("a word >= 10^9", bytes(big_word))]


@pytest.mark.parametrize("which", range(5))
def test_bad_cell_fails_the_push_and_leaves_the_table(which):
    import torch
    p, s = 15, 2
    name, bad = _bad_cells()[which]
    rng = np.random.default_rng(100 + which)
    good_chunk, good_vals = make_rows(rng, 20_000, 300, p, s)
    bad_chunk, _ = make_rows(rng, 20_000, 300, p, s)
    cells = bad_chunk.columns[1].data.copy()
    row = int(np.flatnonzero(~bad_chunk.columns[1].nulls())[7])
    cells[row] = np.frombuffer(bad, dtype=np.uint8)
    bad_chunk = Chunk([bad_chunk.columns[0], Column(cells, bad_chunk.columns[1].nulls())] + bad_chunk.columns[2:])
    plan = plans(p, s, local=False)[-1]
    lib = abi.load_lib()
    for route in ("device", "host"):
        e = HashAggExec(plan, MockDataSource(plan.col_types, []))
        e.open()
        h = e._h
        try:
            # the good rows go in first (a host push flushed by the device push, or a device push)
            if route == "device":
                chk, keep = dev_columns(good_chunk)
                abi.check(lib.tg_agg_push_dev(h, C.byref(chk)))
                chk, keep2 = dev_columns(bad_chunk)
                assert lib.tg_agg_push_dev(h, C.byref(chk)) == abi.TG_ERR_INVALID, name
            else:
                cs = good_chunk.to_struct()
                abi.check(lib.tg_agg_push(h, C.byref(cs)))
                cs2 = bad_chunk.to_struct()
                abi.check(lib.tg_agg_push(h, C.byref(cs2)))      # staged on the host: checked when the batch is flushed
                assert lib.tg_agg_finish(h) == abi.TG_ERR_INVALID, name
            assert b"column 1" in lib.tg_last_error(), lib.tg_last_error()
            before = e.stats()
            e._prepared = True
            abi.check(lib.tg_agg_finish(h))   # host route: the failed flush took the good rows with it, the table is still empty
            rows = []
            while True:
                c = e.next(1 << 20)
                if c.num_rows() == 0:
                    break
                rows.extend(rows_of(c))
            if route == "device":
                check(plan, good_vals, rows)
                assert before.input_rows == good_chunk.num_rows()
            else:
                assert rows == [] and before.input_rows == 0
        finally:
            assert lib.tg_agg_close(h) == abi.TG_OK
            e._h = C.c_void_p()
        torch.cuda.synchronize()


def test_host_push_then_bad_device_push_keeps_the_host_rows():
    p, s = 18, 0
    rng = np.random.default_rng(110)
    good_chunk, good_vals = make_rows(rng, 30_000, 200, p, s)
    bad_chunk, _ = make_rows(rng, 1000, 10, p, s)
    cells = bad_chunk.columns[2].data.copy()
    cells[5, 1] = 1                                        # digitsFrac 1 in a DECIMAL(18, 0) column
    bad_chunk = Chunk(bad_chunk.columns[:2] + [Column(cells)] + bad_chunk.columns[3:])
    plan = plans(p, s)[1]                                   # SUM / AVG of column 2
    lib = abi.load_lib()
    e = HashAggExec(plan, MockDataSource(plan.col_types, []))
    e.open()
    try:
        for c in good_chunk.split(4096):
            cs = c.to_struct()
            abi.check(lib.tg_agg_push(e._h, C.byref(cs)))
        chk, keep = dev_columns(bad_chunk)
        assert lib.tg_agg_push_dev(e._h, C.byref(chk)) == abi.TG_ERR_INVALID
        assert b"column 2" in lib.tg_last_error()
        abi.check(lib.tg_agg_finish(e._h))
        e._prepared = True
        rows = rows_of(e.next(1 << 20))
        check(plan, good_vals, rows)
    finally:
        e.close()


# ---- scale -----------------------------------------------------------------------------------------------------
def test_full_scale_100m_rows_1m_groups():
    # SUM(DECIMAL(15,2)) + COUNT over 100 M device-resident rows in 1 M groups; the cells are built on the device in FromBin's
    # form (digitsInt 13: two integer words, one fraction word); the sums stay below 2^63, so an int64 index_add is exact
    import torch
    from tidb_b200.device import DeviceAgg
    n, G = 100_000_000, 1_000_000
    gen = torch.Generator(device="cuda").manual_seed(21)
    keys = torch.randint(0, G, (n,), device="cuda", dtype=torch.int64, generator=gen)
    vals = torch.randint(-(10 ** 15 - 1), 10 ** 15, (n,), device="cuda", dtype=torch.int64, generator=gen)
    m = vals.abs()
    ip = m // 100
    w = torch.zeros((n, 10), dtype=torch.int32, device="cuda")
    w[:, 0] = (13 | (2 << 8) | ((vals < 0).to(torch.int32) << 24)).to(torch.int32)
    w[:, 1] = (ip // 10 ** 9).to(torch.int32)
    w[:, 2] = (ip % 10 ** 9).to(torch.int32)
    w[:, 3] = ((m % 100) * 10 ** 7).to(torch.int32)
    del m, ip
    cells = w.view(torch.uint8).view(n, 40)
    torch.cuda.synchronize()   # the aggregation reads its input on a stream of its own: it must be written first
    plan = AggPlan([INT_NN, FieldType(DEC, abi.FLAG_NOT_NULL, 15, 2)], [0], [AggFunc(P.AGG_FIRSTROW, 0), dsum(1, 2), AggFunc(P.AGG_COUNT, -1)],
                   expected_groups=G)
    agg = DeviceAgg(plan)
    try:
        agg.push([keys, cells])
        rows, cols, _ = agg.finish()
        assert rows == G
        k = np.zeros(rows, dtype=np.int64)
        out = np.zeros((rows, 40), dtype=np.uint8)
        cnt = np.zeros(rows, dtype=np.int64)
        lib = abi.load_lib()
        for dst, src in ((k, cols[0]), (out, cols[1]), (cnt, cols[2])):
            abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(dst.ctypes.data), C.c_void_p(src), C.c_size_t(dst.nbytes)))
    finally:
        agg.close()
    del cells, w
    want = torch.zeros(G, dtype=torch.int64, device="cuda").index_add_(0, keys, vals).cpu().numpy()[k]
    assert np.array_equal(cnt, torch.bincount(keys, minlength=G).cpu().numpy()[k])
    c = out.view(np.int32).astype(np.int64)
    hdr = c[:, 0]
    ni = (hdr & 0xFF) // 9                                   # integer words: |sum| < 10^17, its integer part < 10^15
    assert np.isin(ni, (1, 2)).all() and (((hdr >> 8) & 0xFFFF) == (2 | (2 << 8))).all()   # digitsFrac = resultFrac = 2
    ipart = np.where(ni == 2, c[:, 1] * 10 ** 9 + c[:, 2], c[:, 1])
    fw = np.where(ni == 2, c[:, 3], c[:, 2])
    mag = ipart * 100 + fw // 10 ** 7
    assert (fw % 10 ** 7 == 0).all()
    neg = ((hdr >> 24) & 0xFF) == 1
    assert np.array_equal(np.where(neg, -mag, mag), want) and np.array_equal(neg, want < 0)
    for r in np.random.default_rng(0).integers(0, G, 200):   # spot checks through the codec
        assert bytes(out[r]) == A.sum_result(int(want[r]), 2)
