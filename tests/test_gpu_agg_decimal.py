"""DECIMAL SUM / AVG of integer columns on every update path of the CUDA hash aggregation, compared exactly.

Each case forces one path through the TG_AGG_* switches, proves from tg_agg_stats.paths / local_rows that it ran, and
compares every group's 40-byte MyDecimal cell byte for byte with the canonical cell of the exact answer
(tests/mydecimal.py: SUM is the Python-int sum, AVG the truncate-or-round rule at the requested scale).  The data holds
full-range signed values with groups made only of INT64_MIN, unsigned groups of UINT64_MAX whose sums pass 2^64 and 2^65,
x / -x pairs whose sums cross zero and groups that cancel to exactly 0, all-NULL groups (NULL results), NOT NULL and
nullable arguments.  DOUBLE SUM / AVG, COUNT, MIN and MAX in the same plans are checked with tests/agg_reference.py."""
import ctypes as C

import numpy as np
import pytest

import agg_reference as R
import mydecimal as D
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.executor import HashAggExec, MockDataSource
from tidb_b200.plan import AggFunc, AggPlan, FieldType

pytestmark = pytest.mark.gpu

P = abi
DEC = abi.TYPE_NEWDECIMAL
I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1
INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
UINT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
SWITCHES = ("TG_AGG_LOCAL", "TG_AGG_LOCAL_SLOTS", "TG_AGG_V1")
K_ALLNULL, K_IMIN, K_UMAX, K_CANCEL, K_IMAX = (7_000_000_000_000 + j for j in range(5))
SPECIAL = (K_ALLNULL, K_IMIN, K_UMAX, K_CANCEL, K_IMAX)


@pytest.fixture(autouse=True)
def _default_switches(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)


# ---- data --------------------------------------------------------------------------------------------------------
# columns: 0 g key (nullable) | 1 i BIGINT (nullable, full range) | 2 u BIGINT UNSIGNED (nullable, full range)
#          3 inn BIGINT NOT NULL (full range) | 4 c BIGINT (nullable, x / -x pairs in one group) | 5 d DOUBLE (nullable)
TYPES = [INT, INT, UINT, INT_NN, INT, DBL]


def make_rows(rng, n, ngroups):
    half = n // 2
    gp = (rng.integers(0, ngroups, half) * 2654435761 % (1 << 40) - (1 << 39)).astype(np.int64)
    sp = rng.random(half) < 0.02
    gp[sp] = rng.choice(np.array(SPECIAL, dtype=np.int64), int(sp.sum()))
    gp[rng.random(half) < 0.002] = I64_MIN                   # the key equal to the table's empty sentinel
    gnp = rng.random(half) < 0.01                            # the NULL group
    g = np.repeat(gp, 2); gn = np.repeat(gnp, 2)
    v = rng.integers(I64_MIN + 1, I64_MAX, half, endpoint=True, dtype=np.int64)
    c = np.stack([v, -v], axis=1).ravel()                    # pairs: every group's sum crosses zero on the way
    rem = rng.random(n) < 0.3
    c[rem] = rng.integers(-1000, 1000, int(rem.sum()))       # ... and ends near it
    cn = np.repeat(rng.random(half) < 0.05, 2)
    i = rng.integers(I64_MIN, I64_MAX, n, endpoint=True, dtype=np.int64)
    u = rng.integers(0, 1 << 64, n, dtype=np.uint64).view(np.int64)
    inn = rng.integers(I64_MIN, I64_MAX, n, endpoint=True, dtype=np.int64)
    d = rng.standard_normal(n) * 1e3
    iN, uN, dN = rng.random(n) < 0.05, rng.random(n) < 0.05, rng.random(n) < 0.05
    key = np.where(gn, 0, g)
    for k, col, val in ((K_IMIN, i, I64_MIN), (K_IMIN, inn, I64_MIN), (K_UMAX, u, -1), (K_IMAX, i, I64_MAX), (K_IMAX, inn, I64_MAX)):
        col[key == k] = val
    m = key == K_CANCEL
    c[m] = np.stack([v, -v], axis=1).ravel()[m]             # pairs only: the sum is exactly 0
    m = key == K_ALLNULL
    iN = iN | m; uN = uN | m; cn = cn | m; dN = dN | m
    perm = rng.permutation(n)
    cols = [Column(g, gn), Column(i, iN), Column(u, uN), Column(inn), Column(c, cn), Column(d, dN)]
    return Chunk([Column(col.data[perm], col.nulls()[perm]) for col in cols])


def sum_(c):
    return AggFunc(P.AGG_SUM, c, P.TYPE_LONGLONG, ret_type=DEC)


def avg_(c, f):
    return AggFunc(P.AGG_AVG, c, P.TYPE_LONGLONG, ret_type=DEC, ret_frac=f)


def plans(group_by=(0,), expected_groups=0, types=TYPES, a=1):
    """DECIMAL SUM / AVG (at scales 0, 4, 9, 30) over every argument kind, at most 4 device states per plan so that the
    CTA-local level accepts them, plus one plan mixing them with DOUBLE SUM / AVG, COUNT, MIN and MAX"""
    fr = [AggFunc(P.AGG_FIRSTROW, g) for g in group_by]
    i, u, inn, c, d = a, a + 1, a + 2, a + 3, a + 4
    lists = [[sum_(i)], [sum_(u)], [sum_(inn), avg_(inn, 4)], [sum_(c)], [avg_(i, 0)], [avg_(u, 9)], [avg_(c, 30)],
             [avg_(i, 4), AggFunc(P.AGG_COUNT, -1)],
             [sum_(inn), AggFunc(P.AGG_COUNT, c), AggFunc(P.AGG_MIN, i), AggFunc(P.AGG_MAX, u), AggFunc(P.AGG_SUM, d, P.TYPE_DOUBLE),
              avg_(u, 4), AggFunc(P.AGG_AVG, d, P.TYPE_DOUBLE), avg_(inn, 30)]]
    return [AggPlan(types, list(group_by), fr + fs, expected_groups=expected_groups) for fs in lists]


# ---- exact reference ---------------------------------------------------------------------------------------------
def _logical(chunks, c):
    data = np.concatenate([ch.columns[c].data if ch.sel is None else ch.columns[c].data[ch.sel] for ch in chunks])
    nl = np.concatenate([ch.columns[c].nulls() if ch.sel is None else ch.columns[c].nulls()[ch.sel] for ch in chunks])
    return data, nl


def dec_expected(plan, chunks):
    """group key tuple -> {function index: expected cell bytes or None} for the DECIMAL functions of the plan.  Sums are
    exact: the 32-bit halves of the arguments are summed per group as float64, exact while a group has < 2^21 rows"""
    keys = [_logical(chunks, g) for g in plan.group_by]
    n = len(_logical(chunks, 0)[0])
    if keys:
        kmat = np.stack([a for v, nl in keys for a in (nl.astype(np.int64), np.where(nl, 0, v))], axis=1)
        uk, inv = np.unique(kmat, axis=0, return_inverse=True)
        inv = inv.ravel()
        tuples = [tuple(None if r[2 * j] else int(r[2 * j + 1]) for j in range(len(keys))) for r in uk]
    else:
        if n == 0:
            return {(): {k: None for k, f in enumerate(plan.funcs) if f.ret_type == DEC}}
        inv, tuples = np.zeros(n, dtype=np.int64), [()]
    assert n < (1 << 21)
    ng = len(tuples)
    out = {t: {} for t in tuples}
    for k, f in enumerate(plan.funcs):
        if f.ret_type != DEC:
            continue
        v, nl = _logical(chunks, f.arg_col)
        keep = ~nl
        if plan.col_types[f.arg_col].unsigned:
            uv = v.view(np.uint64)
            lo, hi = (uv & np.uint64(0xFFFFFFFF)).astype(np.float64), (uv >> np.uint64(32)).astype(np.float64)
        else:
            lo, hi = (v & 0xFFFFFFFF).astype(np.float64), (v >> 32).astype(np.float64)
        slo = np.bincount(inv[keep], weights=lo[keep], minlength=ng)
        shi = np.bincount(inv[keep], weights=hi[keep], minlength=ng)
        cnt = np.bincount(inv[keep], minlength=ng)
        for gi, t in enumerate(tuples):
            if cnt[gi] == 0:
                out[t][k] = None
                continue
            s = (int(shi[gi]) << 32) + int(slo[gi])
            out[t][k] = D.sum_result(s) if f.name == P.AGG_SUM else D.avg_result(s, int(cnt[gi]), f.ret_frac)
    return out


def rows_of(chunk):
    cols = []
    for col in chunk.columns:
        nl = col.nulls()
        if col.data.ndim == 2:
            cols.append([None if nl[r] else bytes(col.data[r]) for r in range(col.length)])
        else:
            cols.append([None if n else v for v, n in zip(col.data.tolist(), nl.tolist())])
    return list(zip(*cols))


def check(plan, chunks, got_rows):
    """every group's DECIMAL cells equal the canonical cell of the exact answer; the other functions through the DOUBLE /
    integer reference"""
    exp = dec_expected(plan, chunks)
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
            assert D.well_formed(g), (key, k, D.decode(g))
            assert g == cell, f"group {key!r} aggregate {k}: got {D.to_string(g)} {D.decode(g)}, want {D.to_string(cell)} {D.decode(cell)}"
    others = [k for k, f in enumerate(plan.funcs) if f.ret_type != DEC]
    if any(plan.funcs[k].name != P.AGG_FIRSTROW for k in others):
        sub = AggPlan(plan.col_types, plan.group_by, [plan.funcs[k] for k in others])
        R.check(sub, chunks, [tuple(r[k] for k in others) for r in got_rows])
    return len(exp)


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


def run_dev(plan, batches):
    import torch
    e = HashAggExec(plan, MockDataSource(plan.col_types, []))
    e.open()
    try:
        lib = abi.load_lib()
        for b in batches:
            keep = []
            cs = (abi.TgColumn * len(b.columns))()
            for c, col in enumerate(b.columns):
                t = torch.from_numpy(np.ascontiguousarray(col.data).view(np.int64)).cuda(); keep.append(t)
                cs[c].length, cs[c].data, cs[c].elem_len = col.length, t.data_ptr(), 8
                if col.null_bitmap is not None:
                    nb = torch.from_numpy(np.ascontiguousarray(col.null_bitmap)).cuda(); keep.append(nb)
                    cs[c].null_bitmap = nb.data_ptr()
            chk = abi.TgChunk(); chk.ncols = len(b.columns); chk.cols = C.cast(cs, C.POINTER(abi.TgColumn))
            torch.cuda.synchronize()
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


def check_all(plan_list, chunks, want, dont=0, local=None, runner=None):
    st = None
    for plan in plan_list:
        rows, st = (runner or run_host)(plan, chunks)
        check(plan, chunks, rows)
        assert st.paths & want == want, (hex(st.paths), hex(want))
        assert st.paths & dont == 0, (hex(st.paths), hex(dont))
        if local is not None:
            assert (st.local_rows > 0) == local, st.local_rows
    return st


# ---- paths -----------------------------------------------------------------------------------------------------
def test_no_group_by():
    rng = np.random.default_rng(11)
    check_all(plans(group_by=()), make_rows(rng, 300_000, 50).split(1 << 15), want=P.AGG_PATH_NOGROUP, dont=~P.AGG_PATH_NOGROUP)
    # one group of only INT64_MIN / UINT64_MAX: the sums pass -2^63 * n and 2^64 * n
    n = 70_000
    one = Chunk([Column(np.zeros(n, dtype=np.int64)), Column(np.full(n, I64_MIN)), Column(np.full(n, -1, dtype=np.int64)),
                 Column(np.full(n, I64_MIN)), Column(np.full(n, I64_MAX)), Column(np.zeros(n))])
    check_all(plans(group_by=()), one.split(1 << 14), want=P.AGG_PATH_NOGROUP)
    # no input at all: SUM and AVG are NULL
    rows, _ = run_host(plans(group_by=())[2], [])
    assert rows == [(None, None)]


@pytest.mark.parametrize("ngroups", [40, 60_000])
def test_v2_global_only(ngroups, monkeypatch):
    monkeypatch.setenv("TG_AGG_LOCAL", "0")
    rng = np.random.default_rng(12 + ngroups)
    check_all(plans(), make_rows(rng, 200_000, ngroups).split(1 << 15), want=P.AGG_PATH_V2_GLOBAL,
              dont=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE, local=False)


def test_v2_two_level_low_cardinality():
    rng = np.random.default_rng(13)
    check_all(plans()[:-1], make_rows(rng, 400_000, 60).split(1 << 15), want=P.AGG_PATH_V2_LOCAL, local=True)


def test_v2_local_forced_high_cardinality_spills_and_merges(monkeypatch):
    monkeypatch.setenv("TG_AGG_LOCAL", "2")
    rng = np.random.default_rng(14)
    st = check_all(plans(expected_groups=64)[:-1], make_rows(rng, 300_000, 100_000).split(1 << 16),
                   want=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE, local=True)
    assert st.table_slots > 1024


@pytest.mark.parametrize("ngroups,hint,want", [(60, 0, P.AGG_PATH_V1_LOCAL | P.AGG_PATH_MERGE),
                                               (60_000, 0, P.AGG_PATH_V1_LOCAL | P.AGG_PATH_MERGE | P.AGG_PATH_V1_GLOBAL),
                                               (60_000, 60_000, P.AGG_PATH_V1_GLOBAL)])
def test_v1_paths(ngroups, hint, want, monkeypatch):
    monkeypatch.setenv("TG_AGG_V1", "1")
    monkeypatch.setenv("TG_AGG_LOCAL_SLOTS", "512")
    rng = np.random.default_rng(15 + ngroups + hint)
    v2 = P.AGG_PATH_V2_LOCAL | P.AGG_PATH_V2_GLOBAL
    check_all(plans(expected_groups=hint)[:-1], make_rows(rng, 300_000, ngroups).split(1 << 15), want=want, dont=v2, local=False)


@pytest.mark.parametrize("ncols", [2, 3, 4])
def test_multi_key(ncols):
    rng = np.random.default_rng(16 + ncols)
    base = make_rows(rng, 200_000, 50)
    n = base.num_rows()
    keys, types = [base.columns[0]], [INT]
    for _ in range(ncols - 1):
        keys.append(Column(rng.integers(-3, 4, n).astype(np.int64))); types.append(INT_NN)
    chk = Chunk(keys + base.columns[1:])
    check_all(plans(group_by=tuple(range(ncols)), expected_groups=16, types=types + TYPES[1:], a=ncols),
              chk.split(1 << 15), want=P.AGG_PATH_MULTI_KEY, dont=~P.AGG_PATH_MULTI_KEY)


def test_several_device_pushes_with_growth():
    rng = np.random.default_rng(17)
    batches = [make_rows(rng, n, g) for n, g in ((50_000, 30), (100_000, 3000), (100_000, 30_000), (50_000, 40_000))]
    for plan in plans(expected_groups=16):
        rows, st = run_dev(plan, batches)
        check(plan, batches, rows)
        assert st.table_slots > 1024 and st.paths & (P.AGG_PATH_V2_LOCAL | P.AGG_PATH_V2_GLOBAL)
    rows, st = run_dev(plans(group_by=())[0], batches)
    check(plans(group_by=())[0], batches, rows)


def test_sel_vectors(monkeypatch):
    rng = np.random.default_rng(18)
    chunks = []
    for c in make_rows(rng, 300_000, 500).split(1 << 14):
        sel = np.sort(rng.choice(c.num_rows(), c.num_rows() // 3, replace=False))
        chunks.append(Chunk(c.columns, sel))
    check_all(plans()[:-1], chunks, want=P.AGG_PATH_V2_LOCAL)
    check_all(plans()[-1:], chunks, want=P.AGG_PATH_V2_GLOBAL)
    monkeypatch.setenv("TG_AGG_V1", "1")
    check_all(plans()[:3], chunks, want=P.AGG_PATH_V1_LOCAL)


# ---- AVG rounding on the device ----------------------------------------------------------------------------------
AVG_CASES = [(1, 2), (-1, 2), (3, 2), (-3, 2), (1, 8), (-1, 8), (1, 32), (-1, 32), (2, 3), (-2, 3), (-1, 20000), (-1, 30000),
             (99999, 100000), (-99999, 100000), (-1, 3), (7, 7), (0, 5), (5, 10), (-5, 10), (1, 2 * 10 ** 5)]


@pytest.mark.parametrize("local", ["0", "2"])
def test_avg_ties_and_signs(local, monkeypatch):
    # one group per (sum, count): a row holding the sum and count - 1 zero rows; ties of both signs, results that round
    # or truncate to zero (no negative zero), carries into the integer part
    monkeypatch.setenv("TG_AGG_LOCAL", local)
    g, x = [], []
    for j, (s, n) in enumerate(AVG_CASES):
        g += [j] * n
        x += [s] + [0] * (n - 1)
    rng = np.random.default_rng(19)
    perm = rng.permutation(len(g))
    chk = Chunk([Column(np.array(g, dtype=np.int64)[perm]), Column(np.array(x, dtype=np.int64)[perm])])
    fs = [AggFunc(P.AGG_FIRSTROW, 0)] + [avg_(1, f) for f in (0, 4, 9, 30)]
    for plan in (AggPlan([INT_NN, INT_NN], [0], fs[:3]), AggPlan([INT_NN, INT_NN], [0], fs[:1] + fs[3:])):
        rows, st = run_host(plan, chk.split(1 << 15))
        assert check(plan, chk.split(1 << 15), rows) == len(AVG_CASES)
        for r in rows:
            for cell in r[1:]:
                c = D.decode(cell)
                assert not (c.negative and D.value(cell) == 0), D.to_string(cell)


# ---- the C ABI around DECIMAL results ----------------------------------------------------------------------------
def test_next_paging_result_dev_and_elem_len():
    rng = np.random.default_rng(20)
    chunks = make_rows(rng, 100_000, 3000).split(1 << 15)
    plan = AggPlan(TYPES, [0], [AggFunc(P.AGG_FIRSTROW, 0), sum_(1), AggFunc(P.AGG_COUNT, -1), avg_(2, 4)], expected_groups=3000)
    rows, _ = run_host(plan, chunks, page=37)          # 37-row pages: cells and bitmaps start inside a byte
    assert check(plan, chunks, rows) > 3000
    lib = abi.load_lib()
    e = HashAggExec(plan, MockDataSource(plan.col_types, chunks))
    e.open()
    try:
        e.next(8)
        # a DECIMAL column needs 40-byte cells: an 8-byte output column is refused before anything is copied
        from tidb_b200.chunk import MutChunk
        bad = MutChunk([8, 8, 8, 40], 16, [np.int64, np.int64, np.int64, np.dtype((np.uint8, 40))])
        n = C.c_int64(0)
        assert lib.tg_agg_next(e._h, C.byref(bad.struct), C.c_int64(16), C.byref(n)) == abi.TG_ERR_INVALID
        assert b"elem_len 40" in lib.tg_last_error()
        bad = MutChunk([8, 40, 8, 8], 16, [np.int64, np.dtype((np.uint8, 40)), np.int64, np.int64])
        assert lib.tg_agg_next(e._h, C.byref(bad.struct), C.c_int64(16), C.byref(n)) == abi.TG_ERR_INVALID
        # tg_agg_result_dev: the device column holds 40-byte cells
        nrows = C.c_int64(0)
        cols = (C.c_void_p * 4)(); nulls = (C.c_void_p * 4)()
        abi.check(lib.tg_agg_result_dev(e._h, C.byref(nrows), cols, nulls))
        m = nrows.value
        host = np.zeros((m, 40), dtype=np.uint8)
        keys = np.zeros(m, dtype=np.int64)
        abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(host.ctypes.data), C.c_void_p(cols[1]), C.c_size_t(m * 40)))
        abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(keys.ctypes.data), C.c_void_p(cols[0]), C.c_size_t(m * 8)))
        knb = np.zeros((m + 7) // 8, dtype=np.uint8); snb = np.zeros((m + 7) // 8, dtype=np.uint8)
        abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(knb.ctypes.data), C.c_void_p(nulls[0]), C.c_size_t(len(knb))))
        abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(snb.ctypes.data), C.c_void_p(nulls[1]), C.c_size_t(len(snb))))
        from tidb_b200.chunk import unpack_nulls
        kn, sn = unpack_nulls(knb, m), unpack_nulls(snb, m)
        exp = dec_expected(plan, chunks)
        for r in range(m):
            key = (None if kn[r] else int(keys[r]),)
            want = exp[key][1]
            assert (None if sn[r] else bytes(host[r])) == want, key
    finally:
        e.close()


def test_uint64_max_groups_pass_2_64_and_2_65():
    # groups of 1, 2, 3, 4 and 5 UINT64_MAX rows: sums just below 2^64, then past 2^64, 2^65 and 2^66
    g = np.repeat(np.arange(5, dtype=np.int64), np.arange(1, 6))
    u = np.full(len(g), -1, dtype=np.int64)
    chk = Chunk([Column(g), Column(u)])
    plan = AggPlan([INT_NN, FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED | abi.FLAG_NOT_NULL)], [0],
                   [AggFunc(P.AGG_FIRSTROW, 0), sum_(1), avg_(1, 4)])
    rows, _ = run_host(plan, [chk])
    got = {r[0]: D.to_string(r[1]) for r in rows}
    assert got == {j: str(U64_MAX * (j + 1)) for j in range(5)}
    assert all(D.to_string(r[2]) == "18446744073709551615.0000" for r in rows)


def test_full_scale_100m_rows_1m_groups():
    # SUM(bigint) + COUNT over 100 M device-resident rows in 1 M groups, values below 2^31: an int64 bincount is exact
    import torch
    from tidb_b200.device import DeviceAgg
    n, G = 100_000_000, 1_000_000
    gen = torch.Generator(device="cuda").manual_seed(21)
    keys = torch.randint(0, G, (n,), device="cuda", dtype=torch.int64, generator=gen)
    vals = torch.randint(-(1 << 31), 1 << 31, (n,), device="cuda", dtype=torch.int64, generator=gen)
    torch.cuda.synchronize()   # the aggregation reads its input on a stream of its own: it must be written first
    plan = AggPlan([INT_NN, INT_NN], [0], [AggFunc(P.AGG_FIRSTROW, 0), sum_(1), AggFunc(P.AGG_COUNT, -1)], expected_groups=G)
    agg = DeviceAgg(plan)
    try:
        agg.push([keys, vals])
        rows, cols, _ = agg.finish()
        assert rows == G
        k = np.zeros(rows, dtype=np.int64)
        cells = np.zeros((rows, 40), dtype=np.uint8)
        cnt = np.zeros(rows, dtype=np.int64)
        lib = abi.load_lib()
        for dst, src in ((k, cols[0]), (cells, cols[1]), (cnt, cols[2])):
            abi.check(lib.tg_memcpy_d2h(0, C.c_void_p(dst.ctypes.data), C.c_void_p(src), C.c_size_t(dst.nbytes)))
    finally:
        agg.close()
    want = torch.zeros(G, dtype=torch.int64, device="cuda").index_add_(0, keys, vals).cpu().numpy()
    want_cnt = torch.bincount(keys, minlength=G).cpu().numpy()
    assert np.array_equal(cnt, want_cnt[k])
    # the cells: header, then base-10^9 words of |sum| < 2^31 * 10^4 < 10^18 (at most two words)
    c = cells.view(np.int32).astype(np.int64)
    w = want[k]
    hdr = c[:, 0]
    neg = (hdr >> 24) & 0xFF
    words = np.where((hdr & 0xFF) == 18, c[:, 1] * 10 ** 9 + c[:, 2], c[:, 1])
    assert np.array_equal(np.where(neg == 1, -words, words), w)
    assert np.array_equal(neg == 1, w < 0)
    big = np.abs(w) >= 10 ** 9
    assert np.array_equal(hdr & 0xFF, np.where(big, 18, 9)) and np.array_equal((hdr >> 8) & 0xFFFF, np.zeros_like(hdr))
    assert not c[:, 3:].any() and not c[~big, 2].any()
    for r in np.random.default_rng(0).integers(0, G, 200):   # spot checks through the codec
        assert bytes(cells[r]) == D.sum_result(int(w[r]))
