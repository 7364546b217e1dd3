"""COUNT / SUM / AVG with DISTINCT on every update path of the CUDA hash aggregation, against the plain-Python reference
of tests/agg_distinct_reference.py.

Each path is forced through the TG_AGG_* switches and proven from tg_agg_stats.paths.  COUNT and DECIMAL cells are
compared exactly (cells byte for byte); DOUBLE SUM / AVG within the order-free bound of tests/agg_reference.py.  The data
repeats its values within and across groups and pushes: signed and unsigned BIGINT (values above 2^63), DOUBLE with -0.0,
+0.0 and NaN, DECIMAL(18,2) / (15,2) / (18,18), NULL group keys, a DOUBLE group key with both zeros, and a NOT NULL
argument."""
import ctypes as C

import numpy as np
import pytest

import agg_distinct_reference as DR
import mydecimal as D
import mydecimal_args as A
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.executor import HashAggExec, MockDataSource
from tidb_b200.plan import AggFunc, AggPlan, FieldType

pytestmark = pytest.mark.gpu

P = abi
DEC = abi.TYPE_NEWDECIMAL
INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
UINT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
SWITCHES = ("TG_AGG_LOCAL", "TG_AGG_LOCAL_SLOTS", "TG_AGG_V1")
SCALES = [(18, 2), (15, 2), (18, 18)]
# columns: 0 g BIGINT | 1 k2 BIGINT NOT NULL | 2 k3 BIGINT | 3 k4 DOUBLE (keys)
#          4 x BIGINT | 5 u BIGINT UNSIGNED | 6 d DOUBLE | 7 a DECIMAL(p, s) | 8 xn BIGINT NOT NULL (arguments)
G, K2, K3, K4, X, U, DD, DA, XN = range(9)


@pytest.fixture(autouse=True)
def _default_switches(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)


def types_of(p, s):
    return [INT, INT_NN, INT, DBL, INT, UINT, DBL, FieldType(DEC, 0, p, s), INT_NN]


# ---- data --------------------------------------------------------------------------------------------------------
def dec_cells(v, p, s):
    n = len(v)
    return A.cells_np(v, p, s, np.full(n, p - s), np.zeros(n, dtype=np.int64), v < 0)


def make_vals(rng, n, ngroups, p, s, pool=40):
    """{column: (values, nulls)}: every argument drawn from a small pool, so values repeat within groups and pushes"""
    lim = 10 ** p - 1
    g = (rng.integers(0, ngroups, n) * 2654435761 % (1 << 40) - (1 << 39)).astype(np.int64)
    xpool = np.concatenate([np.array([-(1 << 63), (1 << 63) - 1, 0, -1, 1], dtype=np.int64), rng.integers(-(1 << 62), 1 << 62, pool)])
    upool = np.concatenate([np.array([(1 << 64) - 1, 1 << 63, 0], dtype=np.uint64), rng.integers(0, 1 << 64, pool, dtype=np.uint64)]).view(np.int64)
    dpool = np.concatenate([np.array([0.0, -0.0, np.nan, 1.5, -2.25, 1e300]), rng.standard_normal(pool) * 1e3])
    apool = np.concatenate([np.array([lim, -lim, 0, 150, 15], dtype=np.int64), rng.integers(-lim, lim, pool, endpoint=True)])
    nl = lambda q: rng.random(n) < q
    return {G: (g, nl(0.01)), K2: (rng.integers(-2, 3, n).astype(np.int64), np.zeros(n, dtype=bool)),
            K3: (rng.integers(0, 3, n).astype(np.int64), nl(0.05)),
            K4: (rng.choice(np.array([0.0, -0.0, 1.5]), n), nl(0.05)),
            X: (rng.choice(xpool, n), nl(0.05)), U: (rng.choice(upool, n), nl(0.05)),
            DD: (rng.choice(dpool, n), nl(0.05)), DA: (rng.choice(apool, n), nl(0.05)),
            XN: (rng.integers(0, 7, n).astype(np.int64), np.zeros(n, dtype=bool))}


def to_chunk(vals, p, s, lo=0, hi=None):
    cols = []
    for c in range(9):
        v, nl = vals[c][0][lo:hi], vals[c][1][lo:hi]
        cols.append(Column(dec_cells(v, p, s) if c == DA else v, nl if nl.any() else None))
    return Chunk(cols)


def concat(*parts):
    return {c: (np.concatenate([q[c][0] for q in parts]), np.concatenate([q[c][1] for q in parts])) for c in parts[0]}


def cnt(c):
    return AggFunc(P.AGG_COUNT, c, distinct=True)


def dsum(c):
    return AggFunc(P.AGG_SUM, c, P.TYPE_LONGLONG, ret_type=DEC, distinct=True)


def davg(c, frac, t=P.TYPE_LONGLONG):
    return AggFunc(P.AGG_AVG, c, t, ret_type=DEC, ret_frac=frac, distinct=True)


def plans(p, s, group_by=(G,), expected_groups=0, small=False):
    """function lists; small=True keeps each list at <= 4 state words (the CTA-local levels take no more)"""
    fr = [AggFunc(P.AGG_FIRSTROW, g) for g in group_by]
    dd = lambda name: AggFunc(name, DD, P.TYPE_DOUBLE, distinct=True)
    if small:
        lists = [[cnt(X), AggFunc(P.AGG_COUNT, X)], [davg(XN, 4)], [dd(P.AGG_SUM)], [cnt(DA), cnt(U), cnt(DD)],
                 [AggFunc(P.AGG_SUM, DA, DEC, ret_type=DEC, ret_frac=s, distinct=True)]]
    else:
        lists = [[cnt(X), AggFunc(P.AGG_COUNT, X), dsum(X), davg(X, 4)],
                 [cnt(U), dsum(U), cnt(DD), dd(P.AGG_SUM), dd(P.AGG_AVG), AggFunc(P.AGG_SUM, DD, P.TYPE_DOUBLE)],
                 [cnt(DA), AggFunc(P.AGG_SUM, DA, DEC, ret_type=DEC, ret_frac=s, distinct=True), davg(DA, min(s + 4, 30), DEC),
                  AggFunc(P.AGG_MAX, DA, DEC, ret_type=DEC, ret_frac=s, distinct=True), AggFunc(P.AGG_COUNT, DA)],
                 [davg(XN, 4), cnt(XN), AggFunc(P.AGG_AVG, XN, ret_type=DEC, ret_frac=4), AggFunc(P.AGG_COUNT, -1), cnt(X)]]
    return [AggPlan(types_of(p, s), list(group_by), fr + fs, expected_groups=expected_groups) for fs in lists]


# ---- running -----------------------------------------------------------------------------------------------------
def rows_of(chunk):
    cols = []
    for col in chunk.columns:
        nl = col.nulls()
        if col.data.ndim == 2:
            cols.append([None if nl[r] else bytes(col.data[r]) for r in range(col.length)])
        else:
            cols.append([None if x else v for v, x in zip(col.data.tolist(), nl.tolist())])
    return list(zip(*cols))


def drain(e):
    rows = []
    while True:
        c = e.next(1 << 20)
        if c.num_rows() == 0:
            return rows
        rows.extend(rows_of(c))


def run_host(plan, chunks):
    e = HashAggExec(plan, MockDataSource(plan.col_types, chunks))
    e.open()
    try:
        return drain(e), e.stats(), e.distinct_stats()
    finally:
        e.close()


def dev_columns(chunk, misalign=False):
    """device copies of the chunk's columns; misalign=True puts DECIMAL columns 8 bytes past a 16-byte boundary"""
    import torch
    keep, cs = [], (abi.TgColumn * len(chunk.columns))()
    for c, col in enumerate(chunk.columns):
        raw = np.ascontiguousarray(col.data).view(np.uint8).ravel()
        if col.data.ndim == 2 and misalign:
            buf = torch.zeros(raw.size + 8, dtype=torch.uint8, device="cuda")
            buf[8:] = torch.from_numpy(raw).cuda()
            ptr = buf.data_ptr() + 8
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


def push_dev(e, chunk, misalign=False):
    chk, keep = dev_columns(chunk, misalign)
    abi.check(abi.load_lib().tg_agg_push_dev(e._h, C.byref(chk)))


def check_paths(plan_list, chunks, vals, want, dont=0, local=None):
    for plan in plan_list:
        rows, st, ds = run_host(plan, chunks)
        DR.check(plan, vals, rows)
        assert st.paths & want == want, (hex(st.paths), hex(want))
        assert st.paths & dont == 0, (hex(st.paths), hex(dont))
        if local is not None:
            assert (st.local_rows > 0) == local, st.local_rows
        assert ds.launches >= 1 and ds.mark_ms > 0


# ---- paths -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p,s", SCALES)
def test_no_group_by(p, s):
    vals = make_vals(np.random.default_rng(1 + s), 120_000, 1, p, s)
    ch = to_chunk(vals, p, s).split(1 << 15)
    check_paths(plans(p, s, group_by=()) + plans(p, s, group_by=(), small=True), ch, vals,
                want=P.AGG_PATH_NOGROUP, dont=~P.AGG_PATH_NOGROUP)


@pytest.mark.parametrize("p,s", SCALES)
def test_v2_global(p, s, monkeypatch):
    monkeypatch.setenv("TG_AGG_LOCAL", "0")
    vals = make_vals(np.random.default_rng(10 + s), 120_000, 5000, p, s)
    check_paths(plans(p, s) + plans(p, s, small=True), to_chunk(vals, p, s).split(1 << 15), vals,
                want=P.AGG_PATH_V2_GLOBAL, dont=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE, local=False)


@pytest.mark.parametrize("p,s", SCALES)
def test_v2_cta_local(p, s):
    vals = make_vals(np.random.default_rng(20 + s), 150_000, 60, p, s)
    check_paths(plans(p, s, small=True), to_chunk(vals, p, s).split(1 << 15), vals, want=P.AGG_PATH_V2_LOCAL, local=True)


def test_v2_local_spills_and_merges(monkeypatch):
    monkeypatch.setenv("TG_AGG_LOCAL", "2")
    p, s = 18, 2
    vals = make_vals(np.random.default_rng(30), 120_000, 5000, p, s)
    check_paths(plans(p, s, expected_groups=64, small=True), to_chunk(vals, p, s).split(1 << 16), vals,
                want=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE, local=True)


@pytest.mark.parametrize("ngroups,hint,want", [(60, 0, P.AGG_PATH_V1_LOCAL | P.AGG_PATH_MERGE), (60_000, 60_000, P.AGG_PATH_V1_GLOBAL)])
def test_v1_paths(ngroups, hint, want, monkeypatch):
    monkeypatch.setenv("TG_AGG_V1", "1")
    monkeypatch.setenv("TG_AGG_LOCAL_SLOTS", "512")
    p, s = 15, 2
    vals = make_vals(np.random.default_rng(40 + ngroups), 150_000, ngroups, p, s)
    v2 = P.AGG_PATH_V2_LOCAL | P.AGG_PATH_V2_GLOBAL
    check_paths(plans(p, s, expected_groups=hint, small=True), to_chunk(vals, p, s).split(1 << 15), vals, want=want, dont=v2, local=False)


@pytest.mark.parametrize("group_by", [(G, K2), (K3, K4), (G, K2, K3), (G, K2, K3, K4)])
def test_multi_key(group_by):
    p, s = 18, 2
    vals = make_vals(np.random.default_rng(50 + len(group_by)), 120_000, 50, p, s)
    check_paths(plans(p, s, group_by=group_by, expected_groups=16), to_chunk(vals, p, s).split(1 << 15), vals,
                want=P.AGG_PATH_MULTI_KEY, dont=~P.AGG_PATH_MULTI_KEY)


def test_double_group_key_zeros_form_one_group():
    p, s = 18, 2
    vals = make_vals(np.random.default_rng(55), 50_000, 1, p, s)
    check_paths(plans(p, s, group_by=(K4,), small=True), to_chunk(vals, p, s).split(1 << 14), vals, want=P.AGG_PATH_V2_LOCAL)


# ---- known answers -------------------------------------------------------------------------------------------------
def test_integration_answers():
    # the reference's tests/integrationtest/r/executor/aggregate.result: t1(a int, b int) grouped by a
    t1 = [(1, 1), (2, 2), (3, 3), (1, 4), (1, 1), (3, 5), (2, 2), (3, 5), (3, 3)]
    a = np.array([r[0] for r in t1], dtype=np.int64)
    b = np.array([r[1] for r in t1], dtype=np.int64)
    plan = AggPlan([INT, INT], [0], [AggFunc(P.AGG_FIRSTROW, 0), davg(1, 4), dsum(1), cnt(1), AggFunc(P.AGG_MAX, 1, distinct=True)])
    rows, _, ds = run_host(plan, [Chunk([Column(a), Column(b)])])
    got = sorted((r[0], D.to_string(r[1]), D.to_string(r[2]), r[3], r[4]) for r in rows)
    assert got == [(1, "2.5000", "5", 2, 4), (2, "2.0000", "2", 1, 2), (3, "4.0000", "8", 2, 5)]
    assert ds.pairs == 5
    # no GROUP BY over no rows: the default row; over all-NULL rows: COUNT 0, SUM / AVG NULL
    plan = AggPlan([INT, INT], [], [cnt(1), dsum(1), davg(1, 4)])
    assert run_host(plan, [])[0] == [(0, None, None)]
    assert run_host(plan, [Chunk([Column(a), Column(b, np.ones(len(b), dtype=bool))])])[0] == [(0, None, None)]


# ---- across pushes -----------------------------------------------------------------------------------------------
def test_host_pushes_with_sel_skip_unselected_rows():
    p, s = 18, 2
    rng = np.random.default_rng(60)
    vals = make_vals(rng, 90_000, 300, p, s)
    n = len(vals[G][0])
    other = make_vals(np.random.default_rng(61), n, 300, p, s, pool=400)   # values the selected rows never hold
    phys = {c: (np.empty(2 * n, dtype=vals[c][0].dtype), np.empty(2 * n, dtype=bool)) for c in vals}
    for c in vals:
        phys[c][0][0::2], phys[c][1][0::2] = vals[c]
        phys[c][0][1::2], phys[c][1][1::2] = other[c]
    big = to_chunk(phys, p, s)
    chunks = []
    for lo in range(0, 2 * n, 1 << 14):
        part = Chunk([c.slice(lo, min(2 * n, lo + (1 << 14))) for c in big.columns])
        chunks.append(Chunk(part.columns, np.arange(0, part.num_rows(), 2)))
    check_paths(plans(p, s), chunks, vals, want=P.AGG_PATH_V2_GLOBAL)


@pytest.mark.parametrize("misalign", [False, True])
def test_device_pushes_repeat_values(misalign):
    p, s = 15, 2
    rng = np.random.default_rng(70 + misalign)
    parts = [make_vals(rng, n, g, p, s) for n, g in ((50_001, 30), (100_000, 3000), (99_999, 3000))]
    vals = concat(*parts)
    for plan in plans(p, s) + plans(p, s, group_by=()) + plans(p, s, group_by=(G, K3), expected_groups=16):
        e = HashAggExec(plan, MockDataSource(plan.col_types, []))
        e.open()
        try:
            for q in parts:
                push_dev(e, to_chunk(q, p, s), misalign)
            DR.check(plan, vals, drain(e))
            ds = e.distinct_stats()
            cols = sorted({f.arg_col for f in plan.funcs if f.distinct and f.name != P.AGG_MAX})
            assert ds.pairs == sum(DR.pair_count(plan, vals, c) for c in cols)
        finally:
            e.close()


@pytest.mark.parametrize("group_by", [(), (G,), (G, K2)])
def test_set_grows(group_by):
    p, s = 18, 2
    rng = np.random.default_rng(80 + len(group_by))
    small = make_vals(rng, 1000, 10, p, s)
    n = 1_000_000
    big = make_vals(rng, n, 1000, p, s)
    big[X] = (rng.permutation(n).astype(np.int64) * 7919 - (1 << 40), np.zeros(n, dtype=bool))   # ~1 M new pairs
    big[DD] = (rng.standard_normal(n), np.zeros(n, dtype=bool))
    vals = concat(small, big)
    plan = AggPlan(types_of(p, s), list(group_by), [AggFunc(P.AGG_FIRSTROW, g) for g in group_by] +
                   [cnt(X), dsum(X), cnt(DD), AggFunc(P.AGG_AVG, DD, P.TYPE_DOUBLE, distinct=True)])
    e = HashAggExec(plan, MockDataSource(plan.col_types, []))
    e.open()
    try:
        push_dev(e, to_chunk(small, p, s))
        push_dev(e, to_chunk(big, p, s))
        DR.check(plan, vals, drain(e))
        ds = e.distinct_stats()
        assert ds.set_grows > 0 and ds.launches > 4
        assert ds.pairs == DR.pair_count(plan, vals, X) + DR.pair_count(plan, vals, DD)
        assert ds.set_slots >= ds.pairs
    finally:
        e.close()


def test_bad_decimal_cell_leaves_groups_and_sets_unchanged():
    p, s = 15, 2
    rng = np.random.default_rng(90)
    one, two = make_vals(rng, 20_000, 100, p, s), make_vals(rng, 20_000, 100, p, s)
    plan = plans(p, s)[2]
    e = HashAggExec(plan, MockDataSource(plan.col_types, []))
    e.open()
    try:
        push_dev(e, to_chunk(one, p, s))
        pairs = e.distinct_stats().pairs
        bad = to_chunk(two, p, s)
        r = int(np.flatnonzero(~two[DA][1])[-1])
        cells = bad.columns[DA].data.copy()
        cells[r, 1] = s + 1                                  # digitsFrac != the column's scale
        bad = Chunk(bad.columns[:DA] + [Column(cells, two[DA][1] if two[DA][1].any() else None)] + bad.columns[DA + 1:])
        with pytest.raises(abi.TgError) as ei:
            push_dev(e, bad)
        assert ei.value.code == abi.TG_ERR_INVALID
        assert e.distinct_stats().pairs == pairs
        push_dev(e, to_chunk(two, p, s))                     # the same values again: counted once
        vals = concat(one, two)
        DR.check(plan, vals, drain(e))
        assert e.distinct_stats().pairs == DR.pair_count(plan, vals, DA)
    finally:
        e.close()


# ---- full scale ----------------------------------------------------------------------------------------------------
def test_full_scale_count_distinct():
    import torch
    from tidb_b200.device import DeviceAgg, fetch_device
    n, ng = 100_000_000, 1_000_000
    g = torch.Generator(device="cuda"); g.manual_seed(7)
    keys = torch.randint(0, ng, (n,), device="cuda", generator=g, dtype=torch.int64)
    v = torch.randint(0, 16, (n,), device="cuda", generator=g, dtype=torch.int64)
    plan = AggPlan([INT_NN, INT_NN], [0], [AggFunc(P.AGG_FIRSTROW, 0), cnt(1)], expected_groups=ng)
    torch.cuda.synchronize()
    agg = DeviceAgg(plan)
    try:
        agg.push([keys, v])
        rows, cols, _ = agg.finish()
        ds = agg.distinct_stats()
        gk = np.frombuffer(fetch_device(cols[0], rows * 8).tobytes(), dtype=np.int64)
        got = np.frombuffer(fetch_device(cols[1], rows * 8).tobytes(), dtype=np.int64)
    finally:
        agg.close()
    pairs = np.unique((keys.cpu().numpy() << 4) | v.cpu().numpy())
    want = np.bincount(pairs >> 4, minlength=ng)
    assert rows == np.count_nonzero(want) and ds.pairs == len(pairs)
    order = np.argsort(gk)
    assert np.array_equal(gk[order], np.flatnonzero(want)) and np.array_equal(got[order], want[want > 0])
