"""Every update path of the CUDA hash aggregation against the exact reference (tests/agg_reference.py).

Each case forces one path through the TG_AGG_* switches and proves from tg_agg_stats.paths / local_rows that the path
ran, then compares every group with the reference: COUNT, MIN, MAX and FIRSTROW bit-exact, SUM and AVG inside the
summation error bound.  The data holds the values where aggregation kernels go wrong: groups made only of the values the
device states start from (MIN of INT64_MAX, MAX of INT64_MIN, unsigned MIN of 2**64-1 and MAX of 0, DOUBLE MAX of -inf),
groups whose arguments are all NULL, the NULL group and the INT64_MIN group, full-range integers, DOUBLE extremes
(+-inf, +-DBL_MAX, -0.0, subnormals), and sums that cancel (x, -x pairs plus a small remainder)."""
import ctypes as C

import numpy as np
import pytest

import agg_reference as R
from nested_loop import columns_to_rows
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.executor import HashAggExec, MockDataSource
from tidb_b200.plan import AggFunc, AggPlan, FieldType

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
UINT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
DBL_NN = FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)
FINAL = abi.AGGMODE_FINAL
SWITCHES = ("TG_AGG_LOCAL", "TG_AGG_LOCAL_SLOTS", "TG_AGG_V1")
P = abi
DMAX = np.finfo(np.float64).max
EXTREMES = np.array([np.inf, -np.inf, DMAX, -DMAX, -0.0, 0.0, 5e-324, -5e-324, 1e-310, -1e-310, 2.2250738585072014e-308, 1.0, -1.0])

# special group keys (far from the regular keys): each group is made of one kind of value
K_ALLNULL, K_IMAX, K_IMIN, K_UMAX, K_UZERO, K_NEGINF, K_POSINF = (7_000_000_000_000 + j for j in range(7))
SPECIAL = (K_ALLNULL, K_IMAX, K_IMIN, K_UMAX, K_UZERO, K_NEGINF, K_POSINF)


@pytest.fixture(autouse=True)
def _default_switches(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)


# ---- data --------------------------------------------------------------------------------------------------------
# columns: 0 g key (nullable) | 1 x DOUBLE (nullable, cancelling) | 2 xnn DOUBLE NOT NULL | 3 i BIGINT (nullable, full range)
#          4 u BIGINT UNSIGNED (nullable, full range) | 5 d DOUBLE (nullable, extremes) | 6 inn BIGINT NOT NULL (full range)
TYPES = [INT, DBL, DBL_NN, INT, UINT, DBL, INT_NN]


def make_rows(rng, n, ngroups):
    """n rows over about ngroups regular groups plus the special, NULL and INT64_MIN groups"""
    half = n // 2
    gp = (rng.integers(0, ngroups, half) * 2654435761 % (1 << 40) - (1 << 39)).astype(np.int64)
    sp = rng.random(half) < 0.004                            # pairs that go to a special group
    gp[sp] = rng.choice(np.array(SPECIAL, dtype=np.int64), int(sp.sum()))
    gp[rng.random(half) < 0.002] = I64_MIN                   # the key equal to the table's empty sentinel
    gnp = rng.random(half) < 0.01                            # the NULL group
    v = (rng.random(half) - 0.5) * 1e12                      # x, -x pairs in one group: the sum cancels
    g = np.repeat(gp, 2); gn = np.repeat(gnp, 2)
    x = np.stack([v, -v], axis=1).ravel()
    rem = rng.random(n) < 0.02
    x[rem] += (rng.random(int(rem.sum())) - 0.5) * 1e-3      # ... plus a small remainder
    xn = np.repeat(rng.random(half) < 0.05, 2)
    xnn = (rng.random(n) - 0.5) * 1e6
    i = rng.integers(I64_MIN, I64_MAX, n, endpoint=True, dtype=np.int64)
    u = rng.integers(0, 1 << 64, n, dtype=np.uint64).view(np.int64)
    d = np.where(rng.random(n) < 0.3, rng.choice(EXTREMES, n), rng.standard_normal(n) * 1e3)
    inn = rng.integers(I64_MIN, I64_MAX, n, endpoint=True, dtype=np.int64)
    iN, uN, dN = rng.random(n) < 0.05, rng.random(n) < 0.05, rng.random(n) < 0.05
    key = np.where(gn, 0, g)
    for k, col, val, nl in ((K_IMAX, i, I64_MAX, iN), (K_IMIN, i, I64_MIN, iN), (K_UMAX, u, -1, uN), (K_UZERO, u, 0, uN),
                            (K_NEGINF, d, -np.inf, dN), (K_POSINF, d, np.inf, dN)):
        m = key == k
        col[m] = val
        if k == K_IMAX:
            inn[m] = I64_MAX
        if k == K_IMIN:
            inn[m] = I64_MIN
    m = key == K_ALLNULL
    xn = xn | m; iN = iN | m; uN = uN | m; dN = dN | m
    perm = rng.permutation(n)
    cols = [Column(g, gn), Column(x, xn), Column(xnn), Column(i, iN), Column(u, uN), Column(d, dN), Column(inn)]
    return Chunk([Column(c.data[perm], c.nulls()[perm]) for c in cols])


def plans(group_by=(0,), expected_groups=0):
    """the aggregate list split into plans of at most 4 device states each, so that the CTA-local level accepts them"""
    fr = [AggFunc(P.AGG_FIRSTROW, 0)] if group_by else []
    lists = [
        [AggFunc(P.AGG_COUNT, -1), AggFunc(P.AGG_SUM, 1, P.TYPE_DOUBLE), AggFunc(P.AGG_COUNT, 1, P.TYPE_DOUBLE), AggFunc(P.AGG_AVG, 2, P.TYPE_DOUBLE)],
        [AggFunc(P.AGG_MIN, 3), AggFunc(P.AGG_MAX, 3)],
        [AggFunc(P.AGG_MIN, 4), AggFunc(P.AGG_MAX, 4)],
        [AggFunc(P.AGG_MIN, 5, P.TYPE_DOUBLE), AggFunc(P.AGG_MAX, 5, P.TYPE_DOUBLE)],
        [AggFunc(P.AGG_AVG, 1, P.TYPE_DOUBLE), AggFunc(P.AGG_MIN, 6), AggFunc(P.AGG_SUM, 2, P.TYPE_DOUBLE)],
        [AggFunc(P.AGG_MAX, 6), AggFunc(P.AGG_COUNT, 2, P.TYPE_DOUBLE), AggFunc(P.AGG_MAX, 2, P.TYPE_DOUBLE)],
    ]
    return [AggPlan(TYPES, list(group_by), fr + fs, expected_groups=expected_groups) for fs in lists]


def make_partials(rng, n, ngroups):
    """partial results (count, sum) as a TiDB partial worker sends them: a worker that saw no non-NULL row of a group
    sends count 0 and a NULL sum"""
    g = rng.integers(0, ngroups, n).astype(np.int64)
    g[:5] = I64_MIN
    gn = rng.random(n) < 0.01
    cnt = rng.integers(0, 1 << 20, n).astype(np.int64)
    cnt[rng.random(n) < 0.1] = 0
    v = (rng.random(n // 2) - 0.5) * 1e12
    sm = np.stack([v, -v], axis=1).ravel()[:n] + (rng.random(n) - 0.5)
    smn = cnt == 0
    g[(g % 97) == 3] = 3; cnt[g == 3] = 0; smn[g == 3] = True      # group 3: every partial sum NULL, counts 0
    return Chunk([Column(g, gn), Column(cnt), Column(sm, smn)])


def final_plans(group_by=(0,), expected_groups=0):
    types = [INT, INT_NN, DBL]
    fr = [AggFunc(P.AGG_FIRSTROW, 0)] if group_by else []
    return [AggPlan(types, list(group_by), fr + [AggFunc(P.AGG_COUNT, 1, mode=FINAL), AggFunc(P.AGG_SUM, 2, P.TYPE_DOUBLE, mode=FINAL)],
                    expected_groups=expected_groups),
            AggPlan(types, list(group_by), fr + [AggFunc(P.AGG_AVG, 1, P.TYPE_LONGLONG, mode=FINAL, arg_col2=2)], expected_groups=expected_groups)]


# ---- running ---------------------------------------------------------------------------------------------------
def run_host(plan, chunks):
    """tg_agg_push of every chunk (host memory, staged by the library), then finish / next; returns (rows, stats)"""
    e = HashAggExec(plan, MockDataSource(plan.col_types, chunks))
    e.open()
    try:
        rows = []
        while True:
            c = e.next(1 << 20)
            if c.num_rows() == 0:
                break
            rows.extend(columns_to_rows([(col.data, col.nulls()) for col in c.columns]))
        return rows, e.stats()
    finally:
        e.close()


def run_dev(plan, batches):
    """one tg_agg_push_dev per batch (each batch is one device update), then finish / next; returns (rows, stats)"""
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
            rows.extend(columns_to_rows([(col.data, col.nulls()) for col in c.columns]))
        return rows, e.stats()
    finally:
        e.close()


def check_all(plan_list, chunks, want, dont=0, local=None, runner=None):
    """run every plan, compare with the reference, assert the path bits `want` (all set) / `dont` (all clear) and, when
    `local` is given, whether the CTA-local level absorbed rows; returns the stats of the last plan"""
    st = None
    for plan in plan_list:
        rows, st = (runner or run_host)(plan, chunks)
        R.check(plan, chunks, rows)
        assert st.paths & want == want, (hex(st.paths), hex(want))
        assert st.paths & dont == 0, (hex(st.paths), hex(dont))
        if local is not None:
            assert (st.local_rows > 0) == local, st.local_rows
    return st


# ---- paths -----------------------------------------------------------------------------------------------------
def test_no_group_by():
    rng = np.random.default_rng(1)
    chunks = make_rows(rng, 300_000, 50).split(1 << 15)
    check_all(plans(group_by=()), chunks, want=P.AGG_PATH_NOGROUP, dont=~P.AGG_PATH_NOGROUP)
    check_all(final_plans(group_by=()), make_partials(rng, 100_000, 20).split(1 << 14), want=P.AGG_PATH_NOGROUP, dont=~P.AGG_PATH_NOGROUP)
    # a single identity-valued row is still a result
    one = Chunk([Column(np.zeros(1, dtype=np.int64)), Column(np.zeros(1)), Column(np.zeros(1)), Column(np.array([I64_MAX])),
                 Column(np.array([-1], dtype=np.int64)), Column(np.array([-np.inf])), Column(np.array([I64_MIN]))])
    check_all(plans(group_by=()), [one], want=P.AGG_PATH_NOGROUP)


@pytest.mark.parametrize("ngroups", [40, 60_000])
def test_v2_global_only(ngroups, monkeypatch):
    monkeypatch.setenv("TG_AGG_LOCAL", "0")
    rng = np.random.default_rng(2 + ngroups)
    check_all(plans(), make_rows(rng, 200_000, ngroups).split(1 << 15), want=P.AGG_PATH_V2_GLOBAL,
              dont=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE, local=False)
    check_all(final_plans(), make_partials(rng, 100_000, ngroups).split(1 << 15), want=P.AGG_PATH_V2_GLOBAL, dont=P.AGG_PATH_V2_LOCAL, local=False)


@pytest.mark.parametrize("slots", [None, "512"])
def test_v2_two_level_low_cardinality(slots, monkeypatch):
    if slots:
        monkeypatch.setenv("TG_AGG_LOCAL_SLOTS", slots)
    rng = np.random.default_rng(3)
    check_all(plans(), make_rows(rng, 400_000, 60).split(1 << 15), want=P.AGG_PATH_V2_LOCAL, local=True)
    check_all(final_plans(), make_partials(rng, 200_000, 60).split(1 << 15), want=P.AGG_PATH_V2_LOCAL, local=True)


def test_v2_local_forced_high_cardinality_spills_and_merges(monkeypatch):
    # TG_AGG_LOCAL=2 keeps the CTA-local level on a 100 K-group input, and a 64-group hint leaves the global table far too
    # small: local groups that find no global slot spill, the host grows the table and folds them in (merge_partials).
    # This input, the several-push test below and test_agg_two_level_paths_vs_oracle[300-...] emitted groups twice while
    # the rehash and the merge placed keys by another hash than the update kernel looked them up with
    monkeypatch.setenv("TG_AGG_LOCAL", "2")
    rng = np.random.default_rng(4)
    st = check_all(plans(expected_groups=64), make_rows(rng, 300_000, 100_000).split(1 << 16),
                   want=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE, local=True)
    assert st.table_slots > 1024
    check_all(final_plans(expected_groups=64), make_partials(rng, 300_000, 100_000).split(1 << 16), want=P.AGG_PATH_V2_LOCAL | P.AGG_PATH_MERGE)


@pytest.mark.parametrize("ngroups,hint,want", [(60, 0, P.AGG_PATH_V1_LOCAL | P.AGG_PATH_MERGE),
                                               (60_000, 0, P.AGG_PATH_V1_LOCAL | P.AGG_PATH_MERGE | P.AGG_PATH_V1_GLOBAL),
                                               (60_000, 60_000, P.AGG_PATH_V1_GLOBAL)])
def test_v1_paths(ngroups, hint, want, monkeypatch):
    # the legacy update (TG_AGG_V1=1): CTA-local partial pass + merge, then the global kernel for the rows a CTA-local
    # table could not take.  512-slot local tables overflow on the high-cardinality input, so both levels run
    monkeypatch.setenv("TG_AGG_V1", "1")
    monkeypatch.setenv("TG_AGG_LOCAL_SLOTS", "512")
    rng = np.random.default_rng(5 + ngroups + hint)
    v2 = P.AGG_PATH_V2_LOCAL | P.AGG_PATH_V2_GLOBAL
    check_all(plans(expected_groups=hint), make_rows(rng, 300_000, ngroups).split(1 << 15), want=want, dont=v2, local=False)
    check_all(final_plans(expected_groups=hint), make_partials(rng, 300_000, ngroups).split(1 << 15), want=want, dont=v2)


def test_several_device_pushes_with_growth():
    # four tg_agg_push_dev batches into one handle, each with more groups than the last: later batches find the groups of
    # earlier ones, and the table grows between batches
    rng = np.random.default_rng(6)
    batches = [make_rows(rng, n, g) for n, g in ((50_000, 30), (100_000, 3000), (100_000, 30_000), (50_000, 40_000))]
    for plan in plans(expected_groups=16):
        rows, st = run_dev(plan, batches)
        R.check(plan, batches, rows)
        assert st.table_slots > 1024 and st.paths & (P.AGG_PATH_V2_LOCAL | P.AGG_PATH_V2_GLOBAL)
    rows, st = run_dev(plans(group_by=())[0], batches)
    R.check(plans(group_by=())[0], batches, rows)


def test_sel_vectors(monkeypatch):
    # host chunks that carry a selection vector: only the selected rows count
    rng = np.random.default_rng(7)
    chunks = []
    for c in make_rows(rng, 300_000, 500).split(1 << 14):
        sel = np.sort(rng.choice(c.num_rows(), c.num_rows() // 3, replace=False))
        chunks.append(Chunk(c.columns, sel))
    check_all(plans(), chunks, want=P.AGG_PATH_V2_LOCAL)
    monkeypatch.setenv("TG_AGG_V1", "1")
    check_all(plans()[:2], chunks, want=P.AGG_PATH_V1_LOCAL)


def test_host_push_with_null_data_pointer_is_rejected():
    # a needed column of a host chunk with rows but no data pointer is invalid input: the push fails before anything is
    # staged, and the handle aggregates the next pushes as if it had never been offered
    plan = AggPlan([INT_NN, INT_NN], [0], [AggFunc(P.AGG_FIRSTROW, 0), AggFunc(P.AGG_COUNT, -1), AggFunc(P.AGG_MIN, 1),
                                           AggFunc(P.AGG_MAX, 1)])
    vals = np.arange(1000, dtype=np.int64)
    good = Chunk([Column(vals % 7), Column(vals)])
    bad = Chunk(good.columns)
    lib = abi.load_lib()
    e = HashAggExec(plan, MockDataSource(plan.col_types, []))
    e.open()
    try:
        bs = bad.to_struct()
        bs.cols[1].data = None
        assert lib.tg_agg_push(e._h, C.byref(bs)) == abi.TG_ERR_INVALID
        assert b"data is NULL" in lib.tg_last_error()
        gs = good.to_struct()
        abi.check(lib.tg_agg_push(e._h, C.byref(gs)))
        abi.check(lib.tg_agg_finish(e._h))
        e._prepared = True
        out = e.next(1 << 10)
        rows = sorted(zip(*(c.data.tolist() for c in out.columns)))
        assert rows == [(k, len(vals[k::7]), k, int(vals[k::7][-1])) for k in range(7)]
    finally:
        e.close()


# ---- several GROUP BY columns ----------------------------------------------------------------------------------
def mk_rows(rng, n, ncols, card):
    """ncols key columns (column 0 nullable with both 0 and NULL present, column 1 a DOUBLE with -0.0 and +0.0) + the TYPES
    argument columns"""
    base = make_rows(rng, n, 50)
    keys, types = [], []
    for c in range(ncols):
        if c == 0:
            keys.append(Column(rng.integers(-card, card + 1, n).astype(np.int64), rng.random(n) < 0.2)); types.append(INT)
        elif c == 1:
            v = rng.integers(-card, card + 1, n).astype(np.float64) * 0.5
            v[v == 0] = np.where(rng.random(int((v == 0).sum())) < 0.5, -0.0, 0.0)
            keys.append(Column(v)); types.append(DBL_NN)
        else:
            v = rng.integers(-card, card + 1, n).astype(np.int64)
            v[rng.random(n) < 0.001] = I64_MIN
            keys.append(Column(v)); types.append(INT_NN)
    return Chunk(keys + base.columns[1:]), types


def mk_plans(ncols, types):
    a = ncols - 1                        # argument columns follow the keys: x, xnn, i, u, d, inn at a+1 .. a+6
    t = types + TYPES[1:]
    fr = [AggFunc(P.AGG_FIRSTROW, c) for c in range(ncols)]
    lists = [[AggFunc(P.AGG_COUNT, -1), AggFunc(P.AGG_SUM, a + 1, P.TYPE_DOUBLE), AggFunc(P.AGG_COUNT, a + 1, P.TYPE_DOUBLE),
              AggFunc(P.AGG_AVG, a + 1, P.TYPE_DOUBLE), AggFunc(P.AGG_AVG, a + 2, P.TYPE_DOUBLE), AggFunc(P.AGG_SUM, a + 2, P.TYPE_DOUBLE)],
             [AggFunc(P.AGG_MIN, a + 3), AggFunc(P.AGG_MAX, a + 3), AggFunc(P.AGG_MIN, a + 4), AggFunc(P.AGG_MAX, a + 4),
              AggFunc(P.AGG_MIN, a + 5, P.TYPE_DOUBLE), AggFunc(P.AGG_MAX, a + 5, P.TYPE_DOUBLE), AggFunc(P.AGG_MIN, a + 6), AggFunc(P.AGG_MAX, a + 6)]]
    return [AggPlan(t, list(range(ncols)), fr + fs, expected_groups=16) for fs in lists]


@pytest.mark.parametrize("ncols", [2, 3, 4])
def test_multi_key(ncols):
    rng = np.random.default_rng(8 + ncols)
    chk, types = mk_rows(rng, 200_000, ncols, 5)
    check_all(mk_plans(ncols, types), chk.split(1 << 15), want=P.AGG_PATH_MULTI_KEY, dont=~P.AGG_PATH_MULTI_KEY)


def test_multi_key_contention_three_groups():
    # about 1 M rows over 3 distinct 4-column keys: every warp races for the same records (tag claim, the two 128-bit
    # record loads), MIN / AVG / integer MIN / MAX over each
    rng = np.random.default_rng(9)
    n = 1 << 20
    chk, _ = mk_rows(rng, n, 4, 1)
    types = [INT_NN, DBL_NN, INT_NN, INT]
    pick = rng.integers(0, 3, n)
    keys = [np.array([5, -3, 5])[pick], np.array([0.5, -0.0, -0.5])[pick], np.array([I64_MIN, 7, 7])[pick], np.array([0, 0, 1])[pick]]
    kn = (pick == 0)                           # (5, 0.5, INT64_MIN, NULL) and (-3, -0.0, 7, 0) and (5, -0.5, 7, 1)
    cols = [Column(keys[0].astype(np.int64)), Column(keys[1]), Column(keys[2].astype(np.int64)), Column(keys[3].astype(np.int64), kn)] + chk.columns[4:]
    chunks = Chunk(cols).split(1 << 18)
    st = check_all(mk_plans(4, types), chunks, want=P.AGG_PATH_MULTI_KEY)
    assert st.groups == 3


def test_multi_key_null_differs_from_zero():
    # (NULL, x) and (0, x) are different groups: the NULL bits word of the key tells them apart
    g0 = np.array([0, 0, 0, 1, 1, 0], dtype=np.int64)
    g0n = np.array([True, False, True, False, False, False])
    g1 = np.array([4, 4, 4, 4, 4, 5], dtype=np.int64)
    x = np.array([1.0, 2.0, 4.0, 8.0, 16.0, 32.0])
    plan = AggPlan([INT, INT_NN, DBL_NN], [0, 1], [AggFunc(P.AGG_FIRSTROW, 0), AggFunc(P.AGG_FIRSTROW, 1), AggFunc(P.AGG_COUNT, -1),
                                                    AggFunc(P.AGG_SUM, 2, P.TYPE_DOUBLE)])
    chunks = [Chunk([Column(g0, g0n), Column(g1), Column(x)])]
    rows, st = run_host(plan, chunks)
    assert R.check(plan, chunks, rows) == 4
    assert sorted(rows, key=repr) == sorted([(None, 4, 2, 5.0), (0, 4, 1, 2.0), (1, 4, 2, 24.0), (0, 5, 1, 32.0)], key=repr)
