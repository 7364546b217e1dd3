"""Parity of the CUDA hash join against the oracle, through the C-ABI (HashJoinExec → tg_join_*).

Mirrors the reference's join tests: random chunks with forced matches, sel vectors, NULL keys,
duplicate keys, both build sides, every join type (testJoinProbe inner_join_probe_test.go:228 and
siblings); comparison = sorted row multisets (checkChunksEqual :137).  Integer columns bit-exact."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from nested_loop import assert_rows_equal, columns_sorted, columns_to_rows
from test_oracle_join import DBL, INT, INT_NN, JOIN_TYPES, UINT_NN, col, make_case, run_oracle
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.executor import HashJoinExec, MockDataSource, drain
from tidb_b200.plan import FieldType, FilterItem, JoinPlan

pytestmark = pytest.mark.gpu


def run_gpu(plan, left, right, required_rows=1024):
    e = HashJoinExec(plan, MockDataSource(plan.left_types, left), MockDataSource(plan.right_types, right))
    chunks = drain(e, required_rows)
    rows = []
    for c in chunks:
        rows.extend(columns_to_rows([(col_.data, col_.nulls()) for col_ in c.columns]))
    return rows


def run_gpu_stats(plan, left, right, required_rows=1024):
    """run_gpu, plus the handle's tg_join_stats read before close"""
    e = HashJoinExec(plan, MockDataSource(plan.left_types, left), MockDataSource(plan.right_types, right))
    e.open()
    try:
        rows = []
        while True:
            c = e.next(required_rows)
            if c.num_rows() == 0:
                break
            rows.extend(columns_to_rows([(col_.data, col_.nulls()) for col_ in c.columns]))
        return rows, e.stats()
    finally:
        e.close()


def test_device_present():
    lib = abi.load_lib()
    assert lib.tg_device_count() > 0, "GPU tests need a CUDA device"
    name = C.create_string_buffer(128); sm = C.c_int(0); mem = C.c_int64(0)
    abi.check(lib.tg_device_info(0, name, 128, C.byref(sm), C.byref(mem)))
    assert sm.value > 0


def test_sql_hash_join_goldens_on_gpu():
    # tests/integrationtest/r/executor/jointest/hash_join.result:1-22 and :36-60
    t = Chunk([col(list(range(1, 129)), [False] * 128)])
    s = Chunk([col([1, 128], [False, False])])
    plan = JoinPlan(abi.JOIN_INNER, [INT], [INT], [0], [0])
    assert sorted(run_gpu(plan, t.split(32), [s])) == [(1, 1), (128, 128)]
    t = [Chunk([col([148307968, -1327693824, -277544960], [False] * 3)])]
    s = [Chunk([col([-277544960, 2, 2, -277544960, 2, 6], [False] * 6)])]
    inner = JoinPlan(abi.JOIN_INNER, [INT], [INT], [0], [0], lused=[0], rused=[])
    assert sorted(run_gpu(inner, t, s)) == [(-277544960,), (-277544960,)]
    left = JoinPlan(abi.JOIN_LEFT_OUTER, [INT], [INT], [0], [0], lused=[0], rused=[])
    assert sorted(run_gpu(left, t, s)) == [(-1327693824,), (-277544960,), (-277544960,), (148307968,)]
    # pkg/executor/test/jointest/join_test.go:66-80
    t = [Chunk([col([1, 2], [False, False]), col([1, 2], [False, False])])]
    t1 = [Chunk([col([2, 4], [False, False]), col([3, 4], [False, False])])]
    lo = JoinPlan(abi.JOIN_LEFT_OUTER, [INT, INT], [INT, INT], [0], [0])
    assert sorted(run_gpu(lo, t, t1), key=str) == sorted([(1, 1, None, None), (2, 2, 2, 3)], key=str)
    ro = JoinPlan(abi.JOIN_RIGHT_OUTER, [INT, INT], [INT, INT], [0], [0], build_is_right=False)
    assert sorted(run_gpu(ro, t1, t), key=str) == sorted([(None, None, 1, 1), (2, 3, 2, 2)], key=str)


def test_sql_join_result_goldens_multi_key_other_condition_on_gpu():
    # the reference's SQL known answers for several equal conditions, a non-equi residual and date-time keys
    # (tests/sql_goldens.py, from tests/integrationtest/r/executor/jointest/join.result) through the CUDA path
    import sql_goldens
    for name, plan, left, right, count, rows in sql_goldens.cases():
        got = run_gpu(plan, left, right)
        assert len(got) == count, name
        if rows is not None:
            assert sorted(got) == sorted(rows), name


@pytest.mark.parametrize("jt", JOIN_TYPES)
@pytest.mark.parametrize("build_is_right", [True, False])
@pytest.mark.parametrize("nulls,dup,with_sel", [(0.0, False, False), (0.15, True, False), (0.1, True, True)])
def test_gpu_vs_oracle_all_join_types(jt, build_is_right, nulls, dup, with_sel):
    if jt in (abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI) and not build_is_right:
        pytest.skip("NewJoinProbe panics: left outer semi needs right build (base_join_probe.go:913)")
    rng = np.random.default_rng(4321 + jt * 7 + int(build_is_right))
    ltypes, rtypes, l, r = make_case(rng, 3000, 4000, nulls, dup, with_sel)
    semi = jt >= abi.JOIN_SEMI
    plan = JoinPlan(jt, ltypes, rtypes, [1], [0], build_is_right=build_is_right,
                    lused=[0, 1, 2], rused=[] if semi else [2, 0])
    assert_rows_equal(run_oracle(plan, l, r), run_gpu(plan, l, r))


@pytest.mark.parametrize("jt", [abi.JOIN_INNER, abi.JOIN_LEFT_OUTER, abi.JOIN_RIGHT_OUTER, abi.JOIN_SEMI])
def test_gpu_filters(jt):
    rng = np.random.default_rng(77 + jt)
    ltypes, rtypes, l, r = make_case(rng, 2000, 3000, 0.1, True, False)
    semi = jt >= abi.JOIN_SEMI
    signed = ([FilterItem(abi.CMP_GT, 0, const_i64=0)],
              [FilterItem(abi.CMP_LT, 1, const_i64=1 << 39), FilterItem(abi.CMP_NE, 2, rhs_col=1)])
    # UNSIGNED items over the same words: a negative word is a value of at least 2^63 (types.CompareInt)
    unsigned = ([FilterItem(abi.CMP_LT, 0, const_i64=1 << 39, lhs_unsigned=True)],
                [FilterItem(abi.CMP_GT, 1, rhs_col=2, lhs_unsigned=True), FilterItem(abi.CMP_LE, 2, rhs_col=1, rhs_unsigned=True),
                 FilterItem(abi.CMP_LT, 0, const_i64=-20, lhs_unsigned=True, rhs_unsigned=True)])
    for (lf, rf), build_is_right in ((f, b) for f in (signed, unsigned) for b in (True, False)):
        plan = JoinPlan(jt, ltypes, rtypes, [1], [0], build_is_right=build_is_right, lused=None, rused=[] if semi else None,
                        build_filter=rf if build_is_right else lf, probe_filter=lf if build_is_right else rf)
        if jt == abi.JOIN_LEFT_OUTER:
            plan.build_filter, plan.probe_filter = ([], lf) if build_is_right else (lf, [])
        if jt == abi.JOIN_RIGHT_OUTER:
            plan.build_filter, plan.probe_filter = (rf, []) if build_is_right else ([], rf)
        if semi:
            plan.build_filter, plan.probe_filter = ([], lf) if build_is_right else (lf, [])
        assert_rows_equal(run_oracle(plan, l, r), run_gpu(plan, l, r))


@pytest.mark.parametrize("jt,build_is_right", [(abi.JOIN_INNER, True), (abi.JOIN_INNER, False), (abi.JOIN_LEFT_OUTER, True),
                                               (abi.JOIN_RIGHT_OUTER, False), (abi.JOIN_SEMI, True), (abi.JOIN_ANTI_SEMI, True)])
@pytest.mark.parametrize("nulls,dup,with_sel", [(0.0, False, False), (0.12, True, True)])
def test_gpu_other_condition(jt, build_is_right, nulls, dup, with_sel):
    # OtherCondition evaluated on candidate pairs on the device (k_probe_count / k_probe_write, csrc/join_kernels.cuh):
    # column-vs-column across the two sides plus a constant item, NULL operands never pass; unique and duplicate build keys
    from tidb_b200.plan import OtherCond
    rng = np.random.default_rng(31 + jt + 10 * int(build_is_right))
    ltypes, rtypes, l, r = make_case(rng, 3000, 4000, nulls, dup, with_sel)
    semi = jt >= abi.JOIN_SEMI
    other = [OtherCond(abi.CMP_LE, 0, 0, 1, 1), OtherCond(abi.CMP_NE, 1, 2, -1, -1, const_i64=7)]
    plan = JoinPlan(jt, ltypes, rtypes, [1], [0], build_is_right=build_is_right, lused=[0, 1, 2], rused=[] if semi else [2, 0], other_cond=other)
    assert_rows_equal(run_oracle(plan, l, r), run_gpu(plan, l, r))


def test_gpu_other_condition_gate():
    # shapes whose OtherCondition the device does not evaluate are declined by the planner gate, never mis-evaluated
    from tidb_b200.plan import OtherCond
    lib = abi.load_lib()
    other = [OtherCond(abi.CMP_LT, 0, 0, 1, 1)]
    for jt, brt in ((abi.JOIN_LEFT_OUTER, False), (abi.JOIN_SEMI, False), (abi.JOIN_LEFT_OUTER_SEMI, True)):
        plan = JoinPlan(jt, [INT, INT], [INT, INT], [0], [0], build_is_right=brt, lused=[0, 1], rused=[] if jt >= abi.JOIN_SEMI else [1], other_cond=other)
        d, keep = plan.to_struct()
        assert lib.tg_join_supported(C.byref(d)) == abi.TG_ERR_UNSUPPORTED
    mixed = JoinPlan(abi.JOIN_INNER, [INT, DBL], [INT, INT], [0], [0], other_cond=[OtherCond(abi.CMP_LT, 0, 1, 1, 1)])   # double vs int
    d, keep = mixed.to_struct()
    assert lib.tg_join_supported(C.byref(d)) == abi.TG_ERR_UNSUPPORTED


@pytest.mark.parametrize("jt,build_is_right", [(abi.JOIN_INNER, True), (abi.JOIN_INNER, False), (abi.JOIN_LEFT_OUTER, True),
                                               (abi.JOIN_RIGHT_OUTER, False), (abi.JOIN_SEMI, True), (abi.JOIN_ANTI_SEMI, True)])
@pytest.mark.parametrize("nkeys,unsigned_second,nulls", [(2, False, 0.0), (3, False, 0.08), (2, True, 0.08), (4, False, 0.05)])
def test_gpu_multi_column_join_keys(jt, build_is_right, nkeys, unsigned_second, nulls):
    # several equal conditions (FixedSerializedKey mode, join_table_meta.go:174-178, codec.go:822): the device joins on a
    # synthetic 64-bit candidate key (k_composite_key) and re-checks every key column on each candidate pair; key values come
    # from a small range so pairs that agree on some but not all key columns are common, NULL in any key column = no key,
    # signed vs unsigned key columns compare by value
    from test_oracle_join import make_multikey_case
    rng = np.random.default_rng(5100 + jt * 13 + nkeys + int(build_is_right))
    if nkeys == 4:
        INTU = FieldType(abi.TYPE_LONGLONG, 0)
        def side(rows):
            return [Column(rng.integers(-3, 3, rows).astype(np.int64), rng.random(rows) < nulls) for _ in range(4)]
        ltypes = rtypes = [INTU] * 4
        l, r = Chunk(side(5000)).split(1024), Chunk(side(4000)).split(700)
        lk = rk = [0, 1, 2, 3]
    else:
        ltypes, rtypes, l, r = make_multikey_case(rng, 4000, 6000, nulls, nkeys, unsigned_second=unsigned_second)
        lk, rk = list(range(1, 1 + nkeys)), list(range(nkeys))
    semi = jt >= abi.JOIN_SEMI
    plan = JoinPlan(jt, ltypes, rtypes, lk, rk, build_is_right=build_is_right, lused=[0, 1, 2, 3], rused=[] if semi else [3, 0, 1])
    want = run_oracle(plan, l, r)
    assert len(want) > 0 or jt == abi.JOIN_ANTI_SEMI
    assert_rows_equal(want, run_gpu(plan, l, r))


def test_gpu_multi_column_join_keys_with_other_condition_and_filters():
    # the residual key equalities and the user's OtherCondition share one item list; build / probe filters still apply first
    from test_oracle_join import make_multikey_case
    from tidb_b200.plan import OtherCond
    rng = np.random.default_rng(6200)
    ltypes, rtypes, l, r = make_multikey_case(rng, 5000, 8000, 0.05, 2)
    other = [OtherCond(abi.CMP_LT, 0, 0, 1, 3), OtherCond(abi.CMP_NE, 1, 2, -1, -1, const_i64=0)]
    for jt in (abi.JOIN_INNER, abi.JOIN_LEFT_OUTER):
        plan = JoinPlan(jt, ltypes, rtypes, [1, 2], [0, 1], build_is_right=True, lused=[0, 1, 2, 3], rused=[3, 0, 1], other_cond=other,
                        probe_filter=[FilterItem(abi.CMP_GT, 3, const_i64=-(1 << 39))],
                        build_filter=[] if jt == abi.JOIN_LEFT_OUTER else [FilterItem(abi.CMP_LT, 2, const_i64=1 << 39)])
        want = run_oracle(plan, l, r)
        assert len(want) > 0
        assert_rows_equal(want, run_gpu(plan, l, r))


def test_gpu_multi_column_join_keys_large_device_batches():
    # 3 M probe rows against 300 K build rows on (a, b): crosses the general path's sub-batches only at 16 M rows, so this
    # checks the bulk behaviour (hash collisions between distinct key tuples would show up as wrong row counts)
    rng = np.random.default_rng(6300)
    nb, npr = 300_000, 3_000_000
    a, b = rng.integers(0, 1000, nb).astype(np.int64), rng.integers(0, 1000, nb).astype(np.int64)
    pay = np.arange(nb, dtype=np.int64)
    pa, pb = rng.integers(0, 1000, npr).astype(np.int64), rng.integers(0, 1000, npr).astype(np.int64)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN, INT_NN], [0, 1], [0, 1], build_is_right=True, lused=[0, 1], rused=[2])
    got = run_gpu(plan, [Chunk([Column(pa), Column(pb)])], [Chunk([Column(a), Column(b), Column(pay)])], required_rows=1 << 20)
    # expected count by value: pairs per (a, b) tuple
    key_b = a * 1000 + b
    key_p = pa * 1000 + pb
    cnt_b = np.bincount(key_b, minlength=1_000_000)
    assert len(got) == int(cnt_b[key_p].sum())
    g = np.array(got, dtype=np.int64)
    assert np.array_equal(g[:, 0], a[g[:, 2]]) and np.array_equal(g[:, 1], b[g[:, 2]])   # every output row joins equal tuples


@pytest.mark.parametrize("jt,build_is_right", [(abi.JOIN_INNER, True), (abi.JOIN_INNER, False), (abi.JOIN_LEFT_OUTER, True),
                                               (abi.JOIN_LEFT_OUTER, False), (abi.JOIN_SEMI, True), (abi.JOIN_ANTI_SEMI, False)])
def test_gpu_time_join_keys(jt, build_is_right):
    # DATE / DATETIME / TIMESTAMP keys (getKeyProp join_table_meta.go:154, codec.go:697-707): compared by calendar fields, the
    # type / fsp bits of the CoreTime word ignored — a DATE joins the DATETIME at midnight of the same day
    from test_oracle_join import make_time_case
    rng = np.random.default_rng(7400 + jt)
    ltypes, rtypes, l, r = make_time_case(rng, 3000, 5000, 0.07)
    semi = jt >= abi.JOIN_SEMI
    plan = JoinPlan(jt, ltypes, rtypes, [1], [0], build_is_right=build_is_right, lused=[0, 1, 2], rused=[] if semi else [1, 0])
    want = run_oracle(plan, l, r)
    assert len(want) > 0
    assert_rows_equal(want, run_gpu(plan, l, r))


def test_gpu_time_join_keys_unique_build_and_gate():
    # unique DATE build keys: the single-pass / U1 paths read the key through load_key(KEY_TIME) as well; the build key column is
    # an output column, so it must come back with its own type bits, not the masked compare word
    from test_oracle_join import DATE_TT, DATETIME0_TT, DATETIME6_TT, core_time
    days = [(2020 + i // 336, 1 + (i // 28) % 12, 1 + i % 28) for i in range(2000)]
    bkey = np.array([core_time(y, m, d, fsp_tt=DATE_TT) for (y, m, d) in days], dtype=np.int64)
    rng = np.random.default_rng(7500)
    pick = rng.integers(0, 2000, 9000)
    pkey = np.array([core_time(*days[i], fsp_tt=DATETIME6_TT) if rng.random() < 0.6 else core_time(*days[i], 12, 30, 0, 0, DATETIME6_TT) for i in pick], dtype=np.int64)
    DT, D = FieldType(abi.TYPE_DATETIME, abi.FLAG_NOT_NULL), FieldType(abi.TYPE_DATE, abi.FLAG_NOT_NULL)
    left = [Chunk([Column(pkey), Column(np.arange(9000, dtype=np.int64))])]
    right = [Chunk([Column(bkey), Column(np.arange(2000, dtype=np.int64) * 3)])]
    for rused in ([1], [0, 1]):
        plan = JoinPlan(abi.JOIN_INNER, [DT, INT_NN], [D, INT_NN], [0], [0], build_is_right=True, lused=[0, 1], rused=rused)
        want = run_oracle(plan, left, right)
        assert 4000 < len(want) < 7000
        assert_rows_equal(want, run_gpu(plan, left, right))
    lib = abi.load_lib()
    mixed = JoinPlan(abi.JOIN_INNER, [DT], [INT_NN], [0], [0])     # date-time vs integer key: the planner casts first
    d, keep = mixed.to_struct()
    assert lib.tg_join_supported(C.byref(d)) == abi.TG_ERR_UNSUPPORTED


@pytest.mark.parametrize("build_is_right", [True, False])
@pytest.mark.parametrize("uq", ["1", "0"])
def test_gpu_unique_key_single_pass_probe(build_is_right, uq, monkeypatch):
    # k_probe_inner_uq: inner join, unique build keys, two NOT NULL build payload columns (row store), probe filters, a probe
    # key column with NULLs that is not output, the sentinel-valued key; TG_PROBE_UQ=0 sends the same plan down the general
    # count -> scan -> write path, both against the oracle, and tg_join_stats.paths shows which path ran
    monkeypatch.setenv("TG_PROBE_UQ", uq)
    rng = np.random.default_rng(77 + int(build_is_right))
    nb, npr = 40_000, 300_000
    bk = rng.permutation(nb * 3)[:nb].astype(np.int64) * 2654435761 - (1 << 41)
    bk[3] = -(1 << 63)
    build = Chunk([Column(bk), Column(np.arange(nb, dtype=np.int64) * 3), Column(rng.integers(0, 9, nb).astype(np.int64))])
    pick = rng.integers(0, nb * 2, npr)
    pk = np.where(pick < nb, bk[np.minimum(pick, nb - 1)], pick.astype(np.int64) * 11 + 5)
    pkn = rng.random(npr) < 0.05
    f = rng.integers(0, 100, npr).astype(np.int64)
    probe = Chunk([Column(np.arange(npr, dtype=np.int64)), Column(pk, pkn), Column(f), Column(rng.random(npr))])
    ptypes, btypes = [INT_NN, INT, INT_NN, FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)], [INT_NN, INT_NN, INT_NN]
    pf = [FilterItem(abi.CMP_LT, 2, const_i64=60), FilterItem(abi.CMP_GT, 3, is_real=True, const_f64=0.25)]
    if build_is_right:
        plan = JoinPlan(abi.JOIN_INNER, ptypes, btypes, [1], [0], build_is_right=True, lused=[0, 3], rused=[1, 2, 0], probe_filter=pf)
        l, r = probe.split(1 << 15), build.split(1 << 13)
    else:
        plan = JoinPlan(abi.JOIN_INNER, btypes, ptypes, [0], [1], build_is_right=False, lused=[2, 1], rused=[0, 2], probe_filter=pf)
        l, r = build.split(1 << 13), probe.split(1 << 15)
    got, st = run_gpu_stats(plan, l, r, required_rows=1 << 16)
    assert_rows_equal(run_oracle(plan, l, r), got)
    ran, skipped = (abi.JOIN_PATH_PROBE_UQ, abi.JOIN_PATH_PROBE_GENERAL) if uq == "1" else (abi.JOIN_PATH_PROBE_GENERAL, abi.JOIN_PATH_PROBE_UQ)
    assert st.paths & ran and not st.paths & skipped, hex(st.paths)


@pytest.mark.parametrize("required_rows", [1, 3, 13])
def test_next_serves_any_required_rows_with_null_bitmaps(required_rows):
    # exec.Executor: Next fills at most RequiredRows rows and RequiredRows may be 1 (LIMIT 1, MaxOneRow): a left outer join whose
    # output carries NULL bitmaps must be drainable one row at a time (the library re-aligns its bit-packed bitmaps on the host)
    rng = np.random.default_rng(5 + required_rows)
    ltypes, rtypes, l, r = make_case(rng, 120, 150, 0.2, True, False)
    plan = JoinPlan(abi.JOIN_LEFT_OUTER, ltypes, rtypes, [1], [0], build_is_right=True, lused=[0, 1, 2], rused=[2, 0])
    e = HashJoinExec(plan, MockDataSource(plan.left_types, l), MockDataSource(plan.right_types, r))
    chunks = drain(e, required_rows)
    assert all(0 < c.num_rows() <= required_rows for c in chunks)
    rows = []
    for c in chunks:
        rows.extend(columns_to_rows([(col_.data, col_.nulls()) for col_ in c.columns]))
    assert_rows_equal(run_oracle(plan, l, r), rows)


def test_gpu_double_keys_and_mixed_sign():
    rng = np.random.default_rng(5)
    ltypes, rtypes, l, r = make_case(rng, 1500, 2000, 0.1, True, False, key_dtype=np.float64)
    l[0].columns[1].data[0] = -0.0
    r[0].columns[0].data[0] = 0.0
    l[0].columns[1] = Column(l[0].columns[1].data, None)
    r[0].columns[0] = Column(r[0].columns[0].data, None)
    plan = JoinPlan(abi.JOIN_INNER, ltypes, rtypes, [1], [0])
    got = run_gpu(plan, l, r)
    assert_rows_equal(run_oracle(plan, l, r), got)
    assert any(row[1] == 0 for row in got)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN], [UINT_NN], [0], [0])
    assert sorted(run_gpu(plan, [Chunk([col([-1, 5, 7])])], [Chunk([col([-1, 5, 9])])])) == [(5, 5)]
    # the int64 value equal to the table's empty sentinel is a legal key
    mn = -(1 << 63)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    lch = [Chunk([col([mn, 1, mn, 3]), col([10, 11, 12, 13])])]
    rch = [Chunk([col([mn, 3, 4]), col([100, 300, 400])])]
    assert_rows_equal(run_oracle(plan, lch, rch), run_gpu(plan, lch, rch))
    rch = [Chunk([col([mn, 3, mn]), col([100, 300, 500])])]   # duplicates of the sentinel key (mode G)
    assert_rows_equal(run_oracle(plan, lch, rch), run_gpu(plan, lch, rch))


def test_gpu_empty_sides():
    e = [Chunk([Column(np.zeros(0, dtype=np.int64))])]
    f = [Chunk([col([1, 2, 3])])]
    for jt in (abi.JOIN_INNER, abi.JOIN_LEFT_OUTER, abi.JOIN_SEMI, abi.JOIN_ANTI_SEMI):
        semi = jt >= abi.JOIN_SEMI
        plan = JoinPlan(jt, [INT], [INT], [0], [0], rused=[] if semi else None)
        assert_rows_equal(run_oracle(plan, f, e), run_gpu(plan, f, []))
        assert_rows_equal(run_oracle(plan, e, f), run_gpu(plan, [], f))


def test_gpu_heavy_duplicate_skew():
    # all build rows share ONE key: the count-then-place build is O(n) (the reference chains rows)
    nb, npr = 200_000, 50
    b = [Chunk([Column(np.full(nb, 7, dtype=np.int64)), Column(np.arange(nb, dtype=np.int64))])]
    p = [Chunk([Column(np.array([7] * 3 + [8] * (npr - 3), dtype=np.int64)), Column(np.arange(npr, dtype=np.int64))])]
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    e = HashJoinExec(plan, MockDataSource(plan.left_types, p), MockDataSource(plan.right_types, b))
    chunks = drain(e, 1 << 20)
    total = sum(c.num_rows() for c in chunks)
    assert total == 3 * nb
    pay = np.concatenate([c.columns[3].data for c in chunks])
    assert np.array_equal(np.sort(pay), np.sort(np.tile(np.arange(nb), 3)))


def _config1(nb=100_000, npr=1_000_000):
    # BASELINE.md config 1: build k = perm(0..nb-1), v = k*7; probe k = uniform[0, nb), v = rowid
    rng = np.random.default_rng(42)
    bk = rng.permutation(nb).astype(np.int64)
    build = Chunk([Column(bk), Column(bk * 7)])
    rng = np.random.default_rng(43)
    pk = rng.integers(0, nb, npr).astype(np.int64)
    probe = Chunk([Column(pk), Column(np.arange(npr, dtype=np.int64))])
    return build, probe


def test_config1_plumbing_1024_row_chunks():
    # 1M ⋈ 100K int64 through Open/Next/Close with tidb_max_chunk_size = 1024 on both sides
    build, probe = _config1()
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    e = HashJoinExec(plan, MockDataSource(plan.left_types, probe.split(1024)), MockDataSource(plan.right_types, build.split(1024)))
    chunks = drain(e, 1024)
    assert all(c.num_rows() <= 1024 for c in chunks)
    total = sum(c.num_rows() for c in chunks)
    assert total == 1_000_000   # bit-exact output row count
    got = [np.concatenate([c.columns[i].data for c in chunks]) for i in range(4)]
    # every output row is (k, rowid, k, 7k) and every probe row appears exactly once
    assert np.array_equal(got[0], got[2]) and np.array_equal(got[3], got[0] * 7)
    assert np.array_equal(np.sort(got[1]), np.arange(1_000_000))
    assert np.array_equal(got[0], probe.columns[0].data[got[1]])
    # and the full multiset equals the oracle's (sorted, column-wise, bit-exact)
    n, ocols = O.OracleJoin(plan, 8).run(build.split(1024), probe.split(1024))
    assert n == total
    assert np.array_equal(columns_sorted(ocols), columns_sorted([(g, np.zeros(len(g), dtype=bool)) for g in got]))


def test_large_direct_push_and_big_next():
    # chunks ≥ 128K rows take the direct H2D path; Next with a large RequiredRows copies D2H directly
    build, probe = _config1(200_000, 2_000_000)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    e = HashJoinExec(plan, MockDataSource(plan.left_types, probe.split(1 << 19)), MockDataSource(plan.right_types, [build]))
    e.open()
    chunks = []
    while True:
        c = e.next(1 << 20)
        if c.num_rows() == 0:
            break
        chunks.append(c)
    st = e.stats()
    e.close()
    assert sum(c.num_rows() for c in chunks) == 2_000_000
    assert st.table_mode == 1 and st.max_dup == 1 and st.distinct_keys == 200_000   # unique-inline table
    got = [np.concatenate([c.columns[i].data for c in chunks]) for i in range(4)]
    assert np.array_equal(got[3], got[0] * 7) and np.array_equal(np.sort(got[1]), np.arange(2_000_000))


def test_partial_match_and_stats():
    # 50 % match variant of config 2's shape (probe keys uniform over 2× the build key range)
    rng = np.random.default_rng(1)
    nb, npr = 50_000, 400_000
    bk = (rng.permutation(nb).astype(np.int64) * 2654435761) % (1 << 40)
    build = Chunk([Column(bk), Column(np.arange(nb, dtype=np.int64))])
    pick = rng.integers(0, 2 * nb, npr)
    pk = np.where(pick < nb, bk[np.minimum(pick, nb - 1)], -pick.astype(np.int64) - 1)
    probe = Chunk([Column(pk), Column(np.arange(npr, dtype=np.int64))])
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    e = HashJoinExec(plan, MockDataSource(plan.left_types, [probe]), MockDataSource(plan.right_types, [build]))
    chunks = drain(e, 1 << 20)
    total = sum(c.num_rows() for c in chunks)
    assert total == int((pick < nb).sum())
    n, ocols = O.OracleJoin(plan, 8).run([build], probe.split(1 << 16))
    got = [np.concatenate([c.columns[i].data for c in chunks]) for i in range(4)]
    assert np.array_equal(columns_sorted(ocols), columns_sorted([(g, np.zeros(len(g), dtype=bool)) for g in got]))


def _fused_variant_paths(env):
    """(bits that must be set, bits that must be clear) in tg_join_stats.paths for a test_fused_probe_variants_forced env"""
    J = abi
    seg, bulk, other, direct = J.JOIN_PATH_PROBE_SEG, J.JOIN_PATH_SCATTER_BULK, J.JOIN_PATH_SCATTER, J.JOIN_PATH_PROBE_DIRECT
    never = J.JOIN_PATH_PROBE_UQ | J.JOIN_PATH_PROBE_GENERAL | 1 << 4   # bit 4 is unassigned
    if env.get("TG_PROBE_PARTITION", "1") == "0":
        return direct, never | seg | bulk | other
    return direct | bulk | seg, never | other   # count-free pass: bulk scatter, segment probe, gated fallback + tail


@pytest.mark.parametrize("env", [dict(TG_PROBE_PARTITION="1", TG_PROBE_PARTS=p) for p in ("2", "4", "5", "6", "7", "9", "16")]
                         + [dict(TG_PROBE_PARTITION="0")])
def test_fused_probe_variants_forced(env, monkeypatch):
    # the fused fast path with the L2 partition pass at several slice counts, and without the pass, must give the same
    # multiset; odd sizes exercise the tail tiles; PART_MIN_MB=0 forces the partition pass on a small table
    monkeypatch.delenv("TG_PROBE_UQ", raising=False)
    for k, v in dict(env, TG_PROBE_PART_MIN_MB="0", TG_PROBE_PART_MIN_ROWS="0").items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(17)
    nb, npr = 300_001, 2_500_003
    bk = rng.permutation(nb).astype(np.int64) * 2654435761 - (1 << 40)
    bk[5] = -(1 << 63)                       # the sentinel-valued key
    build = Chunk([Column(bk), Column(np.arange(nb, dtype=np.int64) * 3)])
    pick = rng.integers(0, int(nb * 1.25), npr)
    pk = np.where(pick < nb, bk[np.minimum(pick, nb - 1)], pick.astype(np.int64) * 7 + 1)   # ~80 % match
    probe = Chunk([Column(pk), Column(np.arange(npr, dtype=np.int64))])
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    e = HashJoinExec(plan, MockDataSource(plan.left_types, [probe]), MockDataSource(plan.right_types, [build]))
    e.open()
    chunks = []
    while True:
        c = e.next(1 << 22)
        if c.num_rows() == 0:
            break
        chunks.append(c)
    paths = e.stats().paths
    e.close()
    # the kernel families this environment selects ran, and no other
    want, dont = _fused_variant_paths(env)
    assert paths & want == want and paths & dont == 0, (hex(paths), hex(want), hex(dont))
    got = [np.concatenate([c.columns[i].data for c in chunks]) for i in range(4)]
    order = np.argsort(bk); sb = bk[order]
    pos = np.searchsorted(sb, pk); pos[pos >= nb] = nb - 1
    hit = sb[pos] == pk
    assert len(got[0]) == int(hit.sum())
    assert np.array_equal(np.sort(got[1]), np.nonzero(hit)[0])                       # each matching probe row exactly once
    assert np.array_equal(got[0], pk[got[1]]) and np.array_equal(got[2], got[0])     # keys travel with their row
    exp_pay = (order[pos] * 3)[got[1]]
    assert np.array_equal(got[3], exp_pay)                                           # and with the right build payload


@pytest.mark.parametrize("lused,rused", [([0, 1, 2, 3, 4], [0, 1]),   # four probe payload columns
                                         ([0, 1, 1], [1]),             # one probe column output twice
                                         ([0, 0, 1], [0, 1])])         # three outputs carry the join key
def test_unique_key_shapes_the_warp_kernels_do_not_cover(lused, rused):
    # a U1 table (unique keys, one 8-byte payload) and an output shape the fused warp kernels are not instantiated for:
    # the single-pass unique-key kernel takes the batch
    rng = np.random.default_rng(31)
    nb, npr = 60_000, 400_001
    bk = rng.permutation(nb).astype(np.int64) * 2654435761 - (1 << 40)
    bv = np.arange(nb, dtype=np.int64) * 3 + 1
    pk = np.where(rng.random(npr) < 0.7, bk[rng.integers(0, nb, npr)], rng.integers(1 << 50, 1 << 51, npr))
    pcols = [pk] + [np.arange(npr, dtype=np.int64) * m + a for m, a in ((1, 0), (5, 2), (-7, 1), (11, -3))]
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN] * 5, [INT_NN, INT_NN], [0], [0], lused=lused, rused=rused)
    e = HashJoinExec(plan, MockDataSource(plan.left_types, [Chunk([Column(c) for c in pcols])]),
                     MockDataSource(plan.right_types, [Chunk([Column(bk), Column(bv)])]))
    e.open()
    chunks = []
    while True:
        c = e.next(1 << 20)
        if c.num_rows() == 0:
            break
        chunks.append(c)
    st = e.stats()
    e.close()
    assert st.table_mode == 1
    assert st.paths & abi.JOIN_PATH_PROBE_UQ, hex(st.paths)
    assert not st.paths & (abi.JOIN_PATH_PROBE_DIRECT | abi.JOIN_PATH_PROBE_SEG | abi.JOIN_PATH_PROBE_GENERAL | 1 << 4), hex(st.paths)
    got = [np.concatenate([c.columns[i].data for c in chunks]) for i in range(len(lused) + len(rused))]
    order = np.argsort(bk)
    pos = np.minimum(np.searchsorted(bk[order], pk), nb - 1)
    rows = np.nonzero(bk[order][pos] == pk)[0]                     # matching probe rows, ascending
    want = [pcols[c][rows] for c in lused] + [(bk, bv)[c][order[pos[rows]]] for c in rused]
    by_row = np.argsort(got[lused.index(1)])                       # probe column 1 is the probe row index
    for g, w in zip(got, want):
        assert np.array_equal(g[by_row], w)


def test_partitioned_probe_overflow_falls_back(monkeypatch):
    # count-free L2 partitioning gives every segment a fixed capacity; a skewed probe side (70 % of the rows carry ONE key)
    # overflows its segment, the partitioned probe launch exits on the device-side flag and the gated direct launch
    # produces the result instead — same multiset either way
    for k, v in dict(TG_PROBE_PARTITION="1", TG_PROBE_PARTS="8", TG_PROBE_PART_MIN_MB="0", TG_PROBE_PART_MIN_ROWS="0").items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(23)
    nb, npr = 200_000, 2_000_000
    bk = rng.permutation(nb).astype(np.int64) * 2654435761 + 11
    build = Chunk([Column(bk), Column(np.arange(nb, dtype=np.int64) + 5)])
    pk = bk[rng.integers(0, nb, npr)]
    pk[rng.random(npr) < 0.7] = bk[12345]
    probe = Chunk([Column(pk), Column(np.arange(npr, dtype=np.int64))])
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    e = HashJoinExec(plan, MockDataSource(plan.left_types, [probe]), MockDataSource(plan.right_types, [build]))
    chunks = drain(e, 1 << 22)
    got = [np.concatenate([c.columns[i].data for c in chunks]) for i in range(4)]
    assert len(got[0]) == npr
    assert np.array_equal(np.sort(got[1]), np.arange(npr))
    assert np.array_equal(got[0], pk[got[1]]) and np.array_equal(got[2], got[0])
    order = np.argsort(bk)
    assert np.array_equal(got[3], order[np.searchsorted(bk[order], got[0])] + 5)


def test_concurrent_push_and_next_wait_and_rewind():
    # one thread pushes probe chunks while another blocks in tg_join_next_wait (the reference's probe fetcher goroutine vs
    # the consumer of joinResultCh, hash_join_v2.go:840/:1176); then a second pass after tg_join_probe_rewind
    import threading
    from tidb_b200.chunk import MutChunk
    lib = abi.load_lib()
    build, probe = _config1(150_000, 3_000_000)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    desc, keep = plan.to_struct()
    h = C.c_void_p()
    abi.check(lib.tg_join_open(C.byref(desc), C.byref(h)))
    bs = build.to_struct()
    abi.check(lib.tg_join_build_push(h, C.byref(bs)))
    abi.check(lib.tg_join_build_finish(h))
    chunks = probe.split(1 << 18)
    for _pass in range(2):
        errs = []

        def pusher():
            try:
                for c in chunks:
                    cs = c.to_struct()
                    abi.check(lib.tg_join_probe_push(h, C.byref(cs)))
                abi.check(lib.tg_join_probe_finish(h))
            except Exception as e:   # noqa: BLE001
                errs.append(e)
                lib.tg_join_probe_finish(h)

        th = threading.Thread(target=pusher)
        th.start()
        out = MutChunk([8, 8, 8, 8], 1 << 18)
        rows, parts = 0, [[], [], [], []]
        n = C.c_int64(0)
        while True:
            abi.check(lib.tg_join_next_wait(h, C.byref(out.struct), C.c_int64(1 << 18), C.byref(n)))
            if n.value == 0:
                break
            rows += n.value
            for i, (v, _) in enumerate(out.columns(n.value)):
                parts[i].append(v)
        th.join()
        assert not errs, errs
        assert rows == 3_000_000
        got = [np.concatenate(p) for p in parts]
        assert np.array_equal(np.sort(got[1]), np.arange(3_000_000)) and np.array_equal(got[3], got[0] * 7)
        abi.check(lib.tg_join_probe_rewind(h))
    lib.tg_join_close(h)


def test_close_during_next_wait_and_double_close():
    # exec.Executor: "Close may be called ... with Next() at the same time" (executor.go:65).  A consumer parked in
    # tg_join_next_wait must come back with TG_ERR_CANCELLED when another thread closes the handle; a second close and any
    # call made with the stale handle afterwards must be harmless (the shell outlives the close, csrc/join.cu).
    import threading
    import time
    from tidb_b200.chunk import MutChunk
    lib = abi.load_lib()
    build, probe = _config1(50_000, 200_000)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    for _round in range(3):
        desc, keep = plan.to_struct()
        h = C.c_void_p()
        abi.check(lib.tg_join_open(C.byref(desc), C.byref(h)))
        bs = build.to_struct()
        abi.check(lib.tg_join_build_push(h, C.byref(bs)))
        abi.check(lib.tg_join_build_finish(h))
        rcs = []

        def consumer():
            out = MutChunk([8, 8, 8, 8], 1 << 16)
            n = C.c_int64(0)
            while True:   # nothing was pushed and probe_finish is never called: parks on the result queue
                rc = lib.tg_join_next_wait(h, C.byref(out.struct), C.c_int64(1 << 16), C.byref(n))
                if rc != abi.TG_OK or n.value == 0:
                    rcs.append(rc)
                    return

        th = threading.Thread(target=consumer)
        th.start()
        time.sleep(0.05 * (_round + 1))
        assert lib.tg_join_close(h) == abi.TG_OK
        th.join(timeout=10)
        assert not th.is_alive(), "tg_join_next_wait did not return after tg_join_close"
        assert rcs == [abi.TG_ERR_CANCELLED]
        assert lib.tg_join_close(h) == abi.TG_OK                      # idempotent
        ps = probe.to_struct()
        assert lib.tg_join_probe_push(h, C.byref(ps)) == abi.TG_ERR_CANCELLED
        st = abi.TgJoinStats()
        assert lib.tg_join_get_stats(h, C.byref(st)) == abi.TG_ERR_CANCELLED


def test_close_while_pusher_is_probing():
    # close from a second thread while tg_join_probe_push is inside a probe: close waits for the push, later pushes see
    # TG_ERR_CANCELLED; the pusher never touches freed memory
    import threading
    lib = abi.load_lib()
    build, probe = _config1(100_000, 2_000_000)
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    desc, keep = plan.to_struct()
    h = C.c_void_p()
    abi.check(lib.tg_join_open(C.byref(desc), C.byref(h)))
    bs = build.to_struct()
    abi.check(lib.tg_join_build_push(h, C.byref(bs)))
    abi.check(lib.tg_join_build_finish(h))
    chunks = probe.split(1 << 16)
    seen = []

    def pusher():
        for c in chunks * 4:
            cs = c.to_struct()
            rc = lib.tg_join_probe_push(h, C.byref(cs))
            if rc != abi.TG_OK:
                seen.append(rc)
                return
        seen.append(abi.TG_OK)

    th = threading.Thread(target=pusher)
    th.start()
    import time
    time.sleep(0.02)
    assert lib.tg_join_close(h) == abi.TG_OK
    th.join(timeout=30)
    assert not th.is_alive()
    assert seen and seen[0] in (abi.TG_ERR_CANCELLED, abi.TG_OK)


def test_probe_device_segments_matches_dense_probe(monkeypatch):
    # the shape a count-free exchange delivers: `nseg` fixed-capacity regions, each valid for its first seg_cnt[s] rows.
    # The segmented device probe must return exactly what the dense device probe returns for the concatenated valid rows,
    # with and without the L2 partition pass.
    import torch
    from tidb_b200.device import DeviceJoin
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(5)
    nb, cap, nseg = 120_000, 300 * 1024, 5
    fill = [cap, 0, 123_457, cap - 1, 77]
    bk = rng.permutation(nb).astype(np.int64) * 2654435761 + 3
    pk_all, pv_all = [], []
    kcol = np.full(nseg * cap, -7, dtype=np.int64); vcol = np.full(nseg * cap, -9, dtype=np.int64)    # padding never matches
    for s_, f in enumerate(fill):
        k = np.where(rng.random(f) < 0.9, bk[rng.integers(0, nb, f)], rng.integers(1 << 50, 1 << 51, f))
        v = np.arange(f, dtype=np.int64) + s_ * 10_000_000
        kcol[s_ * cap:s_ * cap + f] = k; vcol[s_ * cap:s_ * cap + f] = v
        pk_all.append(k); pv_all.append(v)
    pk, pv = np.concatenate(pk_all), np.concatenate(pv_all)
    t = lambda a: torch.from_numpy(a).to(dev)
    for env in (dict(TG_PROBE_PARTITION="0"), dict(TG_PROBE_PARTITION="1", TG_PROBE_PARTS="6", TG_PROBE_PART_MIN_MB="0", TG_PROBE_PART_MIN_ROWS="0")):
        for k_, v_ in env.items():
            monkeypatch.setenv(k_, v_)
        plan = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0], device=0)
        j = DeviceJoin(plan)
        j.build([t(bk), t(np.arange(nb, dtype=np.int64) * 5)])
        rows_d, cols_d, _ = j.probe([t(pk), t(pv)])
        dense = [_dev_to_np(p, rows_d) for p in cols_d]
        rows_s, cols_s, _ = j.probe_segments([t(kcol), t(vcol)], t(np.array(fill, dtype=np.int64)), cap)
        seg = [_dev_to_np(p, rows_s) for p in cols_s]
        j.close()
        assert rows_s == rows_d == int(np.isin(pk, bk).sum())
        od, os_ = np.argsort(dense[1]), np.argsort(seg[1])
        for a, b in zip(dense, seg):
            assert np.array_equal(a[od], b[os_])


def _dev_to_np(ptr, n):
    import torch
    class _A:
        pass
    a = _A()
    a.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}
    return torch.as_tensor(a, device=torch.device("cuda", 0)).cpu().numpy()
