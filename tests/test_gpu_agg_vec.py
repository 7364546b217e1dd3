"""Parity of the CUDA hash aggregation, VecEval kernels and repartition kernel against the oracle,
through the C-ABI.  COUNT / MIN / MAX / integer results bit-exact; SUM / AVG(double) within 1e-6
relative (BASELINE.json north_star; the reference's own summation order is nondeterministic)."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from nested_loop import columns_to_rows
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.executor import HashAggExec, MockDataSource, drain
from tidb_b200.plan import AggFunc, AggPlan, FieldType, FilterItem, filter_array

pytestmark = pytest.mark.gpu

INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
DBL_NN = FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)
REL = 1e-6


def run_gpu_agg(plan, chunks, required_rows=1024):
    e = HashAggExec(plan, MockDataSource(plan.col_types, chunks))
    out = drain(e, required_rows)
    rows = []
    for c in out:
        rows.extend(columns_to_rows([(col.data, col.nulls()) for col in c.columns]))
    return rows


def run_gpu_agg_stats(plan, chunks, required_rows=1024):
    """run_gpu_agg, plus the handle's tg_agg_stats read before close"""
    e = HashAggExec(plan, MockDataSource(plan.col_types, chunks))
    e.open()
    try:
        rows = []
        while True:
            c = e.next(required_rows)
            if c.num_rows() == 0:
                break
            rows.extend(columns_to_rows([(col.data, col.nulls()) for col in c.columns]))
        return rows, e.stats()
    finally:
        e.close()


def run_orc_agg(plan, chunks):
    a = O.OracleAgg(plan, 5, 5)
    n, cols = a.run(chunks)
    a.close()
    return columns_to_rows(cols) if n else []


def assert_agg_equal(exp, got, float_cols):
    assert len(exp) == len(got)
    key = lambda r: tuple((0, 0) if v is None else (1, v) for i, v in enumerate(r) if i not in float_cols)
    exp, got = sorted(exp, key=key), sorted(got, key=key)
    for e, g in zip(exp, got):
        for i, (a, b) in enumerate(zip(e, g)):
            if i in float_cols and a is not None and b is not None:
                assert b == pytest.approx(a, rel=REL), (e, g)
            else:
                assert a == b, (e, g)


def test_aggfunc_kats_on_gpu():
    # aggfuncs/func_sum_test.go:39 (10.0 / NULL), func_count_test.go (5 / 0), func_avg_test.go:38 (2.0 / NULL)
    plan = AggPlan([DBL], [], [AggFunc(abi.AGG_SUM, 0, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 0, abi.TYPE_DOUBLE),
                               AggFunc(abi.AGG_AVG, 0, abi.TYPE_DOUBLE)])
    assert run_gpu_agg(plan, [Chunk([Column(np.arange(5, dtype=np.float64))])]) == [(10.0, 5, 2.0)]
    assert run_gpu_agg(plan, []) == [(None, 0, None)]
    # merge of partials 10 + 9 = 19, 5 + 3 = 8, 2.375 (func_sum_test.go:28, func_avg_test.go:25)
    a = Chunk([Column(np.arange(5, dtype=np.float64))]); b = Chunk([Column(np.arange(2, 5, dtype=np.float64))])
    assert run_gpu_agg(plan, [a, b]) == [(19.0, 8, 2.375)]


def test_sql_aggregate_goldens_on_gpu():
    # tests/integrationtest/r/executor/aggregate.result:11-14, :18-21, :53-58
    t = Chunk([Column(np.array([1, 2], dtype=np.int64)), Column(np.array([0, 1], dtype=np.int64), np.array([True, False]))])
    plan = AggPlan([INT, INT], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_COUNT, 1)])
    assert sorted(run_gpu_agg(plan, [t])) == [(1, 0), (2, 1)]
    plan = AggPlan([INT, DBL], [0], [AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE)])
    got = sorted(run_gpu_agg(plan, [Chunk([Column(np.array([1, 2], dtype=np.int64)), Column(np.array([1.0 / 3.0, 1.0 / 6.0]))])]))
    assert [repr(r[0]) for r in got] == ["0.16666666666666666", "0.3333333333333333"]
    empty = Chunk([Column(np.zeros(0, dtype=np.int64))])
    assert run_gpu_agg(AggPlan([INT], [], [AggFunc(abi.AGG_COUNT, 0)]), [empty]) == [(0,)]
    assert run_gpu_agg(AggPlan([INT], [0], [AggFunc(abi.AGG_COUNT, 0)]), [empty]) == []
    # TestParallelHashAgg (aggregate_test.go:385): 20 groups × 20 rows of 1 → SUM 20 each
    g = np.tile(np.arange(20, dtype=np.int64), 20)
    chunks = Chunk([Column(g), Column(np.ones(400))]).split(32)
    plan = AggPlan([INT, DBL], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE)])
    assert sorted(run_gpu_agg(plan, chunks)) == [(i, 20.0) for i in range(20)]


@pytest.mark.parametrize("ngroups,nullg", [(40, True), (5000, False), (1, False)])
def test_agg_random_vs_oracle(ngroups, nullg):
    rng = np.random.default_rng(7 + ngroups)
    n = 60_000
    g = rng.integers(-ngroups // 2, ngroups // 2 + 1, n).astype(np.int64)
    g[0] = -(1 << 63)   # the sentinel-valued key is a legal group
    gn = (rng.random(n) < 0.05) if nullg else None
    x = rng.random(n) * 1e7
    xn = rng.random(n) < 0.1
    y = rng.integers(-1000, 1000, n).astype(np.int64)
    chunks = Chunk([Column(g, gn), Column(x, xn), Column(y)]).split(1024)
    plan = AggPlan([INT if nullg else INT_NN, DBL, INT_NN], [0], [
        AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE),
        AggFunc(abi.AGG_AVG, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_MIN, 2), AggFunc(abi.AGG_MAX, 2),
        AggFunc(abi.AGG_MIN, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_MAX, 1, abi.TYPE_DOUBLE)], expected_groups=16)   # tiny hint → table growth
    assert_agg_equal(run_orc_agg(plan, chunks), run_gpu_agg(plan, chunks), {1, 3})


def test_agg_no_group_by_and_double_key():
    rng = np.random.default_rng(3)
    n = 100_000
    x = rng.random(n) * 100; xn = rng.random(n) < 0.2
    y = rng.integers(-5, 5, n).astype(np.int64)
    chunks = Chunk([Column(x, xn), Column(y)]).split(4096)
    plan = AggPlan([DBL, INT_NN], [], [AggFunc(abi.AGG_SUM, 0, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 0, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, -1),
                                       AggFunc(abi.AGG_AVG, 0, abi.TYPE_DOUBLE), AggFunc(abi.AGG_MIN, 1), AggFunc(abi.AGG_MAX, 0, abi.TYPE_DOUBLE)])
    assert_agg_equal(run_orc_agg(plan, chunks), run_gpu_agg(plan, chunks), {0, 3})
    # double group key: -0.0 and +0.0 are one group (codec float.go:23)
    k = np.array([0.0, -0.0, 1.5, 1.5, np.nan, np.nan, -2.0])
    chunks = [Chunk([Column(k), Column(np.ones(7))])]
    plan = AggPlan([DBL_NN, DBL_NN], [0], [AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE)])
    assert sorted(run_gpu_agg(plan, chunks)) == sorted(run_orc_agg(plan, chunks)) == [(1, 1.0), (2, 2.0), (2, 2.0), (2, 2.0)]


def test_agg_config3_shape_reduced():
    # config 3 shape at 1/50 scale: SELECT g, SUM(x), COUNT(x) GROUP BY g; uniform g, x = uniform[0,1e7); 1 % NULL x
    rng = np.random.default_rng(44)
    n, G = 2_000_000, 20_000
    g = rng.integers(0, G, n).astype(np.int64)
    x = np.floor(rng.random(n) * 1e7)
    for xn in (None, rng.random(n) < 0.01):
        chunk = Chunk([Column(g), Column(x, xn)])
        plan = AggPlan([INT_NN, DBL if xn is not None else DBL_NN], [0],
                       [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE)],
                       expected_groups=G)
        e = HashAggExec(plan, MockDataSource(plan.col_types, chunk.split(1 << 18)))
        out = drain(e, 1 << 16)
        gk = np.concatenate([c.columns[0].data for c in out]); s = np.concatenate([c.columns[1].data for c in out])
        cnt = np.concatenate([c.columns[2].data for c in out])
        assert len(gk) == G and np.array_equal(np.sort(gk), np.arange(G))
        m = np.ones(n, dtype=bool) if xn is None else ~xn
        exp_cnt = np.bincount(g[m], minlength=G); exp_sum = np.bincount(g[m], weights=x[m], minlength=G)
        assert np.array_equal(cnt, exp_cnt[gk])           # COUNT bit-exact
        assert np.allclose(s, exp_sum[gk], rtol=REL, atol=0)


@pytest.mark.parametrize("hint,local_env", [(0, None), (300, None), (200_000, None), (0, "0"), (200_000, "2")])
def test_agg_two_level_paths_vs_oracle(hint, local_env, monkeypatch):
    # the round-2 two-level update (csrc/agg_update.cuh): CTA-local tables + global table, every combination of
    # hint / forced mode, on skewed keys (a few hot groups + a long tail), NULL groups, the sentinel-valued key, 1 % NULL x.
    # The CTA-local level takes at most 4 device states, so the aggregates are split over two plans; tg_agg_stats shows
    # which level ran
    monkeypatch.delenv("TG_AGG_LOCAL", raising=False)
    monkeypatch.delenv("TG_AGG_V1", raising=False)
    if local_env is not None:
        monkeypatch.setenv("TG_AGG_LOCAL", local_env)
    # the CTA-local level runs for hints up to 4096 groups (or no hint) unless TG_AGG_LOCAL=0; TG_AGG_LOCAL=2 forces it
    local = local_env == "2" or (local_env != "0" and hint <= 4096)
    rng = np.random.default_rng(11 + hint)
    n = 400_000
    hot = rng.integers(0, 8, n)
    tail = rng.integers(-60_000, 60_000, n)
    g = np.where(rng.random(n) < 0.5, hot, tail).astype(np.int64)
    g[:3] = -(1 << 63)
    gn = rng.random(n) < 0.02
    x = np.floor(rng.random(n) * 1e7); xn = rng.random(n) < 0.01
    y = rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)
    chunks = Chunk([Column(g, gn), Column(x, xn), Column(y)]).split(1 << 16)
    for funcs, float_cols in (([AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE),
                                AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_MAX, 2)], {1}),
                              ([AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_MIN, 1, abi.TYPE_DOUBLE)], set())):
        plan = AggPlan([INT, DBL, INT_NN], [0], funcs, expected_groups=hint)
        got, st = run_gpu_agg_stats(plan, chunks)
        assert_agg_equal(run_orc_agg(plan, chunks), got, float_cols)
        if local:
            assert st.paths & abi.AGG_PATH_V2_LOCAL and st.local_rows > 0, (hex(st.paths), st.local_rows)
        else:
            assert st.paths & abi.AGG_PATH_V2_GLOBAL and not st.paths & abi.AGG_PATH_V2_LOCAL and st.local_rows == 0, (hex(st.paths), st.local_rows)


@pytest.mark.parametrize("ncols,nullable", [(2, False), (3, True), (4, True)])
def test_agg_multi_column_group_by_vs_oracle(ncols, nullable):
    # GetGroupKey concatenates the encodings of every GROUP BY item (agg_util.go:106, codec.go:1761): groups differ when ANY
    # column differs, NULL is a value of its own in every column, -0.0 groups with +0.0.  Tag-claimed multi-word slots
    # (csrc/agg.cu k_agg_update_mk), tiny hint -> several table growths.
    rng = np.random.default_rng(100 + ncols)
    n = 300_000
    cols, types = [], []
    for c in range(ncols):
        if c == 1:
            v = rng.integers(-3, 4, n).astype(np.float64) * 0.5
            v[rng.random(n) < 0.1] = -0.0
            tp = FieldType(abi.TYPE_DOUBLE, 0 if nullable else abi.FLAG_NOT_NULL)
        else:
            v = rng.integers(0, 40 if c else 300, n).astype(np.int64)
            if c == 0:
                v[:5] = -(1 << 63)
            tp = FieldType(abi.TYPE_LONGLONG, 0 if nullable else abi.FLAG_NOT_NULL)
        nl = (rng.random(n) < 0.05) if nullable else None
        cols.append(Column(v, nl)); types.append(tp)
    x = np.floor(rng.random(n) * 1e6); xn = rng.random(n) < 0.02
    cols.append(Column(x, xn)); types.append(DBL)
    chunks = Chunk(cols).split(1 << 15)
    funcs = [AggFunc(abi.AGG_FIRSTROW, c, types[c].tp) for c in range(ncols)] + [
        AggFunc(abi.AGG_SUM, ncols, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, ncols, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, -1),
        AggFunc(abi.AGG_MAX, ncols, abi.TYPE_DOUBLE)]
    plan = AggPlan(types, list(range(ncols)), funcs, expected_groups=64)
    assert_agg_equal(run_orc_agg(plan, chunks), run_gpu_agg(plan, chunks), {ncols})


@pytest.mark.parametrize("group_cols", [[], [0], [0, 1]])
def test_agg_fused_argument_expression(group_cols):
    # SUM(l_extendedprice * (1 - l_discount)) with the projection fused into the update kernels (tg_agg_func.arg_expr): the
    # reference evaluates Args[0] per row (func_sum.go:90 through builtinArithmeticMinusRealSig / MultiplyRealSig): NULL when
    # an operand is NULL; ErrOverflow when a non-NULL row leaves the DOUBLE range
    rng = np.random.default_rng(21 + len(group_cols))
    n = 150_000
    g0 = rng.integers(0, 700, n).astype(np.int64); g1 = rng.integers(0, 3, n).astype(np.int64)
    price = np.floor(rng.random(n) * 1e7) / 100; pn = rng.random(n) < 0.03
    disc = np.floor(rng.random(n) * 11) / 100; dn = rng.random(n) < 0.03
    chunks = Chunk([Column(g0), Column(g1), Column(price, pn), Column(disc, dn)]).split(1 << 14)
    funcs = [AggFunc(abi.AGG_FIRSTROW, c) for c in group_cols] + [
        AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, arg_col2=3, arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=1.0),
        AggFunc(abi.AGG_AVG, 2, abi.TYPE_DOUBLE, arg_col2=3, arg_expr=abi.ARGEXPR_MUL), AggFunc(abi.AGG_COUNT, -1)]
    plan = AggPlan([INT_NN, INT_NN, DBL, DBL], group_cols, funcs, expected_groups=100)
    k = len(group_cols)
    assert_agg_equal(run_orc_agg(plan, chunks), run_gpu_agg(plan, chunks), {k, k + 1})
    # overflow: 1e308 * (3 - (-1e308))  ->  ErrOverflow on both sides
    big = [Chunk([Column(np.zeros(4, dtype=np.int64)), Column(np.zeros(4, dtype=np.int64)), Column(np.array([1.0, 1e308, 2.0, 3.0])), Column(np.array([0.5, -1e308, 0.1, 0.2]))])]
    oplan = AggPlan([INT_NN, INT_NN, DBL_NN, DBL_NN], group_cols, [AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, arg_col2=3, arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=3.0)])
    with pytest.raises(RuntimeError):
        run_orc_agg(oplan, big)
    with pytest.raises(abi.TgError) as ei:
        run_gpu_agg(oplan, big)
    assert ei.value.code == abi.TG_ERR_OVERFLOW


def test_agg_next_small_required_rows():
    # HashAggExec.Next with RequiredRows = 3 on a result that carries NULL bitmaps (SUM over all-NULL groups is NULL)
    rng = np.random.default_rng(8)
    n = 5000
    g = rng.integers(0, 37, n).astype(np.int64)
    x = rng.random(n); xn = (g % 5 == 0) | (rng.random(n) < 0.1)
    chunks = Chunk([Column(g), Column(x, xn)]).split(512)
    plan = AggPlan([INT_NN, DBL], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE)])
    assert_agg_equal(run_orc_agg(plan, chunks), run_gpu_agg(plan, chunks, required_rows=3), {1})


def test_agg_multi_push_same_table():
    # several device batches into one handle (fetchChildData loop, agg_hash_executor.go:449): later batches find the groups
    # of earlier ones; the table grows between batches
    rng = np.random.default_rng(5)
    parts = []
    for b in range(3):
        n = 5_000_000 if b == 1 else 70_000       # the middle batch is large enough to be flushed on its own (4M-row staging)
        g = rng.integers(0, 3000 * (b + 1), n).astype(np.int64)
        x = np.floor(rng.random(n) * 1000)
        parts.append(Chunk([Column(g), Column(x)]))
    chunks = [c for p_ in parts for c in p_.split(1 << 18)]
    plan = AggPlan([INT_NN, DBL_NN], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE)])
    out = drain(HashAggExec(plan, MockDataSource(plan.col_types, chunks)), 1 << 16)
    gk = np.concatenate([c.columns[0].data for c in out]); s_ = np.concatenate([c.columns[1].data for c in out]); cnt = np.concatenate([c.columns[2].data for c in out])
    gall = np.concatenate([p_.columns[0].data for p_ in parts]); xall = np.concatenate([p_.columns[1].data for p_ in parts])
    G = 9000
    assert np.array_equal(np.sort(gk), np.flatnonzero(np.bincount(gall, minlength=G)))
    assert np.array_equal(cnt, np.bincount(gall, minlength=G)[gk])
    assert np.allclose(s_, np.bincount(gall, weights=xall, minlength=G)[gk], rtol=REL, atol=0)


# ---- VecEval ----------------------------------------------------------------------------------------------
def _call_vec(fn, *args):
    return fn(*args)


def gpu_vec(kind, op, a: Column, b, bc, au=False, bu=False):
    lib = abi.load_lib()
    n = a.length
    res = np.zeros(n, dtype=np.float64 if kind == "arith_real" else np.int64)
    nulls = np.zeros((n + 7) // 8, dtype=np.uint8)
    sa = a.to_struct(); sb = b.to_struct() if b is not None else None
    pb = C.byref(sb) if sb is not None else None
    rp, np_ = res.ctypes.data_as(C.c_void_p), nulls.ctypes.data_as(C.c_void_p)
    if kind == "cmp_int":
        rc = lib.tg_vec_compare_int(0, 0, op, int(au), int(bu), C.byref(sa), pb, C.c_int64(bc), rp, np_, None)
    elif kind == "cmp_real":
        rc = lib.tg_vec_compare_real(0, 0, op, C.byref(sa), pb, C.c_double(bc), rp, np_, None)
    elif kind == "arith_int":
        rc = lib.tg_vec_arith_int(0, 0, op, int(au), int(bu), C.byref(sa), pb, C.c_int64(bc), rp, np_, None)
    else:
        rc = lib.tg_vec_arith_real(0, 0, op, C.byref(sa), pb, C.c_double(bc), rp, np_, None)
    return rc, res, np.unpackbits(nulls, bitorder="little")[:n] == 0


def test_vec_compare_vs_row_oracle():
    # testVectorizedBuiltinFunc (expression/bench_test.go:1562): random 1024-row chunk, vec vs row evaluator
    rng = np.random.default_rng(11)
    n = 1024 + 37
    a = Column(rng.integers(-50, 50, n).astype(np.int64), rng.random(n) < 0.1)
    b = Column(rng.integers(-50, 50, n).astype(np.int64), rng.random(n) < 0.1)
    fa = Column(np.where(rng.random(n) < 0.05, np.nan, rng.integers(-5, 5, n) / 2.0), rng.random(n) < 0.1)
    fb = Column(np.where(rng.random(n) < 0.05, np.nan, rng.integers(-5, 5, n) / 2.0))
    for op in range(6):
        for (au, bu) in ((False, False), (True, False), (False, True), (True, True)):
            rc, r, nl = gpu_vec("cmp_int", op, a, b, 0, au, bu); assert rc == 0
            er, enl = O.vec_compare_int(op, a, b, 0, au, bu)
            assert np.array_equal(nl, enl) and np.array_equal(r[~nl], er[~enl])
        rc, r, nl = gpu_vec("cmp_int", op, a, None, 3); assert rc == 0
        er, enl = O.vec_compare_int(op, a, None, 3)
        assert np.array_equal(nl, enl) and np.array_equal(r[~nl], er[~enl])
        rc, r, nl = gpu_vec("cmp_real", op, fa, fb, 0.0); assert rc == 0
        er, enl = O.vec_compare_real(op, fa, fb)
        assert np.array_equal(nl, enl) and np.array_equal(r[~nl], er[~enl])


def test_vec_arith_vs_row_oracle_and_overflow():
    rng = np.random.default_rng(12)
    n = 3000
    a = Column(rng.integers(-1 << 40, 1 << 40, n).astype(np.int64), rng.random(n) < 0.1)
    b = Column(rng.integers(-1 << 20, 1 << 20, n).astype(np.int64), rng.random(n) < 0.1)
    for op in (abi.ARITH_PLUS, abi.ARITH_MINUS, abi.ARITH_MUL):
        rc, r, nl = gpu_vec("arith_int", op, a, b, 0); erc, er, enl = O.vec_arith_int(op, a, b)
        assert rc == erc == 0 and np.array_equal(nl, enl) and np.array_equal(r[~nl], er[~enl])
    fa = Column(rng.random(n) * 1e6, rng.random(n) < 0.1); fb = Column(rng.random(n))
    for op in (abi.ARITH_PLUS, abi.ARITH_MINUS, abi.ARITH_MUL):
        rc, r, nl = gpu_vec("arith_real", op, fa, fb, 0.0); erc, er, enl = O.vec_arith_real(op, fa, fb)
        assert rc == erc == 0 and np.array_equal(nl, enl) and np.array_equal(r[~nl], er[~enl])   # IEEE: bit-exact
    mx, mn = (1 << 63) - 1, -(1 << 63)
    cases = [("arith_int", abi.ARITH_PLUS, [mx], 1, False, False), ("arith_int", abi.ARITH_PLUS, [-1], 1, True, True),
             ("arith_int", abi.ARITH_MINUS, [mn], 1, False, False), ("arith_int", abi.ARITH_MINUS, [0], 1, True, True),
             ("arith_int", abi.ARITH_MUL, [-1], mn, False, False), ("arith_int", abi.ARITH_MUL, [1 << 32], 1 << 31, False, False)]
    for kind, op, av, bc, au, bu in cases:
        col = Column(np.array(av, dtype=np.int64))
        rc, _, _ = gpu_vec(kind, op, col, None, bc, au, bu)
        erc, _, _ = O.vec_arith_int(op, col, None, bc, au, bu)
        assert rc == erc == abi.TG_ERR_OVERFLOW
        ncol = Column(np.array(av, dtype=np.int64), np.array([True]))   # NULL rows never raise
        rc, _, nl = gpu_vec(kind, op, ncol, None, bc, au, bu); assert rc == 0 and nl[0]
    rc, _, _ = gpu_vec("arith_real", abi.ARITH_PLUS, Column(np.array([1.7e308])), None, 1.7e308); assert rc == abi.TG_ERR_OVERFLOW
    rc, _, _ = gpu_vec("arith_real", abi.ARITH_PLUS, Column(np.array([np.nan])), None, 1.0); assert rc == abi.TG_ERR_OVERFLOW
    rc, r, _ = gpu_vec("arith_real", abi.ARITH_MUL, Column(np.array([np.nan])), None, 1.0); assert rc == 0 and np.isnan(r[0])


def test_vec_filter_vs_oracle():
    rng = np.random.default_rng(13)
    n = 5000
    a = Column(rng.integers(-10, 10, n).astype(np.int64), rng.random(n) < 0.1)
    b = Column(rng.random(n) * 10)
    c = Column(rng.integers(-10, 10, n).astype(np.int64))
    items = [FilterItem(abi.CMP_GT, 0, const_i64=-3), FilterItem(abi.CMP_LT, 1, is_real=True, const_f64=7.5), FilterItem(abi.CMP_NE, 0, rhs_col=2)]
    for sel in (None, np.sort(rng.choice(n, n // 2, replace=False)).astype(np.int64)):
        chk = Chunk([a, b, c], sel)
        exp, ecnt = O.vec_filter(chk, items)
        got = np.zeros(n, dtype=np.uint8); cnt = C.c_int64(0)
        cs = chk.to_struct(); fa = filter_array(items)
        abi.check(abi.load_lib().tg_vec_filter(0, 0, C.byref(cs), fa, len(items), got.ctypes.data_as(C.c_void_p), C.byref(cnt), None))
        assert np.array_equal(got.astype(bool), exp) and cnt.value == ecnt


# ---- repartition ---------------------------------------------------------------------------------------------
def test_partition_by_key_properties():
    import torch
    lib = abi.load_lib()
    rng = np.random.default_rng(21)
    n, P = 1_000_003, 8
    key = torch.from_numpy(rng.integers(-1 << 62, 1 << 62, n).astype(np.int64)).cuda()
    pay = torch.arange(n, dtype=torch.int64, device="cuda")
    dk = torch.empty_like(key); dp = torch.empty_like(pay)
    offs = torch.zeros(P + 1, dtype=torch.int64, device="cuda")
    src = (C.c_void_p * 2)(key.data_ptr(), pay.data_ptr()); dst = (C.c_void_p * 2)(dk.data_ptr(), dp.data_ptr())
    abi.check(lib.tg_partition_by_key(0, C.c_void_p(key.data_ptr()), None, C.c_int64(n), P, 2, src, dst, C.c_void_p(offs.data_ptr()), None))
    torch.cuda.synchronize()
    o = offs.cpu().numpy(); k = key.cpu().numpy(); outk = dk.cpu().numpy(); outp = dp.cpu().numpy()
    assert o[0] == 0 and o[-1] == n and np.all(np.diff(o) >= 0)
    exp_part = np.array([lib.tg_partition_of_key(int(v), P) for v in k[:2000]])
    assert np.array_equal(np.sort(outp), np.arange(n))            # a permutation: nothing lost or duplicated
    assert np.array_equal(outk, k[outp])                          # key and payload moved together
    part_of_out = np.searchsorted(o, np.arange(n), side="right") - 1
    idx = np.where(outp < 2000)[0]
    assert np.array_equal(part_of_out[idx], exp_part[outp[idx]])  # every row sits in its hash partition
    counts = torch.zeros(P, dtype=torch.int64, device="cuda")
    abi.check(lib.tg_partition_count(0, C.c_void_p(key.data_ptr()), C.c_int64(n), P, C.c_void_p(counts.data_ptr()), None))
    torch.cuda.synchronize()
    assert np.array_equal(counts.cpu().numpy(), np.diff(o))
