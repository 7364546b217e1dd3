"""tests/agg_reference.py pinned on the CPU: the reference's known answers, hand-worked identity-value and Final-mode
cases, the summation bound, and agreement with the C++ oracle on random data."""
import math

import numpy as np
import pytest

import agg_reference as R
import oracle_lib as O
from nested_loop import columns_to_rows
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.plan import AggFunc, AggPlan, FieldType

INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
UINT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1
FINAL = abi.AGGMODE_FINAL


def values(plan, chunks):
    """reference result as {key: tuple of expected values}"""
    return {k: tuple(e.value for e in es) for k, es in R.expected(plan, chunks).items()}


def test_aggfunc_kats():
    # aggfuncs/func_sum_test.go:39 (10.0 / NULL), func_count_test.go (5 / 0), func_avg_test.go:38 (2.0 / NULL)
    plan = AggPlan([DBL], [], [AggFunc(abi.AGG_SUM, 0, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 0, abi.TYPE_DOUBLE),
                               AggFunc(abi.AGG_AVG, 0, abi.TYPE_DOUBLE)])
    assert values(plan, [Chunk([Column(np.arange(5, dtype=np.float64))])]) == {(): (10.0, 5, 2.0)}
    assert values(plan, []) == {(): (None, 0, None)}
    # merge of partials 10 + 9 = 19, 5 + 3 = 8, 2.375 (func_sum_test.go:28, func_avg_test.go:25)
    a, b = Chunk([Column(np.arange(5, dtype=np.float64))]), Chunk([Column(np.arange(2, 5, dtype=np.float64))])
    assert values(plan, [a, b]) == {(): (19.0, 8, 2.375)}


def test_sql_aggregate_goldens():
    # tests/integrationtest/r/executor/aggregate.result:11-14, :18-21, :53-58
    t = Chunk([Column(np.array([1, 2], dtype=np.int64)), Column(np.array([0, 1], dtype=np.int64), np.array([True, False]))])
    plan = AggPlan([INT, INT], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_COUNT, 1)])
    assert values(plan, [t]) == {(1,): (1, 0), (2,): (2, 1)}
    plan = AggPlan([INT, DBL], [0], [AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE)])
    got = values(plan, [Chunk([Column(np.array([1, 2], dtype=np.int64)), Column(np.array([1.0 / 3.0, 1.0 / 6.0]))])])
    assert [repr(got[(k,)][0]) for k in (1, 2)] == ["0.3333333333333333", "0.16666666666666666"]
    empty = Chunk([Column(np.zeros(0, dtype=np.int64))])
    assert values(AggPlan([INT], [], [AggFunc(abi.AGG_COUNT, 0)]), [empty]) == {(): (0,)}
    assert values(AggPlan([INT], [0], [AggFunc(abi.AGG_COUNT, 0)]), [empty]) == {}


def test_identity_values_are_results():
    # groups made only of the values the device states start from (ordered domain: MIN ~0, MAX 0): the result is the value,
    # never NULL
    g = np.array([1, 1, 2, 2, 3, 4, 5, 6], dtype=np.int64)
    i = np.array([I64_MAX, I64_MAX, I64_MIN, I64_MIN, 0, 0, 0, 0], dtype=np.int64)
    u = np.array([0, 0, 0, 0, -1, 0, 0, 0], dtype=np.int64)          # -1 is 2**64 - 1 read as uint64
    d = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, -np.inf, -0.0])
    un = np.array([True] * 4 + [False] * 4)
    plan = AggPlan([INT_NN, INT, UINT, DBL], [0], [
        AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_MIN, 1), AggFunc(abi.AGG_MAX, 1), AggFunc(abi.AGG_MIN, 2), AggFunc(abi.AGG_MAX, 2),
        AggFunc(abi.AGG_MAX, 3, abi.TYPE_DOUBLE)])
    got = values(plan, [Chunk([Column(g), Column(i), Column(u, un), Column(d)])])
    assert got[(1,)][1:3] == (I64_MAX, I64_MAX)
    assert got[(2,)][1:3] == (I64_MIN, I64_MIN)
    assert got[(1,)][3:5] == (None, None)                 # all-NULL argument: NULL
    assert got[(3,)][3:5] == (U64_MAX, U64_MAX)
    assert got[(4,)][3:5] == (0, 0)
    assert got[(5,)][5] == -math.inf
    # a zero MIN/MAX(double) may come back with either sign; other results are bit-exact
    e = R.expected(plan, [Chunk([Column(g), Column(i), Column(u, un), Column(d)])])[(6,)][5]
    assert e.matches(0.0) and e.matches(-0.0) and not e.matches(5e-324)
    e = R.expected(plan, [Chunk([Column(g), Column(i), Column(u, un), Column(d)])])[(3,)][3]
    assert e.matches(U64_MAX) and not e.matches(U64_MAX - 1) and not e.matches(None)


def test_group_keys_null_sentinel_and_negative_zero():
    k = np.array([0.0, -0.0, 1.5, 2.0, 2.0])
    kn = np.array([False, False, False, True, True])
    g2 = np.array([I64_MIN, I64_MIN, 7, 7, 0], dtype=np.int64)
    g2n = np.array([False, False, False, False, True])
    plan = AggPlan([DBL, INT], [0, 1], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_FIRSTROW, 1), AggFunc(abi.AGG_COUNT, -1)])
    got = values(plan, [Chunk([Column(k, kn), Column(g2, g2n)])])
    assert got == {(0.0, I64_MIN): (0.0, I64_MIN, 2), (1.5, 7): (1.5, 7, 1), (None, 7): (None, 7, 1), (None, None): (None, None, 1)}
    # a result row is matched to its group through the FIRSTROW outputs; a -0.0 key reads as +0.0
    assert R.check(plan, [Chunk([Column(k, kn), Column(g2, g2n)])], [(-0.0, I64_MIN, 2), (1.5, 7, 1), (None, 7, 1), (None, None, 1)]) == 4
    with pytest.raises(AssertionError):
        R.check(plan, [Chunk([Column(k, kn), Column(g2, g2n)])], [(0.0, I64_MIN, 2), (1.5, 7, 1), (None, None, 2)])


def test_final_mode_hand_worked():
    # partial results of three workers for two groups: (group, partial count, partial sum); worker 3 saw no row of group 2
    g = np.array([1, 1, 1, 2, 2, 2], dtype=np.int64)
    cnt = np.array([2, 3, 0, 4, 0, 0], dtype=np.int64)
    sm = np.array([1.5, -0.25, 0.0, 8.0, 0.0, 0.0])
    smn = np.array([False, False, True, False, True, True])
    plan = AggPlan([INT_NN, INT_NN, DBL], [0], [
        AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_COUNT, 1, mode=FINAL), AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, mode=FINAL),
        AggFunc(abi.AGG_AVG, 1, abi.TYPE_LONGLONG, mode=FINAL, arg_col2=2)])
    got = values(plan, [Chunk([Column(g), Column(cnt), Column(sm, smn)])])
    assert got == {(1,): (1, 5, 1.25, 0.25), (2,): (2, 4, 8.0, 2.0)}
    # every partial sum NULL and every count 0: SUM and AVG are NULL, COUNT is 0
    got = values(plan, [Chunk([Column(g[4:]), Column(cnt[4:]), Column(sm[4:], smn[4:])])])
    assert got == {(2,): (2, 0, None, None)}


def test_sum_bound_catches_a_single_precision_accumulator():
    # x, -x pairs plus a small remainder: the exact sum is the remainder.  Any double summation order stays inside the
    # bound; a float32 accumulator (an error of about 2**-24 of the magnitudes) does not
    rng = np.random.default_rng(1)
    big = rng.random(5000) * 1e9
    xs = np.concatenate([big, -big, rng.random(10) * 1e-3])
    plan = AggPlan([DBL], [], [AggFunc(abi.AGG_SUM, 0, abi.TYPE_DOUBLE), AggFunc(abi.AGG_AVG, 0, abi.TYPE_DOUBLE)])
    e = R.expected(plan, [Chunk([Column(xs)])])[()]
    assert e[0].value == math.fsum(xs[-10:])
    for _ in range(5):
        rng.shuffle(xs)
        s = 0.0
        for v in xs.tolist():
            s += v
        assert e[0].matches(s) and e[1].matches(s / len(xs))
        s32 = np.float32(0)
        for v in xs.astype(np.float32):
            s32 = np.float32(s32 + v)
        assert not e[0].matches(float(s32))
    assert not e[0].matches(e[0].value + 2 * e[0].tol) and e[0].matches(e[0].value - e[0].tol)


def test_fused_argument_rounds_each_operation():
    a, b = np.array([0.1, 3.0, 1e300]), np.array([0.7, 0.3, 1e-300])
    plan = AggPlan([DBL, DBL], [], [AggFunc(abi.AGG_SUM, 0, abi.TYPE_DOUBLE, arg_col2=1, arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=1.0)])
    e = R.expected(plan, [Chunk([Column(a), Column(b)])])[()][0]
    assert e.value == math.fsum([0.1 * (1.0 - 0.7), 3.0 * (1.0 - 0.3), 1e300 * (1.0 - 1e-300)])


def test_sel_vector_is_applied():
    g = np.array([1, 2, 1, 2, 3], dtype=np.int64)
    x = np.array([1.0, 2.0, 4.0, 8.0, 16.0])
    plan = AggPlan([INT_NN, DBL], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE)])
    assert values(plan, [Chunk([Column(g), Column(x)], np.array([0, 3, 4]))]) == {(1,): (1, 1.0), (2,): (2, 8.0), (3,): (3, 16.0)}


@pytest.mark.parametrize("seed,nullg", [(1, True), (2, False)])
def test_reference_agrees_with_oracle(seed, nullg):
    # COUNT and MIN/MAX bit-exact, SUM / AVG within the bound, on mixed-sign data and full-range integers
    rng = np.random.default_rng(seed)
    n = 20_000
    g = rng.integers(-30, 30, n).astype(np.int64)
    g[:3] = I64_MIN
    gn = (rng.random(n) < 0.05) if nullg else None
    x = (rng.random(n) - 0.5) * 1e6
    xn = rng.random(n) < 0.1
    y = rng.integers(I64_MIN, I64_MAX, n, endpoint=True).astype(np.int64)
    d = rng.standard_normal(n) * 1e300
    chunks = Chunk([Column(g, gn), Column(x, xn), Column(y), Column(d)]).split(1000)
    plan = AggPlan([INT if nullg else INT_NN, DBL, INT_NN, FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)], [0], [
        AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE),
        AggFunc(abi.AGG_AVG, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_MIN, 2), AggFunc(abi.AGG_MAX, 2),
        AggFunc(abi.AGG_MIN, 3, abi.TYPE_DOUBLE), AggFunc(abi.AGG_MAX, 3, abi.TYPE_DOUBLE)])
    orc = O.OracleAgg(plan, 4, 3)
    nrows, cols = orc.run(chunks)
    orc.close()
    assert R.check(plan, chunks, columns_to_rows(cols)) == nrows
