"""CPU checks of tests/agg_distinct_reference.py: the reference's integration answers for COUNT / SUM / AVG / MAX with
DISTINCT, and the Go map semantics of -0.0, +0.0 and NaN."""
import math

import numpy as np

import agg_distinct_reference as DR
import mydecimal as D
from tidb_b200 import abi
from tidb_b200.plan import AggFunc, AggPlan, FieldType

INT = FieldType(abi.TYPE_LONGLONG, 0)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
DEC = abi.TYPE_NEWDECIMAL

# tests/integrationtest/r/executor/aggregate.result of the reference: t1(a int, b int), grouped by a
T1 = [(1, 1), (2, 2), (3, 3), (1, 4), (1, 1), (3, 5), (2, 2), (3, 5), (3, 3)]


def t1_vals():
    a = np.array([r[0] for r in T1], dtype=np.int64)
    b = np.array([r[1] for r in T1], dtype=np.int64)
    z = np.zeros(len(T1), dtype=bool)
    return {0: (a, z), 1: (b, z)}


def test_integration_answers():
    plan = AggPlan([INT, INT], [0], [AggFunc(abi.AGG_FIRSTROW, 0),
                                     AggFunc(abi.AGG_AVG, 1, ret_type=DEC, ret_frac=4, distinct=True),
                                     AggFunc(abi.AGG_SUM, 1, ret_type=DEC, distinct=True),
                                     AggFunc(abi.AGG_COUNT, 1, distinct=True),
                                     AggFunc(abi.AGG_MAX, 1, distinct=True)])
    exp = DR.expected(plan, t1_vals())
    got = {k: (D.to_string(v[1]), D.to_string(v[2]), v[3], v[4]) for k, v in exp.items()}
    assert got == {(1,): ("2.5000", "5", 2, 4), (2,): ("2.0000", "2", 1, 2), (3,): ("4.0000", "8", 2, 5)}


def test_zero_and_nan_follow_go_maps():
    nan = float("nan")
    assert DR.distinct_values([0.0, -0.0, 1.0, 1.0], True) == [0.0, 1.0]
    xs = DR.distinct_values([nan, nan, 2.0, nan], True)
    assert len(xs) == 4 and sum(math.isnan(x) for x in xs) == 3
    assert DR.distinct_values([-1, (1 << 64) - 1, 5, 5], False) == [-1, (1 << 64) - 1, 5]
    d = np.array([0.0, -0.0, nan, nan, 3.0, 3.0, 1.5], dtype=np.float64)
    g = np.array([1, 1, 1, 1, 1, 2, 2], dtype=np.int64)
    z = np.zeros(len(d), dtype=bool)
    plan = AggPlan([INT, DBL], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_COUNT, 1, distinct=True),
                                     AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE, distinct=True),
                                     AggFunc(abi.AGG_AVG, 1, abi.TYPE_DOUBLE, distinct=True), AggFunc(abi.AGG_COUNT, 1)])
    exp = DR.expected(plan, {0: (g, z), 1: (d, z)})
    assert exp[(1,)][1] == 4 and exp[(1,)][2] is DR.NAN and exp[(1,)][4] == 5
    assert exp[(2,)][1] == 2 and exp[(2,)][2].matches(4.5) and exp[(2,)][3].matches(2.25)
    assert DR.pair_count(plan, {0: (g, z), 1: (d, z)}, 1) == 4   # NaN rows enter no set


def test_nulls_empty_input_and_decimal_scale():
    v = np.array([150, 150, 0, 7], dtype=np.int64)        # DECIMAL(5,2): 1.50 twice, a NULL, 0.07
    nl = np.array([False, False, True, False])
    plan = AggPlan([FieldType(DEC, 0, 5, 2)], [], [AggFunc(abi.AGG_COUNT, 0, distinct=True),
                                                   AggFunc(abi.AGG_SUM, 0, DEC, ret_type=DEC, ret_frac=2, distinct=True),
                                                   AggFunc(abi.AGG_AVG, 0, DEC, ret_type=DEC, ret_frac=6, distinct=True)])
    e = DR.expected(plan, {0: (v, nl)})[()]
    assert (e[0], D.to_string(e[1]), D.to_string(e[2])) == (2, "1.57", "0.785000")
    # no GROUP BY over no rows: the default row (COUNT 0, SUM and AVG NULL)
    assert DR.expected(plan, {0: (v[:0], nl[:0])}) == {(): [0, None, None]}
    # all-NULL group: COUNT 0, SUM / AVG NULL
    assert DR.expected(plan, {0: (v[2:3], nl[2:3])}) == {(): [0, None, None]}
