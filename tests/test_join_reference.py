"""tests/join_reference.py against the nested-loop restatement (row for row, small random cases over every join type, both
build sides, filters, OtherCondition, 1-4 key columns, FLOAT / DOUBLE / date-time / mixed-signedness keys, NULLs, sel vectors and
constructed candidate-key collisions) and against oracle/join.cpp on cases of about 200 K rows."""
import numpy as np
import pytest

import join_keys as K
import oracle_lib as O
from join_reference import assert_same_rows, join_reference, to_rows
from nested_loop import assert_rows_equal, nested_loop_join
from test_oracle_join import DATE_TT, DATETIME6_TT, JOIN_TYPES, core_time
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.plan import FieldType, FilterItem, JoinPlan, OtherCond

INT = FieldType(abi.TYPE_LONGLONG, 0)
UINT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED)
FLT = FieldType(abi.TYPE_FLOAT, 0)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
DATE = FieldType(abi.TYPE_DATE, 0)
DATETIME = FieldType(abi.TYPE_DATETIME, 0)

F32_POOL = np.array([0.0, -0.0, 0.1, 0.5, -0.5, 1.0, 3.4028234663852886e38, -3.4028234663852886e38, 1e-40, -1e-40, np.inf, -np.inf,
                     1.5, 2.25], dtype=np.float32)
F64_EXTRA = np.array([0.1, float(np.float32(0.1)), 0.5, -0.0, 1e-40, float(np.float32(1e-40)), np.inf, 2.25, 7.0], dtype=np.float64)
TIME_DAYS = [(2023, 1 + m, 1 + d) for m in range(3) for d in range(5)]


def key_values(rng, kind, side, n, key_range):
    """(values, type) of one key column; side 0 = left, 1 = right"""
    if kind == "int":
        return rng.integers(-key_range, key_range, n).astype(np.int64), INT
    if kind == "mixed":   # left UNSIGNED, right signed: the same bits of a negative value must not match
        v = rng.integers(-key_range, key_range, n).astype(np.int64)
        ext = np.array([-1, -(1 << 63), (1 << 63) - 1, 0], dtype=np.int64)
        pick = rng.random(n) < 0.02
        v[pick] = ext[rng.integers(0, len(ext), int(pick.sum()))]
        return v, (UINT if side == 0 else INT)
    if kind == "float":
        return F32_POOL[rng.integers(0, len(F32_POOL), n)], FLT
    if kind == "float_double":
        if side == 0:
            return F32_POOL[rng.integers(0, len(F32_POOL), n)], FLT
        pool = np.concatenate([F32_POOL.astype(np.float64), F64_EXTRA])
        return pool[rng.integers(0, len(pool), n)], DBL
    if kind == "double":
        return rng.integers(-key_range, key_range, n).astype(np.float64) / 4, DBL
    if kind == "time":
        tt = DATETIME6_TT if side == 0 else DATE_TT
        w = [core_time(*TIME_DAYS[int(i)], fsp_tt=tt) if (side == 1 or rng.random() < 0.5) else core_time(*TIME_DAYS[int(i)], 1, 2, 3, 4, tt)
             for i in rng.integers(0, len(TIME_DAYS), n)]
        return np.array(w, dtype=np.int64), (DATETIME if side == 0 else DATE)
    raise ValueError(kind)


def gen_case(rng, nl, nr, kind="int", nkeys=1, nulls=0.1, sel=False, key_range=40, chunk_rows=(37, 29)):
    """left: [payload, key_1 .. key_nkeys, payload], right: [key_1 .. key_nkeys, payload]; a third of the left rows copy a
    right row's keys"""
    def payload(n):
        return rng.integers(-1 << 40, 1 << 40, n).astype(np.int64)

    def nl_mask(n):
        return rng.random(n) < nulls if nulls > 0 else None
    lkeys = [key_values(rng, kind, 0, nl, key_range) for _ in range(nkeys)]
    rkeys = [key_values(rng, kind, 1, nr, key_range) for _ in range(nkeys)]
    if nl and nr:
        src, dst = rng.integers(0, nr, nl // 3), rng.choice(nl, nl // 3, replace=False)
        for (lv, lt), (rv, rt) in zip(lkeys, rkeys):
            lv[dst] = rv[src].astype(lv.dtype)
    lcols = [Column(payload(nl), nl_mask(nl))] + [Column(v, nl_mask(nl)) for v, _ in lkeys] + [Column(payload(nl), nl_mask(nl))]
    rcols = [Column(v, nl_mask(nr)) for v, _ in rkeys] + [Column(payload(nr), nl_mask(nr))]
    ltypes = [INT] + [t for _, t in lkeys] + [INT]
    rtypes = [t for _, t in rkeys] + [INT]
    left, right = Chunk(lcols).split(chunk_rows[0]), Chunk(rcols).split(chunk_rows[1])
    if sel:
        for lst in (left, right):
            for ch in lst:
                m = ch.columns[0].length
                ch.sel = np.sort(rng.choice(m, max(1, m * 2 // 3), replace=False)).astype(np.int64)
    return ltypes, rtypes, left, right


def plan_for(jt, brt, ltypes, rtypes, nkeys, filters=False, other=False):
    semi = jt >= abi.JOIN_SEMI
    lf = [FilterItem(abi.CMP_GT, 0, const_i64=-(1 << 39))]
    rf = [FilterItem(abi.CMP_LT, nkeys, const_i64=1 << 39)]
    oc = [OtherCond(abi.CMP_LE, 0, 0, 1, nkeys), OtherCond(abi.CMP_NE, 1, nkeys, -1, -1, const_i64=7)] if other else []
    return JoinPlan(jt, ltypes, rtypes, list(range(1, 1 + nkeys)), list(range(nkeys)), build_is_right=brt,
                    lused=list(range(nkeys + 2)), rused=[] if semi else [nkeys, 0],
                    probe_filter=(lf if brt else rf) if filters else [], build_filter=(rf if brt else lf) if filters else [],
                    other_cond=oc)


def needs_build_scan(jt, brt):
    """the outer side of an outer join, or the left side of a semi / anti join, is the build side"""
    return (jt == abi.JOIN_LEFT_OUTER and not brt) or (jt == abi.JOIN_RIGHT_OUTER and brt) or (jt in (abi.JOIN_SEMI, abi.JOIN_ANTI_SEMI) and not brt)


def allowed(jt, brt):
    if jt in (abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI) and not brt:
        return False      # NewJoinProbe: left outer semi needs the right side as build side
    return True


CASES = [dict(kind=k, nkeys=nk, nulls=nu, sel=s, filters=f, other=o)
         for k, nk, nu, s, f, o in [("int", 1, 0.0, False, False, False), ("int", 1, 0.15, True, True, False),
                                    ("int", 1, 0.1, False, False, True), ("int", 2, 0.08, True, True, True),
                                    ("int", 3, 0.05, False, False, False), ("int", 4, 0.05, True, False, True),
                                    ("mixed", 1, 0.1, False, True, False), ("mixed", 2, 0.05, True, False, False),
                                    ("float", 1, 0.1, True, False, False), ("float_double", 1, 0.1, False, True, False),
                                    ("double", 1, 0.1, True, True, False), ("time", 1, 0.1, False, False, False)]]


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("jt", JOIN_TYPES)
@pytest.mark.parametrize("brt", [True, False])
def test_reference_vs_nested_loop(case, jt, brt):
    if not allowed(jt, brt):
        pytest.skip("NewJoinProbe: left outer semi needs the right side as build side")
    c = CASES[case]
    rng = np.random.default_rng(100 * case + 10 * jt + int(brt))
    ltypes, rtypes, l, r = gen_case(rng, 300, 250, c["kind"], c["nkeys"], c["nulls"], c["sel"], key_range=8 if c["nkeys"] > 1 else 40)
    other = c["other"] and jt not in (abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI)   # nested_loop: no residual there
    plan = plan_for(jt, brt, ltypes, rtypes, c["nkeys"], c["filters"], other)
    want = nested_loop_join(plan, l, r)
    assert_rows_equal(want, to_rows(join_reference(plan, l, r)))


def test_reference_special_float_keys_known_answers():
    # 0.1f != 0.1 but == float64(0.1f); 0.5f == 0.5; -0.0f == 0.0; inf == inf; a subnormal f32 equals its float64 value only
    lk = np.array([0.1, 0.5, -0.0, np.inf, 1e-40, 3.4028234663852886e38], dtype=np.float32)
    rk = np.array([0.1, float(np.float32(0.1)), 0.5, 0.0, np.inf, 1e-40, float(np.float32(1e-40)), 3.4028234663852886e38], dtype=np.float64)
    plan = JoinPlan(abi.JOIN_INNER, [FLT], [DBL], [0], [0])
    got = to_rows(join_reference(plan, [Chunk([Column(lk)])], [Chunk([Column(rk)])]))
    f = lambda x: float(np.float32(x))
    assert sorted(got) == sorted([(f(0.1), f(0.1)), (0.5, 0.5), (-0.0, 0.0), (np.inf, np.inf), (f(1e-40), f(1e-40)),
                                  (f(3.4028234663852886e38), 3.4028234663852886e38)])


@pytest.mark.parametrize("ncols", [2, 3, 4])
@pytest.mark.parametrize("jt,brt", [(abi.JOIN_INNER, True), (abi.JOIN_LEFT_OUTER, True), (abi.JOIN_RIGHT_OUTER, False),
                                    (abi.JOIN_SEMI, True), (abi.JOIN_ANTI_SEMI, True)])
def test_reference_constructed_collisions_vs_nested_loop(ncols, jt, brt):
    # probe tuples with the same candidate key as a build tuple but another value: never a match
    rng = np.random.default_rng(ncols * 10 + jt)
    b = rng.integers(-1000, 1000, (200, ncols)).astype(np.int64)
    p = b[rng.integers(0, 200, 300)].copy()
    for i in range(0, 300, 3):
        p[i] = K.colliding_keys(tuple(int(x) for x in p[i]), ncols, delta=int(rng.integers(1, 50)))
    bcols = [Column(b[:, c]) for c in range(ncols)] + [Column(np.arange(200, dtype=np.int64))]
    pcols = [Column(np.arange(300, dtype=np.int64))] + [Column(p[:, c], rng.random(300) < 0.05) for c in range(ncols)] + [Column(np.zeros(300, np.int64))]
    probe, build = [Chunk(pcols)], [Chunk(bcols)]
    lt, rt = [INT] * (ncols + 2), [INT] * (ncols + 1)
    plan = plan_for(jt, brt, lt, rt, ncols)
    l, r = (probe, build) if brt else (build, probe)
    if not brt:
        plan = JoinPlan(jt, rt, lt, list(range(ncols)), list(range(1, 1 + ncols)), build_is_right=False, lused=list(range(ncols + 1)),
                        rused=list(range(ncols + 2)))
    want = nested_loop_join(plan, l, r)
    assert_rows_equal(want, to_rows(join_reference(plan, l, r)))


def run_oracle_cols(plan, left, right):
    build, probe = (right, left) if plan.build_is_right else (left, right)
    j = O.OracleJoin(plan, 5)
    n, cols = j.run(build, probe)
    j.close()
    return cols


@pytest.mark.parametrize("jt", JOIN_TYPES)
@pytest.mark.parametrize("brt", [True, False])
@pytest.mark.parametrize("kind,nkeys,other", [("int", 1, False), ("int", 2, True), ("double", 1, False), ("mixed", 1, False)])
def test_reference_vs_oracle_medium(jt, brt, kind, nkeys, other):
    if not allowed(jt, brt):
        pytest.skip("NewJoinProbe: left outer semi needs the right side as build side")
    if other and (jt in (abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI) or needs_build_scan(jt, brt)):
        pytest.skip("OtherCondition / several keys with a build-side scan or a left outer semi join are not offloaded")
    rng = np.random.default_rng(9000 + jt * 3 + int(brt) + 50 * nkeys)
    ltypes, rtypes, l, r = gen_case(rng, 200_000, 150_000, kind, nkeys, 0.05, True, key_range=300 if nkeys > 1 else 60_000,
                                    chunk_rows=(4096, 4096))
    plan = plan_for(jt, brt, ltypes, rtypes, nkeys, True, other)
    want = join_reference(plan, l, r)
    assert len(want[0][0]) > 1000
    assert_same_rows(want, run_oracle_cols(plan, l, r), "oracle")
