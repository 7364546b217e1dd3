"""Pins the exact references the GPU tests use (tests/vec_reference.py for the VecEval builtins, oracle/topn.py for
TopN's order) with known answers, and runs the Python VecEval reference against the C++ oracle (oracle/vec.cpp) on an
edge set and on random full-range rows.  CPU only."""
import math
import os
import sys

import numpy as np
import pytest

import oracle_lib as O
import vec_reference as R
from tidb_b200 import abi
from tidb_b200.chunk import Chunk, Column
from tidb_b200.plan import FilterItem

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import topn as OT   # noqa: E402

MIN, MAX, UMAX = R.INT64_MIN, R.INT64_MAX, R.UINT64_MAX
SIGNS = [(False, False), (False, True), (True, False), (True, True)]
OPS = [abi.CMP_LT, abi.CMP_LE, abi.CMP_GT, abi.CMP_GE, abi.CMP_EQ, abi.CMP_NE]
INT_EDGES, REAL_EDGES = R.INT_EDGES, R.REAL_EDGES


# ---- known answers ---------------------------------------------------------------------------------------
def _ai(op, a, au, b, bu):
    r, o, rule = R.arith_int(op, R.word(a), au, R.word(b), bu)
    return R.value(r, au or bu), o, rule


def test_arith_int_known_answers_from_reference_tests():
    # builtin_arithmetic_test.go:278-287 TestArithmeticMultiply
    assert _ai(R.MUL, 11, False, 11, False) == (121, False, None)
    assert _ai(R.MUL, -1, False, MIN, False)[1]
    assert _ai(R.MUL, MIN, False, -1, False)[1]
    # :289-291 unsigned operands
    assert _ai(R.MUL, 11, True, 11, True) == (121, False, None)
    # TestArithmeticPlus :99 / TestArithmeticMinus :195
    assert _ai(R.PLUS, 12, False, 1, False) == (13, False, None)
    assert _ai(R.MINUS, 12, False, 1, False) == (11, False, None)


@pytest.mark.parametrize("op,a,au,b,bu,exp", [
    # plus, signed + signed
    (R.PLUS, MAX, False, 1, False, None), (R.PLUS, MIN, False, -1, False, None), (R.PLUS, MAX, False, MIN, False, -1),
    (R.PLUS, MIN, False, MAX, False, -1), (R.PLUS, MAX - 1, False, 1, False, MAX),
    # unsigned + unsigned
    (R.PLUS, UMAX, True, 1, True, None), (R.PLUS, UMAX, True, 0, True, UMAX), (R.PLUS, 1 << 63, True, MAX, True, UMAX),
    # unsigned + signed, signed + unsigned
    (R.PLUS, 0, True, -1, False, None), (R.PLUS, 5, True, -5, False, 0), (R.PLUS, UMAX, True, -1, False, UMAX - 1),
    (R.PLUS, 1 << 63, True, MIN, False, 0), (R.PLUS, 1, True, MAX, False, 1 << 63), (R.PLUS, UMAX, True, 1, False, None),
    (R.PLUS, -1, False, 1, True, 0), (R.PLUS, MIN, False, 1 << 63, True, 0), (R.PLUS, -1, False, 0, True, None),
    (R.PLUS, 1, False, UMAX, True, None), (R.PLUS, MAX, False, 1 << 63, True, UMAX),
    # minus
    (R.MINUS, MIN, False, 1, False, None), (R.MINUS, MAX, False, -1, False, None), (R.MINUS, -1, False, MIN, False, MAX),
    (R.MINUS, -2, False, MAX, False, None), (R.MINUS, -1, False, MAX, False, MIN),
    (R.MINUS, 0, True, 1, True, None), (R.MINUS, 5, True, 5, True, 0), (R.MINUS, UMAX, True, 0, True, UMAX),
    (R.MINUS, 0, True, 1, False, None), (R.MINUS, 0, True, -1, False, 1), (R.MINUS, UMAX, True, -1, False, None),
    (R.MINUS, 1 << 63, True, MAX, False, 1), (R.MINUS, MAX, True, MIN, False, UMAX), (R.MINUS, 1 << 63, True, MIN, False, None),
    (R.MINUS, -22, False, 10, True, None), (R.MINUS, 5, False, 5, True, 0), (R.MINUS, MAX, False, 0, True, MAX),
    (R.MINUS, 0, False, 1, True, None), (R.MINUS, MIN, False, 3, True, None),
    # multiply
    (R.MUL, MAX, False, 2, False, None), (R.MUL, 1 << 32, False, 1 << 31, False, None), (R.MUL, -(1 << 32), False, 1 << 31, False, MIN),
    (R.MUL, 3037000499, False, 3037000499, False, 3037000499 ** 2), (R.MUL, 3037000500, False, 3037000500, False, None),
    (R.MUL, -1, False, MAX, False, -MAX), (R.MUL, 1 << 32, True, 1 << 32, True, None),
    (R.MUL, (1 << 32) - 1, True, (1 << 32) + 1, True, UMAX), (R.MUL, 0, True, UMAX, True, 0),
])
def test_arith_int_boundaries(op, a, au, b, bu, exp):
    r, o, _ = _ai(op, a, au, b, bu)
    assert o == (exp is None)
    if exp is not None:
        assert r == exp


def test_arith_int_go_rules():
    # the two places where TiDB's vectorized code departs from exact arithmetic
    assert _ai(R.MINUS, 0, False, MIN, False) == (MIN, False, "ZERO_MINUS_INT64_MIN")      # exact 2^63 would overflow
    assert _ai(R.MINUS, 1, False, MIN, False)[1]                                           # ... but 1 - INT64_MIN does
    assert _ai(R.MINUS, -1, False, MIN, False) == (MAX, False, None)
    assert _ai(R.MUL, -1, False, 1, True) == (UMAX, False, "MUL_UNSIGNED_BITS")            # exact -1 would overflow
    assert _ai(R.MUL, 1, True, -1, False) == (UMAX, False, "MUL_UNSIGNED_BITS")
    assert _ai(R.MUL, -1, False, 0, True) == (0, False, "MUL_UNSIGNED_BITS")
    assert _ai(R.MUL, -1, False, 2, True)[1]
    assert _ai(R.MUL, MIN, False, 2, True)[1]                                              # 2^63 * 2 = 2^64
    assert _ai(R.MUL, MIN, False, 1, True) == (1 << 63, False, "MUL_UNSIGNED_BITS")
    # no other pair of edge values is decided by a rule
    for a in INT_EDGES:
        for b in INT_EDGES:
            for au, bu in SIGNS:
                for op in (R.PLUS, R.MINUS, R.MUL):
                    rule = R.arith_int(op, a, au, b, bu)[2]
                    if rule == "ZERO_MINUS_INT64_MIN":
                        assert (op, a, b, au, bu) == (R.MINUS, 0, MIN, False, False)
                    elif rule == "MUL_UNSIGNED_BITS":
                        assert op == R.MUL and au != bu


def test_compare_known_answers():
    assert R.compare_int(-1, False, -1, True) == -1          # -1 < 2^64 - 1
    assert R.compare_int(-1, True, -1, False) == 1
    assert R.compare_int(MIN, True, MAX, False) == 1          # 2^63 > 2^63 - 1
    assert R.compare_int(MAX, True, MAX, False) == 0
    assert R.compare_int(MIN, False, MIN, True) == -1
    assert R.compare_int(5, True, 5, False) == 0
    assert R.compare_int(-1, True, -2, True) == 1
    assert R.compare_real(math.nan, -math.inf) == -1 and R.compare_real(math.nan, -math.nan) == 0
    assert R.compare_real(-0.0, 0.0) == 0 and R.compare_real(5e-324, 0.0) == 1 and R.compare_real(-math.inf, -1e308) == -1


def test_arith_real_known_answers():
    r, o = R.arith_real(R.MUL, math.inf, 0.0)
    assert math.isnan(r) and not o                            # * overflows only on +-Inf
    r, o = R.arith_real(R.MUL, math.nan, 2.0)
    assert math.isnan(r) and not o
    r, o = R.arith_real(R.PLUS, math.nan, 2.0)
    assert math.isnan(r) and o                                # + / - overflow on any non-finite result
    assert R.arith_real(R.MINUS, math.inf, math.inf)[1]
    assert R.arith_real(R.MUL, 1e308, 10.0) == (math.inf, True)
    assert R.arith_real(R.PLUS, 1.7976931348623157e308, 1e292) == (math.inf, True)
    assert math.copysign(1.0, R.arith_real(R.PLUS, -0.0, -0.0)[0]) == -1.0
    assert math.copysign(1.0, R.arith_real(R.PLUS, -0.0, 0.0)[0]) == 1.0
    assert math.copysign(1.0, R.arith_real(R.MINUS, -0.0, 0.0)[0]) == -1.0
    assert math.copysign(1.0, R.arith_real(R.MUL, 0.0, -3.0)[0]) == -1.0
    assert R.arith_real(R.MUL, 5e-324, 0.5) == (0.0, False)   # subnormal rounds to even
    assert R.arith_real(R.MUL, 2.2250738585072014e-308, 0.5) == (1.1125369292536007e-308, False)


def test_compare_vec_matches_scalar_on_edges():
    a = np.array([x for x in INT_EDGES for _ in INT_EDGES], np.int64)
    b = np.array([y for _ in INT_EDGES for y in INT_EDGES], np.int64)
    for au, bu in SIGNS:
        exp = [R.compare_int(int(x), au, int(y), bu) for x, y in zip(a, b)]
        assert R.compare_int_vec(a, au, b, bu).tolist() == exp
        for k in INT_EDGES:
            assert R.compare_int_vec(a, au, k, bu).tolist() == [R.compare_int(int(x), au, k, bu) for x in a]
    x = np.array([p for p in REAL_EDGES for _ in REAL_EDGES]); y = np.array([q for _ in REAL_EDGES for q in REAL_EDGES])
    assert R.compare_real_vec(x, y).tolist() == [R.compare_real(p, q) for p, q in zip(x.tolist(), y.tolist())]


# ---- the Python reference against the C++ oracle -----------------------------------------------------------
def _int_cases(rng, n):
    """(a, b) int64 words: every pair of edge values, then n random rows (full range, small, edges, edge +- small)"""
    ea = np.array([x for x in INT_EDGES for _ in INT_EDGES], np.int64)
    eb = np.array([y for _ in INT_EDGES for y in INT_EDGES], np.int64)
    def col():
        kind = rng.integers(0, 4, n)
        full = rng.integers(MIN, MAX, n, endpoint=True, dtype=np.int64)
        small = rng.integers(-100, 100, n).astype(np.int64)
        edge = np.array(INT_EDGES, np.int64)[rng.integers(0, len(INT_EDGES), n)]
        with np.errstate(over="ignore"):
            near = edge + rng.integers(-3, 4, n).astype(np.int64)      # wraps at the int64 ends: still a valid word
        return np.select([kind == 0, kind == 1, kind == 2], [full, small, edge], near)
    return np.concatenate([ea, col()]), np.concatenate([eb, col()])


@pytest.mark.parametrize("n", [0, 200_000])
def test_vec_int_reference_vs_oracle(n):
    rng = np.random.default_rng(2024 + n)
    a, b = _int_cases(rng, n)
    m = len(a)
    an, bn = rng.random(m) < 0.05, rng.random(m) < 0.05
    for au, bu in SIGNS:
        for op in OPS:
            exp, enul = R.compare_int_col(op, a, an, b, bn, 0, au, bu)
            got, gnul = O.vec_compare_int(op, Column(a, an), Column(b, bn), 0, au, bu)
            assert np.array_equal(got, exp) and np.array_equal(gnul, enul), (op, au, bu)
            for k in (0, -1, MIN, MAX, 1 << 32):
                exp, enul = R.compare_int_col(op, a, an, None, None, k, au, bu)
                got, gnul = O.vec_compare_int(op, Column(a, an), None, k, au, bu)
                assert np.array_equal(got, exp) and np.array_equal(gnul, enul), (op, au, bu, k)
        for op in (R.PLUS, R.MINUS, R.MUL):
            ovf = R.arith_int_overflow_rows(op, a, b, 0, au, bu)
            nl = an | ovf                           # every overflowing row under NULL: the whole column is computed
            err, exp, enul = R.arith_int_vec(op, a, nl, b, bn, 0, au, bu)
            assert not err
            rc, got, gnul = O.vec_arith_int(op, Column(a, nl), Column(b, bn), 0, au, bu)
            assert rc == 0 and np.array_equal(gnul, enul), (op, au, bu)
            bad = np.flatnonzero(got != exp)
            assert len(bad) == 0, (op, au, bu, [(int(a[i]), int(b[i]), int(got[i]), int(exp[i])) for i in bad[:5]])
            if ovf.any():                           # one overflowing row left non-NULL fails the call
                i = int(np.flatnonzero(ovf)[-1])
                nl2 = nl.copy(); nl2[i] = False
                b2n = bn.copy(); b2n[i] = False
                assert R.arith_int_vec(op, a, nl2, b, b2n, 0, au, bu)[0]
                assert O.vec_arith_int(op, Column(a, nl2), Column(b, b2n), 0, au, bu)[0] == abi.TG_ERR_OVERFLOW


@pytest.mark.parametrize("n", [0, 200_000])
def test_vec_real_reference_vs_oracle(n):
    rng = np.random.default_rng(77 + n)
    ea = np.array([x for x in REAL_EDGES for _ in REAL_EDGES]); eb = np.array([y for _ in REAL_EDGES for y in REAL_EDGES])
    def col():
        kind = rng.integers(0, 3, n)
        bits = rng.integers(MIN, MAX, n, endpoint=True, dtype=np.int64).view(np.float64)     # any double, NaNs included
        return np.select([kind == 0, kind == 1], [bits, rng.normal(0, 1e3, n)], np.array(REAL_EDGES)[rng.integers(0, len(REAL_EDGES), n)])
    a, b = np.concatenate([ea, col()]), np.concatenate([eb, col()])
    m = len(a)
    an, bn = rng.random(m) < 0.05, rng.random(m) < 0.05
    for op in OPS:
        exp, enul = R.compare_real_col(op, a, an, b, bn)
        got, gnul = O.vec_compare_real(op, Column(a, an), Column(b, bn))
        assert np.array_equal(got, exp) and np.array_equal(gnul, enul), op
        for k in (0.0, -0.0, math.nan, -math.inf):
            exp, enul = R.compare_real_col(op, a, an, None, None, k)
            got, gnul = O.vec_compare_real(op, Column(a, an), None, k)
            assert np.array_equal(got, exp) and np.array_equal(gnul, enul), (op, k)
    for op in (R.PLUS, R.MINUS, R.MUL):
        ovf = R.arith_real_vec(op, a, an, b, bn)[3]
        nl = an | ovf
        err, exp, enul, _ = R.arith_real_vec(op, a, nl, b, bn)
        assert not err
        rc, got, gnul = O.vec_arith_real(op, Column(a, nl), Column(b, bn))
        assert rc == 0 and np.array_equal(gnul, enul)
        assert np.array_equal(got.view(np.int64), exp.view(np.int64)), op      # same IEEE operations on the same CPU
        if ovf.any():
            nl2 = nl.copy(); nl2[np.flatnonzero(ovf)[0]] = False
            assert R.arith_real_vec(op, a, nl2, b, bn)[0]
            assert O.vec_arith_real(op, Column(a, nl2), Column(b, bn))[0] == abi.TG_ERR_OVERFLOW


def test_vec_filter_reference_vs_oracle():
    rng = np.random.default_rng(5)
    a, b = _int_cases(rng, 50_000)
    m = len(a)
    x = np.array(REAL_EDGES)[rng.integers(0, len(REAL_EDGES), m)]
    y = np.array(REAL_EDGES)[rng.integers(0, len(REAL_EDGES), m)]
    nls = [rng.random(m) < 0.03 for _ in range(4)]
    chk = Chunk([Column(a, nls[0]), Column(b, nls[1]), Column(x, nls[2]), Column(y, nls[3])])
    cols = [(c.data, c.nulls()) for c in chk.columns]
    item_sets = [
        [FilterItem(abi.CMP_GT, 0, const_i64=-1, lhs_unsigned=True)],
        [FilterItem(abi.CMP_LT, 0, rhs_col=1, lhs_unsigned=True, rhs_unsigned=False)],
        [FilterItem(abi.CMP_GE, 1, rhs_col=0, lhs_unsigned=False, rhs_unsigned=True)],
        [FilterItem(abi.CMP_EQ, 0, const_i64=MIN, rhs_unsigned=True)],                   # no signed value equals 2^63
        [FilterItem(abi.CMP_EQ, 0, const_i64=MIN, rhs_unsigned=True, lhs_unsigned=True)],
        [FilterItem(abi.CMP_NE, 2, rhs_col=3, is_real=True)],
        [FilterItem(abi.CMP_LE, 2, is_real=True, const_f64=-0.0), FilterItem(abi.CMP_GE, 3, is_real=True, const_f64=math.nan)],
        [FilterItem(abi.CMP_GE, 0, const_i64=0), FilterItem(abi.CMP_LT, 1, const_i64=-1, rhs_unsigned=True),
         FilterItem(abi.CMP_NE, 0, rhs_col=1, lhs_unsigned=True, rhs_unsigned=True), FilterItem(abi.CMP_LE, 1, const_i64=MAX),
         FilterItem(abi.CMP_GT, 2, is_real=True, const_f64=-math.inf), FilterItem(abi.CMP_NE, 3, is_real=True, const_f64=0.0),
         FilterItem(abi.CMP_LE, 0, const_i64=-2, rhs_unsigned=True, lhs_unsigned=True), FilterItem(abi.CMP_GE, 2, rhs_col=3, is_real=True)],
    ]
    sel = np.sort(rng.choice(m, m // 3, replace=False)).astype(np.int64)
    for items in item_sets:
        exp = R.filter_rows(cols, items)
        got, cnt = O.vec_filter(chk, items)
        assert np.array_equal(got, exp) and cnt == int(exp.sum()), items
        exp = R.filter_rows(cols, items, sel)
        got, cnt = O.vec_filter(Chunk(chk.columns, sel), items)
        assert np.array_equal(got, exp) and cnt == int(exp.sum()), items


# ---- TopN order -------------------------------------------------------------------------------------------
def test_topn_reference_zero_and_nan():
    rows = [(-0.0, 2), (0.0, 1)]
    assert OT.topn_rows(rows, ["real", "int"], [(0, False), (1, False)], 0, 1) == [(0.0, 1)]
    assert OT.topn_rows(rows[::-1], ["real", "int"], [(0, False), (1, False)], 0, 1) == [(0.0, 1)]
    rows = [(0.0, 2), (-0.0, 1)]
    assert OT.topn_rows(rows, ["real", "int"], [(0, True), (1, False)], 0, 1) == [(-0.0, 1)]
    nan2 = R.f64_from_bits(-0x0007FFFFFFFFFF00)
    rows = [(1.0, 0), (math.nan, 1), (None, 2), (-math.inf, 3), (nan2, 4)]
    got = OT.topn_rows(rows, ["real", "int"], [(0, False), (1, True)], 0, 5)
    assert [r[1] for r in got] == [2, 4, 1, 3, 0]                 # NULL, the two NaNs (equal), -Inf, 1
    got = OT.topn_rows(rows, ["real", "int"], [(0, True), (1, False)], 0, 5)
    assert [r[1] for r in got] == [0, 3, 1, 4, 2]


def test_topn_reference_time_ignores_fsp_bits():
    t = OT.pack_time(2024, 2, 29, 23, 59, 58, 999999)
    assert OT.time_fields(t) == dict(year=2024, month=2, day=29, hour=23, minute=59, second=58, microsecond=999999)
    rows = [(t | 0x5, 2), (t | 0x3, 1), (OT.pack_time(2024, 2, 29, 23, 59, 59, 0), 0)]
    assert OT.topn_rows(rows, ["time", "int"], [(0, False), (1, False)], 0, 2) == [(t | 0x3, 1), (t | 0x5, 2)]
    assert OT.topn_rows(rows, ["time", "int"], [(0, True), (1, True)], 0, 2)[0][1] == 0
    assert OT._cmp_time(OT.pack_time(1999, 12, 31, 23, 59, 59, 999999), OT.pack_time(2000, 1, 1)) == -1
    assert OT._cmp_time(OT.pack_time(0, 0, 0), OT.pack_time(0, 0, 0, fsp_tt=0xF)) == 0


def _edge_table(rng, n):
    ints = np.array(INT_EDGES, np.int64)[rng.integers(0, len(INT_EDGES), n)]
    reals = np.array(REAL_EDGES)[rng.integers(0, len(REAL_EDGES), n)]
    times = np.array([OT.pack_time(y, mo, d, h, mi, s, us, f) for y, mo, d, h, mi, s, us, f in zip(
        rng.choice([0, 1969, 2024, 9999], n), rng.integers(0, 13, n), rng.integers(0, 32, n), rng.integers(0, 2, n),
        rng.integers(0, 2, n), rng.integers(0, 60, n), rng.choice([0, 1, 999999], n), rng.integers(0, 16, n))],
        dtype=np.uint64).view(np.int64)
    small = rng.integers(0, 3, n).astype(np.int64)
    vals = [ints, ints.copy(), reals, times, small]
    rng.shuffle(vals[1])
    nulls = [rng.random(n) < 0.1 for _ in vals]
    return vals, nulls, ["int", "uint", "real", "time", "int"]


@pytest.mark.parametrize("seed", range(4))
def test_topn_order_matches_topn_rows(seed):
    rng = np.random.default_rng(seed)
    n = 3000
    vals, nulls, kinds = _edge_table(rng, n)
    rows = [tuple(None if nulls[c][i] else (vals[c][i].item() if kinds[c] != "real" else float(vals[c][i])) for c in range(len(vals))) + (i,)
            for i in range(n)]
    cols = [(v, nl) for v, nl in zip(vals, nulls)]
    for by in ([(0, False)], [(1, True), (4, False)], [(2, False), (4, True)], [(2, True), (3, False)], [(3, True), (2, False), (1, False)],
               [(4, False), (3, False), (2, True), (1, True), (0, False)]):
        for offset, count in ((0, n), (7, 100), (n - 1, 5)):
            exp = [r[-1] for r in OT.topn_rows(rows, kinds + ["int"], by, offset, count)]
            assert OT.topn_order(cols, kinds, by, offset, count).tolist() == exp, (by, offset, count)
