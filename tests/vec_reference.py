"""Exact reference of the VecEval builtins (tg_vec_compare_*, tg_vec_arith_*, tg_vec_filter), used only by tests/.

A restatement over mathematical values in plain Python integers and floats, written from the semantics and not from
the C++ code, so that a defect shared by the kernels and the C++ oracle can still be seen:

- An integer argument is an 8-byte word.  A signed argument's value is the two's-complement int64; an UNSIGNED
  argument's value is the word mod 2^64.
- Comparison (types.CompareInt, pkg/types/compare.go:86) orders those values.  REAL comparison is Go cmp.Compare:
  NaN below everything, NaN == NaN, -0 == +0.
- Integer +, - and * are computed exactly.  The result overflows when it falls outside int64 with both arguments
  signed, and outside [0, 2^64) otherwise (the result is UNSIGNED when either argument is: builtin_arithmetic.go:207,
  :378, :583).  Where TiDB's vectorized code departs from exact arithmetic the Go code wins; each such place is a named
  rule below that cites its line.
- REAL + and - overflow on a non-finite result (mathutil.IsFinite, builtin_arithmetic_vec.go:496-523, :300-322),
  * only on +-Inf (math.IsInf, :40-62).  An overflow on a NULL row is not an error.
- A result row is NULL when either argument is (Column.MergeNulls, column.go:906).  The library writes 0 as the value
  of an integer row that overflows under NULL; every other row holds its computed value, NULL or not.
- The filter follows VecEvalBool (expression.go:409-494): a row is selected when every item is non-NULL and true.

The scalar functions are the definition.  The *_vec wrappers apply them to numpy columns: arithmetic evaluates each
distinct (lhs, rhs) pair once, comparison uses an order-preserving numeric key that tests/test_vec_topn_reference.py
pins against the scalar compare.
"""
from __future__ import annotations

import math
import struct
from typing import Optional, Sequence, Tuple

import numpy as np

TWO64 = 1 << 64
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
UINT64_MAX = TWO64 - 1

CMP_LT, CMP_LE, CMP_GT, CMP_GE, CMP_EQ, CMP_NE = 0, 1, 2, 3, 4, 5
PLUS, MINUS, MUL = 0, 1, 2


def value(word: int, unsigned: bool) -> int:
    """the mathematical value of an 8-byte integer word (any Python int; only its low 64 bits count)"""
    u = word % TWO64
    if unsigned:
        return u
    return u - TWO64 if u >= 1 << 63 else u


def word(v: int) -> int:
    """the int64 bit pattern (as a signed Python int, the way an int64 numpy column holds it) of v mod 2^64"""
    return value(v, False)


def f64_bits(x: float) -> int:
    return struct.unpack("<q", struct.pack("<d", x))[0]


def f64_from_bits(w: int) -> float:
    return struct.unpack("<d", struct.pack("<q", word(w)))[0]


# edge values the tests draw from
# int64 words: read as UNSIGNED, -1 is 2^64 - 1 and INT64_MIN is 2^63
INT_EDGES = [0, 1, -1, 2, -2, 7, -7, 1 << 31, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, -(1 << 32), 3037000499, 3037000500,
             -3037000500, 1 << 62, -(1 << 62), INT64_MAX, INT64_MAX - 1, INT64_MIN, INT64_MIN + 1]
REAL_EDGES = [0.0, -0.0, 1.0, -1.0, 0.5, 2.0, 1e308, -1e308, 1.7976931348623157e308, math.inf, -math.inf, math.nan,
              f64_from_bits(0x7FF0000000000123), f64_from_bits(-0x000FFFFFFFFFF001),   # NaNs of both signs with payloads
              5e-324, -5e-324, 2.2250738585072009e-308, 3.0, -0.1]


# ---- comparison ---------------------------------------------------------------------------------------
def compare_int(a: int, a_unsigned: bool, b: int, b_unsigned: bool) -> int:
    x, y = value(a, a_unsigned), value(b, b_unsigned)
    return (x > y) - (x < y)


def compare_real(x: float, y: float) -> int:
    xn, yn = math.isnan(x), math.isnan(y)
    if xn or yn:
        return 0 if (xn and yn) else (-1 if xn else 1)
    return (x > y) - (x < y)          # -0.0 == 0.0 in Python as in IEEE 754


def holds(op: int, c: int) -> bool:
    return {CMP_LT: c < 0, CMP_LE: c <= 0, CMP_GT: c > 0, CMP_GE: c >= 0, CMP_EQ: c == 0, CMP_NE: c != 0}[op]


# ---- arithmetic -----------------------------------------------------------------------------------------
# Rule ZERO_MINUS_INT64_MIN: builtinArithmeticMinusIntSig.overflowCheck (builtin_arithmetic.go:491-535) flags a
# signed a - b only for a > 0, b < 0 past INT64_MAX and for a < 0, b > 0 that wraps.  a = 0, b = INT64_MIN fits
# neither, so 0 - INT64_MIN returns the wrapped INT64_MIN without an error, although the exact 2^63 is out of range.
# Rule MUL_UNSIGNED_BITS: with either argument UNSIGNED the planner picks builtinArithmeticMultiplyIntUnsignedSig
# (builtin_arithmetic.go:583-587), which multiplies the two words as uint64 (builtin_arithmetic_vec.go:1010-1040):
# a negative signed argument counts as 2^64 + v.  So -1 * 1u is 2^64 - 1 without an error, and -1 * 0u is 0.
RULES = ("ZERO_MINUS_INT64_MIN", "MUL_UNSIGNED_BITS")


def arith_int(op: int, a: int, a_unsigned: bool, b: int, b_unsigned: bool) -> Tuple[int, bool, Optional[str]]:
    """-> (result word, overflow, name of the rule that decided it or None)"""
    unsigned = a_unsigned or b_unsigned
    if op == MUL and unsigned:
        p = (a % TWO64) * (b % TWO64)
        rule = "MUL_UNSIGNED_BITS" if not (a_unsigned and b_unsigned) else None
        return word(p), p > UINT64_MAX, rule
    x, y = value(a, a_unsigned), value(b, b_unsigned)
    if op == MINUS and not unsigned and x == 0 and y == INT64_MIN:
        return INT64_MIN, False, "ZERO_MINUS_INT64_MIN"
    exact = x + y if op == PLUS else (x - y if op == MINUS else x * y)
    lo, hi = (0, UINT64_MAX) if unsigned else (INT64_MIN, INT64_MAX)
    return word(exact), not lo <= exact <= hi, None


def arith_real(op: int, x: float, y: float) -> Tuple[float, bool]:
    """-> (IEEE double result, overflow)"""
    r = x + y if op == PLUS else (x - y if op == MINUS else x * y)
    return r, (math.isinf(r) if op == MUL else not math.isfinite(r))


# ---- numpy columns --------------------------------------------------------------------------------------
def _merge_nulls(an: np.ndarray, bn: Optional[np.ndarray]) -> np.ndarray:
    return an.copy() if bn is None else (an | bn)


def _pairs(a: np.ndarray, b: Optional[np.ndarray], b_const):
    """distinct (lhs, rhs) pairs of two 8-byte columns (or a column and a constant) and each row's pair index"""
    a = np.ascontiguousarray(a).view(np.int64)
    if b is None:
        ua, inv = np.unique(a, return_inverse=True)
        return [(int(x), b_const) for x in ua], inv.reshape(-1)
    b = np.ascontiguousarray(b).view(np.int64)
    both = np.stack([a, b], axis=1)
    u, inv = np.unique(both, axis=0, return_inverse=True)
    return [(int(x), int(y)) for x, y in u], inv.reshape(-1)


def arith_int_vec(op, a, a_nulls, b, b_nulls, b_const=0, a_unsigned=False, b_unsigned=False):
    """-> (error: overflow on a non-NULL row, result int64 column, result NULL flags)"""
    nulls = _merge_nulls(np.asarray(a_nulls, bool), None if b is None else np.asarray(b_nulls, bool))
    if len(a) == 0:
        return False, np.zeros(0, np.int64), nulls
    pairs, inv = _pairs(a, b, int(b_const))
    outs = [arith_int(op, x, a_unsigned, y, b_unsigned) for x, y in pairs]
    res_u = np.array([0 if o else r for r, o, _ in outs], dtype=np.int64)
    ovf_u = np.array([o for _, o, _ in outs], dtype=bool)
    ovf = ovf_u[inv]
    return bool((ovf & ~nulls).any()), res_u[inv], nulls


def arith_int_overflow_rows(op, a, b, b_const=0, a_unsigned=False, b_unsigned=False) -> np.ndarray:
    """rows whose result overflows, NULL or not"""
    if len(a) == 0:
        return np.zeros(0, bool)
    pairs, inv = _pairs(a, b, int(b_const))
    return np.array([arith_int(op, x, a_unsigned, y, b_unsigned)[1] for x, y in pairs], dtype=bool)[inv]


def arith_real_vec(op, a, a_nulls, b, b_nulls, b_const=0.0):
    """-> (error, result float64 column, result NULL flags, overflow rows)"""
    nulls = _merge_nulls(np.asarray(a_nulls, bool), None if b is None else np.asarray(b_nulls, bool))
    if len(a) == 0:
        return False, np.zeros(0, np.float64), nulls, np.zeros(0, bool)
    pairs, inv = _pairs(np.asarray(a, np.float64), None if b is None else np.asarray(b, np.float64), f64_bits(float(b_const)))
    outs = [arith_real(op, f64_from_bits(x), f64_from_bits(y)) for x, y in pairs]
    res = np.array([r for r, _ in outs], dtype=np.float64)[inv]
    ovf = np.array([o for _, o in outs], dtype=bool)[inv]
    return bool((ovf & ~nulls).any()), res, nulls, ovf


def int_order_key(words: np.ndarray, unsigned: bool) -> Tuple[np.ndarray, np.ndarray]:
    """(sign class, uint64) per row, lexicographically ordered as the values: negative values are class 0 and their
    words as uint64 ascend with the value; non-negative values are class 1 and their word is the value"""
    w = np.ascontiguousarray(words).view(np.int64)
    cls = np.ones(len(w), np.int8) if unsigned else (w >= 0).astype(np.int8)
    return cls, w.view(np.uint64)


def compare_int_vec(a, a_unsigned, b, b_unsigned) -> np.ndarray:
    """-1 / 0 / 1 per row; b is a column or an int broadcast to every row"""
    if np.isscalar(b) or isinstance(b, int):
        b = np.full(len(a), word(int(b)), np.int64)
    ca, wa = int_order_key(a, a_unsigned)
    cb, wb = int_order_key(b, b_unsigned)
    lt = (ca < cb) | ((ca == cb) & (wa < wb))
    gt = (ca > cb) | ((ca == cb) & (wa > wb))
    return gt.astype(np.int64) - lt.astype(np.int64)


def compare_real_vec(x, y) -> np.ndarray:
    x = np.asarray(x, np.float64)
    y = np.broadcast_to(np.asarray(y, np.float64), x.shape)
    xn, yn = np.isnan(x), np.isnan(y)
    with np.errstate(invalid="ignore"):
        c = (x > y).astype(np.int64) - (x < y).astype(np.int64)
    c = np.where(xn & yn, 0, c)
    c = np.where(xn & ~yn, -1, c)
    return np.where(~xn & yn, 1, c)


def holds_vec(op: int, c: np.ndarray) -> np.ndarray:
    return {CMP_LT: c < 0, CMP_LE: c <= 0, CMP_GT: c > 0, CMP_GE: c >= 0, CMP_EQ: c == 0, CMP_NE: c != 0}[op]


def compare_int_col(op, a, a_nulls, b, b_nulls, b_const=0, a_unsigned=False, b_unsigned=False):
    """tg_vec_compare_int: -> (0/1 int64 column, NULL flags)"""
    nulls = _merge_nulls(np.asarray(a_nulls, bool), None if b is None else np.asarray(b_nulls, bool))
    c = compare_int_vec(a, a_unsigned, b_const if b is None else b, b_unsigned)
    return holds_vec(op, c).astype(np.int64), nulls


def compare_real_col(op, a, a_nulls, b, b_nulls, b_const=0.0):
    nulls = _merge_nulls(np.asarray(a_nulls, bool), None if b is None else np.asarray(b_nulls, bool))
    c = compare_real_vec(a, b_const if b is None else b)
    return holds_vec(op, c).astype(np.int64), nulls


def filter_rows(cols: Sequence[Tuple[np.ndarray, np.ndarray]], items: Sequence, sel: Optional[np.ndarray] = None) -> np.ndarray:
    """tg_vec_filter: `selected` per physical row.  cols[c] = (8-byte values, NULL flags); items are
    tidb_b200.plan.FilterItem; only the rows in `sel` (all rows without it) can be selected."""
    n = len(cols[0][0])
    ok = np.ones(n, bool)
    for it in items:
        lv, ln = cols[it.lhs_col]
        ok &= ~ln
        rv = None
        if it.rhs_col >= 0:
            rv, rn = cols[it.rhs_col]
            ok &= ~rn
        if it.is_real:
            c = compare_real_vec(np.asarray(lv).view(np.float64), it.const_f64 if rv is None else np.asarray(rv).view(np.float64))
        else:
            c = compare_int_vec(lv, it.lhs_unsigned, word(it.const_i64) if rv is None else rv, it.rhs_unsigned)
        ok &= holds_vec(it.op, c)
    if sel is not None:
        keep = np.zeros(n, bool)
        keep[np.asarray(sel, np.int64)] = True
        ok &= keep
    return ok
