"""Plain-Python reference for COUNT, SUM and AVG with DISTINCT, independent of the CUDA code.

Each group keeps the set of its distinct non-NULL argument values, with the semantics of the Go maps the reference's
functions use (aggfuncs/func_count_distinct.go, func_sum.go, func_avg.go):
  - an integer column is keyed on its 64 bits (unsigned columns read as uint64: the same bits);
  - a DOUBLE -0.0 and +0.0 are one value, and NaN != NaN makes every NaN row a new value;
  - a DECIMAL column is handed in as its int64 values at the column's scale (MyDecimal.ToHashKey: 1.50 = 1.5).
Groups are formed as tests/agg_reference.py forms them (NULL is None, a DOUBLE key -0.0 is +0.0).  MIN / MAX ignore the
DISTINCT flag.  Expected values are ints (COUNT, MIN, MAX, FIRSTROW), 40-byte DECIMAL cells from tests/mydecimal_args.py,
agg_reference.Expect for DOUBLE SUM / AVG (the order-free error bound), NAN for a DOUBLE SUM / AVG over a NaN, or None.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence, Tuple

import numpy as np

import agg_reference as R
import mydecimal_args as A
from tidb_b200 import abi

NAN = "NaN"   # expected DOUBLE result: any NaN


def distinct_values(xs: Sequence, is_real: bool) -> list:
    """the distinct values of xs in first-seen order, by Go map semantics"""
    seen, out = set(), []
    for x in xs:
        if is_real:
            if x != x:            # NaN: never found in the map, so every NaN row is inserted and counted
                out.append(x)
                continue
            k = 0.0 if x == 0 else x
        else:
            k = x
        if k not in seen:
            seen.add(k)
            out.append(x)
    return out


def _unsigned(t) -> bool:
    return t.tp not in (abi.TYPE_DOUBLE, abi.TYPE_NEWDECIMAL) and bool(t.flag & abi.FLAG_UNSIGNED)


def _lists(plan, vals) -> Dict[int, Tuple[list, list]]:
    out = {}
    for c, (v, nl) in vals.items():
        v = np.asarray(v)
        if _unsigned(plan.col_types[c]):
            v = v.view(np.uint64)
        out[c] = (v.tolist(), np.asarray(nl, dtype=bool).tolist())
    return out


def group_rows(plan, cols) -> Dict[Tuple, List[int]]:
    n = len(next(iter(cols.values()))[0]) if cols else 0
    if not plan.group_by:
        return {(): list(range(n))}   # no GROUP BY: one group, also over no rows (the default row)
    kv = [R._key_values(*cols[g], plan.col_types[g].tp == abi.TYPE_DOUBLE) for g in plan.group_by]
    groups: Dict[Tuple, List[int]] = {}
    for i, k in enumerate(zip(*kv)):
        groups.setdefault(k, []).append(i)
    return groups


def _one(plan, f, cols, rows, key):
    if f.name == abi.AGG_FIRSTROW:
        return key[plan.group_by.index(f.arg_col)]
    if f.arg_col < 0:
        return len(rows)
    t = plan.col_types[f.arg_col]
    is_real, is_dec = t.tp == abi.TYPE_DOUBLE, t.tp == abi.TYPE_NEWDECIMAL
    v, nl = cols[f.arg_col]
    xs = [v[r] for r in rows if not nl[r]]
    if f.distinct and f.name in (abi.AGG_COUNT, abi.AGG_SUM, abi.AGG_AVG):
        xs = distinct_values(xs, is_real)
    if f.name == abi.AGG_COUNT:
        return len(xs)
    if not xs:
        return None
    if f.name in (abi.AGG_MIN, abi.AGG_MAX):
        pick = min(xs) if f.name == abi.AGG_MIN else max(xs)
        return A.sum_result(pick, t.decimal) if is_dec else pick
    if f.ret_type == abi.TYPE_NEWDECIMAL:
        s = t.decimal if is_dec else 0
        total = sum(xs)
        return A.sum_result(total, s) if f.name == abi.AGG_SUM else A.avg_result(total, len(xs), s, f.ret_frac)
    if any(x != x for x in xs):
        return NAN
    return R._sum_expect(xs, None if f.name == abi.AGG_SUM else len(xs))


def expected(plan, vals) -> Dict[Tuple, list]:
    """vals: {column: (values, nulls)} over every row pushed, in push order.  -> group key tuple -> one expected value per
    function"""
    cols = _lists(plan, vals)
    return {k: [_one(plan, f, cols, rows, k) for f in plan.funcs] for k, rows in group_rows(plan, cols).items()}


def pair_count(plan, vals, col) -> int:
    """the (group, value) pairs a dedup set of column `col` holds: distinct non-NULL, non-NaN values per group"""
    cols = _lists(plan, vals)
    v, nl = cols[col]
    is_real = plan.col_types[col].tp == abi.TYPE_DOUBLE
    return sum(sum(1 for x in distinct_values([v[r] for r in rows if not nl[r]], is_real) if x == x)
               for rows in group_rows(plan, cols).values())


def matches(want, got) -> bool:
    if isinstance(want, R.Expect):
        return want.matches(got)
    if want is NAN:
        return isinstance(got, float) and math.isnan(got)
    if want is None or got is None:
        return want is None and got is None
    return want == got


def check(plan, vals, got_rows) -> int:
    """every result row equals the reference's, group by group (FIRSTROW of each GROUP BY column names the group)"""
    exp = expected(plan, vals)
    got = {}
    for r in got_rows:
        k = R.result_key(plan, r) if plan.group_by else ()
        assert k not in got, f"group {k} emitted twice"
        got[k] = r
    assert set(got) == set(exp), (len(got), len(exp), sorted(set(map(repr, exp)) ^ set(map(repr, got)))[:10])
    for k, ws in exp.items():
        for i, w in enumerate(ws):
            g = got[k][i]
            if plan.funcs[i].name in (abi.AGG_MIN, abi.AGG_MAX, abi.AGG_FIRSTROW) and isinstance(g, int) and _unsigned(plan.col_types[plan.funcs[i].arg_col]):
                g &= R.MASK64
            assert matches(w, g), f"group {k!r} aggregate {i} ({plan.funcs[i]}): got {g!r}, want {w!r}"
    return len(exp)
