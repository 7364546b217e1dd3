"""Exact reference for the hash aggregation, in plain Python and numpy, independent of oracle/agg.cpp.

Groups are formed with a dict over key tuples (NULL is None, -0.0 is +0.0 in DOUBLE keys, unsigned columns read as
uint64).  COUNT, MIN, MAX and FIRSTROW are exact.  SUM and AVG are compared with the exact sum S = math.fsum(x) of a
group's non-NULL arguments through an error bound that holds for ANY summation order (atomics in any order, local
tables merged later, several pushes):

    |got - S| <= gamma(m - 1) * sum(|x_i|) + ulp(S),     gamma(k) = k*u / (1 - k*u),  u = 2**-53

for a group of m non-NULL arguments; AVG gets that bound divided by its count, plus 2 ulp for the division.  A relative
tolerance would mean nothing for a sum that cancels; this bound does not depend on the size of the result.

Final mode (the inputs are partial results): COUNT sums the partial counts, SUM adds the non-NULL partial sums (NULL if
there are none), AVG(count, sum) is sum(sum) / sum(count) over the rows where both are non-NULL, NULL when the counts
add up to 0.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from tidb_b200 import abi

U = 2.0 ** -53
MASK64 = (1 << 64) - 1


def gamma(k: int) -> float:
    return k * U / (1 - k * U) if k > 0 else 0.0


@dataclass
class Expect:
    """expected value of one aggregate in one group: exact (value, tol = None) or within tol of value"""
    value: object
    tol: Optional[float] = None
    real_minmax: bool = False    # MIN/MAX(double): a zero may come back with either sign

    def matches(self, got) -> bool:
        if self.value is None or got is None:
            return self.value is None and got is None
        if self.tol is not None:
            return abs(got - self.value) <= self.tol
        if self.real_minmax and self.value == 0:
            return got == 0
        return got == self.value and type(got) is type(self.value)


def _logical(col, sel):
    data, nulls = col.data, col.nulls()
    if sel is not None:
        data, nulls = data[sel], nulls[sel]
    return data, nulls


def _gather(plan, chunks):
    """the logical rows of every chunk (sel applied), one (values, nulls) pair of Python lists per column"""
    ncols = len(plan.col_types)
    vals: List[list] = [[] for _ in range(ncols)]
    nls: List[list] = [[] for _ in range(ncols)]
    for ch in chunks:
        for c in range(ncols):
            v, nl = _logical(ch.columns[c], ch.sel)
            vals[c].append(v); nls[c].append(nl)
    out = []
    for c, t in enumerate(plan.col_types):
        v = np.concatenate(vals[c]) if vals[c] else np.zeros(0, dtype=np.float64 if t.tp == abi.TYPE_DOUBLE else np.int64)
        nl = np.concatenate(nls[c]) if nls[c] else np.zeros(0, dtype=bool)
        if t.tp != abi.TYPE_DOUBLE and (t.flag & abi.FLAG_UNSIGNED):
            v = v.view(np.uint64)
        out.append((v.tolist(), nl.tolist()))
    return out


def _key_values(v, nl, is_real):
    if is_real:
        v = [0.0 if x == 0 else x for x in v]     # -0.0 and +0.0 are one group key
    return [None if n else x for x, n in zip(v, nl)]


def _sum_expect(xs: list, m_div: Optional[int] = None) -> Expect:
    """SUM (m_div None) or AVG = sum / m_div of the list of float64 arguments"""
    if not xs:
        return Expect(None)
    s = math.fsum(xs)
    err = gamma(len(xs) - 1) * math.fsum(abs(x) for x in xs) + math.ulp(s)
    if m_div is None:
        return Expect(s, err)
    a = s / m_div
    return Expect(a, err / m_div + 2 * math.ulp(a))


def _arg_real(f, cols, rows):
    """per-row float64 arguments of SUM / AVG over `rows`, NULL rows dropped; a fused expression is evaluated with one
    rounding per operation, like the kernel (no fused multiply-add)"""
    a, an = cols[f.arg_col]
    if f.arg_expr == abi.ARGEXPR_COL:
        return [a[r] for r in rows if not an[r]]
    b, bn = cols[f.arg_col2]
    c = float(f.arg_const)
    # Python float arithmetic is IEEE binary64 with one rounding per operation
    if f.arg_expr == abi.ARGEXPR_MUL:
        return [a[r] * b[r] for r in rows if not (an[r] or bn[r])]
    return [a[r] * (c - b[r]) for r in rows if not (an[r] or bn[r])]


def _one(plan, f, cols, rows, key) -> Expect:
    final = f.mode == abi.AGGMODE_FINAL
    if f.name == abi.AGG_COUNT:
        if f.arg_col < 0:
            return Expect(len(rows))
        v, nl = cols[f.arg_col]
        if final:
            return Expect(sum(v[r] for r in rows if not nl[r]))
        return Expect(sum(1 for r in rows if not nl[r]))
    if f.name == abi.AGG_SUM:
        return _sum_expect(_arg_real(f, cols, rows))
    if f.name == abi.AGG_AVG:
        if final:
            c, cn = cols[f.arg_col]
            s, sn = cols[f.arg_col2]
            keep = [r for r in rows if not cn[r] and not sn[r]]
            total = sum(c[r] for r in keep)
            if total == 0:
                return Expect(None)
            return _sum_expect([s[r] for r in keep], total)
        xs = _arg_real(f, cols, rows)
        return _sum_expect(xs, len(xs)) if xs else Expect(None)
    if f.name in (abi.AGG_MIN, abi.AGG_MAX):
        v, nl = cols[f.arg_col]
        xs = [v[r] for r in rows if not nl[r]]
        if not xs:
            return Expect(None)
        pick = min(xs) if f.name == abi.AGG_MIN else max(xs)
        is_real = plan.col_types[f.arg_col].tp == abi.TYPE_DOUBLE
        return Expect(float(pick) if is_real else int(pick), real_minmax=is_real)
    if f.name == abi.AGG_FIRSTROW:
        return Expect(key[plan.group_by.index(f.arg_col)])
    raise ValueError(f"no reference for aggregate {f.name}")


def expected(plan, chunks) -> Dict[Tuple, List[Expect]]:
    """group key tuple (GROUP BY columns in plan order) -> one Expect per aggregate function"""
    cols = _gather(plan, chunks)
    n = len(cols[0][0]) if cols else 0
    groups: Dict[Tuple, List[int]] = {}
    if plan.group_by:
        kv = [_key_values(*cols[g], plan.col_types[g].tp == abi.TYPE_DOUBLE) for g in plan.group_by]
        for i, k in enumerate(zip(*kv)):
            groups.setdefault(k, []).append(i)
    elif n:
        groups[()] = list(range(n))
    else:   # no GROUP BY over no rows: one row of defaults (COUNT 0, everything else NULL)
        return {(): [Expect(0 if f.name == abi.AGG_COUNT else None) for f in plan.funcs]}
    return {k: [_one(plan, f, cols, rows, k) for f in plan.funcs] for k, rows in groups.items()}


def _normalize(plan, f, v):
    """a result value as the reference states it: unsigned integer columns read as uint64"""
    if v is None or f.arg_col < 0 or f.name not in (abi.AGG_MIN, abi.AGG_MAX, abi.AGG_FIRSTROW):
        return v
    t = plan.col_types[f.arg_col]
    if t.tp != abi.TYPE_DOUBLE and (t.flag & abi.FLAG_UNSIGNED):
        return int(v) & MASK64
    if t.tp == abi.TYPE_DOUBLE and f.name == abi.AGG_FIRSTROW and v == 0:
        return 0.0
    return v


def result_key(plan, row) -> Tuple:
    """the group key of a result row, read from its FIRSTROW(group column) outputs"""
    pos = {}
    for i, f in enumerate(plan.funcs):
        if f.name == abi.AGG_FIRSTROW:
            pos.setdefault(f.arg_col, i)
    missing = [g for g in plan.group_by if g not in pos]
    assert not missing, f"the plan needs FIRSTROW of every GROUP BY column to match groups (missing {missing})"
    return tuple(_normalize(plan, plan.funcs[pos[g]], row[pos[g]]) for g in plan.group_by)


def check(plan, chunks, got_rows: Sequence[Tuple]) -> int:
    """assert that the result rows equal the reference, group by group; returns the number of groups"""
    exp = expected(plan, chunks)
    got = {}
    for r in got_rows:
        k = result_key(plan, r)
        assert k not in got, f"group {k} emitted twice"
        got[k] = r
    assert len(got) == len(exp), (len(got), len(exp), sorted(set(map(repr, exp)) ^ set(map(repr, got)))[:10])
    assert set(got) == set(exp), sorted(set(map(repr, exp)) ^ set(map(repr, got)))[:10]
    for k, es in exp.items():
        r = got[k]
        for i, (f, e) in enumerate(zip(plan.funcs, es)):
            v = _normalize(plan, f, r[i])
            assert e.matches(v), f"group {k!r} aggregate {i} (name {f.name}, mode {f.mode}): got {v!r}, want {e.value!r} tol {e.tol!r}"
    return len(exp)
