"""TEST INFRASTRUCTURE (oracle): CPU restatement of TopNExec's row order, used only by tests/.

Follows pkg/executor/sortexec/topn.go: rows are compared item by item with the column type's CompareFunc
(pkg/util/chunk/compare.go:64 cmpNull — NULL before every value; :74 cmpInt64, :82 cmpUint64, :112 cmpFloat64 = Go
cmp.Compare, NaN before everything, -0 == +0; :129 cmpTime -> types/core_time.go:256 compareTime, which compares the
calendar fields and the microseconds, not the fsp / type bits) and DESC negates the comparison (topn.go:157
greaterRow); the result is rows [offset, offset + count) of that order (topn.go:285 heap of offset+count rows, :346
final sort).  Ties keep no particular order in the reference (heap), so callers compare the ORDER BY columns of tied
rows, not their identity.
Parity pinning: no golden vectors exist in the reference for TopN beyond SQL results on tiny tables
(tests/integrationtest/r/executor/sort.result-style); pinned by this restatement + the hand cases in
tests/test_vec_topn_reference.py.

Two forms of the same order: topn_rows (a comparator over Python values, the definition) and topn_order (a numpy key
transform for inputs where a Python comparator is too slow).  Both sort stably, so on the same input they return the
same rows in the same order; tests/test_vec_topn_reference.py checks that on the edge set.
"""
from __future__ import annotations

import functools
import math
from typing import List, Sequence, Tuple

import numpy as np

# packed CoreTime (pkg/types/time.go:235-251): (name, bit offset, width), most significant first; bits 0..3 are fspTt
TIME_FIELDS = (("year", 50, 14), ("month", 46, 4), ("day", 41, 5), ("hour", 36, 5), ("minute", 30, 6),
               ("second", 24, 6), ("microsecond", 4, 20))


def pack_time(year, month, day, hour=0, minute=0, second=0, microsecond=0, fsp_tt=0) -> int:
    """the uint64 word of a types.Time (as an unsigned Python int)"""
    w = fsp_tt & 0xF
    for (_, off, width), v in zip(TIME_FIELDS, (year, month, day, hour, minute, second, microsecond)):
        assert 0 <= v < (1 << width)
        w |= v << off
    return w


def time_fields(w: int) -> dict:
    w %= 1 << 64
    return {name: (w >> off) & ((1 << width) - 1) for name, off, width in TIME_FIELDS}


def _cmp_time(a: int, b: int) -> int:
    """compareTime: datetimeToUint64 (core_time.go:354), then the microseconds"""
    def key(w):
        f = time_fields(w)
        return (f["year"] * 10**10 + f["month"] * 10**8 + f["day"] * 10**6 + f["hour"] * 10**4 + f["minute"] * 100 + f["second"],
                f["microsecond"])
    ka, kb = key(a), key(b)
    return -1 if ka < kb else (1 if ka > kb else 0)


def _cmp_value(a, b, kind: str) -> int:
    if kind == "real":          # Go cmp.Compare on float64: NaN < everything, NaN == NaN
        an, bn = isinstance(a, float) and math.isnan(a), isinstance(b, float) and math.isnan(b)
        if an or bn:
            return 0 if (an and bn) else (-1 if an else 1)
    if kind == "time":
        return _cmp_time(a, b)
    return -1 if a < b else (1 if a > b else 0)


def topn_rows(rows: Sequence[Tuple], kinds: Sequence[str], by_items: Sequence[Tuple[int, bool]], offset: int, count: int) -> List[Tuple]:
    """rows: tuples with None for NULL; kinds[c] in {"int", "uint", "real", "time"}; by_items: (column, desc).
    "uint" and "time" values may be given as int64 bit patterns."""
    def cmp_rows(x, y):
        for col, desc in by_items:
            a, b = x[col], y[col]
            if a is None or b is None:
                c = 0 if (a is None and b is None) else (-1 if a is None else 1)     # cmpNull
            else:
                if kinds[col] == "uint":
                    a, b = a % (1 << 64), b % (1 << 64)
                c = _cmp_value(a, b, kinds[col])
            if desc:
                c = -c
            if c:
                return c
        return 0
    ordered = sorted(rows, key=functools.cmp_to_key(cmp_rows))
    return ordered[offset:offset + count]


def order_key(values: np.ndarray, nulls: np.ndarray, kind: str, desc: bool) -> Tuple[np.ndarray, np.ndarray]:
    """(null key, value key) arrays whose ascending lexicographic order is the item's order; equal keys = equal values"""
    w = np.ascontiguousarray(values).view(np.uint64).copy()
    if kind == "int":
        k = w ^ np.uint64(1 << 63)
    elif kind == "uint":
        k = w
    elif kind == "time":
        k = w & np.uint64(~0xF & ((1 << 64) - 1))
    elif kind == "real":
        x = np.ascontiguousarray(values).view(np.float64)
        w[np.isnan(x)] = np.uint64(0xFFF8000000000000)        # every NaN: one value below -Inf
        w[x == 0.0] = np.uint64(0)                            # -0 == +0
        neg = (w >> np.uint64(63)) == np.uint64(1)
        k = np.where(neg, ~w, w | np.uint64(1 << 63))
    else:
        raise ValueError(kind)
    nk = (~np.asarray(nulls, bool)).astype(np.uint8)          # NULL first
    k = np.where(np.asarray(nulls, bool), np.uint64(0), k)
    if desc:
        return (1 - nk).astype(np.uint8), ~k
    return nk, k


def topn_order(cols: Sequence[Tuple[np.ndarray, np.ndarray]], kinds: Sequence[str], by_items: Sequence[Tuple[int, bool]],
               offset: int, count: int) -> np.ndarray:
    """row indices of rows [offset, offset + count) in ORDER BY order (stable: ties keep input order).
    cols[c] = (8-byte values, NULL flags)."""
    keys = []
    for col, desc in by_items:
        keys.extend(order_key(cols[col][0], cols[col][1], kinds[col], desc))
    order = np.lexsort(keys[::-1]) if keys else np.arange(len(cols[0][0]))
    return order[offset:offset + count]


def item_keys(cols, kinds, by_items, rows: np.ndarray) -> np.ndarray:
    """the ORDER BY key of the given rows as an (len(rows), 2 * items) uint64 matrix: equal rows = equal keys"""
    out = []
    for col, desc in by_items:
        nk, k = order_key(cols[col][0][rows], cols[col][1][rows], kinds[col], desc)
        out += [nk.astype(np.uint64), k]
    return np.stack(out, axis=1) if out else np.zeros((len(rows), 0), np.uint64)
