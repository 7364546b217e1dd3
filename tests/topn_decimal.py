"""Test-only reference: oracle/topn.py's TopN order extended with a "decimal" kind, 40-byte MyDecimal cells compared as
cmpMyDecimal (pkg/util/chunk/compare.go:120) -> MyDecimal.Compare (pkg/types/mydecimal.go:1623).  Every other kind is
oracle/topn.py's, unchanged.

Two forms of the same order, as in oracle/topn.py: topn_rows (a comparator over Python values, the definition; DECIMAL
values are the cells as bytes) and topn_order / item_keys (numpy keys; a DECIMAL key is a dense rank over the column's
distinct values).  Both sort stably, so on the same input they return the same rows in the same order;
tests/test_topn_decimal_reference.py checks that on the edge set and pins cmp_decimal with TestCompareMyDecimal
(pkg/types/mydecimal_test.go:520) and hand cases.
"""
from __future__ import annotations

import functools
import os
import struct
import sys
from typing import List, Sequence, Tuple

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import topn as OT   # noqa: E402

# ---- DECIMAL: 40-byte MyDecimal cells (types/mydecimal.go:236-248): int8 digitsInt, int8 digitsFrac, int8 resultFrac,
# bool negative, int32 wordBuf[9] in base 10^9 (ceil(digitsInt / 9) integer words, then ceil(digitsFrac / 9) fraction words)
DEC_BASE = 10 ** 9


def _dec_parts(cell):
    """(negative, integer words, fraction words) of a well-formed cell"""
    b = bytes(cell)
    di, df, _rf, neg = struct.unpack_from("<bbbB", b, 0)
    words = struct.unpack_from("<9i", b, 4)
    wi, wf = (di + 8) // 9, (df + 8) // 9
    assert di >= 0 and df >= 0 and wi + wf <= 9 and all(0 <= w < DEC_BASE for w in words[:wi + wf]), "malformed cell"
    return bool(neg), list(words[:wi]), list(words[wi:wi + wf])


def cmp_decimal(a, b) -> int:
    """MyDecimal.Compare: the sign first (a negative zero is below +0 and above every negative value), then doSub
    (mydecimal.go:1726): leading zero integer words and trailing zero fraction words dropped, the longer integer part is
    larger, else the first differing word decides, and the side with words left over is larger"""
    na, ia, fa = _dec_parts(a)
    nb, ib, fb = _dec_parts(b)
    if na != nb:
        return -1 if na else 1
    while ia and ia[0] == 0:
        ia = ia[1:]
    while ib and ib[0] == 0:
        ib = ib[1:]
    if len(ia) != len(ib):
        c = -1 if len(ia) < len(ib) else 1
    else:
        while fa and fa[-1] == 0:
            fa = fa[:-1]
        while fb and fb[-1] == 0:
            fb = fb[:-1]
        x, y = ia + fa, ib + fb
        k = 0
        while k < len(x) and k < len(y) and x[k] == y[k]:
            k += 1
        if k < len(x) and k < len(y):
            c = -1 if x[k] < y[k] else 1
        else:
            c = 0 if len(x) == len(y) else (-1 if len(x) < len(y) else 1)
    return -c if na else c


def decimal_dense_rank(cells: np.ndarray, nulls: np.ndarray) -> np.ndarray:
    """uint64 dense rank of each non-NULL cell over the column's distinct values, in Compare's order: rows sort by
    (sign class, signed aligned words), where the 9 integer word slots are right-aligned and the 9 fraction word slots
    left-aligned on the point.  NULL rows get 0 (callers key NULLs separately)."""
    n = len(cells)
    w = np.ascontiguousarray(cells).reshape(n, 40).view(np.int32).astype(np.int64)       # (n, 10)
    live = ~np.asarray(nulls, bool)
    hdr = w[:, 0]
    di, df = ((hdr & 0xFF) ^ 0x80) - 0x80, (((hdr >> 8) & 0xFF) ^ 0x80) - 0x80
    neg = ((hdr >> 24) & 0xFF) != 0
    wi, wf = (di + 8) // 9, (df + 8) // 9
    ok = (di >= 0) & (df >= 0) & (wi + wf <= 9)
    for j in range(9):
        ok &= (j >= wi + wf) | ((w[:, 1 + j] >= 0) & (w[:, 1 + j] < DEC_BASE))
    assert ok[live].all(), "malformed cell"
    wi, wf = np.where(live, wi, 0), np.where(live, wf, 0)
    aligned = np.zeros((n, 18), np.int64)
    rows = np.arange(n)
    for j in range(9):
        used = live & (j < wi + wf)
        slot = np.where(j < wi, 9 - wi + j, 9 + j - wi)
        aligned[rows[used], slot[used]] = w[used, 1 + j]
    aligned[neg] = -aligned[neg]
    key = np.concatenate([(~neg).astype(np.int64)[:, None], aligned], axis=1)
    key[~live] = 0
    order = np.lexsort(key.T[::-1])
    ks = key[order]
    rank = np.empty(n, np.uint64)
    rank[order] = np.cumsum(np.r_[False, (ks[1:] != ks[:-1]).any(axis=1)]).astype(np.uint64)
    return np.where(live, rank, np.uint64(0))


def cmp_value(a, b, kind: str) -> int:
    return cmp_decimal(a, b) if kind == "decimal" else OT._cmp_value(a, b, kind)


def topn_rows(rows: Sequence[Tuple], kinds: Sequence[str], by_items: Sequence[Tuple[int, bool]], offset: int, count: int) -> List[Tuple]:
    """oracle/topn.py topn_rows with kinds[c] = "decimal" allowed (values: 40-byte cells)"""
    def cmp_rows(x, y):
        for col, desc in by_items:
            a, b = x[col], y[col]
            if a is None or b is None:
                c = 0 if (a is None and b is None) else (-1 if a is None else 1)     # cmpNull
            else:
                if kinds[col] == "uint":
                    a, b = a % (1 << 64), b % (1 << 64)
                c = cmp_value(a, b, kinds[col])
            if desc:
                c = -c
            if c:
                return c
        return 0
    return sorted(rows, key=functools.cmp_to_key(cmp_rows))[offset:offset + count]


def order_key(values: np.ndarray, nulls: np.ndarray, kind: str, desc: bool) -> Tuple[np.ndarray, np.ndarray]:
    """oracle/topn.py order_key with a "decimal" kind: the value key is a dense rank over the given cells, so keys of
    different row sets compare only for the same set"""
    if kind != "decimal":
        return OT.order_key(values, nulls, kind, desc)
    nl = np.asarray(nulls, bool)
    k = decimal_dense_rank(values, nl)
    nk = (~nl).astype(np.uint8)                                # NULL first
    if desc:
        return (1 - nk).astype(np.uint8), ~k
    return nk, k


def topn_order(cols, kinds, by_items, offset: int, count: int) -> np.ndarray:
    """row indices of rows [offset, offset + count) in ORDER BY order (stable).  cols[c] = (8-byte values or (n, 40) uint8
    DECIMAL cells, NULL flags)."""
    keys = []
    for col, desc in by_items:
        keys.extend(order_key(cols[col][0], cols[col][1], kinds[col], desc))
    order = np.lexsort(keys[::-1]) if keys else np.arange(len(cols[0][0]))
    return order[offset:offset + count]


def item_keys(cols, kinds, by_items, rows: np.ndarray) -> np.ndarray:
    """the ORDER BY key of the given rows as an (len(rows), 2 * items) uint64 matrix: equal rows = equal keys.  A DECIMAL
    item is ranked over the whole column, so the keys of any two row sets compare."""
    out = []
    for col, desc in by_items:
        if kinds[col] == "decimal":
            nk, k = order_key(cols[col][0], cols[col][1], kinds[col], desc)
            nk, k = nk[rows], k[rows]
        else:
            nk, k = order_key(cols[col][0][rows], cols[col][1][rows], kinds[col], desc)
        out += [nk.astype(np.uint64), k]
    return np.stack(out, axis=1) if out else np.zeros((len(rows), 0), np.uint64)
