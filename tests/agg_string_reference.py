"""Exact reference for the hash aggregation with string GROUP BY columns, in plain Python.

Groups are formed over a tuple of group keys: a string column contributes collator.ImmutableKey of its bytes
(codec.go HashGroupKey with new collations enabled): the bytes under binary (63) and utf8mb4_0900_bin (309), the bytes
with trailing 0x20 cut under the PAD collations utf8mb4_bin (46), utf8_bin (83), ascii_bin (65) and latin1_bin (47).
NULL is its own group (None), apart from b"".  Integer and DOUBLE columns contribute their value as agg_reference.py
states it.

FIRSTROW of a string GROUP BY column is firstRow4String with one worker (aggfuncs/func_first_row.go): the raw bytes,
trailing spaces included, of the group's earliest row in push order; within a chunk, logical row order (sel order).
Every other aggregate is agg_reference.py's, over the same groups.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

import agg_reference as R
from tidb_b200 import abi

PAD_COLLATIONS = (46, 83, 65, 47)
BYTE_COLLATIONS = (63, 309)


def collation_key(b: Optional[bytes], collation: int) -> Optional[bytes]:
    """collator.ImmutableKey of one value under an offloaded collation; None stays None (the NULL group)"""
    if b is None:
        return None
    if collation in PAD_COLLATIONS:
        return bytes(b).rstrip(b" ")     # truncateTailingSpace: 0x20 only, a tab is kept
    if collation in BYTE_COLLATIONS:
        return bytes(b)
    raise ValueError(f"collation {collation} is not offloaded")


def is_string(t) -> bool:
    return t.tp in abi.STRING_TYPES


def _logical_rows(col, sel):
    if col.is_varlen:
        vals = col.values()
        if sel is not None:
            vals = [vals[i] for i in sel]
        return vals, [v is None for v in vals]
    data, nulls = col.data, col.nulls()
    if sel is not None:
        data, nulls = data[sel], nulls[sel]
    return data, nulls


def gather(plan, chunks) -> List[Tuple[list, list]]:
    """the logical rows of every chunk in push order, one (values, nulls) pair of lists per column; a string column's
    values are bytes (None where NULL)"""
    out = []
    for c, t in enumerate(plan.col_types):
        vals: list = []
        nls: list = []
        for ch in chunks:
            v, nl = _logical_rows(ch.columns[c], ch.sel)
            if is_string(t):
                vals.extend(v); nls.extend(nl)
            else:
                v = np.asarray(v)
                if t.tp != abi.TYPE_DOUBLE and (t.flag & abi.FLAG_UNSIGNED):
                    v = v.view(np.uint64)
                vals.extend(v.tolist()); nls.extend(np.asarray(nl).tolist())
        out.append((vals, nls))
    return out


def _key_of(plan, cols, g, i):
    t = plan.col_types[g]
    v, nl = cols[g]
    if nl[i]:
        return None
    if is_string(t):
        return collation_key(v[i], t.collation)
    x = v[i]
    return 0.0 if t.tp == abi.TYPE_DOUBLE and x == 0 else x


def expected(plan, chunks) -> Dict[Tuple, List[R.Expect]]:
    """group key tuple (GROUP BY columns in plan order, string keys as collation keys) -> one Expect per function"""
    cols = gather(plan, chunks)
    n = len(cols[0][0]) if cols else 0
    groups: Dict[Tuple, List[int]] = {}
    for i in range(n):
        groups.setdefault(tuple(_key_of(plan, cols, g, i) for g in plan.group_by), []).append(i)
    out = {}
    for k, rows in groups.items():
        es = []
        for f in plan.funcs:
            if f.name == abi.AGG_FIRSTROW and is_string(plan.col_types[f.arg_col]):
                v, nl = cols[f.arg_col]
                es.append(R.Expect(None if nl[rows[0]] else bytes(v[rows[0]])))   # the earliest row, raw bytes
            else:
                es.append(R._one(plan, f, cols, rows, k))
        out[k] = es
    return out


def result_key(plan, row) -> Tuple:
    """the group key of a result row, from its FIRSTROW(group column) outputs"""
    pos = {}
    for i, f in enumerate(plan.funcs):
        if f.name == abi.AGG_FIRSTROW:
            pos.setdefault(f.arg_col, i)
    missing = [g for g in plan.group_by if g not in pos]
    assert not missing, f"the plan needs FIRSTROW of every GROUP BY column to match groups (missing {missing})"
    key = []
    for g in plan.group_by:
        t, v = plan.col_types[g], row[pos[g]]
        if is_string(t):
            key.append(collation_key(v, t.collation))
        else:
            key.append(R._normalize(plan, plan.funcs[pos[g]], v))
    return tuple(key)


def check(plan, chunks, got_rows: Sequence[Tuple]) -> int:
    """assert that the result rows equal the reference, group by group; returns the number of groups"""
    exp = expected(plan, chunks)
    got = {}
    for r in got_rows:
        k = result_key(plan, r)
        assert k not in got, f"group {k!r} emitted twice"
        got[k] = r
    assert set(got) == set(exp), sorted(set(map(repr, exp)) ^ set(map(repr, got)))[:10]
    for k, es in exp.items():
        r = got[k]
        for i, (f, e) in enumerate(zip(plan.funcs, es)):
            v = r[i]
            if not (f.name == abi.AGG_FIRSTROW and is_string(plan.col_types[f.arg_col])):
                v = R._normalize(plan, f, v)
            assert e.matches(v), f"group {k!r} aggregate {i} (name {f.name}): got {v!r}, want {e.value!r} tol {e.tol!r}"
    return len(exp)
