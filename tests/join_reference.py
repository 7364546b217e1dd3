"""Exact, vectorized reference of the hash join for all seven join types, fast enough for tens of millions of rows.

A restatement of the semantics tests/nested_loop.py pins, written with numpy instead of a nested loop (and independently of
oracle/join.cpp):
  * a row whose filter fails, or with a NULL in any key column, has no key and never matches;
  * mixed signed / unsigned key columns compare by value: a negative signed key never equals an unsigned one;
  * FLOAT and DOUBLE keys compare as float64 values (a FLOAT key is float64(f32): 0.1f != 0.1, 0.5f == 0.5), -0 == +0;
  * DATE / DATETIME / TIMESTAMP keys ignore the low 4 bits (type / fsp) of the CoreTime word;
  * several key columns match iff every column matches;
  * filters and OtherCondition are CNF lists compared as FilterItem / OtherCond say (signed / unsigned per operand), and an
    item with a NULL operand fails.

The build keys are sorted, each probe row finds its match range with searchsorted, duplicates expand with np.repeat, the
OtherCondition runs on the candidate pairs, and outer padding, semi, anti and the left outer semi flag follow from the per
probe row pass counts; the build-side rows of the outer / semi / anti joins whose outer side is the build side follow from
bincount marks over the passing pairs.

Several key columns are matched through a 64-bit mix of their values (not the library's mix), and every candidate pair is
then checked column by column, so a collision of the mix never adds a row.

Results are lists of (values, nulls) per output column; assert_same_rows compares two of them as multisets of rows, where
NULL != 0 and FLOAT / DOUBLE / DECIMAL cells compare by their bits.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from tidb_b200 import abi
from tidb_b200.executor import np_dtype_of
from tidb_b200.plan import JoinPlan

TIME_TYPES = (abi.TYPE_DATE, abi.TYPE_DATETIME, abi.TYPE_TIMESTAMP)
REAL_TYPES = (abi.TYPE_FLOAT, abi.TYPE_DOUBLE)
Cols = List[Tuple[np.ndarray, np.ndarray]]


def flatten(chunks, types) -> Cols:
    """the logical rows of a list of chunks (sel applied) as one (values, nulls) pair per column"""
    out = []
    for c, t in enumerate(types):
        vals, nls = [], []
        for ch in chunks:
            col = ch.columns[c]
            idx = ch.sel if ch.sel is not None else slice(None)
            vals.append(col.data[idx])
            nls.append(col.nulls()[idx] if col.null_bitmap is not None else np.zeros(len(col.data[idx]), dtype=bool))
        if not vals:
            dt = np_dtype_of(t)
            vals, nls = [np.zeros((0,) + np.dtype(dt).shape, dtype=np.dtype(dt).base)], [np.zeros(0, dtype=bool)]
        out.append((np.concatenate(vals), np.concatenate(nls)))
    return out


def key_unsigned(t) -> bool:
    if t.tp == abi.TYPE_YEAR:
        return True
    if t.tp == abi.TYPE_DURATION:
        return False
    return t.unsigned


# ---- compares (types.CompareInt / cmp.Compare) ----------------------------------------------------------------
def cmp_int(a, ua: bool, b, ub: bool) -> np.ndarray:
    """-1 / 0 / 1 of two int64 arrays (or scalars) read as signed or unsigned values"""
    a = np.asarray(a, dtype=np.int64)
    b = np.asarray(b, dtype=np.int64)
    a, b = np.broadcast_arrays(a, b)
    if ua and ub:
        x, y = a.view(np.uint64), b.view(np.uint64)
        return np.where(x < y, -1, np.where(x == y, 0, 1))
    r = np.where(a < b, -1, np.where(a == b, 0, 1))
    if ua:       # a unsigned, b signed: a >= 2^63 or b < 0 means a > b
        r = np.where((a < 0) | (b < 0), 1, r)
    elif ub:
        r = np.where((a < 0) | (b < 0), -1, r)
    return r


def cmp_real(a, b) -> np.ndarray:
    a, b = np.broadcast_arrays(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64))
    return np.where(a < b, -1, np.where(a > b, 1, 0))


def apply_cmp(op: int, r: np.ndarray) -> np.ndarray:
    return {abi.CMP_LT: r < 0, abi.CMP_LE: r <= 0, abi.CMP_GT: r > 0, abi.CMP_GE: r >= 0,
            abi.CMP_EQ: r == 0, abi.CMP_NE: r != 0}[op]


def filter_pass(cols: Cols, items) -> np.ndarray:
    n = len(cols[0][0]) if cols else 0
    ok = np.ones(n, dtype=bool)
    for it in items:
        a, an = cols[it.lhs_col]
        if it.rhs_col >= 0:
            b, bn = cols[it.rhs_col]
        else:
            b, bn = (it.const_f64 if it.is_real else it.const_i64), np.zeros(n, dtype=bool)
        r = cmp_real(a, b) if it.is_real else cmp_int(a, it.lhs_unsigned, b, it.rhs_unsigned)
        ok &= ~an & ~bn & apply_cmp(it.op, r)
    return ok


# ---- keys ---------------------------------------------------------------------------------------------------------
def key_word(vals: np.ndarray, t) -> np.ndarray:
    """one int64 word per row that is equal for two rows iff their keys are equal (within one key column pair)"""
    if t.tp in REAL_TYPES:
        f = vals.astype(np.float64)
        return np.where(f == 0, 0.0, f).view(np.int64)
    if t.tp in TIME_TYPES:
        return vals.view(np.int64) & ~np.int64(0xF)
    return vals.view(np.int64)


def side_keys(cols: Cols, types, keys: Sequence[int], other_types, other_keys, passed: np.ndarray):
    """(valid, words[nkeys, n]) of one side: valid = filter passed, no NULL key column, no negative signed value against
    an unsigned key column"""
    valid = passed.copy()
    words = []
    for c, oc in zip(keys, other_keys):
        v, nl = cols[c]
        w = key_word(v, types[c])
        valid &= ~nl
        if types[c].tp not in REAL_TYPES + TIME_TYPES and key_unsigned(other_types[oc]) and not key_unsigned(types[c]):
            valid &= w >= 0
        words.append(w)
    return valid, words


def row_key(words):
    """one int64 per row for the match search: the word itself for one key column; for several, a mix of the words (any
    two equal tuples get equal mixes; the pairs a collision of the mix adds are removed by join_pairs)"""
    if len(words) == 1:
        return words[0]
    h = np.zeros(len(words[0]), dtype=np.uint64)
    with np.errstate(over="ignore"):
        for w in words:
            h ^= w.view(np.uint64)
            h *= np.uint64(0xD6E8FEB86659FD93)
            h ^= h >> np.uint64(32)
    return h.view(np.int64)


def other_pass(plan: JoinPlan, L: Cols, R: Cols, li: np.ndarray, ri: np.ndarray) -> np.ndarray:
    ok = np.ones(len(li), dtype=bool)
    for it in plan.other_cond or []:
        def operand(side, col):
            v, nl = (L if side == 0 else R)[col]
            idx = li if side == 0 else ri
            return v[idx], nl[idx]
        a, an = operand(it.lhs_side, it.lhs_col)
        if it.rhs_side >= 0:
            b, bn = operand(it.rhs_side, it.rhs_col)
        else:
            b, bn = (it.const_f64 if it.is_real else it.const_i64), np.zeros(len(li), dtype=bool)
        r = cmp_real(a, b) if it.is_real else cmp_int(a, it.lhs_unsigned, b, it.rhs_unsigned)
        ok &= ~an & ~bn & apply_cmp(it.op, r)
    return ok


# ---- the join -------------------------------------------------------------------------------------------------------
def join_pairs(plan: JoinPlan, L: Cols, R: Cols):
    """(li, ri) of every (left row, right row) pair with equal keys that passes the OtherCondition"""
    lf = plan.probe_filter if plan.build_is_right else plan.build_filter
    rf = plan.build_filter if plan.build_is_right else plan.probe_filter
    lvalid, lw = side_keys(L, plan.left_types, plan.left_keys, plan.right_types, plan.right_keys, filter_pass(L, lf))
    rvalid, rw = side_keys(R, plan.right_types, plan.right_keys, plan.left_types, plan.left_keys, filter_pass(R, rf))
    lk, rk = row_key(lw), row_key(rw)
    (bk, bvalid), (pk, pvalid) = ((rk, rvalid), (lk, lvalid)) if plan.build_is_right else ((lk, lvalid), (rk, rvalid))
    brows = np.nonzero(bvalid)[0]
    order = np.argsort(bk[brows], kind="stable")
    sb, srow = bk[brows][order], brows[order]
    prows = np.nonzero(pvalid)[0]
    # search in key order (sorted needles walk the sorted keys once), then put the ranges back in row order
    porder = np.argsort(pk[prows])
    needles = pk[prows][porder]
    lo, cnt = np.empty(len(prows), np.int64), np.empty(len(prows), np.int64)
    lo[porder] = np.searchsorted(sb, needles, "left")
    cnt[porder] = np.searchsorted(sb, needles, "right")
    cnt -= lo
    total = int(cnt.sum())
    prep = np.repeat(prows, cnt)
    start = np.cumsum(cnt) - cnt
    pos = np.arange(total, dtype=np.int64) - np.repeat(start - lo, cnt)
    brep = srow[pos]
    li, ri = (prep, brep) if plan.build_is_right else (brep, prep)
    if len(lw) > 1:
        ok = np.ones(len(li), dtype=bool)
        for a, b in zip(lw, rw):
            ok &= a[li] == b[ri]
        li, ri = li[ok], ri[ok]
    if plan.other_cond:
        ok = other_pass(plan, L, R, li, ri)
        li, ri = li[ok], ri[ok]
    return li, ri


def _gather(vals, nulls, idx):
    """rows idx of a column; idx < 0 = a NULL-padded row"""
    pad = idx < 0
    j = np.where(pad, 0, idx)
    if len(vals) == 0:
        v = np.zeros((len(idx),) + vals.shape[1:], dtype=vals.dtype)
        return v, np.ones(len(idx), dtype=bool)
    v = vals[j].copy()
    v[pad] = 0
    return v, nulls[j] | pad


def join_reference(plan: JoinPlan, left, right, flat: bool = False):
    """the result of `plan` over the chunk lists left / right (flat=True: already flattened Cols) as (values, nulls) per
    output column"""
    L = left if flat else flatten(left, plan.left_types)
    R = right if flat else flatten(right, plan.right_types)
    nl, nr = len(L[0][0]), len(R[0][0])
    li, ri = join_pairs(plan, L, R)
    jt = plan.join_type
    flag = None
    if jt == abi.JOIN_INNER:
        pass
    elif jt == abi.JOIN_LEFT_OUTER:
        miss = np.nonzero(np.bincount(li, minlength=nl) == 0)[0]
        li, ri = np.concatenate([li, miss]), np.concatenate([ri, np.full(len(miss), -1, np.int64)])
    elif jt == abi.JOIN_RIGHT_OUTER:
        miss = np.nonzero(np.bincount(ri, minlength=nr) == 0)[0]
        li, ri = np.concatenate([li, np.full(len(miss), -1, np.int64)]), np.concatenate([ri, miss])
    elif jt in (abi.JOIN_SEMI, abi.JOIN_ANTI_SEMI):
        hit = np.bincount(li, minlength=nl) > 0
        li = np.nonzero(hit if jt == abi.JOIN_SEMI else ~hit)[0]
        ri = np.full(len(li), -1, np.int64)
    elif jt in (abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI):
        hit = np.bincount(li, minlength=nl) > 0
        flag = (hit != (jt == abi.JOIN_ANTI_LEFT_OUTER_SEMI)).astype(np.int64)
        li = np.arange(nl, dtype=np.int64)
        ri = np.full(nl, -1, np.int64)
    else:
        raise ValueError("join type")
    lu = plan.lused if plan.lused is not None else list(range(len(plan.left_types)))
    ru = plan.rused if plan.rused is not None else list(range(len(plan.right_types)))
    out = [_gather(*L[c], li) for c in lu] + [_gather(*R[c], ri) for c in ru]
    if flag is not None:
        out.append((flag, np.zeros(len(flag), dtype=bool)))
    return out


# ---- comparison -------------------------------------------------------------------------------------------------------
def _words(vals: np.ndarray) -> np.ndarray:
    """the bits of a column as int64 words, [n, w]"""
    v = np.ascontiguousarray(vals)
    if v.dtype.itemsize == 4 and v.ndim == 1:
        return v.view(np.uint32).astype(np.int64)[:, None]
    return v.reshape(len(v), -1).view(np.int64) if v.ndim == 2 else v.view(np.int64)[:, None]


def canonical(cols: Cols) -> np.ndarray:
    """rows as an int64 matrix (a word of NULL flags, then every column's value words, zero under NULL), in an order that
    only depends on the multiset of rows"""
    if not cols:
        return np.zeros((0, 0), dtype=np.int64)
    n = len(cols[0][1])
    words = [_words(v) for v, _ in cols]
    m = np.empty((n, 1 + sum(w.shape[1] for w in words)), dtype=np.int64)
    mask = np.zeros(n, dtype=np.int64)
    h = np.zeros(n, dtype=np.uint64)
    j = 1
    with np.errstate(over="ignore"):
        for c, ((_, nl), w) in enumerate(zip(cols, words)):
            nl = np.asarray(nl, dtype=bool)
            mask |= nl.astype(np.int64) << c
            for k in range(w.shape[1]):
                x = np.where(nl, 0, w[:, k])
                m[:, j] = x
                j += 1
                h ^= x.view(np.uint64)
                h *= np.uint64(0x9E3779B97F4A7C15)
                h ^= h >> np.uint64(29)
        m[:, 0] = mask
        h ^= mask.view(np.uint64)
        h *= np.uint64(0xBF58476D1CE4E5B9)
    return m[np.argsort(h)]


def assert_same_rows(want: Cols, got: Cols, what: str = "") -> None:
    assert len(want) == len(got), f"{what}: {len(got)} output columns, expected {len(want)}"
    w, g = canonical(want), canonical(got)
    assert w.shape == g.shape, f"{what}: {g.shape[0]} rows, expected {w.shape[0]}"
    bad = np.nonzero((w != g).any(axis=1))[0] if len(w) else []
    assert len(bad) == 0, f"{what}: {len(bad)} rows differ; first got {g[bad[0]].tolist()}, expected {w[bad[0]].tolist()}"


def to_rows(cols: Cols) -> list:
    """(values, nulls) columns -> row tuples with None for NULL (for comparing with nested_loop_join)"""
    if not cols:
        return []
    n = len(cols[0][0])
    pyc = [[None if nl[i] else (v[i].tobytes() if v.ndim == 2 else v[i].item()) for i in range(n)] for v, nl in cols]
    return list(zip(*pyc))
