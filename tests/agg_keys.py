"""Keys that land where a test wants them in the GPU hash aggregation's tables, and a model of how those tables grow.

A restatement of the aggregation's slot functions (tidb_b200/csrc/agg.cu, agg_update.cuh) on top of tests/join_keys.py's
hash64, hash64_inv and slot32:
  agg_home(k, n)      = slot32(hash64(k), n)                       a single-column key's home in the group table
  local_home(k, ls)   = slot32(hash64(k) * LOCAL_MUL, ls)          its home in k_agg_update2's CTA-local table
  key_words(row)      = load_key_words: one word per column (NULL as 0, DOUBLE -0 as +0), then the NULL-bits word when
                        a column is nullable; a DISTINCT set's key appends the value word
  hash_words(w)       = h = hash64(w0), then h = hash64(h ^ (w_j * WORD_MUL + j)) for j >= 1: the home (slot32) and the
                        tag (h | 3) of a multi-column row or a DISTINCT pair
A home depends only on the top 32 bits of its hash, and hash64 is a bijection, so keys whose hashes share those bits
share a home at every table size: top_keys() makes them.  Every step of hash_words inverts (WORD_MUL is odd), so a row
can be solved for any hash through one of its BIGINT columns: solve_column().

The growth model restates grow_and_retry: a round gives up on an item after MAX_PROBE steps; when the table stays at most
a quarter full once the deferred items join (long_run_not_full), the next round walks without that limit, else the
table grows to grown_slots().
"""
from __future__ import annotations

import math
import struct
from typing import Dict, List, Optional, Sequence, Tuple

from join_keys import M64, SENTINEL, hash64, hash64_inv, i64, slot32, u64

MAX_PROBE = 48                       # kAggMaxProbe
LOCAL_MUL = 0xD6E8FEB86659FD93       # k_agg_update2's second multiply for the CTA-local home
WORD_MUL = 0xD6E8FEB86659FD93        # hash_words' multiplier of key words
WORD_MUL_INV = pow(WORD_MUL, -1, 1 << 64)
LOCAL_MUL_INV = pow(LOCAL_MUL, -1, 1 << 64)
NEG_ZERO = 0x8000000000000000
MAX_SLOTS = (1 << 32) - 1            # alloc_table refuses 2^32 slots


# ---- single-column keys -------------------------------------------------------------------------------------------
def agg_home(k: int, nslots: int) -> int:
    return slot32(hash64(k), nslots)


def local_home(k: int, ls: int) -> int:
    return slot32((hash64(k) * LOCAL_MUL) & M64, ls)


def top32(k: int) -> int:
    return hash64(k) >> 32


def top_keys(n: int, top: int, low0: int = 0) -> List[int]:
    """n distinct BIGINT keys (int64; the same bits are the BIGINT UNSIGNED key) whose hash64 has the top 32 bits `top`:
    one home at every table size.  The INT64_MIN sentinel, which lives in a side slot, is skipped."""
    out, low = [], low0
    while len(out) < n:
        k = hash64_inv((top << 32) | (low & 0xFFFFFFFF))
        low += 1
        if k != SENTINEL:
            out.append(k)
    return out


def window_keys(n: int, top: int, width: int) -> List[int]:
    """n distinct BIGINT keys with top 32 hash bits spread over [top, top + width): homes within a short window"""
    return [hash64_inv((((top + j % width) & 0xFFFFFFFF) << 32) | (j // width)) for j in range(n)]


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def bits_f64(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", u64(b)))[0]


def double_key_bits(x: float) -> int:
    """the word a DOUBLE group key is hashed as: its bits, with -0 as +0"""
    return 0 if x == 0 else f64_bits(x)


def top_doubles(n: int, top: int) -> List[float]:
    """n distinct DOUBLE keys whose hash has the top 32 bits `top`: preimages that are finite, not NaN and not -0 (a -0
    key is hashed as +0), found by trying further low hash bits"""
    out, low = [], 0
    while len(out) < n:
        b = u64(hash64_inv((top << 32) | low))
        low += 1
        if (b >> 52) & 0x7FF == 0x7FF or b == NEG_ZERO:
            continue
        out.append(bits_f64(b))
    return out


def local_top_keys(n: int, top: int = 0xFFFFFFFF) -> List[int]:
    """n distinct BIGINT keys that share one CTA-local home at every local table size: top 32 bits of hash64(k) * LOCAL_MUL
    equal `top` (0xFFFFFFFF: the last slot, so their run wraps at ls).  Their global homes are spread."""
    out, low = [], 0
    while len(out) < n:
        k = hash64_inv(((((top << 32) | low) * LOCAL_MUL_INV) & M64))
        low += 1
        if k != SENTINEL:
            out.append(k)
    return out


def outside_window(keys, tops: Sequence[Tuple[int, int]], min_slots: int, margin: int = 64):
    """boolean mask (numpy) of the keys whose home stays at least `margin` slots away from every cluster (top, size) at
    every table of min_slots slots or more: their top 32 hash bits keep out of [top - margin, top + size + margin]
    slot widths of a min_slots table, with wrap-around at 2^32"""
    import numpy as np
    from join_keys import hash64_np
    return outside_window_h(hash64_np(np.asarray(keys, dtype=np.int64)), tops, min_slots, margin)


# ---- multi-column rows and DISTINCT pairs ---------------------------------------------------------------------------
def key_words(row: Sequence, kinds: Sequence[str], nullable: bool) -> List[int]:
    """load_key_words of one row: kinds[j] is 'i' (BIGINT, signed or not: the same 8 bytes) or 'f' (DOUBLE); None is NULL"""
    w, nb = [], 0
    for j, (v, kd) in enumerate(zip(row, kinds)):
        if v is None:
            nb |= 1 << j
            w.append(0)
        else:
            w.append(double_key_bits(v) if kd == "f" else u64(int(v)))
    if nullable:
        w.append(nb)
    return w


def hash_words(words: Sequence[int]) -> int:
    h = hash64(words[0])
    for j in range(1, len(words)):
        h = hash64(h ^ ((u64(words[j]) * WORD_MUL + j) & M64))
    return h


def mk_home(words: Sequence[int], nslots: int) -> int:
    return slot32(hash_words(words), nslots)


def tag(words: Sequence[int]) -> int:
    """the published tag of a record: hash | 3 (mk_find_or_insert's `ready`)"""
    return hash_words(words) | 3


def solve_column(words: Sequence[int], col: int, target: int) -> int:
    """the word of column `col` (a BIGINT word, any value) that gives `words` the hash_words value `target`, the other
    words kept: the steps after `col` are undone from the target, then col's own step"""
    h = u64(target)
    for j in range(len(words) - 1, col, -1):
        h = u64(hash64_inv(h)) ^ ((u64(words[j]) * WORD_MUL + j) & M64)
    if col == 0:
        return u64(hash64_inv(h))
    prev = hash_words(words[:col])
    x = u64(hash64_inv(h)) ^ prev
    return ((x - col) * WORD_MUL_INV) & M64


def row_with_hash(row: Sequence, kinds: Sequence[str], nullable: bool, col: int, target: int) -> Tuple:
    """`row` with BIGINT column `col` (non-NULL) solved so that the row's key words hash to `target`"""
    assert kinds[col] == "i" and row[col] is not None
    w = key_words(row, kinds, nullable)
    out = list(row)
    out[col] = i64(solve_column(w, col, target))
    assert hash_words(key_words(out, kinds, nullable)) == u64(target)
    return tuple(out)


def rows_with_top(n: int, top: int, kinds: Sequence[str], nullable: bool, seed_row: Sequence, vary: int = 0,
                  col: Optional[int] = None) -> List[Tuple]:
    """n different rows whose hash_words has the top 32 bits `top` (one home at every table size): column `vary` counts
    up from seed_row's value, the last BIGINT column (or `col`) is solved"""
    col = max(j for j, k in enumerate(kinds) if k == "i") if col is None else col
    assert vary != col
    out = []
    for j in range(n):
        r = list(seed_row)
        r[vary] = (r[vary] + j) if kinds[vary] == "i" else float(r[vary] + j)
        out.append(row_with_hash(r, kinds, nullable, col, (top << 32) | (j * 0x9E3779B1 & 0xFFFFFFFF)))
    return out


def equal_hash_rows(n: int, row: Sequence, kinds: Sequence[str], nullable: bool, vary: int = 0,
                    col: Optional[int] = None) -> List[Tuple]:
    """n different rows with the same 64-bit hash_words as `row` (so the same home and the same tag): column `vary` steps,
    column `col` (default: the last BIGINT column) is solved.  They reach mk_find_or_insert's ordered-load compare."""
    col = max(j for j, k in enumerate(kinds) if k == "i") if col is None else col
    target = hash_words(key_words(row, kinds, nullable))
    out = [tuple(row)]
    for j in range(1, n):
        r = list(row)
        r[vary] = (r[vary] + j) if kinds[vary] == "i" else float(r[vary] + j)
        out.append(row_with_hash(r, kinds, nullable, col, target))
    assert len(set(out)) == n
    return out


def pair_words(group_words: Sequence[int], value_word: int) -> List[int]:
    """a DISTINCT set's key: the group table's words followed by the value (k_agg_distinct_mark)"""
    return list(group_words) + [u64(value_word)]


def values_with_set_top(n: int, group_words: Sequence[int], top: int) -> List[int]:
    """n different int64 DISTINCT values that, paired with one group's words, share the set home of `top` at every size"""
    w = list(group_words) + [0]
    return [i64(solve_column(w, len(w) - 1, (top << 32) | (j * 0x9E3779B1 & 0xFFFFFFFF))) for j in range(n)]


def equal_hash_pairs(n: int, group_words_fn, groups: Sequence, value: int) -> List[Tuple]:
    """(group, value) pairs of different groups with one set hash: the value is solved for each group's words so that
    every pair hashes like (groups[0], value).  group_words_fn(g) gives a group's words."""
    target = hash_words(pair_words(group_words_fn(groups[0]), value))
    out = [(groups[0], value)]
    for g in groups[1:n]:
        w = pair_words(group_words_fn(g), 0)
        out.append((g, i64(solve_column(w, len(w) - 1, target))))
    return out


# ---- can two rows that differ only in the NULL-bits word share a tag? ---------------------------------------------------
def _y(x: int) -> int:
    """hash64's xor-fold, linear over GF(2) and its own inverse"""
    return x ^ (x >> 32)


def null_word_tag_pairs(ncols: int = 4) -> List[Tuple[Tuple, Tuple]]:
    """Every way two rows of `ncols` nullable BIGINT columns that differ only in their NULL-bits word (NULL stored as 0,
    so a NULL and a 0 in the same column) can share a tag, as a list of row pairs; empty when no such pair exists.

    The words before the NULL word are equal, so both hashes are hash64(u ^ A_i) with one u and A_i = nb_i * WORD_MUL +
    ncols.  hash64(x) = _y(x) * MUL with _y linear, so the two hashes are MUL * (Y ^ a_1) and MUL * (Y ^ a_2) with Y = _y(u),
    a_i = _y(A_i).  Sharing a tag needs the hashes to differ by d in -3..3 (d != 0), that is (Y ^ a_1) - (Y ^ a_2) =
    d * MUL^-1.  Over the bits c = a_1 ^ a_2 the left side is a sum of +-2^i, one sign per bit of c chosen by Y, and the
    other bits cancel: it reaches t exactly when (t + c) / 2 or (t + c) / 2 + 2^63 is a subset of c.  Every candidate Y is
    then completed over the bits outside c that reach the tag's low bits, and the rows are built by solving a column that
    is not NULL in either row; each candidate is verified on the restated tags."""
    from join_keys import MUL_INV
    kinds = ["i"] * ncols
    found = []
    for nb1 in range(1 << ncols):
        for nb2 in range(nb1 + 1, 1 << ncols):
            a1, a2 = _y((nb1 * WORD_MUL + ncols) & M64), _y((nb2 * WORD_MUL + ncols) & M64)
            c = a1 ^ a2
            free_cols = [j for j in range(ncols) if not ((nb1 | nb2) >> j) & 1]
            for d in (-3, -2, -1, 1, 2, 3):
                t = (d * MUL_INV) & M64
                v = (t + c) & M64
                if v & 1:
                    continue
                for s in {v >> 1, (v >> 1) | (1 << 63)}:
                    if s & ~c & M64:
                        continue
                    base = (a1 & ~c) | ((~a1 & c) & s) | ((a1 & c) & ~s)   # Y on c: bit i flips a1's when i is in s
                    for low in range(4):
                        y = (base & ~(3 & ~c)) | (low & ~c & 3)
                        u = _y(y)
                        if not free_cols:
                            rows = [tuple(None if (nb >> j) & 1 else 0 for j in range(ncols)) for nb in (nb1, nb2)]
                            w = [key_words(r, kinds, True) for r in rows]
                            if hash_words(w[0][:ncols]) != u:
                                continue
                        else:
                            col = free_cols[-1]
                            r = [None if ((nb1 | nb2) >> j) & 1 else 0 for j in range(ncols)]
                            w = key_words(r, kinds, True)[:ncols]
                            r[col] = i64(solve_column(w, col, u))
                            rows = [tuple(None if (nb >> j) & 1 else r[j] for j in range(ncols)) for nb in (nb1, nb2)]
                        w1, w2 = (key_words(r, kinds, True) for r in rows)
                        if w1[:ncols] == w2[:ncols] and w1 != w2 and tag(w1) == tag(w2):
                            found.append((rows[0], rows[1]))
    return found


# ---- probing and growth ---------------------------------------------------------------------------------------------
def insert_run(homes: Sequence[int], nslots: int, max_probe: int = MAX_PROBE, taken: Optional[Dict[int, int]] = None):
    """linear probing of distinct keys given by their homes, in order, into a table of nslots slots (`taken`: slot ->
    key index, updated): returns the indices of the keys that found no slot within max_probe steps.  A key at offset i
    from its home needs i steps: offsets 0 .. max_probe are reachable."""
    taken = {} if taken is None else taken
    deferred = []
    for idx, h in enumerate(homes):
        s, steps = h, 0
        while s in taken:
            steps += 1
            if steps > max_probe:
                deferred.append(idx)
                break
            s = (s + 1) % nslots
        else:
            taken[s] = idx
    return deferred


def grown_slots(cur: int, more: int) -> int:
    """agg.cu grown_slots: x4, or more: at most half full once `more` new entries join a table that was 60 % full"""
    return max(cur * 4, int((cur * 0.6 + more) * 2))


def first_slots(rows: int, expected_groups: int = 0) -> int:
    """the group table's (and a DISTINCT set's, without a hint) first size: twice the hint, else twice the first push's
    rows up to 4 M, at least 1024"""
    if expected_groups > 0:
        return max(1024, 2 * expected_groups)
    return max(1024, 2 * min(rows, 1 << 22))


def long_run_not_full(used: int, nd: int, slots: int) -> bool:
    """agg.cu long_run_not_full: the table stays at most a quarter full once the deferred items join"""
    return (used + nd) * 4 <= slots


def grow_rounds(keys: Sequence[int], first: int, fixed: bool = True, max_rounds: int = 40):
    """grow_and_retry over one pass of distinct single-column keys into a table of `first` slots.  fixed=False restates
    the rule before long_run_not_full: every deferral grows the table.  Returns (slots, rounds, error): error is "oom"
    when the table would reach 2^32 slots (alloc_table's TG_ERR_OOM)."""
    slots, probe, todo, taken = first, MAX_PROBE, list(keys), {}
    for rnd in range(max_rounds):
        dl = insert_run([agg_home(k, slots) for k in todo], slots, probe, taken)
        if not dl:
            return slots, rnd + 1, None
        todo = [todo[i] for i in dl]
        if fixed and probe == MAX_PROBE and long_run_not_full(len(taken), len(todo), slots):
            probe = slots
            continue
        want = grown_slots(slots, len(todo))
        if want > MAX_SLOTS:
            return slots, rnd + 1, "oom"
        # the rehash places every key of the old table in the grown one (k_agg_rehash walks without a limit)
        pending = set(todo)
        slots, probe, taken = want, MAX_PROBE, {}
        insert_run([agg_home(k, slots) for k in keys if k not in pending], slots, slots, taken)
    return slots, max_rounds, "no convergence"


def slots_bound(first: int, entries: int) -> int:
    """the largest table grow_and_retry can reach from `first` slots when every round's used + deferred count is at most
    `entries` (the table's groups plus the rows that can be deferred): a table of 4 * entries slots or more always has
    room, so the last growth starts below that and adds at most `entries`"""
    if 4 * entries <= first:
        return first
    return max(first, grown_slots(4 * entries - 1, entries))


def chernoff_run_bound(load: float, k: int = MAX_PROBE + 1) -> float:
    """an upper bound on the chance that a run of k occupied slots starts at a given slot of a linear-probing table of
    uniform homes at `load`: at least k of the keys home within those k slots, a sum of independent Bernoulli draws of
    mean k * load, so P <= exp(-mu) (e mu / k)^k = (load * e^(1 - load))^k.  A probe longer than MAX_PROBE steps needs such
    a run of MAX_PROBE + 1 slots."""
    return (load * math.exp(1 - load)) ** k


def hash_words_np(words) -> "np.ndarray":
    """hash_words over columns of words (a list of equal-length uint64 / int64 arrays, one per key word)"""
    import numpy as np
    from join_keys import hash64_np
    h = hash64_np(np.asarray(words[0]).astype(np.int64))
    with np.errstate(over="ignore"):
        for j in range(1, len(words)):
            w = np.asarray(words[j]).astype(np.int64).view(np.uint64)
            h = hash64_np((h ^ (w * np.uint64(WORD_MUL) + np.uint64(j))).view(np.int64))
    return h


def outside_window_h(h, tops: Sequence[Tuple[int, int]], min_slots: int, margin: int = 64):
    """outside_window for items given by their 64-bit hashes (uint64 array)"""
    import numpy as np
    t = (np.asarray(h, dtype=np.uint64) >> np.uint64(32)).astype(np.int64)
    width = -(-(1 << 32) // min_slots)
    ok = np.ones(len(t), dtype=bool)
    for top, size in tops:
        ok &= (t - (top - margin * width)) % (1 << 32) > (size + 2 * margin) * width
    return ok
