"""Keys that land where a test wants them in the GPU join table.

A restatement of the join's hashing (tidb_b200/csrc/common.cuh, join_kernels.cuh) with inverses:
  hash64(k)        = (k ^ k >> 32) * 0x9E3779B97F4A7C15 mod 2^64   an xor-fold and an odd multiply: both invert
  slot32(h, n)     = mulhi32(hi32(h), n)                           the table slot, monotone in hi32(h)
  home_slot(h, n)  = slot32(h, n) rounded down to a multiple of 4  where a key's linear-probe run starts
  l2_slice(h, P)   = mulhi32(hi32(h), P)                           the L2 slice of the partitioned probe
  candidate_key(t) = k_composite_key's mix of 2-4 key columns: h = t0, then h = fmix(h) + t_c * C + c per column, C odd

key_with_home(slot, nslots) returns a key whose home is `slot`; colliding_keys(row, ncols) returns a different key tuple with
the same candidate key.  Keys are int64 values (the bits of an unsigned key).
"""
from __future__ import annotations

from typing import Sequence, Tuple

import numpy as np

M64 = (1 << 64) - 1
MUL = 0x9E3779B97F4A7C15
MUL_INV = pow(MUL, -1, 1 << 64)
HOME_WIDTH = 4
SENTINEL = -(1 << 63)     # the table's empty-slot key; a build key with this value lives in the side slot `nslots`
_F1, _F2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB
_F1_INV, _F2_INV = pow(_F1, -1, 1 << 64), pow(_F2, -1, 1 << 64)


def u64(k: int) -> int:
    return k & M64


def i64(u: int) -> int:
    u &= M64
    return u - (1 << 64) if u >> 63 else u


def hash64(k: int) -> int:
    k = u64(k)
    return ((k ^ (k >> 32)) * MUL) & M64


def hash64_inv(h: int) -> int:
    """the int64 key whose hash64 is h (the xor-fold by 32 is its own inverse)"""
    x = (u64(h) * MUL_INV) & M64
    return i64(x ^ (x >> 32))


def mulhi32(a: int, b: int) -> int:
    return (a * b) >> 32


def slot32(h: int, nslots: int) -> int:
    return mulhi32(u64(h) >> 32, nslots)


def home_slot(h: int, nslots: int) -> int:
    return slot32(h, nslots) & ~(HOME_WIDTH - 1)


def home_of_key(k: int, nslots: int) -> int:
    return home_slot(hash64(k), nslots)


def l2_slice(h: int, parts: int) -> int:
    return mulhi32(u64(h) >> 32, parts)


def key_with_home(slot: int, nslots: int, salt: int = 0) -> int:
    """a key whose home slot is `slot` (a multiple of HOME_WIDTH below nslots); `salt` picks one of 2^32 such keys"""
    assert slot % HOME_WIDTH == 0 and 0 <= slot < nslots < (1 << 32)
    hi = -(-(slot << 32) // nslots)            # the smallest hi32 with mulhi32(hi, nslots) >= slot
    k = hash64_inv((hi << 32) | (salt & 0xFFFFFFFF))
    assert k != SENTINEL and home_of_key(k, nslots) == slot
    return k


def first_hi32_of_slice(p: int, parts: int) -> int:
    """the smallest hi32(h) in L2 slice p"""
    return -(-(p << 32) // parts)


def fmix(h: int) -> int:
    h = u64(h)
    h ^= h >> 30
    h = (h * _F1) & M64
    h ^= h >> 27
    h = (h * _F2) & M64
    return h ^ (h >> 31)


def _unxorshift(h: int, s: int) -> int:
    x = h
    for _ in range(64 // s + 1):
        x = h ^ (x >> s)
    return x & M64


def fmix_inv(h: int) -> int:
    h = _unxorshift(u64(h), 31)
    h = (h * _F2_INV) & M64
    h = _unxorshift(h, 27)
    h = (h * _F1_INV) & M64
    return _unxorshift(h, 30)


def candidate_key(row: Sequence[int]) -> int:
    """k_composite_key's 64-bit candidate key of one key tuple (int64 values)"""
    h = u64(row[0])
    for c in range(1, len(row)):
        h = (fmix(h) + u64(row[c]) * MUL + c) & M64
    return i64(h)


def colliding_keys(row: Sequence[int], ncols: int, delta: int = 1) -> Tuple[int, ...]:
    """a key tuple != row with the same candidate key: the first column moves by `delta`, the others up to the last stay,
    and the last column is solved for: b_last = (target - fmix(h') - (ncols - 1)) * C^-1 mod 2^64"""
    assert len(row) == ncols >= 2 and delta != 0
    target = u64(candidate_key(row))
    new = [i64(row[0] + delta)] + [int(v) for v in row[1:ncols - 1]]
    h = u64(new[0])
    for c in range(1, ncols - 1):
        h = (fmix(h) + u64(new[c]) * MUL + c) & M64
    last = ((target - fmix(h) - (ncols - 1)) * MUL_INV) & M64
    out = tuple(new + [i64(last)])
    assert out != tuple(int(v) for v in row) and candidate_key(out) == i64(target)
    return out


def hash64_np(k: np.ndarray) -> np.ndarray:
    k = np.asarray(k).view(np.uint64)
    with np.errstate(over="ignore"):
        return (k ^ (k >> np.uint64(32))) * np.uint64(MUL)


def home_slot_np(k: np.ndarray, nslots: int) -> np.ndarray:
    hi = hash64_np(k) >> np.uint64(32)
    return ((hi * np.uint64(nslots)) >> np.uint64(32)).astype(np.int64) & ~(HOME_WIDTH - 1)
