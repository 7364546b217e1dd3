"""The rules of the slice index of a sliced unique-key join table (tidb_b200/csrc/join.cu build_slice_index, SliceIndex in
join_kernels.cuh), restated in Python over numpy uint64 arrays: the key hash, the slice and bucket a key falls in, the
index sizes the build picks and whether it builds the index at all.  Also the inverse of the hash, so tests can craft
build sides with a chosen number of keys per slice and chosen bucket sizes."""
import math

import numpy as np

GOLD = 0x9E3779B97F4A7C15          # hash64: (k ^ (k >> 32)) * GOLD mod 2^64
GOLD_INV = pow(GOLD, -1, 1 << 64)
SENTINEL = -(1 << 63)              # kEmptyKey: the key value that marks empty slots, kept in the table's side slot
LOAD = 0.7                         # kPidxLoad: keys per index slot of the fullest slice
KEYS_PER_BUCKET = 4.0              # kPidxKeysPerBucket
MAX_PILOT_BYTES = 160 << 10        # kPidxMaxPilotBytes: pilot bytes of one slice, held in shared memory by the probe
MAX_BUCKET = 32                    # kPidxMaxBucket: a bucket with more keys is never placed
_M32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def _u64(a):
    a = np.asarray(a)
    return a if a.dtype == np.uint64 else a.astype(np.int64).view(np.uint64)


def hash64(keys):
    """hash64 of int64 keys, as uint64"""
    k = _u64(keys)
    with np.errstate(over="ignore"):
        return (k ^ (k >> _S32)) * np.uint64(GOLD)


def mulhi32(a, n):
    """(a * n) >> 32 for 32-bit a (uint64 array) and n < 2^32: the product fits in 64 bits"""
    return (a * np.uint64(n)) >> _S32


def slot32(h, n):
    """slot32: the top 32 hash bits scaled to [0, n) — the slice of a key among P slices"""
    return mulhi32(h >> _S32, n)


def pidx_bucket(h, B):
    """pidx_bucket: the low 32 hash bits scaled to [0, B) — a key's bucket within its slice"""
    return mulhi32(h & _M32, B)


def key_of_hash(h):
    """the int64 keys whose hash64 is h (uint64 array): GOLD is odd, so the product inverts mod 2^64, and the
    xor-shift inverts by xoring the high half into the low half again"""
    with np.errstate(over="ignore"):
        kp = _u64(h) * np.uint64(GOLD_INV)
    hi = kp >> _S32
    return ((hi << _S32) | ((kp & _M32) ^ hi)).view(np.int64)


def part_counts(keys, P):
    """keys per slice of the build keys; the sentinel key lives in the side slot and is not counted"""
    k = np.asarray(keys, dtype=np.int64)
    k = k[k != SENTINEL]
    return np.bincount(slot32(hash64(k), P).astype(np.int64), minlength=P)


def index_params(part_counts, P):
    """(S, B, built) as build_slice_index decides them: S index slots and B pilot bytes per slice (a multiple of 16),
    both sized by the fullest slice; the index is built when there are at least 2 slices and B fits kPidxMaxPilotBytes"""
    mx = int(max(part_counts))
    S = math.ceil(mx / LOAD) + 1
    B = (math.ceil(mx / KEYS_PER_BUCKET) + 16) & ~15
    return S, B, P >= 2 and B <= MAX_PILOT_BYTES


def _range32(i, n):
    """[lo, hi): the 32-bit values a with mulhi32(a, n) == i"""
    return -(-(i << 32) // n), -(-((i + 1) << 32) // n)


def hashes_in_slice(rng, p, P, count, lo_range=(0, 1 << 32), avoid_buckets=None, B=1):
    """`count` random hashes whose slice is p of P, their low halves drawn from lo_range ([lo, hi)) and never in one of
    the buckets `avoid_buckets` of B"""
    a, b = _range32(p, P)
    hi = rng.integers(a, b, count, dtype=np.uint64)
    lo = rng.integers(lo_range[0], lo_range[1], count, dtype=np.uint64)
    if avoid_buckets is not None and len(avoid_buckets):
        bad = np.isin(pidx_bucket(lo, B), avoid_buckets)
        while bad.any():
            lo[bad] = rng.integers(lo_range[0], lo_range[1], int(bad.sum()), dtype=np.uint64)
            bad = np.isin(pidx_bucket(lo, B), avoid_buckets)
    return (hi << _S32) | lo


def hashes_in_bucket(rng, p, P, b, B, count):
    """`count` random hashes of slice p of P and bucket b of B"""
    return hashes_in_slice(rng, p, P, count, lo_range=_range32(b, B))


def craft_build(counts, P, buckets=(), seed=0):
    """unique int64 build keys with exactly counts[p] keys in slice p of P, none of them the sentinel.
    buckets: (slice, bucket, size) triples; bucket None picks a random one.  Each named bucket holds exactly `size` keys
    (the slice's other keys avoid it), with B the pilot bytes the build will size for these counts.  -> (keys, [(slice,
    bucket, size)] with every bucket resolved)"""
    rng = np.random.default_rng(seed)
    _, B, _ = index_params(counts, P)
    chosen, taken = [], set()
    for p, b, size in buckets:
        while b is None or (p, b) in taken:
            b = int(rng.integers(0, B))
        taken.add((p, b))
        chosen.append((p, b, size))
    parts = []
    for p in range(P):
        mine = [(b, size) for q, b, size in chosen if q == p]
        rest = counts[p] - sum(size for _, size in mine)
        assert rest >= 0, (p, counts[p], len(mine))
        parts.append(hashes_in_slice(rng, p, P, rest, avoid_buckets=np.array([b for b, _ in mine], np.uint64), B=B))
        parts += [hashes_in_bucket(rng, p, P, b, B, size) for b, size in mine]
    h = np.concatenate(parts)
    keys = key_of_hash(h)
    sentinel_hash = hash64(np.array([SENTINEL], np.int64))[0]
    hs = np.sort(h)
    assert (hs[1:] != hs[:-1]).all() and not (h == sentinel_hash).any(), "a repeated hash: pick another seed"
    return keys[rng.permutation(len(keys))], chosen


def bucket_sizes(keys, P, B):
    """(slice, bucket) -> keys, for the non-sentinel keys: the bucket counts k_pidx_bucket_count makes"""
    k = np.asarray(keys, dtype=np.int64)
    h = hash64(k[k != SENTINEL])
    gid = slot32(h, P).astype(np.int64) * B + pidx_bucket(h, B).astype(np.int64)
    return np.bincount(gid, minlength=P * B).reshape(P, B)
