"""The key-crafting model of the hash aggregation's tables (tests/agg_keys.py), and its model of grow_and_retry.

CPU only: the crafted homes, the wrap keys, the equal-hash rows, the cluster size either side of the probe limit, the
answer to whether a row can share a tag with a row that differs only in the NULL-bits word, and the bound on table size
that the growth rule gives a crafted cluster."""
import random

import numpy as np
import pytest

import agg_keys as K
from join_keys import SENTINEL, hash64, hash64_inv, i64, u64

SIZES = [1024, 4096, 12_345, 1 << 20, 3_000_017, 1 << 31, (1 << 32) - 4]


def test_top_keys_share_a_home_at_every_size():
    # the issue's example: j < 50 keys i64(hash64_inv(0x12345678_00000000 | j)) share one home at every size
    ks = K.top_keys(50, 0x12345678)
    assert ks == [i64(hash64_inv(0x12345678_00000000 | j)) for j in range(50)]
    for n in SIZES:
        assert len({K.agg_home(k, n) for k in ks}) == 1, n
    # BIGINT UNSIGNED keys are the same 8 bytes
    assert all(K.agg_home(u64(k), 4096) == K.agg_home(k, 4096) for k in ks)


def test_top_keys_skip_the_sentinel():
    top = hash64(SENTINEL) >> 32
    low = hash64(SENTINEL) & 0xFFFFFFFF
    ks = K.top_keys(3, top, low0=low)
    assert SENTINEL not in ks and len(set(ks)) == 3 and all(K.top32(k) == top for k in ks)


def test_wrap_keys_home_on_the_last_slot():
    # mulhi32(0xFFFFFFFF, n) = n - 1: the run wraps to slot 0; top 0 homes on slot 0
    for n in SIZES:
        assert {K.agg_home(k, n) for k in K.top_keys(20, 0xFFFFFFFF)} == {n - 1}
        assert {K.agg_home(k, n) for k in K.top_keys(20, 0)} == {0}
    taken = {}
    assert K.insert_run([K.agg_home(k, 1024) for k in K.top_keys(30, 0xFFFFFFFF)], 1024, K.MAX_PROBE, taken) == []
    assert sorted(taken) == list(range(29)) + [1023]


def test_double_keys_are_finite_and_not_negative_zero():
    xs = K.top_doubles(300, 0x0BADCAFE)
    assert len(set(K.f64_bits(x) for x in xs)) == 300
    assert all(np.isfinite(x) and K.f64_bits(x) != K.NEG_ZERO for x in xs)
    for n in SIZES:
        assert len({K.slot32(hash64(K.double_key_bits(x)), n) for x in xs}) == 1
    assert K.double_key_bits(-0.0) == K.double_key_bits(0.0) == 0


@pytest.mark.parametrize("ls", [512, 1024, 2048, 4096])
def test_local_keys_share_the_last_local_slot(ls):
    ks = K.local_top_keys(100)
    assert {K.local_home(k, ls) for k in ks} == {ls - 1}
    assert len({K.agg_home(k, 1 << 20) for k in ks}) > 90      # their global homes are spread


def test_window_keys_and_background_filter():
    ks = K.window_keys(40, 0x80000000, 8)
    assert len(set(ks)) == 40 and all(0x80000000 <= K.top32(k) < 0x80000008 for k in ks)
    rng = np.random.default_rng(0)
    bg = rng.integers(-(1 << 62), 1 << 62, 200_000)
    ok = K.outside_window(bg, [(0x80000000, 40), (0xFFFFFFFF, 50)], 1 << 17)
    assert 0.8 < ok.mean() < 1.0
    for n in (1 << 17, 1 << 20, 1 << 24):
        homes = np.array([K.agg_home(int(k), n) for k in bg[ok][:5000]])
        c0, c1 = K.agg_home(ks[0], n), n - 1
        assert np.all(np.minimum(np.abs(homes - c0), n - np.abs(homes - c0)) > 64)
        assert np.all(np.minimum(np.abs(homes - c1), n - np.abs(homes - c1)) > 64)


def test_cluster_size_either_side_of_the_probe_limit():
    # a key at offset i from its home needs i steps: offsets 0 .. 48 fit, so 49 keys fit and the 50th is deferred
    for c, deferred in ((48, 0), (49, 0), (50, 1), (51, 2), (200, 151)):
        homes = [K.agg_home(k, 4096) for k in K.top_keys(c, 0x12345678)]
        assert len(K.insert_run(homes, 4096)) == deferred, c
    # at any size, and whichever key comes first
    ks = K.top_keys(50, 0x12345678)
    random.Random(1).shuffle(ks)
    for n in SIZES[:4]:
        assert len(K.insert_run([K.agg_home(k, n) for k in ks], n)) == 1


@pytest.mark.parametrize("ncols", [2, 3, 4])
@pytest.mark.parametrize("nullable", [False, True])
def test_rows_solved_through_the_last_column(ncols, nullable):
    kinds, seed = {2: (["f", "i"], [0.5, 0]), 3: (["i", "f", "i"], [7, None if nullable else 0.5, 3]),
                   4: (["i", "f", "i", "i"], [7, 0.5, None if nullable else 3, 11])}[ncols]
    rows = K.rows_with_top(60, 0x00C0FFEE, kinds, nullable, seed)
    assert len(set(rows)) == 60
    for n in SIZES:
        assert {K.mk_home(K.key_words(r, kinds, nullable), n) for r in rows} == {K.slot32(0x00C0FFEE << 32, n)}
    nkw = ncols + (1 if nullable else 0)
    assert all(len(K.key_words(r, kinds, nullable)) == nkw for r in rows)


@pytest.mark.parametrize("ncols", [2, 3, 4])
@pytest.mark.parametrize("nullable", [False, True])
def test_equal_hash_rows_share_the_tag(ncols, nullable):
    kinds = ["i"] * ncols
    row = [5, None if nullable and ncols > 2 else 9, 13, -2][:ncols]
    rows = K.equal_hash_rows(8, row, kinds, nullable)
    words = [K.key_words(r, kinds, nullable) for r in rows]
    assert len({tuple(w) for w in words}) == 8
    assert len({K.hash_words(w) for w in words}) == 1 and len({K.tag(w) for w in words}) == 1


def test_key_words_restate_load_key_words():
    # NULL stored as 0 plus the NULL-bits word; DOUBLE -0 stored as +0
    assert K.key_words([None, -0.0, 4], ["i", "f", "i"], True) == [0, 0, 4, 0b001]
    assert K.key_words([0, 0.0, 4], ["i", "f", "i"], True) == [0, 0, 4, 0]
    assert K.key_words([-1, 1.0], ["i", "f"], False) == [u64(-1), K.f64_bits(1.0)]
    w1, w2 = K.key_words([None, 1, 2, 3], ["i"] * 4, True), K.key_words([0, 1, 2, 3], ["i"] * 4, True)
    assert w1[:4] == w2[:4] and K.hash_words(w1) != K.hash_words(w2)


def test_no_row_shares_a_tag_with_one_that_differs_only_in_the_null_word():
    # mk_find_or_insert compares a 4-column group table's first four words and leaves the fifth, the NULL-bits word, to the
    # tag.  The model decides exactly whether two rows that differ only in that word can share a tag: they cannot, for
    # 2, 3 and 4 nullable columns, so (NULL, a, b, c) and (0, a, b, c) never merge
    for ncols in (2, 3, 4):
        assert K.null_word_tag_pairs(ncols) == []


def test_null_word_decision_restates_the_sign_sums():
    # the decision rests on: (Y ^ a1) - (Y ^ a2) mod 2^64 is a sum of +-2^i over the bits of c = a1 ^ a2, so
    # ((diff + c) / 2) mod 2^63 is a subset of c.  Check it on random draws
    r = random.Random(3)
    for _ in range(2000):
        y, a1, a2 = (r.getrandbits(64) for _ in range(3))
        c = a1 ^ a2
        diff = ((y ^ a1) - (y ^ a2)) & K.M64
        v = (diff + c) & K.M64
        assert v & 1 == 0
        s = v >> 1
        assert (s & ~c & K.M64) == 0 or ((s | (1 << 63)) & ~c & K.M64) == 0


def test_distinct_values_with_a_set_top_and_equal_hash_pairs():
    gw = lambda g: K.key_words([g], ["i"], True)
    vals = K.values_with_set_top(60, gw(42), 0x55555555)
    assert len(set(vals)) == 60
    for n in SIZES[:5]:
        assert len({K.mk_home(K.pair_words(gw(42), v), n) for v in vals}) == 1
    pairs = K.equal_hash_pairs(6, gw, [1, 2, 3, None, 5, 6], 77)
    hs = {K.hash_words(K.pair_words(gw(g), v)) for g, v in pairs}
    assert len(hs) == 1 and len(set(pairs)) == 6
    # without GROUP BY the set key is the value alone
    vs = K.values_with_set_top(10, [], 0x1234)
    assert len({K.mk_home([u64(v)], 4096) for v in vs}) == 1


# ---- growth ---------------------------------------------------------------------------------------------------------
def test_unfixed_rule_grows_a_50_key_cluster_until_out_of_memory():
    # every deferral grew the table x4: 1024 slots -> 2^30, then alloc_table refuses 2^32 slots
    slots, rounds, err = K.grow_rounds(K.top_keys(50, 0x12345678), 1024, fixed=False)
    assert (slots, err) == (1 << 30, "oom") and rounds == 11


@pytest.mark.parametrize("c", [49, 50, 51, 200, 5000])
def test_fixed_rule_keeps_the_table_for_a_cluster(c):
    first = K.first_slots(100_000)
    slots, rounds, err = K.grow_rounds(K.top_keys(c, 0x12345678), first)
    assert err is None and slots == first and rounds == (1 if c <= 49 else 2)


def test_fixed_rule_grows_a_full_table():
    # 700 uniform keys and a 60-key cluster in 1024 slots: the deferral comes with the table over a quarter full, so it
    # grows as before, then the cluster's long run is walked without the limit
    rng = random.Random(5)
    ks = [rng.getrandbits(63) for _ in range(700)] + K.top_keys(60, 0x42424242)
    slots, rounds, err = K.grow_rounds(ks, 1024)
    assert err is None and slots == 4096 and rounds == 3
    assert slots <= K.slots_bound(1024, len(ks))


def test_slots_bound():
    assert K.slots_bound(1 << 18, 10_000) == 1 << 18
    assert K.slots_bound(1024, 5000) == K.grown_slots(19_999, 5000)
    assert K.slots_bound(1024, 5000) < 1 << 17
    assert K.first_slots(100, 0) == 1024 and K.first_slots(100_000) == 200_000 and K.first_slots(10, 64) == 1024
    assert K.first_slots(1 << 23) == 1 << 23


def test_uniform_data_never_reaches_the_rule():
    # a deferral needs a run of MAX_PROBE + 1 occupied slots; at a quarter load its chance per slot is below 3e-14, so
    # even a 2^32-slot table of uniform keys defers nothing at the load the rule keeps; at half load it is 8e-5
    assert K.chernoff_run_bound(0.25) < 3e-14 and K.chernoff_run_bound(0.25) * (1 << 32) < 2e-4
    assert K.chernoff_run_bound(0.5) > 5e-5
