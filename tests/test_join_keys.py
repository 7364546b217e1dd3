"""The key constructions of tests/join_keys.py round-trip, and the planner gate of FLOAT join columns (tg_join_supported runs
the descriptor checks only: no device needed)."""
import ctypes as C

import numpy as np
import pytest

import join_keys as K
from test_oracle_join import INT, DBL
from tidb_b200 import abi
from tidb_b200.plan import FieldType, FilterItem, JoinPlan, OtherCond

FLT = FieldType(abi.TYPE_FLOAT, 0)


def test_hash64_and_fmix_invert():
    rng = np.random.default_rng(1)
    for k in [0, 1, -1, K.SENTINEL, (1 << 63) - 1] + [int(x) for x in rng.integers(-(1 << 63), (1 << 63) - 1, 200, dtype=np.int64)]:
        assert K.hash64_inv(K.hash64(k)) == k
        assert K.i64(K.fmix_inv(K.fmix(k))) == k
        assert int(K.hash64_np(np.array([k], dtype=np.int64))[0]) == K.hash64(k)


@pytest.mark.parametrize("nslots", [36, 1000, 8632, 2_222_256, (1 << 31) + 4])
def test_key_with_home_lands_on_its_home(nslots):
    for slot in sorted({0, 4, nslots - 4 - nslots % 4, (nslots // 2) & ~3}):
        for salt in (0, 1, 0xFFFFFFFF, 12345):
            k = K.key_with_home(slot, nslots, salt)
            assert K.home_of_key(k, nslots) == slot
            assert int(K.home_slot_np(np.array([k], dtype=np.int64), nslots)[0]) == slot


def test_slice_boundaries_are_monotone_in_the_slot():
    # slot and slice are both mulhi32 of hi32(h): the first hash of slice p lands at or above p/P of the table
    nslots, P = 8632, 8
    for p in range(1, P):
        hi = K.first_hi32_of_slice(p, P)
        assert K.l2_slice(hi << 32, P) == p and K.l2_slice((hi - 1) << 32, P) == p - 1
        assert K.slot32((hi - 1) << 32, nslots) <= p * nslots // P <= K.slot32(hi << 32, nslots)


@pytest.mark.parametrize("ncols", [2, 3, 4])
def test_colliding_keys_share_the_candidate_key(ncols):
    rng = np.random.default_rng(ncols)
    for _ in range(100):
        row = tuple(int(x) for x in rng.integers(-1000, 1000, ncols))
        for delta in (1, -7, 1 << 40):
            other = K.colliding_keys(row, ncols, delta)
            assert other != row and K.candidate_key(other) == K.candidate_key(row)
    # two columns: fmix(a0) + a1*C + 1 (the kernel's formula spelt out)
    a0, a1 = 5, -3
    assert K.candidate_key((a0, a1)) == K.i64(K.fmix(a0) + K.u64(a1) * K.MUL + 1)


def _supported(plan):
    lib = abi.load_lib()
    d, keep = plan.to_struct()
    return lib.tg_join_supported(C.byref(d))


def test_float_columns_gate():
    # accepted: a FLOAT key (against FLOAT or DOUBLE), FLOAT payloads on both sides, any join type
    for jt in (abi.JOIN_INNER, abi.JOIN_LEFT_OUTER, abi.JOIN_SEMI, abi.JOIN_LEFT_OUTER_SEMI):
        semi = jt >= abi.JOIN_SEMI
        for rk in (FLT, DBL):
            plan = JoinPlan(jt, [FLT, FLT, INT], [rk, FLT], [0], [0], lused=[0, 1, 2], rused=[] if semi else [0, 1])
            assert _supported(plan) == abi.TG_OK
    plan = JoinPlan(abi.JOIN_INNER, [INT, FLT], [INT, FLT], [0], [0], build_is_right=False)
    assert _supported(plan) == abi.TG_OK
    # declined: FLOAT in a filter, in an OtherCondition, in a multi-column key, a FLOAT key against an integer key
    declined = [
        JoinPlan(abi.JOIN_INNER, [INT, FLT], [INT], [0], [0], probe_filter=[FilterItem(abi.CMP_GT, 1, is_real=True, const_f64=0.5)]),
        JoinPlan(abi.JOIN_INNER, [INT], [INT, FLT], [0], [0], build_filter=[FilterItem(abi.CMP_GT, 1, is_real=True, const_f64=0.5)]),
        JoinPlan(abi.JOIN_INNER, [INT, FLT], [INT, FLT], [0], [0], other_cond=[OtherCond(abi.CMP_LT, 0, 1, 1, 1, is_real=True)]),
        JoinPlan(abi.JOIN_INNER, [INT, FLT], [INT, FLT], [0, 1], [0, 1]),
        JoinPlan(abi.JOIN_INNER, [FLT], [INT], [0], [0]),
    ]
    for plan in declined:
        assert _supported(plan) == abi.TG_ERR_UNSUPPORTED, plan
