"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol
include/tidbgpu.h declares, validates descriptors without a GPU, and fails loudly (no CPU fallback)
when no device is present."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tidb_b200 import abi
from tidb_b200.chunk import Column
from tidb_b200.plan import AggFunc, AggPlan, FieldType, JoinPlan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
DBL = FieldType(abi.TYPE_DOUBLE, 0)


@pytest.fixture(scope="module")
def lib():
    from tidb_b200 import build
    build.build()
    return abi.load_lib()


def test_header_symbols_all_exported_abi_version_2(lib):
    hdr = open(os.path.join(ROOT, "include", "tidbgpu.h")).read()
    declared = set(re.findall(r"\b(tg_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(abi.EXPORTED_SYMBOLS), declared ^ set(abi.EXPORTED_SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), f"{name} is declared in tidbgpu.h but not exported"
    assert lib.tg_abi_version() == 2


def test_stats_struct_layout_and_path_bits():
    # tg_join_stats / tg_agg_stats as include/tidbgpu.h lays them out (ABI version 2): the Python mirror must agree byte
    # for byte, and the path bits must carry the header's values
    assert C.sizeof(abi.TgJoinStats) == 12 * 8 + 2 * 4 and abi.TgJoinStats.paths.offset == 8 * 8 + 4
    assert C.sizeof(abi.TgAggStats) == 9 * 8 + 2 * 4 and abi.TgAggStats.local_rows.offset == 8 * 8
    assert abi.TgAggStats.paths.offset == 9 * 8
    hdr = open(os.path.join(ROOT, "include", "tidbgpu.h")).read()
    bits = dict((m.group(1), 1 << int(m.group(2))) for m in re.finditer(r"\bTG_((?:JOIN|AGG)_PATH_[A-Z0-9_]+) = 1 << (\d+)", hdr))
    assert len(bits) == 13
    for name, v in bits.items():
        assert getattr(abi, name) == v, name
    assert 1 << 4 not in [v for name, v in bits.items() if name.startswith("JOIN")]   # unassigned, never reused


def test_fixed_len_matches_reference(lib):
    # pkg/util/chunk/codec.go:165-179 getFixedLen
    for tp, n in ((abi.TYPE_FLOAT, 4), (abi.TYPE_TINY, 8), (abi.TYPE_LONGLONG, 8), (abi.TYPE_DOUBLE, 8), (abi.TYPE_YEAR, 8),
                  (abi.TYPE_DURATION, 8), (abi.TYPE_DATETIME, 8), (abi.TYPE_NEWDECIMAL, 40), (abi.TYPE_VARSTRING, -1)):
        assert lib.tg_fixed_len(tp) == n


def test_join_supported_gate(lib):
    ok = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0])
    d, keep = ok.to_struct()
    assert lib.tg_join_supported(C.byref(d)) == abi.TG_OK
    multi = JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0, 1], [0, 1])   # round 2: FixedSerializedKey mode
    d, keep = multi.to_struct()
    assert lib.tg_join_supported(C.byref(d)) == abi.TG_OK
    strkey = JoinPlan(abi.JOIN_INNER, [FieldType(abi.TYPE_VARSTRING)], [FieldType(abi.TYPE_VARSTRING)], [0], [0])
    d, keep = strkey.to_struct()
    assert lib.tg_join_supported(C.byref(d)) == abi.TG_ERR_UNSUPPORTED
    # NewJoinProbe panics for semi joins with right-side output columns (base_join_probe.go:896)
    semi = JoinPlan(abi.JOIN_SEMI, [INT_NN], [INT_NN], [0], [0], rused=[0])
    d, keep = semi.to_struct()
    assert lib.tg_join_supported(C.byref(d)) == abi.TG_ERR_INVALID


def test_agg_supported_gate(lib):
    ok = AggPlan([INT_NN, DBL], [0], [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, 1, abi.TYPE_DOUBLE)])
    d, keep = ok.to_struct()
    assert lib.tg_agg_supported(C.byref(d)) == abi.TG_OK
    # SUM(int) returns DECIMAL in TiDB (aggregation/base_func.go:223): declined
    bad = AggPlan([INT_NN, INT_NN], [0], [AggFunc(abi.AGG_SUM, 1, abi.TYPE_LONGLONG)])
    d, keep = bad.to_struct()
    assert lib.tg_agg_supported(C.byref(d)) == abi.TG_ERR_UNSUPPORTED


def test_no_cpu_fallback_without_device(lib):
    if lib.tg_device_count() > 0:
        pytest.skip("a CUDA device is present")
    plan = JoinPlan(abi.JOIN_INNER, [INT_NN], [INT_NN], [0], [0])
    d, keep = plan.to_struct()
    h = C.c_void_p()
    assert lib.tg_join_open(C.byref(d), C.byref(h)) == abi.TG_ERR_CUDA
    assert b"no CPU fallback" in lib.tg_last_error()
    p = C.c_void_p()
    assert lib.tg_dev_alloc(0, C.c_size_t(16), C.byref(p)) == abi.TG_ERR_CUDA


def test_vec_compare_and_arith_refuse_4_byte_operands_without_a_device(lib):
    # a 4-byte operand, as a or as b, is TG_ERR_UNSUPPORTED on every machine: the argument checks answer before the
    # device is looked for, and a refused call writes nothing
    wide, narrow = Column(np.arange(5, dtype=np.int64)).to_struct(), Column(np.arange(5, dtype=np.int32)).to_struct()
    assert narrow.elem_len == 4
    for name, const in (("tg_vec_compare_int", C.c_int64(1)), ("tg_vec_arith_int", C.c_int64(1)),
                        ("tg_vec_compare_real", C.c_double(1.0)), ("tg_vec_arith_real", C.c_double(1.0))):
        signs = (0, 0) if name.endswith("_int") else ()
        for a, b in ((narrow, None), (narrow, wide), (wide, narrow)):
            res, nulls = np.full(5, 0x5A5A5A5A, np.int64), np.full(1, 0xA5, np.uint8)
            rc = getattr(lib, name)(0, 0, abi.CMP_LT, *signs, C.byref(a), None if b is None else C.byref(b), const,
                                    res.ctypes.data_as(C.c_void_p), nulls.ctypes.data_as(C.c_void_p), None)
            assert rc == abi.TG_ERR_UNSUPPORTED, (name, a is narrow, b is narrow)
            assert b"8-byte columns" in lib.tg_last_error()
            assert (res == 0x5A5A5A5A).all() and nulls[0] == 0xA5


def test_partition_function_is_stable(lib):
    # host mirror of the device partition function: spreads keys, deterministic
    import collections
    cnt = collections.Counter(lib.tg_partition_of_key(k * 2654435761, 8) for k in range(80000))
    assert set(cnt) == set(range(8))
    assert max(cnt.values()) < 1.1 * 10000 and min(cnt.values()) > 0.9 * 10000
    assert lib.tg_partition_of_key(12345, 1) == 0


def test_round2_gates_without_gpu(lib):
    # the planner gates answer on a host without a device: multi-column GROUP BY (up to 4), fused aggregate argument
    # expressions (SUM / AVG over two DOUBLE columns, Complete mode), OtherCondition shapes
    from tidb_b200.plan import OtherCond
    DBL_NN = FieldType(abi.TYPE_DOUBLE, abi.FLAG_NOT_NULL)
    def agg_rc(plan):
        d, keep = plan.to_struct()
        return lib.tg_agg_supported(C.byref(d))
    cols = [INT_NN] * 5 + [DBL_NN, DBL_NN]
    assert agg_rc(AggPlan(cols, [0, 1, 2, 3], [AggFunc(abi.AGG_FIRSTROW, 2), AggFunc(abi.AGG_COUNT, -1)])) == abi.TG_OK
    assert agg_rc(AggPlan(cols, [0, 1, 2, 3, 4], [AggFunc(abi.AGG_COUNT, -1)])) == abi.TG_ERR_UNSUPPORTED
    assert agg_rc(AggPlan(cols, [0], [AggFunc(abi.AGG_FIRSTROW, 1)])) == abi.TG_ERR_UNSUPPORTED           # FIRSTROW of a non-group column
    ok = AggFunc(abi.AGG_SUM, 5, abi.TYPE_DOUBLE, arg_col2=6, arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=1.0)
    assert agg_rc(AggPlan(cols, [0], [ok])) == abi.TG_OK
    assert agg_rc(AggPlan(cols, [0], [AggFunc(abi.AGG_MAX, 5, abi.TYPE_DOUBLE, arg_col2=6, arg_expr=abi.ARGEXPR_MUL)])) == abi.TG_ERR_UNSUPPORTED
    assert agg_rc(AggPlan(cols, [0], [AggFunc(abi.AGG_SUM, 5, abi.TYPE_DOUBLE, arg_col2=1, arg_expr=abi.ARGEXPR_MUL)])) == abi.TG_ERR_UNSUPPORTED   # int operand
    def join_rc(plan):
        d, keep = plan.to_struct()
        return lib.tg_join_supported(C.byref(d))
    oc = [OtherCond(abi.CMP_LT, 0, 1, 1, 1)]
    assert join_rc(JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0], other_cond=oc)) == abi.TG_OK
    assert join_rc(JoinPlan(abi.JOIN_LEFT_OUTER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0], build_is_right=False, other_cond=oc)) == abi.TG_ERR_UNSUPPORTED
    assert join_rc(JoinPlan(abi.JOIN_INNER, [INT_NN, INT_NN], [INT_NN, INT_NN], [0], [0], other_cond=[OtherCond(abi.CMP_LT, 0, 5, 1, 1)])) == abi.TG_ERR_INVALID


def test_multi_column_join_key_gates_without_gpu(lib):
    # several equal conditions (FixedSerializedKey mode, join_table_meta.go:174-178): 2..4 8-byte integer-family key columns
    # on the shapes that need no build-side scan and no NULL-aware flag; everything else is declined, never mis-evaluated
    from tidb_b200.plan import OtherCond
    DBL = FieldType(abi.TYPE_DOUBLE, 0)
    I32 = FieldType(abi.TYPE_LONG, 0)
    def rc(plan):
        d, keep = plan.to_struct()
        return lib.tg_join_supported(C.byref(d))
    four = [INT_NN] * 5
    assert rc(JoinPlan(abi.JOIN_INNER, four, four, [0, 1], [1, 0])) == abi.TG_OK
    assert rc(JoinPlan(abi.JOIN_INNER, four, four, [0, 1, 2, 3], [0, 1, 2, 3], build_is_right=False)) == abi.TG_OK
    assert rc(JoinPlan(abi.JOIN_LEFT_OUTER, four, four, [0, 1], [0, 1], build_is_right=True)) == abi.TG_OK
    assert rc(JoinPlan(abi.JOIN_ANTI_SEMI, four, four, [0, 1], [0, 1], build_is_right=True, rused=[])) == abi.TG_OK
    assert rc(JoinPlan(abi.JOIN_INNER, four, four, [0, 1, 2, 3, 4], [0, 1, 2, 3, 4])) == abi.TG_ERR_UNSUPPORTED        # > 4 keys
    assert rc(JoinPlan(abi.JOIN_LEFT_OUTER, four, four, [0, 1], [0, 1], build_is_right=False)) == abi.TG_ERR_UNSUPPORTED   # build-side scan
    assert rc(JoinPlan(abi.JOIN_LEFT_OUTER_SEMI, four, four, [0, 1], [0, 1], rused=[])) == abi.TG_ERR_UNSUPPORTED        # NULL-aware flag
    assert rc(JoinPlan(abi.JOIN_INNER, [INT_NN, DBL], [INT_NN, DBL], [0, 1], [0, 1])) == abi.TG_ERR_UNSUPPORTED          # real key column
    assert rc(JoinPlan(abi.JOIN_INNER, [INT_NN, I32], [INT_NN, I32], [0, 1], [0, 1])) == abi.TG_OK                       # INT is 8 bytes in a chunk (chunk/codec.go:153)
    assert rc(JoinPlan(abi.JOIN_INNER, four, four, [0, 9], [0, 1])) == abi.TG_ERR_INVALID
    # the residual key equalities share the 8 OtherCondition item slots
    oc = [OtherCond(abi.CMP_LT, 0, 4, 1, 4)] * 5
    assert rc(JoinPlan(abi.JOIN_INNER, four, four, [0, 1, 2], [0, 1, 2], other_cond=oc)) == abi.TG_OK
    assert rc(JoinPlan(abi.JOIN_INNER, four, four, [0, 1, 2, 3], [0, 1, 2, 3], other_cond=oc)) == abi.TG_ERR_UNSUPPORTED


def test_time_join_key_gates_without_gpu(lib):
    # DATE / DATETIME / TIMESTAMP join keys (getKeyProp join_table_meta.go:154) are offloaded against each other only
    DT, D, TS = FieldType(abi.TYPE_DATETIME, 0), FieldType(abi.TYPE_DATE, 0), FieldType(abi.TYPE_TIMESTAMP, 0)
    def rc(plan):
        d, keep = plan.to_struct()
        return lib.tg_join_supported(C.byref(d))
    assert rc(JoinPlan(abi.JOIN_INNER, [DT], [D], [0], [0])) == abi.TG_OK
    assert rc(JoinPlan(abi.JOIN_LEFT_OUTER, [TS, INT_NN], [DT], [0], [0], build_is_right=False)) == abi.TG_OK
    assert rc(JoinPlan(abi.JOIN_INNER, [DT], [INT_NN], [0], [0])) == abi.TG_ERR_UNSUPPORTED
    assert rc(JoinPlan(abi.JOIN_INNER, [FieldType(abi.TYPE_DOUBLE, 0)], [D], [0], [0])) == abi.TG_ERR_UNSUPPORTED
    assert rc(JoinPlan(abi.JOIN_INNER, [DT, INT_NN], [D, INT_NN], [0, 1], [0, 1])) == abi.TG_ERR_UNSUPPORTED   # several keys: integer family only
