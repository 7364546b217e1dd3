"""CPU-side checks of string GROUP BY in the hash aggregation: the tg_agg_desc_ex3, tg_mut_varlen and
tg_agg_string_stats layouts against the header, every accept / decline rule of tg_agg_supported_ex3, ex3 with no
collations answering as ex2, and tg_agg_open_ex3 checking its arguments before it looks for a device."""
import ctypes as C
import os
import re

import pytest

from tidb_b200 import abi
from tidb_b200.plan import AggFunc, AggPlan, FieldType

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, U, INV = abi.TG_OK, abi.TG_ERR_UNSUPPORTED, abi.TG_ERR_INVALID
INT = FieldType(abi.TYPE_LONGLONG, 0)
DBL = FieldType(abi.TYPE_DOUBLE, 0)
DEC = FieldType(abi.TYPE_NEWDECIMAL, 0, 15, 2)
COLLATIONS = (63, 46, 83, 65, 47, 309)


def s(coll=46, tp=abi.TYPE_VARCHAR, flag=0):
    return FieldType(tp, flag, collation=coll)


@pytest.fixture(scope="module")
def lib():
    from tidb_b200 import build
    build.build()
    return abi.load_lib()


def rc3(lib, cols, funcs, group_by=(0,), colls=True):
    d, keep = AggPlan(cols, list(group_by), funcs).to_struct_ex3()
    if not colls:
        d.col_collation = None
    return lib.tg_agg_supported_ex3(C.byref(d))


def rc2(lib, cols, funcs, group_by=(0,)):
    d, keep = AggPlan(cols, list(group_by), funcs).to_struct_ex2()
    return lib.tg_agg_supported_ex2(C.byref(d))


def fr(c):
    return AggFunc(abi.AGG_FIRSTROW, c)


def test_layout():
    assert abi.TgAggDescEx3.ex2.offset == 0 and abi.TgAggDescEx3.col_collation.offset == C.sizeof(abi.TgAggDescEx2) == 88
    assert C.sizeof(abi.TgAggDescEx3) == 96
    assert [(n, getattr(abi.TgMutVarlen, n).offset) for n, _ in abi.TgMutVarlen._fields_] == [("offsets", 0), ("data", 8), ("data_cap", 16)]
    assert C.sizeof(abi.TgMutVarlen) == 24
    assert [(n, getattr(abi.TgAggStringStats, n).offset) for n, _ in abi.TgAggStringStats._fields_] == \
        [("dict_entries", 0), ("dict_bytes", 8), ("dict_slots", 16), ("dict_grows", 24), ("launches", 32), ("encode_ms", 40)]
    assert C.sizeof(abi.TgAggStringStats) == 48
    hdr = open(os.path.join(ROOT, "include", "tidbgpu.h")).read()
    assert re.search(r"typedef struct tg_agg_desc_ex3 \{\s*tg_agg_desc_ex2 ex2;.*?const int32_t\* col_collation;.*?\} tg_agg_desc_ex3;", hdr, re.S)
    assert "typedef struct tg_mut_varlen { int64_t* offsets; uint8_t* data; int64_t data_cap; } tg_mut_varlen;" in hdr
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct tg_agg_string_stats \{(.*?)\} tg_agg_string_stats;", hdr, re.S).group(1), flags=re.S)
    assert " ".join(body.split()) == "int64_t dict_entries, dict_bytes, dict_slots, dict_grows, launches; double encode_ms;"
    assert "TG_AGG_PATH_STRING_KEY = 0x80" in hdr and abi.AGG_PATH_STRING_KEY == 1 << 7
    for sym, args in (("tg_agg_supported_ex3", "const tg_agg_desc_ex3\\* desc"), ("tg_agg_open_ex3", "const tg_agg_desc_ex3\\* desc, tg_agg\\*\\* out"),
                      ("tg_agg_next_ex", "tg_agg\\* a, tg_mut_chunk\\* out, tg_mut_varlen\\* var_out, int64_t max_rows, int64_t\\* nrows"),
                      ("tg_agg_result_dev_ex", "tg_agg\\* a, int64_t\\* out_rows, void\\*\\* out_cols, void\\*\\* out_nulls, void\\*\\* out_offsets"),
                      ("tg_agg_get_string_stats", "tg_agg\\* a, tg_agg_string_stats\\* out")):
        assert sym in abi.EXPORTED_SYMBOLS and re.search(rf"\bint {sym}\({args}\);", hdr), sym
    assert "#define TIDBGPU_ABI_VERSION 2" in hdr
    # the plan renders every column's collation, 46 unless given
    d, keep = AggPlan([s(63), INT], [0], [fr(0)]).to_struct_ex3()
    assert [d.col_collation[i] for i in range(2)] == [63, 46]


def test_exports(lib):
    for sym in ("tg_agg_supported_ex3", "tg_agg_open_ex3", "tg_agg_next_ex", "tg_agg_result_dev_ex", "tg_agg_get_string_stats"):
        assert hasattr(lib, sym), sym


def test_gate_accepts(lib):
    string_types = (abi.TYPE_VARCHAR, abi.TYPE_VARSTRING, abi.TYPE_STRING, abi.TYPE_TINY_BLOB, abi.TYPE_MEDIUM_BLOB,
                    abi.TYPE_LONG_BLOB, abi.TYPE_BLOB)
    for tp in string_types:
        for coll in COLLATIONS:
            assert rc3(lib, [s(coll, tp), INT], [fr(0), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_COUNT, 0)]) == OK, (tp, coll)
    # mixed with integer and DOUBLE keys, up to 4 GROUP BY columns; FIRSTROW of a byte-exact string key with several
    assert rc3(lib, [s(63), INT, DBL, s(309)], [fr(0), fr(1), fr(2), fr(3)], group_by=(0, 1, 2, 3)) == OK
    assert rc3(lib, [s(46), s(47), INT], [AggFunc(abi.AGG_COUNT, -1), fr(2)], group_by=(0, 1, 2)) == OK
    # COUNT(string) without GROUP BY, and under another key; DECIMAL and DISTINCT functions over other columns
    assert rc3(lib, [s(), INT], [AggFunc(abi.AGG_COUNT, 0)], group_by=()) == OK
    assert rc3(lib, [INT, s(17)], [fr(0), AggFunc(abi.AGG_COUNT, 1)]) == OK   # a COUNT argument needs no collation
    assert rc3(lib, [s(), s(), DEC, INT], [fr(0), fr(1), AggFunc(abi.AGG_SUM, 2, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=2),
                                           AggFunc(abi.AGG_COUNT, 3, distinct=True)], group_by=(0, 1)) == OK  # PAD FIRSTROW, 2 keys
    assert rc3(lib, [s(63), s(63), DEC, INT], [fr(0), fr(1), AggFunc(abi.AGG_SUM, 2, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=2),
                                               AggFunc(abi.AGG_AVG, 2, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=6),
                                               AggFunc(abi.AGG_COUNT, 3, distinct=True)], group_by=(0, 1)) == OK


def test_gate_declines(lib):
    for tp in (abi.TYPE_ENUM, abi.TYPE_SET, abi.TYPE_JSON, abi.TYPE_BIT):
        assert rc3(lib, [FieldType(tp, 0), INT], [fr(0)]) == U, tp
        assert rc3(lib, [INT, FieldType(tp, 0)], [fr(0), AggFunc(abi.AGG_COUNT, 1)]) == U, tp
    for coll in (45, 33, 224, 255, 28, 87, 248, 0, -1):   # _ci, gbk, gb18030, none
        assert rc3(lib, [s(coll), INT], [fr(0)]) == U, coll
    assert rc3(lib, [s(), INT, INT, INT, INT], [fr(0)], group_by=(0, 1, 2, 3, 4)) == U   # 5 GROUP BY columns
    for name in (abi.AGG_SUM, abi.AGG_AVG, abi.AGG_MIN, abi.AGG_MAX):
        assert rc3(lib, [INT, s()], [fr(0), AggFunc(name, 1, abi.TYPE_VARCHAR)]) == U, name
        assert rc3(lib, [s(), INT], [fr(0), AggFunc(name, 0, abi.TYPE_VARCHAR)]) == U, name
    assert rc3(lib, [INT, s()], [fr(0), AggFunc(abi.AGG_COUNT, 1, distinct=True)]) == U
    assert rc3(lib, [s(), INT], [AggFunc(abi.AGG_COUNT, 0, distinct=True)]) == U
    assert rc3(lib, [INT, s()], [fr(0), fr(1)]) == U                                       # FIRSTROW of a non-key string
    assert rc3(lib, [s(), s(46), INT], [fr(0), fr(1)], group_by=(0, 2)) == U
    assert rc3(lib, [INT, s(), DBL], [fr(0), AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, arg_col2=1, arg_expr=abi.ARGEXPR_MUL)]) == U
    assert rc3(lib, [INT, s()], [fr(0), AggFunc(abi.AGG_COUNT, 1, mode=abi.AGGMODE_FINAL)]) == U
    # FIRSTROW of a PAD key under several GROUP BY columns takes a free column slot and a hidden aggregate per such key
    assert rc3(lib, [s(46), INT], [fr(0), fr(1)], group_by=(0, 1)) == OK
    assert rc3(lib, [s(46), s(83), s(65), s(47)], [fr(0), fr(1), fr(2), fr(3)], group_by=(0, 1, 2, 3)) == OK
    assert rc3(lib, [s(46)] + [INT] * 15, [fr(0), fr(1)], group_by=(0, 1)) == U                      # no free column slot
    assert rc3(lib, [s(46)] + [INT] * 14, [fr(0), fr(1)], group_by=(0, 1)) == OK
    assert rc3(lib, [s(46), INT], [fr(0), fr(1)] + [AggFunc(abi.AGG_COUNT, -1)] * 10, group_by=(0, 1)) == U   # 13 aggregates
    assert rc3(lib, [s(46), INT], [fr(0), fr(1)] + [AggFunc(abi.AGG_COUNT, -1)] * 9, group_by=(0, 1)) == OK
    assert rc3(lib, [s(63), INT], [fr(0), fr(1)] + [AggFunc(abi.AGG_COUNT, -1)] * 10, group_by=(0, 1)) == OK  # no hidden one


def test_no_collations_answers_as_ex2(lib):
    plans = [
        ([INT, DBL], [fr(0), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE)], (0,)),
        ([INT, INT, DBL], [fr(0), fr(1), AggFunc(abi.AGG_AVG, 2, abi.TYPE_DOUBLE)], (0, 1)),
        ([INT, DEC], [fr(0), AggFunc(abi.AGG_SUM, 1, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=2)], (0,)),
        ([INT, INT], [fr(0), AggFunc(abi.AGG_COUNT, 1, distinct=True)], (0,)),
        ([s(), INT], [fr(0)], (0,)),
        ([INT, s()], [fr(0), AggFunc(abi.AGG_COUNT, 1)], (0,)),
        ([INT, FieldType(abi.TYPE_FLOAT, 0)], [fr(0), AggFunc(abi.AGG_SUM, 1)], (0,)),
        ([INT, DEC], [fr(0), AggFunc(abi.AGG_SUM, 1, ret_type=abi.TYPE_NEWDECIMAL, ret_frac=3)], (0,)),   # INVALID
    ]
    for cols, funcs, gb in plans:
        want = rc2(lib, cols, funcs, gb)
        assert rc3(lib, cols, funcs, gb, colls=False) == want, (cols, funcs)
        if not any(t.tp in abi.STRING_TYPES for t in cols):   # no string column: the collations change nothing
            assert rc3(lib, cols, funcs, gb) == want, (cols, funcs)
    assert rc2(lib, [s(), INT], [fr(0)]) == U


def test_open_checks_arguments_before_the_device(lib):
    if lib.tg_device_count() > 0:
        pytest.skip("the no-device answer needs a machine without a CUDA device")
    for plan, want in ((AggPlan([s(46), INT], [0], [fr(0)]), abi.TG_ERR_CUDA),
                       (AggPlan([s(45), INT], [0], [fr(0)]), U),
                       (AggPlan([INT, s()], [0], [fr(0), AggFunc(abi.AGG_MAX, 1)]), U)):
        d, keep = plan.to_struct_ex3()
        h = C.c_void_p()
        assert lib.tg_agg_open_ex3(C.byref(d), C.byref(h)) == want
        assert not h.value
