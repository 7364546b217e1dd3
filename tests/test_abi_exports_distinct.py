"""CPU-side checks of COUNT / SUM / AVG with DISTINCT: the tg_agg_desc_ex2 and tg_agg_distinct_stats layouts against the
header, every accept / decline / invalid rule of tg_agg_supported_ex2, and the same answer as tg_agg_supported_ex for
every plan without DISTINCT."""
import ctypes as C
import os
import re

import pytest

from tidb_b200 import abi
from tidb_b200.plan import AggFunc, AggPlan, FieldType

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEC = abi.TYPE_NEWDECIMAL
OK, U, INV = abi.TG_OK, abi.TG_ERR_UNSUPPORTED, abi.TG_ERR_INVALID
INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
UINT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED)
DBL = FieldType(abi.TYPE_DOUBLE, 0)


def dec(p, s, flag=0):
    return FieldType(DEC, flag, p, s)


@pytest.fixture(scope="module")
def lib():
    from tidb_b200 import build
    build.build()
    return abi.load_lib()


def rc(lib, cols, funcs, group_by=(0,)):
    d, keep = AggPlan(cols, list(group_by), funcs).to_struct_ex2()
    return lib.tg_agg_supported_ex2(C.byref(d))


def rc_ex(lib, cols, funcs, group_by=(0,)):
    d, keep = AggPlan(cols, list(group_by), funcs).to_struct_ex()
    return lib.tg_agg_supported_ex(C.byref(d))


def cnt(c, **kw):
    return AggFunc(abi.AGG_COUNT, c, distinct=True, **kw)


def test_layout():
    assert abi.TgAggDescEx2.ex.offset == 0 and abi.TgAggDescEx2.has_distinct.offset == C.sizeof(abi.TgAggDescEx) == 80
    assert C.sizeof(abi.TgAggDescEx2) == 88
    assert [(n, getattr(abi.TgAggDistinctStats, n).offset) for n, _ in abi.TgAggDistinctStats._fields_] == \
        [("pairs", 0), ("set_slots", 8), ("set_grows", 16), ("launches", 24), ("mark_ms", 32)]
    assert C.sizeof(abi.TgAggDistinctStats) == 40
    hdr = open(os.path.join(ROOT, "include", "tidbgpu.h")).read()

    def fields(name):
        body = re.search(rf"typedef struct {name} \{{(.*?)\}} {name};", hdr, re.S).group(1)
        return re.findall(r"(\w+\*?)\s+\**(\w+)[;,]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))

    assert fields("tg_agg_desc_ex2") == [("tg_agg_desc_ex", "ex"), ("uint8_t*", "has_distinct")]
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct tg_agg_distinct_stats \{(.*?)\} tg_agg_distinct_stats;", hdr, re.S).group(1), flags=re.S)
    assert " ".join(body.split()) == "int64_t pairs, set_slots, set_grows, launches; double mark_ms;"
    for sym, arg in (("tg_agg_supported_ex2", "const tg_agg_desc_ex2\\* desc"), ("tg_agg_open_ex2", "const tg_agg_desc_ex2\\* desc"),
                     ("tg_agg_get_distinct_stats", "tg_agg\\* a, tg_agg_distinct_stats\\* out")):
        assert sym in abi.EXPORTED_SYMBOLS and re.search(rf"\bint {sym}\({arg}", hdr), sym
    # the plan renders HasDistinct per function, and NULL when no function has it
    d, keep = AggPlan([INT, INT], [0], [AggFunc(abi.AGG_FIRSTROW, 0), cnt(1), AggFunc(abi.AGG_COUNT, 1)]).to_struct_ex2()
    assert [d.has_distinct[i] for i in range(3)] == [0, 1, 0] and d.ex.base.n_funcs == 3
    d, keep = AggPlan([INT, INT], [0], [AggFunc(abi.AGG_COUNT, 1)]).to_struct_ex2()
    assert not d.has_distinct


def test_accepts(lib):
    int_cols = [INT, INT, INT_NN, UINT] + [FieldType(t, 0) for t in (abi.TYPE_TINY, abi.TYPE_SHORT, abi.TYPE_INT24, abi.TYPE_LONG,
                                                                     abi.TYPE_YEAR, abi.TYPE_DURATION)]
    for c in range(1, len(int_cols)):
        assert rc(lib, int_cols, [cnt(c)]) == OK, c
        if int_cols[c].tp != abi.TYPE_DURATION:   # DECIMAL SUM / AVG take no DURATION argument, with or without DISTINCT
            assert rc(lib, int_cols, [AggFunc(abi.AGG_SUM, c, ret_type=DEC, distinct=True)]) == OK, c
            assert rc(lib, int_cols, [AggFunc(abi.AGG_AVG, c, ret_type=DEC, ret_frac=4, distinct=True)]) == OK, c
        for name in (abi.AGG_MIN, abi.AGG_MAX):
            assert rc(lib, int_cols, [AggFunc(name, c, distinct=True)]) == OK
    cols = [INT, DBL, dec(15, 2), dec(18, 18, abi.FLAG_NOT_NULL), dec(18, 0)]
    for c in (1,):
        for name in (abi.AGG_COUNT, abi.AGG_SUM, abi.AGG_AVG, abi.AGG_MIN, abi.AGG_MAX):
            assert rc(lib, cols, [AggFunc(name, c, abi.TYPE_DOUBLE, distinct=True)]) == OK, name
    for c in (2, 3, 4):
        s = cols[c].decimal
        assert rc(lib, cols, [cnt(c)]) == OK
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, c, DEC, ret_type=DEC, ret_frac=s, distinct=True)]) == OK
        assert rc(lib, cols, [AggFunc(abi.AGG_AVG, c, DEC, ret_type=DEC, ret_frac=min(s + 4, 30), distinct=True)]) == OK
        assert rc(lib, cols, [AggFunc(abi.AGG_MAX, c, DEC, ret_type=DEC, ret_frac=s, distinct=True)]) == OK
    # no GROUP BY, four GROUP BY columns with NULLs, two DISTINCT columns, DISTINCT next to the plain function
    mixed = [cnt(1), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE, distinct=True), AggFunc(abi.AGG_COUNT, 1), cnt(2),
             AggFunc(abi.AGG_AVG, 2, DEC, ret_type=DEC, ret_frac=6, distinct=True), AggFunc(abi.AGG_COUNT, -1)]
    assert rc(lib, cols, mixed, group_by=()) == OK
    assert rc(lib, cols + [INT, INT_NN, INT], [AggFunc(abi.AGG_FIRSTROW, 0)] + mixed, group_by=(0, 5, 6, 7)) == OK
    # the free column slots: 14 child columns + 2 DISTINCT columns fit, 15 + 2 do not
    wide = [INT] * 13 + [DBL]
    two = [cnt(12), cnt(13), AggFunc(abi.AGG_SUM, 13, abi.TYPE_DOUBLE, distinct=True)]
    assert rc(lib, wide, two) == OK
    assert rc(lib, wide + [INT], two) == U
    assert rc(lib, [INT] * 16, [cnt(1)]) == U
    assert rc(lib, [INT] * 16, [AggFunc(abi.AGG_MAX, 1, distinct=True)]) == OK   # MIN / MAX take no set


def test_declines(lib):
    cols = [INT, INT, DBL, FieldType(abi.TYPE_FLOAT, 0), FieldType(abi.TYPE_DATETIME, 0), FieldType(abi.TYPE_DATE, 0),
            FieldType(abi.TYPE_TIMESTAMP, 0), FieldType(abi.TYPE_VARSTRING, 0), dec(19, 2), dec(30, 4), FieldType(DEC, 0)]
    for c in range(3, len(cols)):   # FLOAT, date-time, string, DECIMAL(p > 18) or without precision
        assert rc(lib, cols, [cnt(c)]) == U, c
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, c, ret_type=DEC, distinct=True)]) == U, c
    for mode in (abi.AGGMODE_FINAL, abi.AGGMODE_PARTIAL1, abi.AGGMODE_PARTIAL2):
        for f in (cnt(1), AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, distinct=True), AggFunc(abi.AGG_AVG, 2, abi.TYPE_DOUBLE, distinct=True)):
            f.mode = mode
            assert rc(lib, cols, [f]) == U, (mode, f)
    for expr in (abi.ARGEXPR_MUL, abi.ARGEXPR_MUL_CSUB):   # DISTINCT over an argument expression
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, arg_col2=2, arg_expr=expr)]) == OK
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, arg_col2=2, arg_expr=expr, distinct=True)]) == U
    assert rc(lib, cols, [cnt(1, arg_col2=2)]) == U                                        # COUNT(DISTINCT a, b)
    assert rc(lib, cols, [AggFunc(abi.AGG_FIRSTROW, 0, distinct=True)]) == U
    # the twin without DISTINCT is declined, so DISTINCT is too
    assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 1, distinct=True)]) == U                     # SUM(int) needs DECIMAL
    assert rc_ex(lib, cols, [AggFunc(abi.AGG_SUM, 1)]) == U
    assert rc(lib, [INT, dec(15, 2)], [AggFunc(abi.AGG_COUNT, 1, ret_type=DEC, distinct=True)]) == U
    # the 24-word limit counts a DISTINCT COUNT's own count word
    assert rc(lib, [INT, INT_NN], [AggFunc(abi.AGG_SUM, 1, ret_type=DEC)] * 9) == OK                      # 9 x 2 words
    assert rc(lib, [INT, INT_NN], [AggFunc(abi.AGG_SUM, 1, ret_type=DEC, distinct=True)] * 8) == OK       # 8 x 3 words
    assert rc(lib, [INT, INT_NN], [AggFunc(abi.AGG_SUM, 1, ret_type=DEC, distinct=True)] * 9) == U        # 9 x 3 words
    assert rc(lib, [INT, INT_NN], [AggFunc(abi.AGG_COUNT, 1)] * 12) == OK
    assert rc(lib, [INT, INT_NN], [cnt(1)] * 12) == OK


def test_invalid(lib):
    cols = [INT, INT, dec(15, 2), dec(5, 6)]
    for name in (abi.AGG_COUNT, abi.AGG_SUM, abi.AGG_AVG, abi.AGG_MIN, abi.AGG_MAX):
        assert rc(lib, cols, [AggFunc(name, -1, ret_type=DEC, distinct=True)]) == INV, name
    assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 2, DEC, ret_type=DEC, ret_frac=3, distinct=True)]) == INV   # the twin's scale rule
    assert rc(lib, cols, [cnt(3)]) == INV                                                                   # decimal > flen
    assert rc(lib, cols, [cnt(7)]) == INV                                                                   # out of range
    assert lib.tg_agg_supported_ex2(None) == INV
    h = C.c_void_p()
    assert lib.tg_agg_open_ex2(None, C.byref(h)) == INV


def _existing_plans():
    cols = [INT, DBL, dec(15, 2), INT_NN, UINT, dec(19, 2), FieldType(abi.TYPE_DATETIME, 0)]
    fs = [AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_COUNT, 1), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE), AggFunc(abi.AGG_AVG, 1, abi.TYPE_DOUBLE),
          AggFunc(abi.AGG_SUM, 0, ret_type=DEC), AggFunc(abi.AGG_AVG, 3, ret_type=DEC, ret_frac=4), AggFunc(abi.AGG_SUM, 0),
          AggFunc(abi.AGG_SUM, 2, DEC, ret_type=DEC, ret_frac=2), AggFunc(abi.AGG_AVG, 2, DEC, ret_type=DEC, ret_frac=1),
          AggFunc(abi.AGG_MIN, 4), AggFunc(abi.AGG_MAX, 2, DEC, ret_type=DEC, ret_frac=2), AggFunc(abi.AGG_COUNT, 5),
          AggFunc(abi.AGG_COUNT, 6), AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_FIRSTROW, 1),
          AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE, arg_col2=1, arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=1.0),
          AggFunc(abi.AGG_SUM, 2, DEC, ret_type=DEC, ret_frac=4, arg_col2=2, arg_expr=abi.ARGEXPR_MUL),
          AggFunc(abi.AGG_AVG, 2, DEC, ret_type=DEC, ret_frac=4, arg_col2=2, arg_expr=abi.ARGEXPR_MUL_CSUB, arg_const=3.0),
          AggFunc(abi.AGG_COUNT, 3, mode=abi.AGGMODE_FINAL), AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE, mode=abi.AGGMODE_PARTIAL1),
          AggFunc(abi.AGG_COUNT, 9), AggFunc(abi.AGG_SUM, 2, DEC, ret_type=DEC, ret_frac=5)]
    for gb in ((0,), (), (0, 3), (1,), (2,)):
        for f in fs:
            yield cols, [f], gb
        yield cols, fs[:12], gb
        yield cols, fs[:4] + fs[7:9], gb


def test_without_distinct_ex2_answers_like_ex(lib):
    n = 0
    for cols, funcs, gb in _existing_plans():
        want = rc_ex(lib, cols, funcs, gb)
        d, keep = AggPlan(cols, list(gb), funcs).to_struct_ex2()
        assert not d.has_distinct
        assert lib.tg_agg_supported_ex2(C.byref(d)) == want, (funcs, gb)
        zeros = (C.c_uint8 * len(funcs))()
        d.has_distinct = zeros
        assert lib.tg_agg_supported_ex2(C.byref(d)) == want, (funcs, gb)
        n += 1
    assert n > 100
