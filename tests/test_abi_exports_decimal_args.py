"""CPU-side checks of aggregates over DECIMAL(p <= 18, s) columns: the tg_agg_desc_ex layout, every accept / decline /
invalid rule of tg_agg_supported_ex, the same plans still declined through tg_agg_supported, and HashAggExec's result
schema."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tidb_b200 import abi
from tidb_b200.executor import HashAggExec, MockDataSource, np_dtype_of
from tidb_b200.plan import AggFunc, AggPlan, FieldType

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEC = abi.TYPE_NEWDECIMAL
OK, U, INV = abi.TG_OK, abi.TG_ERR_UNSUPPORTED, abi.TG_ERR_INVALID
INT = FieldType(abi.TYPE_LONGLONG, 0)
DBL = FieldType(abi.TYPE_DOUBLE, 0)


def dec(p, s, flag=0):
    return FieldType(DEC, flag, p, s)


@pytest.fixture(scope="module")
def lib():
    from tidb_b200 import build
    build.build()
    return abi.load_lib()


def rc(lib, cols, funcs, group_by=(0,), ex=True):
    plan = AggPlan(cols, list(group_by), funcs)
    if ex:
        d, keep = plan.to_struct_ex()
        return lib.tg_agg_supported_ex(C.byref(d))
    d, keep = plan.to_struct()
    return lib.tg_agg_supported(C.byref(d))


def sum_(c, f):
    return AggFunc(abi.AGG_SUM, c, DEC, ret_type=DEC, ret_frac=f)


def avg_(c, f):
    return AggFunc(abi.AGG_AVG, c, DEC, ret_type=DEC, ret_frac=f)


def min_(c, f):
    return AggFunc(abi.AGG_MIN, c, DEC, ret_type=DEC, ret_frac=f)


def max_(c, f):
    return AggFunc(abi.AGG_MAX, c, DEC, ret_type=DEC, ret_frac=f)


def test_desc_ex_layout():
    assert C.sizeof(abi.TgAggDesc) == 64
    assert abi.TgAggDescEx.base.offset == 0
    assert abi.TgAggDescEx.col_flen.offset == 64 and abi.TgAggDescEx.col_decimal.offset == 72
    assert C.sizeof(abi.TgAggDescEx) == 80
    hdr = open(os.path.join(ROOT, "include", "tidbgpu.h")).read()
    body = re.search(r"typedef struct tg_agg_desc_ex \{(.*?)\} tg_agg_desc_ex;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert re.findall(r"(\w+\*?)\s+\**(\w+);", body) == [("tg_agg_desc", "base"), ("int32_t*", "col_flen"), ("int32_t*", "col_decimal")]
    for sym in ("tg_agg_supported_ex", "tg_agg_open_ex"):
        assert sym in abi.EXPORTED_SYMBOLS and re.search(rf"\bint {sym}\(const tg_agg_desc_ex\* desc", hdr)
    # the precision and scale travel per child column; FieldType defaults to "not given"
    assert FieldType(abi.TYPE_LONGLONG, 0) == FieldType(abi.TYPE_LONGLONG, 0, -1, -1)
    d, keep = AggPlan([INT, dec(15, 2), dec(18, 9)], [0], [sum_(1, 2)]).to_struct_ex()
    assert [d.col_flen[i] for i in range(3)] == [-1, 15, 18] and [d.col_decimal[i] for i in range(3)] == [-1, 2, 9]
    assert (d.base.n_cols, d.base.n_funcs, d.base.funcs[0].ret_frac) == (3, 1, 2)


def test_accepts(lib):
    for p, s in ((1, 0), (1, 1), (15, 2), (18, 0), (18, 2), (18, 9), (18, 18)):
        cols = [INT, dec(p, s), dec(p, s, abi.FLAG_NOT_NULL), dec(p, s, abi.FLAG_UNSIGNED)]
        for c in (1, 2, 3):
            for fn in (sum_, min_, max_):
                assert rc(lib, cols, [fn(c, s)]) == OK, (p, s, c, fn)
            for f in sorted({s, min(s + 4, 30), 18 if s <= 18 else s, 30}):
                assert rc(lib, cols, [avg_(c, f)]) == OK, (p, s, c, f)
            assert rc(lib, cols, [AggFunc(abi.AGG_COUNT, c)]) == OK
    # no GROUP BY, several GROUP BY columns, and mixed with DOUBLE SUM, COUNT, integer DECIMAL SUM, integer MIN / MAX
    cols = [INT, INT, dec(15, 2), DBL, dec(18, 9)]
    mixed = [AggFunc(abi.AGG_FIRSTROW, 0), sum_(2, 2), avg_(4, 13), AggFunc(abi.AGG_SUM, 3, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, -1),
             AggFunc(abi.AGG_SUM, 1, ret_type=DEC), AggFunc(abi.AGG_MIN, 1), AggFunc(abi.AGG_MAX, 1), min_(4, 9), max_(2, 2),
             AggFunc(abi.AGG_COUNT, 2)]
    assert rc(lib, cols, mixed) == OK
    assert rc(lib, cols, mixed[1:], group_by=()) == OK
    assert rc(lib, cols, [AggFunc(abi.AGG_FIRSTROW, 0)] + mixed[1:], group_by=(0, 1)) == OK


def test_declines(lib):
    cols = [INT, dec(15, 2), DBL, dec(19, 2), FieldType(DEC, 0), FieldType(DEC, 0, 15, -1), FieldType(DEC, 0, -1, 2)]
    for c in (3, 4, 5, 6):                                   # flen > 18, or flen / decimal not given
        for f in (sum_(c, 2), avg_(c, 6), min_(c, 2), max_(c, 2), AggFunc(abi.AGG_COUNT, c)):
            assert rc(lib, cols, [f]) == U, (c, f)
    for mode in (abi.AGGMODE_FINAL, abi.AGGMODE_PARTIAL2, abi.AGGMODE_PARTIAL1):   # DECIMAL partial results
        for f in (sum_(1, 2), avg_(1, 6), min_(1, 2), AggFunc(abi.AGG_COUNT, 1)):
            f.mode = mode
            assert rc(lib, cols, [f]) == U, (mode, f)
    for expr in (abi.ARGEXPR_MUL, abi.ARGEXPR_MUL_CSUB):   # a DECIMAL column in a fused argument expression
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 1, DEC, ret_type=DEC, ret_frac=2, arg_col2=2, arg_expr=expr)]) == U
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, arg_col2=1, arg_expr=expr)]) == U
    assert rc(lib, cols, [AggFunc(abi.AGG_FIRSTROW, 1)], group_by=(1,)) == U          # a DECIMAL GROUP BY column
    assert rc(lib, cols, [AggFunc(abi.AGG_COUNT, -1)], group_by=(0, 1)) == U
    assert rc(lib, cols, [AggFunc(abi.AGG_FIRSTROW, 1)]) == U                          # FIRSTROW over DECIMAL
    for name in (abi.AGG_SUM, abi.AGG_AVG, abi.AGG_MIN, abi.AGG_MAX):                 # a non-DECIMAL ret_type
        for rt in (0, abi.TYPE_DOUBLE, abi.TYPE_LONGLONG):
            assert rc(lib, cols, [AggFunc(name, 1, DEC, ret_type=rt, ret_frac=2)]) == U, (name, rt)
    assert rc(lib, cols, [AggFunc(abi.AGG_COUNT, 1, DEC, ret_type=DEC)]) == U          # COUNT keeps its BIGINT result


def test_invalid(lib):
    cols = [INT, dec(15, 2), dec(18, 18), dec(5, 6), dec(0, 0)]
    for f in (sum_(1, 0), sum_(1, 3), min_(1, 1), max_(1, 4), avg_(1, 1), avg_(1, 31), sum_(2, 17), avg_(2, 17), avg_(2, 31)):
        assert rc(lib, cols, [f]) == INV, f
    for c in (3, 4):                                         # decimal > flen, flen 0
        assert rc(lib, cols, [sum_(c, 6 if c == 3 else 0)]) == INV, c
        assert rc(lib, cols, [AggFunc(abi.AGG_COUNT, c)]) == INV, c


def test_state_words(lib):
    # SUM / AVG take 2-3 state words, MIN / MAX 1-2, under the same 24-word limit
    cols = [INT, dec(15, 2), dec(15, 2, abi.FLAG_NOT_NULL)]
    assert rc(lib, cols, [sum_(1, 2)] * 8) == OK and rc(lib, cols, [sum_(1, 2)] * 9) == U
    assert rc(lib, cols, [avg_(2, 6)] * 12) == OK
    assert rc(lib, cols, [min_(1, 2)] * 12) == OK and rc(lib, cols, [max_(2, 2)] * 12) == OK
    assert rc(lib, cols, [sum_(1, 2)] * 7 + [min_(1, 2), max_(1, 2)]) == U   # 21 + 4 words


def test_without_ex_every_decimal_plan_stays_declined(lib):
    cols = [INT, dec(15, 2), dec(18, 0)]
    for f in (sum_(1, 2), avg_(1, 6), min_(1, 2), max_(2, 0), AggFunc(abi.AGG_COUNT, 1), sum_(1, 0), avg_(1, 31)):
        assert rc(lib, cols, [f], ex=False) == U, f
    # the _ex call with both arrays NULL is the plain call
    d, keep = AggPlan(cols, [0], [sum_(1, 2)]).to_struct_ex()
    d.col_flen = None
    assert lib.tg_agg_supported_ex(C.byref(d)) == U
    d, keep = AggPlan(cols, [0], [sum_(1, 2)]).to_struct_ex()
    d.col_decimal = None
    assert lib.tg_agg_supported_ex(C.byref(d)) == U
    assert lib.tg_agg_supported_ex(None) == INV
    h = C.c_void_p()
    assert lib.tg_agg_open_ex(None, C.byref(h)) == INV
    # plans without DECIMAL columns answer the same through both calls
    for funcs in ([AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE)], [AggFunc(abi.AGG_SUM, 0, ret_type=DEC)], [AggFunc(abi.AGG_SUM, 0)]):
        assert rc(lib, [INT, DBL], funcs) == rc(lib, [INT, DBL], funcs, ex=False)


def test_result_schema():
    cols = [INT, dec(15, 2), dec(18, 9, abi.FLAG_NOT_NULL), DBL]
    plan = AggPlan(cols, [0], [sum_(1, 2), avg_(1, 6), min_(2, 9), max_(1, 2), AggFunc(abi.AGG_COUNT, 1), avg_(2, 30),
                               AggFunc(abi.AGG_SUM, 3, abi.TYPE_DOUBLE), AggFunc(abi.AGG_FIRSTROW, 0), sum_(2, 9)])
    e = HashAggExec(plan, MockDataSource(plan.col_types, []))
    got = [(t.tp, t.flen, t.decimal, t.not_null) for t in e.schema]
    assert got == [(DEC, 37, 2, False), (DEC, 19, 6, False), (DEC, 18, 9, False), (DEC, 15, 2, False),
                   (abi.TYPE_LONGLONG, -1, -1, True), (DEC, 39, 30, False), (abi.TYPE_DOUBLE, -1, -1, False),
                   (abi.TYPE_LONGLONG, -1, -1, False), (DEC, 40, 9, False)]
    for k in (0, 1, 2, 3, 5, 8):
        assert np.dtype(np_dtype_of(e.schema[k])).itemsize == 40
    empty = e.empty_chunk()
    assert empty.columns[2].elem_len == 40 and empty.columns[2].data.shape == (0, 40)
