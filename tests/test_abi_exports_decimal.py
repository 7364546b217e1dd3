"""CPU-side checks of the DECIMAL SUM / AVG boundary: tg_agg_func keeps its size and offsets (ret_type / ret_frac take the
place of a reserved word), and tg_agg_supported accepts exactly the DECIMAL plans the kernels run."""
import ctypes as C
import os
import re

import pytest

from tidb_b200 import abi
from tidb_b200.executor import HashAggExec, MockDataSource, np_dtype_of
from tidb_b200.plan import AggFunc, AggPlan, FieldType

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEC = abi.TYPE_NEWDECIMAL
INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
UINT = FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED)
DBL = FieldType(abi.TYPE_DOUBLE, 0)


@pytest.fixture(scope="module")
def lib():
    from tidb_b200 import build
    build.build()
    return abi.load_lib()


def rc(lib, cols, funcs, group_by=(0,)):
    d, keep = AggPlan(cols, list(group_by), funcs).to_struct()
    return lib.tg_agg_supported(C.byref(d))


def test_agg_func_layout_unchanged():
    assert C.sizeof(abi.TgAggFunc) == 40
    assert abi.TgAggFunc.ret_type.offset == 28 and abi.TgAggFunc.ret_frac.offset == 30
    assert abi.TgAggFunc.arg_const.offset == 32
    hdr = open(os.path.join(ROOT, "include", "tidbgpu.h")).read()
    body = re.search(r"typedef struct tg_agg_func \{(.*?)\} tg_agg_func;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"\b(u?int\d+_t|double)\s+(\w+);", body)
    assert fields[-3:] == [("int16_t", "ret_type"), ("int16_t", "ret_frac"), ("double", "arg_const")]
    d, keep = AggPlan([INT, INT], [0], [AggFunc(abi.AGG_AVG, 1, ret_type=DEC, ret_frac=7)]).to_struct()
    assert (d.funcs[0].ret_type, d.funcs[0].ret_frac) == (DEC, 7)


def test_accepts_integer_sum_and_avg(lib):
    cols = [INT, INT, INT_NN, UINT, FieldType(abi.TYPE_LONG, 0), FieldType(abi.TYPE_TINY, 0), FieldType(abi.TYPE_YEAR, 0)]
    for c in range(1, len(cols)):
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, c, ret_type=DEC)]) == abi.TG_OK, c
        for f in (0, 4, 9, 30):
            assert rc(lib, cols, [AggFunc(abi.AGG_AVG, c, ret_type=DEC, ret_frac=f)]) == abi.TG_OK, (c, f)
    # mixed with the DOUBLE aggregates, no GROUP BY, several GROUP BY columns
    mixed = [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 1, ret_type=DEC), AggFunc(abi.AGG_COUNT, -1),
             AggFunc(abi.AGG_MIN, 1), AggFunc(abi.AGG_MAX, 3), AggFunc(abi.AGG_SUM, 7, abi.TYPE_DOUBLE),
             AggFunc(abi.AGG_AVG, 2, ret_type=DEC, ret_frac=4)]
    assert rc(lib, cols + [DBL], mixed) == abi.TG_OK
    assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 1, ret_type=DEC)], group_by=()) == abi.TG_OK
    assert rc(lib, cols, [AggFunc(abi.AGG_FIRSTROW, 0), AggFunc(abi.AGG_SUM, 3, ret_type=DEC)], group_by=(0, 1, 2)) == abi.TG_OK


def test_ret_type_zero_and_other_types_keep_todays_answers(lib):
    # SUM / AVG of an integer column without a DECIMAL ret_type are declined as before; DOUBLE ones run as before
    assert rc(lib, [INT_NN, INT_NN], [AggFunc(abi.AGG_SUM, 1, abi.TYPE_LONGLONG)]) == abi.TG_ERR_UNSUPPORTED
    assert rc(lib, [INT_NN, INT_NN], [AggFunc(abi.AGG_AVG, 1, abi.TYPE_LONGLONG)]) == abi.TG_ERR_UNSUPPORTED
    assert rc(lib, [INT_NN, INT_NN], [AggFunc(abi.AGG_SUM, 1, ret_type=abi.TYPE_LONGLONG)]) == abi.TG_ERR_UNSUPPORTED
    assert rc(lib, [INT_NN, DBL], [AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE, ret_type=abi.TYPE_DOUBLE)]) == abi.TG_OK
    assert rc(lib, [INT_NN, DBL], [AggFunc(abi.AGG_AVG, 1, abi.TYPE_DOUBLE)]) == abi.TG_OK


def test_invalid_scale(lib):
    cols = [INT, INT]
    assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 1, ret_type=DEC, ret_frac=1)]) == abi.TG_ERR_INVALID
    assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 1, ret_type=DEC, ret_frac=-1)]) == abi.TG_ERR_INVALID
    assert rc(lib, cols, [AggFunc(abi.AGG_AVG, 1, ret_type=DEC, ret_frac=31)]) == abi.TG_ERR_INVALID
    assert rc(lib, cols, [AggFunc(abi.AGG_AVG, 1, ret_type=DEC, ret_frac=-1)]) == abi.TG_ERR_INVALID


def test_declined_shapes(lib):
    cols = [INT, INT, DBL, DBL, FieldType(abi.TYPE_DURATION, 0), FieldType(DEC, 0)]
    U = abi.TG_ERR_UNSUPPORTED
    assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, ret_type=DEC)]) == U           # DOUBLE argument
    assert rc(lib, cols, [AggFunc(abi.AGG_AVG, 2, abi.TYPE_DOUBLE, ret_type=DEC, ret_frac=4)]) == U
    assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 4, ret_type=DEC)]) == U                             # DURATION argument
    assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 5, ret_type=DEC)]) == U                             # DECIMAL input column
    for name in (abi.AGG_COUNT, abi.AGG_MIN, abi.AGG_MAX, abi.AGG_FIRSTROW):                     # another function
        assert rc(lib, cols, [AggFunc(name, 1, ret_type=DEC)]) == U, name
    for mode in (abi.AGGMODE_FINAL, abi.AGGMODE_PARTIAL2):                                        # DECIMAL partial results
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 1, ret_type=DEC, mode=mode)]) == U, mode
    assert rc(lib, cols, [AggFunc(abi.AGG_AVG, 1, ret_type=DEC, ret_frac=4, mode=abi.AGGMODE_FINAL, arg_col2=0)]) == U
    for expr in (abi.ARGEXPR_MUL, abi.ARGEXPR_MUL_CSUB):                                          # a fused expression
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 1, ret_type=DEC, arg_col2=0, arg_expr=expr)]) == U, expr
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, ret_type=DEC, arg_col2=3, arg_expr=expr)]) == U, expr


def test_state_word_gate(lib):
    # a nullable DECIMAL SUM takes three state words, a NOT NULL one two; the table has 24 state slots
    cols = [INT_NN, INT, INT_NN]
    assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 1, ret_type=DEC)] * 8) == abi.TG_OK                   # 24
    assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 1, ret_type=DEC)] * 9) == abi.TG_ERR_UNSUPPORTED      # 27
    assert rc(lib, cols, [AggFunc(abi.AGG_AVG, 2, ret_type=DEC, ret_frac=4)] * 12) == abi.TG_OK       # 24
    assert rc(lib, cols, [AggFunc(abi.AGG_AVG, 2, ret_type=DEC, ret_frac=4)] * 11 + [AggFunc(abi.AGG_SUM, 1, ret_type=DEC)]) == abi.TG_ERR_UNSUPPORTED


def test_result_schema():
    plan = AggPlan([INT, INT, DBL], [0], [AggFunc(abi.AGG_SUM, 1, ret_type=DEC), AggFunc(abi.AGG_AVG, 1, ret_type=DEC, ret_frac=4),
                                           AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE)])
    e = HashAggExec(plan, MockDataSource(plan.col_types, []))
    assert [t.tp for t in e.schema] == [DEC, DEC, abi.TYPE_DOUBLE]
    import numpy as np
    assert np.dtype(np_dtype_of(e.schema[0])).itemsize == 40
    empty = e.empty_chunk()
    assert empty.columns[0].elem_len == 40 and empty.columns[0].data.shape == (0, 40)
