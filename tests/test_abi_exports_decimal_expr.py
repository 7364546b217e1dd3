"""CPU-side checks of SUM / AVG over a product of DECIMAL(p <= 18) columns (a * b, a * (c - b)): every accept / decline /
invalid rule of tg_agg_supported_ex, the plain call still declining, the state-word count, and HashAggExec's result
schema."""
import ctypes as C
import math

import pytest

from tidb_b200 import abi
from tidb_b200.executor import HashAggExec, MockDataSource
from tidb_b200.plan import AggFunc, AggPlan, FieldType

DEC = abi.TYPE_NEWDECIMAL
OK, U, INV = abi.TG_OK, abi.TG_ERR_UNSUPPORTED, abi.TG_ERR_INVALID
MUL, CSUB = abi.ARGEXPR_MUL, abi.ARGEXPR_MUL_CSUB
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
    d, keep = plan.to_struct_ex() if ex else plan.to_struct()
    return (lib.tg_agg_supported_ex if ex else lib.tg_agg_supported)(C.byref(d))


def xsum(a, b, f, expr=MUL, c=0.0, mode=abi.AGGMODE_COMPLETE, ret_type=DEC):
    return AggFunc(abi.AGG_SUM, a, DEC, mode=mode, ret_type=ret_type, ret_frac=f, arg_col2=b, arg_expr=expr, arg_const=c)


def xavg(a, b, f, expr=MUL, c=0.0, mode=abi.AGGMODE_COMPLETE, ret_type=DEC):
    return AggFunc(abi.AGG_AVG, a, DEC, mode=mode, ret_type=ret_type, ret_frac=f, arg_col2=b, arg_expr=expr, arg_const=c)


def test_accepts(lib):
    for (pa, sa), (pb, sb) in (((1, 0), (1, 0)), ((15, 2), (15, 2)), ((18, 0), (18, 0)), ((18, 9), (18, 9)), ((18, 18), (18, 0)),
                               ((18, 12), (18, 18)), ((1, 1), (18, 18))):
        cols = [INT, dec(pa, sa), dec(pb, sb), dec(pa, sa, abi.FLAG_NOT_NULL), dec(pb, sb, abi.FLAG_NOT_NULL)]
        for a, b in ((1, 2), (3, 4), (1, 4), (3, 2), (2, 2)):      # either operand nullable; the same column twice
            s = cols[a].decimal + cols[b].decimal
            if s > 30:                                          # 18 + 18: declined below
                continue
            for expr, c in ((MUL, 0.0), (CSUB, 1.0), (CSUB, -1.0), (CSUB, 0.0), (CSUB, float(10 ** (18 - sb)))):
                assert rc(lib, cols, [xsum(a, b, s, expr, c)]) == OK, (pa, sa, pb, sb, a, b, expr, c)
                for f in sorted({s, min(s + 4, 30), 30}):
                    assert rc(lib, cols, [xavg(a, b, f, expr, c)]) == OK, (pa, sa, pb, sb, a, b, f)
    # the Q1 / Q3 / Q6 shapes over DECIMAL(15,2), with no GROUP BY, one and three GROUP BY columns, mixed with other functions
    cols = [INT, INT, INT, dec(15, 2), dec(15, 2, abi.FLAG_NOT_NULL), DBL]
    mixed = [AggFunc(abi.AGG_FIRSTROW, 0), xsum(3, 4, 4, CSUB, 1.0), xsum(3, 4, 4), xavg(3, 4, 8, CSUB, 1.0),
             AggFunc(abi.AGG_SUM, 5, abi.TYPE_DOUBLE), AggFunc(abi.AGG_COUNT, -1), AggFunc(abi.AGG_SUM, 3, DEC, ret_type=DEC, ret_frac=2)]
    assert rc(lib, cols, mixed) == OK
    assert rc(lib, cols, mixed[1:], group_by=()) == OK
    assert rc(lib, cols, [AggFunc(abi.AGG_FIRSTROW, g) for g in (0, 1, 2)] + [xsum(3, 4, 4, CSUB, 1.0)], group_by=(0, 1, 2)) == OK
    # a decimal literal 1.00 reaches the library as the integer 1.0
    assert rc(lib, cols, [xsum(3, 4, 4, CSUB, 1.00)]) == OK


def test_declines(lib):
    cols = [INT, dec(15, 2), DBL, dec(19, 2), FieldType(DEC, 0), FieldType(DEC, 0, 15, -1), INT, dec(18, 18), dec(18, 13)]
    for expr in (MUL, CSUB):
        for b in (2, 6, 3, 4, 5):                             # DECIMAL x DOUBLE / integer, flen > 18, flen / scale not given
            assert rc(lib, cols, [xsum(1, b, 4, expr, 1.0)]) == U, (expr, b)
            assert rc(lib, cols, [xavg(1, b, 8, expr, 1.0)]) == U, (expr, b)
        for a in (3, 4, 5):
            assert rc(lib, cols, [xsum(a, 1, 4, expr, 1.0)]) == U, (expr, a)
        assert rc(lib, cols, [AggFunc(abi.AGG_SUM, 2, abi.TYPE_DOUBLE, arg_col2=1, arg_expr=expr, arg_const=1.0)]) == U
        for name in (abi.AGG_MIN, abi.AGG_MAX, abi.AGG_COUNT):   # MIN / MAX / COUNT of an expression
            assert rc(lib, cols, [AggFunc(name, 1, DEC, ret_type=DEC, ret_frac=4, arg_col2=1, arg_expr=expr, arg_const=1.0)]) == U
        for mode in (abi.AGGMODE_FINAL, abi.AGGMODE_PARTIAL1, abi.AGGMODE_PARTIAL2):
            assert rc(lib, cols, [xsum(1, 1, 4, expr, 1.0, mode=mode)]) == U, mode
        for rt in (0, abi.TYPE_DOUBLE, abi.TYPE_LONGLONG):   # a non-DECIMAL ret_type
            assert rc(lib, cols, [xsum(1, 1, 4, expr, 1.0, ret_type=rt)]) == U, rt
        assert rc(lib, cols, [xsum(7, 8, 31, expr, 0.0)]) == U   # s = 18 + 13 > 30
        assert rc(lib, cols, [xavg(7, 8, 31, expr, 0.0)]) == U
    # the constant: not an integer, not finite, or |c| * 10^s_b > 10^18
    for c in (0.5, -1.25, math.inf, -math.inf, math.nan, 1e16 + 2, 1e17):
        assert rc(lib, cols, [xsum(1, 1, 4, CSUB, c)]) == U, c
    assert rc(lib, cols, [xsum(1, 1, 4, CSUB, 1e16)]) == OK          # 10^16 * 10^2 = 10^18: the bound itself
    assert rc(lib, cols, [xsum(1, 1, 4, CSUB, -1e16)]) == OK
    assert rc(lib, cols, [xsum(1, 7, 20, CSUB, 2.0)]) == U           # 2 * 10^18 > 10^18
    assert rc(lib, cols, [xsum(1, 7, 20, CSUB, -1.0)]) == OK


def test_invalid(lib):
    cols = [INT, dec(15, 2), dec(18, 9), dec(5, 6), dec(0, 0)]
    for f in (xsum(1, 1, 2), xsum(1, 1, 5), xsum(1, 2, 4), xavg(1, 1, 3), xavg(1, 1, 31), xsum(1, 2, 9, CSUB, 1.0), xavg(1, 2, 10, CSUB, 1.0),
              xavg(2, 2, 17)):
        assert rc(lib, cols, [f]) == INV, f
    for b in (3, 4):                                          # decimal > flen, flen 0
        assert rc(lib, cols, [xsum(1, b, 8 if b == 3 else 2)]) == INV, b


def test_state_words(lib):
    # three words, and a fourth for the count when an operand is nullable, under the 24-word limit
    cols = [INT, dec(15, 2), dec(15, 2, abi.FLAG_NOT_NULL)]
    assert rc(lib, cols, [xsum(2, 2, 4)] * 8) == OK and rc(lib, cols, [xsum(2, 2, 4)] * 9) == U
    assert rc(lib, cols, [xsum(1, 2, 4)] * 6) == OK and rc(lib, cols, [xsum(1, 2, 4)] * 7) == U
    assert rc(lib, cols, [xavg(2, 1, 8, CSUB, 1.0)] * 6) == OK and rc(lib, cols, [xavg(2, 1, 8, CSUB, 1.0)] * 7) == U
    d, keep = AggPlan(cols, [0], [xsum(1, 2, 4)] * 7).to_struct_ex()
    assert lib.tg_agg_supported_ex(C.byref(d)) == U and b"up to 4 over a product" in lib.tg_last_error()


def test_without_ex_every_product_plan_stays_declined(lib):
    cols = [INT, dec(15, 2), dec(18, 0)]
    for f in (xsum(1, 1, 4), xavg(1, 2, 6, CSUB, 1.0), xsum(1, 2, 2, CSUB, 1.0)):
        assert rc(lib, cols, [f], ex=False) == U, f
    # DOUBLE products answer as before through both calls
    dcols = [INT, DBL, DBL]
    for f in (AggFunc(abi.AGG_SUM, 1, abi.TYPE_DOUBLE, arg_col2=2, arg_expr=MUL),
              AggFunc(abi.AGG_AVG, 1, abi.TYPE_DOUBLE, arg_col2=2, arg_expr=CSUB, arg_const=0.5)):
        assert rc(lib, dcols, [f]) == rc(lib, dcols, [f], ex=False) == OK


def test_result_schema():
    # TPC-H lineitem: l_extendedprice, l_discount, l_tax DECIMAL(15,2).  1 - l_discount is DECIMAL(16,2); the product is
    # DECIMAL(31,4) (Q1 / Q3); l_extendedprice * l_discount is DECIMAL(30,4) (Q6); SUM adds 22 digits, AVG the increment
    cols = [INT, dec(15, 2), dec(15, 2, abi.FLAG_NOT_NULL), dec(18, 18), dec(18, 12), dec(10, 0)]
    plan = AggPlan(cols, [0], [xsum(1, 2, 4, CSUB, 1.0), xsum(1, 2, 4), xavg(1, 2, 8, CSUB, 1.0), xsum(3, 4, 30), xavg(3, 4, 30),
                               xsum(5, 5, 0, CSUB, -12345.0), xsum(1, 5, 2, CSUB, 10 ** 12)])
    e = HashAggExec(plan, MockDataSource(plan.col_types, []))
    got = [(t.tp, t.flen, t.decimal) for t in e.schema]
    assert got == [(DEC, 53, 4), (DEC, 52, 4), (DEC, 35, 8), (DEC, 58, 30), (DEC, 36, 30), (DEC, 43, 0), (DEC, 51, 2)]
