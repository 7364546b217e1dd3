"""CPU-side checks of the join gate for DECIMAL payload columns: 40-byte MyDecimal cells are carried through every join
type and build side as output columns, while a DECIMAL key, filter item or OtherCondition operand is still declined."""
import ctypes as C
import os
import re

import pytest

from tidb_b200 import abi
from tidb_b200.plan import FieldType, FilterItem, JoinPlan, OtherCond

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT = FieldType(abi.TYPE_LONGLONG, 0)
INT_NN = FieldType(abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)
DEC = FieldType(abi.TYPE_NEWDECIMAL, 0, 15, 2)
DEC_NN = FieldType(abi.TYPE_NEWDECIMAL, abi.FLAG_NOT_NULL, 15, 2)
JOIN_TYPES = [abi.JOIN_INNER, abi.JOIN_LEFT_OUTER, abi.JOIN_RIGHT_OUTER, abi.JOIN_SEMI, abi.JOIN_ANTI_SEMI,
              abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI]


@pytest.fixture(scope="module")
def lib():
    from tidb_b200 import build
    build.build()
    return abi.load_lib()


def rc(lib, plan):
    d, keep = plan.to_struct()
    return lib.tg_join_supported(C.byref(d))


# left: 0 key | 1 DECIMAL | 2 INT | 3 DECIMAL NOT NULL      right: 0 key | 1 DECIMAL NOT NULL | 2 DECIMAL | 3 INT
LT = [INT, DEC, INT, DEC_NN]
RT = [INT, DEC_NN, DEC, INT]


@pytest.mark.parametrize("jt", JOIN_TYPES)
@pytest.mark.parametrize("build_is_right", [True, False])
def test_gate_accepts_decimal_payload_every_join_type(lib, jt, build_is_right):
    semi = jt >= abi.JOIN_SEMI
    want = abi.TG_OK
    if jt in (abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI) and not build_is_right:
        want = abi.TG_ERR_UNSUPPORTED   # needs the right side as build side, DECIMAL or not
    for lused, rused in (([1, 0, 3], [] if semi else [2, 1]), (None, [] if semi else None), ([3], [] if semi else [1, 1, 2])):
        plan = JoinPlan(jt, LT, RT, [0], [0], build_is_right=build_is_right, lused=lused, rused=rused)
        assert rc(lib, plan) == want, (lused, rused)


def test_gate_accepts_decimal_payload_with_several_keys_filters_and_other_condition(lib):
    for brt in (True, False):
        multi = JoinPlan(abi.JOIN_INNER, [INT, INT] + LT[1:], [INT, INT] + RT[1:], [0, 1], [0, 1], build_is_right=brt,
                         lused=[0, 2, 4], rused=[2, 3])
        assert rc(lib, multi) == abi.TG_OK
        filtered = JoinPlan(abi.JOIN_INNER, LT, RT, [0], [0], build_is_right=brt, lused=[1, 3], rused=[1, 2],
                            build_filter=[FilterItem(abi.CMP_GT, 3 if brt else 2, const_i64=0)],
                            probe_filter=[FilterItem(abi.CMP_NE, 2 if brt else 3, const_i64=5)])
        assert rc(lib, filtered) == abi.TG_OK
    for jt in (abi.JOIN_INNER, abi.JOIN_LEFT_OUTER, abi.JOIN_SEMI, abi.JOIN_ANTI_SEMI):
        other = JoinPlan(jt, LT, RT, [0], [0], build_is_right=True, lused=[1, 2, 3], rused=[] if jt >= abi.JOIN_SEMI else [1, 2],
                         other_cond=[OtherCond(abi.CMP_LT, 0, 2, 1, 3), OtherCond(abi.CMP_NE, 1, 3, -1, -1, const_i64=7)])
        assert rc(lib, other) == abi.TG_OK


def test_gate_declines_decimal_keys_filters_and_other_condition_operands(lib):
    U = abi.TG_ERR_UNSUPPORTED
    assert rc(lib, JoinPlan(abi.JOIN_INNER, LT, RT, [1], [1])) == U                  # DECIMAL key
    assert rc(lib, JoinPlan(abi.JOIN_INNER, LT, RT, [0], [2])) == U                  # DECIMAL against an integer key
    assert rc(lib, JoinPlan(abi.JOIN_INNER, LT, RT, [0, 3], [0, 1])) == U            # one DECIMAL column among several keys
    for brt in (True, False):
        for lf, rf in (([FilterItem(abi.CMP_GT, 1, const_i64=0)], []), ([], [FilterItem(abi.CMP_LT, 3, rhs_col=2)]),
                       ([FilterItem(abi.CMP_EQ, 2, rhs_col=3)], [])):
            plan = JoinPlan(abi.JOIN_INNER, LT, RT, [0], [0], build_is_right=brt,
                            build_filter=rf if brt else lf, probe_filter=lf if brt else rf)
            assert rc(lib, plan) == U, (brt, lf, rf)
    for oc in ([OtherCond(abi.CMP_LT, 0, 1, 1, 3)], [OtherCond(abi.CMP_LT, 0, 2, 1, 2)],
               [OtherCond(abi.CMP_NE, 1, 1, -1, -1, const_i64=0)], [OtherCond(abi.CMP_EQ, 0, 3, 1, 1)]):
        assert rc(lib, JoinPlan(abi.JOIN_INNER, LT, RT, [0], [0], other_cond=oc)) == U, oc


def test_gate_semi_join_with_decimal_right_output_is_invalid(lib):
    for jt in (abi.JOIN_SEMI, abi.JOIN_ANTI_SEMI, abi.JOIN_LEFT_OUTER_SEMI):
        assert rc(lib, JoinPlan(jt, LT, RT, [0], [0], lused=[1], rused=[1])) == abi.TG_ERR_INVALID


def test_header_cell_gather_path_bit(lib):
    hdr = open(os.path.join(ROOT, "include", "tidbgpu.h")).read()
    m = re.search(r"\bTG_JOIN_PATH_CELL_GATHER = (0x[0-9a-fA-F]+|\d+)", hdr)
    assert m and int(m.group(1), 0) == 1 << 7 == abi.JOIN_PATH_CELL_GATHER
    assert not re.search(r"\bTG_JOIN_PATH_[A-Z0-9_]+ = 1 << 4\b", hdr)   # 1 << 4 stays unassigned
    assert lib.tg_abi_version() == 2
    assert C.sizeof(abi.TgJoinDesc) == 160   # tg_join_desc is unchanged: no precision or scale is needed to move a cell
