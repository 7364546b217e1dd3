"""Known answers for tests/mydecimal_expr.py: DecimalMul and DecimalSub rows of pkg/types/mydecimal_test.go within
DECIMAL(p <= 18) operands, and SUM / AVG over products."""
from fractions import Fraction

import numpy as np
import pytest

import mydecimal as D
import mydecimal_expr as X


# TestMulMyDecimal (pkg/types/mydecimal_test.go:671): the rows whose operands fit DECIMAL(18)
@pytest.mark.parametrize("a,b,want", [
    ("12", "10", "120"),
    ("-123.456", "98765.4321", "-12193185.1853376"),
    ("123456", "987654321", "121931851853376"),
    ("123456", "9876543210", "1219318518533760"),
    ("123", "0.01", "1.23"),
    ("123", "0", "0"),
    ("0.5999991229316", "0.918755041726043", "0.5512522192246113614062276588"),
    ("0.5999991229317", "0.918755041726042", "0.5512522192247026369112773314"),
    ("0.000", "-1", "0.000"),
])
def test_mul_known_answers(a, b, want):
    assert X.product_string(a, b) == want


# TestSubMyDecimal (pkg/types/mydecimal_test.go:634): the rows with an integer minuend, run as 1 * (c - b)
@pytest.mark.parametrize("c,b,want", [
    ("10000000", "1", "9999999"),
    ("1000001000", ".1", "1000000999.9"),
    ("1000000000", ".1", "999999999.9"),
    ("12345", "123.45", "12221.55"),
    ("-12345", "-123.45", "-12221.55"),
    ("-12345", "123.45", "-12468.45"),
    ("12345", "-123.45", "12468.45"),
])
def test_sub_known_answers(c, b, want):
    assert X.minus_string(c, b) == want


def test_group_sums_and_results():
    a = np.array([10 ** 18 - 1, 10 ** 18 - 1, 5, -5, 7, 0], dtype=np.int64)
    b = np.array([10 ** 18 - 1, 10 ** 18 - 1, 3, 3, 1, 0], dtype=np.int64)
    inv = np.array([0, 0, 1, 1, 2, 3])
    keep = np.array([True, True, True, True, True, False])
    sums, cnt = X.group_sums(X.products(a, b, X.MUL, 0, 0), keep, inv, 4)
    assert sums == [2 * (10 ** 18 - 1) ** 2, 0, 7, 0] and cnt.tolist() == [2, 2, 1, 0]
    assert sums[0] > 1 << 120
    cells = X.expected_cells(sums, cnt, False, 4, 4)
    assert cells[3] is None and D.to_string(cells[1]) == "0.0000" and D.to_string(cells[2]) == "0.0007"
    # c - b at scale s_b: 1 - 0.05 = 0.95, times 100.00 = 95.0000
    t = X.operand_t(5, X.MUL_CSUB, 1, 2)
    assert t == 95 and D.to_string(X.sum_result(10000 * t, 4)) == "95.0000"
    # AVG of the products at scale 4 rounded half up at 5 digits: 1 / 32 = 0.03125 -> 0.03125, at 4 digits -> 0.0313
    assert D.to_string(X.avg_result(10 ** 4, 32, 4, 4)) == "0.0313"
    assert D.value(X.avg_result(-(10 ** 4), 32, 4, 30)) == Fraction(-1, 32)
