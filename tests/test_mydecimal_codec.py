"""The test-only MyDecimal codec (tests/mydecimal.py) pinned with known answers from the reference's own tests
(pkg/types/mydecimal_test.go), and the DECIMAL AVG rule at the scales the GPU tests use."""
from fractions import Fraction

import pytest

import mydecimal as D

I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1


# TestFromInt (mydecimal_test.go:27-43) and TestFromUint (:45-61)
@pytest.mark.parametrize("v,s", [(-12345, "-12345"), (-1, "-1"), (1, "1"), (-9223372036854775807, "-9223372036854775807"),
                                 (-9223372036854775808, "-9223372036854775808"),
                                 (12345, "12345"), (0, "0"), (18446744073709551615, "18446744073709551615")])
def test_from_int_and_uint(v, s):
    cell = D.encode(v)
    assert D.to_string(cell) == s
    c = D.decode(cell)
    # FromUint: digitsInt = 9 * words, digitsFrac 0, resultFrac untouched (0)
    assert c.digits_int == 9 * max(1, -(-len(str(abs(v))) // 9)) and c.digits_frac == 0 and c.result_frac == 0
    assert c.negative == (v < 0) and D.well_formed(cell) and D.value(cell) == v


def test_int64_min_and_uint64_max_words():
    assert D.decode(D.encode(I64_MIN)).words[:3] == (9, 223372036, 854775808)
    assert D.decode(D.encode(U64_MAX)).words[:3] == (18, 446744073, 709551615)


# TestRoundWithHalfEven (mydecimal_test.go:297-330): it runs ModeHalfUp.  Rows with a non-negative scale
@pytest.mark.parametrize("inp,scale,out", [("123456789.987654321", 1, "123456790.0"), ("15.1", 0, "15"), ("15.5", 0, "16"),
                                           ("15.9", 0, "16"), ("-15.1", 0, "-15"), ("-15.5", 0, "-16"), ("-15.9", 0, "-16"),
                                           ("15.1", 1, "15.1"), ("-15.1", 1, "-15.1"), ("15.17", 1, "15.2"), (".999", 0, "1")])
def test_round_half_up(inp, scale, out):
    digits = len(inp.split(".")[1]) if "." in inp else 0
    v = D.round_half_up(Fraction(inp), scale, digits)
    assert D.to_string(D.encode(v, max(scale, 0))) == out


# TestDivModMyDecimal (mydecimal_test.go:705-741), integer over integer rows, DecimalDiv with fracIncr 5
@pytest.mark.parametrize("a,b,out", [(120, 10, "12.000000000"), (121931851853376, 987654321, "123456.000000000"),
                                     (0, 987, "0.00000"), (1, 3, "0.333333333"), (1, 1, "1.000000000")])
def test_div_integer_rows(a, b, out):
    q, digits = D.div_trunc(a, b, 5)
    assert D.to_string(D.encode(q, digits)) == out


@pytest.mark.parametrize("s,n,f,out", [
    # f = 4: the quotient has 9 digits, rounded half away from zero on the 5th
    (1, 8, 4, "0.1250"), (5, 8, 4, "0.6250"), (1, 16, 4, "0.0625"), (-1, 16, 4, "-0.0625"),
    (1, 32, 4, "0.0313"), (-1, 32, 4, "-0.0313"),            # 0.03125: a tie, both signs
    (2, 3, 4, "0.6667"), (-2, 3, 4, "-0.6667"),
    (-1, 30000, 4, "0.0000"),                                 # rounds to zero: the sign goes (Round :956-967)
    (-1, 20000, 4, "-0.0001"),                                # -0.00005 rounds away from zero
    (99999, 100000, 4, "1.0000"), (-99999, 100000, 4, "-1.0000"),   # carry into the integer part
    # f = 0: truncation (no digit after the scale in the quotient)
    (3, 2, 0, "1"), (-3, 2, 0, "-1"), (5, 3, 0, "1"), (-1, 3, 0, "0"), (1, 2, 0, "0"), (-1, 2, 0, "0"),
    # f = 9: truncation at 9 digits
    (2, 3, 9, "0.666666666"), (-2, 3, 9, "-0.666666666"), (1, 2 * 10 ** 9, 9, "0.000000000"),
    (-1, 2 * 10 ** 9, 9, "0.000000000"), (-1, 3 * 10 ** 9, 9, "0.000000000"),
    # f = 30: 36 quotient digits, rounded on the 31st
    (2, 3, 30, "0.666666666666666666666666666667"), (-2, 3, 30, "-0.666666666666666666666666666667"),
    (1, 3, 30, "0.333333333333333333333333333333"),
    (1, 2 * 10 ** 30, 30, "0.000000000000000000000000000001"),     # 5e-31: a tie
    (-1, 2 * 10 ** 30, 30, "-0.000000000000000000000000000001"),
    (-1, 3 * 10 ** 30, 30, "0.000000000000000000000000000000"),
    # extremes
    (U64_MAX * 3, 3, 4, "18446744073709551615.0000"), (I64_MIN * 2, 2, 0, "-9223372036854775808"),
])
def test_avg_rule(s, n, f, out):
    cell = D.avg_result(s, n, f)
    assert D.to_string(cell) == out
    c = D.decode(cell)
    assert c.digits_frac == f and c.result_frac == f and D.well_formed(cell)
    assert c.negative == (D.value(cell) < 0)


def test_avg_multiple_of_nine_truncates_toward_zero():
    # 9-digit scale: 0.6666666666... is not rounded up; 18 and 27 likewise
    for f in (9, 18, 27):
        assert D.avg_value(2, 3, f) == Fraction(int("6" * f), 10 ** f)
        assert D.avg_value(-2, 3, f) == -Fraction(int("6" * f), 10 ** f)


def test_sum_result_and_well_formed():
    for s in (0, 1, -1, 10 ** 9, -(10 ** 9) + 1, (1 << 127) - 1, -(1 << 127), U64_MAX * 4):
        cell = D.sum_result(s)
        assert D.value(cell) == s and D.well_formed(cell) and D.to_string(cell) == str(s)
        assert D.decode(cell).negative == (s < 0)
    bad = bytearray(D.sum_result(5))
    bad[8:12] = (7).to_bytes(4, "little")          # a word after the integer range
    assert not D.well_formed(bytes(bad))
    assert not D.well_formed(bytes([1]) + D.sum_result(12345)[1:])   # digitsInt 1 does not cover 12345
