"""The reference for aggregates over DECIMAL(p <= 18, s) columns (tests/mydecimal_args.py), pinned by known answers of the
reference project and by its own cross-checks.  CPU only."""
import random
from fractions import Fraction

import numpy as np
import pytest

import mydecimal as D
import mydecimal_args as A


def test_stored_cells_read_back():
    # FromBin's form, digitsInt 0, extra leading zero words, a negative zero, a resultFrac that is not the scale
    for p, s in ((18, 0), (18, 2), (18, 9), (18, 18), (15, 2), (1, 0), (1, 1), (10, 4)):
        for v in (0, 1, -1, 5 * 10 ** (s - 1) if s else 5, 10 ** p - 1, -(10 ** p - 1), 10 ** s, -(10 ** s) + 1):
            if abs(v) >= 10 ** p:
                continue
            want = Fraction(v, 10 ** s)
            forms = [A.cell(v, p, s), A.cell(v, p, s, result_frac=30), A.cell(v, p, s, digits_int=9 * (9 - (s + 8) // 9))]
            if abs(v) < 10 ** s:
                forms.append(A.cell(v, p, s, digits_int=0))
            if v == 0:
                forms.append(A.cell(v, p, s, neg_zero=True))
            for c in forms:
                assert D.value(c) == want, (p, s, v, D.decode(c))
                assert D.decode(c).digits_frac == s
    # 0.5 at scale 1 is the left-aligned word 500000000
    assert D.decode(A.cell(5, 2, 1)).words[:2] == (0, 500_000_000)
    assert D.to_string(A.cell(-123456789012345678, 18, 9)) == "-123456789.012345678"


def test_numpy_encoder_matches_the_scalar_one():
    rng = np.random.default_rng(3)
    for p, s in ((18, 0), (18, 2), (18, 9), (18, 18), (15, 2)):
        n = 2000
        v = rng.integers(-(10 ** p - 1), 10 ** p - 1, n, endpoint=True, dtype=np.int64)
        v[:200] = rng.integers(-(10 ** s) + 1 if s else 0, 10 ** s if s else 1, 200)
        ip = np.abs(v) // 10 ** s
        need = np.where(ip == 0, 0, np.array([len(str(x)) for x in ip.tolist()]))
        di = np.maximum(need, rng.integers(0, 9 * (9 - (s + 8) // 9) + 1, n))
        rf = rng.integers(0, 31, n)
        neg = (v < 0) | ((v == 0) & (rng.random(n) < 0.5))
        cells = A.cells_np(v, p, s, di, rf, neg)
        for r in range(n):
            want = A.cell(int(v[r]), p, s, digits_int=int(di[r]), result_frac=int(rf[r]), neg_zero=bool(neg[r]))
            assert bytes(cells[r]) == want, (p, s, r)


def test_known_answers_of_the_aggregate_functions():
    # executor/aggfuncs tests over NewDecFromInt(0..4) (aggfunc_test.go:484), and a second partial {2, 3, 4}:
    # func_sum_test.go:30 (10, 9, 19), func_avg_test.go:29 (2.0, 3.0, 2.375 at the default increment 4),
    # func_max_min_test.go:113 (MAX 4, 4, 4), :125 (MIN 0, 2, 0)
    first, second = [0, 1, 2, 3, 4], [2, 3, 4]
    for rows, s_, a_, mx, mn in ((first, "10", "2.0000", "4", "0"), (second, "9", "3.0000", "4", "2"),
                                 (first + second, "19", "2.3750", "4", "0")):
        assert D.to_string(A.sum_result(sum(rows), 0)) == s_
        assert D.to_string(A.avg_result(sum(rows), len(rows), 0, 4)) == a_
        assert D.to_string(A.sum_result(max(rows), 0)) == mx and D.to_string(A.sum_result(min(rows), 0)) == mn
    # tests/integrationtest/r/executor/aggregate.result:1085: max(b) of DECIMAL(15,2) per group
    assert D.to_string(A.sum_result(77164, 2)) == "771.64" and D.to_string(A.sum_result(37849, 2)) == "378.49"
    # aggregate.result:1163-1168: DECIMAL(10,4) rows 0, -0.9871, -0.9871, twice: sum(a) = -3.9484
    assert D.to_string(A.sum_result(2 * (0 - 9871 - 9871), 4)) == "-3.9484"


@pytest.mark.parametrize("dividend,divisor,want", [
    ("120", 10, "12.000000000"),                             # types/mydecimal_test.go:713
    ("1", 3, "0.333333333"),                                 # :721
    ("1.000000000000", 3, "0.333333333333333333"),           # :722, digitsFrac 12 + 5 -> 18 digits
    ("10.000000000060", 2, "5.000000000030000000"),          # :726
])
def test_divmod_truncation_point(dividend, divisor, want):
    # TestDivModMyDecimal, DecimalDiv(a, b, 5) with an integer divisor: the quotient is truncated at
    # 9 * ceil((digitsFrac + 5) / 9) fraction digits
    assert A.div_trunc_string(dividend, divisor, 5) == want


def test_avg_rule():
    # truncation when f is a multiple of 9, half up on digit f + 1 otherwise, ties of both signs, no negative zero
    s = 2
    assert D.to_string(A.avg_result(1, 2, s, 4)) == "0.0050"            # 0.005 exactly
    assert D.to_string(A.avg_result(1, 2, s, 2)) == "0.01"              # 0.005 -> half up
    assert D.to_string(A.avg_result(-1, 2, s, 2)) == "-0.01"
    assert D.to_string(A.avg_result(-1, 3, s, 2)) == "0.00"             # rounds to zero: no sign
    assert D.to_string(A.avg_result(2, 3, 0, 9)) == "0.666666666"       # truncated at 9 digits
    assert D.to_string(A.avg_result(2, 3, 0, 8)) == "0.66666667"
    assert D.to_string(A.avg_result(2, 3, 9, 18)) == "0.000000000666666666"
    assert D.to_string(A.avg_result(-(10 ** 18 - 1), 1, 18, 30)) == "-0.999999999999999999000000000000"
    assert A.avg_value(5, 10, 0, 0) == 0 and A.avg_value(-19, 10, 0, 0) == -1   # f = 0 is a multiple of 9: truncated
    assert D.to_string(A.avg_result(-15, 100, 1, 1)) == "0.0"                      # -0.015 at f = 1: rounds to zero, no sign
    assert D.to_string(A.avg_result(-15, 100, 1, 2)) == "-0.02"                    # at f = 2: half up


def test_capped_scale_does_not_depend_on_the_increment():
    # f = 30 when s + incr > 30: doDivMod keeps more digits for a larger incr, and the result is the same for every one of
    # them (Round reads only digit 31), so the library can truncate at 36 digits for all
    rnd = random.Random(5)
    for s in (0, 2, 9, 17, 18):
        for _ in range(300):
            total = rnd.randint(-(10 ** 18 - 1) * 50, (10 ** 18 - 1) * 50)
            n = rnd.choice([1, 2, 3, 7, 8, 9, 11, 13, 50, 10 ** 6 + 3, 2 ** 40 + 1])
            got = {A.avg_result(total, n, s, 30, incr) for incr in range(30 - s, 31)}
            assert len(got) == 1, (total, n, s)
            # and equals the rule stated on f alone: truncate at 36 digits, half up on digit 31
            v = Fraction(total, n * 10 ** s)
            q = Fraction(int(abs(v) * 10 ** 36), 10 ** 36)
            assert got == {D.encode(D.round_half_up(q if v >= 0 else -q, 30, 36), 30)}
