"""Test-only reference for SUM / AVG of a product of DECIMAL(p <= 18) columns, a * b or a * (c - b) with an integer c,
computed with Python ints over tests/mydecimal_args.py.

DecimalMul (types/mydecimal.go:2041) is exact with digitsFrac = s_a + s_b, and c - b (DecimalSub) is exact at scale s_b,
so a row's value is the integer a_scaled * t_scaled at scale s = s_a + s_b, t_scaled = b_scaled or c * 10^s_b - b_scaled.
SUM and AVG over these values follow the rules of DECIMAL columns at scale s (mydecimal_args.sum_result / avg_result).
"""
from __future__ import annotations

from fractions import Fraction
from typing import Sequence, Tuple

import numpy as np

import mydecimal as D
import mydecimal_args as A

MUL, MUL_CSUB = 1, 2          # abi.ARGEXPR_MUL / ARGEXPR_MUL_CSUB


def parse(text: str) -> Tuple[int, int]:
    """'-123.45' -> (-12345, 2)"""
    neg = text.startswith("-")
    ip, _, fp = text.lstrip("-").partition(".")
    v = int((ip or "0") + fp)
    return (-v if neg else v), len(fp)


def operand_t(b_scaled, expr: int, c: int, s_b: int):
    """the second factor at scale s_b: b, or c - b (works on Python ints and object arrays)"""
    return b_scaled if expr == MUL else c * 10 ** s_b - b_scaled


def products(a: np.ndarray, b: np.ndarray, expr: int, c: int, s_b: int) -> np.ndarray:
    """exact per-row products at scale s_a + s_b, as Python ints (object array)"""
    return a.astype(object) * operand_t(b.astype(object), expr, c, s_b)


def product_string(a: str, b: str) -> str:
    """DecimalMul of two literals as MyDecimal.String prints it (digitsFrac = s_a + s_b digits, no negative zero)"""
    (x, sa), (y, sb) = parse(a), parse(b)
    return D.to_string(D.encode(Fraction(x * y, 10 ** (sa + sb)), sa + sb))


def minus_string(c: str, b: str) -> str:
    """1 * (c - b) with an integer c: the product path at scale 0 + s_b"""
    (cv, sc), (y, sb) = parse(c), parse(b)
    assert sc == 0
    return D.to_string(D.encode(Fraction(1 * operand_t(y, MUL_CSUB, cv, sb), 10 ** sb), sb))


def group_sums(values: np.ndarray, keep: np.ndarray, inv: np.ndarray, ngroups: int) -> Tuple[list, np.ndarray]:
    """exact per-group sums of the kept rows (Python ints) and the per-group counts"""
    idx = np.flatnonzero(keep)
    order = idx[np.argsort(inv[idx], kind="stable")]
    g = inv[order]
    cnt = np.bincount(g, minlength=ngroups)
    sums = [0] * ngroups
    if len(order):
        starts = np.flatnonzero(np.r_[True, g[1:] != g[:-1]])
        red = np.add.reduceat(values[order], starts)
        for j, v in zip(g[starts].tolist(), red.tolist()):
            sums[j] = int(v)
    return sums, cnt


def sum_result(total: int, s: int) -> bytes:
    return A.sum_result(total, s)


def avg_result(total: int, n: int, s: int, f: int) -> bytes:
    return A.avg_result(total, n, s, f)


def expected_cells(sums: Sequence[int], cnt: np.ndarray, avg: bool, s: int, f: int) -> list:
    return [None if n == 0 else (avg_result(t, int(n), s, f) if avg else sum_result(t, s)) for t, n in zip(sums, cnt.tolist())]
