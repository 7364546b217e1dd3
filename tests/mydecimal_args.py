"""Test-only reference for aggregates over DECIMAL(p <= 18, s) argument columns: the stored input cells and the exact
result cells, computed with Python ints and Fractions.

Input cells are what MyDecimal.FromBin (types/mydecimal.go:1465) leaves in a chunk column for a DECIMAL(p, s) column:
digitsFrac = s, ceil(digitsInt / 9) integer words (FromBin sets digitsInt = p - s, so small values have leading zero
words), then ceil(s / 9) fraction words, left-aligned.  `cell` writes that form and the variants the library must read
the same way: digitsInt 0, extra leading zero words, a negative zero, any resultFrac.  `cells_np` is the same encoder on
numpy arrays, for large inputs.

Results (tests/mydecimal.py `encode`, the canonical form: digitsFrac = resultFrac = the result scale):
  SUM       the exact sum at scale s (sum4Decimal, executor/aggfuncs/func_sum.go).
  MIN/MAX   the smallest / largest value at scale s (max4Decimal / min4Decimal, func_max_min.go:906).
  AVG       DecimalDiv(sum, count, incr) then Round(f, ModeHalfUp) (baseAvgDecimal, func_avg.go:84), f = min(s + incr, 30).
            doDivMod (mydecimal.go:2203) truncates the quotient at T = 9 * ceil((s + incr) / 9) fraction digits when the
            sum has digitsFrac = s; Round then rounds the magnitude half up on digit f + 1 (truncation when T == f).
"""
from __future__ import annotations

import struct
from fractions import Fraction
from typing import Optional

import numpy as np

import mydecimal as D

BASE = 10 ** 9


def _words(digits: int) -> int:
    return (digits + 8) // 9


def cell(scaled: int, p: int, s: int, digits_int: Optional[int] = None, result_frac: int = 0, neg_zero: bool = False) -> bytes:
    """the stored cell of value scaled / 10^s in a DECIMAL(p, s) column; digits_int defaults to FromBin's p - s"""
    m = abs(scaled)
    assert m < 10 ** p
    ip, fp = divmod(m, 10 ** s)
    di = p - s if digits_int is None else digits_int
    wi, wf = _words(di), _words(s)
    assert wi + wf <= 9 and ip < BASE ** wi
    iw = [(ip // BASE ** (wi - 1 - j)) % BASE for j in range(wi)]
    fpl = fp * 10 ** (9 * wf - s)
    fw = [(fpl // BASE ** (wf - 1 - j)) % BASE for j in range(wf)]
    words = iw + fw + [0] * (9 - wi - wf)
    neg = scaled < 0 or (neg_zero and scaled == 0)
    return struct.pack("<bbbB9i", di, s, result_frac, 1 if neg else 0, *words)


def cells_np(scaled: np.ndarray, p: int, s: int, digits_int: np.ndarray, result_frac: np.ndarray, neg: np.ndarray) -> np.ndarray:
    """`cell` for arrays: int64 values * 10^s (|v| < 10^p <= 10^18), per-row digitsInt / resultFrac / negative flag
    (neg must be set for every negative value; set on a zero it makes a negative zero) -> (n, 40) uint8"""
    n = len(scaled)
    m = np.abs(scaled.astype(np.int64))
    assert (m < 10 ** p).all() and (neg | (scaled >= 0)).all()
    ip, fp = m // 10 ** s, m % 10 ** s
    wi, wf = (digits_int + 8) // 9, _words(s)
    assert (wi + wf <= 9).all() and ((ip < BASE) | (wi >= 2)).all() and ((ip == 0) | (wi >= 1)).all()
    words = np.zeros((n, 9), dtype=np.int64)
    rows = np.arange(n)
    k = wi >= 1
    words[rows[k], wi[k] - 1] = ip[k] % BASE
    k = wi >= 2
    words[rows[k], wi[k] - 2] = ip[k] // BASE
    fpl = fp * 10 ** (9 * wf - s)
    if wf == 1:
        words[rows, wi] = fpl
    elif wf == 2:
        words[rows, wi] = fpl // BASE
        words[rows, wi + 1] = fpl % BASE
    out = np.zeros((n, 10), dtype=np.int32)
    out[:, 0] = (digits_int.astype(np.int32) | (s << 8) | (result_frac.astype(np.int32) << 16) | (neg.astype(np.int32) << 24))
    out[:, 1:] = words
    return out.view(np.uint8).reshape(n, 40)


def sum_result(total_scaled: int, s: int) -> bytes:
    """SUM (and MIN / MAX) of a DECIMAL(p, s) column: the value total_scaled / 10^s at scale s"""
    return D.encode(Fraction(total_scaled, 10 ** s), s)


def avg_value(total_scaled: int, n: int, s: int, f: int, incr: Optional[int] = None) -> Fraction:
    """AVG of n > 0 values of scale s summing to total_scaled / 10^s, at result scale f.  incr = the
    div_precision_increment (default f - s: f = s + incr); f = 30 stands for every incr >= 30 - s"""
    if incr is None:
        incr = f - s
    assert f == min(s + incr, 30)
    if total_scaled == 0:
        return Fraction(0)
    t = 9 * _words(s + incr)                          # doDivMod's fraction digits of the quotient
    q = Fraction(abs(total_scaled) * 10 ** t // (n * 10 ** s), 10 ** t)
    return D.round_half_up(-q if total_scaled < 0 else q, f, t)


def avg_result(total_scaled: int, n: int, s: int, f: int, incr: Optional[int] = None) -> bytes:
    return D.encode(avg_value(total_scaled, n, s, f, incr), f)


def div_trunc_string(dividend: str, divisor: int, incr: int) -> str:
    """DecimalDiv(dividend, divisor, incr) of a decimal string by a positive integer, printed as MyDecimal.ToString prints
    the quotient: truncated at T = 9 * ceil((digitsFrac + incr) / 9) digits, all T of them shown"""
    neg = dividend.startswith("-")
    ip, _, fp = dividend.lstrip("-").partition(".")
    s = len(fp)
    scaled = int(ip + fp)
    t = 9 * _words(s + incr)
    q = scaled * 10 ** t // (divisor * 10 ** s)
    out = f"{q // 10 ** t}.{str(q % 10 ** t).rjust(t, '0')}"
    return ("-" if neg and q else "") + out
