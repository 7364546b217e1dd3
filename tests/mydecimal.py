"""Test-only codec of TiDB's 40-byte MyDecimal cell, and the exact DECIMAL SUM / AVG rules the GPU aggregation must meet.

Cell layout (types/mydecimal.go:236-248, copied whole into a chunk column, util/chunk/column.go:41): int8 digitsInt,
int8 digitsFrac, int8 resultFrac, bool negative, then int32 wordBuf[9] in base 10^9, most significant word first:
integer words, then fraction words.

`to_string` restates MyDecimal.ToString (mydecimal.go:317-392, with removeLeadingZeros :278 and countLeadingZeroes :201),
so a cell is read the way TiDB prints it.  `encode` writes the canonical form the library writes: digitsInt = 9 * the
number of integer words with at least one word (FromUint, mydecimal.go:1069), digitsFrac = resultFrac = the scale.

`sum_result` / `avg_result` state the aggregate rules with Python ints:
  SUM  exact sum, scale 0 (sum4Decimal, executor/aggfuncs/func_sum.go:207-253).
  AVG  DecimalDiv(sum, count, frac) truncates the quotient at 9 * ceil(frac / 9) fraction digits (doDivMod,
       mydecimal.go:2203), then Round(frac, ModeHalfUp) looks only at the first digit after the scale and rounds the
       magnitude (mydecimal.go:811-983).  So AVG rounds half away from zero unless frac is a multiple of 9, where it is
       the truncated quotient.  A zero result is never negative: doDivMod clears the sign of a zero quotient
       (mydecimal.go:2449) and Round clears it when it rounds to zero (:956-967).
"""
from __future__ import annotations

import struct
from fractions import Fraction
from typing import NamedTuple, Tuple

CELL = 40
BASE = 10 ** 9
WORDS = 9


class Cell(NamedTuple):
    digits_int: int
    digits_frac: int
    result_frac: int
    negative: bool
    words: Tuple[int, ...]


def _words_of(digits: int) -> int:
    return (digits + 8) // 9


def decode(cell) -> Cell:
    b = bytes(cell)
    assert len(b) == CELL, len(b)
    di, df, rf, neg = struct.unpack_from("<bbbB", b, 0)
    return Cell(di, df, rf, bool(neg), struct.unpack_from("<9i", b, 4))


def encode(value, frac: int = 0) -> bytes:
    """the canonical cell of `value` (int or Fraction with at most `frac` fraction digits) at scale `frac`"""
    v = Fraction(value)
    scaled = v * 10 ** frac
    assert scaled.denominator == 1, f"{value} has more than {frac} fraction digits"
    m = abs(scaled.numerator)
    ip, fp = divmod(m, 10 ** frac)
    iw = []
    while True:
        iw.append(ip % BASE)
        ip //= BASE
        if ip == 0:
            break
    iw.reverse()
    nfw = _words_of(frac)
    fpw = fp * 10 ** (9 * nfw - frac)
    fw = [(fpw // BASE ** (nfw - 1 - j)) % BASE for j in range(nfw)]
    words = iw + fw
    assert len(words) <= WORDS
    words += [0] * (WORDS - len(words))
    return struct.pack("<bbbB9i", 9 * len(iw), frac, frac, 1 if v < 0 else 0, *words)


def value(cell) -> Fraction:
    """the signed value of a cell (digitsInt / digitsFrac select the words)"""
    c = decode(cell)
    wi, wf = _words_of(c.digits_int), _words_of(c.digits_frac)
    ip = 0
    for w in c.words[:wi]:
        ip = ip * BASE + w
    fp = 0
    for w in c.words[wi:wi + wf]:
        fp = fp * BASE + w
    v = ip + Fraction(fp, BASE ** wf)
    return -v if c.negative else v


def _count_leading_zeroes(i: int, word: int) -> int:
    leading = 0
    while word < 10 ** i:
        i -= 1
        leading += 1
    return leading


def _remove_leading_zeros(c: Cell):
    digits_int = c.digits_int
    i = ((digits_int - 1) % 9) + 1
    idx = 0
    while digits_int > 0 and c.words[idx] == 0:
        digits_int -= i
        i = 9
        idx += 1
    if digits_int > 0:
        digits_int -= _count_leading_zeroes((digits_int - 1) % 9, c.words[idx])
    else:
        digits_int = 0
    return idx, digits_int


def to_string(cell) -> str:
    """MyDecimal.ToString (mydecimal.go:317-392): the printed value, without rounding"""
    c = decode(cell)
    digits_frac = c.digits_frac
    start, digits_int = _remove_leading_zeros(c)
    if digits_int + digits_frac == 0:
        digits_int, start = 1, 0
    out = "-" if c.negative else ""
    if digits_int > 0:
        ip = 0
        for w in c.words[start:start + _words_of(digits_int)]:
            ip = ip * BASE + w
        out += str(ip % 10 ** digits_int).rjust(digits_int, "0")
    else:
        out += "0"
    if digits_frac > 0:
        widx = start + _words_of(digits_int)
        frac_digits = "".join(str(w).rjust(9, "0") for w in c.words[widx:widx + _words_of(digits_frac)])
        out += "." + frac_digits[:digits_frac]
    return out


def well_formed(cell) -> bool:
    """a header TiDB can read: digitsInt covers the significant integer digits and fits the words, every word is below
    10^9, and the words outside the integer and fraction ranges are zero"""
    c = decode(cell)
    if c.digits_int < 0 or c.digits_frac < 0 or c.result_frac < 0:
        return False
    wi, wf = _words_of(c.digits_int), _words_of(c.digits_frac)
    if wi + wf > WORDS or any(not 0 <= w < BASE for w in c.words):
        return False
    if any(c.words[wi + wf:]):
        return False
    if wi and c.words[0] >= 10 ** (c.digits_int - 9 * (wi - 1)):
        return False   # a digit above digitsInt
    return True


# ---- aggregate rules -----------------------------------------------------------------------------------------------
def sum_result(s: int) -> bytes:
    """DECIMAL SUM of integers: the exact sum, scale 0"""
    return encode(s, 0)


def div_trunc(s: int, n: int, frac_incr: int) -> Tuple[Fraction, int]:
    """DecimalDiv(s, n, frac_incr) of two integers: (quotient truncated toward zero at 9 * ceil(frac_incr / 9) fraction
    digits, digitsFrac of the quotient; a zero dividend keeps frac_incr, zeroMyDecimalWithFrac)"""
    if s == 0:
        return Fraction(0), frac_incr
    d = 9 * _words_of(frac_incr)
    q = (abs(s) * 10 ** d) // abs(n)
    q = Fraction(q, 10 ** d)
    return (-q if (s < 0) != (n < 0) else q), d


def round_half_up(v: Fraction, frac: int, digits_frac: int) -> Fraction:
    """Round(v, frac, ModeHalfUp) of a value with digits_frac fraction digits: unchanged when frac >= digits_frac, else the
    magnitude rounded on the first digit after the scale alone"""
    if frac >= digits_frac:
        return v
    a = abs(v)
    keep = int(a * 10 ** frac)
    if int(a * 10 ** (frac + 1)) % 10 >= 5:
        keep += 1
    r = Fraction(keep, 10 ** frac)
    return -r if v < 0 else r


def avg_value(s: int, n: int, frac: int) -> Fraction:
    """DECIMAL AVG of integers with sum s over n > 0 rows at scale frac (DecimalDiv with fracIncr = frac, then Round)"""
    q, d = div_trunc(s, n, frac)
    return round_half_up(q, frac, d)


def avg_result(s: int, n: int, frac: int) -> bytes:
    return encode(avg_value(s, n, frac), frac)
