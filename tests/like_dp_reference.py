"""A second reference for the string VecEval kernels, built differently from string_reference.py.

string_reference.py restates the reference's compile-then-walk LIKE (CompilePatternInner and doMatchInner with its single
restart point), which is also what the kernel runs, so a misreading of the Go code would be shared by both.  This module
answers the same questions another way:

  - LIKE: the pattern is cut into tokens (a literal, '_' = one character, '%' = any run) under the escape-first rule,
    with no "%%" or "%_" rewrite; the string is decoded into Go runes (one U+FFFD per byte that does not start a valid
    UTF-8 sequence, string_reference.decode_rune, which test_string_reference.py pins to Go's tables) or taken as bytes;
    and the match is a dynamic-programming table over (pattern position, string position).  Row i of the table is the
    set of string prefixes that the first i tokens match, kept as an integer bit mask over string positions.
  - Comparisons: Python's bytes ordering, after rstrip(b" ") under the four PAD collation ids.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import string_reference as S

LIT, ONE, ANY = "lit", "one", "any"
PAD_IDS = (46, 83, 65, 47)
BYTE_ORDER_IDS = (63, 309)
RUNE_MODE_IDS = PAD_IDS + (309,)


def over_runes(collation: int) -> bool:
    """LIKE walks runes under every offloaded collation but binary (63)"""
    if collation in RUNE_MODE_IDS:
        return True
    if collation == 63:
        return False
    raise ValueError(f"collation {collation} is not offloaded")


def chars_of(s: bytes, runes: bool) -> List[int]:
    """the characters LIKE sees: Go's []rune(s) (a U+FFFD per invalid byte) or the bytes"""
    if not runes:
        return list(s)
    out, i = [], 0
    while i < len(s):
        r, w = S.decode_rune(s, i)
        out.append(r)
        i += w
    return out


def tokens(pattern: bytes, escape: int, runes: bool) -> List[Tuple[str, int]]:
    """the pattern as (kind, value) tokens.  The escape is tested first, so '%' or '_' may be the escape; an escape with
    nothing after it is a literal escape character.  Over runes the escape is the rune `escape` (0xE9 is 'e acute')."""
    cs = chars_of(pattern, runes)
    out: List[Tuple[str, int]] = []
    i = 0
    while i < len(cs):
        c = cs[i]
        if c == escape:
            if i + 1 < len(cs):
                i += 1
            out.append((LIT, cs[i]))
        elif c == ord("%"):
            out.append((ANY, 0))
        elif c == ord("_"):
            out.append((ONE, 0))
        else:
            out.append((LIT, c))
        i += 1
    return out


def match_tokens(chars: Sequence[int], toks: Sequence[Tuple[str, int]]) -> bool:
    """the DP table: bit j of `row` is set when the tokens so far match chars[:j]"""
    n = len(chars)
    full = (1 << (n + 1)) - 1
    eq = {}
    for kind, v in toks:
        if kind == LIT and v not in eq:
            eq[v] = sum(1 << j for j, c in enumerate(chars) if c == v)   # bit j: chars[j] == v
    row = 1                                              # the empty pattern matches the empty prefix
    for kind, v in toks:
        if kind == LIT:
            row = (row & eq[v]) << 1
        elif kind == ONE:
            row = (row << 1) & full
        else:                                            # '%': every prefix at or after the first one reached
            row = full & ~((row & -row) - 1) if row else 0
        if not row:
            return False
    return bool((row >> n) & 1)


def like(s: bytes, pattern: bytes, escape: int, collation: int) -> bool:
    """`s LIKE pattern ESCAPE escape` for one non-NULL row under an offloaded collation id"""
    r = over_runes(collation)
    return match_tokens(chars_of(s, r), tokens(pattern, escape, r))


def like_bytes_ok(weights: Sequence[int], types: Sequence[int]) -> bool:
    """the host's choice of the byte walk for a rune collation: a compiled pattern of ASCII literals and '%' only"""
    return all(t == S.PAT_ANY or (t == S.PAT_MATCH and 0 <= w < 0x80) for w, t in zip(weights, types))


def cmp_key(s: bytes, collation: int) -> bytes:
    if collation in PAD_IDS:
        return s.rstrip(b" ")
    if collation in BYTE_ORDER_IDS:
        return s
    raise ValueError(f"collation {collation} is not offloaded")


def compare(a: bytes, b: bytes, collation: int) -> int:
    """three-way comparison of two non-NULL values under an offloaded collation id"""
    x, y = cmp_key(a, collation), cmp_key(b, collation)
    return (x > y) - (x < y)
