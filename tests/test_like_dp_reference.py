"""Pins the two LIKE / comparison references against each other on the CPU: like_dp_reference.py (tokens and a DP table)
and string_reference.py (the reference's compile-then-walk, the kernel's algorithm).  Every pattern of up to 4 symbols
over {a, b, %, _, \\, e-acute, 0xFF} meets every string of up to 5 symbols over {a, b, ' ', e-acute, 0xE2, 0x82, 0xFF},
under four escapes, over bytes and over runes.

string_reference.do_match compares a string character with a pattern character only for equality with a literal, and
so does the DP; so a string character that equals no literal of the pattern is replaced by one stand-in (-1) before the
two are run, and each (pattern, reduced string) pair is checked once.  That reduction is exact, and it is what keeps the
whole enumeration to seconds."""
import itertools

import pytest

import like_dp_reference as P
import string_reference as S

PAT_SYMS = [b"a", b"b", b"%", b"_", b"\\", "é".encode(), b"\xff"]
STR_SYMS = [b"a", b"b", b" ", "é".encode(), b"\xe2", b"\x82", b"\xff"]
ESCAPES = [ord("\\"), ord("%"), ord("_"), 0xE9]


def _words(syms, maxlen):
    for k in range(maxlen + 1):
        for t in itertools.product(syms, repeat=k):
            yield b"".join(t)


PATTERNS = sorted(set(_words(PAT_SYMS, 4)))
STRINGS = sorted(set(_words(STR_SYMS, 5)))


_CHARS = {r: [tuple(P.chars_of(s, r)) for s in STRINGS] for r in (False, True)}
_REDUCED = {}


def _reduced(lits, runes):
    """the distinct (reduced characters, reduced bytes) pairs of STRINGS for one set of literals"""
    key = (lits, runes)
    if key not in _REDUCED:
        _REDUCED[key] = sorted({(tuple(c if c in lits else -1 for c in chars), tuple(c if c in lits else -1 for c in bs))
                                for chars, bs in zip(_CHARS[runes], _CHARS[False])})
    return _REDUCED[key]


@pytest.mark.parametrize("runes", [False, True], ids=["bytes", "runes"])
@pytest.mark.parametrize("escape", ESCAPES, ids=["backslash", "percent", "underscore", "e9"])
def test_dp_and_walk_agree_everywhere(escape, runes):
    seen = set()
    checked = fast = 0
    for pat in PATTERNS:
        w, t = S.compile_pattern(pat, escape, runes)
        toks = P.tokens(pat, escape, runes)
        key = (tuple(w), tuple(t), tuple(toks))
        if key in seen:
            continue
        seen.add(key)
        lits = frozenset({x for x, y in zip(w, t) if y == S.PAT_MATCH} | {v for k, v in toks if k == P.LIT})
        bytes_ok = runes and P.like_bytes_ok(w, t)
        fast += bytes_ok
        done = {}
        for rr, rb in _reduced(lits, runes):
            if rr not in done:
                walk = S.do_match(rr, w, t)
                dp = P.match_tokens(rr, toks)
                assert walk == dp, (pat, escape, runes, rr, walk, dp)
                done[rr] = walk
                checked += 1
            if bytes_ok:
                # the byte walk the host picks for this pattern gives the rune walk's answer on every string
                assert S.do_match(rb, w, t) == done[rr], (pat, escape, rr, rb)
    assert checked > 10_000 and (fast > 50 if runes else fast == 0)


def test_like_entry_points_agree():
    # like() of both modules, through the collation ids, on a slice of the enumeration
    for pat in PATTERNS[::37]:
        for s in STRINGS[::53]:
            for coll in (63, 46, 83, 65, 47, 309):
                assert S.like(s, pat, ord("\\"), coll) == P.like(s, pat, ord("\\"), coll), (s, pat, coll)


def test_ascii_bytes_are_whole_runes():
    # what the byte walk relies on: in any byte string, a byte below 0x80 decodes as the rune of its own value, one byte
    # wide, and no longer rune contains such a byte; so an ASCII literal matches at the same places over bytes and over
    # runes, and the byte positions a '%' can stop at that an ASCII literal can follow are rune boundaries
    import numpy as np
    rng = np.random.default_rng(5)
    extra = [bytes(rng.integers(0, 256, int(rng.integers(1, 12)), dtype=np.uint8)) for _ in range(20_000)]
    extra += [bytes(rng.choice([0x41, 0x80, 0xBF, 0xC2, 0xE0, 0xED, 0xF0, 0xF4, 0xA0, 0x9F], 8)) for _ in range(20_000)]
    for s in STRINGS + extra:
        i = 0
        while i < len(s):
            r, width = S.decode_rune(s, i)
            if s[i] < 0x80:
                assert (r, width) == (s[i], 1), s
            else:
                assert r >= 0x80 and all(b >= 0x80 for b in s[i:i + width]), s
            i += width


def test_dp_pins():
    # hand cases the DP answers on its own (no compile rewrites): escape-first, trailing escape, '%_' and '%%'
    bs = ord("\\")
    assert P.tokens(b"a\\", bs, False) == [(P.LIT, 97), (P.LIT, bs)]
    assert P.tokens(b"%%a", ord("%"), True) == [(P.LIT, 37), (P.LIT, 97)]
    assert P.tokens(b"__", ord("_"), True) == [(P.LIT, 95)]
    assert P.tokens("é%".encode(), 0xE9, True) == [(P.LIT, 37)]
    assert P.tokens(b"\xe9%", 0xE9, True) == [(P.LIT, S.RUNE_ERROR), (P.ANY, 0)]
    assert P.like(b"abc", b"%_", bs, 46) and P.like(b"abc", b"%%c", bs, 46) and not P.like(b"", b"%_", bs, 46)
    assert P.like(b"\xe2\x82", b"__", bs, 46) and not P.like(b"\xe2\x82", b"_", bs, 46)
    assert P.like(b"\xe2\x82\xac", b"_", bs, 309) and P.like(b"\xe2\x82\xac", b"___", bs, 63)
    assert P.like(b"\xff", "�".encode(), bs, 46) and not P.like(b"\xff", "�".encode(), bs, 63)
    assert P.like(b"a ", b"a_", bs, 46) and not P.like(b"a ", b"a", bs, 46)   # LIKE does not cut trailing spaces


def test_compare_agrees_with_string_reference():
    vals = sorted(set(_words([b"a", b" ", b"\t", b"\x00", b"\xa0", "　".encode(), b"\xff"], 3)))
    for coll in (63, 46, 83, 65, 47, 309):
        for a in vals:
            for b in vals:
                assert P.compare(a, b, coll) == S.compare(a, b, coll), (a, b, coll)
    assert P.compare(b"a  ", b"a", 46) == 0 and P.compare(b"a  ", b"a", 309) == 1 and P.compare(b"a  ", b"a", 63) == 1
    for kept in (b"\t", b"\x00", b"\xa0", "　".encode()):
        assert P.compare(b"a" + kept, b"a", 46) == 1
