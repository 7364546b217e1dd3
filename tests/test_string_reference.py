"""Pins tests/string_reference.py (the reference of the string VecEval kernels) to the reference's own tables, then to
hand cases for invalid UTF-8, high escapes, '%' as the escape, a trailing escape and the empty pattern."""
import pytest

import string_reference as S

BS = ord("\\")
UTF8MB4_BIN, BINARY, BIN0900 = 46, 63, 309

# stringutil TestPatternMatch (pkg/util/stringutil/string_util_test.go:68): pattern, input, escape, match; CompilePattern
# and DoMatch, the rune walk
PATTERN_MATCH = [
    ("", "a", "\\", False), ("a", "a", "\\", True), ("a", "b", "\\", False), ("aA", "aA", "\\", True),
    ("_", "a", "\\", True), ("_", "ab", "\\", False), ("__", "b", "\\", False), ("%", "abcd", "\\", True),
    ("%", "", "\\", True), ("%b", "AAA", "\\", False), ("%a%", "BBB", "\\", False), ("a%", "BBB", "\\", False),
    ("\\%a", "%a", "\\", True), ("\\%a", "aa", "\\", False), ("\\_a", "_a", "\\", True), ("\\_a", "aa", "\\", False),
    ("\\\\_a", "\\xa", "\\", True), ("\\a\\b", "\\a\\b", "\\", False), ("\\a\\b", "ab", "\\", True),
    ("%%_", "abc", "\\", True), ("%_%_aA", "aaaA", "\\", True), ("+_a", "_a", "+", True), ("+%a", "%a", "+", True),
    ("\\%a", "%a", "+", False), ("++a", "+a", "+", True), ("+a", "a", "+", True), ("++_a", "+xa", "+", True),
    ("___Հ", "䇇Հ", "\\", False),
]

# expression TestLike (pkg/expression/builtin_like_test.go:30): input, pattern, match; escape '\\', the default
# collation utf8mb4_bin
LIKE = [
    ("a", "", 0), ("a", "a", 1), ("a", "b", 0), ("aA", "Aa", 0), ("aAb", "Aa%", 0), ("aAb", "aA_", 1),
    ("baab", "b_%b", 1), ("baab", "b%_b", 1), ("bab", "b_%b", 1), ("bab", "b%_b", 1), ("bb", "b_%b", 0),
    ("bb", "b%_b", 0), ("baabccc", "b_%b%", 1), ("a", "\\a", 1),
]

# collate TestUTF8CollatorCompare (pkg/util/collate/collate_test.go:57): left, right, and the expected Compare under
# binary, utf8mb4_bin and utf8mb4_0900_bin (columns 1, 2 and 6 of the table)
COLLATOR_COMPARE = [
    ("a", "b", (-1, -1, -1)), ("a", "A", (1, 1, 1)), ("À", "A", (1, 1, 1)), ("abc", "abc", (0, 0, 0)),
    ("abc", "ab", (1, 1, 1)), ("😜", "😃", (1, 1, 1)), ("a", "a ", (-1, 0, -1)), ("a ", "a  ", (-1, 0, -1)),
    ("a\t", "a", (1, 1, 1)), ("ß", "s", (1, 1, 1)), ("ß", "ss", (1, 1, 1)), ("啊", "吧", (1, 1, 1)),
    ("中文", "汉字", (-1, -1, -1)), ("æ", "ae", (1, 1, 1)), ("Å", "A", (1, 1, 1)), ("Å", "A", (1, 1, 1)),
    ("\U0001730F", "啊", (1, 1, 1)), ("가", "㉡", (1, 1, 1)), ("갟", "감1", (1, 1, 1)),
    ("\U000FFFFE", "\U000FFFFF", (-1, -1, -1)),
]


@pytest.mark.parametrize("pattern,s,escape,match", PATTERN_MATCH)
def test_pattern_match(pattern, s, escape, match):
    w, t = S.compile_pattern(pattern.encode(), ord(escape), True)
    assert S.do_match(S.runes(s.encode()), w, t) == match


@pytest.mark.parametrize("s,pattern,match", LIKE)
def test_like(s, pattern, match):
    assert S.like(s.encode(), pattern.encode(), BS, UTF8MB4_BIN) == bool(match)
    assert S.like(s.encode(), pattern.encode(), BS, BIN0900) == bool(match)
    assert S.like(s.encode(), pattern.encode(), BS, BINARY) == bool(match)   # ASCII: bytes and runes agree


@pytest.mark.parametrize("a,b,expect", COLLATOR_COMPARE)
def test_collator_compare(a, b, expect):
    for cid, e in zip((BINARY, UTF8MB4_BIN, BIN0900), expect):
        assert S.compare(a.encode(), b.encode(), cid) == e
        assert S.compare(b.encode(), a.encode(), cid) == -e


def test_collation_ids():
    assert [S.collator_of(i) for i in (63, 46, 83, 65, 47, 309)] == [S.BINARY] + [S.PAD_BIN] * 4 + [S.DERIVED]
    for ci in (33, 45, 224, 255, 28, 87, 248, 249, 0, 8):   # _ci, gbk, gb18030, latin1_swedish_ci, ...
        assert S.collator_of(ci) is None


def test_rune_decoding_matches_go():
    # every class of invalid sequence is one U+FFFD per byte (utf8.DecodeRune width 1)
    E = S.RUNE_ERROR
    assert S.runes(b"\xe2\x82") == [E, E]                 # truncated 3-byte sequence
    assert S.runes(b"\xe2\x82\xac") == [0x20AC]
    assert S.runes(b"\xc0\xaf") == [E, E]                 # overlong
    assert S.runes(b"\xe0\x80\xaf") == [E, E, E]          # overlong 3-byte
    assert S.runes(b"\xed\xa0\x80") == [E, E, E]          # surrogate U+D800
    assert S.runes(b"\xf4\x90\x80\x80") == [E, E, E, E]   # above U+10FFFF
    assert S.runes(b"\xf0\x9f\x98") == [E, E, E]
    assert S.runes(b"\x80a\xff") == [E, ord("a"), E]
    assert S.runes(b"\xf0\x9f\x98\x9c") == [0x1F61C]
    assert S.runes("�".encode()) == [E]
    # Python's replacement decoding groups a truncated sequence into one U+FFFD; Go does not
    assert len(b"\xe2\x82".decode("utf-8", errors="replace")) == 1


def test_like_invalid_utf8():
    assert S.like(b"\xe2\x82", b"__", BS, UTF8MB4_BIN)            # two invalid bytes are two runes
    assert not S.like(b"\xe2\x82", b"_", BS, UTF8MB4_BIN)
    assert S.like(b"\xe2\x82", b"__", BS, BINARY)                 # and two bytes
    assert S.like(b"\xe2\x82\xac", b"_", BS, UTF8MB4_BIN) and not S.like(b"\xe2\x82\xac", b"_", BS, BINARY)
    # an invalid byte and a valid U+FFFD match each other, over runes only
    assert S.like(b"\xff", "�".encode(), BS, UTF8MB4_BIN)
    assert S.like("�".encode(), b"\xff", BS, BIN0900)
    assert not S.like(b"\xff", "�".encode(), BS, BINARY)
    assert S.like(b"x\xffy", b"x_y", BS, UTF8MB4_BIN)


def test_high_escape_is_a_rune():
    # rune(0xE9) is 'é': over runes the escape matches the character, not the byte 0xE9
    e9 = 0xE9
    assert S.compile_pattern("é%".encode(), e9, True) == ([ord("%")], [S.PAT_MATCH])
    assert S.like(b"%", "é%".encode(), e9, UTF8MB4_BIN) and not S.like(b"ab", "é%".encode(), e9, UTF8MB4_BIN)
    assert S.compile_pattern(b"\xe9%", e9, False) == ([ord("%")], [S.PAT_MATCH])
    assert S.like(b"%", b"\xe9%", e9, BINARY)
    # the raw byte 0xE9 in a rune pattern decodes to U+FFFD, which is not the escape
    assert S.compile_pattern(b"\xe9%", e9, True) == ([S.RUNE_ERROR, ord("%")], [S.PAT_MATCH, S.PAT_ANY])


def test_percent_and_underscore_as_escape():
    pc = ord("%")
    assert S.compile_pattern(b"%%a", pc, True) == ([ord("%"), ord("a")], [S.PAT_MATCH, S.PAT_MATCH])
    assert S.like(b"%a", b"%%a", pc, UTF8MB4_BIN) and not S.like(b"xa", b"%%a", pc, UTF8MB4_BIN)
    assert S.like(b"ab", b"a_", pc, UTF8MB4_BIN)          # '_' still a wildcard
    us = ord("_")
    assert S.like(b"_", b"__", us, UTF8MB4_BIN) and not S.like(b"x", b"__", us, UTF8MB4_BIN)


def test_trailing_escape_and_empty_pattern():
    assert S.compile_pattern(b"ab\\", BS, True) == ([97, 98, BS], [S.PAT_MATCH] * 3)
    assert S.like(b"ab\\", b"ab\\", BS, UTF8MB4_BIN) and not S.like(b"ab", b"ab\\", BS, UTF8MB4_BIN)
    assert S.like(b"", b"", BS, UTF8MB4_BIN) and not S.like(b" ", b"", BS, UTF8MB4_BIN)
    assert S.like(b"", b"%", BS, BINARY) and not S.like(b"", b"_", BS, BINARY)


def test_compile_rewrites():
    assert S.compile_pattern(b"a%%%b", BS, True) == ([97, 37, 98], [S.PAT_MATCH, S.PAT_ANY, S.PAT_MATCH])
    assert S.compile_pattern(b"%_", BS, True) == ([95, 37], [S.PAT_ONE, S.PAT_ANY])
    assert S.compile_pattern(b"%__%", BS, False) == ([95, 95, 37], [S.PAT_ONE, S.PAT_ONE, S.PAT_ANY])


def test_like_trailing_spaces_count():
    assert not S.like(b"a ", b"a", BS, UTF8MB4_BIN) and S.compare(b"a ", b"a", UTF8MB4_BIN) == 0
    assert S.compare(b"a\t", b"a", UTF8MB4_BIN) == 1 and S.compare(b"\x80", b"\x7f", BINARY) == 1
    assert S.compare(b"a\x00", b"a", UTF8MB4_BIN) == 1 and S.compare(b"a\x00", b"a ", UTF8MB4_BIN) == 1
