"""Plain-Python restatement of what the string VecEval kernels compute, the reference the GPU tests compare against.

Restated from the reference (pkg/util):
  - Go's `[]rune(s)` (unicode/utf8.DecodeRune): a byte that does not start a valid UTF-8 sequence is U+FFFD, width 1
  - stringutil.CompilePatternInner / CompilePatternInnerBinary (stringutil/string_util.go:154, :202)
  - stringutil.doMatchInner (string_util.go:301), with DoMatch / DoMatchBinary around it
  - collate.truncateTailingSpace, strings.Compare, and the collation id -> collator map (collate/collate.go:434-443,
    collate/bin.go)
Python's bytes.decode(errors="replace") groups some invalid sequences into one U+FFFD, which Go does not, so the decoder
here is written out byte by byte.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

RUNE_ERROR = 0xFFFD
PAT_MATCH, PAT_ONE, PAT_ANY = 1, 2, 3

# collator behaviours
BINARY, PAD_BIN, DERIVED = "binary", "pad_bin", "derived"
COLLATIONS = {63: BINARY, 46: PAD_BIN, 83: PAD_BIN, 65: PAD_BIN, 47: PAD_BIN, 309: DERIVED}


def collator_of(collation_id: int) -> Optional[str]:
    """binCollator (63), binPaddingCollator (the four *_bin ids), derivedBinCollator (309); None: not offloaded"""
    return COLLATIONS.get(collation_id)


def decode_rune(s: bytes, i: int) -> Tuple[int, int]:
    """utf8.DecodeRune(s[i:]) -> (rune, width)"""
    b0 = s[i]
    if b0 < 0x80:
        return b0, 1
    if 0xC2 <= b0 <= 0xDF:
        need, lo, hi = 1, 0x80, 0xBF
    elif 0xE0 <= b0 <= 0xEF:
        need, lo, hi = 2, (0xA0 if b0 == 0xE0 else 0x80), (0x9F if b0 == 0xED else 0xBF)
    elif 0xF0 <= b0 <= 0xF4:
        need, lo, hi = 3, (0x90 if b0 == 0xF0 else 0x80), (0x8F if b0 == 0xF4 else 0xBF)
    else:
        return RUNE_ERROR, 1
    if len(s) - i <= need or not lo <= s[i + 1] <= hi:
        return RUNE_ERROR, 1
    for k in range(2, need + 1):
        if not 0x80 <= s[i + k] <= 0xBF:
            return RUNE_ERROR, 1
    r = b0 & (0x1F, 0x0F, 0x07)[need - 1]
    for k in range(1, need + 1):
        r = (r << 6) | (s[i + k] & 0x3F)
    return r, need + 1


def runes(s: bytes) -> List[int]:
    """[]rune(s)"""
    out, i = [], 0
    while i < len(s):
        r, w = decode_rune(s, i)
        out.append(r)
        i += w
    return out


def compile_pattern(pattern: bytes, escape: int, over_runes: bool) -> Tuple[List[int], List[int]]:
    """CompilePatternInner (over_runes: the pattern's runes, the escape is rune(escape)) or CompilePatternInnerBinary"""
    chars = runes(pattern) if over_runes else list(pattern)
    weights: List[int] = []
    types: List[int] = []
    i = 0
    while i < len(chars):
        r = chars[i]
        if r == escape:
            tp = PAT_MATCH
            if i < len(chars) - 1:
                i += 1
                r = chars[i]
        elif r == ord("_"):
            if types and types[-1] == PAT_ANY:            # %_ => _%
                tp, r = PAT_ANY, ord("%")
                weights[-1], types[-1] = ord("_"), PAT_ONE
            else:
                tp = PAT_ONE
        elif r == ord("%"):
            if types and types[-1] == PAT_ANY:            # %% => %
                i += 1
                continue
            tp = PAT_ANY
        else:
            tp = PAT_MATCH
        weights.append(r)
        types.append(tp)
        i += 1
    return weights, types


def do_match(chars: Sequence[int], weights: Sequence[int], types: Sequence[int]) -> bool:
    """doMatchInner over a decoded string (runes, or bytes for DoMatchBinary)"""
    c = p = next_c = next_p = 0
    while p < len(weights) or c < len(chars):
        if p < len(weights):
            tp = types[p]
            if tp == PAT_MATCH:
                if c < len(chars) and chars[c] == weights[p]:
                    p += 1
                    c += 1
                    continue
            elif tp == PAT_ONE:
                if c < len(chars):
                    p += 1
                    c += 1
                    continue
            else:
                next_p, next_c = p, c + 1
                p += 1
                continue
        if 0 < next_c <= len(chars):
            p, c = next_p, next_c
            continue
        return False
    return True


def like(s: bytes, pattern: bytes, escape: int, collation_id: int) -> bool:
    """builtinLikeSig for one non-NULL row: the collator's Pattern().Compile(pattern, escape) then DoMatch(s)"""
    over_runes = collator_of(collation_id) != BINARY
    w, t = compile_pattern(pattern, escape, over_runes)
    return do_match(runes(s) if over_runes else list(s), w, t)


def truncate_tailing_space(s: bytes) -> bytes:
    """collate.truncateTailingSpace: only 0x20 is cut"""
    n = len(s)
    while n > 0 and s[n - 1] == 0x20:
        n -= 1
    return s[:n]


def strings_compare(a: bytes, b: bytes) -> int:
    """strings.Compare: unsigned bytes, a proper prefix first"""
    return (a > b) - (a < b)


def compare(a: bytes, b: bytes, collation_id: int) -> int:
    """Collator.Compare of the collation id's collator"""
    if collator_of(collation_id) == PAD_BIN:
        return strings_compare(truncate_tailing_space(a), truncate_tailing_space(b))
    return strings_compare(a, b)


def apply_cmp(op: int, c: int) -> bool:
    """TG_CMP_LT .. TG_CMP_NE applied to a three-way result"""
    return (c < 0, c <= 0, c > 0, c >= 0, c == 0, c != 0)[op]
