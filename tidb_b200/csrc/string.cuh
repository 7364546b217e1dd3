// string.cuh — var-length string values as the VecEval string kernels read them (host and device share these
// definitions): Go's rune decoding, the three offloaded collator behaviours, LIKE pattern compilation and the
// single-restart match walk.
//
// Replaces (pkg/util): collate.binCollator / binPaddingCollator / derivedBinCollator (collate/bin.go),
// truncateTailingSpace (collate/collate.go), stringutil.CompilePatternInner / CompilePatternInnerBinary / doMatchInner
// (stringutil/string_util.go:154, :202, :301) and unicode/utf8.DecodeRune as `[]rune(s)` uses it.
#pragma once
#include <cstdint>

namespace tg {

// ---- collations --------------------------------------------------------------------------------------------------
// The collator behaviour a MySQL collation id selects (collate.go newCollatorIDMap with new collations enabled).
enum StrColl {
  COLL_BINARY = 0,    // 63 binary: strings.Compare on the bytes, LIKE over bytes
  COLL_PAD_BIN = 1,   // 46 utf8mb4_bin, 83 utf8_bin, 65 ascii_bin, 47 latin1_bin: trailing 0x20 cut, LIKE over runes
  COLL_DERIVED = 2,   // 309 utf8mb4_0900_bin: strings.Compare on the bytes, LIKE over runes
  COLL_NONE = -1
};
__host__ __device__ __forceinline__ int coll_of_id(int32_t id) {
  switch (id) {
    case 63: return COLL_BINARY;
    case 46: case 83: case 65: case 47: return COLL_PAD_BIN;
    case 309: return COLL_DERIVED;
    default: return COLL_NONE;
  }
}

// truncateTailingSpace: the length without trailing 0x20 bytes (a tab is kept)
__host__ __device__ __forceinline__ int64_t str_trim_len(const uint8_t* s, int64_t n) {
  while (n > 0 && s[n - 1] == 0x20) n--;
  return n;
}

// strings.Compare: unsigned bytes, a proper prefix first
__host__ __device__ __forceinline__ int str_cmp_bytes(const uint8_t* a, int64_t na, const uint8_t* b, int64_t nb) {
  const int64_t m = na < nb ? na : nb;
  for (int64_t i = 0; i < m; i++) {
    const uint8_t x = a[i], y = b[i];
    if (x != y) return x < y ? -1 : 1;
  }
  return na < nb ? -1 : (na > nb ? 1 : 0);
}

// ---- Go's rune decoding ------------------------------------------------------------------------------------------
// utf8.DecodeRune: the rune at s[0] and its width.  Every byte that does not start a valid sequence (a stray
// continuation byte, a truncated sequence, an overlong form, a surrogate, a code point above U+10FFFF) is U+FFFD with
// width 1.  n >= 1.
static const int32_t kRuneError = 0xFFFD;
__host__ __device__ __forceinline__ int32_t decode_rune(const uint8_t* s, int64_t n, int* width) {
  const uint32_t b0 = s[0];
  *width = 1;
  if (b0 < 0x80) return (int32_t)b0;
  uint32_t lo = 0x80, hi = 0xBF;   // the accepted range of the second byte
  int need;
  if (b0 >= 0xC2 && b0 <= 0xDF) need = 1;
  else if (b0 >= 0xE0 && b0 <= 0xEF) { need = 2; if (b0 == 0xE0) lo = 0xA0; else if (b0 == 0xED) hi = 0x9F; }
  else if (b0 >= 0xF0 && b0 <= 0xF4) { need = 3; if (b0 == 0xF0) lo = 0x90; else if (b0 == 0xF4) hi = 0x8F; }
  else return kRuneError;
  if (n <= need) return kRuneError;
  const uint32_t b1 = s[1];
  if (b1 < lo || b1 > hi) return kRuneError;
  if (need == 1) { *width = 2; return (int32_t)(((b0 & 0x1F) << 6) | (b1 & 0x3F)); }
  const uint32_t b2 = s[2];
  if (b2 < 0x80 || b2 > 0xBF) return kRuneError;
  if (need == 2) { *width = 3; return (int32_t)(((b0 & 0x0F) << 12) | ((b1 & 0x3F) << 6) | (b2 & 0x3F)); }
  const uint32_t b3 = s[3];
  if (b3 < 0x80 || b3 > 0xBF) return kRuneError;
  *width = 4;
  return (int32_t)(((b0 & 0x07) << 18) | ((b1 & 0x3F) << 12) | ((b2 & 0x3F) << 6) | (b3 & 0x3F));
}

// ---- LIKE patterns -----------------------------------------------------------------------------------------------
enum { PAT_MATCH = 1, PAT_ONE = 2, PAT_ANY = 3 };   // stringutil.PatMatch / PatOne / PatAny

// CompilePatternInner (runes = true: over []rune(pattern), the escape is rune(escape)) or CompilePatternInnerBinary
// (runes = false: over the bytes).  The escape is tested before '_' and '%'; an escape as the last character is a
// literal; "%%" becomes "%" and "%_" becomes "_%".  weights / types need room for n entries; returns the compiled length.
__host__ __device__ inline int64_t compile_pattern(const uint8_t* p, int64_t n, int escape, bool runes, int32_t* weights,
                                                   uint8_t* types) {
  int64_t len = 0;
  for (int64_t i = 0; i < n;) {
    int w = 1;
    int32_t r = runes ? decode_rune(p + i, n - i, &w) : (int32_t)p[i];
    i += w;
    uint8_t tp;
    if (r == escape) {
      tp = PAT_MATCH;
      if (i < n) { r = runes ? decode_rune(p + i, n - i, &w) : (int32_t)p[i]; i += w; }
    } else if (r == '_') {
      if (len > 0 && types[len - 1] == PAT_ANY) { tp = PAT_ANY; r = '%'; weights[len - 1] = '_'; types[len - 1] = PAT_ONE; }
      else tp = PAT_ONE;
    } else if (r == '%') {
      if (len > 0 && types[len - 1] == PAT_ANY) continue;
      tp = PAT_ANY;
    } else {
      tp = PAT_MATCH;
    }
    weights[len] = r; types[len] = tp; len++;
  }
  return len;
}

// doMatchInner over the string's bytes (runes = false: DoMatchBinary) or its runes (DoMatch), positions kept in bytes:
// the single restart point is the position one character past where the last '%' started matching.
template <bool RUNES>
__host__ __device__ inline bool like_match(const uint8_t* s, int64_t n, const int32_t* weights, const uint8_t* types,
                                           int64_t plen) {
  int64_t c = 0, p = 0, next_c = 0, next_p = 0;   // next_c == 0: no restart point yet
  while (p < plen || c < n) {
    if (p < plen) {
      const uint8_t tp = types[p];
      if (tp == PAT_ANY) {
        next_p = p;
        if (c < n) { int w = 1; if (RUNES) decode_rune(s + c, n - c, &w); next_c = c + w; }
        else next_c = n + 1;
        p++;
        continue;
      }
      if (c < n) {
        int w = 1;
        const int32_t r = RUNES ? decode_rune(s + c, n - c, &w) : (int32_t)s[c];
        if (tp == PAT_ONE || r == weights[p]) { p++; c += w; continue; }
      }
    }
    if (0 < next_c && next_c <= n) { p = next_p; c = next_c; continue; }
    return false;
  }
  return true;
}

}  // namespace tg
