// decimal.cuh — the MyDecimal cell of an exact DECIMAL aggregate result (included by agg.cu; only k_agg_finalize uses it).
//
// A cell is the 40-byte types.MyDecimal (types/mydecimal.go:236-248) that chunk.Column copies whole (util/chunk/column.go:41):
//   byte 0 digitsInt (int8), byte 1 digitsFrac (int8), byte 2 resultFrac (int8), byte 3 negative (bool),
//   then int32 wordBuf[9] in base 10^9, most significant word first: integer words, then fraction words, the rest 0.
// The library writes one canonical form: digitsInt = 9 * the number of integer words, at least one word (FromUint,
// mydecimal.go:1069), digitsFrac = resultFrac = the result scale, and a zero result is never negative.  The update
// kernels only see the 128-bit sum in two state words; this header is the one place that knows the layout.
#pragma once

namespace tg {

#define TG_DEC_CELL_BYTES 40
#define TG_DEC_WORD_BASE 1000000000u

__device__ __forceinline__ uint32_t dec_pow10(int k) {
  uint32_t p = 1;
  for (int j = 0; j < k; j++) p *= 10u;
  return p;
}

// integer part `ip` (magnitude) and `nfw` fraction words -> the cell
__device__ __forceinline__ void dec_store(uint8_t* cell, bool neg, unsigned __int128 ip, const uint32_t* fw, int nfw, int frac) {
  uint32_t iw[5];   // < 2^127 has at most 39 digits
  int ni = 0;
  do { iw[ni++] = (uint32_t)(ip % TG_DEC_WORD_BASE); ip /= TG_DEC_WORD_BASE; } while (ip != 0 && ni < 5);
  uint32_t c[10];
  for (int j = 0; j < 10; j++) c[j] = 0;
  c[0] = (uint32_t)(9 * ni) | ((uint32_t)frac << 8) | ((uint32_t)frac << 16) | ((neg ? 1u : 0u) << 24);
  for (int j = 0; j < ni; j++) c[1 + j] = iw[ni - 1 - j];
  for (int j = 0; j < nfw; j++) c[1 + ni + j] = fw[j];
  unsigned long long* o = reinterpret_cast<unsigned long long*>(cell);   // cells are 8-byte aligned (40-byte stride)
  for (int j = 0; j < 5; j++) o[j] = (unsigned long long)c[2 * j] | ((unsigned long long)c[2 * j + 1] << 32);
}

__device__ __forceinline__ void dec_store_null(uint8_t* cell) {
  unsigned long long* o = reinterpret_cast<unsigned long long*>(cell);
  for (int j = 0; j < 5; j++) o[j] = 0;
}

__device__ __forceinline__ __int128 dec_sum_of(unsigned long long lo, unsigned long long hi) {
  return (__int128)(((unsigned __int128)hi << 64) | lo);
}

// SUM: the exact sum at scale 0 (sum4Decimal, func_sum.go:207-253; its final Round to 0 digits leaves an integer alone)
__device__ __noinline__ void dec_sum_cell(uint8_t* cell, unsigned long long lo, unsigned long long hi) {
  const __int128 s = dec_sum_of(lo, hi);
  const bool neg = s < 0;
  dec_store(cell, neg, neg ? (unsigned __int128)(-s) : (unsigned __int128)s, nullptr, 0, 0);
}

// AVG: DecimalDiv(sum, count, frac) then Round(frac, ModeHalfUp) (baseAvgDecimal.AppendFinalResult2Chunk, func_avg.go:84-109).
// doDivMod (mydecimal.go:2203) truncates the quotient at 9 * ceil(frac / 9) fraction digits; Round then looks only at the
// first digit after the scale and rounds the magnitude.  With frac a multiple of 9 there is no such digit in the quotient,
// so the result is the truncated quotient.  A quotient or rounded result of zero loses its sign (doDivMod and Round both
// clear `negative` on zero).  `n` < 2^63, so r * 10^9 fits 128 bits.
__device__ __noinline__ void dec_avg_cell(uint8_t* cell, unsigned long long lo, unsigned long long hi, unsigned long long n, int frac) {
  const __int128 s = dec_sum_of(lo, hi);
  const bool neg = s < 0;
  const unsigned __int128 m = neg ? (unsigned __int128)(-s) : (unsigned __int128)s;
  unsigned __int128 q = m / n;
  unsigned long long r = (unsigned long long)(m % n);
  const int nfw = (frac + 8) / 9;
  uint32_t fw[4];   // frac <= 30
  for (int j = 0; j < nfw; j++) {
    const unsigned __int128 x = (unsigned __int128)r * TG_DEC_WORD_BASE;
    fw[j] = (uint32_t)(x / n);
    r = (unsigned long long)(x % n);
  }
  if (frac % 9) {   // Round, mydecimal.go:892-898: keep the word's first frac % 9 digits, half up on the next one
    const uint32_t p = dec_pow10(9 - frac % 9 - 1);
    unsigned long long sh = fw[nfw - 1] / p;
    const unsigned long long dig = sh % 10;
    if (dig >= 5) sh += 10;
    unsigned long long w = (unsigned long long)p * (sh - dig);
    int j = nfw - 1;
    for (;;) {   // carry into the words before it and the integer part (999.99995 -> 1000.0000)
      if (w < TG_DEC_WORD_BASE) { fw[j] = (uint32_t)w; break; }
      fw[j] = (uint32_t)(w - TG_DEC_WORD_BASE);
      if (--j < 0) { q += 1; break; }
      w = (unsigned long long)fw[j] + 1;
    }
  }
  bool zero = q == 0;
  for (int j = 0; j < nfw; j++) zero &= fw[j] == 0;
  dec_store(cell, neg && !zero, q, fw, nfw, frac);
}

}  // namespace tg
