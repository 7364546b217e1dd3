// decimal.cuh — the MyDecimal cell of an exact DECIMAL aggregate result and of a DECIMAL argument column (included by agg.cu:
// k_agg_finalize writes cells, k_dec_to_scaled parses them), and the order of cells (included by topn.cu, and by vec.cu
// for the DECIMAL compares and filters).
//
// A cell is the 40-byte types.MyDecimal (types/mydecimal.go:236-248) that chunk.Column copies whole (util/chunk/column.go:41):
//   byte 0 digitsInt (int8), byte 1 digitsFrac (int8), byte 2 resultFrac (int8), byte 3 negative (bool),
//   then int32 wordBuf[9] in base 10^9, most significant word first: integer words, then fraction words, the rest 0.
// The library writes one canonical form: digitsInt = 9 * the number of integer words, at least one word (FromUint,
// mydecimal.go:1069), digitsFrac = resultFrac = the result scale, and a zero result is never negative.  The update
// kernels only see the 128-bit sum in two state words (192 bits in three for a product of DECIMAL columns), or the int64
// value * 10^scale of a DECIMAL argument; this header is the one place that knows the layout.
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

__device__ __forceinline__ unsigned long long dec_pow10_u64(int k) {
  unsigned long long p = 1;
  for (int j = 0; j < k; j++) p *= 10ull;
  return p;
}

// ---- input cells of a DECIMAL(flen, scale) argument column, flen <= 18 --------------------------------------------------
// A stored cell (MyDecimal.FromBin, mydecimal.go:1465) has digitsFrac == scale, ceil(digitsInt / 9) integer words (digitsInt
// may be 0, and leading integer words may be 0), then ceil(scale / 9) fraction words, left-aligned: 0.5 at scale 1 is the
// word 500000000.  resultFrac is not looked at, nor are the words after the fraction words.  Returns false for a cell in
// any other form (digitsFrac != scale, a word >= 10^9, digits after the scale, more than flen significant digits); else
// *v = value * 10^scale, |*v| < 10^flen <= 10^18, and a negative zero is 0.  c[0] is the header word (bytes digitsInt,
// digitsFrac, resultFrac, negative), c[1..9] the words; every index is a constant, so c stays in registers.
__device__ __forceinline__ bool dec_parse_cell(const uint32_t (&c)[10], int flen, int scale, long long* v) {
  const int di = (int)(int8_t)(c[0] & 0xffu), df = (int)(int8_t)((c[0] >> 8) & 0xffu);
  const bool neg = (c[0] >> 24) != 0;
  if (df != scale || di < 0) return false;
  const int wi = (di + 8) / 9, wf = (scale + 8) / 9;   // wf <= 2
  if (wi + wf > 9) return false;
  unsigned long long ip = 0, fr = 0;
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 9; j++) {
    const uint32_t w = c[1 + j];
    if (j < wi) {
      // 1844674407 * 10^9 > 10^18 >= the bound checked below: a larger prefix is too many digits, and this keeps ip in 64 bits
      if (w >= TG_DEC_WORD_BASE || ip >= 1844674407ull) ok = false;
      else ip = ip * TG_DEC_WORD_BASE + w;
    } else if (j < wi + wf) {
      if (w >= TG_DEC_WORD_BASE) ok = false;
      fr = fr * TG_DEC_WORD_BASE + w;
    }
  }
  const unsigned long long pad = dec_pow10_u64(9 * wf - scale);
  if (!ok || fr % pad != 0 || ip >= dec_pow10_u64(flen - scale)) return false;
  const unsigned long long m = ip * dec_pow10_u64(scale) + fr / pad;
  *v = neg ? -(long long)m : (long long)m;
  return true;
}

// SUM: the exact sum at the argument's scale (sum4Decimal, func_sum.go:207-253; its final Round to the scale leaves the sum
// alone).  The integer part is |sum| / 10^scale; the remainder, left-aligned, gives the ceil(scale / 9) fraction words.  A
// DECIMAL MIN / MAX writes its int64 here too (hi = the sign extension).
static __device__ __noinline__ void dec_sum_cell(uint8_t* cell, unsigned long long lo, unsigned long long hi, int scale) {
  const __int128 s = dec_sum_of(lo, hi);
  const bool neg = s < 0;
  unsigned __int128 m = neg ? (unsigned __int128)(-s) : (unsigned __int128)s;
  const int nfw = (scale + 8) / 9;   // scale <= 18
  uint32_t fw[2] = {0, 0};
  if (scale) {
    const unsigned long long p = dec_pow10_u64(scale);
    const unsigned long long r = (unsigned long long)(m % p) * dec_pow10_u64(9 * nfw - scale);   // < 10^(9 nfw) <= 10^18
    m /= p;
    if (nfw == 2) { fw[0] = (uint32_t)(r / TG_DEC_WORD_BASE); fw[1] = (uint32_t)(r % TG_DEC_WORD_BASE); }
    else fw[0] = (uint32_t)r;
  }
  dec_store(cell, neg, m, fw, nfw, scale);
}

// AVG: DecimalDiv(sum, count, incr) then Round(frac, ModeHalfUp) (baseAvgDecimal.AppendFinalResult2Chunk, func_avg.go:84-109),
// for a sum of `scale` fraction digits and frac = min(scale + incr, 30) (typeInfer4Avg, base_func.go:274).
// Why the quotient is truncated at 9 * ceil(frac / 9) fraction digits for every div_precision_increment `incr`: every input
// cell has digitsFrac == scale, so the sum does too (DecimalAdd keeps the larger digitsFrac), and the count has 0.  doDivMod
// (mydecimal.go:2203) then computes ceil((9 * ceil(scale / 9) + max(0, incr - (9 * ceil(scale / 9) - scale))) / 9) =
// ceil((scale + incr) / 9) fraction words of the quotient, truncated, i.e. T = 9 * ceil((scale + incr) / 9) digits.  When
// scale + incr <= 30, frac = scale + incr and T = 9 * ceil(frac / 9).  When it is capped (frac = 30), T >= 36 > 31 digits:
// the first 31 digits are those of the exact quotient either way, and Round looks only at the first digit after the scale,
// so truncating at 36 = 9 * ceil(30 / 9) gives the same result.  Round rounds the magnitude half up on digit frac + 1; with
// frac a multiple of 9 (uncapped) there is no such digit in the quotient, so the result is the truncated quotient.  A
// quotient or rounded result of zero loses its sign (doDivMod and Round both clear `negative` on zero).
// The value is sum / (count * 10^scale), and count * 10^scale can pass 64 bits: the digits are those of m / n (m = |sum|),
// with the point moved `scale` places, so the integer part is q / 10^scale (q = m / n), the fraction digits are the low
// `scale` digits of q, then the digits of r / n (r = m % n).  `n` < 2^63, so r * 10^9 fits 128 bits.  frac >= scale.
static __device__ __noinline__ void dec_avg_cell(uint8_t* cell, unsigned long long lo, unsigned long long hi, unsigned long long n, int scale, int frac) {
  const __int128 s = dec_sum_of(lo, hi);
  const bool neg = s < 0;
  const unsigned __int128 m = neg ? (unsigned __int128)(-s) : (unsigned __int128)s;
  unsigned __int128 q = m / n;
  unsigned long long r = (unsigned long long)(m % n);
  const int nfw = (frac + 8) / 9;
  uint32_t fw[4];   // frac <= 30
  // the low `scale` digits of q: its first 9 * (scale / 9) digits as whole words (`top`), then the last scale % 9 digits
  // (`carry`), which shift the words of r / n right by scale % 9 digits (scale 0: top = carry = 0, the words of r / n as they are)
  const int aw = scale / 9;
  const unsigned long long pb = dec_pow10(scale % 9), lift = TG_DEC_WORD_BASE / pb;
  unsigned long long low = 0;
  if (scale) {   // a DECIMAL(p <= 18) argument: |sum| < n * 10^18, so q < 10^18 fits 64 bits
    const unsigned long long q64 = (unsigned long long)q, p = dec_pow10_u64(scale);
    low = q64 % p;
    q = q64 / p;
  }
  const unsigned long long top = low / pb;
  unsigned long long carry = low % pb;
  for (int j = 0; j < nfw; j++) {
    if (j < aw) { fw[j] = (uint32_t)(aw == 2 && j == 0 ? top / TG_DEC_WORD_BASE : top % TG_DEC_WORD_BASE); continue; }
    const unsigned __int128 x = (unsigned __int128)r * TG_DEC_WORD_BASE;
    const unsigned long long e = (unsigned long long)(x / n);
    r = (unsigned long long)(x % n);
    fw[j] = (uint32_t)(carry * lift + e / pb);
    carry = e % pb;
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

// the one call k_agg_finalize makes for a non-NULL DECIMAL result: AVG, or SUM / MIN / MAX (one call site instead of two
// keeps the kernel at 64 registers)
static __device__ __noinline__ void dec_result_cell(uint8_t* cell, bool avg, unsigned long long lo, unsigned long long hi, unsigned long long n, int scale, int frac) {
  if (avg) dec_avg_cell(cell, lo, hi, n, scale, frac);
  else dec_sum_cell(cell, lo, hi, scale);
}

// 192-bit magnitudes, least significant word first: m /= d, returns m % d (d < 2^64; each step's quotient fits 64 bits
// because the running remainder is below d)
__device__ __forceinline__ unsigned long long dec_divmod192(unsigned long long (&m)[3], unsigned long long d) {
  unsigned long long r = 0;
#pragma unroll
  for (int j = 2; j >= 0; j--) {
    const unsigned __int128 x = ((unsigned __int128)r << 64) | m[j];
    m[j] = (unsigned long long)(x / d);
    r = (unsigned long long)(x % d);
  }
  return r;
}

// the two's-complement 192-bit sum (top:mid:lo) -> its magnitude in m; returns the sign
__device__ __forceinline__ bool dec_magnitude(unsigned long long (&m)[3], unsigned long long lo, unsigned long long mid, unsigned long long top) {
  const bool neg = (long long)top < 0;
  m[0] = lo; m[1] = mid; m[2] = top;
  if (neg) {
    m[0] = ~m[0] + 1ull;
    unsigned long long c = m[0] == 0 ? 1ull : 0ull;
    m[1] = ~m[1] + c;
    c = (c && m[1] == 0) ? 1ull : 0ull;
    m[2] = ~m[2] + c;
  }
  return neg;
}

// dec_store for a 192-bit integer part `ip` (magnitude, consumed).  ip < 2^184 has at most 56 digits, 7 words;
// the callers' bounds keep ni + nfw <= 9 (dec3_sum_cell, dec3_avg_cell)
__device__ __forceinline__ void dec3_store(uint8_t* cell, bool neg, unsigned long long (&ip)[3], const uint32_t* fw, int nfw, int frac) {
  uint32_t iw[7];
  int ni = 0;
  do { iw[ni++] = (uint32_t)dec_divmod192(ip, TG_DEC_WORD_BASE); } while ((ip[0] | ip[1] | ip[2]) != 0 && ni < 7);
  uint32_t c[10];
  for (int j = 0; j < 10; j++) c[j] = 0;
  c[0] = (uint32_t)(9 * ni) | ((uint32_t)frac << 8) | ((uint32_t)frac << 16) | ((neg ? 1u : 0u) << 24);
  for (int j = 0; j < ni; j++) c[1 + j] = iw[ni - 1 - j];
  for (int j = 0; j < nfw; j++) c[1 + ni + j] = fw[j];
  unsigned long long* o = reinterpret_cast<unsigned long long*>(cell);   // cells are 8-byte aligned (40-byte stride)
  for (int j = 0; j < 5; j++) o[j] = (unsigned long long)c[2 * j] | ((unsigned long long)c[2 * j + 1] << 32);
}

// ---- cells of a DECIMAL SUM / AVG of a product (k_agg_finalize<true, true>) ------------------------------------------
// The same rules as dec_sum_cell / dec_avg_cell above, for the exact 192-bit two's-complement sum (top:mid:lo) of DECIMAL
// products a * b / a * (c - b) at scale s = s_a + s_b <= 30.  They stay beside the 128-bit writers, which every other plan
// keeps: the long division of three words costs registers (a kernel's count includes its callees').  Why every accepted
// result fits MyDecimal's 9 words, so that fixWordCntError (mydecimal.go) never truncates a fraction word:
//   SUM: |sum| < 2^184 has at most 56 digits.  Its integer part has at most 56 - scale of them, so
//        ceil((56 - scale) / 9) + ceil(scale / 9) <= 8 words at any scale.
//   AVG: |avg| = |sum| / n < 2 * 10^(36 - scale) (|a * t| < 10^18 * 2 * 10^18, in units of 10^-scale): at most 37 - scale
//        integer digits, ceil((37 - scale) / 9) <= 5 words, and frac <= 30 gives at most 4 fraction words; 5 + 4 = 9 only
//        at scale 0.

// SUM: the integer part is |sum| / 10^scale; the remainder, left-aligned, gives the ceil(scale / 9) fraction words: the
// last scale % 9 digits first (padded to a whole word), then whole words towards the point.
static __device__ __noinline__ void dec3_sum_cell(uint8_t* cell, unsigned long long lo, unsigned long long mid, unsigned long long top, int scale) {
  unsigned long long m[3];
  const bool neg = dec_magnitude(m, lo, mid, top);
  const int aw = scale / 9, nfw = (scale + 8) / 9;   // scale <= 30
  uint32_t fw[4] = {0, 0, 0, 0};
  if (scale % 9) {
    const uint32_t pb = dec_pow10(scale % 9);
    fw[aw] = (uint32_t)dec_divmod192(m, pb) * (TG_DEC_WORD_BASE / pb);
  }
  for (int j = aw - 1; j >= 0; j--) fw[j] = (uint32_t)dec_divmod192(m, TG_DEC_WORD_BASE);
  dec3_store(cell, neg, m, fw, nfw, scale);
}

// AVG: dec_avg_cell's rule (the truncation at 9 * ceil(frac / 9) digits derived there holds for any scale <= 30: a product
// has digitsFrac s_a + s_b, so the sum does too).  q = m / n by 192-bit long division (n < 2^63); the integer part is
// q / 10^scale, the fraction digits are the low `scale` digits of q, then the digits of r / n (r * 10^9 fits 128 bits).
static __device__ __noinline__ void dec3_avg_cell(uint8_t* cell, unsigned long long lo, unsigned long long mid, unsigned long long top, unsigned long long n, int scale, int frac) {
  unsigned long long q[3];
  const bool neg = dec_magnitude(q, lo, mid, top);
  unsigned long long r = dec_divmod192(q, n);
  const int nfw = (frac + 8) / 9;
  uint32_t fw[4];   // frac <= 30
  // the low `scale` digits of q: the last scale % 9 of them (`carry`) shift the words of r / n right by scale % 9 digits;
  // the 9 * (scale / 9) before them are whole words (scale 0: no words, carry 0, the words of r / n as they are)
  const int aw = scale / 9;
  const unsigned long long pb = dec_pow10(scale % 9), lift = TG_DEC_WORD_BASE / pb;
  unsigned long long carry = scale % 9 ? dec_divmod192(q, pb) : 0ull;
  for (int j = aw - 1; j >= 0; j--) fw[j] = (uint32_t)dec_divmod192(q, TG_DEC_WORD_BASE);
  for (int j = aw; j < nfw; j++) {
    const unsigned __int128 x = (unsigned __int128)r * TG_DEC_WORD_BASE;
    const unsigned long long e = (unsigned long long)(x / n);
    r = (unsigned long long)(x % n);
    fw[j] = (uint32_t)(carry * lift + e / pb);
    carry = e % pb;
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
      if (--j < 0) { if (++q[0] == 0 && ++q[1] == 0) ++q[2]; break; }
      w = (unsigned long long)fw[j] + 1;
    }
  }
  bool zero = (q[0] | q[1] | q[2]) == 0;
  for (int j = 0; j < nfw; j++) zero &= fw[j] == 0;
  dec3_store(cell, neg && !zero, q, fw, nfw, frac);
}

// the one call k_agg_finalize<true, true> makes for a non-NULL product result (the scale, AVG's scale and the AVG flag in
// one word `how` = scale | frac << 8 | avg << 16: fewer argument registers)
static __device__ __noinline__ void dec3_result_cell(uint8_t* cell, unsigned long long lo, unsigned long long mid, unsigned long long top, unsigned long long n, int how) {
  const int scale = how & 0xff, frac = (how >> 8) & 0xff;
  if (how >> 16) dec3_avg_cell(cell, lo, mid, top, n, scale, frac);
  else dec3_sum_cell(cell, lo, mid, top, scale);
}

// ---- ordering cells of any form (TopN: k_topn_rank_dec on the device, the exact comparator on the host) ---------------
// The order is MyDecimal.Compare (mydecimal.go:1623, through chunk cmpMyDecimal): the sign first, so a negative zero sorts
// after every negative value and before +0 (and all negative zeros are equal); then doSub's word comparison of the
// magnitudes: ceil(digitsInt / 9) integer words, then ceil(digitsFrac / 9) fraction words, left-aligned, with leading zero
// integer words and trailing zero fraction words not counted.  resultFrac and the words after the used ones are not
// looked at.  c[0] is the header word, c[1..9] the words, as in dec_parse_cell.

__host__ __device__ __forceinline__ int dec_int_words(uint32_t hdr) { return ((int)(int8_t)(hdr & 0xffu) + 8) / 9; }
__host__ __device__ __forceinline__ int dec_frac_words(uint32_t hdr) { return ((int)(int8_t)((hdr >> 8) & 0xffu) + 8) / 9; }
__host__ __device__ __forceinline__ bool dec_negative(uint32_t hdr) { return (hdr >> 24) != 0; }

// a cell Compare can read: digitsInt >= 0, digitsFrac >= 0, at most 9 integer and fraction words, each below 10^9
__host__ __device__ __forceinline__ bool dec_cell_ok(const uint32_t (&c)[10]) {
  const int di = (int)(int8_t)(c[0] & 0xffu), df = (int)(int8_t)((c[0] >> 8) & 0xffu);
  if (di < 0 || df < 0) return false;
  const int n = (di + 8) / 9 + (df + 8) / 9;
  if (n > 9) return false;
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 9; j++) ok &= j >= n || c[1 + j] < TG_DEC_WORD_BASE;
  return ok;
}

// Word j (0..8) of a cell, for dec_cmp_words: DecWordsPtr reads a cell in memory (the host comparator, a constant in
// kernel parameter space); DecWordsReg reads a cell held in registers, selecting among its nine words so that every
// index into c is a constant (a dynamic index would move the cell to local memory).
struct DecWordsPtr {
  const uint32_t* c;
  __host__ __device__ __forceinline__ uint32_t operator()(int j) const { return c[1 + j]; }
};
struct DecWordsReg {
  const uint32_t (&c)[10];
  __device__ __forceinline__ uint32_t operator()(int j) const {
    uint32_t w = 0;
#pragma unroll
    for (int t = 0; t < 9; t++) w = t == j ? c[1 + t] : w;
    return w;
  }
};

// -1 / 0 / 1: MyDecimal.Compare of two well-formed cells (header words ha / hb, words read through wa / wb).  Integer
// words are right-aligned and fraction words left-aligned on the point (a missing word is 0), which is doSub's comparison
// once leading and trailing zero words are dropped.  On a malformed cell it returns some value and reads no memory
// outside the cell's nine words through DecWordsReg.
template <typename WA, typename WB>
__host__ __device__ __forceinline__ int dec_cmp_words(uint32_t ha, const WA& wa_at, uint32_t hb, const WB& wb_at) {
  const bool na = dec_negative(ha), nb = dec_negative(hb);
  if (na != nb) return na ? -1 : 1;
  const int ia = dec_int_words(ha), ib = dec_int_words(hb);
  const int ea = ia + dec_frac_words(ha), eb = ib + dec_frac_words(hb);
  const int top = ia > ib ? ia : ib, fr = (ea - ia > eb - ib) ? ea - ia : eb - ib;
  int r = 0;
  for (int k = -top; k < fr && r == 0; k++) {   // k < 0: integer word 10^(9 * (-k - 1)); k >= 0: fraction word k
    const int ja = ia + k, jb = ib + k;
    const uint32_t wa = (ja >= 0 && ja < ea) ? wa_at(ja) : 0u, wb = (jb >= 0 && jb < eb) ? wb_at(jb) : 0u;
    r = wa < wb ? -1 : (wa > wb ? 1 : 0);
  }
  return na ? -r : r;
}

__host__ __device__ inline int dec_cell_cmp(const uint32_t* a, const uint32_t* b) {
  return dec_cmp_words(a[0], DecWordsPtr{a}, b[0], DecWordsPtr{b});
}

// The comparison form of a well-formed cell (host; the constant of a DECIMAL compare or filter item): the same sign (a
// negative zero stays negative) and value, without its leading zero integer words and trailing zero fraction words, so
// digitsInt / digitsFrac = 9 * the integer / fraction words kept; resultFrac and the unused words are 0.  dec_cell_cmp
// orders it against every cell as it orders the input cell, and a row's comparison with it walks no word pair that
// only the constant's zero words would add.
inline void dec_normalize(const uint32_t (&c)[10], uint32_t (&o)[10]) {
  const int wi = dec_int_words(c[0]), n = wi + dec_frac_words(c[0]);
  int lo = 0, hi = n;
  while (lo < wi && c[1 + lo] == 0) lo++;
  while (hi > wi && c[hi] == 0) hi--;   // c[hi] is word hi - 1
  for (int j = 0; j < 10; j++) o[j] = 0;
  o[0] = (uint32_t)(9 * (wi - lo)) | ((uint32_t)(9 * (hi - wi)) << 8) | (dec_negative(c[0]) ? 1u << 24 : 0u);
  for (int j = lo; j < hi; j++) o[1 + j - lo] = c[1 + j];
}

// A monotone 64-bit key of a well-formed cell: a < b implies key(a) <= key(b), equal values give equal keys, and values
// that differ within their first 16 significant digits give different keys.  Bit 63 is 1 for a cell without the negative
// flag; below it the magnitude M = 0 for a zero, else (e + 82) << 54 | m, where e in [-81, 80] is the decimal exponent of
// the leading digit and m in [10^15, 10^16) the first 16 significant digits; a negative cell takes ~M (63 bits).  Every
// index into c is a constant, so c stays in registers.
__host__ __device__ __forceinline__ unsigned long long dec_order_key(const uint32_t (&c)[10]) {
  const int wi = dec_int_words(c[0]), n = wi + dec_frac_words(c[0]);
  uint32_t w = 0, w1 = 0, w2 = 0;   // the first nonzero word and the two after it
  int j0 = -1;
#pragma unroll
  for (int j = 0; j < 9; j++) {
    const uint32_t v = j < n ? c[1 + j] : 0u;
    if (j0 < 0) { if (v) { j0 = j; w = v; } }
    else if (j == j0 + 1) w1 = v;
    else if (j == j0 + 2) w2 = v;
  }
  unsigned long long mag = 0;
  if (j0 >= 0) {
    int d = 1;          // digits of w
    uint32_t p = 10;    // 10^d
#pragma unroll
    for (int k = 1; k < 9; k++) if (w >= p) { d++; p *= 10u; }
    const int e = 9 * (wi - 1 - j0) + d - 1;
    // the first 18 significant digits: w (d digits), w1 (9), then the first 9 - d digits of w2; p = 10^d here
    const unsigned long long z = ((unsigned long long)w * TG_DEC_WORD_BASE + w1) * (TG_DEC_WORD_BASE / p) + w2 / p;
    mag = ((unsigned long long)(e + 82) << 54) | (z / 100ull);
  }
  return dec_negative(c[0]) ? (~mag & 0x7FFFFFFFFFFFFFFFull) : (mag | 0x8000000000000000ull);
}

}  // namespace tg
