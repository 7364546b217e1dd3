// agg.cu — tg_agg_*: GPU hash aggregation behind HashAggExec's Open/Next/Close contract
// (pkg/executor/aggregate/agg_hash_executor.go:93, :237, :441, :164).
//
// What the kernels replace:
//   GetGroupKey + getPartialResultsOfEachRow + per-row af.UpdatePartialResult
//     (agg_util.go:106, agg_hash_partial_worker.go:219, :256)         → k_agg_update / k_agg_update_nogroup
//   HashAggFinalWorker merge + AppendFinalResult2Chunk (agg_hash_final_worker.go:73, :121;
//     func_sum.go:80, func_avg.go:332, func_count.go:43)              → k_agg_finalize
// There is no partial/final split on one GPU: every row updates the single device-resident group table
// with atomics.  The 1M-group table of config 3 is 48 MB, which does NOT stay resident in the 50 MB L2 of an H100: the
// step takes about twice as long as with a 24 MB table (DESIGN.md §4.2).
//
// Layout: structure-of-arrays open-addressing table — keys[S+2] (int64, sentinel = empty), rows[S+2]
// (group row count), and one or two 8-byte state arrays per aggregate.  Slot S holds the NULL group
// (NULL group keys DO form a group: codec.go:1766), slot S+1 the group whose key equals the sentinel.
#include <memory>
#include <algorithm>
#include <cmath>
#include "common.cuh"
#include "tma.cuh"
#include "decimal.cuh"
#include "chunk_io.cuh"
#include "string.cuh"
#include "str_dict.cuh"

namespace tg {

#define TG_MAX_AGG 12
enum { GK_I64 = 0, GK_F64 = 1, GK_NONE = 2 };

struct AggFuncDev {
  int32_t name;         // TG_AGG_*
  int32_t arg_col;      // -1: COUNT(*)
  int32_t is_real;
  int32_t is_unsigned;
  int32_t s0, s1;       // state array indices (-1 = unused): s0 value (sum / min / max / count), s1 non-NULL count
  int32_t final_mode;   // TG_AGGMODE_FINAL: inputs are partial results
  int32_t arg_col2;
  int32_t arg_expr;     // TG_ARGEXPR_*
  int32_t s2;           // >= 0: DECIMAL SUM / AVG, an exact 128-bit sum of the integer (or scaled DECIMAL) argument: s0 its low word, s2 its high word
  int32_t dec_frac;     // DECIMAL AVG: result scale (AggFuncDesc.RetTp decimal)
  int32_t dec_scale;    // >= 0: the result is a DECIMAL cell and the argument's values are integers * 10^-dec_scale (0 for an
                        // integer column, s_a + s_b for a product); -1: an 8-byte result
  int32_t s3;           // >= 0: DECIMAL SUM / AVG of a product of two DECIMAL columns (arg_expr), an exact 192-bit sum: s0, s2, s3
                        // its low, middle and top words
  double arg_const;
  long long dec_c;      // DECIMAL MUL_CSUB: the integer constant c * 10^(s_b), |dec_c| <= 10^18
};
struct AggSpec { int32_t n; int32_t pad; unsigned long long* err; AggFuncDev f[TG_MAX_AGG]; };

// argument of SUM / AVG as a double: a plain column or the fused scalar expression; false = NULL.  A non-finite
// intermediate on a non-NULL row raises *spec.err (types.ErrOverflow: builtin_arithmetic_vec.go:51-58, :312-318)
__device__ __forceinline__ bool agg_arg_real(const AggSpec& spec, const AggFuncDev& f, const DevCols& cols, int64_t row, double& v) {
  const uint8_t* nb = cols.nulls[f.arg_col];
  if (nb && !bit_not_null(nb, row)) return false;
  const double a = __longlong_as_double((long long)__ldcs(reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col]) + row));
  if (f.arg_expr == TG_ARGEXPR_COL) { v = a; return true; }
  const uint8_t* nb2 = cols.nulls[f.arg_col2];
  if (nb2 && !bit_not_null(nb2, row)) return false;
  const double b = __longlong_as_double((long long)__ldcs(reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col2]) + row));
  const double t = f.arg_expr == TG_ARGEXPR_MUL_CSUB ? __dsub_rn(f.arg_const, b) : b;
  const double r = __dmul_rn(a, t);     // separate roundings, like the two builtins (no fused multiply-add)
  if (!isfinite(t) || !isfinite(r)) atomicExch(spec.err, 1ull);
  v = r;
  return true;
}
#define TG_MAX_GROUP_COLS 4
struct AggTable {
  long long* keys;                       // single GROUP BY column: the key itself (kEmptyKey = unoccupied)
  unsigned long long* rows;
  unsigned long long* state[2 * TG_MAX_AGG];
  unsigned long long nslots;
  // several GROUP BY columns (GetGroupKey concatenates their encodings, agg_util.go:106 / codec.go:1761): a slot is claimed
  // through its 64-bit TAG word (0 empty, hash|1 being written, hash|3 published) and holds nkw key words — one per
  // column (NULL stored as 0) plus, when a column is nullable, a word with the columns' NULL bits
  unsigned long long* tags;
  long long* keyw[TG_MAX_GROUP_COLS + 1];
  int32_t nkw;
  // element stride of every array above, in 8-byte words: 1 = structure of arrays (single-key tables: a row's atomics go to
  // different sectors, and same-sector atomics would serialise); multi-key tables are ARRAY OF RECORDS
  // [tag | key words | rows | states], padded to 32 bytes: their groups are mostly cold (Q3: 2.4 rows per group, a 1.4 GB
  // table), and a row should touch one or two DRAM sectors instead of one per array
  uint32_t stride;
};
struct GroupKey { const void* data; const uint8_t* nulls; int32_t kind; int32_t pad; };
struct GroupKeys { int32_t n, nkw; const void* data[TG_MAX_GROUP_COLS]; const uint8_t* nulls[TG_MAX_GROUP_COLS]; int32_t kind[TG_MAX_GROUP_COLS]; };

// order-preserving map double → u64 so that MIN/MAX(double) can use integer atomics
__device__ __forceinline__ unsigned long long f64_to_ordered(double d) {
  unsigned long long u = (unsigned long long)__double_as_longlong(d);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double ordered_to_f64(unsigned long long u) {
  u = (u >> 63) ? (u & 0x7fffffffffffffffull) : ~u;
  return __longlong_as_double((long long)u);
}
__device__ __forceinline__ unsigned long long i64_to_ordered(long long v) { return (unsigned long long)v ^ 0x8000000000000000ull; }

// DECIMAL SUM / AVG: adds the 128-bit value (ext:v) to the 128-bit sum (*hi:*lo).  The atomic that wraps the low word sees
// its own carry, so the sum is exact in any order of the additions.  ext is v's high word: all ones for a negative signed
// argument, 0 for a non-negative or unsigned one, so non-negative data pays the second atomic only on a carry.  The sum
// cannot overflow: fewer than 2^63 rows of magnitude at most 2^64 stay below 2^127.
__device__ __forceinline__ void dec_add(unsigned long long* lo, unsigned long long* hi, unsigned long long v, unsigned long long ext) {
  const unsigned long long old = atomicAdd(lo, v);
  const unsigned long long add = ext + (old + v < old ? 1ull : 0ull);
  if (add) atomicAdd(hi, add);
}
// DECIMAL SUM / AVG of a product: adds the 192-bit value (v2:v1:v0) to the 192-bit sum (*w2:*w1:*w0) with dec_add's carry
// rule, one word after the other: the middle word only when v1 plus the low word's carry is not 0, the top word only on a
// middle carry or a negative value.  A non-negative product below 2^64 costs one atomic, like an integer row.  Products
// are below 2 * 10^36 < 2^121 in magnitude, so fewer than 2^63 rows keep |sum| < 2^184: exact in any order of the additions.
__device__ __forceinline__ void dec3_add(unsigned long long* w0, unsigned long long* w1, unsigned long long* w2, unsigned long long v0,
                                         unsigned long long v1, unsigned long long v2) {
  const unsigned long long old0 = atomicAdd(w0, v0);
  const unsigned long long x1 = v1 + (old0 + v0 < old0 ? 1ull : 0ull);
  unsigned long long x2 = v2 + (x1 < v1 ? 1ull : 0ull);   // v1 = 2^64 - 1 plus a carry wraps to 0
  if (x1) { const unsigned long long old1 = atomicAdd(w1, x1); x2 += old1 + x1 < old1 ? 1ull : 0ull; }
  if (x2) atomicAdd(w2, x2);
}
// the exact signed product a * t as (top:mid:lo): one 64x64 multiply for the low word, its signed high half, the sign
__device__ __forceinline__ void dec_mul(long long a, long long t, unsigned long long& lo, unsigned long long& mid, unsigned long long& top) {
  lo = (unsigned long long)a * (unsigned long long)t;
  mid = (unsigned long long)__mul64hi(a, t);
  top = (unsigned long long)((long long)mid >> 63);
}
// one row of a DECIMAL SUM / AVG of a product: the 192-bit add of a * t and the non-NULL count (nullptr: NOT NULL operands).
// The three words are the consecutive states s0, s2 = s0 + 1, s3 = s0 + 2, so they sit at w0, w0 + step, w0 + 2 * step in
// every table layout.  Out of line, like dec_apply, and with few arguments: a kernel's register count includes its callees'.
__device__ __noinline__ void dec3_apply(unsigned long long* w0, int64_t step, unsigned long long* cnt, long long a, long long t) {
  unsigned long long lo, mid, top;
  dec_mul(a, t, lo, mid, top);
  dec3_add(w0, w0 + step, w0 + 2 * step, lo, mid, top);
  if (cnt) atomicAdd(cnt, 1ull);
}
// the operands of a DECIMAL product row (k_dec_to_scaled has turned both columns into int64 value * 10^scale): a, and
// t = b (MUL) or c * 10^(s_b) - b (MUL_CSUB, |t| < 2 * 10^18); false when b is NULL (the caller has checked a)
__device__ __forceinline__ bool dec_expr_operands(const AggFuncDev& f, const DevCols& cols, int64_t row, long long& a, long long& t) {
  const uint8_t* nb2 = cols.nulls[f.arg_col2];
  if (nb2 && !bit_not_null(nb2, row)) return false;
  a = __ldcs(reinterpret_cast<const long long*>(cols.data[f.arg_col]) + row);
  const long long b = __ldcs(reinterpret_cast<const long long*>(cols.data[f.arg_col2]) + row);
  t = f.arg_expr == TG_ARGEXPR_MUL_CSUB ? f.dec_c - b : b;
  return true;
}
// high word of an integer argument as a 128-bit value
__device__ __forceinline__ unsigned long long dec_ext(const AggFuncDev& f, unsigned long long v) {
  return f.is_unsigned ? 0ull : (unsigned long long)((long long)v >> 63);
}

// home slot of a single-column group key in the global table.  Every kernel that places or looks up such a key uses it —
// the update kernels (k_agg_update, k_agg_update2), the merge of partial results and the rehash into a grown table: a key
// that a rehash or a merge placed by another function is not found by the next lookup, which inserts a second copy of
// its group
__device__ __forceinline__ uint32_t agg_home(long long k, unsigned long long nslots) { return slot32(hash64((unsigned long long)k), (uint32_t)nslots); }

// probe-length limit of every find-or-insert into the group table, a DISTINCT set or a string dictionary: an item whose
// probe sequence is longer is deferred, and the host grows the table, or re-runs the item without the limit when the
// table is far from full (grow_and_retry)
constexpr uint32_t kAggMaxProbe = 48;

// find-or-insert `k` in the global table starting at slot s with the slot's current content `cur` already loaded;
// returns false when the probe sequence exceeds max_probe (table overfull: defer)
__device__ __forceinline__ bool global_find_or_insert(const AggTable& t, long long k, uint32_t& s, long long cur, uint32_t max_probe) {
  const uint32_t S = (uint32_t)t.nslots;
  uint32_t steps = 0;
  for (;;) {
    if (cur == k) return true;
    if (cur == kEmptyKey) {
      unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(&t.keys[s]), (unsigned long long)kEmptyKey, (unsigned long long)k);
      if (old == (unsigned long long)kEmptyKey || old == (unsigned long long)k) return true;
    }
    if (++steps > max_probe) return false;
    if (++s == S) s = 0;
    cur = *reinterpret_cast<volatile long long*>(&t.keys[s]);
  }
}

// fold one partial group (rows + states) into global slot s: MergePartialResult (func_sum.go:106, func_count.go:481,
// func_avg.go:444, func_max_min.go merge)
template <bool WIDE>
__device__ __forceinline__ void agg_merge_into(const AggTable& t, const AggSpec& spec, unsigned long long s, unsigned long long rows, const unsigned long long* st) {
  atomicAdd(&t.rows[s], rows);
  for (int k = 0; k < spec.n; k++) {
    const AggFuncDev& f = spec.f[k];
    if (f.s0 >= 0) {
      unsigned long long v = st[f.s0];
      switch (f.name) {
        case TG_AGG_COUNT: atomicAdd(&t.state[f.s0][s], v); break;
        case TG_AGG_SUM: case TG_AGG_AVG:
          if (WIDE && f.s3 >= 0) dec3_add(&t.state[f.s0][s], &t.state[f.s2][s], &t.state[f.s3][s], v, st[f.s2], st[f.s3]);
          else if (f.s2 >= 0) dec_add(&t.state[f.s0][s], &t.state[f.s2][s], v, st[f.s2]);
          else atomicAdd(reinterpret_cast<double*>(&t.state[f.s0][s]), __longlong_as_double((long long)v));
          break;
        case TG_AGG_MIN: atomicMin(&t.state[f.s0][s], v); break;
        case TG_AGG_MAX: atomicMax(&t.state[f.s0][s], v); break;
        default: break;
      }
    }
    if (f.s1 >= 0) atomicAdd(&t.state[f.s1][s], st[f.s1]);
  }
}

__global__ void k_agg_init(AggTable t, AggSpec spec, unsigned long long n_total) {
  unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (; i < n_total; i += stride) {
    if (t.nkw) { t.tags[(size_t)i * t.stride] = 0; for (int j = 0; j < t.nkw; j++) t.keyw[j][(size_t)i * t.stride] = 0; }
    else t.keys[i] = kEmptyKey;
    t.rows[(size_t)i * t.stride] = 0;
    for (int k = 0; k < spec.n; k++) {
      const AggFuncDev& f = spec.f[k];
      if (f.s0 >= 0) {
        unsigned long long init = 0;
        if (f.name == TG_AGG_MIN) init = ~0ull;          // ordered domain: larger than everything
        t.state[f.s0][(size_t)i * t.stride] = init;
      }
      if (f.s1 >= 0) t.state[f.s1][(size_t)i * t.stride] = 0;
      if (f.s2 >= 0) t.state[f.s2][(size_t)i * t.stride] = 0;
      if (f.s3 >= 0) t.state[f.s3][(size_t)i * t.stride] = 0;
    }
  }
}

// WIDE: the plan has a DECIMAL SUM / AVG of a product (AggFuncDev::s3).  Only the WIDE instantiations of the update, merge
// and finalize kernels carry the 192-bit code: a kernel's register count includes its out-of-line callees', and every other
// plan keeps the kernels it had.
template <bool WIDE>
__device__ __forceinline__ void agg_apply(const AggTable& t, const AggSpec& spec, const DevCols& cols, int64_t row,
                                          unsigned long long s) {
  atomicAdd(&t.rows[(size_t)s * t.stride], 1ull);
  for (int k = 0; k < spec.n; k++) {
    const AggFuncDev& f = spec.f[k];
    if (f.arg_col < 0 || f.s0 < 0) continue;   // COUNT(*) and NOT NULL COUNT(x) read rows[]; FIRSTROW reads the key
    const uint8_t* nb = cols.nulls[f.arg_col];
    if (nb && !bit_not_null(nb, row)) continue;
    if (WIDE && f.s3 >= 0) {   // DECIMAL SUM / AVG of a product
      long long x, y;
      if (dec_expr_operands(f, cols, row, x, y))
        dec3_apply(&t.state[f.s0][(size_t)s * t.stride], t.state[f.s2] - t.state[f.s0], f.s1 >= 0 ? &t.state[f.s1][(size_t)s * t.stride] : nullptr, x, y);
      continue;
    }
    switch (f.name) {
      case TG_AGG_COUNT:
        if (f.final_mode) atomicAdd(&t.state[f.s0][(size_t)s * t.stride], reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col])[row]);
        else atomicAdd(&t.state[f.s0][(size_t)s * t.stride], 1ull);
        break;
      case TG_AGG_SUM: {
        if (f.s2 >= 0) {   // DECIMAL: exact 128-bit sum of the integer argument
          const unsigned long long v = reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col])[row];
          dec_add(&t.state[f.s0][(size_t)s * t.stride], &t.state[f.s2][(size_t)s * t.stride], v, dec_ext(f, v));
          if (f.s1 >= 0) atomicAdd(&t.state[f.s1][(size_t)s * t.stride], 1ull);
          break;
        }
        double v;
        if (!agg_arg_real(spec, f, cols, row, v)) break;
        atomicAdd(reinterpret_cast<double*>(&t.state[f.s0][(size_t)s * t.stride]), v);
        if (f.s1 >= 0) atomicAdd(&t.state[f.s1][(size_t)s * t.stride], 1ull);
        break;
      }
      case TG_AGG_AVG:
        if (f.s2 >= 0) {
          const unsigned long long v = reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col])[row];
          dec_add(&t.state[f.s0][(size_t)s * t.stride], &t.state[f.s2][(size_t)s * t.stride], v, dec_ext(f, v));
          if (f.s1 >= 0) atomicAdd(&t.state[f.s1][(size_t)s * t.stride], 1ull);
        } else if (f.final_mode) {   // args: count column, sum column (func_avg.go:405)
          const uint8_t* nb2 = cols.nulls[f.arg_col2];
          if (nb2 && !bit_not_null(nb2, row)) break;
          atomicAdd(reinterpret_cast<double*>(&t.state[f.s0][(size_t)s * t.stride]), reinterpret_cast<const double*>(cols.data[f.arg_col2])[row]);
          atomicAdd(&t.state[f.s1][(size_t)s * t.stride], reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col])[row]);
        } else {
          double v;
          if (!agg_arg_real(spec, f, cols, row, v)) break;
          atomicAdd(reinterpret_cast<double*>(&t.state[f.s0][(size_t)s * t.stride]), v);
          if (f.s1 >= 0) atomicAdd(&t.state[f.s1][(size_t)s * t.stride], 1ull);
        }
        break;
      case TG_AGG_MIN: case TG_AGG_MAX: {
        unsigned long long v;
        if (f.is_real) v = f64_to_ordered(reinterpret_cast<const double*>(cols.data[f.arg_col])[row]);
        else if (f.is_unsigned) v = reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col])[row];
        else v = i64_to_ordered(reinterpret_cast<const long long*>(cols.data[f.arg_col])[row]);
        if (f.name == TG_AGG_MIN) atomicMin(&t.state[f.s0][(size_t)s * t.stride], v); else atomicMax(&t.state[f.s0][(size_t)s * t.stride], v);
        if (f.s1 >= 0) atomicAdd(&t.state[f.s1][(size_t)s * t.stride], 1ull);
        break;
      }
      default: break;
    }
  }
}

// One thread per row: find-or-insert the group slot, then atomics.  Rows whose NEW key finds no slot within
// max_probe steps are deferred (bit set in `deferred`) so the host can grow the table and re-run
// them; `only` restricts a re-run to those rows.
template <bool WIDE>
__global__ void __launch_bounds__(256)
k_agg_update(GroupKey gk, DevCols cols, int64_t n, AggTable t, AggSpec spec, uint32_t max_probe,
             uint32_t* deferred, const uint32_t* only, unsigned long long* n_deferred) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    if (only && !((only[i >> 5] >> (i & 31)) & 1u)) continue;
    unsigned long long s;
    bool is_null = gk.nulls && !bit_not_null(gk.nulls, i);
    if (is_null) s = t.nslots;
    else {
      long long k;
      if (gk.kind == GK_I64) k = reinterpret_cast<const long long*>(gk.data)[i];
      else {
        double d = reinterpret_cast<const double*>(gk.data)[i];
        if (d == 0) d = 0;   // -0 and +0 encode to the same group key (codec float.go:23)
        k = __double_as_longlong(d);
      }
      if (k == kEmptyKey) s = t.nslots + 1;
      else {
        // No global fill counter: one atomic per NEW key on a single address serialised at ~3 ns each (1 M groups =
        // 3 ms, twice the rest of the kernel).  A probe sequence longer than `max_probe` steps means the table is
        // overfull: the row is deferred and the host grows the table.
        uint32_t sl = agg_home(k, t.nslots);
        if (!global_find_or_insert(t, k, sl, *reinterpret_cast<volatile long long*>(&t.keys[sl]), max_probe)) {
          atomicOr(&deferred[i >> 5], 1u << (i & 31));
          atomicAdd(n_deferred, 1ull);
          continue;
        }
        s = sl;
      }
    }
    agg_apply<WIDE>(t, spec, cols, i, s);
  }
}

// no GROUP BY, DECIMAL SUM / AVG of a product: a 192-bit sum per thread, a warp reduction, one dec3_add per warp (out of
// line: the 192-bit accumulator stays out of k_agg_update_nogroup's other paths)
__device__ __forceinline__ void add192(unsigned long long& s0, unsigned long long& s1, unsigned long long& s2, unsigned long long v0,
                                       unsigned long long v1, unsigned long long v2) {
  asm("add.cc.u64 %0, %0, %3;\n\taddc.cc.u64 %1, %1, %4;\n\taddc.u64 %2, %2, %5;" : "+l"(s0), "+l"(s1), "+l"(s2) : "l"(v0), "l"(v1), "l"(v2));
}
__device__ __noinline__ void dec3_nogroup(const long long* a, const uint8_t* na, const long long* b, const uint8_t* nb, bool csub, long long c,
                                          int64_t i0, int64_t n, int64_t stride, unsigned long long* w0, unsigned long long* w1,
                                          unsigned long long* w2, unsigned long long* cnt_out) {
  unsigned long long s0 = 0, s1 = 0, s2 = 0, cnt = 0;
  for (int64_t i = i0; i < n; i += stride) {
    if ((na && !bit_not_null(na, i)) || (nb && !bit_not_null(nb, i))) continue;
    unsigned long long lo, mid, top;
    dec_mul(a[i], csub ? c - b[i] : b[i], lo, mid, top);
    add192(s0, s1, s2, lo, mid, top);
    cnt++;
  }
  for (int o = 16; o; o >>= 1) {
    const unsigned long long t0 = __shfl_xor_sync(0xffffffffu, s0, o), t1 = __shfl_xor_sync(0xffffffffu, s1, o), t2 = __shfl_xor_sync(0xffffffffu, s2, o);
    add192(s0, s1, s2, t0, t1, t2);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0 && cnt) {
    dec3_add(w0, w1, w2, s0, s1, s2);
    if (cnt_out) atomicAdd(cnt_out, cnt);
  }
}

// no GROUP BY: one group.  Warp-shuffle partial reduction, then one atomic per warp and aggregate.
template <bool WIDE>
__global__ void __launch_bounds__(256)
k_agg_update_nogroup(DevCols cols, int64_t n, AggTable t, AggSpec spec) {
  int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  unsigned long long my_rows = 0;
  for (int64_t i = i0; i < n; i += stride) my_rows++;
  for (int o = 16; o; o >>= 1) my_rows += __shfl_xor_sync(0xffffffffu, my_rows, o);
  if (lane == 0 && my_rows) atomicAdd(&t.rows[t.nslots], my_rows);
  for (int k = 0; k < spec.n; k++) {
    const AggFuncDev& f = spec.f[k];
    if (f.arg_col < 0 || f.s0 < 0) continue;
    const uint8_t* nb = cols.nulls[f.arg_col];
    if (WIDE && f.s3 >= 0) {
      dec3_nogroup(reinterpret_cast<const long long*>(cols.data[f.arg_col]), nb, reinterpret_cast<const long long*>(cols.data[f.arg_col2]),
                   cols.nulls[f.arg_col2], f.arg_expr == TG_ARGEXPR_MUL_CSUB, f.dec_c, i0, n, stride, &t.state[f.s0][t.nslots],
                   &t.state[f.s2][t.nslots], &t.state[f.s3][t.nslots], f.s1 >= 0 ? &t.state[f.s1][t.nslots] : nullptr);
      continue;
    }
    double fs = 0; unsigned long long cnt = 0, ext = f.name == TG_AGG_MIN ? ~0ull : 0ull, isum = 0;
    __int128 dsum = 0;   // DECIMAL SUM / AVG: exact
    for (int64_t i = i0; i < n; i += stride) {
      if (nb && !bit_not_null(nb, i)) continue;
      if (f.s2 >= 0) {
        const unsigned long long v = reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col])[i];
        dsum += f.is_unsigned ? (__int128)v : (__int128)(long long)v;
        cnt++;
        continue;
      }
      if (f.name == TG_AGG_AVG && f.final_mode) {
        const uint8_t* nb2 = cols.nulls[f.arg_col2];
        if (nb2 && !bit_not_null(nb2, i)) continue;
        fs += reinterpret_cast<const double*>(cols.data[f.arg_col2])[i];
        cnt += reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col])[i];
        continue;
      }
      if ((f.name == TG_AGG_SUM || f.name == TG_AGG_AVG) && f.arg_expr) {
        double v;
        if (!agg_arg_real(spec, f, cols, i, v)) continue;
        cnt++; fs += v;
        continue;
      }
      cnt++;
      if (f.name == TG_AGG_SUM || f.name == TG_AGG_AVG) fs += reinterpret_cast<const double*>(cols.data[f.arg_col])[i];
      else if (f.name == TG_AGG_COUNT) { if (f.final_mode) isum += reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col])[i]; else isum++; }
      else {
        unsigned long long v;
        if (f.is_real) v = f64_to_ordered(reinterpret_cast<const double*>(cols.data[f.arg_col])[i]);
        else if (f.is_unsigned) v = reinterpret_cast<const unsigned long long*>(cols.data[f.arg_col])[i];
        else v = i64_to_ordered(reinterpret_cast<const long long*>(cols.data[f.arg_col])[i]);
        ext = f.name == TG_AGG_MIN ? (v < ext ? v : ext) : (v > ext ? v : ext);
      }
    }
    if (f.s2 >= 0) {
      for (int o = 16; o; o >>= 1) {
        const unsigned long long lo = __shfl_xor_sync(0xffffffffu, (unsigned long long)dsum, o);
        const unsigned long long hi = __shfl_xor_sync(0xffffffffu, (unsigned long long)((unsigned __int128)dsum >> 64), o);
        dsum += (__int128)(((unsigned __int128)hi << 64) | lo);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      }
      if (lane == 0 && cnt) {
        dec_add(&t.state[f.s0][t.nslots], &t.state[f.s2][t.nslots], (unsigned long long)dsum, (unsigned long long)((unsigned __int128)dsum >> 64));
        if (f.s1 >= 0) atomicAdd(&t.state[f.s1][t.nslots], cnt);
      }
      continue;
    }
    for (int o = 16; o; o >>= 1) {
      fs += __shfl_xor_sync(0xffffffffu, fs, o);
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      isum += __shfl_xor_sync(0xffffffffu, isum, o);
      unsigned long long e2 = __shfl_xor_sync(0xffffffffu, ext, o);
      ext = f.name == TG_AGG_MIN ? (e2 < ext ? e2 : ext) : (e2 > ext ? e2 : ext);
    }
    if (lane == 0 && cnt) {
      unsigned long long s = t.nslots;
      if (f.name == TG_AGG_SUM || f.name == TG_AGG_AVG) atomicAdd(reinterpret_cast<double*>(&t.state[f.s0][s]), fs);
      else if (f.name == TG_AGG_COUNT) atomicAdd(&t.state[f.s0][s], isum);
      else if (f.name == TG_AGG_MIN) atomicMin(&t.state[f.s0][s], ext);
      else atomicMax(&t.state[f.s0][s], ext);
      if (f.s1 >= 0 && !(f.name == TG_AGG_COUNT)) atomicAdd(&t.state[f.s1][s], cnt);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Two-phase path for low-cardinality GROUP BY (the reference's own benchmark uses NDV 1000, benchmark_test.go:224): the
// same partial → final split as HashAggPartialWorker / HashAggFinalWorker (agg_hash_partial_worker.go:256,
// agg_hash_final_worker.go:73), with a CTA playing the partial worker.  Each CTA aggregates its rows into a
// shared-memory table (2048-4096 slots + the NULL and sentinel groups); rows whose new key does not fit are
// deferred to the global kernel.  At the end the CTA emits its partial results, and k_agg_merge folds them into the
// global table (MergePartialResult semantics) with the usual grow-and-retry protocol.
// ---------------------------------------------------------------------------------------------------------------
#define AGG_LOCAL_SLOTS_MAX 4096   // per-CTA table: 4096 slots with <= 1 state array, 2048 otherwise (about 96 KB, 2 CTAs per SM)
#define AGG_LOCAL_MAX_STATES 4
struct AggPartials {   // columnar partial results, capacity = gridDim.x * (local_slots / 2 + 2)
  long long* keys;
  unsigned char* kind;                 // 0 regular key, 1 NULL group, 2 sentinel-valued key
  unsigned long long* rows;
  unsigned long long* state[AGG_LOCAL_MAX_STATES];
  unsigned long long* count;           // number of tuples emitted
};

template <bool WIDE>
__global__ void __launch_bounds__(256)
k_agg_update_local(GroupKey gk, DevCols cols, int64_t row_lo, int64_t row_hi, AggSpec spec, int nstates, int local_slots,
                   AggPartials out, uint32_t* deferred, unsigned long long* n_deferred) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int LS = local_slots, NT = local_slots + 2;
  const unsigned int max_local_fill = (unsigned int)(local_slots / 2);
  AggTable lt;
  lt.stride = 1; lt.nkw = 0; lt.tags = nullptr;
  lt.nslots = (unsigned long long)LS;
  lt.keys = reinterpret_cast<long long*>(smem_raw);
  lt.rows = reinterpret_cast<unsigned long long*>(smem_raw) + NT;
  for (int s = 0; s < nstates; s++) lt.state[s] = reinterpret_cast<unsigned long long*>(smem_raw) + (size_t)NT * (2 + s);
  __shared__ unsigned int s_fill;
  for (int i = threadIdx.x; i < NT; i += blockDim.x) {
    lt.keys[i] = kEmptyKey; lt.rows[i] = 0;
    for (int k = 0; k < spec.n; k++) {
      const AggFuncDev& f = spec.f[k];
      if (f.s0 >= 0) lt.state[f.s0][i] = f.name == TG_AGG_MIN ? ~0ull : 0ull;
      if (f.s1 >= 0) lt.state[f.s1][i] = 0;
      if (f.s2 >= 0) lt.state[f.s2][i] = 0;
      if (f.s3 >= 0) lt.state[f.s3][i] = 0;
    }
  }
  if (threadIdx.x == 0) s_fill = 0;
  __syncthreads();
  unsigned long long my_deferred = 0;
  for (int64_t i = row_lo + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < row_hi; i += (int64_t)gridDim.x * blockDim.x) {
    unsigned long long s;
    bool is_null = gk.nulls && !bit_not_null(gk.nulls, i);
    bool defer = false;
    if (is_null) s = LS;
    else {
      long long k;
      if (gk.kind == GK_I64) k = reinterpret_cast<const long long*>(gk.data)[i];
      else { double d = reinterpret_cast<const double*>(gk.data)[i]; if (d == 0) d = 0; k = __double_as_longlong(d); }
      if (k == kEmptyKey) s = LS + 1;
      else {
        s = slot32(mix64((uint64_t)k), (uint32_t)LS);
        for (;;) {
          long long cur = *reinterpret_cast<volatile long long*>(&lt.keys[s]);
          if (cur == k) break;
          if (cur == kEmptyKey) {
            unsigned int f = atomicAdd(&s_fill, 1u);
            if (f >= max_local_fill) { atomicSub(&s_fill, 1u); defer = true; break; }
            unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(&lt.keys[s]), (unsigned long long)kEmptyKey, (unsigned long long)k);
            if (old == (unsigned long long)kEmptyKey) break;
            atomicSub(&s_fill, 1u);
            if (old == (unsigned long long)k) break;
          }
          if (++s == (unsigned long long)LS) s = 0;
        }
      }
    }
    if (defer) { atomicOr(&deferred[i >> 5], 1u << (i & 31)); my_deferred++; continue; }
    agg_apply<WIDE>(lt, spec, cols, i, s);
  }
  for (int o = 16; o; o >>= 1) my_deferred += __shfl_xor_sync(0xffffffffu, my_deferred, o);
  if ((threadIdx.x & 31) == 0 && my_deferred) atomicAdd(n_deferred, my_deferred);
  __syncthreads();
  // emit the partial results of this CTA
  for (int i = threadIdx.x; i < NT; i += blockDim.x) {
    bool occ = i < LS ? lt.keys[i] != kEmptyKey : lt.rows[i] != 0;
    if (!occ) continue;
    unsigned long long o = atomicAdd(out.count, 1ull);
    out.keys[o] = i < LS ? lt.keys[i] : 0;
    out.kind[o] = i < LS ? 0 : (i == LS ? 1 : 2);
    out.rows[o] = lt.rows[i];
    for (int s = 0; s < nstates; s++) out.state[s][o] = lt.state[s][i];
  }
}

// fold partial results into the global table; same deferral protocol as k_agg_update
template <bool WIDE>
__global__ void __launch_bounds__(256)
k_agg_merge(AggPartials in, int64_t m, int nstates, AggTable t, AggSpec spec, uint32_t max_probe,
            uint32_t* deferred, const uint32_t* only, unsigned long long* n_deferred) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < m; i += stride) {
    if (only && !((only[i >> 5] >> (i & 31)) & 1u)) continue;
    unsigned long long s;
    if (in.kind[i] == 1) s = t.nslots;
    else if (in.kind[i] == 2) s = t.nslots + 1;
    else {
      const long long k = in.keys[i];
      uint32_t sl = agg_home(k, t.nslots);
      if (!global_find_or_insert(t, k, sl, *reinterpret_cast<volatile long long*>(&t.keys[sl]), max_probe)) {
        atomicOr(&deferred[i >> 5], 1u << (i & 31));
        atomicAdd(n_deferred, 1ull);
        continue;
      }
      s = sl;
    }
    unsigned long long st[AGG_LOCAL_MAX_STATES];
    for (int a = 0; a < nstates; a++) st[a] = in.state[a][i];
    agg_merge_into<WIDE>(t, spec, s, in.rows[i], st);
  }
}

// re-insert every group of an old table into a bigger one (no atomics on the states: keys are unique)
__global__ void k_agg_rehash(AggTable oldt, AggTable newt, int nstates) {
  unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (; i < oldt.nslots + 2; i += stride) {
    unsigned long long s;
    if (i >= oldt.nslots) { if (oldt.rows[i] == 0) continue; s = newt.nslots + (i - oldt.nslots); }
    else {
      long long k = oldt.keys[i];
      if (k == kEmptyKey) continue;
      s = agg_home(k, newt.nslots);
      for (;;) {
        unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(&newt.keys[s]), (unsigned long long)kEmptyKey, (unsigned long long)k);
        if (old == (unsigned long long)kEmptyKey) break;
        if (++s == newt.nslots) s = 0;
      }
    }
    newt.rows[s] = oldt.rows[i];
    for (int a = 0; a < nstates; a++) newt.state[a][s] = oldt.state[a][i];
  }
}

// number of occupied slots (distinct groups), for sizing the result columns
__global__ void k_agg_count(AggTable t, unsigned long long* count) {
  unsigned long long n_total = t.nslots + 2;
  unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  unsigned long long c = 0;
  for (; i < n_total; i += stride) c += i < t.nslots ? (t.nkw ? t.tags[(size_t)i * t.stride] != 0 : t.keys[i] != kEmptyKey) : (t.rows[(size_t)i * t.stride] != 0);
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}

struct AggOut { void* data[TG_MAX_AGG]; uint8_t* valid[TG_MAX_AGG]; };

// compact the occupied slots into the result columns (Go-map iteration order is unspecified in the
// reference too; here it is slot order within warps, warp order by the atomic cursor)
// DEC: the plan has a DECIMAL result column (the cell writers of decimal.cuh); WIDE: one of them is a SUM / AVG of a
// product (the 192-bit writers, which take more registers)
template <bool DEC, bool WIDE>
__global__ void __launch_bounds__(256)
k_agg_finalize(AggTable t, AggSpec spec, int gk_kind, AggOut out, unsigned long long* cursor) {
  unsigned long long n_total = t.nslots + 2;
  unsigned long long base = blockIdx.x * (unsigned long long)blockDim.x;
  unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  for (; base < n_total; base += stride) {
    unsigned long long i = base + threadIdx.x;
    bool occ = false;
    if (i < t.nslots) occ = t.nkw ? t.tags[(size_t)i * t.stride] != 0 : t.keys[i] != kEmptyKey;
    else if (i < n_total) occ = t.rows[(size_t)i * t.stride] != 0;
    unsigned b = __ballot_sync(0xffffffffu, occ);
    // one cursor atomic per CTA iteration (256 slots), not per warp: a 29 M-slot table (Q3) would otherwise put 0.9 M atomics on
    // one address
    __shared__ uint32_t s_wcnt[8];
    __shared__ unsigned long long s_cbase;
    const int warp = threadIdx.x >> 5;
    if (lane == 0) s_wcnt[warp] = __popc(b);
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t tot = 0;
      for (int w = 0; w < 8; w++) tot += s_wcnt[w];
      s_cbase = tot ? atomicAdd(cursor, (unsigned long long)tot) : 0ull;
    }
    __syncthreads();
    unsigned long long wbase = s_cbase;
    for (int w = 0; w < warp; w++) wbase += s_wcnt[w];
    __syncthreads();   // s_wcnt / s_cbase are rewritten by the next iteration
    if (!occ) continue;
    unsigned long long o = wbase + __popc(b & ((1u << lane) - 1));
    unsigned long long rows = t.rows[(size_t)i * t.stride];
    for (int k = 0; k < spec.n; k++) {
      const AggFuncDev& f = spec.f[k];
      unsigned long long nn = f.s1 >= 0 ? t.state[f.s1][(size_t)i * t.stride] : rows;   // non-NULL inputs seen
      if (DEC && f.dec_scale >= 0) {   // DECIMAL SUM / AVG / MIN / MAX: a 40-byte MyDecimal cell, NULL without a non-NULL input (decimal.cuh)
        uint8_t* cell = reinterpret_cast<uint8_t*>(out.data[k]) + (size_t)o * TG_DEC_CELL_BYTES;
        // SUM / AVG: the 128-bit sum (192-bit over a product); MIN / MAX: the int64 of the ordered domain (i64_to_ordered),
        // sign-extended
        unsigned long long lo = t.state[f.s0][(size_t)i * t.stride], hi;
        if (f.s2 >= 0) hi = t.state[f.s2][(size_t)i * t.stride];
        else { lo ^= 0x8000000000000000ull; hi = (unsigned long long)((long long)lo >> 63); }
        if (nn == 0) dec_store_null(cell);
        else if (WIDE && f.s3 >= 0)
          dec3_result_cell(cell, lo, hi, t.state[f.s3][(size_t)i * t.stride], nn, f.dec_scale | (f.dec_frac << 8) | (f.name == TG_AGG_AVG ? 1 << 16 : 0));
        else dec_result_cell(cell, f.name == TG_AGG_AVG, lo, hi, nn, f.dec_scale, f.dec_frac);
        if (out.valid[k]) out.valid[k][o] = nn != 0 ? 1 : 0;
        continue;
      }
      bool valid = true;
      unsigned long long v = 0;
      switch (f.name) {
        case TG_AGG_COUNT: v = (f.arg_col < 0 || f.s0 < 0) ? rows : t.state[f.s0][(size_t)i * t.stride]; break;
        case TG_AGG_SUM: valid = nn != 0; v = t.state[f.s0][(size_t)i * t.stride]; break;   // NULL when no non-NULL input (func_sum.go:80)
        case TG_AGG_AVG:
          valid = nn != 0;
          if (valid) v = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)t.state[f.s0][(size_t)i * t.stride]) / (double)nn);   // func_avg.go:332
          break;
        case TG_AGG_MIN: case TG_AGG_MAX: {
          valid = nn != 0;
          unsigned long long u = t.state[f.s0][(size_t)i * t.stride];
          if (f.is_real) v = (unsigned long long)__double_as_longlong(ordered_to_f64(u));
          else if (f.is_unsigned) v = u;
          else v = u ^ 0x8000000000000000ull;
          break;
        }
        default:   // FIRSTROW(group column): the group key itself (firstRow4Int func_first_row.go:140)
          if (t.nkw) {   // f.arg_col2 = index of the column among the GROUP BY items | word with the NULL bits << 8 (0 = none)
            const int g = f.arg_col2 & 0xff, nullword = (f.arg_col2 >> 8) & 0xff;
            if (nullword && ((unsigned long long)t.keyw[nullword][(size_t)i * t.stride] >> g) & 1ull) valid = false;
            else v = (unsigned long long)t.keyw[g][(size_t)i * t.stride];
          }
          else if (i == t.nslots) valid = false;                       // NULL group
          else if (i == t.nslots + 1) v = (unsigned long long)kEmptyKey;
          else v = (unsigned long long)t.keys[i];
          (void)gk_kind;
          break;
      }
      reinterpret_cast<unsigned long long*>(out.data[k])[o] = valid ? v : 0ull;
      if (out.valid[k]) out.valid[k][o] = valid ? 1 : 0;
    }
  }
}


// ---- several GROUP BY columns: tag-claimed slots, global table only -------------------------------------------------
// N key words: the group table's keys (the GROUP BY words and the NULL word), or a DISTINCT set's (those plus the value)
template <int N> struct KeyWordsN { long long w[N]; };
typedef KeyWordsN<TG_MAX_GROUP_COLS + 1> KeyWords;
template <class K>
__device__ __forceinline__ unsigned long long hash_words(const K& k, int nkw) {
  unsigned long long h = hash64((unsigned long long)k.w[0]);
  for (int j = 1; j < nkw; j++) h = hash64(h ^ ((unsigned long long)k.w[j] * 0xD6E8FEB86659FD93ull + (unsigned long long)j));
  return h;
}
template <class K>
__device__ __forceinline__ void load_key_words(const GroupKeys& gk, int64_t i, K& k) {
  unsigned long long nullbits = 0;
  for (int j = 0; j < gk.n; j++) {
    long long v = 0;
    if (gk.nulls[j] && !bit_not_null(gk.nulls[j], i)) nullbits |= 1ull << j;
    else {
      v = __ldcs(reinterpret_cast<const long long*>(gk.data[j]) + i);
      if (gk.kind[j] == GK_F64) { double d = __longlong_as_double(v); if (d == 0) d = 0; v = __double_as_longlong(d); }
    }
    k.w[j] = v;
  }
  if (gk.nkw > gk.n) k.w[gk.n] = (long long)nullbits;
}
// find-or-insert; returns the slot or ~0 when the probe sequence is longer than max_probe (overfull: defer).  *inserted (when
// given) is set when this call claimed the slot: of all the threads that look up one new key, exactly one sees it set.  T is
// the group table (AggTable) or a DISTINCT set (DistinctSet): both have tags, keyw, nslots, nkw and stride.
template <class T, class K>
__device__ __forceinline__ unsigned long long mk_find_or_insert(const T& t, const K& k, unsigned long long h, uint32_t max_probe,
                                                                bool* inserted = nullptr) {
  const unsigned long long ready = h | 3ull, busy = (h & ~3ull) | 1ull;
  uint32_t s = slot32(h, (uint32_t)t.nslots), steps = 0;
  for (;;) {
    // tag and the first three key words sit in the record's first 32 bytes (records are 32-byte aligned): two L2-coherent
    // 128-bit loads of that one sector (128 bits is the widest load sm_90 has).  A tag that is not yet `ready`, or key words
    // that do not match, fall through to the ordered loads below.
    unsigned long long cur, k0, k1, k2;
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(cur), "=l"(k0) : "l"(&t.tags[(size_t)s * t.stride]) : "memory");
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2+16];" : "=l"(k1), "=l"(k2) : "l"(&t.tags[(size_t)s * t.stride]) : "memory");
    if (cur == 0) {
      cur = atomicCAS(&t.tags[(size_t)s * t.stride], 0ull, busy);
      if (cur == 0) {
        for (int j = 0; j < t.nkw; j++) t.keyw[j][(size_t)s * t.stride] = k.w[j];
        __threadfence();
        *reinterpret_cast<volatile unsigned long long*>(&t.tags[(size_t)s * t.stride]) = ready;   // publish
        if (inserted) *inserted = true;
        return s;
      }
    }
    if ((cur | 2ull) == ready) {
      bool eq = cur == ready && (unsigned long long)k.w[0] == k0 && (t.nkw < 2 || (unsigned long long)k.w[1] == k1) && (t.nkw < 3 || (unsigned long long)k.w[2] == k2);
      if (eq && t.nkw > 3) eq = *reinterpret_cast<volatile long long*>(&t.keyw[3][(size_t)s * t.stride]) == k.w[3];
      // a DISTINCT set compares its words past the fourth too (up to four group words, the NULL word and the value).  The
      // group table keeps its four-word check here: its fifth word, the NULL word of four GROUP BY columns, is left to
      // the tag as before, which keeps k_agg_update_mk at its register count.
      constexpr int NW = (int)(sizeof(k.w) / sizeof(k.w[0]));
      if (NW > TG_MAX_GROUP_COLS + 1) {
#pragma unroll
        for (int j = 4; j < NW; j++)
          if (eq && t.nkw > j) eq = *reinterpret_cast<volatile long long*>(&t.keyw[j][(size_t)s * t.stride]) == k.w[j];
      }
      if (!eq) {   // still being written, or the vector load raced with the writer, or a different key with the same hash: settle it with ordered loads
        while (cur != ready) cur = *reinterpret_cast<volatile unsigned long long*>(&t.tags[(size_t)s * t.stride]);
        eq = true;
        for (int j = 0; j < t.nkw; j++) eq &= *reinterpret_cast<volatile long long*>(&t.keyw[j][(size_t)s * t.stride]) == k.w[j];
      }
      if (eq) return s;
    }
    if (++steps > max_probe) return ~0ull;
    if (++s == (uint32_t)t.nslots) s = 0;
  }
}

template <bool WIDE>
__global__ void __launch_bounds__(256)
k_agg_update_mk(GroupKeys gk, DevCols cols, int64_t n, AggTable t, AggSpec spec, uint32_t max_probe,
                uint32_t* deferred, const uint32_t* only, unsigned long long* n_deferred) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long my_deferred = 0;
  for (; i < n; i += stride) {
    if (only && !((only[i >> 5] >> (i & 31)) & 1u)) continue;
    KeyWords k;
    load_key_words(gk, i, k);
    const unsigned long long s = mk_find_or_insert(t, k, hash_words(k, t.nkw), max_probe);
    if (s == ~0ull) { atomicOr(&deferred[i >> 5], 1u << (i & 31)); my_deferred++; continue; }
    agg_apply<WIDE>(t, spec, cols, i, s);
  }
  for (int o = 16; o; o >>= 1) my_deferred += __shfl_xor_sync(0xffffffffu, my_deferred, o);
  if ((threadIdx.x & 31) == 0 && my_deferred) atomicAdd(n_deferred, my_deferred);
}

// re-insert every group of an old multi-key table into a bigger one (keys are distinct: claim with the published tag)
__global__ void k_agg_rehash_mk(AggTable oldt, AggTable newt, int nstates) {
  unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (; i < oldt.nslots; i += stride) {
    const unsigned long long tag = oldt.tags[(size_t)i * oldt.stride];
    if (tag == 0) continue;
    uint32_t s = slot32(tag, (uint32_t)newt.nslots);
    for (;;) {
      if (atomicCAS(&newt.tags[(size_t)s * newt.stride], 0ull, tag) == 0ull) break;
      if (++s == (uint32_t)newt.nslots) s = 0;
    }
    for (int j = 0; j < oldt.nkw; j++) newt.keyw[j][(size_t)s * newt.stride] = oldt.keyw[j][(size_t)i * oldt.stride];
    newt.rows[(size_t)s * newt.stride] = oldt.rows[(size_t)i * oldt.stride];
    for (int a = 0; a < nstates; a++) newt.state[a][(size_t)s * newt.stride] = oldt.state[a][(size_t)i * oldt.stride];
  }
}

// ---- DISTINCT arguments: one dedup set per argument column ----------------------------------------------------------
// A set holds the (group key words, value word) pairs seen so far, in HBM, for the life of the handle.  Its records are
// [tag | key words], claimed like the multi-key table's (mk_find_or_insert) and carrying no states; the key words are the
// group table's (load_key_words: NULL group keys as 0 plus the NULL word, a DOUBLE -0 as +0) followed by the value.
#define TG_SET_MAX_WORDS (TG_MAX_GROUP_COLS + 2)
struct DistinctSet {
  unsigned long long* tags;
  long long* keyw[TG_SET_MAX_WORDS];
  unsigned long long nslots;
  int32_t nkw;
  uint32_t stride;     // 8-byte words per record: 2 for a value alone, else a multiple of 4 (32-byte records)
};
typedef KeyWordsN<TG_SET_MAX_WORDS> SetKey;

// One thread per row: bit i of `mark` = row i's argument is not NULL and row i claimed a new (group, value) pair — exactly
// one row per pair, the one whose CAS claimed the slot.  The update kernels then read the argument column with `mark` as
// its null bitmap, so COUNT / SUM / AVG(DISTINCT x) are the plain functions over it.  A DOUBLE value is keyed with -0 as
// +0, and a NaN row is always new (Go map[float64]: NaN != NaN) without entering the set.  A row whose probe runs past
// max_probe is deferred like the group table's; `only` restricts a re-run to those rows, whose bits are then ORed in.
// Warps run whole 32-row words: lane 0 stores the ballot.  counters[0] = rows deferred, counters[1] = pairs inserted.
__global__ void __launch_bounds__(256)
k_agg_distinct_mark(GroupKeys gk, const long long* __restrict__ vals, const uint8_t* __restrict__ vnulls, int is_real, int64_t n,
                    DistinctSet t, uint32_t max_probe, uint32_t* mark, uint32_t* deferred, const uint32_t* only,
                    unsigned long long* counters) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long my_deferred = 0, my_new = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i - lane < n; i += stride) {
    bool win = false;
    if (i < n && (!only || ((only[i >> 5] >> (i & 31)) & 1u)) && (!vnulls || bit_not_null(vnulls, i))) {
      long long v = __ldcs(vals + i);
      bool nan = false;
      if (is_real) { double d = __longlong_as_double(v); if (d == 0) d = 0; nan = d != d; v = __double_as_longlong(d); }
      if (nan) win = true;
      else {
        SetKey k;
        load_key_words(gk, i, k);
#pragma unroll
        for (int j = 0; j < TG_SET_MAX_WORDS; j++) if (j == gk.nkw) k.w[j] = v;   // the value follows the group words
        bool ins = false;
        const unsigned long long s = mk_find_or_insert(t, k, hash_words(k, t.nkw), max_probe, &ins);
        if (s == ~0ull) { atomicOr(&deferred[i >> 5], 1u << (i & 31)); my_deferred++; }
        else if (ins) { win = true; my_new++; }
      }
    }
    const uint32_t b = __ballot_sync(0xffffffffu, win);
    if (lane == 0) { if (only) mark[i >> 5] |= b; else mark[i >> 5] = b; }
  }
  for (int o = 16; o; o >>= 1) {
    my_deferred += __shfl_xor_sync(0xffffffffu, my_deferred, o);
    my_new += __shfl_xor_sync(0xffffffffu, my_new, o);
  }
  if (lane == 0 && my_deferred) atomicAdd(&counters[0], my_deferred);
  if (lane == 0 && my_new) atomicAdd(&counters[1], my_new);
}

// re-insert every pair of an old set into a bigger one (pairs are distinct: claim with the published tag)
__global__ void k_agg_distinct_rehash(DistinctSet oldt, DistinctSet newt) {
  unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (; i < oldt.nslots; i += stride) {
    const unsigned long long tag = oldt.tags[(size_t)i * oldt.stride];
    if (tag == 0) continue;
    uint32_t s = slot32(tag, (uint32_t)newt.nslots);
    for (;;) {
      if (atomicCAS(&newt.tags[(size_t)s * newt.stride], 0ull, tag) == 0ull) break;
      if (++s == (uint32_t)newt.nslots) s = 0;
    }
    for (int j = 0; j < oldt.nkw; j++) newt.keyw[j][(size_t)s * newt.stride] = oldt.keyw[j][(size_t)i * oldt.stride];
  }
}

// A DECIMAL(flen <= 18, scale) argument column of 40-byte cells -> value * 10^scale as int64 (dec_parse_cell), once per batch
// and column, so that every update kernel sees an 8-byte integer column (40 bytes read + 8 written per row).  A thread owns
// two adjacent rows: 80 bytes, five 16-byte loads when the column is 16-byte aligned (V16; then so is every pair), else ten
// 8-byte loads (a caller's device column is only guaranteed 8-byte alignment).  A cell under NULL is not parsed and its
// loads are skipped (the 16-byte load in the middle of a pair may still fetch 8 of its bytes); its output is 0.  A
// non-NULL cell not in the column's stored form raises *err to `tag` (atomicMax: the host names the column).
template <bool V16>
__global__ void __launch_bounds__(256)
k_dec_to_scaled(const uint8_t* __restrict__ cells, const uint8_t* __restrict__ nulls, int64_t n, int flen, int scale,
                long long* __restrict__ out, unsigned long long* err, unsigned long long tag) {
  const int64_t npair = (n + 1) >> 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < npair; p += stride) {
    const int64_t r0 = 2 * p;
    const bool two = r0 + 1 < n;
    const bool nn0 = !nulls || bit_not_null(nulls, r0), nn1 = two && (!nulls || bit_not_null(nulls, r0 + 1));
    uint32_t c0[10], c1[10];
#pragma unroll
    for (int j = 0; j < 10; j++) { c0[j] = 0; c1[j] = 0; }
    if (V16 && two) {
      const uint4* q = reinterpret_cast<const uint4*>(cells + (size_t)r0 * TG_DEC_CELL_BYTES);
      const uint4 z = make_uint4(0, 0, 0, 0);
      const uint4 a = nn0 ? __ldcs(q) : z, b = nn0 ? __ldcs(q + 1) : z, m = (nn0 || nn1) ? __ldcs(q + 2) : z;
      const uint4 d = nn1 ? __ldcs(q + 3) : z, e = nn1 ? __ldcs(q + 4) : z;
      c0[0] = a.x; c0[1] = a.y; c0[2] = a.z; c0[3] = a.w; c0[4] = b.x; c0[5] = b.y; c0[6] = b.z; c0[7] = b.w; c0[8] = m.x; c0[9] = m.y;
      c1[0] = m.z; c1[1] = m.w; c1[2] = d.x; c1[3] = d.y; c1[4] = d.z; c1[5] = d.w; c1[6] = e.x; c1[7] = e.y; c1[8] = e.z; c1[9] = e.w;
    } else {
      const unsigned long long* q = reinterpret_cast<const unsigned long long*>(cells + (size_t)r0 * TG_DEC_CELL_BYTES);
#pragma unroll
      for (int j = 0; j < 5; j++) {
        if (nn0) { const unsigned long long w = __ldcs(q + j); c0[2 * j] = (uint32_t)w; c0[2 * j + 1] = (uint32_t)(w >> 32); }
        if (nn1) { const unsigned long long w = __ldcs(q + 5 + j); c1[2 * j] = (uint32_t)w; c1[2 * j + 1] = (uint32_t)(w >> 32); }
      }
    }
    long long v0 = 0, v1 = 0;
    bool bad = nn0 && !dec_parse_cell(c0, flen, scale, &v0);
    bad |= nn1 && !dec_parse_cell(c1, flen, scale, &v1);
    if (bad) atomicMax(err, tag);
    if (two) __stcs(reinterpret_cast<longlong2*>(out) + p, make_longlong2(v0, v1));   // `out` is a 256-byte aligned scratch column
    else out[r0] = v0;
  }
}

}  // namespace tg
#include "agg_update.cuh"
namespace tg {

// words of AggImpl::scalars, the handle's device counters
enum {
  SC_COUNT = 0,            // k_agg_count: occupied slots
  SC_DEFERRED = 1,         // rows an update round deferred
  SC_CURSOR = 2,           // k_agg_finalize's output cursor
  SC_V1_TUPLES = 3,        // partial tuples a v1 CTA-local pass emitted
  SC_MERGE_DEFERRED = 4,   // partial tuples a merge round deferred
  SC_SPILLED = 5,          // local groups a round-2 update spilled
  SC_LOCAL_ROWS = 6,       // rows the CTA-local level absorbed, since the table was created (zeroed with it)
  SC_OVERFLOW = 7,         // spec.err: a fused argument expression left the DOUBLE range
  SC_DEC_ERR = 8,          // k_dec_to_scaled: a DECIMAL cell not in its column's stored form
};

}  // namespace tg

using namespace tg;

struct AggImpl;

// shell + implementation, like tg_join (join.cu): close frees the implementation, the shell stays readable
struct tg_agg {
  std::mutex mu;
  std::atomic<bool> closed{false};
  AggImpl* impl = nullptr;
};

// What the gate compiles from a descriptor (agg_compile): the child schema, the group keys, the device functions and
// their state words, and the shape of every result.  tg_agg_supported* compiles one on the stack; a handle keeps its own.
struct AggPlan {
  int ncols = 0;
  std::vector<int> types, elem;
  std::vector<uint32_t> flags;
  std::vector<int> col_flen, col_dec;   // tg_agg_desc_ex: precision / scale per child column, -1 = not given
  std::vector<char> str_col;            // a string column of a descriptor with collations (tg_agg_desc_ex3)
  std::vector<int> coll;                // per child column: StrColl of its collation (COLL_NONE: not given / not one)
  std::vector<char> needed;
  int group_col = -1;          // -1: no GROUP BY (several GROUP BY columns: the first one)
  int gk_kind = GK_NONE;
  std::vector<int> group_cols, group_kinds;   // all GROUP BY columns
  int nkw = 0;                 // > 0: multi-key table (key words per slot)
  AggSpec spec{};
  int nstates = 0;
  std::vector<char> dec_decode;         // DECIMAL argument column of SUM / AVG / MIN / MAX: k_dec_to_scaled runs on every batch
  bool wide = false;        // a DECIMAL SUM / AVG of a product: the WIDE kernel instantiations
  bool dec_out = false;     // a DECIMAL result column: k_agg_finalize<true, wide>
  std::vector<char> out_nullable;
  std::vector<int> out_elem;   // bytes per result cell: 8, or 40 for a DECIMAL (MyDecimal) column

  // DISTINCT arguments (tg_agg_desc_ex2): set j dedups child column dist_cols[j] and feeds the virtual column ncols + j
  // (the column's values, null bitmap = the set's mark bits), which the DISTINCT functions read as their argument
  std::vector<char> fdistinct;          // per function: COUNT / SUM / AVG with HasDistinct
  std::vector<int> dist_cols;
  int dist_gkw = 0;                     // group key words of a set record (the value word follows)

  // string columns (tg_agg_desc_ex3): a string GROUP BY column is encoded to ids by its dictionary (str_dict.cuh) before
  // the DISTINCT sets and the update kernels see the batch; its FIRSTROW finalizes to the id, then gathers the bytes
  std::vector<char> is_str;             // a string column the plan reads (GROUP BY key or COUNT argument)
  std::vector<char> needed_fixed;       // `needed` without the string columns (validate_chunk / device_view)
  std::vector<int> dict_of;             // per child column: its dictionary, -1
  std::vector<int> out_dict;            // per result: the dictionary of a string result, -1
  // FIRSTROW of a PAD-collation string key with several GROUP BY columns: the dictionary's earliest row of a key value
  // is not each group's, so the encode pass writes a tail column (ordinal << kTailBits | trailing spaces cut) and a
  // hidden unsigned MIN per group keeps its earliest row's: that row's raw bytes are the key plus that many spaces
  int n_out = 0;                        // functions of the descriptor; spec.n counts the hidden MINs after them
  std::vector<int> tail_col;            // per child column: the virtual column of its tail values, -1
  std::vector<int> tail_fn;             // per result: the hidden MIN of its tail values, -1
};

struct AggImpl : DeviceHandle, AggPlan {
  std::vector<std::unique_ptr<DevBuf>> dscaled;   // per DECIMAL argument column: its int64 value * 10^scale, pooled scratch

  struct SetMem { DevBuf mem, mark; DistinctSet t{}; unsigned long long used = 0; };   // used: the pairs the set holds
  std::vector<std::unique_ptr<SetMem>> dsets;
  DevBuf dcounters;                     // k_agg_distinct_mark: [0] rows deferred [1] pairs inserted
  bool broken = false;                  // a push failed after a set was touched: every later push / finish fails
  tg_agg_distinct_stats dstats{};

  std::vector<std::unique_ptr<StrDict>> dicts;
  std::vector<std::unique_ptr<DevBuf>> sids, doffs;   // per child column: the id column of a batch, a batch's offsets
  DevBuf sflag;                         // bad-offsets flag of a device push
  int64_t str_ords = 0;                 // logical rows encoded so far: the ordinal of the next batch's first row
  double encode_ms = 0;
  std::vector<std::unique_ptr<DevBuf>> stails;   // per child column: a batch's tail values
  std::vector<std::unique_ptr<DevBuf>> out_soffs, out_sbytes;
  std::vector<std::vector<int64_t>> host_soffs;   // the string results' offsets, read back once at finish

  // table
  DevBuf tbl_mem;
  AggTable tbl{};
  unsigned long long nslots = 0;
  DevBuf scalars;              // counters, SC_* words
  DevBuf deferred[2];          // row bitmaps of grow_and_retry: one round's input and the next round's
  DevBuf partials_mem;
  int64_t expected_groups = 0;
  int local_mode = -1;            // -1 undecided, 0 global atomics only, 1 CTA-local partial aggregation first

  // staging
  HostStage stage;
  std::vector<std::unique_ptr<DevBuf>> dcols, dnulls;

  // result
  bool finished = false;
  std::vector<std::unique_ptr<DevBuf>> out_cols, out_valid, out_bitmaps;
  int64_t out_rows = 0, consumed = 0;
  tg_agg_stats stats{};
};

namespace tg {

static long long pow10_i64(int k) { long long p = 1; while (k-- > 0) p *= 10; return p; }

// TG_TYPE_VARCHAR, VARSTRING, STRING and the BLOB / TEXT types (ENUM, SET, JSON and BIT are var-length, not strings)
static bool agg_string_type(int32_t tp) {
  return tp == TG_TYPE_VARCHAR || tp == TG_TYPE_VARSTRING || tp == TG_TYPE_STRING || (tp >= TG_TYPE_TINY_BLOB && tp <= TG_TYPE_BLOB);
}

// What a function's argument is, once the schema is read: the class decides which rules the function runs
enum ArgClass { ARG_NONE, ARG_INT, ARG_REAL, ARG_DEC, ARG_DEC_PRODUCT, ARG_STR, ARG_OTHER };
static int arg_class(const AggPlan* p, const tg_agg_func& f) {
  if (f.arg_col < 0 || f.arg_col >= p->ncols) return ARG_NONE;
  const int t = p->types[f.arg_col];
  if (p->str_col[f.arg_col]) return ARG_STR;
  if (t == TG_TYPE_NEWDECIMAL) return f.arg_expr == TG_ARGEXPR_MUL || f.arg_expr == TG_ARGEXPR_MUL_CSUB ? ARG_DEC_PRODUCT : ARG_DEC;
  if (t == TG_TYPE_DOUBLE) return ARG_REAL;
  return is_int_family(t) ? ARG_INT : ARG_OTHER;
}

// A DECIMAL result keeps the argument's scale s, except AVG, which rounds to s .. 30 digits (typeInfer4Sum / typeInfer4Avg)
static int ret_frac_rule(const tg_agg_func& f, int s, const char* avg_msg, const char* msg) {
  if (f.name == TG_AGG_AVG ? (f.ret_frac < s || f.ret_frac > 30) : f.ret_frac != s) return fail(TG_ERR_INVALID, f.name == TG_AGG_AVG ? avg_msg : msg);
  return TG_OK;
}

// A DECIMAL argument column is decoded to one int64 at its scale: it needs its precision (1..18) and scale
static int dec_col_rules(const AggPlan* p, int c) {
  const int prec = p->col_flen[c], s = p->col_dec[c];
  if (prec < 0 || s < 0) return fail(TG_ERR_UNSUPPORTED, "a DECIMAL argument column needs its precision and scale (tg_agg_desc_ex col_flen / col_decimal)");
  if (prec > 18) return fail(TG_ERR_UNSUPPORTED, "DECIMAL arguments are offloaded up to precision 18 (one int64 at the column's scale)");
  if (prec < 1 || s > prec) return fail(TG_ERR_INVALID, "a DECIMAL column needs 1 <= flen and 0 <= decimal <= flen");
  return TG_OK;
}

// SUM / AVG of a * b or a * (c - b) over two DECIMAL(p <= 18) columns (dec_arg_rules has checked a and the mode): the exact
// product (DecimalMul, mydecimal.go:2041) has scale s = s_a + s_b, and c - b (DecimalSub) is exact at scale s_b
static int dec_product_rules(const AggPlan* p, const tg_agg_func& f) {
  const int c2 = f.arg_col2;
  if (c2 < 0 || c2 >= p->ncols || p->types[c2] != TG_TYPE_NEWDECIMAL)
    return fail(TG_ERR_UNSUPPORTED, "a DECIMAL argument expression takes two DECIMAL columns");
  TG_TRY(dec_col_rules(p, c2));
  if (f.name != TG_AGG_SUM && f.name != TG_AGG_AVG) return fail(TG_ERR_UNSUPPORTED, "argument expressions are fused for SUM / AVG only");
  if (f.ret_type != TG_TYPE_NEWDECIMAL) return fail(TG_ERR_UNSUPPORTED, "SUM / AVG of a DECIMAL product need a DECIMAL ret_type");
  const int s2 = p->col_dec[c2], s = p->col_dec[f.arg_col] + s2;
  // TiDB types the product with frac min(s, 30) but keeps digitsFrac min(s, 31) in the value: past 30 the two disagree
  if (s > 30) return fail(TG_ERR_UNSUPPORTED, "a DECIMAL product is offloaded up to scale 30 (s_a + s_b)");
  if (f.arg_expr == TG_ARGEXPR_MUL_CSUB) {   // c * 10^s_b - b must fit int64: |c| * 10^s_b <= 10^18 keeps it below 2 * 10^18
    const double c = f.arg_const;
    const double lim = 1e18 / (double)pow10_i64(s2);   // 10^(18 - s_b), exact in a double
    if (!std::isfinite(c) || c != std::trunc(c) || std::fabs(c) > lim)
      return fail(TG_ERR_UNSUPPORTED, "a DECIMAL c - b takes an integer constant c with |c| * 10^scale(b) <= 10^18");
  }
  return ret_frac_rule(f, s, "DECIMAL AVG of a product: scale must be s_a + s_b .. 30", "DECIMAL SUM of a product has the scale s_a + s_b");
}

// A function over a DECIMAL column (tg_agg_desc_ex), alone or in a product: TG_OK when it is offloaded
static int dec_arg_rules(const AggPlan* p, const tg_agg_func& f) {
  TG_TRY(dec_col_rules(p, f.arg_col));
  if (f.mode != TG_AGGMODE_COMPLETE) return fail(TG_ERR_UNSUPPORTED, "aggregates over DECIMAL columns are offloaded in Complete mode only (no DECIMAL partial results)");
  if (f.arg_expr == TG_ARGEXPR_MUL || f.arg_expr == TG_ARGEXPR_MUL_CSUB) return dec_product_rules(p, f);
  if (f.arg_expr != TG_ARGEXPR_COL) return fail(TG_ERR_UNSUPPORTED, "a DECIMAL column is not offloaded in this argument expression");
  switch (f.name) {
    case TG_AGG_COUNT:   // reads the null bitmap only
      return f.ret_type == TG_TYPE_NEWDECIMAL ? fail(TG_ERR_UNSUPPORTED, "a DECIMAL result is offloaded for SUM / AVG / MIN / MAX only") : TG_OK;
    case TG_AGG_SUM: case TG_AGG_AVG: case TG_AGG_MIN: case TG_AGG_MAX:
      if (f.ret_type != TG_TYPE_NEWDECIMAL) return fail(TG_ERR_UNSUPPORTED, "SUM / AVG / MIN / MAX over a DECIMAL column need a DECIMAL ret_type");
      return ret_frac_rule(f, p->col_dec[f.arg_col], "DECIMAL AVG scale must be the column's scale .. 30",
                           "DECIMAL SUM / MIN / MAX of a DECIMAL column have the column's scale");
    default: return fail(TG_ERR_UNSUPPORTED, "this aggregate function is not offloaded over a DECIMAL column");
  }
}

// DECIMAL SUM / AVG of an integer column (typeInfer4Sum / typeInfer4Avg, aggregation/base_func.go); any other ret_type
// keeps the result type each function has always had here
static int dec_result_rules(const AggPlan* p, const tg_agg_func& f) {
  if (f.name != TG_AGG_SUM && f.name != TG_AGG_AVG) return fail(TG_ERR_UNSUPPORTED, "a DECIMAL result is offloaded for SUM / AVG only");
  if (f.mode != TG_AGGMODE_COMPLETE) return fail(TG_ERR_UNSUPPORTED, "DECIMAL SUM / AVG are offloaded in Complete mode only (no DECIMAL partial results)");
  if (f.arg_expr != TG_ARGEXPR_COL) return fail(TG_ERR_UNSUPPORTED, "DECIMAL SUM / AVG take a plain column argument");
  if (f.arg_col < 0 || f.arg_col >= p->ncols) return fail(TG_ERR_INVALID, "aggregate argument column out of range");
  const int t = p->types[f.arg_col];
  if (!is_int_family(t) || t == TG_TYPE_DURATION || p->elem[f.arg_col] != 8)
    return fail(TG_ERR_UNSUPPORTED, "DECIMAL SUM / AVG are offloaded over 8-byte integer columns only");
  return ret_frac_rule(f, 0, "DECIMAL AVG scale must be 0..30", "DECIMAL SUM of an integer column has scale 0");
}

// COUNT / SUM / AVG with HasDistinct (tg_agg_desc_ex2), checked before the rules of the same function without it, which
// must accept it too: TG_OK when its dedup pass is offloaded, else the status and message
static int distinct_rules(const AggPlan* p, const tg_agg_func& f) {
  if (f.arg_col < 0 || f.arg_col >= p->ncols) return fail(TG_ERR_INVALID, "a DISTINCT aggregate needs an argument column");
  if (f.name == TG_AGG_FIRSTROW) return fail(TG_ERR_UNSUPPORTED, "FIRSTROW with DISTINCT is not offloaded");
  if (f.mode != TG_AGGMODE_COMPLETE) return fail(TG_ERR_UNSUPPORTED, "DISTINCT aggregates are offloaded in Complete mode only");
  if (f.arg_expr != TG_ARGEXPR_COL) return fail(TG_ERR_UNSUPPORTED, "DISTINCT aggregates take a plain column argument");
  if (f.name == TG_AGG_COUNT && f.arg_col2 >= 0) return fail(TG_ERR_UNSUPPORTED, "COUNT(DISTINCT a, b) over several arguments is not offloaded");
  const int t = p->types[f.arg_col];
  if (!((is_int_family(t) && p->elem[f.arg_col] == 8) || t == TG_TYPE_DOUBLE || t == TG_TYPE_NEWDECIMAL))
    return fail(TG_ERR_UNSUPPORTED, "DISTINCT aggregates are offloaded over integer-family, DOUBLE and DECIMAL(p <= 18) columns");
  return TG_OK;
}

// A function over a string column (tg_agg_desc_ex3): TG_OK when it is offloaded, else the status and message
static int str_arg_rules(const AggPlan* p, const tg_agg_func& f) {
  if (f.arg_expr != TG_ARGEXPR_COL) return fail(TG_ERR_UNSUPPORTED, "a string column is not offloaded in an argument expression");
  switch (f.name) {
    case TG_AGG_COUNT:   // reads the null bitmap only
      if (f.mode != TG_AGGMODE_COMPLETE) return fail(TG_ERR_UNSUPPORTED, "COUNT over a string column is offloaded in Complete mode only");
      if (f.ret_type == TG_TYPE_NEWDECIMAL) return fail(TG_ERR_UNSUPPORTED, "a DECIMAL result is offloaded for SUM / AVG / MIN / MAX only");
      return TG_OK;
    case TG_AGG_FIRSTROW:
      if (p->dict_of[f.arg_col] < 0) return fail(TG_ERR_UNSUPPORTED, "FIRSTROW of a string column is offloaded only for GROUP BY columns");
      return TG_OK;
    default: return fail(TG_ERR_UNSUPPORTED, "only FIRSTROW (of a GROUP BY column) and COUNT are offloaded over string columns");
  }
}

static AggFuncDev func_dev(const tg_agg_func& f) {   // no state words yet, an 8-byte result
  return AggFuncDev{f.name, f.arg_col, 0, 0, -1, -1, 0, f.arg_col2, f.arg_expr, -1, 0, -1, -1, f.arg_const, 0};
}

// The state words of one function: its value in `words` words (1; 2 or 3 for the 128 / 192-bit sum of a DECIMAL SUM /
// AVG: dec3_apply / sdec3_apply find them one state stride apart, so they are consecutive), then a non-NULL count
static void add_states(AggPlan* p, AggFuncDev& o, int words, bool count) {
  o.s0 = p->nstates++;
  if (words > 1) o.s2 = p->nstates++;
  if (words > 2) o.s3 = p->nstates++;
  if (count) o.s1 = p->nstates++;
}

static bool nullable_col(const AggPlan* p, int c) { return !(p->flags[c] & TG_FLAG_NOT_NULL); }

static int compile_schema(AggPlan* p, const tg_agg_desc_ex3& d) {
  const tg_agg_desc& b = d.ex2.ex.base;
  if (b.n_cols <= 0 || b.n_cols > TG_MAX_COLS) return fail(TG_ERR_UNSUPPORTED, "child schema must have 1..16 columns");
  p->ncols = b.n_cols;
  for (int c = 0; c < b.n_cols; c++) {
    const int t = b.col_types[c];
    const bool str = d.col_collation && agg_string_type(t);
    p->types.push_back(t);
    p->flags.push_back(b.col_flags ? b.col_flags[c] : 0);
    p->elem.push_back(fixed_len(t));
    p->col_flen.push_back(d.ex2.ex.col_flen ? d.ex2.ex.col_flen[c] : -1);
    p->col_dec.push_back(d.ex2.ex.col_decimal ? d.ex2.ex.col_decimal[c] : -1);
    p->str_col.push_back(str);
    p->coll.push_back(str ? coll_of_id(d.col_collation[c]) : COLL_NONE);
  }
  p->needed.assign(b.n_cols, 0);
  p->dec_decode.assign(b.n_cols, 0);
  p->dict_of.assign(b.n_cols, -1);
  return TG_OK;
}

static int compile_group_keys(AggPlan* p, const tg_agg_desc& b) {
  if (b.n_group_by > TG_MAX_GROUP_COLS) return fail(TG_ERR_UNSUPPORTED, "GPU hash aggregation handles up to 4 GROUP BY columns");
  bool any_nullable = false;
  int ndicts = 0;
  for (int q = 0; q < b.n_group_by; q++) {
    const int g = b.group_by_cols[q];
    if (g < 0 || g >= p->ncols) return fail(TG_ERR_INVALID, "group-by column out of range");
    const int t = p->types[g];
    if (!is_int_family(t) && t != TG_TYPE_DOUBLE && !p->str_col[g]) return fail(TG_ERR_UNSUPPORTED, "GROUP BY column type is not offloaded (int family / double only)");
    if (p->str_col[g]) {   // encoded to a dense int64 id column (encode_strings)
      if (p->coll[g] == COLL_NONE) return fail(TG_ERR_UNSUPPORTED, "string GROUP BY collation not offloaded (binary, *_bin and utf8mb4_0900_bin are)");
      if (p->dict_of[g] < 0) p->dict_of[g] = ndicts++;
    } else if (p->elem[g] != 8) return fail(TG_ERR_UNSUPPORTED, "GROUP BY columns must be 8-byte columns");
    const int kind = t == TG_TYPE_DOUBLE ? GK_F64 : GK_I64;
    if (q == 0) { p->group_col = g; p->gk_kind = kind; }
    p->group_cols.push_back(g); p->group_kinds.push_back(kind);
    any_nullable |= nullable_col(p, g);
    p->needed[g] = 1;
  }
  p->dist_gkw = b.n_group_by + (any_nullable ? 1 : 0);
  if (b.n_group_by > 1) p->nkw = p->dist_gkw;
  return TG_OK;
}

// The rules of function k that do not depend on its function name: its argument's class decides which ones run
static int func_rules(AggPlan* p, const tg_agg_desc_ex3& d, int k) {
  const tg_agg_func& f = d.ex2.ex.base.funcs[k];
  if (d.ex2.has_distinct && d.ex2.has_distinct[k]) {
    if (f.arg_col < 0) return fail(TG_ERR_INVALID, "a DISTINCT aggregate needs an argument column");
    // MIN / MAX: DISTINCT changes nothing (buildMaxMin ignores HasDistinct)
    if (f.name != TG_AGG_MIN && f.name != TG_AGG_MAX) { TG_TRY(distinct_rules(p, f)); p->fdistinct[k] = 1; }
  }
  const int cls = arg_class(p, f);
  const bool dec_arg = cls == ARG_DEC || cls == ARG_DEC_PRODUCT;
  if (cls == ARG_STR) {
    TG_TRY(str_arg_rules(p, f));
    if (f.name == TG_AGG_FIRSTROW) p->out_dict[k] = p->dict_of[f.arg_col];
  }
  if (dec_arg) TG_TRY(dec_arg_rules(p, f));
  else if (f.ret_type == TG_TYPE_NEWDECIMAL) TG_TRY(dec_result_rules(p, f));
  if (f.arg_expr != TG_ARGEXPR_COL) {
    if (f.arg_expr != TG_ARGEXPR_MUL && f.arg_expr != TG_ARGEXPR_MUL_CSUB) return fail(TG_ERR_INVALID, "unknown aggregate argument expression");
    if ((f.name != TG_AGG_SUM && f.name != TG_AGG_AVG) || f.mode != TG_AGGMODE_COMPLETE)
      return fail(TG_ERR_UNSUPPORTED, "argument expressions are fused for SUM / AVG in Complete mode only");
    if (!dec_arg && (cls != ARG_REAL || f.arg_col2 < 0 || f.arg_col2 >= p->ncols || p->types[f.arg_col2] != TG_TYPE_DOUBLE))
      return fail(TG_ERR_UNSUPPORTED, "argument expressions take two DOUBLE columns");
    p->needed[f.arg_col2] = 1;
  }
  if (f.mode != TG_AGGMODE_COMPLETE && f.mode != TG_AGGMODE_FINAL) return fail(TG_ERR_UNSUPPORTED, "only Complete and Final aggregate modes are offloaded");
  if (f.arg_col >= p->ncols || f.arg_col2 >= p->ncols) return fail(TG_ERR_INVALID, "aggregate argument column out of range");
  if (cls != ARG_NONE) {
    if (p->elem[f.arg_col] != 8 && !dec_arg && cls != ARG_STR) return fail(TG_ERR_UNSUPPORTED, "aggregate arguments must be 8-byte columns");
    p->needed[f.arg_col] = 1;
  }
  return TG_OK;
}

// The device function, state words and result shape of function k, with the rules that depend on its function name
static int compile_func(AggPlan* p, const tg_agg_desc_ex3& d, int k) {
  const tg_agg_func& f = d.ex2.ex.base.funcs[k];
  AggFuncDev& o = p->spec.f[k] = func_dev(f);
  TG_TRY(func_rules(p, d, k));
  const int cls = arg_class(p, f);   // the argument columns are in range now: ARG_NONE is arg_col < 0
  // a DECIMAL(p <= 18, s) argument column: decoded to int64 value * 10^s on every batch, then the integer update paths run
  const bool dec_arg = cls == ARG_DEC || cls == ARG_DEC_PRODUCT, dec = f.ret_type == TG_TYPE_NEWDECIMAL;
  // a DISTINCT argument is NULL on every row that brought no new value: COUNT needs its own count, AVG its divisor
  const bool distinct = p->fdistinct[k] != 0;
  const bool nullable = distinct || (cls != ARG_NONE && nullable_col(p, f.arg_col)) ||
                        (f.arg_expr != TG_ARGEXPR_COL && f.arg_col2 >= 0 && nullable_col(p, f.arg_col2));
  o.final_mode = f.mode == TG_AGGMODE_FINAL;
  o.is_real = cls == ARG_REAL;
  o.is_unsigned = cls != ARG_NONE && !dec_arg && (p->flags[f.arg_col] & TG_FLAG_UNSIGNED) != 0;   // a decoded DECIMAL is a signed int64
  if (dec_arg && (f.name != TG_AGG_COUNT || distinct)) p->dec_decode[f.arg_col] = 1;   // COUNT(DISTINCT dec): the set is keyed on the value
  if (dec_arg && f.name != TG_AGG_COUNT) o.dec_scale = p->col_dec[f.arg_col];
  else if (dec) o.dec_scale = 0;
  if (cls == ARG_DEC_PRODUCT) {
    const int sb = p->col_dec[f.arg_col2];
    o.dec_scale += sb;
    p->dec_decode[f.arg_col2] = 1;
    if (f.arg_expr == TG_ARGEXPR_MUL_CSUB) o.dec_c = (long long)f.arg_const * pow10_i64(sb);
  }
  p->dec_out |= o.dec_scale >= 0;
  switch (f.name) {
    case TG_AGG_COUNT:
      if (o.final_mode && cls == ARG_NONE) return fail(TG_ERR_INVALID, "final COUNT needs the partial count column");
      if (o.final_mode || (cls != ARG_NONE && nullable)) add_states(p, o, 1, false);   // NOT NULL COUNT(x) == COUNT(*) == rows[]
      return TG_OK;
    case TG_AGG_SUM: case TG_AGG_AVG:
      p->out_nullable[k] = 1;
      if (dec) {   // the exact sum (a product's in 3 words), non-NULL count (NOT NULL arguments count with rows[])
        add_states(p, o, cls == ARG_DEC_PRODUCT ? 3 : 2, nullable);
        p->wide |= cls == ARG_DEC_PRODUCT;
        if (f.name == TG_AGG_AVG) o.dec_frac = f.ret_frac;
        p->out_elem[k] = TG_DEC_CELL_BYTES;
      } else if (f.name == TG_AGG_AVG && o.final_mode) {
        if (cls == ARG_NONE || f.arg_col2 < 0 || p->types[f.arg_col2] != TG_TYPE_DOUBLE || !is_int_family(p->types[f.arg_col]))
          return fail(TG_ERR_UNSUPPORTED, "final AVG takes (count BIGINT, sum DOUBLE)");
        p->needed[f.arg_col2] = 1;
        add_states(p, o, 1, true);
      } else {   // SUM(int) yields DECIMAL in TiDB (aggregation/base_func.go:223-245): offloaded only when ret_type asks for it
        if (cls != ARG_REAL) return fail(TG_ERR_UNSUPPORTED, f.name == TG_AGG_SUM ? "SUM is offloaded for DOUBLE arguments only (SUM(int) is DECIMAL)"
                                                                                 : "AVG is offloaded for DOUBLE arguments only");
        add_states(p, o, 1, nullable);
      }
      return TG_OK;
    case TG_AGG_MIN: case TG_AGG_MAX:
      if (!dec_arg && cls != ARG_INT && cls != ARG_REAL) return fail(TG_ERR_UNSUPPORTED, "MIN/MAX are offloaded for int family / DOUBLE / DECIMAL");
      add_states(p, o, 1, nullable);
      p->out_nullable[k] = 1;
      if (dec_arg) p->out_elem[k] = TG_DEC_CELL_BYTES;   // the signed int64 MIN / MAX at the column's scale
      return TG_OK;
    case TG_AGG_FIRSTROW: {
      int gi = -1;   // the last GROUP BY item of the column
      for (size_t q = 0; q < p->group_cols.size(); q++) if (p->group_cols[q] == f.arg_col) gi = (int)q;
      if (cls == ARG_NONE || gi < 0) return fail(TG_ERR_UNSUPPORTED, "FIRSTROW is offloaded only for GROUP BY columns (deterministic)");
      p->out_nullable[k] = nullable_col(p, f.arg_col);
      o.arg_col2 = gi | ((p->nkw > (int)p->group_cols.size() ? (int)p->group_cols.size() : 0) << 8);
      return TG_OK;
    }
    default: return fail(TG_ERR_UNSUPPORTED, "aggregate function is not offloaded");
  }
}

// One dedup set per DISTINCT argument column; its functions read the virtual column ncols + j (free DevCols slots)
static int compile_distinct(AggPlan* p) {
  for (int k = 0; k < p->n_out; k++) {
    if (!p->fdistinct[k]) continue;
    int& c = p->spec.f[k].arg_col;
    const size_t j = std::find(p->dist_cols.begin(), p->dist_cols.end(), c) - p->dist_cols.begin();
    if (j == p->dist_cols.size()) p->dist_cols.push_back(c);
    c = p->ncols + (int)j;
  }
  if (p->ncols + (int)p->dist_cols.size() > TG_MAX_COLS)
    return fail(TG_ERR_UNSUPPORTED, "DISTINCT aggregates need one free column slot per argument column (child columns + DISTINCT columns <= 16)");
  return TG_OK;
}

// FIRSTROW of a PAD string key under several GROUP BY columns: one tail column and one hidden MIN per such column
static int compile_tail_mins(AggPlan* p, int n_group_by) {
  p->tail_col.assign(p->ncols, -1);
  p->tail_fn.assign(p->n_out, -1);
  std::vector<int> min_of(p->ncols, -1);
  int nvirt = p->ncols + (int)p->dist_cols.size();
  for (int k = 0; k < p->n_out; k++) {
    const int c = p->spec.f[k].arg_col;
    if (p->out_dict[k] < 0 || p->coll[c] != COLL_PAD_BIN || n_group_by < 2) continue;
    if (min_of[c] < 0) {
      if (nvirt >= TG_MAX_COLS) return fail(TG_ERR_UNSUPPORTED, "FIRSTROW of a PAD string key with several GROUP BY columns needs a free column slot (child columns + DISTINCT columns + such keys <= 16)");
      if (p->spec.n >= TG_MAX_AGG) return fail(TG_ERR_UNSUPPORTED, "FIRSTROW of a PAD string key with several GROUP BY columns takes a hidden aggregate slot (at most 12 in all)");
      p->tail_col[c] = nvirt++;
      min_of[c] = p->spec.n++;
      AggFuncDev& o = p->spec.f[min_of[c]] = func_dev(tg_agg_func{TG_AGG_MIN, TG_AGGMODE_COMPLETE, p->tail_col[c], 0, 0, -1, TG_ARGEXPR_COL, 0, 0, 0.0});
      o.is_unsigned = 1;
      add_states(p, o, 1, false);
      p->out_nullable.push_back(0); p->out_elem.push_back(8); p->out_dict.push_back(-1); p->fdistinct.push_back(0);
    }
    p->tail_fn[k] = min_of[c];
  }
  return TG_OK;
}

// The gate: compiles a descriptor into a fresh *p, or returns the status and message of the first rule it breaks
static int agg_compile(AggPlan* p, const tg_agg_desc_ex3& d) {
  const tg_agg_desc& b = d.ex2.ex.base;
  TG_TRY(compile_schema(p, d));
  TG_TRY(compile_group_keys(p, b));
  if (b.n_funcs <= 0 || b.n_funcs > TG_MAX_AGG) return fail(TG_ERR_UNSUPPORTED, "1..12 aggregate functions are offloaded");
  p->spec.n = p->n_out = b.n_funcs;
  p->out_nullable.assign(b.n_funcs, 0);
  p->out_elem.assign(b.n_funcs, 8);
  p->fdistinct.assign(b.n_funcs, 0);
  p->out_dict.assign(b.n_funcs, -1);
  for (int k = 0; k < b.n_funcs; k++) TG_TRY(compile_func(p, d, k));
  TG_TRY(compile_distinct(p));
  TG_TRY(compile_tail_mins(p, b.n_group_by));
  if (p->nstates > 2 * TG_MAX_AGG) return fail(TG_ERR_UNSUPPORTED, "the aggregate list needs more than 24 state words (a DECIMAL SUM / AVG takes up to 3, up to 4 over a product)");
  p->is_str.assign(p->ncols, 0);
  p->needed_fixed = p->needed;
  for (int c = 0; c < p->ncols; c++)
    if (p->needed[c] && p->str_col[c]) { p->is_str[c] = 1; p->needed_fixed[c] = 0; }
  return TG_OK;
}

static int table_record_words(const AggImpl* a) { return a->nkw ? ((1 + a->nkw + 1 + a->nstates + 3) / 4) * 4 : (2 + a->nstates); }
static void layout_table(AggImpl* a, uint8_t* mem, unsigned long long nslots, AggTable& t) {
  size_t n = (size_t)nslots + 2;
  t.nslots = nslots;
  t.nkw = a->nkw;
  if (a->nkw) {   // array of records: [tag | nkw key words | rows | states], padded to a multiple of 32 bytes
    unsigned long long* w = reinterpret_cast<unsigned long long*>(mem);
    t.stride = (uint32_t)table_record_words(a);
    t.tags = w; t.keys = reinterpret_cast<long long*>(w);
    for (int j = 0; j < a->nkw; j++) t.keyw[j] = reinterpret_cast<long long*>(w + 1 + j);
    t.rows = w + 1 + a->nkw;
    for (int s = 0; s < a->nstates; s++) t.state[s] = w + 2 + a->nkw + s;
    return;
  }
  t.stride = 1;
  t.keys = reinterpret_cast<long long*>(mem);
  t.tags = reinterpret_cast<unsigned long long*>(mem);
  t.rows = reinterpret_cast<unsigned long long*>(mem + n * 8);
  for (int s = 0; s < a->nstates; s++) t.state[s] = reinterpret_cast<unsigned long long*>(mem + n * 8 * (2 + s));
}

static int alloc_table(AggImpl* a, unsigned long long nslots, DevBuf& mem, AggTable& t) {
  // slots are 32-bit (agg_home, slot32): a bigger table would send every key to one slot
  if (nslots >= (1ull << 32)) return fail(TG_ERR_OOM, "the aggregation table would need 2^32 slots or more");
  size_t n = (size_t)nslots + 2;
  TG_TRY(mem.ensure(a->device, n * 8 * (size_t)table_record_words(a) + 64));
  layout_table(a, mem.as<uint8_t>(), nslots, t);
  k_agg_init<<<grid_size(a->nsm, (int64_t)n, 256, 8), 256, 0, a->stream>>>(t, a->spec, n);
  a->stats.kernel_launches++;
  return TG_OK;
}

// x4, or more: the grown table is at most half full once `more` new groups (deferred items) join a table that was 60 % full
static unsigned long long grown_slots(unsigned long long cur, unsigned long long more) {
  return std::max<unsigned long long>(cur * 4, (unsigned long long)((cur * 0.6 + (double)more) * 2));
}

// grow the group table for `more` new groups: rehash into a grown_slots table
static int grow_table(AggImpl* a, unsigned long long more) {
  const unsigned long long want_slots = grown_slots(a->nslots, more);
  std::unique_ptr<DevBuf> nm(new DevBuf());
  AggTable nt{};
  TG_TRY(alloc_table(a, want_slots, *nm, nt));
  if (a->nkw) k_agg_rehash_mk<<<grid_size(a->nsm, (int64_t)a->tbl.nslots, 256, 8), 256, 0, a->stream>>>(a->tbl, nt, a->nstates);
  else k_agg_rehash<<<grid_size(a->nsm, (int64_t)a->tbl.nslots + 2, 256, 8), 256, 0, a->stream>>>(a->tbl, nt, a->nstates);
  a->stats.kernel_launches++;
  TG_CUDA(cudaStreamSynchronize(a->stream));
  std::swap(a->tbl_mem.p, nm->p); std::swap(a->tbl_mem.cap, nm->cap); std::swap(a->tbl_mem.device, nm->device);
  a->tbl = nt;
  a->nslots = want_slots;
  return TG_OK;
}

__global__ void k_mark_range(uint32_t* bits, int64_t lo, int64_t hi) {
  int64_t i = lo + blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < hi; i += stride) atomicOr(&bits[i >> 5], 1u << (i & 31));
}
static int mark_range_deferred(AggImpl* a, int64_t lo, int64_t hi) {
  // whole 32-bit words with memset, ragged edges with a tiny kernel
  int64_t wlo = (lo + 31) / 32, whi = hi / 32;
  uint32_t* bits = a->deferred[0].as<uint32_t>();
  if (whi > wlo) TG_CUDA(cudaMemsetAsync(bits + wlo, 0xff, (size_t)(whi - wlo) * 4, a->stream));
  int64_t e1 = std::min<int64_t>(hi, wlo * 32);
  if (lo < e1) { k_mark_range<<<1, 64, 0, a->stream>>>(bits, lo, e1); a->stats.kernel_launches++; }
  int64_t s2 = std::max<int64_t>(std::max<int64_t>(lo, e1), whi * 32);
  if (s2 < hi) { k_mark_range<<<1, 64, 0, a->stream>>>(bits, s2, hi); a->stats.kernel_launches++; }
  return TG_OK;
}

// A round deferred nd items from a table of `slots` slots with `used` of them taken: true when the table stays at most a
// quarter full once they join, so a probe ran long because the keys share a home, not because the table is full.  A
// home depends only on the top 32 bits of a 64-bit hash, so keys that share those bits share a home at every size, and
// growing would never shorten their run.  Uniform keys at a quarter load start a run long enough to defer an item with a
// probability below 3e-14 per slot (a Chernoff bound, tests/agg_keys.py), so this does not change how uniform data grows;
// at half load the same bound is 8e-5 per slot, which a table of millions of slots does reach.
static bool long_run_not_full(unsigned long long used, unsigned long long nd, unsigned long long slots) {
  return (used + nd) * 4 <= slots;
}

// Grow-and-retry, the protocol of every find-or-insert pass into the group table, a DISTINCT set or a string dictionary.
// launch(deferred, only, max_probe, nd) runs one round over the pass's `nitems` items (only == nullptr: all of them, else
// those whose bit is set), sets in `deferred` the bit of every item that found no slot within max_probe steps, and reads
// back their number into nd.  fill(used, slots) reads how many slots the table has and how many are taken.
// grow(nd, room) makes room for nd new entries; room: the table has it already (long_run_not_full), and grow only
// extends what else the pass sizes by its entries (a dictionary's per-id arrays).  The next round re-runs just the
// deferred items: with room, through an unbounded probe (max_probe = slots) on the same table — nothing is ever deleted
// from it, so a walk past kAggMaxProbe steps still meets an existing key before any empty slot — else with kAggMaxProbe
// on the grown table.  bits[0] and bits[1] take turns as the bitmap a round writes and the one it reads; `resume`: the
// items of the first round are the ones already marked in bits[0].
template <class Launch, class Fill, class Grow>
static int grow_and_retry(AggImpl* a, DevBuf (&bits)[2], int64_t nitems, bool resume, const char* what, Launch launch, Fill fill, Grow grow) {
  const size_t bytes = (size_t)((nitems + 31) / 32) * 4;
  int cur = resume ? 1 : 0;
  const uint32_t* only = resume ? bits[0].as<uint32_t>() : nullptr;
  uint32_t max_probe = kAggMaxProbe;
  for (int round = 0;; round++) {
    TG_TRY(bits[cur].ensure(a->device, bytes + 16));
    TG_CUDA(cudaMemsetAsync(bits[cur].p, 0, bytes, a->stream));
    unsigned long long nd = 0;
    TG_TRY(launch(bits[cur].as<uint32_t>(), only, max_probe, nd));
    if (nd == 0) return TG_OK;
    // x4 per growth, and an unbounded round only follows a bounded one: 40 rounds are never reached
    if (round == 39) return fail(TG_ERR_CUDA, std::string("internal: ") + what + " failed to converge");
    unsigned long long used = 0, slots = 0;
    if (max_probe == kAggMaxProbe) TG_TRY(fill(used, slots));
    const bool room = max_probe == kAggMaxProbe && long_run_not_full(used, nd, slots);
    TG_TRY(grow(nd, room));
    max_probe = room ? (uint32_t)slots : kAggMaxProbe;
    only = bits[cur].as<uint32_t>();
    cur ^= 1;
  }
}

// one 8-byte counter back to the host (synchronises the stream)
static int read_back(AggImpl* a, const unsigned long long* counter, unsigned long long& v) {
  TG_CUDA(cudaMemcpyAsync(&v, counter, 8, cudaMemcpyDeviceToHost, a->stream));
  TG_CUDA(cudaStreamSynchronize(a->stream));
  return TG_OK;
}

// occupied slots of the group table, the NULL and sentinel groups included (k_agg_count; synchronises the stream)
static int table_used(AggImpl* a, unsigned long long* sc, unsigned long long& used) {
  TG_CUDA(cudaMemsetAsync(sc + SC_COUNT, 0, 8, a->stream));
  k_agg_count<<<grid_size(a->nsm, (int64_t)a->nslots + 2, 256, 8), 256, 0, a->stream>>>(a->tbl, sc + SC_COUNT);
  a->stats.kernel_launches++;
  return read_back(a, sc + SC_COUNT, used);
}

// grow_and_retry's fill and grow for the group table
static auto table_fill(AggImpl* a, unsigned long long* sc) {
  return [a, sc](unsigned long long& used, unsigned long long& slots) -> int { slots = a->nslots; return table_used(a, sc, used); };
}
static auto table_grow(AggImpl* a) {
  return [a](unsigned long long nd, bool room) -> int { return room ? TG_OK : grow_table(a, nd); };
}

// fold `m` partial-result tuples into the global table, growing it until every tuple found a slot
static int merge_partials(AggImpl* a, const AggPartials& pp, unsigned long long m, unsigned long long* sc) {
  if (m == 0) return TG_OK;
  DevBuf bits[2];
  return grow_and_retry(a, bits, (int64_t)m, false, "aggregation merge", [&](uint32_t* deferred, const uint32_t* only, uint32_t max_probe, unsigned long long& nd) -> int {
    TG_CUDA(cudaMemsetAsync(sc + SC_MERGE_DEFERRED, 0, 8, a->stream));
    (a->wide ? k_agg_merge<true> : k_agg_merge<false>)<<<grid_size(a->nsm, (int64_t)m, 256, 8), 256, 0, a->stream>>>(pp, (int64_t)m, a->nstates, a->tbl, a->spec, max_probe, deferred, only, sc + SC_MERGE_DEFERRED);
    a->stats.kernel_launches++;
    a->stats.paths |= TG_AGG_PATH_MERGE;
    return read_back(a, sc + SC_MERGE_DEFERRED, nd);
  }, table_fill(a, sc), table_grow(a));
}

// columnar partial-result tuples of `cap` entries in partials_mem: keys, rows, one array per state, kind
static int alloc_partials(AggImpl* a, size_t cap, unsigned long long* count, AggPartials& pp) {
  TG_TRY(a->partials_mem.ensure(a->device, cap * (8 + 8 + 8 * (size_t)a->nstates + 1) + 256));
  uint8_t* base = a->partials_mem.as<uint8_t>();
  pp.keys = reinterpret_cast<long long*>(base); base += cap * 8;
  pp.rows = reinterpret_cast<unsigned long long*>(base); base += cap * 8;
  for (int s = 0; s < a->nstates; s++) { pp.state[s] = reinterpret_cast<unsigned long long*>(base); base += cap * 8; }
  pp.kind = base;
  pp.count = count;
  return TG_OK;
}

// TG_AGG_LOCAL_SLOTS, the CTA-local table's slots for sweeps: 512, 1024, 2048 or 4096; 0 when unset or any other value
static int env_local_slots() {
  const int v = env_int("TG_AGG_LOCAL_SLOTS", 0);
  return (v == 512 || v == 1024 || v == 2048 || v == 4096) ? v : 0;
}

// several GROUP BY columns: global tag-claimed table only (k_agg_update_mk)
static int update_grouped_mk(AggImpl* a, const DevCols& cols, int64_t n, unsigned long long* sc) {
  GroupKeys gk{};
  gk.n = (int)a->group_cols.size(); gk.nkw = a->nkw;
  for (int q = 0; q < gk.n; q++) { gk.data[q] = cols.data[a->group_cols[q]]; gk.nulls[q] = cols.nulls[a->group_cols[q]]; gk.kind[q] = a->group_kinds[q]; }
  return grow_and_retry(a, a->deferred, n, false, "aggregation table", [&](uint32_t* deferred, const uint32_t* only, uint32_t max_probe, unsigned long long& nd) -> int {
    TG_CUDA(cudaMemsetAsync(sc + SC_DEFERRED, 0, 8, a->stream));
    (a->wide ? k_agg_update_mk<true> : k_agg_update_mk<false>)<<<grid_size(a->nsm, n, 256, 8), 256, 0, a->stream>>>(gk, cols, n, a->tbl, a->spec, max_probe, deferred, only, sc + SC_DEFERRED);
    a->stats.kernel_launches++;
    a->stats.paths |= TG_AGG_PATH_MULTI_KEY;
    return read_back(a, sc + SC_DEFERRED, nd);
  }, table_fill(a, sc), table_grow(a));
}

// Round-2 update path (agg_update.cuh): one two-level kernel per round; rows / local groups that found no slot are re-run
// after the table has grown.
static int update_grouped_v2(AggImpl* a, const GroupKey& gk, const DevCols& cols, int64_t n, unsigned long long* sc) {
  // CTA-local level: on for small / unknown cardinalities (a CTA turns it off by itself when its hit rate is low)
  const int env_local = env_int("TG_AGG_LOCAL", 1), env_slots = env_local_slots();
  bool local = env_local != 0 && a->nstates <= AGG_LOCAL_MAX_STATES && (a->expected_groups == 0 || a->expected_groups <= 4096);
  if (env_local == 2) local = a->nstates <= AGG_LOCAL_MAX_STATES;
  int local_slots = env_slots ? env_slots : 2048;
  size_t smem = (size_t)(local_slots + 2) * 8 * (2 + a->nstates);
  while (local && smem > (100u << 10) && local_slots > 512) { local_slots /= 2; smem = (size_t)(local_slots + 2) * 8 * (2 + a->nstates); }
  int per_sm = local ? (int)std::max<size_t>(1, std::min<size_t>(4, (200u << 10) / smem)) : 8;
  int grid = (int)std::min<int64_t>((n + AGG2_TILE - 1) / AGG2_TILE, (int64_t)a->nsm * per_sm);
  if (grid < 1) grid = 1;
  Agg2Params p{};
  p.gk = gk; p.n = n; p.max_probe = kAggMaxProbe; p.nstates = a->nstates; p.local_slots = local ? local_slots : 0;
  p.n_deferred = sc + SC_DEFERRED; p.local_rows = sc + SC_LOCAL_ROWS;
  if (local) {
    p.spill_cap = (unsigned long long)grid * (size_t)(local_slots + 2);
    TG_TRY(alloc_partials(a, (size_t)p.spill_cap, sc + SC_SPILLED, p.spill));
    TG_CUDA(cudaFuncSetAttribute(a->wide ? k_agg_update2<true, true> : k_agg_update2<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  // local groups of the first round that found no global slot (p.spill): they count as entries of the table's fill, the
  // table grows for them as well, then merges them; a table with room for them merges them after the last round
  unsigned long long spilled = 0;
  auto merge_spill = [&]() {
    const unsigned long long m = spilled;
    spilled = 0;
    return merge_partials(a, p.spill, m, sc);
  };
  auto fill = [&](unsigned long long& used, unsigned long long& slots) -> int {
    slots = a->nslots;
    TG_TRY(table_used(a, sc, used));
    used += spilled;
    return TG_OK;
  };
  auto grow = [&](unsigned long long nd, bool room) -> int {
    if (room) return TG_OK;
    TG_TRY(grow_table(a, nd + spilled));
    return merge_spill();
  };
  TG_TRY(grow_and_retry(a, a->deferred, n, false, "aggregation table", [&](uint32_t* deferred, const uint32_t* only, uint32_t max_probe, unsigned long long& nd) -> int {
    const bool lvl = local && !only;   // the CTA-local level runs in the first round
    TG_CUDA(cudaMemsetAsync(sc + SC_DEFERRED, 0, 8, a->stream));
    TG_CUDA(cudaMemsetAsync(sc + SC_SPILLED, 0, 8, a->stream));
    p.deferred = deferred; p.only = only; p.max_probe = max_probe;
    if (lvl) (a->wide ? k_agg_update2<true, true> : k_agg_update2<true, false>)<<<grid, AGG2_BLOCK, smem, a->stream>>>(p, cols, a->tbl, a->spec);
    else (a->wide ? k_agg_update2<false, true> : k_agg_update2<false, false>)<<<grid, AGG2_BLOCK, 0, a->stream>>>(p, cols, a->tbl, a->spec);
    a->stats.kernel_launches++;
    a->stats.paths |= lvl ? TG_AGG_PATH_V2_LOCAL : TG_AGG_PATH_V2_GLOBAL;
    unsigned long long back[8] = {0};
    TG_CUDA(cudaMemcpyAsync(back, sc, 64, cudaMemcpyDeviceToHost, a->stream));
    TG_CUDA(cudaStreamSynchronize(a->stream));
    a->stats.local_rows = (int64_t)back[SC_LOCAL_ROWS];
    nd = back[SC_DEFERRED];
    if (lvl) spilled = back[SC_SPILLED];
    if (spilled > p.spill_cap) return fail(TG_ERR_CUDA, "internal: aggregation spill buffer overflow");
    return TG_OK;
  }, fill, grow));
  if (spilled == 0) return TG_OK;
  unsigned long long used = 0;
  TG_TRY(table_used(a, sc, used));
  if (!long_run_not_full(used, spilled, a->nslots)) TG_TRY(grow_table(a, spilled));
  return merge_spill();
}

// rows [lo, hi): CTA-local partial aggregation, then merge of the partial results into the global table
static int local_partial_pass(AggImpl* a, const GroupKey& gk, const DevCols& cols, int64_t lo, int64_t hi, unsigned long long* sc) {
  const int env_slots = env_local_slots();
  const int local_slots = env_slots ? env_slots : 1024;   // bigger tables lose more to occupancy than they gain
  const size_t smem = (size_t)(local_slots + 2) * 8 * (2 + a->nstates);
  const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (200u << 10) / smem));
  const int grid = grid_size(a->nsm, hi - lo, 256, per_sm);
  AggPartials pp{};
  TG_TRY(alloc_partials(a, (size_t)grid * (local_slots / 2 + 2), sc + SC_V1_TUPLES, pp));
  TG_CUDA(cudaMemsetAsync(sc + SC_V1_TUPLES, 0, 8, a->stream));
  TG_CUDA(cudaFuncSetAttribute(a->wide ? k_agg_update_local<true> : k_agg_update_local<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  (a->wide ? k_agg_update_local<true> : k_agg_update_local<false>)<<<grid, 256, smem, a->stream>>>(gk, cols, lo, hi, a->spec, a->nstates, local_slots, pp, a->deferred[0].as<uint32_t>(), sc + SC_DEFERRED);
  a->stats.kernel_launches++;
  a->stats.paths |= TG_AGG_PATH_V1_LOCAL;
  unsigned long long m = 0;
  TG_TRY(read_back(a, sc + SC_V1_TUPLES, m));
  return merge_partials(a, pp, m, sc);
}

// Legacy update (TG_AGG_V1=1).  Phase 1 (low cardinality): CTA-local partial passes, decided on a 1M-row sample when there
// is no hint; phase 2: global atomics on every row, or on the rows phase 1 deferred, growing the table on demand.
static int update_grouped_v1(AggImpl* a, const GroupKey& gk, const DevCols& cols, int64_t n, unsigned long long* sc) {
  const bool try_local = a->nstates <= AGG_LOCAL_MAX_STATES && a->local_mode != 0 &&
                         (a->local_mode == 1 || a->expected_groups == 0 || a->expected_groups <= 2 * AGG_LOCAL_SLOTS_MAX);
  if (try_local) {
    const size_t bytes = (size_t)((n + 31) / 32) * 4;
    TG_TRY(a->deferred[0].ensure(a->device, bytes + 16));
    TG_CUDA(cudaMemsetAsync(a->deferred[0].p, 0, bytes, a->stream));
    TG_CUDA(cudaMemsetAsync(sc + SC_DEFERRED, 0, 8, a->stream));
    unsigned long long nd = 0;   // rows the passes so far deferred
    int64_t done = 0;
    while (done < n) {
      int64_t hi = (a->local_mode == 1) ? n : std::min<int64_t>(n, done + (1ll << 20));
      TG_TRY(local_partial_pass(a, gk, cols, done, hi, sc));
      TG_TRY(read_back(a, sc + SC_DEFERRED, nd));
      int64_t span = hi - done;
      done = hi;
      // Keep the CTA-local phase while it absorbs a useful share of the rows: shared-memory atomics (LSU) and L2 atomics
      // are different engines, so splitting the rows between them beats sending all of them to either one.
      if (a->local_mode < 0) a->local_mode = (nd * 10 <= (unsigned long long)span * 7) ? 1 : 0;
      if (a->local_mode == 0) break;
    }
    if (done < n) TG_TRY(mark_range_deferred(a, done, n));   // the rest of the batch goes through the global kernel
    else if (nd == 0) return TG_OK;
  }
  return grow_and_retry(a, a->deferred, n, try_local, "aggregation table", [&](uint32_t* deferred, const uint32_t* only, uint32_t max_probe, unsigned long long& nd) -> int {
    TG_CUDA(cudaMemsetAsync(sc + SC_DEFERRED, 0, 8, a->stream));
    (a->wide ? k_agg_update<true> : k_agg_update<false>)<<<grid_size(a->nsm, n, 256, 8), 256, 0, a->stream>>>(gk, cols, n, a->tbl, a->spec, max_probe, deferred, only, sc + SC_DEFERRED);
    a->stats.kernel_launches++;
    a->stats.paths |= TG_AGG_PATH_V1_GLOBAL;
    return read_back(a, sc + SC_DEFERRED, nd);
  }, table_fill(a, sc), table_grow(a));
}

// aggregate n device-resident rows
static int update_device_impl(AggImpl* a, const DevCols& cols, int64_t n) {
  if (n == 0) return TG_OK;
  a->stats.input_rows += n;
  TG_TRY(a->scalars.ensure(a->device, 64));
  unsigned long long* sc = a->scalars.as<unsigned long long>();
  a->spec.err = sc + SC_OVERFLOW;    // raised by a fused argument expression that left the DOUBLE range (types.ErrOverflow)
  if (a->nslots == 0) {
    unsigned long long want = 1024;
    if (a->group_col >= 0) {
      if (a->expected_groups > 0) want = std::max<unsigned long long>(1024, (unsigned long long)a->expected_groups * 2);
      else want = std::max<unsigned long long>(1024, (unsigned long long)std::min<int64_t>(n, 1ll << 22) * 2);
    }
    TG_CUDA(cudaMemsetAsync(sc, 0, 64, a->stream));
    TG_TRY(alloc_table(a, want, a->tbl_mem, a->tbl));
    a->nslots = want;
  }
  TG_CUDA(cudaEventRecord(a->ev0, a->stream));
  if (a->group_col < 0) {
    (a->wide ? k_agg_update_nogroup<true> : k_agg_update_nogroup<false>)<<<grid_size(a->nsm, n, 256, 4), 256, 0, a->stream>>>(cols, n, a->tbl, a->spec);
    a->stats.kernel_launches++;
    a->stats.paths |= TG_AGG_PATH_NOGROUP;
  } else if (a->nkw) {
    TG_TRY(update_grouped_mk(a, cols, n, sc));
  } else {
    const GroupKey gk{cols.data[a->group_col], cols.nulls[a->group_col], a->gk_kind, 0};
    TG_TRY(env_int("TG_AGG_V1", 0) ? update_grouped_v1(a, gk, cols, n, sc) : update_grouped_v2(a, gk, cols, n, sc));
  }
  TG_CUDA(cudaEventRecord(a->ev1, a->stream));
  TG_CUDA(cudaStreamSynchronize(a->stream));
  TG_CUDA(cudaGetLastError());
  a->stats.update_ms += a->elapsed_ms();
  return TG_OK;
}

// DECIMAL argument columns of the batch -> int64 scratch columns (k_dec_to_scaled), checked before any update kernel runs:
// a cell not in its column's stored form fails the push with the group table untouched.  One 8-byte read-back and one
// synchronisation per batch; the error word is scalars[SC_DEC_ERR], next to the overflow word of spec.err.
static int decode_decimal_args(AggImpl* a, DevCols& cols, int64_t n) {
  if (n == 0 || std::find(a->dec_decode.begin(), a->dec_decode.end(), 1) == a->dec_decode.end()) return TG_OK;
  TG_TRY(a->scalars.ensure(a->device, 72));
  unsigned long long* err = a->scalars.as<unsigned long long>() + SC_DEC_ERR;
  TG_CUDA(cudaMemsetAsync(err, 0, 8, a->stream));
  for (int c = 0; c < a->ncols; c++) {
    if (!a->dec_decode[c]) continue;
    TG_TRY(a->dscaled[c]->ensure(a->device, (size_t)n * 8 + 16));
    const uint8_t* cells = static_cast<const uint8_t*>(cols.data[c]);
    long long* out = a->dscaled[c]->as<long long>();
    const int grid = grid_size(a->nsm, (n + 1) / 2, 256, 8);
    if ((reinterpret_cast<uintptr_t>(cells) & 15) == 0)
      k_dec_to_scaled<true><<<grid, 256, 0, a->stream>>>(cells, cols.nulls[c], n, a->col_flen[c], a->col_dec[c], out, err, (unsigned long long)c + 1);
    else
      k_dec_to_scaled<false><<<grid, 256, 0, a->stream>>>(cells, cols.nulls[c], n, a->col_flen[c], a->col_dec[c], out, err, (unsigned long long)c + 1);
    a->stats.kernel_launches++;
    cols.data[c] = out;
    cols.elem_len[c] = 8;
  }
  unsigned long long e = 0;
  TG_CUDA(cudaMemcpyAsync(&e, err, 8, cudaMemcpyDeviceToHost, a->stream));
  TG_CUDA(cudaStreamSynchronize(a->stream));
  TG_CUDA(cudaGetLastError());
  if (e) {
    const int c = (int)e - 1;
    return fail(TG_ERR_INVALID, "DECIMAL(" + std::to_string(a->col_flen[c]) + ", " + std::to_string(a->col_dec[c]) + ") column " + std::to_string(c) +
                                ": a non-NULL cell is not in the column's stored form (digitsFrac must equal the scale, at most flen digits)");
  }
  return TG_OK;
}

// ---- DISTINCT sets ------------------------------------------------------------------------------------------------
// records of 2 words (tag, value) without GROUP BY, else padded to 32-byte multiples like the multi-key table's
static int set_record_words(int nkw) { return nkw == 1 ? 2 : ((1 + nkw + 3) / 4) * 4; }
static int alloc_set(AggImpl* a, unsigned long long nslots, DevBuf& mem, DistinctSet& t) {
  if (nslots >= (1ull << 32)) return fail(TG_ERR_OOM, "a DISTINCT set would need 2^32 slots or more");
  const int nkw = a->dist_gkw + 1, w = set_record_words(nkw);
  const size_t bytes = (size_t)nslots * w * 8 + 64;   // mk_find_or_insert reads 32 bytes from a 16-byte record's start
  TG_TRY(mem.ensure(a->device, bytes));
  TG_CUDA(cudaMemsetAsync(mem.p, 0, bytes, a->stream));   // tag 0 = empty
  unsigned long long* base = mem.as<unsigned long long>();
  t = DistinctSet{};
  t.tags = base;
  for (int j = 0; j < nkw; j++) t.keyw[j] = reinterpret_cast<long long*>(base + 1 + j);
  t.nslots = nslots; t.nkw = nkw; t.stride = (uint32_t)w;
  return TG_OK;
}
static int grow_set(AggImpl* a, AggImpl::SetMem& m, unsigned long long want) {
  DevBuf nm;
  DistinctSet nt{};
  TG_TRY(alloc_set(a, want, nm, nt));
  k_agg_distinct_rehash<<<grid_size(a->nsm, (int64_t)m.t.nslots, 256, 8), 256, 0, a->stream>>>(m.t, nt);
  a->stats.kernel_launches++;
  TG_CUDA(cudaStreamSynchronize(a->stream));
  std::swap(m.mem.p, nm.p); std::swap(m.mem.cap, nm.cap); std::swap(m.mem.device, nm.device);
  m.t = nt;
  a->dstats.set_grows++;
  return TG_OK;
}

// k_agg_distinct_mark for every DISTINCT argument column of the batch (after decode_decimal_args: a DECIMAL value is its
// int64 at the column's scale), then the virtual columns ncols + j point at the values and the mark bits.  A set is sized
// from its first batch like the group table and grows x4 through the same grow_and_retry.
static int distinct_mark(AggImpl* a, DevCols& cols, int64_t n) {
  if (a->dist_cols.empty() || n == 0) return TG_OK;
  TG_TRY(a->dcounters.ensure(a->device, 16));
  unsigned long long* cnt = a->dcounters.as<unsigned long long>();
  GroupKeys gk{};
  gk.n = (int)a->group_cols.size(); gk.nkw = a->dist_gkw;
  for (int q = 0; q < gk.n; q++) { gk.data[q] = cols.data[a->group_cols[q]]; gk.nulls[q] = cols.nulls[a->group_cols[q]]; gk.kind[q] = a->group_kinds[q]; }
  TG_CUDA(cudaEventRecord(a->ev0, a->stream));
  for (size_t j = 0; j < a->dist_cols.size(); j++) {
    AggImpl::SetMem& m = *a->dsets[j];
    const int c = a->dist_cols[j];
    if (m.t.nslots == 0) TG_TRY(alloc_set(a, std::max<unsigned long long>(1024, (unsigned long long)std::min<int64_t>(n, 1ll << 22) * 2), m.mem, m.t));
    TG_TRY(m.mark.ensure(a->device, (size_t)((n + 31) / 32) * 4 + 16));
    TG_TRY(grow_and_retry(a, a->deferred, n, false, "DISTINCT set", [&](uint32_t* deferred, const uint32_t* only, uint32_t max_probe, unsigned long long& nd) -> int {
      TG_CUDA(cudaMemsetAsync(cnt, 0, 16, a->stream));
      k_agg_distinct_mark<<<grid_size(a->nsm, n, 256, 8), 256, 0, a->stream>>>(gk, static_cast<const long long*>(cols.data[c]), cols.nulls[c],
                                                               a->types[c] == TG_TYPE_DOUBLE, n, m.t, max_probe, m.mark.as<uint32_t>(),
                                                               deferred, only, cnt);
      a->stats.kernel_launches++;
      a->dstats.launches++;
      unsigned long long back[2] = {0, 0};
      TG_CUDA(cudaMemcpyAsync(back, cnt, 16, cudaMemcpyDeviceToHost, a->stream));
      TG_CUDA(cudaStreamSynchronize(a->stream));
      a->dstats.pairs += (int64_t)back[1];
      m.used += back[1];
      nd = back[0];
      return TG_OK;
    }, [&](unsigned long long& used, unsigned long long& slots) -> int { used = m.used; slots = m.t.nslots; return TG_OK; },
    [&](unsigned long long nd, bool room) -> int { return room ? TG_OK : grow_set(a, m, grown_slots(m.t.nslots, nd)); }));
    cols.data[a->ncols + j] = cols.data[c];
    cols.nulls[a->ncols + j] = m.mark.as<uint8_t>();
    cols.elem_len[a->ncols + j] = 8;
  }
  TG_CUDA(cudaEventRecord(a->ev1, a->stream));
  TG_CUDA(cudaStreamSynchronize(a->stream));
  TG_CUDA(cudaGetLastError());
  a->dstats.mark_ms += a->elapsed_ms();
  return TG_OK;
}

static int update_after_decode(AggImpl* a, DevCols& cols, int64_t n) {
  TG_TRY(distinct_mark(a, cols, n));
  TG_TRY(update_device_impl(a, cols, n));
  bool has_expr = false;
  for (int k = 0; k < a->spec.n; k++) has_expr |= a->spec.f[k].arg_expr != TG_ARGEXPR_COL;
  if (!has_expr || n == 0) return TG_OK;
  unsigned long long e = 0;
  TG_CUDA(cudaMemcpyAsync(&e, a->scalars.as<unsigned long long>() + SC_OVERFLOW, 8, cudaMemcpyDeviceToHost, a->stream));
  TG_CUDA(cudaStreamSynchronize(a->stream));
  if (e) return fail(TG_ERR_OVERFLOW, "ErrOverflow: DOUBLE value is out of range in an aggregate argument expression");
  return TG_OK;
}

static int broken_fail() {
  return fail(TG_ERR_STATE, "an earlier push failed after the DISTINCT sets or string dictionaries had taken its values: this handle's results are lost");
}

// every string GROUP BY column of the batch -> its dictionary's ids (str_dict.cuh), through the grow-and-retry of the
// other find-or-insert passes; then the id column, with the column's own NULL bitmap, stands in for the string column.
// Row i of the batch has the ordinal str_ords + i, so a key's earliest row is the first in push order.
static int encode_strings(AggImpl* a, DevCols& cols, const StrColDev* sv, int64_t n, bool& touched) {
  if (a->dicts.empty() || n == 0) return TG_OK;
  if ((unsigned long long)(a->str_ords + n) >> (64 - kTailBits))
    return fail(TG_ERR_UNSUPPORTED, "a string-key aggregation is offloaded for fewer than 2^41 input rows");
  TG_CUDA(cudaEventRecord(a->ev0, a->stream));
  for (int c = 0; c < a->ncols; c++) {
    const int j = a->dict_of[c];
    if (j < 0) continue;
    StrDict& d = *a->dicts[j];
    TG_TRY(str_dict_prepare(d, a->device, n, a->expected_groups, a->stream));
    TG_TRY(a->sids[c]->ensure(a->device, (size_t)n * 8 + 16));
    long long* ids = a->sids[c]->as<long long>();
    unsigned long long* tails = nullptr;
    if (a->tail_col[c] >= 0) { TG_TRY(a->stails[c]->ensure(a->device, (size_t)n * 8 + 16)); tails = a->stails[c]->as<unsigned long long>(); }
    touched = true;   // from the first round on, the dictionary may hold entries of this batch
    TG_TRY(grow_and_retry(a, a->deferred, n, false, "string dictionary", [&](uint32_t* deferred, const uint32_t* only, uint32_t max_probe, unsigned long long& nd) -> int {
      a->stats.kernel_launches++;
      return str_dict_round(d, sv[c], n, a->str_ords, max_probe, ids, deferred, only, nd, tails, a->nsm, a->stream);
    }, [&](unsigned long long& used, unsigned long long& slots) -> int { slots = d.nslots; return str_dict_used(d, used, a->stream); },
    [&](unsigned long long nd, bool room) -> int { return str_dict_grow(d, nd, room, a->device, a->nsm, a->stream); }));
    if (tails) {
      bool wide = false;
      TG_TRY(str_dict_tail_overflow(d, wide, a->stream));
      if (wide) return fail(TG_ERR_UNSUPPORTED, "a string GROUP BY value with 2^23 or more trailing spaces under a PAD collation, whose FIRSTROW is asked with several GROUP BY columns");
      cols.data[a->tail_col[c]] = tails;
      cols.nulls[a->tail_col[c]] = nullptr;
      cols.elem_len[a->tail_col[c]] = 8;
    }
    TG_TRY(str_dict_commit(d, sv[c], ids, n, a->str_ords, a->device, a->nsm, a->stream));
    cols.data[c] = ids;
    cols.elem_len[c] = 8;
  }
  a->str_ords += n;
  a->stats.paths |= TG_AGG_PATH_STRING_KEY;
  TG_CUDA(cudaEventRecord(a->ev1, a->stream));
  TG_CUDA(cudaStreamSynchronize(a->stream));
  TG_CUDA(cudaGetLastError());
  a->encode_ms += a->elapsed_ms();
  return TG_OK;
}

// aggregate n device-resident rows (sv: the string columns, by child column; nullptr without any); a fused argument
// expression that overflowed fails the call (types.ErrOverflow).  A bad DECIMAL cell fails the push before the
// dictionaries and the DISTINCT sets see it; a failure once a dictionary round has run, or any later one with DISTINCT
// sets, leaves a dictionary or a set holding values whose rows were not aggregated, so the handle refuses every later
// push and finish instead of counting them twice or never.
static int update_device(AggImpl* a, const DevCols& in, const StrColDev* sv, int64_t n) {
  if (a->broken) return broken_fail();
  DevCols cols = in;
  TG_TRY(decode_decimal_args(a, cols, n));
  bool touched = false;
  int rc = encode_strings(a, cols, sv, n, touched);
  if (rc == TG_OK) rc = update_after_decode(a, cols, n);
  if (rc != TG_OK && (!a->dist_cols.empty() || touched)) a->broken = true;
  return rc;
}

static int aflush(AggImpl* a) {
  HostStage& st = a->stage;
  if (st.rows == 0) return TG_OK;
  DevCols v{};
  StrColDev sv[TG_MAX_COLS] = {};
  for (int c = 0; c < a->ncols; c++) {
    v.elem_len[c] = a->elem[c];
    if (!a->needed[c]) continue;
    if (a->is_str[c]) {   // staged offsets (from 0) and bytes
      TG_TRY(a->doffs[c]->ensure(a->device, (size_t)(st.rows + 1) * 8 + 16));
      TG_CUDA(cudaMemcpyAsync(a->doffs[c]->p, st.offs[c]->p, (size_t)(st.rows + 1) * 8, cudaMemcpyHostToDevice, a->stream));
      TG_TRY(upload_column(a->device, a->stream, st.data[c]->p, nullptr, (int64_t)st.data[c]->used, 1, *a->dcols[c], *a->dnulls[c],
                           &a->stats.h2d_bytes));
      a->stats.h2d_bytes += (st.rows + 1) * 8;
      if (st.has_nulls[c]) {
        const size_t nb = (size_t)((st.rows + 7) / 8);
        TG_TRY(a->dnulls[c]->ensure(a->device, nb + 16));
        if (nb) TG_CUDA(cudaMemcpyAsync(a->dnulls[c]->p, st.nulls[c]->p, nb, cudaMemcpyHostToDevice, a->stream));
        a->stats.h2d_bytes += (int64_t)nb;
      }
      v.data[c] = a->dcols[c]->p;
      if (st.has_nulls[c]) v.nulls[c] = a->dnulls[c]->as<uint8_t>();
      sv[c] = StrColDev{a->doffs[c]->as<int64_t>(), a->dcols[c]->as<uint8_t>(), 0, v.nulls[c]};
      continue;
    }
    TG_TRY(upload_column(a->device, a->stream, st.data[c]->p, st.has_nulls[c] ? st.nulls[c]->p : nullptr, st.rows, a->elem[c],
                         *a->dcols[c], *a->dnulls[c], &a->stats.h2d_bytes));
    v.data[c] = a->dcols[c]->p;
    if (st.has_nulls[c]) v.nulls[c] = a->dnulls[c]->as<uint8_t>();
  }
  int rc = update_device(a, v, sv, st.rows);
  st.reset();
  return rc;
}

static int afinalize(AggImpl* a) {
  TG_TRY(a->scalars.ensure(a->device, 64));
  unsigned long long* sc = a->scalars.as<unsigned long long>();
  int nf = a->spec.n;
  a->out_cols.clear(); a->out_valid.clear(); a->out_bitmaps.clear();
  for (int k = 0; k < nf; k++) { a->out_cols.emplace_back(new DevBuf()); a->out_valid.emplace_back(new DevBuf()); a->out_bitmaps.emplace_back(new DevBuf()); }
  // agg_hash_executor.go:654: empty input and no GROUP BY → one row of default values (COUNT 0, rest NULL)
  bool default_row = a->stats.input_rows == 0 && a->group_col < 0;
  if (a->nslots == 0) {
    if (!default_row) {   // no input rows: no groups, and a string result has the one offset 0
      a->out_rows = 0;
      for (int k = 0; k < nf; k++) {
        if (a->out_dict[k] < 0) continue;
        TG_TRY(a->out_soffs[k]->ensure(a->device, 16));
        TG_TRY(a->out_sbytes[k]->ensure(a->device, 16));
        TG_CUDA(cudaMemsetAsync(a->out_soffs[k]->p, 0, 8, a->stream));
        a->host_soffs[k].assign(1, 0);
      }
      TG_CUDA(cudaStreamSynchronize(a->stream));
      return TG_OK;
    }
    TG_CUDA(cudaMemsetAsync(sc, 0, 64, a->stream));
    TG_TRY(alloc_table(a, 1024, a->tbl_mem, a->tbl));
    a->nslots = 1024;
  }
  unsigned long long fill = 0;
  TG_TRY(table_used(a, sc, fill));
  int64_t cap = (int64_t)fill + 2 + 1;
  AggOut ao{};
  for (int k = 0; k < nf; k++) {
    TG_TRY(a->out_cols[k]->ensure(a->device, (size_t)cap * a->out_elem[k] + 16));
    ao.data[k] = a->out_cols[k]->p;
    ao.valid[k] = nullptr;
    if (a->out_nullable[k] || default_row) { TG_TRY(a->out_valid[k]->ensure(a->device, (size_t)cap + 16)); ao.valid[k] = a->out_valid[k]->as<uint8_t>(); }
  }
  TG_CUDA(cudaEventRecord(a->ev0, a->stream));
  TG_CUDA(cudaMemsetAsync(sc + SC_CURSOR, 0, 8, a->stream));
  (a->wide ? k_agg_finalize<true, true> : a->dec_out ? k_agg_finalize<true, false> : k_agg_finalize<false, false>)<<<grid_size(a->nsm, (int64_t)a->nslots + 2, 256, 8), 256, 0, a->stream>>>(a->tbl, a->spec, a->gk_kind, ao, sc + SC_CURSOR);
  a->stats.kernel_launches++;
  unsigned long long nrows = 0;
  TG_CUDA(cudaMemcpyAsync(&nrows, sc + SC_CURSOR, 8, cudaMemcpyDeviceToHost, a->stream));
  TG_CUDA(cudaStreamSynchronize(a->stream));
  if (default_row && nrows == 0) {
    // write the default row on the host side: COUNT → 0, everything else NULL
    for (int k = 0; k < nf; k++) {
      uint8_t v = a->spec.f[k].name == TG_AGG_COUNT ? 1 : 0;
      TG_CUDA(cudaMemsetAsync(a->out_cols[k]->p, 0, (size_t)a->out_elem[k], a->stream));
      TG_CUDA(cudaMemcpyAsync(a->out_valid[k]->p, &v, 1, cudaMemcpyHostToDevice, a->stream));
      TG_CUDA(cudaStreamSynchronize(a->stream));
    }
    nrows = 1;
  }
  a->out_rows = (int64_t)nrows;
  a->stats.groups = a->out_rows;
  a->stats.table_slots = (int64_t)a->nslots;
  for (int k = 0; k < nf; k++) {
    if (!ao.valid[k]) continue;
    TG_TRY(a->out_bitmaps[k]->ensure(a->device, (size_t)((a->out_rows + 7) / 8) + 16));
    if (a->out_rows) { launch_pack_bitmap(ao.valid[k], a->out_rows, a->out_bitmaps[k]->as<uint8_t>(), a->nsm, a->stream); a->stats.kernel_launches++; }
  }
  // string results: the ids k_agg_finalize wrote -> offsets and bytes from the dictionary, the offsets also on the host
  for (int k = 0; k < nf; k++) {
    const int j = a->out_dict[k];
    if (j < 0) continue;
    int64_t total = 0;
    const unsigned long long* tails = a->tail_fn[k] >= 0 ? a->out_cols[a->tail_fn[k]]->as<unsigned long long>() : nullptr;
    TG_TRY(str_dict_gather(*a->dicts[j], a->out_cols[k]->as<long long>(), ao.valid[k], tails, a->out_rows, *a->out_soffs[k], *a->out_sbytes[k],
                           &total, a->device, a->nsm, a->stream));
    a->stats.kernel_launches += 5;
    a->host_soffs[k].assign((size_t)a->out_rows + 1, 0);
    TG_CUDA(cudaMemcpyAsync(a->host_soffs[k].data(), a->out_soffs[k]->p, (size_t)(a->out_rows + 1) * 8, cudaMemcpyDeviceToHost, a->stream));
  }
  TG_CUDA(cudaEventRecord(a->ev1, a->stream));
  TG_CUDA(cudaStreamSynchronize(a->stream));
  TG_CUDA(cudaGetLastError());
  a->stats.finalize_ms += a->elapsed_ms();
  return TG_OK;
}

// every descriptor version as a tg_agg_desc_ex3 whose arrays that version lacks are NULL
static tg_agg_desc_ex3 ex3_view(const tg_agg_desc& d) { tg_agg_desc_ex3 v{}; v.ex2.ex.base = d; return v; }
static tg_agg_desc_ex3 ex3_view(const tg_agg_desc_ex& d) { tg_agg_desc_ex3 v{}; v.ex2.ex = d; return v; }
static tg_agg_desc_ex3 ex3_view(const tg_agg_desc_ex2& d) { tg_agg_desc_ex3 v{}; v.ex2 = d; return v; }
static tg_agg_desc_ex3 ex3_view(const tg_agg_desc_ex3& d) { return d; }

template <class Desc> static int agg_supported(const Desc* desc) {
  if (!desc) return fail(TG_ERR_INVALID, "desc is NULL");
  AggPlan p;
  return agg_compile(&p, ex3_view(*desc));
}

template <class Desc> static int agg_open(const Desc* desc, tg_agg** out) {
  if (!out) return fail(TG_ERR_INVALID, "out is NULL");
  *out = nullptr;
  if (!desc) return fail(TG_ERR_INVALID, "desc is NULL");
  const tg_agg_desc_ex3 d = ex3_view(*desc);
  std::unique_ptr<tg_agg> shell(new tg_agg());
  std::unique_ptr<AggImpl> a(new AggImpl());
  TG_TRY(agg_compile(a.get(), d));
  a->device = d.ex2.ex.base.device;
  a->expected_groups = d.ex2.ex.base.expected_groups;
  int ndev = 0;
  TG_TRY(require_device("the GPU hash aggregation", &ndev));
  if (a->device < 0 || a->device >= ndev) return fail(TG_ERR_INVALID, "device ordinal out of range");
  DeviceGuard g(a->device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed");
  TG_TRY(a->open(a->device, d.ex2.ex.base.stream));
  a->stage.init(a->ncols);
  for (int c = 0; c < a->ncols; c++) {
    a->dcols.emplace_back(new DevBuf()); a->dnulls.emplace_back(new DevBuf()); a->dscaled.emplace_back(new DevBuf());
    a->sids.emplace_back(new DevBuf()); a->doffs.emplace_back(new DevBuf()); a->stails.emplace_back(new DevBuf());
    if (a->dict_of[c] >= 0) { a->dicts.emplace_back(new StrDict()); a->dicts.back()->coll = a->coll[c]; }
  }
  for (int k = 0; k < a->spec.n; k++) { a->out_soffs.emplace_back(new DevBuf()); a->out_sbytes.emplace_back(new DevBuf()); }
  a->host_soffs.resize(a->spec.n);
  for (size_t j = 0; j < a->dist_cols.size(); j++) a->dsets.emplace_back(new AggImpl::SetMem());
  shell->impl = a.release();
  *out = shell.release();
  return TG_OK;
}

}  // namespace tg

extern "C" {

int tg_agg_supported(const tg_agg_desc* desc) { return agg_supported(desc); }
int tg_agg_supported_ex(const tg_agg_desc_ex* desc) { return agg_supported(desc); }
int tg_agg_supported_ex2(const tg_agg_desc_ex2* desc) { return agg_supported(desc); }
int tg_agg_supported_ex3(const tg_agg_desc_ex3* desc) { return agg_supported(desc); }
int tg_agg_open(const tg_agg_desc* desc, tg_agg** out) { return agg_open(desc, out); }
int tg_agg_open_ex(const tg_agg_desc_ex* desc, tg_agg** out) { return agg_open(desc, out); }
int tg_agg_open_ex2(const tg_agg_desc_ex2* desc, tg_agg** out) { return agg_open(desc, out); }
int tg_agg_open_ex3(const tg_agg_desc_ex3* desc, tg_agg** out) { return agg_open(desc, out); }

int tg_agg_push(tg_agg* h, const tg_chunk* chk) {
  TG_LOCK(h, AggImpl, a);
  if (a->finished) return fail(TG_ERR_STATE, "push after finish");
  if (a->broken) return broken_fail();
  TG_TRY(validate_chunk(a->ncols, a->needed_fixed, a->elem, chk));
  // string columns: every row's offsets are checked before anything is staged (staging copies the rows' bytes)
  const int64_t phys = chk->ncols ? chk->cols[0].length : 0;
  for (int c = 0; c < a->ncols; c++) {
    if (!a->is_str[c]) continue;
    TG_TRY(check_varlen_rows(chk->cols[c], chk));
    if (chk->cols[c].length != phys) return fail(TG_ERR_INVALID, "chunk columns have different lengths");
  }
  TG_TRY(stage_append(a->stage, a->needed, a->elem, chk));
  if (a->stage.rows >= kStageBatchRows) TG_TRY(aflush(a));
  return TG_OK;
}

int tg_agg_push_dev(tg_agg* h, const tg_chunk* chk) {
  TG_LOCK(h, AggImpl, a);
  if (a->finished) return fail(TG_ERR_STATE, "push after finish");
  DevCols v;
  TG_TRY(device_view(chk, a->ncols, a->needed_fixed, a->elem, v));
  const int64_t n = logical_rows(chk);
  StrColDev sv[TG_MAX_COLS] = {};
  bool any_str = false;
  for (int c = 0; c < a->ncols; c++) {
    if (!a->is_str[c]) continue;
    const tg_column& col = chk->cols[c];
    if (col.elem_len != -1 || !col.offsets) return fail(TG_ERR_INVALID, "a string column is var-length: elem_len -1 and offsets");
    if (col.length != n) return fail(TG_ERR_INVALID, "chunk columns have different lengths");
    if (reinterpret_cast<uintptr_t>(col.offsets) & 7) return fail(TG_ERR_INVALID, "device string offsets must be 8-byte aligned");
    v.data[c] = col.data; v.nulls[c] = col.null_bitmap;
    sv[c] = StrColDev{col.offsets, col.data, 0, col.null_bitmap};
    any_str = true;
  }
  if (any_str && n > 0) {   // every row's offsets, on the device, before a dictionary sees the batch
    TG_TRY(a->sflag.ensure(a->device, 16));
    TG_CUDA(cudaMemsetAsync(a->sflag.p, 0, 4, a->stream));
    for (int c = 0; c < a->ncols; c++)
      if (a->is_str[c]) { str_check_offsets(sv[c].offs, sv[c].data, n, a->sflag.as<unsigned int>(), a->nsm, a->stream); a->stats.kernel_launches++; }
    unsigned int bad = 0;
    TG_CUDA(cudaMemcpyAsync(&bad, a->sflag.p, 4, cudaMemcpyDeviceToHost, a->stream));
    TG_CUDA(cudaStreamSynchronize(a->stream));
    TG_CUDA(cudaGetLastError());
    if (bad) return fail(TG_ERR_INVALID, "a string column has a row with bad offsets (offsets[r] > offsets[r+1], or outside [offsets[0], offsets[length]])");
  }
  TG_TRY(aflush(a));
  return update_device(a, v, sv, n);
}

int tg_agg_finish(tg_agg* h) {
  TG_LOCK(h, AggImpl, a);
  if (a->finished) return TG_OK;
  if (a->broken) return broken_fail();
  TG_TRY(aflush(a));
  TG_TRY(afinalize(a));
  a->finished = true;
  return TG_OK;
}

static bool has_string_result(const AggImpl* a) {
  return std::find_if(a->out_dict.begin(), a->out_dict.end(), [](int j) { return j >= 0; }) != a->out_dict.end();
}

// tg_agg_next (ex false, var_out NULL: a plan with a string result is refused) and tg_agg_next_ex
static int agg_next(tg_agg* h, tg_mut_chunk* out, tg_mut_varlen* var_out, int64_t max_rows, int64_t* nrows, bool ex) {
  TG_LOCK(h, AggImpl, a);
  const bool str = has_string_result(a);
  if (!out || !nrows || (str && ex && !var_out)) return fail(TG_ERR_INVALID, str && ex ? "out / var_out / nrows is NULL" : "out / nrows is NULL");
  if (str && !ex) return fail(TG_ERR_INVALID, "the plan has a string result: read it with tg_agg_next_ex");
  *nrows = 0;
  if (!a->finished) return fail(TG_ERR_STATE, "next before finish (hash aggregation is a pipeline breaker)");
  if (out->ncols != a->n_out) return fail(TG_ERR_INVALID, "output chunk column count does not match the aggregate list");
  const int64_t lo = a->consumed;
  int64_t want = std::min<int64_t>(std::min<int64_t>(max_rows, out->capacity_rows), a->out_rows - lo);
  if (want <= 0) return TG_OK;
  // every output column is checked before the first copy is enqueued: a rejected call writes nothing
  if (!str) TG_TRY(check_out_columns(a->out_bitmaps, a->out_elem, out));
  for (int k = 0; str && k < a->n_out; k++) {
    const bool sk = a->out_dict[k] >= 0;
    if (out->cols[k].elem_len != (sk ? -1 : a->out_elem[k]))
      return fail(TG_ERR_INVALID, "output column elem_len does not match its result column (-1 for a string result, 40 for a DECIMAL one, else 8)");
    if (a->out_bitmaps[k]->p && !out->cols[k].null_bitmap) return fail(TG_ERR_INVALID, "output column can be NULL but the caller passed no null bitmap");
    if (!sk) continue;
    const tg_mut_varlen& vo = var_out[k];
    if (!vo.offsets || (vo.data_cap > 0 && !vo.data) || vo.data_cap < 0) return fail(TG_ERR_INVALID, "a string result needs offsets and data_cap bytes of data");
    // the largest prefix of rows whose bytes fit data_cap
    const int64_t* ho = a->host_soffs[k].data() + lo;
    want = std::min<int64_t>(want, std::upper_bound(ho, ho + want + 1, ho[0] + vo.data_cap) - ho - 1);
  }
  if (want <= 0) return fail(TG_ERR_CAPACITY, "the next result row's string bytes do not fit data_cap");
  for (int k = 0; k < a->n_out; k++) {
    if (a->out_dict[k] >= 0) {
      const int64_t* ho = a->host_soffs[k].data() + lo;
      const int64_t bytes = ho[want] - ho[0];
      if (bytes) TG_CUDA(cudaMemcpyAsync(var_out[k].data, a->out_sbytes[k]->as<uint8_t>() + ho[0], (size_t)bytes, cudaMemcpyDeviceToHost, a->stream));
      for (int64_t r = 0; r <= want; r++) var_out[k].offsets[r] = ho[r] - ho[0];
      a->stats.d2h_bytes += bytes + (want + 1) * 8;
      continue;
    }
    const size_t el = (size_t)a->out_elem[k];
    TG_CUDA(cudaMemcpyAsync(out->cols[k].data, a->out_cols[k]->as<uint8_t>() + (size_t)lo * el, (size_t)want * el, cudaMemcpyDeviceToHost, a->stream));
    a->stats.d2h_bytes += want * (int64_t)el;
  }
  // any RequiredRows >= 1 is served (download_bitmaps re-aligns bitmaps that start inside a byte); d2h_bytes counts the
  // result cells only
  TG_TRY(download_bitmaps(a->out_bitmaps, out, lo, want, a->stream, nullptr));
  a->consumed += want;
  *nrows = want;
  return TG_OK;
}

// tg_agg_result_dev (ex false: a plan with a string result is refused) and tg_agg_result_dev_ex
static int agg_result_dev(tg_agg* h, int64_t* out_rows, void** out_cols, void** out_nulls, void** out_offsets, bool ex) {
  TG_LOCK(h, AggImpl, a);
  if (!ex && has_string_result(a)) return fail(TG_ERR_INVALID, "the plan has a string result: read it with tg_agg_result_dev_ex");
  if (!a->finished) return fail(TG_ERR_STATE, "result before finish");
  if (out_rows) *out_rows = a->out_rows;
  for (int k = 0; k < a->n_out; k++) {
    const bool str = a->out_dict[k] >= 0;
    if (out_cols) out_cols[k] = str ? a->out_sbytes[k]->p : a->out_cols[k]->p;
    if (out_nulls) out_nulls[k] = a->out_bitmaps[k]->p;
    if (out_offsets) out_offsets[k] = str ? a->out_soffs[k]->p : nullptr;
  }
  return TG_OK;
}

int tg_agg_next(tg_agg* h, tg_mut_chunk* out, int64_t max_rows, int64_t* nrows) { return agg_next(h, out, nullptr, max_rows, nrows, false); }

int tg_agg_next_ex(tg_agg* h, tg_mut_chunk* out, tg_mut_varlen* var_out, int64_t max_rows, int64_t* nrows) {
  return agg_next(h, out, var_out, max_rows, nrows, true);
}

int tg_agg_result_dev(tg_agg* h, int64_t* out_rows, void** out_cols, void** out_nulls) {
  return agg_result_dev(h, out_rows, out_cols, out_nulls, nullptr, false);
}

int tg_agg_result_dev_ex(tg_agg* h, int64_t* out_rows, void** out_cols, void** out_nulls, void** out_offsets) {
  return agg_result_dev(h, out_rows, out_cols, out_nulls, out_offsets, true);
}

int tg_agg_get_string_stats(tg_agg* h, tg_agg_string_stats* out) {
  TG_LOCK(h, AggImpl, a);
  if (!out) return fail(TG_ERR_INVALID, "out is NULL");
  *out = tg_agg_string_stats{};
  for (const auto& d : a->dicts) {
    out->dict_entries += d->entries;
    out->dict_bytes += (int64_t)d->arena_used;
    out->dict_slots += (int64_t)d->nslots;
    out->dict_grows += d->grows;
    out->launches += d->launches;
  }
  out->encode_ms = a->encode_ms;
  return TG_OK;
}

int tg_agg_get_stats(tg_agg* h, tg_agg_stats* out) {
  TG_LOCK(h, AggImpl, a);
  if (!out) return fail(TG_ERR_INVALID, "out is NULL");
  *out = a->stats;
  return TG_OK;
}

int tg_agg_get_distinct_stats(tg_agg* h, tg_agg_distinct_stats* out) {
  TG_LOCK(h, AggImpl, a);
  if (!out) return fail(TG_ERR_INVALID, "out is NULL");
  *out = a->dstats;
  out->set_slots = 0;
  for (const auto& m : a->dsets) out->set_slots += (int64_t)m->t.nslots;
  return TG_OK;
}

int tg_agg_close(tg_agg* h) {
  if (!h) return TG_OK;
  bool was = h->closed.exchange(true);
  if (was) return TG_OK;
  {
    std::lock_guard<std::mutex> lock(h->mu);   // waits for an in-flight call; later calls see `closed`
    AggImpl* a = h->impl;
    h->impl = nullptr;
    if (a) {
      DeviceGuard g(a->device);
      a->release();
      cudaGetLastError();
      delete a;
    }
  }
  bury_handle(h);
  return TG_OK;
}

}  // extern "C"
