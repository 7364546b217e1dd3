// oracle/vec.cpp — row-at-a-time restatement of the VecEval* builtins on the path (TEST
// INFRASTRUCTURE, see oracle.h) plus helpers shared by join.cpp / agg.cpp.
//
// Follows the reference's pkg/expression:
//   builtin_compare_vec.go  builtinLTIntSig.vecEvalInt :524-561, vecCompareInt :619
//   builtin_compare_vec_generated.go :54 (real compare through cmp.Compare)
//   builtin_arithmetic_vec.go  PlusInt :856-990 (plusUU/US/SU/SS), MinusInt :365-411 with
//       overflowCheck builtin_arithmetic.go:491-535, MultiplyInt :646-679, MultiplyIntUnsigned :1011,
//       PlusReal :496-523, MinusReal :300-322, MultiplyReal :40-62
//   chunk_executor.go VectorizedFilter :413, expression.go VecEvalBool :409-494, toBool :496
//   pkg/types/compare.go CompareInt :86
//   pkg/util/chunk/column.go MergeNulls :906
#include <mutex>
#include <limits>
#include "common.hpp"

namespace orc {

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }

int compare_int(int64_t a, bool ua, int64_t b, bool ub) {
  auto cmp_u = [](uint64_t x, uint64_t y) { return x < y ? -1 : (x == y ? 0 : 1); };
  auto cmp_s = [](int64_t x, int64_t y) { return x < y ? -1 : (x == y ? 0 : 1); };
  if (ua && ub) return cmp_u((uint64_t)a, (uint64_t)b);
  if (ua && !ub) { if (b < 0 || (uint64_t)a > (uint64_t)INT64_MAX) return 1; return cmp_s(a, b); }
  if (!ua && ub) { if (a < 0 || (uint64_t)b > (uint64_t)INT64_MAX) return -1; return cmp_s(a, b); }
  return cmp_s(a, b);
}

// Go cmp.Compare(float64): NaN is less than any non-NaN, NaN == NaN
int compare_real(double a, double b) {
  bool an = std::isnan(a), bn = std::isnan(b);
  if (an) return bn ? 0 : -1;
  if (bn) return 1;
  return a < b ? -1 : (a > b ? 1 : 0);
}

static inline bool apply_cmp(int op, int c) {
  switch (op) {
    case TG_CMP_LT: return c < 0;
    case TG_CMP_LE: return c <= 0;
    case TG_CMP_GT: return c > 0;
    case TG_CMP_GE: return c >= 0;
    case TG_CMP_EQ: return c == 0;
    default: return c != 0;
  }
}

// one CNF item on one physical row: returns -1 NULL, 0 false, 1 true
static int eval_item(const tg_chunk& chk, int64_t p, const tg_filter_item& it) {
  const tg_column& a = chk.cols[it.lhs_col];
  if (col_is_null(a, p)) return -1;
  if (it.rhs_col >= 0 && col_is_null(chk.cols[it.rhs_col], p)) return -1;
  int c;
  if (it.is_real) {
    double y = it.rhs_col >= 0 ? col_f64(chk.cols[it.rhs_col], p) : it.const_f64;
    c = compare_real(col_f64(a, p), y);
  } else {
    int64_t y = it.rhs_col >= 0 ? col_i64(chk.cols[it.rhs_col], p) : it.const_i64;
    c = compare_int(col_i64(a, p), it.lhs_unsigned != 0, y, it.rhs_unsigned != 0);
  }
  return apply_cmp(it.op, c) ? 1 : 0;
}

bool filter_row(const tg_chunk& chk, int64_t p, const tg_filter_item* items, int n) {
  for (int i = 0; i < n; i++) if (eval_item(chk, p, items[i]) != 1) return false;
  return true;
}

int fetch_result(const std::vector<std::vector<OColumn>*>& parts, int ncols, tg_mut_chunk* out) {
  if (out->ncols != ncols) { set_error("fetch: column count mismatch"); return TG_ERR_INVALID; }
  int64_t total = 0;
  for (auto* p : parts) if (!p->empty()) total += (*p)[0].length;
  if (total > out->capacity_rows) { set_error("fetch: capacity too small"); return TG_ERR_CAPACITY; }
  for (int c = 0; c < ncols; c++) {
    tg_mut_column& dst = out->cols[c];
    int64_t row = 0;
    if (dst.null_bitmap) std::memset(dst.null_bitmap, 0, (size_t)((total + 7) / 8));
    for (auto* p : parts) {
      if (p->empty()) continue;
      OColumn& src = (*p)[c];
      std::memcpy(dst.data + row * src.elem_len, src.data.data(), (size_t)src.length * src.elem_len);
      for (int64_t r = 0; r < src.length; r++) {
        bool nn = !src.is_null(r);
        if (dst.null_bitmap) { if (nn) dst.null_bitmap[(row + r) >> 3] |= (uint8_t)(1u << ((row + r) & 7)); }
        else if (!nn) { set_error("fetch: NULL produced for a column without null bitmap"); return TG_ERR_INVALID; }
      }
      row += src.length;
    }
  }
  return 0;
}

// Column.MergeNulls column.go:906 for the result of a binary builtin
static void merge_nulls(const tg_column* a, const tg_column* b, int64_t n, uint8_t* out) {
  for (int64_t i = 0; i < (n + 7) / 8; i++) {
    uint8_t x = a->null_bitmap ? a->null_bitmap[i] : 0xff;
    uint8_t y = (b && b->null_bitmap) ? b->null_bitmap[i] : 0xff;
    out[i] = x & y;
  }
  if (n & 7) out[(n - 1) >> 3] &= (uint8_t)((1u << (n & 7)) - 1);
}
static inline bool res_is_null(const uint8_t* nulls, int64_t i) { return ((nulls[i >> 3] >> (i & 7)) & 1) == 0; }

}  // namespace orc

using namespace orc;

extern "C" {

const char* orc_last_error(void) { return orc::g_err.c_str(); }

int orc_vec_compare_int(int op, int ua, int ub, const tg_column* a, const tg_column* b, int64_t bc,
                        int64_t* result, uint8_t* nulls) {
  int64_t n = a->length;
  merge_nulls(a, b, n, nulls);
  for (int64_t i = 0; i < n; i++) {
    int64_t y = b ? col_i64(*b, i) : bc;
    result[i] = apply_cmp(op, compare_int(col_i64(*a, i), ua != 0, y, ub != 0)) ? 1 : 0;
  }
  return 0;
}

int orc_vec_compare_real(int op, const tg_column* a, const tg_column* b, double bc, int64_t* result,
                         uint8_t* nulls) {
  int64_t n = a->length;
  merge_nulls(a, b, n, nulls);
  for (int64_t i = 0; i < n; i++) {
    double y = b ? col_f64(*b, i) : bc;
    result[i] = apply_cmp(op, compare_real(col_f64(*a, i), y)) ? 1 : 0;
  }
  return 0;
}

// builtinArithmeticMinusIntSig.overflowCheck builtin_arithmetic.go:491 (forceToSigned = false)
static bool minus_overflow(bool lu, bool ru, int64_t a, int64_t b) {
  bool is_signed = !lu && !ru;
  int64_t res = (int64_t)((uint64_t)a - (uint64_t)b);
  uint64_t ua = (uint64_t)a, ub = (uint64_t)b;
  bool resUnsigned = false;
  if (lu) {
    if (ru) { if (ua < ub) { if (res >= 0) return true; } else resUnsigned = true; }
    else {
      if (b >= 0) { if (ua > ub) resUnsigned = true; }
      else { if (UINT64_MAX - ua < (uint64_t)(-(uint64_t)b)) return true; resUnsigned = true; }
    }
  } else {
    if (ru) { if ((uint64_t)a - (uint64_t)INT64_MIN < ub) return true; }
    else { if (a > 0 && b < 0) resUnsigned = true; else if (a < 0 && b > 0 && res >= 0) return true; }
  }
  if ((!is_signed && !resUnsigned && res < 0) || (is_signed && resUnsigned && (uint64_t)res > (uint64_t)INT64_MAX)) return true;
  return false;
}

int orc_vec_arith_int(int op, int ua, int ub, const tg_column* a, const tg_column* b, int64_t bc,
                      int64_t* result, uint8_t* nulls) {
  int64_t n = a->length;
  merge_nulls(a, b, n, nulls);
  bool lu = ua != 0, ru = ub != 0;
  for (int64_t i = 0; i < n; i++) {
    int64_t lh = col_i64(*a, i), rh = b ? col_i64(*b, i) : bc;
    bool overflow = false;
    int64_t r = 0;
    switch (op) {
      case TG_ARITH_PLUS:
        if (lu && ru) overflow = (uint64_t)lh > UINT64_MAX - (uint64_t)rh;                       // plusUU
        else if (lu && !ru) overflow = (rh < 0 && (uint64_t)(-(uint64_t)rh) > (uint64_t)lh) ||   // plusUS
                                       (rh > 0 && (uint64_t)lh > UINT64_MAX - (uint64_t)rh);
        else if (!lu && ru) overflow = (lh < 0 && (uint64_t)(-(uint64_t)lh) > (uint64_t)rh) ||   // plusSU
                                       (lh > 0 && (uint64_t)rh > UINT64_MAX - (uint64_t)lh);
        else overflow = (lh > 0 && rh > INT64_MAX - lh) || (lh < 0 && rh < INT64_MIN - lh);      // plusSS
        r = (int64_t)((uint64_t)lh + (uint64_t)rh);
        break;
      case TG_ARITH_MINUS:
        overflow = minus_overflow(lu, ru, lh, rh);
        r = (int64_t)((uint64_t)lh - (uint64_t)rh);
        break;
      default:   // multiply
        if (lu || ru) {   // builtinArithmeticMultiplyIntUnsignedSig :1011
          uint64_t x = (uint64_t)lh, y = (uint64_t)rh, res = x * y;
          overflow = x != 0 && res / x != y;
          r = (int64_t)res;
        } else {          // builtinArithmeticMultiplyIntSig :646
          int64_t tmp = (int64_t)((uint64_t)lh * (uint64_t)rh);
          bool special = (tmp == INT64_MIN && lh == -1);   // Go wraps MinInt64 / -1; C would trap
          overflow = special || (lh != 0 && tmp / lh != rh);
          r = tmp;
        }
    }
    if (overflow) {
      if (res_is_null(nulls, i)) { result[i] = 0; continue; }
      set_error("ErrOverflow: BIGINT value is out of range");
      return TG_ERR_OVERFLOW;
    }
    result[i] = r;
  }
  return 0;
}

int orc_vec_arith_real(int op, const tg_column* a, const tg_column* b, double bc, double* result,
                       uint8_t* nulls) {
  int64_t n = a->length;
  merge_nulls(a, b, n, nulls);
  for (int64_t i = 0; i < n; i++) {
    double x = col_f64(*a, i), y = b ? col_f64(*b, i) : bc;
    double r;
    bool overflow;
    switch (op) {
      case TG_ARITH_PLUS: r = x + y; overflow = !std::isfinite(r); break;    // mathutil.IsFinite
      case TG_ARITH_MINUS: r = x - y; overflow = !std::isfinite(r); break;
      default: r = x * y; overflow = std::isinf(r); break;                   // math.IsInf only
    }
    if (overflow) {
      if (res_is_null(nulls, i)) { result[i] = r; continue; }
      set_error("ErrOverflow: DOUBLE value is out of range");
      return TG_ERR_OVERFLOW;
    }
    result[i] = r;
  }
  return 0;
}

int orc_vec_filter(const tg_chunk* chk, const tg_filter_item* items, int32_t n_items, uint8_t* selected,
                   int64_t* n_selected) {
  int64_t phys = chunk_physical_rows(*chk);
  std::memset(selected, 0, (size_t)phys);
  int64_t cnt = 0;
  int64_t n = chunk_logical_rows(*chk);
  for (int64_t l = 0; l < n; l++) {
    int64_t p = chk->sel ? chk->sel[l] : l;
    bool s = filter_row(*chk, p, items, n_items);
    selected[p] = s ? 1 : 0;
    cnt += s;
  }
  if (n_selected) *n_selected = cnt;
  return 0;
}

}  // extern "C"
