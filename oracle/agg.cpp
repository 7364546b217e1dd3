// oracle/agg.cpp — CPU restatement of HashAggExec (TEST INFRASTRUCTURE, see oracle.h).
//
// Follows the reference's pkg/executor/aggregate:
//   agg_hash_executor.go   parallelExec :635, fetchChildData :449, DefaultVal on empty input :654
//   agg_hash_partial_worker.go  updatePartialResult :256, getPartialResultsOfEachRow :219
//                               (murmur3.Sum32(key) % finalConcurrency), shuffleIntermData :287
//   agg_hash_final_worker.go    mergeInputIntoResultMap :73, generateResultAndSend :121
//   agg_util.go            GetGroupKey :106 → codec.HashGroupKey util/codec/codec.go:1761
// and pkg/executor/aggfuncs: func_count.go (:28-47, :73, :481), func_sum.go (:39, :65-114),
// func_avg.go (:317, :332-340, :366, :444), func_max_min.go, func_first_row.go.
// Third-party: github.com/twmb/murmur3 v1.1.6 (go.mod:130) Sum32 = MurmurHash3_x86_32 seed 0; it only
// selects the final worker, never the result.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <thread>
#include <unordered_map>
#include <memory>
#include "common.hpp"

namespace orc {

static const uint8_t NilFlag = 0, floatFlag = 5, varintFlag = 8;   // codec.go:41-52

// encoding/binary.PutVarint (zig-zag + uvarint), used by codec.EncodeVarint number.go:123
static int put_varint(uint8_t* buf, int64_t x) {
  uint64_t ux = (uint64_t)x << 1;
  if (x < 0) ux = ~ux;
  int i = 0;
  while (ux >= 0x80) { buf[i++] = (uint8_t)ux | 0x80; ux >>= 7; }
  buf[i++] = (uint8_t)ux;
  return i;
}
// codec.HashGroupKey ETInt branch: NilFlag | varintFlag + EncodeVarint (encodeSignedInt :249)
int group_key_int(int64_t v, bool is_null, uint8_t* out) {
  if (is_null) { out[0] = NilFlag; return 1; }
  out[0] = varintFlag;
  return 1 + put_varint(out + 1, v);
}
// ETReal branch: floatFlag + EncodeFloat (float.go:44: encodeFloatToCmpUint64 then big-endian u64)
int group_key_real(double f, bool is_null, uint8_t* out) {
  if (is_null) { out[0] = NilFlag; return 1; }
  out[0] = floatFlag;
  uint64_t u; std::memcpy(&u, &f, 8);
  if (f >= 0) u |= 0x8000000000000000ull; else u = ~u;
  for (int i = 0; i < 8; i++) out[1 + i] = (uint8_t)(u >> (56 - 8 * i));
  return 9;
}

// MurmurHash3_x86_32, seed 0 (github.com/twmb/murmur3 Sum32)
static uint32_t murmur3_sum32(const uint8_t* data, size_t len) {
  const uint32_t c1 = 0xcc9e2d51, c2 = 0x1b873593;
  uint32_t h1 = 0;
  size_t nblocks = len / 4;
  for (size_t i = 0; i < nblocks; i++) {
    uint32_t k1; std::memcpy(&k1, data + 4 * i, 4);
    k1 *= c1; k1 = (k1 << 15) | (k1 >> 17); k1 *= c2;
    h1 ^= k1; h1 = (h1 << 13) | (h1 >> 19); h1 = h1 * 5 + 0xe6546b64;
  }
  const uint8_t* tail = data + nblocks * 4;
  uint32_t k1 = 0;
  switch (len & 3) {
    case 3: k1 ^= (uint32_t)tail[2] << 16; [[fallthrough]];
    case 2: k1 ^= (uint32_t)tail[1] << 8; [[fallthrough]];
    case 1: k1 ^= tail[0]; k1 *= c1; k1 = (k1 << 15) | (k1 >> 17); k1 *= c2; h1 ^= k1;
  }
  h1 ^= (uint32_t)len;
  h1 ^= h1 >> 16; h1 *= 0x85ebca6b; h1 ^= h1 >> 13; h1 *= 0xc2b2ae35; h1 ^= h1 >> 16;
  return h1;
}

// PartialResult of one aggregate function (union of the reference's partialResult4* structs)
struct PR {
  double fval = 0;      // SUM/AVG sum, MIN/MAX double, FIRSTROW double
  int64_t ival = 0;     // COUNT, AVG count, SUM notNullRowCount, MIN/MAX/FIRSTROW int
  bool isNull = true;   // MIN/MAX/FIRSTROW: no value yet (partialResult4MaxMinInt.isNull)
  bool gotFirstRow = false;
};

struct Agg {
  std::vector<FieldType> colTypes;
  std::vector<int> groupBy;
  std::vector<tg_agg_func> funcs;
  int partialConcurrency = 5, finalConcurrency = 5;
  std::vector<int> outElemLen;
  std::vector<std::vector<OColumn>> results;   // one per final worker
  std::vector<OColumn> defaultRow;             // DefaultVal row for empty input, no group by
  bool emittedDefault = false;
  double seconds = 0;
};

using GroupMap = std::unordered_map<std::string, std::vector<PR>>;

static bool arg_is_real(const tg_agg_func& f) { return f.arg_type == TypeDouble || f.arg_type == TypeFloat; }

static bool check_supported(const Agg& a, std::string& err) {
  for (int g : a.groupBy) {
    int tp = a.colTypes[g].tp;
    if (fixed_len(tp) != 8 || tp == TypeDate || tp == TypeDatetime || tp == TypeTimestamp) {
      err = "oracle: group-by column type not restated"; return false;
    }
  }
  for (auto& f : a.funcs) {
    if (f.mode != TG_AGGMODE_COMPLETE && f.mode != TG_AGGMODE_FINAL) { err = "oracle: agg mode not restated"; return false; }
    switch (f.name) {
      case TG_AGG_COUNT: break;
      case TG_AGG_SUM: case TG_AGG_AVG:
        if (f.arg_type != TypeDouble) { err = "oracle: SUM/AVG only over DOUBLE (SUM(int) is DECIMAL, base_func.go:223)"; return false; }
        break;
      case TG_AGG_MIN: case TG_AGG_MAX: case TG_AGG_FIRSTROW:
        if (f.arg_col < 0 || fixed_len(f.arg_type) != 8) { err = "oracle: MIN/MAX/FIRSTROW arg type not restated"; return false; }
        break;
      default: err = "oracle: unknown aggregate"; return false;
    }
  }
  return true;
}

// af.UpdatePartialResult for one row (Complete mode: original input) or af.MergePartialResult-like
// consumption of a partial-result input row (Final mode)
// AggFuncDesc.Args[0] as the fused scalar expression (tg_agg_func.arg_expr): args[0].EvalReal(row) through
// builtinArithmeticMinusRealSig / MultiplyRealSig (builtin_arithmetic.go evalReal: NULL if an operand is NULL, ErrOverflow
// when the result leaves the DOUBLE range).  Returns false for NULL; sets *overflow.
static bool arg_real(const tg_chunk& chk, const tg_agg_func& f, int64_t p, double& v, bool* overflow) {
  if (col_is_null(chk.cols[f.arg_col], p)) return false;
  double x = col_f64(chk.cols[f.arg_col], p);
  if (f.arg_expr == TG_ARGEXPR_COL) { v = x; return true; }
  if (col_is_null(chk.cols[f.arg_col2], p)) return false;
  double y = col_f64(chk.cols[f.arg_col2], p);
  volatile double t = f.arg_expr == TG_ARGEXPR_MUL_CSUB ? f.arg_const - y : y;
  volatile double r = x * t;
  if (!std::isfinite((double)t) || !std::isfinite((double)r)) *overflow = true;
  v = r;
  return true;
}
static std::atomic<bool> g_arg_overflow_any{false};
static thread_local bool g_arg_overflow = false;

static void update_row(const Agg& a, const tg_chunk& chk, int64_t p, std::vector<PR>& prs) {
  for (size_t k = 0; k < a.funcs.size(); k++) {
    const tg_agg_func& f = a.funcs[k];
    PR& pr = prs[k];
    bool final_mode = f.mode == TG_AGGMODE_FINAL;
    switch (f.name) {
      case TG_AGG_COUNT:
        if (final_mode) {   // countPartial.UpdatePartialResult func_count.go:461: p += input count
          if (!col_is_null(chk.cols[f.arg_col], p)) pr.ival += col_i64(chk.cols[f.arg_col], p);
        } else if (f.arg_col < 0) pr.ival++;   // COUNT(*) / count(1)
        else if (!col_is_null(chk.cols[f.arg_col], p)) pr.ival++;   // countOriginal4*.Update :73
        break;
      case TG_AGG_SUM: {   // sum4Float64.UpdatePartialResult func_sum.go:90
        double v;
        if (arg_real(chk, f, p, v, &g_arg_overflow)) { pr.fval += v; pr.ival++; }
        break;
      }
      case TG_AGG_AVG:
        if (final_mode) {   // avgPartial4Float64 func_avg.go:405: args[0]=count, args[1]=sum
          const tg_column& cc = chk.cols[f.arg_col]; const tg_column& sc = chk.cols[f.arg_col2];
          if (!col_is_null(sc, p) && !col_is_null(cc, p)) { pr.fval += col_f64(sc, p); pr.ival += col_i64(cc, p); }
        } else {   // avgOriginal4Float64 :366
          double v;
          if (arg_real(chk, f, p, v, &g_arg_overflow)) { pr.fval += v; pr.ival++; }
        }
        break;
      case TG_AGG_MIN: case TG_AGG_MAX: {   // maxMin4Int / maxMin4Float64 func_max_min.go
        const tg_column& c = chk.cols[f.arg_col];
        if (col_is_null(c, p)) break;
        bool isMax = f.name == TG_AGG_MAX;
        if (arg_is_real(f)) {
          double v = col_f64(c, p);
          if (pr.isNull) { pr.fval = v; pr.isNull = false; }
          else if ((isMax && v > pr.fval) || (!isMax && v < pr.fval)) pr.fval = v;
        } else if (f.arg_flag & UnsignedFlag) {
          uint64_t v = (uint64_t)col_i64(c, p);
          if (pr.isNull) { pr.ival = (int64_t)v; pr.isNull = false; }
          else if ((isMax && v > (uint64_t)pr.ival) || (!isMax && v < (uint64_t)pr.ival)) pr.ival = (int64_t)v;
        } else {
          int64_t v = col_i64(c, p);
          if (pr.isNull) { pr.ival = v; pr.isNull = false; }
          else if ((isMax && v > pr.ival) || (!isMax && v < pr.ival)) pr.ival = v;
        }
        break;
      }
      case TG_AGG_FIRSTROW: {   // firstRow4Int func_first_row.go:140-161
        if (pr.gotFirstRow) break;
        const tg_column& c = chk.cols[f.arg_col];
        pr.gotFirstRow = true;
        pr.isNull = col_is_null(c, p);
        if (!pr.isNull) { if (arg_is_real(f)) pr.fval = col_f64(c, p); else pr.ival = col_i64(c, p); }
        break;
      }
    }
  }
}

// af.MergePartialResult (func_sum.go:106, func_count.go:481, func_avg.go:444, max_min, first_row)
static void merge_prs(const Agg& a, const std::vector<PR>& src, std::vector<PR>& dst) {
  for (size_t k = 0; k < a.funcs.size(); k++) {
    const tg_agg_func& f = a.funcs[k];
    const PR& s = src[k]; PR& d = dst[k];
    switch (f.name) {
      case TG_AGG_COUNT: d.ival += s.ival; break;
      case TG_AGG_SUM: case TG_AGG_AVG: d.fval += s.fval; d.ival += s.ival; break;
      case TG_AGG_MIN: case TG_AGG_MAX: {
        if (s.isNull) break;
        bool isMax = f.name == TG_AGG_MAX;
        if (d.isNull) { d = s; break; }
        if (arg_is_real(f)) { if ((isMax && s.fval > d.fval) || (!isMax && s.fval < d.fval)) d.fval = s.fval; }
        else if (f.arg_flag & UnsignedFlag) {
          if ((isMax && (uint64_t)s.ival > (uint64_t)d.ival) || (!isMax && (uint64_t)s.ival < (uint64_t)d.ival)) d.ival = s.ival;
        } else { if ((isMax && s.ival > d.ival) || (!isMax && s.ival < d.ival)) d.ival = s.ival; }
        break;
      }
      case TG_AGG_FIRSTROW: if (!d.gotFirstRow && s.gotFirstRow) d = s; break;
    }
  }
}

// af.AppendFinalResult2Chunk (func_sum.go:80-88, func_avg.go:332-340, func_count.go:43-47)
static void append_final(const Agg& a, const std::vector<PR>& prs, std::vector<OColumn>& out) {
  for (size_t k = 0; k < a.funcs.size(); k++) {
    const tg_agg_func& f = a.funcs[k];
    const PR& p = prs[k];
    OColumn& c = out[k];
    switch (f.name) {
      case TG_AGG_COUNT: c.append_i64(p.ival); break;
      case TG_AGG_SUM: if (p.ival == 0) c.append_null(); else c.append_f64(p.fval); break;
      case TG_AGG_AVG: if (p.ival == 0) c.append_null(); else c.append_f64(p.fval / (double)p.ival); break;
      case TG_AGG_MIN: case TG_AGG_MAX: case TG_AGG_FIRSTROW:
        if (p.isNull) c.append_null();
        else if (arg_is_real(f)) c.append_f64(p.fval); else c.append_i64(p.ival);
        break;
    }
  }
}

static void group_key_of(const Agg& a, const tg_chunk& chk, int64_t p, std::string& key) {
  key.clear();
  uint8_t buf[16];
  for (int g : a.groupBy) {
    const tg_column& c = chk.cols[g];
    bool isNull = col_is_null(c, p);
    int n = (a.colTypes[g].tp == TypeDouble) ? group_key_real(col_f64(c, p), isNull, buf)
                                              : group_key_int(col_i64(c, p), isNull, buf);
    key.append(reinterpret_cast<char*>(buf), n);
  }
}

static bool run_agg(Agg& a, const tg_chunk* chunks, int64_t nchunks) {
  auto t0 = std::chrono::steady_clock::now();
  int M = a.partialConcurrency, N = a.finalConcurrency;
  g_arg_overflow_any = false;
  // partial workers: partialResultsMap[finalWorkerIdx] (agg_hash_partial_worker.go:219)
  std::vector<std::vector<GroupMap>> partial(M, std::vector<GroupMap>(N));
  std::atomic<int64_t> next{0};
  std::atomic<int64_t> totalRows{0};
  {
    std::vector<std::thread> th;
    for (int w = 0; w < M; w++) th.emplace_back([&, w] {
      std::string key;
      g_arg_overflow = false;
      for (;;) {
        int64_t i = next.fetch_add(1);
        if (i >= nchunks) { if (g_arg_overflow) g_arg_overflow_any = true; break; }
        const tg_chunk& chk = chunks[i];
        int64_t n = chunk_logical_rows(chk);
        totalRows += n;
        for (int64_t l = 0; l < n; l++) {
          int64_t p = chk.sel ? chk.sel[l] : l;
          group_key_of(a, chk, p, key);
          // int(murmur3.Sum32(key)) % finalConcurrency — Go int is 64-bit, so the value is non-negative
          int fw = (int)(murmur3_sum32((const uint8_t*)key.data(), key.size()) % (uint32_t)N);
          auto it = partial[w][fw].find(key);
          if (it == partial[w][fw].end()) it = partial[w][fw].emplace(key, std::vector<PR>(a.funcs.size())).first;
          update_row(a, chk, p, it->second);
        }
      }
    });
    for (auto& t : th) t.join();
  }
  if (g_arg_overflow_any.load()) { set_error("ErrOverflow: DOUBLE value is out of range in an aggregate argument expression"); return false; }
  // final workers: merge the M partial maps destined to them, then generate results
  a.results.clear(); a.results.resize(N);
  for (auto& r : a.results) for (int el : a.outElemLen) r.emplace_back(el);
  {
    std::vector<std::thread> th;
    for (int fw = 0; fw < N; fw++) th.emplace_back([&, fw] {
      GroupMap result;
      for (int w = 0; w < M; w++) {
        for (auto& kv : partial[w][fw]) {
          auto it = result.find(kv.first);
          if (it == result.end()) result.emplace(kv.first, kv.second);
          else merge_prs(a, kv.second, it->second);
        }
      }
      for (auto& kv : result) append_final(a, kv.second, a.results[fw]);
    });
    for (auto& t : th) t.join();
  }
  // agg_hash_executor.go:654: child returned nothing and DefaultVal != nil (no GROUP BY,
  // builder.go:2114-2137): a single row of default values (COUNT → 0, everything else NULL)
  if (totalRows.load() == 0 && a.groupBy.empty()) {
    std::vector<PR> empty(a.funcs.size());
    append_final(a, empty, a.results[0]);
  }
  a.seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return true;
}

}  // namespace orc

using namespace orc;
struct orc_agg { Agg a; };

extern "C" {

int32_t orc_group_key_int(int64_t v, int is_null, uint8_t* out) { return group_key_int(v, is_null != 0, out); }
int32_t orc_group_key_real(double v, int is_null, uint8_t* out) { return group_key_real(v, is_null != 0, out); }

int orc_agg_open(const tg_agg_desc* d, int32_t pc, int32_t fc, orc_agg** out) {
  auto* h = new orc_agg();
  Agg& a = h->a;
  a.colTypes.resize(d->n_cols);
  for (int i = 0; i < d->n_cols; i++) { a.colTypes[i].tp = d->col_types[i]; a.colTypes[i].flag = d->col_flags ? d->col_flags[i] : 0; }
  a.groupBy.assign(d->group_by_cols, d->group_by_cols + d->n_group_by);
  a.funcs.assign(d->funcs, d->funcs + d->n_funcs);
  a.partialConcurrency = std::max(1, pc); a.finalConcurrency = std::max(1, fc);
  std::string err;
  if (!check_supported(a, err)) { set_error(err); delete h; return TG_ERR_UNSUPPORTED; }
  for (auto& f : a.funcs) a.outElemLen.push_back(8);
  *out = h;
  return 0;
}
int orc_agg_run(orc_agg* h, const tg_chunk* chunks, int64_t n) { return run_agg(h->a, chunks, n) ? 0 : TG_ERR_UNSUPPORTED; }
int64_t orc_agg_result_rows(orc_agg* h) { int64_t n = 0; for (auto& r : h->a.results) if (!r.empty()) n += r[0].length; return n; }
int orc_agg_result_fetch(orc_agg* h, tg_mut_chunk* out) {
  std::vector<std::vector<OColumn>*> parts;
  for (auto& r : h->a.results) parts.push_back(&r);
  return fetch_result(parts, (int)h->a.funcs.size(), out);
}
double orc_agg_seconds(orc_agg* h) { return h->a.seconds; }
void orc_agg_close(orc_agg* h) { delete h; }

}  // extern "C"
