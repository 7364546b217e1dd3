// join.cu — tg_join_*: the GPU hash join behind HashJoinV2Exec's Open/Next/Close contract
// (pkg/executor/join/hash_join_v2.go:608, :690, :1161, :647).  Host-side orchestration only; the
// kernels live in join_kernels.cuh.
#include <memory>
#include <deque>
#include <algorithm>
#include <cmath>
#include <condition_variable>
#include "join_kernels.cuh"
#include "partition_kernels.cuh"
#include "chunk_io.cuh"

namespace tg {

static const int64_t kGeneralBatchRows = 16ll << 20;   // sub-batch of the general probe path (bounds temp memory)
static const int64_t kDirectPushRows = 128ll << 10;    // chunks at least this big are copied straight from the caller
static const int64_t kNextWindowRows = 1ll << 20;      // D2H window that serves small tg_join_next calls

struct Side {
  int ncols = 0;
  std::vector<int> types;
  std::vector<uint32_t> flags;
  std::vector<int> elem;
  std::vector<int> kelem;         // width the kernels see: a DECIMAL column reaches them as 8-byte row ids (kernel_view)
  bool has_cells = false;         // some needed column is DECIMAL
  std::vector<char> needed;       // staged to the device (key ∪ used ∪ filter columns)
  int key_col = -1;               // the single equal-condition key; -1 when the join has several (key_cols)
  std::vector<int> key_cols;      // several equal conditions: the key columns in condition order
  std::vector<int> key_reject;    //   per key column: mixed-signedness pair and this is the signed side (negative = no key)
  std::vector<int> used;          // columns of this side that appear in the output
  DevFilter filter{};
};

// device-resident columns of one side for one batch
struct ColStore {
  std::vector<std::unique_ptr<DevBuf>> data, nulls;
  std::vector<char> has_nulls;
  int64_t rows = 0, cap_rows = 0;
  void init(int ncols) {
    data.clear(); nulls.clear();
    for (int i = 0; i < ncols; i++) { data.emplace_back(new DevBuf()); nulls.emplace_back(new DevBuf()); }
    has_nulls.assign(ncols, 0);
    rows = cap_rows = 0;
  }
  DevCols view(const Side& s) const {
    DevCols v{};
    for (int c = 0; c < s.ncols && c < TG_MAX_COLS; c++) {
      v.data[c] = s.needed[c] ? data[c]->p : nullptr;
      v.nulls[c] = (s.needed[c] && has_nulls[c]) ? nulls[c]->as<uint8_t>() : nullptr;
      v.elem_len[c] = s.elem[c];
    }
    return v;
  }
};

struct ResultBatch {
  std::vector<std::unique_ptr<DevBuf>> cols, bitmaps;
  int64_t rows = 0;
  int64_t consumed = 0;
};

}  // namespace tg

using namespace tg;

struct JoinImpl;

// The C-ABI handle is a small SHELL that outlives tg_join_close: close frees the implementation (GPU buffers, streams,
// staging) but parks the shell in a bounded graveyard (common.cuh), so a caller that raced with close — parked in
// tg_join_next_wait, blocked on `mu`, or about to enter with a pointer it read just before the close — finds a live
// `closed` flag and gets TG_ERR_CANCELLED instead of touching freed memory (exec.Executor: "Close may be called ...
// with Next() at the same time", executor.go:65).  A second close is a no-op.
struct tg_join {
  std::mutex mu;                     // build / probe-input side (one pushing thread)
  std::mutex res_mu;                 // result queue (one pulling thread may run concurrently with the pusher, like the
  std::condition_variable res_cv;    //   reference's probe fetcher vs joinResultCh consumer, hash_join_v2.go:840 / :1176)
  std::atomic<bool> closed{false};
  JoinImpl* impl = nullptr;          // guarded by mu + res_mu; nullptr once closed
};

struct JoinImpl : DeviceHandle {
  std::mutex& res_mu;                // the shell's (see tg_join)
  std::condition_variable& res_cv;
  explicit JoinImpl(tg_join& shell) : res_mu(shell.res_mu), res_cv(shell.res_cv) {}
  cudaStream_t d2h_stream = nullptr; // tg_join_next copies results on its own stream: D2H overlaps the next H2D + probe
  double load_factor = 0.5;
  bool default_load_factor = true;

  int join_type = 0;
  bool build_is_right = true;
  Side build, probe;
  int n_lused = 0, n_rused = 0;
  std::vector<int> lused, rused;
  int probe_kind = PK_INNER;
  bool need_scan = false;          // JoinProbe.NeedScanRowTable
  int scan_mode = 0;
  bool has_flag_col = false;
  int n_out = 0;
  std::vector<int> out_elem;          // bytes per output cell, 40 for DECIMAL
  std::vector<int> kout_elem;         // what the kernels write: 8-byte row ids for DECIMAL (gather_cells makes the cells)
  KeySpec build_key{}, probe_key{};   // data pointers filled per launch
  bool multi_key = false;             // several equal conditions: synthetic 64-bit candidate key + residual equalities (k_composite_key)
  DevBuf bkey_syn, bkey_syn_nn, pkey_syn, pkey_syn_nn;
  std::vector<tg_other_item> other;   // OtherCondition (sides already mapped: 0 = probe child, 1 = build child)
  std::vector<int> other_build_cols;  // build columns it reads (kept in the row store although they may not be output)
  DevOther dev_other{};               // compiled after the build (row-store word of every build operand)

  // build state
  HostStage bstage;
  ColStore bcols;
  bool built = false;
  DevBuf table, rows_store, row_slot, row_rank, slot_used, scalars;
  TableView tv{};
  DevBuf pidx_slots, pidx_pilot;   // slice index of a sliced U1 table (build_slice_index); pidx.P == 0: none
  SliceIndex pidx{};
  RowSpec rowspec{};
  std::vector<int> build_word_of_col;   // build column → row-store word (mode G)
  int u1_payload_col = -1;

  // probe state
  HostStage pstage;
  ColStore pcols_dev;
  DevBuf tmp_cnt, tmp_slot, tmp_off, tmp_sums, out_cursor;
  DevBuf part_scratch;                               // counts | cursors | offsets of the L2 partition pass
  DevBuf tile_cnt;                                   // rows each 128-row tile keeps in the in-place segment probe
  double seg_match = 1.0;                            // output / input rows of the last partitioned probe whose count the host read
  // the fills of that probe's segments, for the in-place segment capacity (inplace_seg_cap): its P (0 = nothing learned:
  // no such call yet, or it overflowed a segment), the rows it scattered and its largest segment fill
  int seg_parts = 0;
  int64_t seg_rows = 0, seg_fill_max = 0;
  std::unique_ptr<DevBuf> part_cols[1 + TG_FAST_MAX_PCOLS];   // partitioned copies of the probe key and payload columns
  std::vector<std::unique_ptr<DevBuf>> tmp_valid;
  std::deque<std::unique_ptr<ResultBatch>> results;
  std::vector<std::unique_ptr<ResultBatch>> free_batches;   // recycled (cudaFree would synchronise the whole device)
  std::unique_ptr<ResultBatch> dev_result;      // tg_join_probe_dev output (reused across calls)
  DevBuf iota;                                  // int64 0, 1, 2, ...: the row-id stand-in of every DECIMAL column
  int64_t iota_rows = 0;
  std::vector<std::unique_ptr<DevBuf>> out_ids; // per DECIMAL output column: the source row ids the kernels wrote
  std::atomic<bool> probe_finished{false};
  std::atomic<int64_t> d2h_bytes{0};
  // small-Next window
  PinBuf win;
  int64_t win_lo = 0, win_hi = 0;
  ResultBatch* win_batch = nullptr;

  tg_join_stats stats{};
};

namespace tg {

// ---- descriptor → handle -------------------------------------------------------------------------------
static int fill_side(Side& s, int n, const int32_t* types, const uint32_t* flags) {
  if (n <= 0 || n > TG_MAX_COLS) return fail(TG_ERR_UNSUPPORTED, "child schema must have 1..16 columns");
  s.ncols = n;
  s.types.assign(types, types + n);
  s.flags.resize(n);
  for (int i = 0; i < n; i++) s.flags[i] = flags ? flags[i] : 0;
  s.elem.resize(n);
  for (int i = 0; i < n; i++) s.elem[i] = fixed_len(types[i]);
  s.kelem.resize(n);
  for (int i = 0; i < n; i++) s.kelem[i] = s.elem[i] == kCellBytes ? 8 : s.elem[i];
  s.needed.assign(n, 0);
  return TG_OK;
}

static int key_kind_of(int tp) {
  if (is_int_family(tp)) return KEY_I64;
  if (tp == TG_TYPE_DOUBLE) return KEY_F64;
  if (tp == TG_TYPE_FLOAT) return KEY_F32;
  if (tp == TG_TYPE_DATE || tp == TG_TYPE_DATETIME || tp == TG_TYPE_TIMESTAMP) return KEY_TIME;   // getKeyProp join_table_meta.go:154
  return -1;
}
static bool key_unsigned(int tp, uint32_t flag) {
  // getKeyProp join_table_meta.go:130: YEAR always unsigned, DURATION always signed
  if (tp == TG_TYPE_YEAR) return true;
  if (tp == TG_TYPE_DURATION) return false;
  return (flag & TG_FLAG_UNSIGNED) != 0;
}

static int check_filter(const Side& s, const tg_filter_item* items, int n, DevFilter& out) {
  if (n < 0 || n > TG_MAX_FILTER) return fail(TG_ERR_UNSUPPORTED, "at most 8 CNF filter items are offloaded");
  out.n = n;
  if (n > 0 && !items) return fail(TG_ERR_INVALID, "filter items are NULL");
  for (int i = 0; i < n; i++) {
    const tg_filter_item& it = items[i];
    if (it.lhs_col < 0 || it.lhs_col >= s.ncols || it.rhs_col >= s.ncols) return fail(TG_ERR_INVALID, "filter column out of range");
    // the compare family must fit the column types: a real compare on integer columns (or the reverse) would reinterpret bits
    const bool lreal = s.types[it.lhs_col] == TG_TYPE_DOUBLE;
    if ((it.is_real != 0) != lreal || (it.rhs_col >= 0 && (s.types[it.rhs_col] == TG_TYPE_DOUBLE) != lreal))
      return fail(TG_ERR_UNSUPPORTED, "filter compares columns of different families (the planner casts before the filter)");
    if (s.elem[it.lhs_col] != 8 || (it.rhs_col >= 0 && s.elem[it.rhs_col] != 8))
      return fail(TG_ERR_UNSUPPORTED, "filters are offloaded on 8-byte columns only");
    if (it.op < TG_CMP_LT || it.op > TG_CMP_NE) return fail(TG_ERR_INVALID, "bad filter op");
    out.items[i] = it;
  }
  return TG_OK;
}

static int setup(JoinImpl* j, const tg_join_desc* d) {
  if (!d) return fail(TG_ERR_INVALID, "desc is NULL");
  j->join_type = d->join_type;
  j->build_is_right = d->build_is_right != 0;
  Side left, right;
  TG_TRY(fill_side(left, d->n_left_cols, d->left_types, d->left_flags));
  TG_TRY(fill_side(right, d->n_right_cols, d->right_types, d->right_flags));
  if (d->nkeys < 1 || d->nkeys > TG_MAX_JOIN_KEYS) return fail(TG_ERR_UNSUPPORTED, "GPU hash join handles 1..4 equal-condition keys");
  if (!d->left_key_idx || !d->right_key_idx) return fail(TG_ERR_INVALID, "key index arrays are NULL");
  j->multi_key = d->nkeys > 1;
  std::vector<tg_other_item> residual;   // several keys: `left_key_i = right_key_i`, re-checked on every candidate pair
  if (!j->multi_key) {
    int lk = d->left_key_idx[0], rk = d->right_key_idx[0];
    if (lk < 0 || lk >= left.ncols || rk < 0 || rk >= right.ncols) return fail(TG_ERR_INVALID, "key column out of range");
    left.key_col = lk; right.key_col = rk;
    int lkind = key_kind_of(left.types[lk]), rkind = key_kind_of(right.types[rk]);
    if (lkind < 0 || rkind < 0) return fail(TG_ERR_UNSUPPORTED, "join key type is not offloaded (int family / float / double / date-time only)");
    if ((lkind == KEY_I64) != (rkind == KEY_I64)) return fail(TG_ERR_UNSUPPORTED, "integer vs real join keys are cast by the planner before the join");
    if ((lkind == KEY_TIME) != (rkind == KEY_TIME)) return fail(TG_ERR_UNSUPPORTED, "date-time keys only join date-time keys (codec.go:707)");
  } else {
    // FixedSerializedKey mode (join_table_meta.go:174-178) restricted to 8-byte integer-family columns
    for (int q = 0; q < d->nkeys; q++) {
      int lk = d->left_key_idx[q], rk = d->right_key_idx[q];
      if (lk < 0 || lk >= left.ncols || rk < 0 || rk >= right.ncols) return fail(TG_ERR_INVALID, "key column out of range");
      if (!is_int_family(left.types[lk]) || !is_int_family(right.types[rk]) || left.elem[lk] != 8 || right.elem[rk] != 8)
        return fail(TG_ERR_UNSUPPORTED, "joins on several key columns are offloaded for 8-byte integer-family keys only");
      const bool lu = key_unsigned(left.types[lk], left.flags[lk]), ru = key_unsigned(right.types[rk], right.flags[rk]);
      left.key_cols.push_back(lk); right.key_cols.push_back(rk);
      left.key_reject.push_back(lu != ru && !lu); right.key_reject.push_back(lu != ru && !ru);
      tg_other_item it{};
      it.op = TG_CMP_EQ; it.is_real = 0; it.lhs_side = 0; it.lhs_col = lk; it.rhs_side = 1; it.rhs_col = rk;
      it.lhs_unsigned = lu; it.rhs_unsigned = ru;
      residual.push_back(it);
    }
  }
  auto used_list = [&](int n, const int32_t* v, int ncols, std::vector<int>& out) -> int {
    out.clear();
    if (n < 0) { for (int i = 0; i < ncols; i++) out.push_back(i); return TG_OK; }
    for (int i = 0; i < n; i++) { if (v[i] < 0 || v[i] >= ncols) return fail(TG_ERR_INVALID, "used column out of range"); out.push_back(v[i]); }
    return TG_OK;
  };
  TG_TRY(used_list(d->n_lused, d->lused, left.ncols, j->lused));
  TG_TRY(used_list(d->n_rused, d->rused, right.ncols, j->rused));
  left.used = j->lused; right.used = j->rused;
  j->has_flag_col = false;
  // NewJoinProbe base_join_probe.go:850-932
  bool brt = j->build_is_right;
  switch (j->join_type) {
    case TG_JOIN_INNER: j->probe_kind = PK_INNER; j->need_scan = false; break;
    case TG_JOIN_LEFT_OUTER:
      j->need_scan = !brt; j->probe_kind = j->need_scan ? PK_INNER : PK_PROBE_OUTER; j->scan_mode = 0; break;
    case TG_JOIN_RIGHT_OUTER:
      j->need_scan = brt; j->probe_kind = j->need_scan ? PK_INNER : PK_PROBE_OUTER; j->scan_mode = 0; break;
    case TG_JOIN_SEMI: case TG_JOIN_ANTI_SEMI:
      if (!j->rused.empty()) return fail(TG_ERR_INVALID, "len(rUsed) != 0 for semi join");
      j->need_scan = !brt;
      if (brt) j->probe_kind = j->join_type == TG_JOIN_SEMI ? PK_SEMI : PK_ANTI;
      else { j->probe_kind = PK_MARK_ONLY; j->scan_mode = j->join_type == TG_JOIN_SEMI ? 1 : 0; }
      break;
    case TG_JOIN_LEFT_OUTER_SEMI: case TG_JOIN_ANTI_LEFT_OUTER_SEMI:
      if (!j->rused.empty()) return fail(TG_ERR_INVALID, "len(rUsed) != 0 for left outer semi join");
      if (!brt) return fail(TG_ERR_UNSUPPORTED, "left outer semi join needs the right side as build side");
      j->probe_kind = j->join_type == TG_JOIN_LEFT_OUTER_SEMI ? PK_LEFT_OUTER_SEMI : PK_ANTI_LEFT_OUTER_SEMI;
      j->need_scan = false; j->has_flag_col = true;
      break;
    default: return fail(TG_ERR_INVALID, "unknown join type");
  }
  j->build = brt ? right : left;
  j->probe = brt ? left : right;
  TG_TRY(check_filter(j->build, d->build_filter, d->n_build_filter, j->build.filter));
  TG_TRY(check_filter(j->probe, d->probe_filter, d->n_probe_filter, j->probe.filter));
  // OtherCondition (inner_join_probe.go:72-79): sides re-mapped to probe (0) / build (1)
  j->other.clear(); j->other_build_cols.clear();
  if (d->n_other_cond < 0 || d->n_other_cond + (int)residual.size() > TG_MAX_OTHER)
    return fail(TG_ERR_UNSUPPORTED, "at most 8 OtherCondition items (key equalities of a multi-column key included) are offloaded");
  if (d->n_other_cond > 0 && !d->other_cond) return fail(TG_ERR_INVALID, "other_cond is NULL");
  std::vector<tg_other_item> items = residual;
  for (int i = 0; i < d->n_other_cond; i++) items.push_back(d->other_cond[i]);
  if (!items.empty()) {
    if (j->need_scan || j->probe_kind == PK_MARK_ONLY) return fail(TG_ERR_UNSUPPORTED, "OtherCondition / several key columns with a build-side scan (outer side / left side is the build side) are not offloaded");
    if (j->has_flag_col) return fail(TG_ERR_UNSUPPORTED, "OtherCondition / several key columns on left outer semi joins (NULL-aware match flag) are not offloaded");
    for (size_t i = 0; i < items.size(); i++) {
      tg_other_item it = items[i];
      if (it.op < TG_CMP_LT || it.op > TG_CMP_NE) return fail(TG_ERR_INVALID, "bad OtherCondition op");
      auto remap = [&](int32_t& side, int32_t col, bool may_be_const) -> int {
        if (side < 0) return may_be_const ? TG_OK : fail(TG_ERR_INVALID, "OtherCondition: the left operand must be a column");
        if (side > 1) return fail(TG_ERR_INVALID, "OtherCondition side must be 0 (left) or 1 (right)");
        const Side& sd = side == 0 ? left : right;
        if (col < 0 || col >= sd.ncols) return fail(TG_ERR_INVALID, "OtherCondition column out of range");
        if (sd.elem[col] != 8) return fail(TG_ERR_UNSUPPORTED, "OtherCondition is offloaded on 8-byte columns only");
        if ((sd.types[col] == TG_TYPE_DOUBLE) != (it.is_real != 0)) return fail(TG_ERR_UNSUPPORTED, "OtherCondition compares columns of different families (the planner casts first)");
        const bool is_build = (side == 1) == brt;
        Side& mine = is_build ? j->build : j->probe;
        mine.needed[col] = 1;
        if (is_build && std::find(j->other_build_cols.begin(), j->other_build_cols.end(), col) == j->other_build_cols.end()) j->other_build_cols.push_back(col);
        side = is_build ? 1 : 0;
        return TG_OK;
      };
      TG_TRY(remap(it.lhs_side, it.lhs_col, false));
      TG_TRY(remap(it.rhs_side, it.rhs_col, true));
      j->other.push_back(it);
    }
  }
  for (Side* s : {&j->build, &j->probe}) {
    if (s->key_col >= 0) s->needed[s->key_col] = 1;
    for (int c : s->key_cols) s->needed[c] = 1;
    for (int c : s->used) {
      if (s->elem[c] != 8 && s->elem[c] != 4 && s->elem[c] != kCellBytes)
        return fail(TG_ERR_UNSUPPORTED, "only 4/8-byte fixed-width columns and DECIMAL cells are offloaded (no var-len yet)");
      s->needed[c] = 1;
      s->has_cells |= s->elem[c] == kCellBytes;
    }
    for (int i = 0; i < s->filter.n; i++) {
      s->needed[s->filter.items[i].lhs_col] = 1;
      if (s->filter.items[i].rhs_col >= 0) s->needed[s->filter.items[i].rhs_col] = 1;
    }
  }
  // key specs; mixed signedness (NeedSignFlag, join_table_meta.go:296-303): the signed side's negative
  // values can never match
  int bk = j->build.key_col, pk = j->probe.key_col;
  j->build_key = KeySpec{nullptr, nullptr, j->multi_key ? KEY_I64 : key_kind_of(j->build.types[bk]), 0};
  j->probe_key = KeySpec{nullptr, nullptr, j->multi_key ? KEY_I64 : key_kind_of(j->probe.types[pk]), 0};
  if (!j->multi_key && j->build_key.kind == KEY_I64) {
    bool bu = key_unsigned(j->build.types[bk], j->build.flags[bk]), pu = key_unsigned(j->probe.types[pk], j->probe.flags[pk]);
    if (bu != pu) { j->build_key.reject_negative = !bu; j->probe_key.reject_negative = !pu; }
  }
  // output schema: LUsed of left ‖ RUsed of right [‖ matched flag]
  j->n_lused = (int)j->lused.size(); j->n_rused = (int)j->rused.size();
  j->out_elem.clear(); j->kout_elem.clear();
  for (int c : j->lused) { j->out_elem.push_back(left.elem[c]); j->kout_elem.push_back(left.kelem[c]); }
  for (int c : j->rused) { j->out_elem.push_back(right.elem[c]); j->kout_elem.push_back(right.kelem[c]); }
  if (j->has_flag_col) { j->out_elem.push_back(8); j->kout_elem.push_back(8); }
  j->n_out = (int)j->out_elem.size();
  if (j->n_out > TG_MAX_OUT) return fail(TG_ERR_UNSUPPORTED, "too many output columns");
  j->device = d->device;
  j->default_load_factor = !(d->load_factor > 0.05 && d->load_factor <= 0.95);
  j->load_factor = (d->load_factor > 0.05 && d->load_factor <= 0.95) ? d->load_factor : 0.35;   // sparse enough for short probe runs, dense enough for the L2 slices of the partitioned probe
  return TG_OK;
}

// ---- host chunk → device ---------------------------------------------------------------------------
// the rows of side s → cs (replaces its contents): from the host staging st, or (st = nullptr) straight from the
// buffers of a big pushed chunk
static int upload_side(JoinImpl* j, const Side& s, const HostStage* st, const tg_chunk* chk, ColStore& cs) {
  cs.rows = st ? st->rows : chk->cols[0].length;
  for (int c = 0; c < s.ncols; c++) {
    if (!s.needed[c]) continue;
    const void* data = st ? st->data[c]->p : chk->cols[c].data;
    const uint8_t* nulls = st ? (st->has_nulls[c] ? st->nulls[c]->p : nullptr) : chk->cols[c].null_bitmap;
    cs.has_nulls[c] = nulls != nullptr;
    TG_TRY(upload_column(j->device, j->stream, data, nulls, cs.rows, s.elem[c], *cs.data[c], *cs.nulls[c], &j->stats.h2d_bytes));
  }
  return TG_OK;
}

// device chunk → device column store (device-to-device, appended)
static int devchunk_append(JoinImpl* j, const tg_chunk* chk, const Side& s, ColStore& cs) {
  if (chk->sel) return fail(TG_ERR_UNSUPPORTED, "device-resident chunks must not carry a sel vector");
  int64_t n = chk->ncols ? chk->cols[0].length : 0;
  if (n == 0) return TG_OK;
  for (int c = 0; c < s.ncols; c++) {
    if (!s.needed[c]) continue;
    int el = s.elem[c];
    TG_TRY(cs.data[c]->ensure_preserve(j->device, (size_t)(cs.rows + n) * el + 16, (size_t)cs.rows * el, j->stream));
    TG_CUDA(cudaMemcpyAsync(cs.data[c]->as<uint8_t>() + (size_t)cs.rows * el, chk->cols[c].data, (size_t)n * el, cudaMemcpyDeviceToDevice, j->stream));
    if (chk->cols[c].null_bitmap || cs.has_nulls[c]) {
      if (cs.rows % 8 != 0) return fail(TG_ERR_UNSUPPORTED, "device-resident chunks with NULL bitmaps must start at a multiple of 8 rows");
      size_t need = (size_t)((cs.rows + n + 7) / 8) + 16;
      size_t had = (size_t)((cs.rows + 7) / 8);
      TG_TRY(cs.nulls[c]->ensure_preserve(j->device, need, cs.has_nulls[c] ? had : 0, j->stream));
      if (!cs.has_nulls[c]) { TG_CUDA(cudaMemsetAsync(cs.nulls[c]->p, 0xff, had, j->stream)); cs.has_nulls[c] = 1; }
      if (chk->cols[c].null_bitmap) TG_CUDA(cudaMemcpyAsync(cs.nulls[c]->as<uint8_t>() + had, chk->cols[c].null_bitmap, (size_t)((n + 7) / 8), cudaMemcpyDeviceToDevice, j->stream));
      else TG_CUDA(cudaMemsetAsync(cs.nulls[c]->as<uint8_t>() + had, 0xff, (size_t)((n + 7) / 8), j->stream));
    }
  }
  cs.rows += n;
  return TG_OK;
}

// borrow a device chunk of the probe side as a column view (no copy)
static int probe_view(JoinImpl* j, const tg_chunk* chk, DevCols& v) {
  const Side& s = j->probe;
  TG_TRY(device_view(chk, s.ncols, s.needed, s.elem, v));
  for (int c = 0; c < s.ncols; c++)
    if (s.needed[c] && s.elem[c] == kCellBytes && (reinterpret_cast<uintptr_t>(v.data[c]) & 7)) return fail(TG_ERR_INVALID, "DECIMAL device columns must be 8-byte aligned");
  return TG_OK;
}

// several equal conditions: the synthetic candidate-key column of one side's `n` device-resident rows (k_composite_key)
static int composite_key(JoinImpl* j, const Side& s, const DevCols& v, int64_t n, DevBuf& key, DevBuf& not_null) {
  TG_TRY(key.ensure(j->device, (size_t)(n + 1) * 8 + 16));
  TG_TRY(not_null.ensure(j->device, (size_t)((n + 31) / 32) * 4 + 16));
  if (n <= 0) return TG_OK;
  MultiKeySrc src{};
  src.nk = (int)s.key_cols.size();
  for (int q = 0; q < src.nk; q++) {
    const int c = s.key_cols[q];
    src.data[q] = reinterpret_cast<const int64_t*>(v.data[c]);
    src.nulls[q] = v.nulls[c];
    src.reject[q] = s.key_reject[q];
    if (!src.data[q]) return fail(TG_ERR_INVALID, "key column data is NULL");
  }
  k_composite_key<<<grid_size(j->nsm, n, 256, 8), 256, 0, j->stream>>>(src, n, key.as<int64_t>(), not_null.as<uint32_t>());
  j->stats.kernel_launches++;
  return TG_OK;
}

// ---- DECIMAL cells: late materialisation --------------------------------------------------------------
// The build and probe kernels move 8-byte words.  A used DECIMAL column (40-byte MyDecimal cells, moved, never interpreted)
// reaches them as a row-id column instead: the shared iota of int64 row numbers, under the column's own null bitmap.  So
// every path (U1 payload, row-store word, build-side scan, NULL padding) writes the source row's id and valid byte where
// the cell belongs, and gather_cells then copies the 40 raw bytes of that row, or zero bytes under NULL.
static int ensure_iota(JoinImpl* j, int64_t rows) {
  if (rows <= j->iota_rows) return TG_OK;
  rows = std::max(rows, 2 * j->iota_rows);
  TG_TRY(j->iota.ensure(j->device, (size_t)rows * 8 + 16));
  k_iota<<<grid_size(j->nsm, rows, 256, 8), 256, 0, j->stream>>>(j->iota.as<int64_t>(), rows);
  j->stats.kernel_launches++;
  j->iota_rows = rows;
  return TG_OK;
}

// the view the kernels get of `rows` rows of side s: each needed DECIMAL column becomes the iota (8-byte row ids)
static int kernel_view(JoinImpl* j, const Side& s, DevCols& v, int64_t rows) {
  if (!s.has_cells) return TG_OK;
  TG_TRY(ensure_iota(j, rows));
  for (int c = 0; c < s.ncols; c++)
    if (s.needed[c] && s.elem[c] == kCellBytes) { v.data[c] = j->iota.p; v.elem_len[c] = 8; }
  return TG_OK;
}

// ---- fast-path launch tuning (the defaults are the production choice; the overrides let tests and tools force the
// partition pass, or no pass, on any input) ----
struct ProbeTuning { int ctas_per_sm; bool partition; int parts; int part_min_mb; int part_min_rows; int inplace; };
static ProbeTuning probe_tuning() {
  ProbeTuning t;
  t.ctas_per_sm = env_int("TG_PROBE_CTAS_PER_SM", 0);   // 0 = exactly the resident CTA count (occupancy query)
  t.partition = env_int("TG_PROBE_PARTITION", 1) != 0;   // regroup big probes into L2-sized partitions first (0 = never)
  t.parts = env_int("TG_PROBE_PARTS", 0);           // 0 = auto (probe_slices), at most TG_MAX_SLICES
  t.part_min_mb = env_int("TG_PROBE_PART_MIN_MB", 64);
  t.part_min_rows = env_int("TG_PROBE_PART_MIN_ROWS", 1 << 22);
  t.inplace = env_int("TG_PROBE_INPLACE", -1);      // -1 = by the last match fraction (kInplaceMinMatch), 0 / 1 = never / always
  return t;
}

// ---- L2 slices of the partitioned probe -------------------------------------------------------------------
// The partition pass cuts the table into P contiguous slices and probes one at a time; a slice only stays L2 resident while
// it is a fraction of L2, because the probe's input and output columns stream through the same cache.  On an H100 (50 MiB
// L2) the segment probe's time per row stops falling at slices of about a quarter of L2: 100 M probe rows against a 109 MiB
// table took 2.81 / 2.56 / 2.44 ms with slices of 27 / 13.6 / 6.8 MiB (tools/probe_slices.py --sweep slice, DESIGN.md §4.1).
static size_t l2_slice_target(int device) {
  static size_t cache[64];
  if (device >= 0 && device < 64 && cache[device]) return cache[device];
  int l2 = 0;
  if (cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, device) != cudaSuccess || l2 <= 0) { cudaGetLastError(); l2 = 50 << 20; }
  const size_t t = (size_t)l2 / 4;
  if (device >= 0 && device < 64) cache[device] = t;
  return t;
}
// P for a table of `table_bytes`: slices of at most l2_slice_target, at most TG_MAX_PARTS (TG_PROBE_PARTS > 0 overrides, up
// to TG_MAX_SLICES)
static int probe_slices(size_t table_bytes, int device, int parts_override) {
  if (parts_override > 0) return std::min(parts_override, TG_MAX_SLICES);
  const size_t target = l2_slice_target(device);
  return (int)std::min<size_t>((table_bytes + target - 1) / target, TG_MAX_PARTS);
}
// A U1 table the partitioned probe will slice is built dense enough for TG_MAX_PARTS slices of l2_slice_target, but no
// denser than this: longer linear-probe runs cost more than the L2 hits gain.  10 M keys, 100 M probe rows, 16 slices, home
// width 4 (tools/probe_slices.py --sweep shape, H100 at 400 W): load factor 0.5 4.30 ms (50 % match 4.51), 0.6 4.66 (5.57),
// 0.7 5.47 (7.80), against 4.80 (4.40) for the 0.35 table the build used to keep
static const double kMaxDenseLoad = 0.5;
// The in-place segment probe (probe_device) is taken while the last partitioned call of the handle matched at least this
// fraction of its rows: below it, tiles with misses are compacted and the hole fill moves more rows.  bench.py's join
// forced in place / not (tools/probe_slices.py --sweep match, H100 SXM at 700 W): 100 % match 3.63 / 4.25 ms, 99.9 % 3.79 /
// 4.34, 99 % 4.63 / 4.35, 50 % 5.63 / 4.33.
static const double kInplaceMinMatch = 0.995;

// ---- slice index of a sliced U1 table (SliceIndex, join_kernels.cuh) ----------------------------------------------------
// Load factor and mean keys per bucket: tools/scratch/pilot_lab.cu on bench.py's 10 M keys in 16 slices (H100 80GB HBM3,
// 700 W) — load factor 0.7 with 4 keys per bucket places every key with one-byte pilots (153 KiB of pilots per slice), and
// the in-place probe kernel with the pilots in shared memory took 1.70 ms against 2.07 ms on the linear-probe table.
// Denser or with bigger buckets, one-byte pilots leave keys unplaced (0.9 with 4–6 keys: 1–10 % of them); with more
// pilot bytes per CTA than kPidxMaxPilotBytes the kernel lost a third (204 KiB: 2.71–2.83 ms).  DESIGN.md §4.1.
static const double kPidxLoad = 0.7;
static const double kPidxKeysPerBucket = 4.0;
static const size_t kPidxMaxPilotBytes = 160 << 10;
static int enqueue_scan(JoinImpl* j, int64_t n, int64_t* nblocks_out);
static int build_slice_index(JoinImpl* j, const Slot* slots, unsigned long long nslots) {
  const ProbeTuning& tune = probe_tuning();
  const uint32_t P = (uint32_t)probe_slices((size_t)nslots * sizeof(Slot), j->device, tune.parts);
  if (P < 2) return TG_OK;
  DevBuf cnt;
  TG_TRY(cnt.ensure(j->device, (size_t)(TG_MAX_SLICES + 1) * 8));
  unsigned long long* pcnt = cnt.as<unsigned long long>();
  TG_CUDA(cudaMemsetAsync(pcnt, 0, (size_t)(TG_MAX_SLICES + 1) * 8, j->stream));
  k_pidx_part_count<<<grid_size(j->nsm, (int64_t)nslots, 256, 8), 256, 0, j->stream>>>(slots, nslots, P, pcnt);
  unsigned long long hc[TG_MAX_SLICES];
  TG_CUDA(cudaMemcpyAsync(hc, pcnt, P * 8, cudaMemcpyDeviceToHost, j->stream));
  TG_CUDA(cudaStreamSynchronize(j->stream));
  unsigned long long mx = 0;
  for (uint32_t p = 0; p < P; p++) mx = std::max(mx, hc[p]);
  SliceIndex ix{};
  ix.P = P;
  ix.S = (uint32_t)std::ceil((double)mx / kPidxLoad) + 1;
  ix.B = ((uint32_t)std::ceil((double)mx / kPidxKeysPerBucket) + 16) & ~15u;
  int optin = 0;
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, j->device);
  if (ix.B > kPidxMaxPilotBytes || ix.B + 16 > (uint32_t)optin) return TG_OK;   // slices too big: the linear-probe kernels
  ix.nbuf = 2 * ix.B <= kPidxMaxPilotBytes && 2 * (ix.B + 8) <= (uint32_t)optin ? 2 : 1;
  const size_t nb = (size_t)P * ix.B, ns = (size_t)P * ix.S;
  TG_TRY(j->pidx_slots.ensure(j->device, ns * sizeof(Slot)));
  TG_TRY(j->pidx_pilot.ensure(j->device, nb));
  DevBuf owner, list;
  TG_TRY(owner.ensure(j->device, ns * 4));
  TG_TRY(list.ensure(j->device, (size_t)(mx * P + 1) * 4));
  TG_TRY(j->tmp_cnt.ensure(j->device, (nb + 1) * 4));
  Slot* islots = j->pidx_slots.as<Slot>();
  ix.slots = islots;
  ix.pilot = j->pidx_pilot.as<uint8_t>();
  TG_CUDA(cudaMemsetAsync(j->pidx_pilot.p, (int)kPilotNone, nb, j->stream));
  TG_CUDA(cudaMemsetAsync(owner.p, 0xFF, ns * 4, j->stream));
  TG_CUDA(cudaMemsetAsync(j->tmp_cnt.p, 0, (nb + 1) * 4, j->stream));
  k_table_init<<<grid_size(j->nsm, (int64_t)ns, 256, 8), 256, 0, j->stream>>>(islots, ns, ns);   // all empty: no side slot
  const unsigned g = (unsigned)grid_size(j->nsm, (int64_t)nslots, 256, 8);
  k_pidx_bucket_count<<<g, 256, 0, j->stream>>>(slots, nslots, ix, j->tmp_cnt.as<uint32_t>());
  int64_t nblocks = 0;
  TG_TRY(enqueue_scan(j, (int64_t)nb, &nblocks));
  const unsigned long long* off = j->tmp_off.as<unsigned long long>();
  k_pidx_lists<<<g, 256, 0, j->stream>>>(slots, nslots, ix, off, j->tmp_cnt.as<uint32_t>(), list.as<uint32_t>());
  const unsigned gb = (unsigned)grid_size(j->nsm, (int64_t)nb, 256, 8);
  for (uint32_t size = kPidxMaxBucket; size >= 1; size--)   // largest buckets first
    k_pidx_place<<<gb, 256, 0, j->stream>>>(slots, ix, off, list.as<uint32_t>(), size, owner.as<uint32_t>(), j->pidx_pilot.as<uint8_t>());
  unsigned long long* bad = pcnt + TG_MAX_SLICES;
  k_pidx_write<<<g, 256, 0, j->stream>>>(slots, nslots, ix, islots, 0, bad);
  k_pidx_write<<<g, 256, 0, j->stream>>>(slots, nslots, ix, islots, 1, bad);
  j->stats.kernel_launches += 8 + kPidxMaxBucket;
  unsigned long long hbad = 0;
  TG_CUDA(cudaMemcpyAsync(&hbad, bad, 8, cudaMemcpyDeviceToHost, j->stream));
  TG_CUDA(cudaStreamSynchronize(j->stream));
  if (hbad) { j->pidx_slots.release(); j->pidx_pilot.release(); return TG_OK; }   // never seen: the linear-probe kernels
  j->pidx = ix;
  return TG_OK;
}


// Segment capacity of the in-place segment probe.  The fallback C0 = 1.05·n/P + 16 K leaves ≈ 330 K rows of slack per segment
// at 100 M rows and P = 16, about 130 σ of a uniform multinomial fill (σ ≈ sqrt(n/P) ≈ 2.5 K), and every unused row below the
// output count costs the hole fill a move of the whole output row.  So once the host has read the fills of a partitioned
// call of the handle that overflowed no segment, a call with the same P sizes its segments from that call's largest fill,
// scaled to its own rows: f = max_p fill_p · n / n_learned, C = f + 8·sqrt(f) + 4 K, never above C0.  The largest fill
// carries any systematic skew of the key distribution; a fresh batch from the same distribution moves each fill by about
// σ = sqrt(f), and the largest of P fills sits a few σ above the mean at most, so 8 σ overflows with a probability far
// below 1e-9 per call; the 4 K is a floor for small fills, where 8 σ is a few hundred rows.  A batch that overflows all the
// same is probed from its original input by the gated fallback (slower, never wrong), and a synced overflow drops the
// learned fills.  The lean segment probe keeps C0: it has no hole fill, so a tighter capacity saves it only memory.
static int64_t inplace_seg_cap(const JoinImpl* j, int P, int64_t n_main, int64_t C0) {
  if (j->seg_parts != P || j->seg_rows <= 0) return C0;
  const double f = (double)j->seg_fill_max * (double)n_main / (double)j->seg_rows;
  const int64_t C = ((int64_t)(f + 8.0 * std::sqrt(f)) + 4096 + 127) / 128 * 128;
  return std::min(C, C0);
}

// ---- build --------------------------------------------------------------------------------------------
static int build_table(JoinImpl* j) {
  const Side& b = j->build;
  int64_t n = j->bcols.rows;
  j->stats.build_rows = n;
  DevCols bview = j->bcols.view(b);
  TG_TRY(kernel_view(j, b, bview, n));
  KeySpec ks = j->build_key;
  if (j->multi_key) {
    TG_TRY(composite_key(j, b, bview, n, j->bkey_syn, j->bkey_syn_nn));
    ks.data = j->bkey_syn.p; ks.nulls = j->bkey_syn_nn.as<uint8_t>();
  } else { ks.data = bview.data[b.key_col]; ks.nulls = bview.nulls[b.key_col]; }
  unsigned long long nslots = (unsigned long long)((double)(n > 0 ? n : 1) / j->load_factor) + 32;
  // with the DEFAULT load factor a table bigger than TG_MAX_PARTS x 33 MB is made denser, down to load factor 0.5 (bounds the
  // memory of big G tables; U1 tables are resized for the L2 slices below, once the build knows it is U1)
  if (j->default_load_factor) {
    const unsigned long long fit = ((unsigned long long)TG_MAX_PARTS * (33ull << 20)) / sizeof(Slot);
    const unsigned long long dense = (unsigned long long)((double)(n > 0 ? n : 1) / 0.5) + 32;
    if (nslots > fit) nslots = std::max(fit, dense);
  }
  const unsigned long long align = kHomeWidth;   // whole homes; even, as runs continue by 32-byte pairs
  nslots &= ~(align - 1);
  if (nslots + 1 >= 0xFFFFFFFFull) return fail(TG_ERR_UNSUPPORTED, "build side too large for 32-bit slot ids");
  TG_TRY(j->table.ensure(j->device, (size_t)(nslots + 2) * sizeof(Slot)));   // + the side slot and a spare (probe_rows_u1)
  TG_TRY(j->row_slot.ensure(j->device, (size_t)(n + 1) * 4));
  TG_TRY(j->row_rank.ensure(j->device, (size_t)(n + 1) * 4));
  TG_TRY(j->scalars.ensure(j->device, 64));
  Slot* slots = j->table.as<Slot>();
  unsigned long long* sc = j->scalars.as<unsigned long long>();   // [0] distinct [1] maxcnt [2] cursor
  TG_CUDA(cudaEventRecord(j->ev0, j->stream));
  TG_CUDA(cudaMemsetAsync(sc, 0, 64, j->stream));
  k_table_init<<<grid_size(j->nsm, (int64_t)nslots + 1, 256, 8), 256, 0, j->stream>>>(slots, nslots + 1, nslots);
  j->stats.kernel_launches++;
  if (n > 0) {
    k_build_insert<<<grid_size(j->nsm, n, 256, 8), 256, 0, j->stream>>>(ks, bview, b.filter, n, slots, nslots,
                                                                  j->row_slot.as<uint32_t>(), j->row_rank.as<uint32_t>());
    j->stats.kernel_launches++;
  }
  k_table_stats<<<grid_size(j->nsm, (int64_t)nslots + 1, 256, 8), 256, 0, j->stream>>>(slots, nslots + 1, sc, sc + 1);
  j->stats.kernel_launches++;
  unsigned long long host_sc[3] = {0, 0, 0};
  TG_CUDA(cudaMemcpyAsync(host_sc, sc, 16, cudaMemcpyDeviceToHost, j->stream));
  TG_CUDA(cudaStreamSynchronize(j->stream));
  j->stats.distinct_keys = (int64_t)host_sc[0];
  j->stats.max_dup = (int64_t)host_sc[1];
  j->stats.table_slots = (int64_t)nslots;
  if (host_sc[1] > kCntMask) return fail(TG_ERR_UNSUPPORTED, "a single join key repeats more than 2^28 times on the build side");

  // choose the table mode.  U1: unique keys and the build side contributes at most its key (int64) and one
  // 8-byte NOT NULL payload column, and no build-side scan is needed afterwards.
  std::vector<int> payload;   // used build columns other than the key
  bool key_out = false;
  for (int c : b.used) { if (c == b.key_col) key_out = true; else if (std::find(payload.begin(), payload.end(), c) == payload.end()) payload.push_back(c); }
  bool u1 = host_sc[1] <= 1 && !j->need_scan && payload.size() <= 1 && (!key_out || j->build_key.kind == KEY_I64) && j->other.empty();
  if (u1 && payload.size() == 1) {
    int pc = payload[0];
    if (b.kelem[pc] != 8 || j->bcols.has_nulls[pc]) u1 = false;
  }
  bool sliced = false;   // a U1 table rebuilt dense for the partitioned probe: it gets a slice index (build_slice_index)
  j->pidx = SliceIndex{};
  j->pidx_slots.release(); j->pidx_pilot.release();
  if (u1 && j->default_load_factor && n > 0) {
    // the partitioned probe will slice this table: rebuild it dense enough for TG_MAX_PARTS L2-sized slices (probe_slices)
    const ProbeTuning& tune = probe_tuning();
    const size_t part_min = (size_t)tune.part_min_mb << 20;
    const unsigned long long dense = std::max<unsigned long long>((unsigned long long)TG_MAX_PARTS * l2_slice_target(j->device) / sizeof(Slot),
                                                                  (unsigned long long)((double)n / kMaxDenseLoad) + 32) & ~(align - 1);
    if (tune.partition && nslots * sizeof(Slot) > part_min && dense < nslots && dense * sizeof(Slot) > part_min) {
      nslots = dense;
      j->table.release();
      TG_TRY(j->table.ensure(j->device, (size_t)(nslots + 2) * sizeof(Slot)));   // + the side slot and a spare (probe_rows_u1)
      slots = j->table.as<Slot>();
      k_table_init<<<grid_size(j->nsm, (int64_t)nslots + 1, 256, 8), 256, 0, j->stream>>>(slots, nslots + 1, nslots);
      k_build_insert<<<grid_size(j->nsm, n, 256, 8), 256, 0, j->stream>>>(ks, bview, b.filter, n, slots, nslots,
                                                                    j->row_slot.as<uint32_t>(), j->row_rank.as<uint32_t>());
      j->stats.kernel_launches += 2;
      j->stats.table_slots = (int64_t)nslots;
      sliced = true;
    }
  }
  j->tv = TableView{slots, nslots, nullptr, 0, -1, TABLE_NONE};
  j->build_word_of_col.assign(b.ncols, -1);
  if (u1) {
    j->u1_payload_col = payload.empty() ? -1 : payload[0];
    if (n > 0) {
      const unsigned long long* pl = j->u1_payload_col >= 0 ? reinterpret_cast<const unsigned long long*>(bview.data[j->u1_payload_col]) : nullptr;
      k_build_scatter_u1<<<grid_size(j->nsm, n, 256, 8), 256, 0, j->stream>>>(j->row_slot.as<uint32_t>(), pl, n, slots);
      j->stats.kernel_launches++;
      if (sliced) TG_TRY(build_slice_index(j, slots, nslots));
    }
    j->tv.mode = TABLE_U1;
  } else {
    RowSpec rs{};
    int w = 0;
    bool any_nullable = false;
    std::vector<int> cols;
    for (int c : b.used) if (std::find(cols.begin(), cols.end(), c) == cols.end()) cols.push_back(c);
    for (int c : j->other_build_cols) if (std::find(cols.begin(), cols.end(), c) == cols.end()) cols.push_back(c);   // read by OtherCondition only
    if ((int)cols.size() + 1 > TG_MAX_COLS) return fail(TG_ERR_UNSUPPORTED, "too many build columns");
    for (int c : cols) {
      rs.col[w] = c; rs.elem_len[w] = b.kelem[c];
      rs.null_bit[w] = j->bcols.has_nulls[c] ? w : -1;
      any_nullable |= j->bcols.has_nulls[c] != 0;
      j->build_word_of_col[c] = w;
      w++;
    }
    rs.null_word = any_nullable ? w : -1;
    rs.nwords = w + (any_nullable ? 1 : 0);
    if (rs.nwords == 0) rs.nwords = 1;   // semi joins: no payload at all, keep a dummy word so offsets stay valid
    j->rowspec = rs;
    k_table_assign<<<grid_size(j->nsm, (int64_t)nslots + 1, 256, 8), 256, 0, j->stream>>>(slots, nslots + 1, sc + 2);
    j->stats.kernel_launches++;
    TG_TRY(j->rows_store.ensure(j->device, (size_t)(n + 1) * rs.nwords * 8));
    if (n > 0 && w > 0) {
      k_build_scatter_rows<<<grid_size(j->nsm, n, 256, 8), 256, 0, j->stream>>>(j->row_slot.as<uint32_t>(), j->row_rank.as<uint32_t>(), n, slots,
                                                                          bview, rs, j->rows_store.as<unsigned long long>());
      j->stats.kernel_launches++;
    }
    j->tv.mode = TABLE_G;
    j->tv.rows = j->rows_store.as<unsigned long long>();
    j->tv.row_words = rs.nwords;
    j->tv.null_word = rs.null_word;
    // compile OtherCondition against the row store
    j->dev_other = DevOther{};
    j->dev_other.n = (int)j->other.size();
    for (size_t q = 0; q < j->other.size(); q++) {
      const tg_other_item& it = j->other[q];
      OtherItemDev& o = j->dev_other.it[q];
      o.op = it.op; o.is_real = it.is_real; o.l_unsigned = it.lhs_unsigned; o.r_unsigned = it.rhs_unsigned;
      o.const_i64 = it.const_i64; o.const_f64 = it.const_f64;
      auto operand = [&](int side, int col, int32_t& src, int32_t& idx, int32_t& nbit) {
        nbit = -1;
        if (side < 0) { src = OSRC_CONST; idx = 0; }
        else if (side == 0) { src = OSRC_PROBE; idx = col; }
        else { src = OSRC_BUILD; idx = j->build_word_of_col[col]; nbit = rs.null_bit[idx]; }
      };
      operand(it.lhs_side, it.lhs_col, o.l_src, o.l_idx, o.l_null_bit);
      operand(it.rhs_side, it.rhs_col, o.r_src, o.r_idx, o.r_null_bit);
    }
  }
  if (j->need_scan) {
    TG_TRY(j->slot_used.ensure(j->device, (size_t)nslots + 1));
    TG_CUDA(cudaMemsetAsync(j->slot_used.p, 0, (size_t)nslots + 1, j->stream));
  }
  TG_CUDA(cudaEventRecord(j->ev1, j->stream));
  TG_CUDA(cudaStreamSynchronize(j->stream));
  TG_CUDA(cudaGetLastError());
  j->stats.build_ms = j->elapsed_ms();
  j->stats.table_mode = j->tv.mode;
  // valid keys = rows that landed in the table
  j->stats.build_valid_keys = -1;
  j->built = true;
  return TG_OK;
}

// ---- output plumbing -------------------------------------------------------------------------------------
static int ensure_result(JoinImpl* j, ResultBatch& rb, int64_t cap_rows, bool preserve, int64_t used_rows) {
  if ((int)rb.cols.size() != j->n_out) {
    rb.cols.clear(); rb.bitmaps.clear();
    for (int i = 0; i < j->n_out; i++) { rb.cols.emplace_back(new DevBuf()); rb.bitmaps.emplace_back(new DevBuf()); }
  }
  if ((int)j->out_ids.size() != j->n_out) {
    j->out_ids.clear();
    for (int i = 0; i < j->n_out; i++) j->out_ids.emplace_back(new DevBuf());
  }
  for (int c = 0; c < j->n_out; c++) {
    size_t bytes = (size_t)(cap_rows + 8) * j->out_elem[c];
    if (preserve) TG_TRY(rb.cols[c]->ensure_preserve(j->device, bytes, (size_t)used_rows * j->out_elem[c], j->stream));
    else TG_TRY(rb.cols[c]->ensure(j->device, bytes));
    if (j->out_elem[c] != kCellBytes) continue;
    // the ids of a call's output rows, laid out like its cells (every probe starts a fresh batch: ids index from row 0)
    if (preserve) TG_TRY(j->out_ids[c]->ensure_preserve(j->device, (size_t)(cap_rows + 8) * 8, (size_t)used_rows * 8, j->stream));
    else TG_TRY(j->out_ids[c]->ensure(j->device, (size_t)(cap_rows + 8) * 8));
  }
  return TG_OK;
}

// where the kernels write output column c of rb: the cells themselves, or the row ids of a DECIMAL column
static uint8_t* kernel_out(JoinImpl* j, ResultBatch& rb, int c) {
  return (j->out_elem[c] == kCellBytes ? j->out_ids[c] : rb.cols[c])->as<uint8_t>();
}

// Turn the row ids of every DECIMAL output column of rb into cells: rows [0, rb.rows), or [0, *dev_rows) when the fused
// paths leave the count on the device.  `probe_cells` = the view the probe ids index (nullptr: the build-side scan, where
// every probe-side cell is NULL); build ids index bcols, which hold the build rows for the handle's lifetime.  Enqueued
// behind the last kernel that moves rows, before anything can reuse the probe batch's buffers.
static int gather_cells(JoinImpl* j, ResultBatch& rb, const DevCols* probe_cells, const unsigned long long* dev_rows) {
  const bool probe_is_left = j->build_is_right;
  for (int o = 0; o < j->n_out; o++) {
    if (j->out_elem[o] != kCellBytes) continue;
    if (!dev_rows && rb.rows == 0) continue;
    const bool from_left = o < j->n_lused;
    const int col = from_left ? j->lused[o] : j->rused[o - j->n_lused];
    const void* src = from_left == probe_is_left ? (probe_cells ? probe_cells->data[col] : nullptr) : j->bcols.data[col]->p;
    launch_gather_cells(j->out_ids[o]->as<int64_t>(), rb.bitmaps[o]->as<uint8_t>(), src, rb.cols[o]->p, rb.rows, dev_rows,
                        j->nsm, j->stream);
    j->stats.kernel_launches++;
    j->stats.paths |= TG_JOIN_PATH_CELL_GATHER;
  }
  return TG_OK;
}

// which output columns can carry NULLs for this probe batch
static void out_nullable(const JoinImpl* j, const DevCols& pview, std::vector<char>& nullable) {
  nullable.assign(j->n_out, 0);
  bool probe_is_left = j->build_is_right;
  int n_l = j->n_lused;
  for (int o = 0; o < j->n_out; o++) {
    if (j->has_flag_col && o == j->n_out - 1) { nullable[o] = 0; continue; }
    bool from_left = o < n_l;
    bool from_probe = from_left == probe_is_left;
    int col = from_left ? j->lused[o] : j->rused[o - n_l];
    if (from_probe) nullable[o] = pview.nulls[col] != nullptr || j->need_scan;   // scan phase NULL-pads the probe side
    else nullable[o] = j->bcols.has_nulls[col] || j->probe_kind == PK_PROBE_OUTER;
  }
}

static void fill_outspec_probe(const JoinImpl* j, OutCols& oc) {
  bool probe_is_left = j->build_is_right;
  int n_l = j->n_lused;
  oc.n = j->n_out;
  for (int o = 0; o < j->n_out; o++) {
    OutSpec& sp = oc.spec[o];
    sp.elem_len = j->kout_elem[o];
    sp.null_bit = -1;
    if (j->has_flag_col && o == j->n_out - 1) { sp.src = SRC_FLAG; sp.idx = 0; continue; }
    bool from_left = o < n_l;
    int col = from_left ? j->lused[o] : j->rused[o - n_l];
    if (from_left == probe_is_left) { sp.src = SRC_PROBE_COL; sp.idx = col; continue; }
    if (j->tv.mode == TABLE_U1) { sp.src = col == j->build.key_col ? SRC_BUILD_KEY : SRC_BUILD_META; sp.idx = 0; }
    else { sp.src = SRC_BUILD_WORD; sp.idx = j->build_word_of_col[col]; sp.null_bit = j->rowspec.null_bit[sp.idx]; }
  }
}

// exclusive scan of the n counts in tmp_cnt into tmp_off (n + 1 entries), enqueued only; returns the block count
static int enqueue_scan(JoinImpl* j, int64_t n, int64_t* nblocks_out) {
  int64_t nblocks = (n + TG_SCAN_BLOCK * TG_SCAN_ITEMS - 1) / (TG_SCAN_BLOCK * TG_SCAN_ITEMS);
  TG_TRY(j->tmp_sums.ensure(j->device, (size_t)(nblocks + 2) * 8));
  TG_TRY(j->tmp_off.ensure(j->device, (size_t)(n + 2) * 8));
  k_scan_block_sums<<<(unsigned)nblocks, TG_SCAN_BLOCK, 0, j->stream>>>(j->tmp_cnt.as<uint32_t>(), n, j->tmp_sums.as<unsigned long long>());
  k_scan_sums<<<1, 1024, 0, j->stream>>>(j->tmp_sums.as<unsigned long long>(), nblocks);
  k_scan_write<<<(unsigned)nblocks, TG_SCAN_BLOCK, 0, j->stream>>>(j->tmp_cnt.as<uint32_t>(), n, j->tmp_sums.as<unsigned long long>(),
                                                                  j->tmp_off.as<unsigned long long>());
  j->stats.kernel_launches += 3;
  *nblocks_out = nblocks;
  return TG_OK;
}

static int scan_counts(JoinImpl* j, int64_t n, unsigned long long* total_out) {
  int64_t nblocks = 0;
  TG_TRY(enqueue_scan(j, n, &nblocks));
  TG_CUDA(cudaMemcpyAsync(total_out, j->tmp_sums.as<unsigned long long>() + nblocks, 8, cudaMemcpyDeviceToHost, j->stream));
  TG_CUDA(cudaStreamSynchronize(j->stream));
  return TG_OK;
}

// valid-byte streams → bitmaps for the nullable output columns
static int finish_bitmaps(JoinImpl* j, ResultBatch& rb, const std::vector<char>& nullable) {
  for (int c = 0; c < j->n_out; c++) {
    if (!nullable[c]) { rb.bitmaps[c]->release(); continue; }
    TG_TRY(rb.bitmaps[c]->ensure(j->device, (size_t)((rb.rows + 7) / 8) + 16));
    if (rb.rows) {
      launch_pack_bitmap(j->tmp_valid[c]->as<uint8_t>(), rb.rows, rb.bitmaps[c]->as<uint8_t>(), j->nsm, j->stream);
      j->stats.kernel_launches++;
    }
  }
  return TG_OK;
}

static bool fast_path_ok(const JoinImpl* j, const DevCols& pview) {
  if (j->tv.mode != TABLE_U1 || j->probe_kind != PK_INNER || j->need_scan) return false;
  if (j->probe.filter.n || j->probe_key.kind != KEY_I64 || j->probe_key.reject_negative) return false;
  if (pview.nulls[j->probe.key_col]) return false;
  for (int c : j->probe.used) if (j->probe.kelem[c] != 8 || pview.nulls[c]) return false;
  for (int e : j->kout_elem) if (e != 8) return false;
  return true;
}

// single-pass unique-key probe (k_probe_inner_uq): inner join, every build key unique, no OtherCondition, 8-byte output
// columns that cannot be NULL (probe used columns without a bitmap in this batch, build columns without NULLs)
static bool uq_path_ok(const JoinImpl* j, const DevCols& pview) {
  if (!env_int("TG_PROBE_UQ", 1) ||j->probe_kind != PK_INNER || j->need_scan || !j->other.empty() || j->stats.max_dup > 1) return false;
  if (j->tv.mode != TABLE_U1 && j->tv.mode != TABLE_G) return false;
  for (int c : j->probe.used) if (j->probe.kelem[c] != 8 || pview.nulls[c]) return false;
  for (int c : j->build.used) if (j->build.kelem[c] != 8 || j->bcols.has_nulls[c]) return false;
  for (int e : j->kout_elem) if (e != 8) return false;
  return true;
}

// classify the output columns of the fused fast path by the register that feeds them, with the destinations oc.data
// holds; false = shape not covered by the warp kernels (k_probe_inner_uq or the general path takes it)
static bool build_fast_out(const JoinImpl* j, const OutCols& oc, const DevCols& pview, FastOut& fo) {
  std::memset(&fo, 0, sizeof(fo));
  int pcol_of[TG_FAST_MAX_PCOLS];
  for (int c = 0; c < oc.n; c++) {
    const OutSpec& sp = oc.spec[c];
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(oc.data[c]);
    if (sp.src == SRC_BUILD_KEY || (sp.src == SRC_PROBE_COL && sp.idx == j->probe.key_col)) {
      if (fo.n_key_dst >= TG_FAST_MAX_KEYDST) return false;
      fo.key_dst[fo.n_key_dst++] = dst;
    } else if (sp.src == SRC_BUILD_META) {
      if (fo.n_meta_dst >= TG_FAST_MAX_METADST) return false;
      fo.meta_dst[fo.n_meta_dst++] = dst;
    } else if (sp.src == SRC_PROBE_COL) {
      for (int q = 0; q < fo.n_pcols; q++) if (pcol_of[q] == sp.idx) return false;   // same column twice
      if (fo.n_pcols >= TG_FAST_MAX_PCOLS) return false;
      int k = fo.n_pcols++;
      pcol_of[k] = sp.idx;
      fo.psrc[k] = reinterpret_cast<const unsigned long long*>(pview.data[sp.idx]);
      fo.pdst[k] = dst;
    } else return false;
  }
  return true;
}

// (NPC, NKD, NMD) dispatch: f(npc, nkd, nmd), the shape of fo as std::integral_constant values
template <typename F>
static int dispatch_shape(const FastOut& fo, F&& f) {
  using std::integral_constant;
#define TG_SHAPE(P, K, M) if (fo.n_pcols == P && fo.n_key_dst == K && fo.n_meta_dst == M) return f(integral_constant<int, P>(), integral_constant<int, K>(), integral_constant<int, M>());
#define TG_SHAPE_KM(P) TG_SHAPE(P, 0, 0) TG_SHAPE(P, 0, 1) TG_SHAPE(P, 1, 0) TG_SHAPE(P, 1, 1) TG_SHAPE(P, 2, 0) TG_SHAPE(P, 2, 1)
  TG_SHAPE_KM(0) TG_SHAPE_KM(1) TG_SHAPE_KM(2) TG_SHAPE_KM(3)
#undef TG_SHAPE_KM
#undef TG_SHAPE
  return fail(TG_ERR_CUDA, "internal: fused probe shape not instantiated");
}

// Launch the persistent fused probe kernel K with `ctas` CTAs at most, and one wave at most: TG_PROBE_CTAS_PER_SM, or the
// CTAs of K one SM holds (register-bound: queried once per instantiation, 3 if the query fails), per SM
template <auto K, typename... A>
static int launch_resident(JoinImpl* j, const char* name, const FastOut& fo, int64_t ctas, const ProbeTuning& t, A... args) {
  static int resident = 0;
  if (!resident) {
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, K, 256, 0) != cudaSuccess || nb < 1) { cudaGetLastError(); nb = 3; }
    resident = nb;
    if (getenv("TG_DEBUG")) fprintf(stderr, "[tidbgpu] %s<%d,%d,%d>: %d resident CTAs per SM\n", name, fo.n_pcols, fo.n_key_dst, fo.n_meta_dst, nb);
  }
  const int per_sm = t.ctas_per_sm > 0 ? t.ctas_per_sm : resident;
  K<<<(int)std::min<int64_t>(ctas, (int64_t)j->nsm * per_sm), 256, 0, j->stream>>>(args...);
  return TG_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// the fast paths write every output column from row rb.rows on, and no NULLs
static void bind_fast_outputs(JoinImpl* j, ResultBatch& rb, OutCols& oc) {
  for (int c = 0; c < j->n_out; c++) { oc.data[c] = kernel_out(j, rb, c) + (size_t)rb.rows * 8; oc.valid[c] = nullptr; if (rb.bitmaps[c]->p) rb.bitmaps[c]->release(); }
}

// wait for the probe and append the `got` = *cur rows it wrote to rb (copies enqueued before this land as well)
static int read_cursor(JoinImpl* j, ResultBatch& rb, const unsigned long long* cur, unsigned long long& got) {
  TG_CUDA(cudaMemcpyAsync(&got, cur, 8, cudaMemcpyDeviceToHost, j->stream));
  TG_CUDA(cudaStreamSynchronize(j->stream));
  TG_CUDA(cudaGetLastError());
  rb.rows += (int64_t)got;
  j->stats.output_rows += (int64_t)got;
  return TG_OK;
}

static void ensure_tmp_valid(JoinImpl* j) {
  if ((int)j->tmp_valid.size() != j->n_out) { j->tmp_valid.clear(); for (int i = 0; i < j->n_out; i++) j->tmp_valid.emplace_back(new DevBuf()); }
}

// ---- fused path: the warp kernels, behind an optional L2 partition pass ------------------------------------
// The partition pass of one call: P segments of C rows (P = 0: no pass, the direct launch), the n_main rows it scatters in
// tiles of ptile, and whether the segment probe runs in place
struct FusedPlan { int P; int64_t C; int64_t ptile, n_main; bool inplace; };

static FusedPlan fused_plan(const JoinImpl* j, const ResultBatch& rb, const int64_t* pkey, int64_t n, const FastOut& fo,
                            const ProbeTuning& tune, bool seg_input) {
  FusedPlan fp{};
  const size_t table_bytes = (size_t)j->tv.nslots * sizeof(Slot);
  bool src16 = aligned16(pkey);
  for (int c = 0; c < fo.n_pcols; c++) src16 = src16 && aligned16(fo.psrc[c]);
  fp.ptile = scatter_tile_rows(true, seg_input, 1 + fo.n_pcols);   // rows per scatter tile: 4096, or 1024
  fp.n_main = n / fp.ptile * fp.ptile;
  // L2 partition pass, count-free: regroup the probe rows by the TOP hash bits into P fixed-capacity segments of C rows.
  // slot = mulhi(hash, nslots) is monotone in the hash, so segment p only touches the contiguous table slice
  // [p/P, (p+1)/P) while the probe kernel sweeps the segment.  The pass trades 32 B/row of extra streaming traffic for
  // random HBM traffic, which only pays while a slice stays L2 resident (probe_slices; U1 tables are built dense
  // enough for that, build_table).  A skewed probe side that overflows a segment raises `flag`; the partitioned probe
  // launch then exits at once and the gated direct launch behind it does the work — no host round trip.
  // Fewer than ptile rows leave the scatter nothing to do: the whole input would be the tail, and the gated launch,
  // which probes the tail from row n_main on, reads n_main = 0 as "no tail".  Such a probe takes the direct launch.
  if (fp.n_main > 0 && tune.partition && src16 && n >= (int64_t)tune.part_min_rows && table_bytes > ((size_t)tune.part_min_mb << 20)) {
    fp.P = probe_slices(table_bytes, j->device, tune.parts);
    fp.C = ((int64_t)((double)fp.n_main / fp.P * 1.05) + 16384 + 127) / 128 * 128;
    if (!(fp.P >= 2 && (int64_t)fp.P * fp.C / 128 < (1ll << 31))) fp.P = 0;
  }
  // In place (k_probe_inner_u1_seg_inplace): the scatter writes the probe columns straight into the output columns, which
  // then take the segment layout, P·C rows.  It moves fewer bytes than the lean segment probe only when nearly every
  // 128-row tile matches in full, so it follows the match fraction of the last partitioned call whose count the host read
  // (the first call takes it); a mispredicted call is slower, never wrong.  Dense input and a fresh batch only: the
  // segment layout starts at the allocation.
  fp.inplace = fp.P && !seg_input && rb.rows == 0 && fo.n_key_dst >= 1 &&
               (tune.inplace >= 0 ? tune.inplace != 0 : j->seg_match >= kInplaceMinMatch);
  if (fp.inplace) fp.C = inplace_seg_cap(j, fp.P, fp.n_main, fp.C);
  return fp;
}

// the partition pass: the probe key and payload columns into P segments of C rows (the output columns themselves when in
// place, else part_cols); `seg` describes them, gated on the pass's overflow flag
static int scatter_segments(JoinImpl* j, const FusedPlan& fp, const int64_t* pkey, const FastOut& fo, const SegSpec* in_seg, SegSpec& seg) {
  const int nc = 1 + fo.n_pcols;
  if (!fp.inplace) {
    for (int c = 0; c < nc; c++) {
      if (!j->part_cols[c]) j->part_cols[c].reset(new DevBuf());
      TG_TRY(j->part_cols[c]->ensure(j->device, (size_t)fp.P * fp.C * 8 + 64));
    }
  }
  TG_TRY(j->part_scratch.ensure(j->device, (size_t)3 * TG_MAX_SLICES * 8 + 64));
  unsigned long long* cursors = j->part_scratch.as<unsigned long long>();      // fill count per segment
  long long* bases = reinterpret_cast<long long*>(cursors + TG_MAX_SLICES);   // first row of each segment
  unsigned long long* flag = cursors + 2 * TG_MAX_SLICES;                      // overflow
  PartDst d{};
  d.nparts = fp.P; d.ncols = nc;
  d.src[0] = pkey;
  for (int c = 0; c < fo.n_pcols; c++) d.src[1 + c] = fo.psrc[c];
  for (int c = 0; c < nc; c++)
    for (int q = 0; q < fp.P; q++) d.dst[q][c] = fp.inplace ? (c == 0 ? (void*)fo.key_dst[0] : (void*)fo.pdst[c - 1]) : j->part_cols[c]->p;
  k_segment_bases<<<1, 32, 0, j->stream>>>(cursors, bases, flag, fp.P, fp.C);
  j->stats.kernel_launches++;
  d.dst_base = bases; d.capacity = fp.C; d.overflow = flag;
  if (in_seg) { d.in_cnt = in_seg->cnt; d.in_cap = in_seg->cap; d.in_tiles_per_seg = (uint32_t)(in_seg->cap / fp.ptile); }
  TG_TRY(launch_partition_scatter<true>(j->device, j->stream, reinterpret_cast<const long long*>(pkey), nullptr, fp.n_main, d, cursors,
                                        &j->stats.kernel_launches, 0, &j->stats.paths));
  seg = SegSpec{cursors, (uint32_t)(fp.C / 128), 0, fp.C, flag};
  return TG_OK;
}

// the segment probe: in place, then the output made dense (the rows at or beyond R = *cur fill the holes below R); or lean,
// from the segment copies in part_cols
static int probe_segments(JoinImpl* j, const FusedPlan& fp, const FastOut& fo, unsigned long long* cur, const ProbeTuning& tune, const SegSpec& seg) {
  const int64_t rows = (int64_t)fp.P * fp.C, ntiles = rows / 128;
  j->stats.paths |= TG_JOIN_PATH_PROBE_SEG;
  if (fp.inplace) {
    TG_TRY(j->tile_cnt.ensure(j->device, (size_t)ntiles * 4 + 16));
    TG_TRY(j->tmp_cnt.ensure(j->device, (size_t)(2 * ntiles + 1) * 4));
    uint32_t* tile_cnt = j->tile_cnt.as<uint32_t>();
    TG_TRY(dispatch_shape(fo, [&](auto npc, auto nkd, auto nmd) -> int {
      if constexpr (nkd == 0) {
        return fail(TG_ERR_CUDA, "internal: the in-place segment probe needs an output fed by the join key");
      } else if (j->pidx.P == (uint32_t)fp.P) {
        // the slice index of this table, cut for this P: one CTA per SM holding nbuf slices' pilots and their mbarriers.
        // The shared-memory limit is an attribute of the current device, so it is raised on every launch, as the
        // aggregation does.
        const int smem = (int)(j->pidx.nbuf * (j->pidx.B + 8));
        TG_CUDA(cudaFuncSetAttribute(k_probe_inner_u1_seg_inplace_pidx<npc, nkd, nmd>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        k_probe_inner_u1_seg_inplace_pidx<npc, nkd, nmd><<<j->nsm, kPidxThreads, smem, j->stream>>>(rows, j->tv, j->pidx, fo, cur, seg, tile_cnt);
        j->stats.paths |= TG_JOIN_PATH_PROBE_INDEX;
        return TG_OK;
      } else {
        return launch_resident<k_probe_inner_u1_seg_inplace<npc, nkd, nmd>>(j, "k_probe_inner_u1_seg_inplace", fo, (rows / 128 + 7) / 8, tune,
                                                                            rows, j->tv, fo, cur, seg, tile_cnt);
      }
    }));
    k_inplace_holes<<<grid_size(j->nsm, ntiles, 256, 4), 256, 0, j->stream>>>(tile_cnt, ntiles, cur, seg.gate, j->tmp_cnt.as<uint32_t>());
    int64_t nblocks = 0;
    TG_TRY(enqueue_scan(j, 2 * ntiles, &nblocks));
    k_inplace_fill<<<j->nsm * 8, 256, 0, j->stream>>>(tile_cnt, ntiles, j->tmp_off.as<unsigned long long>(), cur, seg.gate, fo);
    j->stats.kernel_launches += 3;
    return TG_OK;
  }
  FastOut pf = fo;
  for (int c = 0; c < fo.n_pcols; c++) pf.psrc[c] = j->part_cols[1 + c]->as<unsigned long long>();
  // the 128-bit stores of the segment kernel need 16-byte aligned output columns: every caller passes a fresh
  // batch (rb.rows == 0), so the columns start at the allocation
  const int64_t* pkey = j->part_cols[0]->as<int64_t>();
  TG_TRY(dispatch_shape(pf, [&](auto npc, auto nkd, auto nmd) {
    return launch_resident<k_probe_inner_u1_seg_lean<npc, nkd, nmd>>(j, "k_probe_inner_u1_seg_lean", pf, (rows / 128 + 7) / 8, tune,
                                                                     pkey, rows, j->tv, pf, cur, seg);
  }));
  j->stats.kernel_launches++;
  return TG_OK;
}

// the warp kernel over the caller's input (n rows, segmented as in_seg when given).  gate != nullptr: it runs only when
// *gate is set (the partition pass overflowed a segment), except that dense rows from ungated_from on are probed either way
static int probe_direct(JoinImpl* j, const int64_t* pkey, int64_t n, const FastOut& fo, unsigned long long* cur, const ProbeTuning& tune,
                        const SegSpec* in_seg, const unsigned long long* gate, int64_t ungated_from) {
  const SegSpec seg = in_seg ? SegSpec{in_seg->cnt, in_seg->tiles_per_seg, gate != nullptr, in_seg->cap, gate, 0}
                             : SegSpec{nullptr, 0, gate != nullptr, 0, gate, ungated_from};
  constexpr int R = 4;
  const int64_t tiles = (n + 32 * R - 1) / (32 * R);
  j->stats.paths |= TG_JOIN_PATH_PROBE_DIRECT;
  TG_TRY(dispatch_shape(fo, [&](auto npc, auto nkd, auto nmd) {
    return launch_resident<k_probe_inner_u1_w<R, npc, nkd, nmd>>(j, "k_probe_inner_u1_w", fo, (tiles + 7) / 8, tune, pkey, n, j->tv, fo, cur, seg);
  }));
  j->stats.kernel_launches++;
  return TG_OK;
}

static int probe_fused(JoinImpl* j, const DevCols& pcells, const DevCols& pview, const KeySpec& ks, int64_t n, ResultBatch& rb,
                       bool sync_count, const SegSpec* in_seg, OutCols& oc, FastOut& fo) {
  const ProbeTuning& tune = probe_tuning();
  const int64_t* pkey = reinterpret_cast<const int64_t*>(ks.data);
  const FusedPlan fp = fused_plan(j, rb, pkey, n, fo, tune, in_seg != nullptr);
  TG_TRY(ensure_result(j, rb, fp.inplace ? std::max<int64_t>(n, (int64_t)fp.P * fp.C) : rb.rows + n, rb.rows > 0, rb.rows));
  bind_fast_outputs(j, rb, oc);
  build_fast_out(j, oc, pview, fo);
  unsigned long long* cur = j->out_cursor.as<unsigned long long>();
  TG_CUDA(cudaMemsetAsync(cur, 0, 8, j->stream));
  if (fp.P) {
    SegSpec seg;
    TG_TRY(scatter_segments(j, fp, pkey, fo, in_seg, seg));
    TG_TRY(probe_segments(j, fp, fo, cur, tune, seg));
    // gated fallback: probes the ORIGINAL input only after an overflow; the < ptile-row tail the scatter left behind
    // (dense input only) rides on the same launch — it is probed whatever the flag says, and appended at R
    TG_TRY(probe_direct(j, pkey, in_seg ? fp.n_main : n, fo, cur, tune, in_seg, seg.gate, fp.n_main < n ? fp.n_main : 0));
  } else if (n > 0) {
    TG_TRY(probe_direct(j, pkey, n, fo, cur, tune, in_seg, nullptr, 0));
  }
  TG_TRY(gather_cells(j, rb, &pcells, cur));   // after the hole fill and the gated fallback: *cur rows from row 0
  if (!sync_count) return TG_OK;
  unsigned long long got = 0, part[2 * TG_MAX_SLICES + 1];   // fill counts | segment bases | overflow flag
  const bool learn = fp.P && !in_seg;
  if (learn) TG_CUDA(cudaMemcpyAsync(part, j->part_scratch.p, sizeof(part), cudaMemcpyDeviceToHost, j->stream));
  TG_TRY(read_cursor(j, rb, cur, got));
  if (fp.P) j->seg_match = (double)got / (double)n;
  if (learn) {
    j->seg_parts = part[2 * TG_MAX_SLICES] ? 0 : fp.P;
    j->seg_rows = fp.n_main;
    j->seg_fill_max = (int64_t)*std::max_element(part, part + fp.P);
  }
  return TG_OK;
}

// single-pass path: inner join on unique build keys with filters / several payload columns (k_probe_inner_uq)
static int probe_uq(JoinImpl* j, const DevCols& pcells, const DevCols& pview, const KeySpec& ks, int64_t n, ResultBatch& rb, OutCols& oc) {
  TG_TRY(ensure_result(j, rb, rb.rows + n, rb.rows > 0, rb.rows));
  bind_fast_outputs(j, rb, oc);
  unsigned long long* cur = j->out_cursor.as<unsigned long long>();
  TG_CUDA(cudaMemsetAsync(cur, 0, 8, j->stream));
  if (n > 0) {
    int64_t tiles = (n + 256 * UQ_R - 1) / (256 * UQ_R);
    int grid = (int)std::min<int64_t>(tiles, (int64_t)j->nsm * 8);
    k_probe_inner_uq<<<grid, 256, 0, j->stream>>>(ks, pview, j->probe.filter, n, j->tv, oc, cur);
    j->stats.kernel_launches++;
    j->stats.paths |= TG_JOIN_PATH_PROBE_UQ;
  }
  TG_TRY(gather_cells(j, rb, &pcells, cur));
  // the output row count decides rb.rows (and the next append position): always needed on the host
  unsigned long long got = 0;
  return read_cursor(j, rb, cur, got);
}

// general path (any join type, NULLs, filters, duplicates): count → scan → write, in sub-batches
static int probe_general(JoinImpl* j, const DevCols& pcells, const DevCols& pview, const KeySpec& ks, int64_t n, ResultBatch& rb, OutCols& oc) {
  const Side& p = j->probe;
  std::vector<char> nullable;
  out_nullable(j, pview, nullable);
  ensure_tmp_valid(j);
  // valid bytes are produced for the whole call, so size them after counting all sub-batches: run count+scan
  // per sub-batch, remembering totals, then write.  Sub-batching keeps the temporaries bounded.
  for (int64_t lo = 0; lo < n; lo += kGeneralBatchRows) {
    int64_t m = std::min<int64_t>(kGeneralBatchRows, n - lo);
    DevCols sub = pview;
    if (lo) {
      if (lo % 8) return fail(TG_ERR_CUDA, "internal: sub-batch offset not byte aligned");
      for (int c = 0; c < p.ncols; c++) {
        if (sub.data[c]) sub.data[c] = reinterpret_cast<const uint8_t*>(sub.data[c]) + (size_t)lo * p.kelem[c];
        if (sub.nulls[c]) sub.nulls[c] += lo / 8;
      }
    }
    KeySpec sks = ks;
    if (j->multi_key) { sks.data = reinterpret_cast<const int64_t*>(ks.data) + lo; sks.nulls = ks.nulls + lo / 8; }
    else { sks.data = sub.data[p.key_col]; sks.nulls = sub.nulls[p.key_col]; }
    TG_TRY(j->tmp_cnt.ensure(j->device, (size_t)(m + 1) * 4));
    TG_TRY(j->tmp_slot.ensure(j->device, (size_t)(m + 1) * 4));
    k_probe_count<<<grid_size(j->nsm, m, 256, 8), 256, 0, j->stream>>>(sks, sub, p.filter, j->dev_other, m, j->tv, j->probe_kind, j->tmp_cnt.as<uint32_t>(),
                                                                 j->tmp_slot.as<uint32_t>(), j->need_scan ? j->slot_used.as<uint8_t>() : nullptr);
    j->stats.kernel_launches++;
    j->stats.paths |= TG_JOIN_PATH_PROBE_GENERAL;
    unsigned long long total = 0;
    TG_TRY(scan_counts(j, m, &total));
    if (total) {
      TG_TRY(ensure_result(j, rb, rb.rows + (int64_t)total, true, rb.rows));
      for (int c = 0; c < j->n_out; c++) {
        oc.data[c] = kernel_out(j, rb, c);
        oc.valid[c] = nullptr;
        if (nullable[c]) {
          TG_TRY(j->tmp_valid[c]->ensure_preserve(j->device, (size_t)(rb.rows + total) + 16, (size_t)rb.rows, j->stream));
          oc.valid[c] = j->tmp_valid[c]->as<uint8_t>();
        }
      }
      k_probe_write<<<grid_size(j->nsm, m, 256, 8), 256, 0, j->stream>>>(m, j->tmp_off.as<unsigned long long>(), j->tmp_slot.as<uint32_t>(),
                                                                   reinterpret_cast<const int64_t*>(sks.data), sks, j->tv, sub, oc, j->probe_kind,
                                                                   (unsigned long long)rb.rows, j->dev_other);
      j->stats.kernel_launches++;
      rb.rows += (int64_t)total;
      j->stats.output_rows += (int64_t)total;
    }
  }
  if ((int)rb.cols.size() != j->n_out) TG_TRY(ensure_result(j, rb, 8, false, 0));
  TG_TRY(finish_bitmaps(j, rb, nullable));
  TG_TRY(gather_cells(j, rb, &pcells, nullptr));
  TG_CUDA(cudaStreamSynchronize(j->stream));
  TG_CUDA(cudaGetLastError());
  return TG_OK;
}

// probe `n` device-resident rows; results are appended to rb (rb.rows advanced)
static int probe_device(JoinImpl* j, const DevCols& pcells, int64_t n, ResultBatch& rb, bool sync_count, const SegSpec* in_seg = nullptr) {
  const Side& p = j->probe;
  DevCols pview = pcells;
  TG_TRY(kernel_view(j, p, pview, n));
  j->stats.probe_rows += n;
  KeySpec ks = j->probe_key;
  if (j->multi_key) {
    if (in_seg) return fail(TG_ERR_UNSUPPORTED, "segmented device chunks: joins on several key columns take the general path");
    TG_TRY(composite_key(j, p, pview, n, j->pkey_syn, j->pkey_syn_nn));
    ks.data = j->pkey_syn.p; ks.nulls = j->pkey_syn_nn.as<uint8_t>();
  } else { ks.data = pview.data[p.key_col]; ks.nulls = pview.nulls[p.key_col]; }
  TG_TRY(j->out_cursor.ensure(j->device, 64));
  OutCols oc{};
  fill_outspec_probe(j, oc);
  FastOut fo{};
  // the output shape decides the path before any output is allocated: the fused warp kernels, else the single-pass
  // unique-key kernel, else the general path.  build_fast_out runs again once the output pointers are known.
  const bool fast = fast_path_ok(j, pview) && build_fast_out(j, oc, pview, fo);
  if (in_seg && !fast) return fail(TG_ERR_UNSUPPORTED, "segmented device chunks are only accepted by the fused fast path (unique build keys, <= 1 payload, no filters, an output shape the warp kernels cover)");
  if (fast) return probe_fused(j, pcells, pview, ks, n, rb, sync_count, in_seg, oc, fo);
  if (uq_path_ok(j, pview)) return probe_uq(j, pcells, pview, ks, n, rb, oc);
  return probe_general(j, pcells, pview, ks, n, rb, oc);
}

// ScanRowTable after the probe side is exhausted (hash_join_v2.go:877)
static int scan_build_side(JoinImpl* j, ResultBatch& rb) {
  const Side& b = j->build;
  int64_t n = j->bcols.rows;
  if (n == 0) { if ((int)rb.cols.size() != j->n_out) TG_TRY(ensure_result(j, rb, 8, false, 0)); return TG_OK; }
  DevCols bview = j->bcols.view(b);
  TG_TRY(kernel_view(j, b, bview, n));
  TG_TRY(j->tmp_cnt.ensure(j->device, (size_t)(n + 1) * 4));
  k_build_scan_count<<<grid_size(j->nsm, n, 256, 8), 256, 0, j->stream>>>(j->row_slot.as<uint32_t>(), j->slot_used.as<uint8_t>(), n, j->scan_mode, j->tmp_cnt.as<uint32_t>());
  j->stats.kernel_launches++;
  unsigned long long total = 0;
  TG_TRY(scan_counts(j, n, &total));
  std::vector<char> nullable(j->n_out, 0);
  bool probe_is_left = j->build_is_right;
  OutCols oc{};
  oc.n = j->n_out;
  ensure_tmp_valid(j);
  TG_TRY(ensure_result(j, rb, rb.rows + (int64_t)total, false, 0));
  for (int o = 0; o < j->n_out; o++) {
    bool from_left = o < j->n_lused;
    int col = from_left ? j->lused[o] : j->rused[o - j->n_lused];
    bool from_probe = from_left == probe_is_left;
    oc.spec[o].elem_len = j->kout_elem[o];
    oc.spec[o].null_bit = -1;
    oc.spec[o].src = from_probe ? SRC_PROBE_COL : SRC_BUILD_WORD;
    oc.spec[o].idx = col;
    nullable[o] = from_probe || j->bcols.has_nulls[col];
    oc.data[o] = kernel_out(j, rb, o);
    oc.valid[o] = nullptr;
    if (nullable[o]) { TG_TRY(j->tmp_valid[o]->ensure(j->device, (size_t)total + 16)); oc.valid[o] = j->tmp_valid[o]->as<uint8_t>(); }
  }
  if (total) {
    k_build_scan_write<<<grid_size(j->nsm, n, 256, 8), 256, 0, j->stream>>>(n, j->tmp_off.as<unsigned long long>(), bview, oc, 0ull);
    j->stats.kernel_launches++;
  }
  rb.rows = (int64_t)total;
  j->stats.output_rows += (int64_t)total;
  TG_TRY(finish_bitmaps(j, rb, nullable));
  TG_TRY(gather_cells(j, rb, nullptr, nullptr));
  TG_CUDA(cudaStreamSynchronize(j->stream));
  TG_CUDA(cudaGetLastError());
  return TG_OK;
}

static std::unique_ptr<ResultBatch> new_batch(JoinImpl* j) {
  std::lock_guard<std::mutex> lk(j->res_mu);
  if (!j->free_batches.empty()) {
    std::unique_ptr<ResultBatch> rb = std::move(j->free_batches.back());
    j->free_batches.pop_back();
    rb->rows = 0; rb->consumed = 0;
    return rb;
  }
  return std::unique_ptr<ResultBatch>(new ResultBatch());
}

static void queue_result(JoinImpl* j, std::unique_ptr<ResultBatch> rb) {
  if (rb->rows <= 0) { std::lock_guard<std::mutex> lk(j->res_mu); j->free_batches.push_back(std::move(rb)); return; }
  { std::lock_guard<std::mutex> lk(j->res_mu); j->results.push_back(std::move(rb)); }
  j->res_cv.notify_all();
}

// probe n rows into rb, timed into probe_ms; with sync_count = false the probe is left in flight and its time uncounted
static int timed_probe(JoinImpl* j, const DevCols& pview, int64_t n, ResultBatch& rb, bool sync_count, const SegSpec* seg = nullptr) {
  TG_CUDA(cudaEventRecord(j->ev0, j->stream));
  TG_TRY(probe_device(j, pview, n, rb, sync_count, seg));
  TG_CUDA(cudaEventRecord(j->ev1, j->stream));
  if (!sync_count) return TG_OK;
  TG_CUDA(cudaStreamSynchronize(j->stream));
  j->stats.probe_ms += j->elapsed_ms();
  return TG_OK;
}

// probe a batch of host rows (the staging st, or a big chunk when st = nullptr) and queue its result for *_next
static int probe_host_rows(JoinImpl* j, const HostStage* st, const tg_chunk* chk) {
  TG_TRY(upload_side(j, j->probe, st, chk, j->pcols_dev));
  std::unique_ptr<ResultBatch> rb = new_batch(j);
  TG_TRY(timed_probe(j, j->pcols_dev.view(j->probe), j->pcols_dev.rows, *rb, true));
  queue_result(j, std::move(rb));
  return TG_OK;
}

static int flush_probe_stage(JoinImpl* j) {
  if (j->pstage.rows == 0) return TG_OK;
  TG_TRY(probe_host_rows(j, &j->pstage, nullptr));
  j->pstage.reset();
  return TG_OK;
}

// tg_join_probe_dev(_seg): probe a device-resident chunk into dev_result; seg = the segment layout of its rows
static int probe_dev_chunk(JoinImpl* j, const tg_chunk* dev_chk, const SegSpec* seg, int64_t nseg, int64_t* out_rows,
                           void** out_cols, void** out_nulls) {
  DevCols pview;
  TG_TRY(probe_view(j, dev_chk, pview));
  const int64_t n = logical_rows(dev_chk);
  if (seg) {
    if (n != nseg * seg->cap) return fail(TG_ERR_INVALID, "column length must be nseg * seg_cap");
    if (n / 128 >= (1ll << 31)) return fail(TG_ERR_UNSUPPORTED, "segmented chunk too large");
  }
  if (!j->dev_result) j->dev_result.reset(new ResultBatch());
  ResultBatch& rb = *j->dev_result;
  rb.rows = 0; rb.consumed = 0;
  TG_TRY(timed_probe(j, pview, n, rb, out_rows != nullptr, seg));
  if (out_rows) *out_rows = rb.rows;
  for (int c = 0; c < j->n_out; c++) {
    if (out_cols) out_cols[c] = rb.cols[c]->p;
    if (out_nulls) out_nulls[c] = rb.bitmaps[c]->p;
  }
  return TG_OK;
}

}  // namespace tg

// ---------------------------------------------------------------------------------------------------
// C entry points
// ---------------------------------------------------------------------------------------------------
extern "C" {

int tg_join_supported(const tg_join_desc* desc) {
  tg_join shell;
  JoinImpl tmp(shell);
  return setup(&tmp, desc);
}

int tg_join_open(const tg_join_desc* desc, tg_join** out) {
  if (!out) return fail(TG_ERR_INVALID, "out is NULL");
  *out = nullptr;
  std::unique_ptr<tg_join> shell(new tg_join());
  std::unique_ptr<JoinImpl> j(new JoinImpl(*shell));
  TG_TRY(setup(j.get(), desc));
  int ndev = 0;
  TG_TRY(require_device("the GPU hash join", &ndev));
  if (j->device < 0 || j->device >= ndev) return fail(TG_ERR_INVALID, "device ordinal out of range");
  DeviceGuard g(j->device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed");
  TG_TRY(j->open(j->device, desc->stream));
  TG_CUDA(cudaStreamCreateWithFlags(&j->d2h_stream, cudaStreamNonBlocking));
  j->bstage.init(j->build.ncols); j->bcols.init(j->build.ncols);
  j->pstage.init(j->probe.ncols); j->pcols_dev.init(j->probe.ncols);
  shell->impl = j.release();
  *out = shell.release();
  return TG_OK;
}

int tg_join_build_push(tg_join* h, const tg_chunk* chk) {
  TG_LOCK(h, JoinImpl, j);
  if (j->built) return fail(TG_ERR_STATE, "build_push after build_finish");
  TG_TRY(validate_chunk(j->build.ncols, j->build.needed, j->build.elem, chk));
  return stage_append(j->bstage, j->build.needed, j->build.elem, chk);
}

int tg_join_build_push_dev(tg_join* h, const tg_chunk* chk) {
  TG_LOCK(h, JoinImpl, j);
  if (j->built) return fail(TG_ERR_STATE, "build_push after build_finish");
  if (j->bstage.rows) return fail(TG_ERR_STATE, "host and device build pushes cannot be mixed");
  TG_TRY(validate_chunk(j->build.ncols, j->build.needed, j->build.elem, chk));
  return devchunk_append(j, chk, j->build, j->bcols);
}

int tg_join_build_finish(tg_join* h) {
  TG_LOCK(h, JoinImpl, j);
  if (j->built) return fail(TG_ERR_STATE, "build_finish called twice");
  if (j->bstage.rows) { TG_TRY(upload_side(j, j->build, &j->bstage, nullptr, j->bcols)); }
  int rc = build_table(j);
  // pinned staging of the build side is no longer needed
  j->bstage.init(j->build.ncols);
  return rc;
}

int tg_join_probe_push(tg_join* h, const tg_chunk* chk) {
  TG_LOCK(h, JoinImpl, j);
  if (!j->built) return fail(TG_ERR_STATE, "probe_push before build_finish");
  if (j->probe_finished.load()) return fail(TG_ERR_STATE, "probe_push after probe_finish");
  TG_TRY(validate_chunk(j->probe.ncols, j->probe.needed, j->probe.elem, chk));
  int64_t n = logical_rows(chk);
  if (n == 0) return TG_OK;
  if (!chk->sel && n >= kDirectPushRows) {
    TG_TRY(flush_probe_stage(j));
    return probe_host_rows(j, nullptr, chk);
  }
  TG_TRY(stage_append(j->pstage, j->probe.needed, j->probe.elem, chk));
  if (j->pstage.rows >= kStageBatchRows) TG_TRY(flush_probe_stage(j));
  return TG_OK;
}

int tg_join_probe_finish(tg_join* h) {
  TG_LOCK(h, JoinImpl, j);
  if (!j->built) return fail(TG_ERR_STATE, "probe_finish before build_finish");
  if (j->probe_finished.load()) return TG_OK;
  TG_TRY(flush_probe_stage(j));
  if (j->need_scan) {
    std::unique_ptr<ResultBatch> rb = new_batch(j);
    TG_TRY(scan_build_side(j, *rb));
    queue_result(j, std::move(rb));
  }
  { std::lock_guard<std::mutex> lk(j->res_mu); j->probe_finished.store(true); }
  j->res_cv.notify_all();
  return TG_OK;
}

static int join_next_impl(tg_join* h, tg_mut_chunk* out, int64_t max_rows, int64_t* nrows, bool wait) {
  if (!h) return fail(TG_ERR_INVALID, "handle is NULL");
  if (h->closed.load()) return fail(TG_ERR_CANCELLED, "handle is closed");
  if (!out || !nrows) return fail(TG_ERR_INVALID, "out / nrows is NULL");
  *nrows = 0;
  std::unique_lock<std::mutex> lock__(h->res_mu);
  if (h->closed.load() || !h->impl) return fail(TG_ERR_CANCELLED, "handle is closed");
  JoinImpl* j = h->impl;
  if (out->ncols != j->n_out) return fail(TG_ERR_INVALID, "output chunk column count does not match the join schema");
  for (int c = 0; c < j->n_out; c++) if (out->cols[c].elem_len != j->out_elem[c]) return fail(TG_ERR_INVALID, "output column elem_len mismatch");
  tg::DeviceGuard guard__(j->device);
  if (!guard__.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed (no usable CUDA device)");
  for (;;) {
    while (!j->results.empty() && j->results.front()->consumed >= j->results.front()->rows) {
      if (j->win_batch == j->results.front().get()) { j->win_batch = nullptr; j->win_lo = j->win_hi = 0; }
      j->free_batches.push_back(std::move(j->results.front()));
      j->results.pop_front();
    }
    if (!j->results.empty()) break;
    if (!wait || j->probe_finished.load()) return TG_OK;   // 0 rows: EOF iff probe_finish was called, else "push more"
    h->res_cv.wait(lock__);
    if (h->closed.load() || !h->impl) return fail(TG_ERR_CANCELLED, "handle is closed");
  }
  cudaStream_t cstream = j->d2h_stream;
  ResultBatch& rb = *j->results.front();
  int64_t want = std::min<int64_t>(std::min<int64_t>(max_rows, out->capacity_rows), rb.rows - rb.consumed);
  if (want <= 0) return TG_OK;
  // every output column is checked before the first copy is enqueued: a rejected call writes nothing
  TG_TRY(check_out_columns(rb.bitmaps, j->out_elem, out));
  // any RequiredRows >= 1 is served (LIMIT 1, MaxOneRow): the result's bit-packed NULL bitmaps are re-aligned on the host
  // when the read cursor is not on a byte boundary (download_bitmaps)
  int64_t lo = rb.consumed;
  // row bytes of all columns, for the small-request window
  size_t row_bytes = 0;
  for (int c = 0; c < j->n_out; c++) row_bytes += j->out_elem[c];
  if (want >= 64 * 1024) {
    for (int c = 0; c < j->n_out; c++) {
      size_t el = j->out_elem[c];
      TG_CUDA(cudaMemcpyAsync(out->cols[c].data, rb.cols[c]->as<uint8_t>() + (size_t)lo * el, (size_t)want * el, cudaMemcpyDeviceToHost, cstream));
      j->d2h_bytes += (int64_t)want * el;
    }
  } else {
    // serve from a pinned window of up to kNextWindowRows rows fetched with one copy per column
    if (j->win_batch != &rb || lo < j->win_lo || lo + want > j->win_hi) {
      int64_t wn = std::min<int64_t>(kNextWindowRows, rb.rows - lo);
      TG_TRY(j->win.reserve((size_t)wn * row_bytes));
      size_t offb = 0;
      for (int c = 0; c < j->n_out; c++) {
        size_t el = j->out_elem[c];
        TG_CUDA(cudaMemcpyAsync(j->win.p + offb, rb.cols[c]->as<uint8_t>() + (size_t)lo * el, (size_t)wn * el, cudaMemcpyDeviceToHost, cstream));
        j->d2h_bytes += (int64_t)wn * el;
        offb += (size_t)wn * el;
      }
      TG_CUDA(cudaStreamSynchronize(cstream));
      j->win_batch = &rb; j->win_lo = lo; j->win_hi = lo + wn;
    }
    int64_t wn = j->win_hi - j->win_lo;
    size_t offb = 0;
    for (int c = 0; c < j->n_out; c++) {
      size_t el = j->out_elem[c];
      std::memcpy(out->cols[c].data, j->win.p + offb + (size_t)(lo - j->win_lo) * el, (size_t)want * el);
      offb += (size_t)wn * el;
    }
  }
  int64_t bitmap_bytes = 0;
  TG_TRY(download_bitmaps(rb.bitmaps, out, lo, want, cstream, &bitmap_bytes));
  j->d2h_bytes += bitmap_bytes;
  rb.consumed += want;
  *nrows = want;
  return TG_OK;
}

int tg_join_probe_rewind(tg_join* h) {
  TG_LOCK(h, JoinImpl, j);
  if (!j->built) return fail(TG_ERR_STATE, "rewind before build_finish");
  if (j->need_scan) return fail(TG_ERR_UNSUPPORTED, "joins that scan the build side afterwards cannot be re-probed (used flags accumulate)");
  j->pstage.reset();
  std::lock_guard<std::mutex> lk(j->res_mu);
  while (!j->results.empty()) { j->free_batches.push_back(std::move(j->results.front())); j->results.pop_front(); }
  j->win_batch = nullptr; j->win_lo = j->win_hi = 0;
  j->probe_finished.store(false);
  return TG_OK;
}

int tg_join_next(tg_join* h, tg_mut_chunk* out, int64_t max_rows, int64_t* nrows) { return join_next_impl(h, out, max_rows, nrows, false); }
int tg_join_next_wait(tg_join* h, tg_mut_chunk* out, int64_t max_rows, int64_t* nrows) { return join_next_impl(h, out, max_rows, nrows, true); }

int tg_join_probe_dev(tg_join* h, const tg_chunk* dev_chk, int64_t* out_rows, void** out_cols, void** out_nulls) {
  TG_LOCK(h, JoinImpl, j);
  if (!j->built) return fail(TG_ERR_STATE, "probe before build_finish");
  return probe_dev_chunk(j, dev_chk, nullptr, 0, out_rows, out_cols, out_nulls);
}

int tg_join_probe_dev_seg(tg_join* h, const tg_chunk* dev_chk, const int64_t* seg_cnt_dev, int32_t nseg, int64_t seg_cap,
                          int64_t* out_rows, void** out_cols, void** out_nulls) {
  TG_LOCK(h, JoinImpl, j);
  if (!j->built) return fail(TG_ERR_STATE, "probe before build_finish");
  if (!seg_cnt_dev || nseg < 1 || seg_cap < 1024 || seg_cap % 1024) return fail(TG_ERR_INVALID, "seg_cnt_dev required; seg_cap must be a positive multiple of 1024");
  SegSpec seg{reinterpret_cast<const unsigned long long*>(seg_cnt_dev), (uint32_t)(seg_cap / 128), 0, seg_cap, nullptr};
  return probe_dev_chunk(j, dev_chk, &seg, nseg, out_rows, out_cols, out_nulls);
}

int tg_join_get_stats(tg_join* h, tg_join_stats* out) {
  TG_LOCK(h, JoinImpl, j);
  if (!out) return fail(TG_ERR_INVALID, "out is NULL");
  TG_CUDA(cudaStreamSynchronize(j->stream));
  *out = j->stats;
  out->d2h_bytes = j->d2h_bytes.load();
  return TG_OK;
}

int tg_join_close(tg_join* h) {
  if (!h) return TG_OK;
  bool was = h->closed.exchange(true);
  if (was) return TG_OK;
  // wake a consumer parked in tg_join_next_wait; notifying under res_mu closes the window between its predicate check
  // and its wait (it holds res_mu across both)
  { std::lock_guard<std::mutex> rlock(h->res_mu); h->res_cv.notify_all(); }
  {
    // waits for an in-flight push and an in-flight next; later calls see `closed`
    std::lock_guard<std::mutex> lock(h->mu);
    std::lock_guard<std::mutex> rlock(h->res_mu);
    JoinImpl* j = h->impl;
    h->impl = nullptr;
    if (j) {
      DeviceGuard g(j->device);
      if (j->stream) cudaStreamSynchronize(j->stream);
      if (j->d2h_stream) { cudaStreamSynchronize(j->d2h_stream); cudaStreamDestroy(j->d2h_stream); }
      j->results.clear();
      j->free_batches.clear();
      j->dev_result.reset();
      j->release();
      cudaGetLastError();
      delete j;
    }
    h->res_cv.notify_all();
  }
  bury_handle(h);   // the shell stays readable for late callers; freed after kGraveyardDepth further closes
  return TG_OK;
}

}  // extern "C"
