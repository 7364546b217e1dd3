// vec_string.cu — VecEval over var-length string columns: the six comparisons and LIKE / NOT LIKE, as a column result
// (tg_vec_compare_string, tg_vec_like) or as STRING items of a Selection CNF (tg_vec_filter_ex2).
//
// Replaces (pkg/expression): builtin{LT,LE,GT,GE,EQ,NE}StringSig.vecEvalInt (builtin_compare_vec_generated.go,
// types.CompareString) and builtinLikeSig.vecEvalInt (builtin_like_vec.go) with a constant pattern, under the binary,
// *_bin and utf8mb4_0900_bin collators (string.cuh).
//
// Layout: a warp takes a tile of 32 consecutive rows, lane l row base + l, and loads their offsets.  When every row of
// the tile has good offsets and the tile's bytes fit kStageCap, the warp copies them into its shared-memory buffer with
// 16-byte loads (byte loads for the unaligned head and tail) and each lane evaluates its row from there; otherwise, and
// for every row reached through a sel vector, lanes read their rows from global memory.  Column-against-column items
// stage both operands, one buffer each.
#include "vec.cuh"
#include "string.cuh"

namespace tg {

static constexpr int kStageCap = 2048;                 // bytes of one warp's buffer
static constexpr int kStageStride = kStageCap + 16;    // + room to keep the global alignment mod 16
static constexpr int kWarpsPerBlock = 8;

// one STRING item: a comparison (op, lhs `op` rhs column or the constant k) or a LIKE match of lhs against the compiled
// pattern (pw, pt, klen entries).  Device pointers into the call's one constant upload.
struct StrItem {
  int32_t kind, op, lhs, rhs;
  int32_t pad_space;    // COLL_PAD_BIN comparison: trailing 0x20 cut (k is already cut)
  int32_t runes;        // LIKE over runes; 0: over bytes (binary, or a pattern only bytes can match: see like_bytes_ok)
  int64_t klen;
  const uint8_t* k;
  const int32_t* pw;
  const uint8_t* pt;
};
struct StrFilter { int32_t n, pad; StrItem items[TG_MAX_FILTER]; };

// a lane's row of column c: good offsets, and where its bytes are
struct RowRef { const uint8_t* p; int64_t len; bool good; };

// Copy `len` bytes from src into buf (16-byte aligned, kStageStride bytes) at the same alignment mod 16; the whole warp
// calls it.  Returns where src[0] landed.
__device__ __forceinline__ const uint8_t* stage_bytes(uint8_t* buf, const uint8_t* src, int64_t len, int lane) {
  const int mis = (int)(reinterpret_cast<uintptr_t>(src) & 15);
  uint8_t* dst = buf + mis;
  int64_t head = (16 - mis) & 15;
  if (head > len) head = len;
  if (lane < head) dst[lane] = src[lane];
  const int64_t nvec = (len - head) >> 4;
  const uint4* vs = reinterpret_cast<const uint4*>(src + head);
  uint4* vd = reinterpret_cast<uint4*>(dst + head);
  for (int64_t v = lane; v < nvec; v += 32) vd[v] = __ldcs(vs + v);
  const int64_t done = head + (nvec << 4);
  if (lane < len - done) dst[done + lane] = src[done + lane];
  __syncwarp();
  return dst;
}

// The row bytes of column c for the warp's 32 rows (lane's row p, in = the lane has a row).  Checks the offsets of every
// row that is in, and stages the tile into buf when `tile` (rows base .. base + 31 in order, no sel) allows it.
__device__ __forceinline__ RowRef load_rows(const StrCols& sc, int c, int64_t nphys, int64_t p, bool in, bool tile,
                                            int64_t base_row, int64_t n, uint8_t* buf, int lane, bool& bad) {
  const int64_t* offs = sc.offs[c];
  const int64_t lo = offs[0], hi = offs[nphys];
  int64_t o0 = 0, o1 = 0;
  if (in) { o0 = offs[p]; o1 = offs[p + 1]; }
  const bool good = in && lo <= o0 && o0 <= o1 && o1 <= hi;
  bad |= in && !good;
  const uint8_t* g = sc.data[c] - sc.base[c];
  RowRef r{g + o0, o1 - o0, good};
  if (tile && __all_sync(0xffffffffu, good || !in)) {
    const int last = (int)(n - base_row < 32 ? n - base_row - 1 : 31);
    const int64_t s0 = __shfl_sync(0xffffffffu, o0, 0), s1 = __shfl_sync(0xffffffffu, o1, last);
    if (s1 - s0 <= kStageCap) {
      const uint8_t* d = stage_bytes(buf, g + s0, s1 - s0, lane);
      r.p = d + (o0 - s0);
    }
  }
  return r;
}

// every STRING item of sf for the warp's rows; true when each is non-NULL true (lanes without a row get false)
__device__ __forceinline__ bool eval_str_items(const StrFilter& sf, const StrCols& sc, const DevCols& cols, int64_t nphys,
                                               int64_t p, bool in, bool tile, int64_t base_row, int64_t n, uint8_t* buf0,
                                               uint8_t* buf1, int lane, bool& bad) {
  bool s = in;
  for (int q = 0; q < sf.n; q++) {
    const StrItem& it = sf.items[q];
    const RowRef a = load_rows(sc, it.lhs, nphys, p, in, tile, base_row, n, buf0, lane, bad);
    const uint8_t* an = cols.nulls[it.lhs];
    bool valid = a.good && (!an || bit_not_null(an, p));
    bool r = false;
    if (it.kind == TG_STR_CMP) {
      const uint8_t* kp = it.k;
      int64_t klen = it.klen;
      if (it.rhs >= 0) {
        const RowRef b = load_rows(sc, it.rhs, nphys, p, in, tile, base_row, n, buf1, lane, bad);
        const uint8_t* bn = cols.nulls[it.rhs];
        valid = valid && b.good && (!bn || bit_not_null(bn, p));
        kp = b.p; klen = b.len;
        if (valid && it.pad_space) klen = str_trim_len(kp, klen);
      }
      if (valid) {
        const int64_t alen = it.pad_space ? str_trim_len(a.p, a.len) : a.len;
        r = apply_cmp(it.op, str_cmp_bytes(a.p, alen, kp, klen));
      }
    } else if (valid) {
      r = it.runes ? like_match<true>(a.p, a.len, it.pw, it.pt, it.klen) : like_match<false>(a.p, a.len, it.pw, it.pt, it.klen);
      if (it.kind == TG_STR_NOT_LIKE) r = !r;
    }
    s &= valid && r;
    __syncwarp();   // the buffers are refilled by the next item
  }
  return s;
}

// COLUMN = false: tg_vec_filter_ex2, selected[p] = every STRING item (sf), then every DECIMAL item (d), then the INT /
// REAL items (f) are non-NULL true; the STRING and DECIMAL items are evaluated at every row, so every offset and cell
// is checked (*bad_offs, *bad_cell).  COLUMN = true: tg_vec_compare_string / tg_vec_like, one STRING item, result[i] =
// its value (0 under NULL) and its validity bits.
template <bool COLUMN>
__global__ void __launch_bounds__(256)
k_vec_string(StrCols sc, DevCols cols, const __grid_constant__ StrFilter sf, const __grid_constant__ DecFilter d,
             DevFilter f, const long long* __restrict__ sel, int64_t nsel, int64_t nphys, uint8_t* __restrict__ selected,
             unsigned long long* count, long long* __restrict__ result, uint8_t* __restrict__ rnulls,
             unsigned int* __restrict__ bad_offs, unsigned int* __restrict__ bad_cell) {
  extern __shared__ __align__(16) uint8_t smem[];   // one buffer per warp, a second one when an item has two columns
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  uint8_t* buf0 = smem + (size_t)wib * kStageStride;
  uint8_t* buf1 = buf0 + (size_t)kWarpsPerBlock * kStageStride;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n = sel ? nsel : nphys;
  bool bad = false, malformed = false;
  unsigned long long local = 0;
  for (int64_t base = warp * 32; base < n; base += nwarps * 32) {
    const int64_t i = base + lane;
    const bool in = i < n;
    const int64_t p = in ? (sel ? sel[i] : i) : 0;
    bool s = eval_str_items(sf, sc, cols, nphys, p, in, sel == nullptr, base, n, buf0, buf1, lane, bad);
    if (COLUMN) {
      const StrItem& it = sf.items[0];
      const uint8_t* an = cols.nulls[it.lhs];
      const uint8_t* bn = it.rhs >= 0 ? cols.nulls[it.rhs] : nullptr;
      const bool valid = in && (!an || bit_not_null(an, p)) && (!bn || bit_not_null(bn, p));
      if (in) __stcs(result + i, s ? 1ll : 0ll);
      store_valid_word(rnulls, base, n, __ballot_sync(0xffffffffu, valid), lane);
    } else if (in) {
      s = eval_dec_items(d, cols, p, malformed) && s;
      s = s && eval_filter(f, cols, p);
      selected[p] = s ? 1 : 0;
      local += s;
    }
  }
  if (!COLUMN) {
    for (int o = 16; o; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if (lane == 0 && local) atomicAdd(count, local);
  }
  if (bad) *bad_offs = 1u;
  if (malformed) *bad_cell = 1u;
}

// TG_TYPE_VARCHAR, VARSTRING, STRING and the BLOB / TEXT types (ENUM, SET, JSON and BIT are var-length, not strings)
static bool is_string_type(int32_t tp) {
  return tp == TG_TYPE_VARCHAR || tp == TG_TYPE_VARSTRING || tp == TG_TYPE_STRING ||
         (tp >= TG_TYPE_TINY_BLOB && tp <= TG_TYPE_BLOB);
}

// the checks of a string operand column that need no device
static int check_str_column(const tg_column& c, int on_device) {
  if (c.elem_len != -1 || !c.offsets) return fail(TG_ERR_INVALID, "a string operand column is var-length: elem_len -1 and offsets");
  if (c.length < 0) return fail(TG_ERR_INVALID, "negative column length");
  if (on_device) {
    if (reinterpret_cast<uintptr_t>(c.offsets) & 7) return fail(TG_ERR_INVALID, "device string offsets must be 8-byte aligned");
    if (c.length > 0 && !c.data) return fail(TG_ERR_INVALID, "string operand column without data");
    return TG_OK;
  }
  if (c.offsets[c.length] < c.offsets[0]) return fail(TG_ERR_INVALID, "string column offsets[length] < offsets[0]");
  if (c.offsets[c.length] > c.offsets[0] && !c.data) return fail(TG_ERR_INVALID, "string operand column without data");
  return TG_OK;
}

// A pattern that matches over bytes exactly as over runes: ASCII literals and '%' only.  An ASCII byte is always a whole
// rune and never part of another one, so a literal matches at the same places either way and '%' can only stop on a
// rune boundary; '_' (one rune, several bytes) and non-ASCII literals need the rune walk.
static bool like_bytes_ok(const std::vector<int32_t>& w, const std::vector<uint8_t>& t, int64_t n) {
  for (int64_t i = 0; i < n; i++)
    if (t[i] == PAT_ONE || (t[i] == PAT_MATCH && (w[i] < 0 || w[i] >= 0x80))) return false;
  return true;
}

// The STRING items of a call, checked and prepared on the host: constants cut when the collation cuts trailing
// spaces, patterns compiled, all of it in one blob uploaded once (item pointers hold blob offsets until then).
struct StrPrep {
  StrFilter sf{};
  std::vector<uint8_t> blob;
  DevBuf dev;
  size_t put(const void* p, size_t bytes) {
    const size_t at = (blob.size() + 15) & ~(size_t)15;
    blob.resize(at + bytes);
    if (bytes) std::memcpy(blob.data() + at, p, bytes);
    return at;
  }
  // item q of sf over columns lhs (rhs): a comparison (kind TG_STR_CMP) or a LIKE
  int add(int kind, int op, int lhs, int rhs, int32_t collation, const uint8_t* bytes, int64_t len, int32_t escape) {
    if (kind < TG_STR_CMP || kind > TG_STR_NOT_LIKE) return fail(TG_ERR_INVALID, "unknown string item kind");
    const int coll = coll_of_id(collation);
    if (coll == COLL_NONE) return fail(TG_ERR_UNSUPPORTED, "string collation not offloaded (binary, *_bin and utf8mb4_0900_bin are)");
    if (kind == TG_STR_CMP && (op < TG_CMP_LT || op > TG_CMP_NE)) return fail(TG_ERR_INVALID, "unknown comparison");
    if (kind != TG_STR_CMP && (escape < 0 || escape > 255)) return fail(TG_ERR_INVALID, "LIKE escape must be a byte 0..255");
    const bool has_const = kind != TG_STR_CMP || rhs < 0;
    if (has_const && (len < 0 || (len > 0 && !bytes))) return fail(TG_ERR_INVALID, "string constant / pattern: negative length or NULL bytes");
    StrItem& it = sf.items[sf.n++];
    it.kind = kind; it.op = op; it.lhs = lhs; it.rhs = kind == TG_STR_CMP ? rhs : -1;
    it.pad_space = kind == TG_STR_CMP && coll == COLL_PAD_BIN;
    if (kind == TG_STR_CMP) {
      if (rhs < 0) {
        it.klen = it.pad_space ? str_trim_len(bytes, len) : len;
        it.k = reinterpret_cast<const uint8_t*>(put(bytes, (size_t)it.klen));
      }
      return TG_OK;
    }
    std::vector<int32_t> w((size_t)len + 1);
    std::vector<uint8_t> t((size_t)len + 1);
    const bool runes = coll != COLL_BINARY;
    it.klen = compile_pattern(bytes, len, escape, runes, w.data(), t.data());
    it.runes = runes && !like_bytes_ok(w, t, it.klen);
    it.pw = reinterpret_cast<const int32_t*>(put(w.data(), (size_t)it.klen * 4));
    it.pt = reinterpret_cast<const uint8_t*>(put(t.data(), (size_t)it.klen));
    return TG_OK;
  }
  // upload the blob; item pointers become device pointers into dev
  int upload(int device, cudaStream_t st) {
    TG_TRY(dev.ensure(device, blob.size() + 16));
    if (!blob.empty()) TG_CUDA(cudaMemcpyAsync(dev.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
    const uint8_t* b = dev.as<uint8_t>();
    for (int q = 0; q < sf.n; q++) {
      StrItem& it = sf.items[q];
      if (it.kind == TG_STR_CMP) { if (it.rhs < 0) it.k = b + reinterpret_cast<size_t>(it.k); }
      else { it.pw = reinterpret_cast<const int32_t*>(b + reinterpret_cast<size_t>(it.pw)); it.pt = b + reinterpret_cast<size_t>(it.pt); }
    }
    return TG_OK;
  }
};

int launch_string(const VecLaunch& v, StrPrep& prep, const DecFilter& d, const DevFilter& f) {
  TG_TRY(prep.upload(v.device, v.st));
  bool two = false;
  for (int q = 0; q < prep.sf.n; q++) two |= prep.sf.items[q].rhs >= 0;
  const size_t smem = (size_t)kWarpsPerBlock * kStageStride * (two ? 2 : 1);
  const int grid = grid_size(v.nsm, v.n, 32 * kWarpsPerBlock, 8);
  const auto kernel = v.selected ? k_vec_string<false> : k_vec_string<true>;
  kernel<<<grid, 32 * kWarpsPerBlock, smem, v.st>>>(v.sc, v.cols, prep.sf, d, f, v.sel, v.nsel, v.nphys, v.selected, &v.flags->count,
                                                    v.result, v.rnulls, &v.flags->fault[0], &v.flags->fault[1]);
  return TG_OK;
}

// tg_vec_compare_string / tg_vec_like: the column a (and b) with one STRING item
static int run_string_column(int device, int on_device, int kind, int op, int32_t collation, const tg_column* a,
                             const tg_column* b, const uint8_t* bytes, int64_t len, int32_t escape, int64_t* result,
                             uint8_t* result_nulls, void* stream) {
  if (!a || !result || !result_nulls) return fail(TG_ERR_INVALID, "a / result / result_nulls is NULL");
  if (b && b->length != a->length) return fail(TG_ERR_INVALID, "argument columns have different lengths");
  TG_TRY(check_str_column(*a, on_device));
  if (b) TG_TRY(check_str_column(*b, on_device));
  StrPrep prep;
  TG_TRY(prep.add(kind, op, 0, b ? 1 : -1, collation, bytes, len, escape));
  return run_column(device, on_device, a, b, result, result_nulls, stream, {FAULT_BAD_OFFSETS},
                    [&](const VecLaunch& v) { return launch_string(v, prep, DecFilter{}, DevFilter{}); });
}

}  // namespace tg

using namespace tg;

extern "C" {

int tg_vec_compare_string(int device, int on_device, int op, int32_t collation, const tg_column* a, const tg_column* b,
                          const uint8_t* b_const, int64_t b_len, int64_t* result, uint8_t* result_nulls, void* stream) {
  return run_string_column(device, on_device, TG_STR_CMP, op, collation, a, b, b_const, b_len, 0, result, result_nulls, stream);
}

int tg_vec_like(int device, int on_device, int32_t collation, const tg_column* a, const uint8_t* pattern,
                int64_t pattern_len, int32_t escape, int64_t* result, uint8_t* result_nulls, void* stream) {
  return run_string_column(device, on_device, TG_STR_LIKE, TG_CMP_EQ, collation, a, nullptr, pattern, pattern_len, escape,
                           result, result_nulls, stream);
}

int tg_vec_filter_ex2(int device, int on_device, const tg_chunk* chk, const int32_t* col_types,
                      const tg_filter_item* items, int32_t n_items, const uint8_t* dec_consts,
                      const tg_str_arg* str_args, uint8_t* selected, int64_t* n_selected, void* stream) {
  if (!chk || !selected || !col_types) return fail(TG_ERR_INVALID, "chunk / col_types / selected is NULL");
  if (n_items < 0 || n_items > TG_MAX_FILTER) return fail(TG_ERR_UNSUPPORTED, "at most 8 CNF filter items are offloaded");
  if (n_items > 0 && !items) return fail(TG_ERR_INVALID, "items is NULL");
  if (chk->ncols <= 0 || chk->ncols > TG_MAX_COLS || !chk->cols) return fail(TG_ERR_UNSUPPORTED, "chunk must have 1..16 columns");
  const int64_t nphys = chk->cols[0].length;
  StrPrep prep;
  std::vector<char> is_str(n_items, 0), needed(chk->ncols, 0);
  for (int i = 0; i < n_items; i++) {
    const tg_filter_item& it = items[i];
    if (it.is_real != TG_FILTER_STRING) continue;
    is_str[i] = 1;
    if (!str_args) return fail(TG_ERR_INVALID, "a STRING item but str_args is NULL");
    const tg_str_arg& sa = str_args[i];
    const bool like = sa.kind == TG_STR_LIKE || sa.kind == TG_STR_NOT_LIKE;
    const int rhs = like ? -1 : it.rhs_col;
    if (it.lhs_col < 0 || it.lhs_col >= chk->ncols || rhs >= chk->ncols) return fail(TG_ERR_INVALID, "filter column out of range");
    for (int c : {it.lhs_col, rhs}) {
      if (c < 0) continue;
      if (!is_string_type(col_types[c])) return fail(TG_ERR_UNSUPPORTED, "a STRING filter item over a column that is not a string type");
      const tg_column& col = chk->cols[c];
      TG_TRY(check_str_column(col, on_device));
      if (col.length != nphys) return fail(TG_ERR_INVALID, "chunk columns have different lengths");
      needed[c] = 1;
    }
    TG_TRY(prep.add(sa.kind, it.op, it.lhs_col, rhs, sa.collation, sa.bytes, sa.len, sa.escape));
  }
  DecFilter d{};
  DevFilter f{};
  TG_TRY(check_filter_items(on_device, chk, col_types, items, n_items, dec_consts, is_str, d, f, needed));
  // a string-typed column in an INT / REAL / DECIMAL item: refused by its type, whatever its elem_len says
  for (int i = 0; i < n_items; i++) {
    if (is_str[i]) continue;
    if (is_string_type(col_types[items[i].lhs_col]) || (items[i].rhs_col >= 0 && is_string_type(col_types[items[i].rhs_col])))
      return fail(TG_ERR_UNSUPPORTED, "a string column in an INT / REAL / DECIMAL filter item");
  }
  return run_filter(device, on_device, chk, needed, prep.sf.n ? &prep : nullptr, d, f, selected, n_selected, stream);
}

}  // extern "C"
