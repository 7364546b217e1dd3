// vec.cu — VecEval* kernels: column-at-a-time scalar builtins over 8-byte chunk columns.
//
// Replaces (pkg/expression): builtinLTIntSig.vecEvalInt & the other five integer comparisons
// (builtin_compare_vec.go:524-561, vecCompareInt :619), the real comparisons
// (builtin_compare_vec_generated.go:54), builtinArithmetic{Plus,Minus,Multiply}{Int,Real}Sig
// (builtin_arithmetic_vec.go:856, :365, :646, :1011, :496, :300, :40) and
// expression.VectorizedFilter (chunk_executor.go:413).  All are streaming kernels bounded by HBM:
// 8 B (+8 B) read and 8 B written per row, null bitmaps merged bytewise (Column.MergeNulls column.go:906).
// The DECIMAL compare and filter (tg_vec_compare_decimal, tg_vec_filter_ex) read 40-byte MyDecimal cells and compare
// them as MyDecimal.Compare (builtin{LT,LE,GT,GE,EQ,NE}DecimalSig, builtin_compare_vec_generated.go:64, :960, :1184).
#include "vec.cuh"

namespace tg {

// Streaming layout: lane l of a warp owns rows base+l, base+32+l, ... (VEC_ITEMS per thread, all loads issued before
// use) so every load/store instruction is one fully coalesced 256-byte request; the 32 validity bits of a warp-row are
// one ballot, written as one aligned 32-bit word of the result bitmap.
#define VEC_ITEMS 4

template <bool REAL>
__global__ void __launch_bounds__(256)
k_vec_compare(int op, int ua, int ub, VArg a, VArg b, long long bc_i, double bc_f, int64_t n,
              long long* __restrict__ result, uint8_t* __restrict__ rnulls) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t tile = 32 * VEC_ITEMS;
  for (int64_t base = warp * tile; base < n; base += nwarps * tile) {
    unsigned long long x[VEC_ITEMS], y[VEC_ITEMS];
    bool in[VEC_ITEMS];
#pragma unroll
    for (int j = 0; j < VEC_ITEMS; j++) {
      int64_t i = base + j * 32 + lane;
      in[j] = i < n;
      x[j] = in[j] ? __ldcs(reinterpret_cast<const unsigned long long*>(a.data) + i) : 0ull;
      y[j] = (in[j] && b.data) ? __ldcs(reinterpret_cast<const unsigned long long*>(b.data) + i) : 0ull;
    }
#pragma unroll
    for (int j = 0; j < VEC_ITEMS; j++) {
      int64_t i = base + j * 32 + lane;
      bool valid = in[j] && arg_valid(a, i) && arg_valid(b, i);
      int c;
      if (REAL) c = cmp_real(__longlong_as_double((long long)x[j]), b.data ? __longlong_as_double((long long)y[j]) : bc_f);
      else c = cmp_int((long long)x[j], ua != 0, b.data ? (long long)y[j] : bc_i, ub != 0);
      if (in[j]) __stcs(result + i, apply_cmp(op, c) ? 1ll : 0ll);
      unsigned bal = __ballot_sync(0xffffffffu, valid);
      store_valid_word(rnulls, base + j * 32, n, bal, lane);
    }
  }
}

// builtinArithmeticMinusIntSig.overflowCheck (builtin_arithmetic.go:491), forceToSigned = false
__device__ __forceinline__ bool minus_overflow(bool lu, bool ru, long long a, long long b) {
  bool is_signed = !lu && !ru;
  long long res = (long long)((unsigned long long)a - (unsigned long long)b);
  unsigned long long ua = (unsigned long long)a, ub = (unsigned long long)b;
  bool resUnsigned = false;
  if (lu) {
    if (ru) { if (ua < ub) { if (res >= 0) return true; } else resUnsigned = true; }
    else {
      if (b >= 0) { if (ua > ub) resUnsigned = true; }
      else { if (~0ull - ua < (unsigned long long)(-(unsigned long long)b)) return true; resUnsigned = true; }
    }
  } else {
    if (ru) { if ((unsigned long long)a - 0x8000000000000000ull < ub) return true; }
    else { if (a > 0 && b < 0) resUnsigned = true; else if (a < 0 && b > 0 && res >= 0) return true; }
  }
  return (!is_signed && !resUnsigned && res < 0) || (is_signed && resUnsigned && (unsigned long long)res > 0x7fffffffffffffffull);
}

__global__ void __launch_bounds__(256)
k_vec_arith_int(int op, int lu, int ru, VArg a, VArg b, long long bc, int64_t n, long long* __restrict__ result,
                uint8_t* __restrict__ rnulls, int* overflow) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t tile = 32 * VEC_ITEMS;
  const long long MAXI = 0x7fffffffffffffffll, MINI = (long long)0x8000000000000000ull;
  for (int64_t base = warp * tile; base < n; base += nwarps * tile) {
    long long xs[VEC_ITEMS], ys[VEC_ITEMS];
    bool in[VEC_ITEMS];
#pragma unroll
    for (int j = 0; j < VEC_ITEMS; j++) {
      int64_t i = base + j * 32 + lane;
      in[j] = i < n;
      xs[j] = in[j] ? __ldcs(reinterpret_cast<const long long*>(a.data) + i) : 0ll;
      ys[j] = in[j] ? (b.data ? __ldcs(reinterpret_cast<const long long*>(b.data) + i) : bc) : 0ll;
    }
#pragma unroll
    for (int j = 0; j < VEC_ITEMS; j++) {
      int64_t i = base + j * 32 + lane;
      long long lh = xs[j], rh = ys[j];
      bool ovf;
      long long r;
      if (op == TG_ARITH_PLUS) {
        if (lu && ru) ovf = (unsigned long long)lh > ~0ull - (unsigned long long)rh;
        else if (lu && !ru) ovf = (rh < 0 && (unsigned long long)(-(unsigned long long)rh) > (unsigned long long)lh) || (rh > 0 && (unsigned long long)lh > ~0ull - (unsigned long long)rh);
        else if (!lu && ru) ovf = (lh < 0 && (unsigned long long)(-(unsigned long long)lh) > (unsigned long long)rh) || (lh > 0 && (unsigned long long)rh > ~0ull - (unsigned long long)lh);
        else ovf = (lh > 0 && rh > MAXI - lh) || (lh < 0 && rh < MINI - lh);
        r = (long long)((unsigned long long)lh + (unsigned long long)rh);
      } else if (op == TG_ARITH_MINUS) {
        ovf = minus_overflow(lu != 0, ru != 0, lh, rh);
        r = (long long)((unsigned long long)lh - (unsigned long long)rh);
      } else if (lu || ru) {
        unsigned long long x = (unsigned long long)lh, y = (unsigned long long)rh, res = x * y;
        ovf = x != 0 && res / x != y;
        r = (long long)res;
      } else {
        long long tmp = (long long)((unsigned long long)lh * (unsigned long long)rh);
        bool special = tmp == MINI && lh == -1;
        ovf = special || (lh != 0 && tmp / lh != rh);
        r = tmp;
      }
      bool valid = in[j] && arg_valid(a, i) && arg_valid(b, i);
      if (ovf) { if (valid) atomicExch(overflow, 1); r = 0; }
      if (in[j]) __stcs(result + i, r);
      unsigned bal = __ballot_sync(0xffffffffu, valid);
      store_valid_word(rnulls, base + j * 32, n, bal, lane);
    }
  }
}

__global__ void __launch_bounds__(256)
k_vec_arith_real(int op, VArg a, VArg b, double bc, int64_t n, double* __restrict__ result, uint8_t* __restrict__ rnulls,
                 int* overflow) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t tile = 32 * VEC_ITEMS;
  for (int64_t base = warp * tile; base < n; base += nwarps * tile) {
    double xs[VEC_ITEMS], ys[VEC_ITEMS];
    bool in[VEC_ITEMS];
#pragma unroll
    for (int j = 0; j < VEC_ITEMS; j++) {
      int64_t i = base + j * 32 + lane;
      in[j] = i < n;
      xs[j] = in[j] ? __ldcs(reinterpret_cast<const double*>(a.data) + i) : 0.0;
      ys[j] = in[j] ? (b.data ? __ldcs(reinterpret_cast<const double*>(b.data) + i) : bc) : 0.0;
    }
#pragma unroll
    for (int j = 0; j < VEC_ITEMS; j++) {
      int64_t i = base + j * 32 + lane;
      double r;
      bool ovf;
      if (op == TG_ARITH_PLUS) { r = xs[j] + ys[j]; ovf = !isfinite(r); }          // mathutil.IsFinite
      else if (op == TG_ARITH_MINUS) { r = xs[j] - ys[j]; ovf = !isfinite(r); }
      else { r = xs[j] * ys[j]; ovf = isinf(r); }                                    // math.IsInf only (:51-58)
      bool valid = in[j] && arg_valid(a, i) && arg_valid(b, i);
      if (ovf && valid) atomicExch(overflow, 1);
      if (in[j]) __stcs(result + i, r);
      unsigned bal = __ballot_sync(0xffffffffu, valid);
      store_valid_word(rnulls, base + j * 32, n, bal, lane);
    }
  }
}

// selected[physical row] = every CNF item is non-NULL true and the row is in sel (if any)
__global__ void __launch_bounds__(256)
k_vec_filter(DevCols cols, DevFilter f, const long long* __restrict__ sel, int64_t nsel, int64_t nphys,
             uint8_t* __restrict__ selected, unsigned long long* count) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long local = 0;
  int64_t n = sel ? nsel : nphys;
  for (; i < n; i += stride) {
    int64_t p = sel ? sel[i] : i;
    bool s = eval_filter(f, cols, p);
    selected[p] = s ? 1 : 0;
    local += s;
  }
  for (int o = 16; o; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0 && local) atomicAdd(count, local);
}

// ---- DECIMAL compares and filters: 40-byte MyDecimal cells (dec_load, DecFilter: vec.cuh) ----------------------------
// a constant cell in its comparison form (dec_normalize), passed by value
struct DecConst { uint32_t c[10]; };

// tg_vec_compare_decimal: k_vec_compare's warp-row layout over cells.  A NULL row's value is 0 and its cells are not
// compared; a malformed non-NULL cell of either operand sets *bad (decimal.cuh dec_cell_ok) whatever the other side holds.
__global__ void __launch_bounds__(256)
k_vec_compare_dec(int op, VArg a, VArg b, const __grid_constant__ DecConst k, int64_t n, long long* __restrict__ result,
                  uint8_t* __restrict__ rnulls, unsigned int* __restrict__ bad) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t tile = 32 * VEC_ITEMS;
  bool malformed = false;
  for (int64_t base = warp * tile; base < n; base += nwarps * tile) {
    uint32_t x[VEC_ITEMS][10], y[VEC_ITEMS][10];
#pragma unroll
    for (int j = 0; j < VEC_ITEMS; j++) {
      const int64_t i = base + j * 32 + lane;
      if (i < n) {
        dec_load(a.data, i, x[j]);
        if (b.data) dec_load(b.data, i, y[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < VEC_ITEMS; j++) {
      const int64_t i = base + j * 32 + lane;
      const bool in = i < n;
      const bool va = in && arg_valid(a, i), vb = in && arg_valid(b, i);
      malformed |= va && !dec_cell_ok(x[j]);
      bool r = false;
      if (b.data) {
        malformed |= vb && !dec_cell_ok(y[j]);
        if (va && vb) r = apply_cmp(op, dec_cmp_words(x[j][0], DecWordsReg{x[j]}, y[j][0], DecWordsReg{y[j]}));
      } else if (va) {
        r = apply_cmp(op, dec_cmp_words(x[j][0], DecWordsReg{x[j]}, k.c[0], DecWordsPtr{k.c}));
      }
      if (in) __stcs(result + i, r ? 1ll : 0ll);
      const unsigned bal = __ballot_sync(0xffffffffu, va && vb);
      store_valid_word(rnulls, base + j * 32, n, bal, lane);
    }
  }
  if (malformed) *bad = 1u;
}

// tg_vec_filter_ex with DECIMAL items: k_vec_filter's row loop; the DECIMAL items are evaluated first and all of them
// (eval_dec_items), so every non-NULL cell of their operands is checked at every row evaluated (*bad), then the INT /
// REAL items by eval_filter, unchanged.
__global__ void __launch_bounds__(256)
k_vec_filter_dec(DevCols cols, DevFilter f, const __grid_constant__ DecFilter d, const long long* __restrict__ sel,
                 int64_t nsel, int64_t nphys, uint8_t* __restrict__ selected, unsigned long long* count,
                 unsigned int* __restrict__ bad) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long local = 0;
  bool malformed = false;
  const int64_t n = sel ? nsel : nphys;
  for (; i < n; i += stride) {
    const int64_t p = sel ? sel[i] : i;
    bool s = eval_dec_items(d, cols, p, malformed);
    s = s && eval_filter(f, cols, p);
    selected[p] = s ? 1 : 0;
    local += s;
  }
  for (int o = 16; o; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0 && local) atomicAdd(count, local);
  if (malformed) *bad = 1u;
}

static const char* const kMalformedCell =
    "malformed DECIMAL cell (digitsInt / digitsFrac < 0, more than 9 words, or a word >= 10^9)";

// the checks of a DECIMAL operand column that need no device
static int check_dec_column(const tg_column& c, int on_device) {
  if (c.elem_len != TG_DEC_CELL_BYTES) return fail(TG_ERR_INVALID, "a DECIMAL operand column must have elem_len 40 (MyDecimal cells)");
  if (c.length < 0 || (c.length > 0 && !c.data)) return fail(TG_ERR_INVALID, "DECIMAL operand column without data");
  if (on_device && (reinterpret_cast<uintptr_t>(c.data) & 7)) return fail(TG_ERR_INVALID, "DECIMAL device columns must be 8-byte aligned");
  return TG_OK;
}

// a constant cell (host memory) -> its comparison form; a missing or malformed cell is TG_ERR_INVALID
static int load_dec_const(const uint8_t* cell, uint32_t (&k)[10]) {
  if (!cell) return fail(TG_ERR_INVALID, "DECIMAL comparison with a constant, but the constant cell is NULL");
  uint32_t c[10];
  std::memcpy(c, cell, TG_DEC_CELL_BYTES);
  if (!dec_cell_ok(c)) return fail(TG_ERR_INVALID, std::string(kMalformedCell) + " as the constant");
  dec_normalize(c, k);
  return TG_OK;
}

int check_filter_items(int on_device, const tg_chunk* chk, const int32_t* col_types, const tg_filter_item* items,
                       int32_t n_items, const uint8_t* dec_consts, const std::vector<char>& skip, DecFilter& d,
                       DevFilter& f, std::vector<char>& needed) {
  const int64_t nphys = chk->cols[0].length;
  for (int i = 0; i < n_items; i++) {
    if (skip[i]) continue;
    const tg_filter_item& it = items[i];
    if (it.lhs_col < 0 || it.lhs_col >= chk->ncols || it.rhs_col >= chk->ncols) return fail(TG_ERR_INVALID, "filter column out of range");
    if (it.op < TG_CMP_LT || it.op > TG_CMP_NE) return fail(TG_ERR_INVALID, "unknown comparison");
    if (it.is_real < TG_FILTER_INT || it.is_real > TG_FILTER_DECIMAL) return fail(TG_ERR_INVALID, "unknown filter item kind (is_real)");
    const bool dec = it.is_real == TG_FILTER_DECIMAL;
    for (int side = 0; side < 2; side++) {
      const int c = side ? it.rhs_col : it.lhs_col;
      if (c < 0) continue;
      const tg_column& col = chk->cols[c];
      const bool dec_col = col_types[c] == TG_TYPE_NEWDECIMAL;
      if (dec && !dec_col) return fail(TG_ERR_UNSUPPORTED, "a DECIMAL filter item compares DECIMAL columns only (the planner casts the other operand)");
      if (!dec && dec_col) return fail(TG_ERR_UNSUPPORTED, "a DECIMAL column in an INT / REAL filter item");
      if (dec) TG_TRY(check_dec_column(col, on_device));
      else if (col.elem_len != 8) return fail(TG_ERR_UNSUPPORTED, "VecEval kernels take 8-byte columns");
      if (col.length != nphys) return fail(TG_ERR_INVALID, "chunk columns have different lengths");
      needed[c] = 1;
    }
    if (dec) {
      DecItem& di = d.items[d.n++];
      di.op = it.op; di.lhs_col = it.lhs_col; di.rhs_col = it.rhs_col;
      if (it.rhs_col < 0) TG_TRY(load_dec_const(dec_consts ? dec_consts + (size_t)TG_DEC_CELL_BYTES * i : nullptr, di.k));
    } else {
      f.items[f.n++] = it;
    }
  }
  return TG_OK;
}

static const char* const kBadOffsets =
    "malformed string offsets: offsets[r] > offsets[r+1], or an offset outside [offsets[0], offsets[length]], at a row the call evaluates";

static int fault_status(VecFault f) {
  if (f == FAULT_OVERFLOW) return fail(TG_ERR_OVERFLOW, "ErrOverflow: value is out of range in arithmetic VecEval kernel");
  return fail(TG_ERR_INVALID, f == FAULT_BAD_CELL ? kMalformedCell : kBadOffsets);
}

// one VecFlags block per device, allocated on first use and never freed; its mutex holds the block from the zeroing
// through the read-back of one call
struct FlagSlot { std::mutex mu; VecFlags* p = nullptr; };
static FlagSlot& flag_slot(int device, int ndev) {
  static std::unique_ptr<FlagSlot[]> slots(new FlagSlot[ndev]);
  return slots[device];
}

int run_vec(int device, int on_device, const tg_chunk* chk, const std::vector<char>& needed, uint8_t* selected,
            int64_t* n_selected, void* result, uint8_t* rnulls, void* stream, std::initializer_list<VecFault> faults,
            const VecKernel& launch) {
  int ndev = 0;
  TG_TRY(require_device("VecEval", &ndev));
  DeviceGuard g(device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed");
  const bool filter = selected != nullptr;
  const int64_t nphys = chk->cols[0].length;
  const size_t nb = (size_t)((nphys + 7) / 8);
  VecLaunch v{};
  v.device = device; v.nsm = device_sm_count(device); v.ncols = chk->ncols; v.st = (cudaStream_t)stream;
  v.sel = reinterpret_cast<const long long*>(chk->sel); v.nsel = chk->nsel; v.nphys = nphys;
  v.n = chk->sel ? chk->nsel : nphys;
  v.selected = selected; v.result = static_cast<long long*>(result); v.rnulls = rnulls;
  // the needed columns: borrowed when device-resident, else uploaded (a var-length one from its offsets[0])
  DevBuf offs[TG_MAX_COLS], data[TG_MAX_COLS], nulls[TG_MAX_COLS];
  for (int c = 0; c < chk->ncols; c++) {
    const tg_column& col = chk->cols[c];
    v.cols.elem_len[c] = col.elem_len;
    if (!needed[c]) continue;
    const bool varlen = col.elem_len < 0;
    if (on_device) {
      if (varlen) { v.sc.offs[c] = col.offsets; v.sc.data[c] = col.data; }
      else v.cols.data[c] = col.data;
      v.cols.nulls[c] = col.null_bitmap;
      continue;
    }
    if (varlen) {
      TG_TRY(upload_varlen_column(device, v.st, col, offs[c], data[c], nulls[c], nullptr));
      v.sc.offs[c] = offs[c].as<int64_t>(); v.sc.data[c] = data[c].as<uint8_t>(); v.sc.base[c] = col.offsets[0];
    } else {
      TG_TRY(upload_column(device, v.st, col.data, col.null_bitmap, col.length, col.elem_len, data[c], nulls[c], nullptr));
      v.cols.data[c] = data[c].p;
    }
    if (col.null_bitmap) v.cols.nulls[c] = nulls[c].as<uint8_t>();
  }
  // a host chunk: its sel vector goes up, and the outputs are computed into device scratch
  DevBuf dsel, dout, dnul;
  if (!on_device) {
    if (chk->sel) {
      TG_TRY(dsel.ensure(device, (size_t)chk->nsel * 8 + 16));
      TG_CUDA(cudaMemcpyAsync(dsel.p, chk->sel, (size_t)chk->nsel * 8, cudaMemcpyHostToDevice, v.st));
      v.sel = dsel.as<long long>();
    }
    if (filter) {
      TG_TRY(dout.ensure(device, (size_t)nphys + 16));
      v.selected = dout.as<uint8_t>();
    } else {
      TG_TRY(dout.ensure(device, (size_t)nphys * 8 + 16)); TG_TRY(dnul.ensure(device, nb + 16));
      v.result = dout.as<long long>(); v.rnulls = dnul.as<uint8_t>();
    }
  }
  VecFlags flags{};
  std::unique_lock<std::mutex> flag_lock;
  if (filter || faults.size()) {
    FlagSlot& slot = flag_slot(device, ndev);
    flag_lock = std::unique_lock<std::mutex>(slot.mu);
    if (!slot.p) TG_CUDA(cudaMalloc(reinterpret_cast<void**>(&slot.p), sizeof(VecFlags)));
    v.flags = slot.p;
    TG_CUDA(cudaMemsetAsync(v.flags, 0, sizeof(VecFlags), v.st));
  }
  if (filter) TG_CUDA(cudaMemsetAsync(v.selected, 0, (size_t)nphys, v.st));
  if (v.n > 0) TG_TRY(launch(v));
  if (v.flags) TG_CUDA(cudaMemcpyAsync(&flags, v.flags, sizeof(VecFlags), cudaMemcpyDeviceToHost, v.st));
  TG_CUDA(cudaStreamSynchronize(v.st));
  if (flag_lock) flag_lock.unlock();
  TG_CUDA(cudaGetLastError());
  for (size_t w = 0; w < faults.size(); w++)
    if (flags.fault[w]) return fault_status(faults.begin()[w]);
  if (!on_device && nphys > 0) {
    if (filter) {
      TG_CUDA(cudaMemcpyAsync(selected, v.selected, (size_t)nphys, cudaMemcpyDeviceToHost, v.st));
    } else {
      TG_CUDA(cudaMemcpyAsync(result, v.result, (size_t)nphys * 8, cudaMemcpyDeviceToHost, v.st));
      TG_CUDA(cudaMemcpyAsync(rnulls, v.rnulls, nb, cudaMemcpyDeviceToHost, v.st));
    }
    TG_CUDA(cudaStreamSynchronize(v.st));
  }
  if (n_selected) *n_selected = (int64_t)flags.count;
  return TG_OK;
}

int run_column(int device, int on_device, const tg_column* a, const tg_column* b, void* result, uint8_t* rnulls,
               void* stream, std::initializer_list<VecFault> faults, const VecKernel& launch) {
  const tg_column cols[2] = {*a, b ? *b : *a};
  const tg_chunk chk{b ? 2 : 1, 0, cols, nullptr, 0};
  return run_vec(device, on_device, &chk, std::vector<char>(chk.ncols, 1), nullptr, nullptr, result, rnulls, stream,
                 faults, launch);
}

int run_filter(int device, int on_device, const tg_chunk* chk, const std::vector<char>& needed, StrPrep* prep,
               const DecFilter& d, const DevFilter& f, uint8_t* selected, int64_t* n_selected, void* stream) {
  // fault word 0: bad string offsets (STRING items only); word 1: malformed DECIMAL cells
  return run_vec(device, on_device, chk, needed, selected, n_selected, nullptr, nullptr, stream,
                 {FAULT_BAD_OFFSETS, FAULT_BAD_CELL}, [&](const VecLaunch& v) -> int {
    if (prep) return launch_string(v, *prep, d, f);
    const int grid = grid_size(v.nsm, v.n, 256, 8);
    if (d.n)
      k_vec_filter_dec<<<grid, 256, 0, v.st>>>(v.cols, f, d, v.sel, v.nsel, v.nphys, v.selected, &v.flags->count, &v.flags->fault[1]);
    else
      k_vec_filter<<<grid, 256, 0, v.st>>>(v.cols, f, v.sel, v.nsel, v.nphys, v.selected, &v.flags->count);
    return TG_OK;
  });
}

// the checks of the four compare / arith calls
static int check_binary(const tg_column* a, const tg_column* b, const void* result, const uint8_t* rnulls) {
  if (!a || !result || !rnulls) return fail(TG_ERR_INVALID, "a / result / result_nulls is NULL");
  if (b && b->length != a->length) return fail(TG_ERR_INVALID, "argument columns have different lengths");
  if (a->elem_len != 8 || (b && b->elem_len != 8)) return fail(TG_ERR_UNSUPPORTED, "VecEval kernels take 8-byte columns");
  return TG_OK;
}

// the grid of the warp-row kernels: VEC_ITEMS rows per thread
static int warp_row_grid(const VecLaunch& v) { return grid_size(v.nsm, (v.n + VEC_ITEMS - 1) / VEC_ITEMS, 256, 8); }

}  // namespace tg

using namespace tg;

extern "C" {

int tg_vec_compare_int(int device, int on_device, int op, int a_unsigned, int b_unsigned, const tg_column* a,
                       const tg_column* b, int64_t b_const, int64_t* result, uint8_t* result_nulls, void* stream) {
  TG_TRY(check_binary(a, b, result, result_nulls));
  return run_column(device, on_device, a, b, result, result_nulls, stream, {}, [&](const VecLaunch& v) {
    k_vec_compare<false><<<warp_row_grid(v), 256, 0, v.st>>>(op, a_unsigned, b_unsigned, v.arg(0), v.arg(1), (long long)b_const,
                                                             0.0, v.n, v.result, v.rnulls);
    return TG_OK;
  });
}

int tg_vec_compare_real(int device, int on_device, int op, const tg_column* a, const tg_column* b, double b_const,
                        int64_t* result, uint8_t* result_nulls, void* stream) {
  TG_TRY(check_binary(a, b, result, result_nulls));
  return run_column(device, on_device, a, b, result, result_nulls, stream, {}, [&](const VecLaunch& v) {
    k_vec_compare<true><<<warp_row_grid(v), 256, 0, v.st>>>(op, 0, 0, v.arg(0), v.arg(1), 0, b_const, v.n, v.result, v.rnulls);
    return TG_OK;
  });
}

int tg_vec_arith_int(int device, int on_device, int op, int a_unsigned, int b_unsigned, const tg_column* a,
                     const tg_column* b, int64_t b_const, int64_t* result, uint8_t* result_nulls, void* stream) {
  TG_TRY(check_binary(a, b, result, result_nulls));
  return run_column(device, on_device, a, b, result, result_nulls, stream, {FAULT_OVERFLOW}, [&](const VecLaunch& v) {
    k_vec_arith_int<<<warp_row_grid(v), 256, 0, v.st>>>(op, a_unsigned, b_unsigned, v.arg(0), v.arg(1), (long long)b_const, v.n,
                                                        v.result, v.rnulls, reinterpret_cast<int*>(&v.flags->fault[0]));
    return TG_OK;
  });
}

int tg_vec_arith_real(int device, int on_device, int op, const tg_column* a, const tg_column* b, double b_const,
                      double* result, uint8_t* result_nulls, void* stream) {
  TG_TRY(check_binary(a, b, result, result_nulls));
  return run_column(device, on_device, a, b, result, result_nulls, stream, {FAULT_OVERFLOW}, [&](const VecLaunch& v) {
    k_vec_arith_real<<<warp_row_grid(v), 256, 0, v.st>>>(op, v.arg(0), v.arg(1), b_const, v.n, reinterpret_cast<double*>(v.result),
                                                         v.rnulls, reinterpret_cast<int*>(&v.flags->fault[0]));
    return TG_OK;
  });
}

int tg_vec_filter(int device, int on_device, const tg_chunk* chk, const tg_filter_item* items, int32_t n_items,
                  uint8_t* selected, int64_t* n_selected, void* stream) {
  if (!chk || !selected) return fail(TG_ERR_INVALID, "chunk / selected is NULL");
  if (n_items < 0 || n_items > TG_MAX_FILTER) return fail(TG_ERR_UNSUPPORTED, "at most 8 CNF filter items are offloaded");
  if (chk->ncols <= 0 || chk->ncols > TG_MAX_COLS) return fail(TG_ERR_UNSUPPORTED, "chunk must have 1..16 columns");
  DevFilter f{}; f.n = n_items;
  std::vector<char> needed(chk->ncols, 0);
  for (int i = 0; i < n_items; i++) {
    const tg_filter_item& it = items[i];
    if (it.lhs_col < 0 || it.lhs_col >= chk->ncols || it.rhs_col >= chk->ncols) return fail(TG_ERR_INVALID, "filter column out of range");
    f.items[i] = it; needed[it.lhs_col] = 1; if (it.rhs_col >= 0) needed[it.rhs_col] = 1;
  }
  for (int c = 0; c < chk->ncols; c++)
    if (needed[c] && chk->cols[c].elem_len != 8) return fail(TG_ERR_UNSUPPORTED, "VecEval kernels take 8-byte columns");
  return run_filter(device, on_device, chk, needed, nullptr, DecFilter{}, f, selected, n_selected, stream);
}

int tg_decimal_normalize(const uint8_t* cell, uint8_t* out) {
  if (!out) return fail(TG_ERR_INVALID, "out is NULL");
  uint32_t k[10];
  TG_TRY(load_dec_const(cell, k));
  std::memcpy(out, k, TG_DEC_CELL_BYTES);
  return TG_OK;
}

int tg_vec_compare_decimal(int device, int on_device, int op, const tg_column* a, const tg_column* b,
                           const uint8_t* b_const_cell, int64_t* result, uint8_t* result_nulls, void* stream) {
  if (!a || !result || !result_nulls) return fail(TG_ERR_INVALID, "a / result / result_nulls is NULL");
  if (op < TG_CMP_LT || op > TG_CMP_NE) return fail(TG_ERR_INVALID, "unknown comparison");
  if (b && b->length != a->length) return fail(TG_ERR_INVALID, "argument columns have different lengths");
  TG_TRY(check_dec_column(*a, on_device));
  if (b) TG_TRY(check_dec_column(*b, on_device));
  DecConst k{};
  if (!b) TG_TRY(load_dec_const(b_const_cell, k.c));
  return run_column(device, on_device, a, b, result, result_nulls, stream, {FAULT_BAD_CELL}, [&](const VecLaunch& v) {
    k_vec_compare_dec<<<warp_row_grid(v), 256, 0, v.st>>>(op, v.arg(0), v.arg(1), k, v.n, v.result, v.rnulls, &v.flags->fault[0]);
    return TG_OK;
  });
}

int tg_vec_filter_ex(int device, int on_device, const tg_chunk* chk, const int32_t* col_types,
                     const tg_filter_item* items, int32_t n_items, const uint8_t* dec_consts,
                     uint8_t* selected, int64_t* n_selected, void* stream) {
  if (!chk || !selected || !col_types) return fail(TG_ERR_INVALID, "chunk / col_types / selected is NULL");
  if (n_items < 0 || n_items > TG_MAX_FILTER) return fail(TG_ERR_UNSUPPORTED, "at most 8 CNF filter items are offloaded");
  if (n_items > 0 && !items) return fail(TG_ERR_INVALID, "items is NULL");
  if (chk->ncols <= 0 || chk->ncols > TG_MAX_COLS || !chk->cols) return fail(TG_ERR_UNSUPPORTED, "chunk must have 1..16 columns");
  DecFilter d{};
  DevFilter f{};
  std::vector<char> needed(chk->ncols, 0);
  TG_TRY(check_filter_items(on_device, chk, col_types, items, n_items, dec_consts, std::vector<char>(n_items, 0), d, f, needed));
  return run_filter(device, on_device, chk, needed, nullptr, d, f, selected, n_selected, stream);
}

}  // extern "C"
