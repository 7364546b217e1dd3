// vec.cuh — what the VecEval translation units share (vec.cu: 8-byte and DECIMAL columns; vec_string.cu: var-length
// string columns): column arguments, the result bitmap store, the DECIMAL CNF items, the host-side check of a
// tg_vec_filter_ex CNF and the host path every VecEval call runs through.
#pragma once
#include <functional>
#include "common.cuh"
#include "chunk_io.cuh"
#include "decimal.cuh"

namespace tg {

struct VArg { const void* data; const uint8_t* nulls; };

__device__ __forceinline__ bool arg_valid(const VArg& a, int64_t i) { return !a.nulls || bit_not_null(a.nulls, i); }

// write the 32 validity bits of rows [wbase, wbase+32) (wbase % 32 == 0); tail rows are masked off
__device__ __forceinline__ void store_valid_word(uint8_t* rnulls, int64_t wbase, int64_t n, unsigned bal, int lane) {
  if (lane == 0 && wbase < n) {
    int64_t rem = n - wbase;
    if (rem >= 32) *reinterpret_cast<uint32_t*>(rnulls + (wbase >> 3)) = bal;
    else {
      bal &= (1u << rem) - 1u;
      for (int b = 0; b < (int)((rem + 7) / 8); b++) rnulls[(wbase >> 3) + b] = (uint8_t)(bal >> (8 * b));
    }
  }
}

// ---- DECIMAL compares and filters: 40-byte MyDecimal cells (decimal.cuh) -------------------------------------------
// The cell of row i in registers: five 8-byte loads.  Lane l's cell starts 40 * l bytes into its warp's 1280 contiguous
// bytes, so the warp's five loads cover those bytes and L1 serves the sectors each load leaves to the next (TopN's
// k_topn_rank_dec reads its cells the same way; see DESIGN.md §6b for the measurement).
__device__ __forceinline__ void dec_load(const void* data, int64_t i, uint32_t (&c)[10]) {
  const unsigned long long* p = reinterpret_cast<const unsigned long long*>(data) + i * 5;
#pragma unroll
  for (int j = 0; j < 5; j++) {
    const unsigned long long v = p[j];
    c[2 * j] = (uint32_t)v; c[2 * j + 1] = (uint32_t)(v >> 32);
  }
}

// the DECIMAL items of a tg_vec_filter_ex CNF: `op` lhs_col (rhs_col, or the constant k when rhs_col < 0)
struct DecItem { int32_t op, lhs_col, rhs_col, pad; uint32_t k[10]; };
struct DecFilter { int32_t n, pad; DecItem items[TG_MAX_FILTER]; };

// every DECIMAL item of `d` at physical row p, all of them, so every non-NULL cell of their operands is checked
// (*malformed); true when each one is non-NULL true
__device__ __forceinline__ bool eval_dec_items(const DecFilter& d, const DevCols& cols, int64_t p, bool& malformed) {
  bool s = true;
  for (int q = 0; q < d.n; q++) {
    const DecItem& it = d.items[q];
    uint32_t x[10];
    dec_load(cols.data[it.lhs_col], p, x);
    const uint8_t* ln = cols.nulls[it.lhs_col];
    const bool vx = !ln || bit_not_null(ln, p);
    malformed |= vx && !dec_cell_ok(x);
    int c;
    bool vy = true;
    if (it.rhs_col >= 0) {
      uint32_t y[10];
      dec_load(cols.data[it.rhs_col], p, y);
      const uint8_t* rn = cols.nulls[it.rhs_col];
      vy = !rn || bit_not_null(rn, p);
      malformed |= vy && !dec_cell_ok(y);
      c = dec_cmp_words(x[0], DecWordsReg{x}, y[0], DecWordsReg{y});
    } else {
      c = dec_cmp_words(x[0], DecWordsReg{x}, it.k[0], DecWordsPtr{it.k});
    }
    s &= vx && vy && apply_cmp(it.op, c);
  }
  return s;
}

// The INT / REAL / DECIMAL items of a tg_vec_filter_ex CNF (the items whose `skip` entry is set are the caller's): checks
// them without a device, marks their operand columns in `needed` and sorts them into d (DECIMAL) and f (the rest).
int check_filter_items(int on_device, const tg_chunk* chk, const int32_t* col_types, const tg_filter_item* items,
                       int32_t n_items, const uint8_t* dec_consts, const std::vector<char>& skip, DecFilter& d,
                       DevFilter& f, std::vector<char>& needed);

// ---- the host path of a VecEval call (vec.cu run_vec) --------------------------------------------------------------
// the string columns of a call: data[c] points at the byte of offset base[c] (an uploaded column starts there)
struct StrCols {
  const int64_t* offs[TG_MAX_COLS];
  const uint8_t* data[TG_MAX_COLS];
  int64_t base[TG_MAX_COLS];
};

// what a kernel reports back, zeroed before the launch and read once after it: a filter's selected rows and up to two
// fault words, each meaning one VecFault of the call
struct VecFlags { unsigned long long count; unsigned int fault[2]; };
enum VecFault { FAULT_OVERFLOW, FAULT_BAD_CELL, FAULT_BAD_OFFSETS };

// what a launch gets: the call's columns and outputs on the device, and `n` rows to evaluate (the sel vector's when the
// chunk has one, else its physical rows; never 0)
struct VecLaunch {
  int device, nsm, ncols;
  cudaStream_t st;
  DevCols cols;                  // fixed-width columns, and the NULL bitmaps of all needed columns
  StrCols sc;                    // var-length columns
  const long long* sel;
  int64_t nsel, nphys, n;
  uint8_t* selected;             // a filter's output
  long long* result;             // a column call's outputs
  uint8_t* rnulls;
  VecFlags* flags;               // NULL for a call with neither a count nor a fault word
  // operand c of a column call, or no column when the call has fewer
  VArg arg(int c) const { return c < ncols ? VArg{cols.data[c], cols.nulls[c]} : VArg{nullptr, nullptr}; }
};
using VecKernel = std::function<int(const VecLaunch&)>;

// Runs one VecEval call once its arguments are checked: the device, its guard and the stream; the needed columns of chk
// borrowed when device-resident, else uploaded; the outputs (a filter's `selected`, or a column call's result / rnulls
// for chk's physical rows) in device scratch for host buffers; the flags; the launch; the read-back.  A set fault word
// fails the call with its VecFault's status, and host outputs and *n_selected are written only when none is set.
int run_vec(int device, int on_device, const tg_chunk* chk, const std::vector<char>& needed, uint8_t* selected,
            int64_t* n_selected, void* result, uint8_t* rnulls, void* stream, std::initializer_list<VecFault> faults,
            const VecKernel& launch);

// run_vec for a column call: operand a, and b when given (already checked to have a's length)
int run_column(int device, int on_device, const tg_column* a, const tg_column* b, void* result, uint8_t* rnulls,
               void* stream, std::initializer_list<VecFault> faults, const VecKernel& launch);

// the STRING items of a call (vec_string.cu), and k_vec_string over them: a filter's when v has `selected`, then its
// DECIMAL items d and INT / REAL items f; else one item's column result
struct StrPrep;
int launch_string(const VecLaunch& v, StrPrep& prep, const DecFilter& d, const DevFilter& f);

// tg_vec_filter, _ex and _ex2 once each has checked its CNF: k_vec_string when there are STRING items (prep is given),
// else k_vec_filter_dec when d has items, else k_vec_filter
int run_filter(int device, int on_device, const tg_chunk* chk, const std::vector<char>& needed, StrPrep* prep,
               const DecFilter& d, const DevFilter& f, uint8_t* selected, int64_t* n_selected, void* stream);

}  // namespace tg
