// vec.cuh — what the VecEval translation units share (vec.cu: 8-byte and DECIMAL columns; vec_string.cu: var-length
// string columns): column arguments, the result bitmap store, the DECIMAL CNF items and the host-side check of a
// tg_vec_filter_ex CNF.
#pragma once
#include <memory>
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

// a column argument made device-resident (copies host buffers when on_device == 0); `elem` is the width the kernel
// reads: 8, or 40 for DECIMAL cells
struct ArgDev {
  DevBuf data, nulls;
  VArg v{nullptr, nullptr};
  int load(int device, int on_device, const tg_column* c, cudaStream_t st, int elem = 8) {
    if (!c) return TG_OK;
    if (c->elem_len != elem) return fail(TG_ERR_UNSUPPORTED, elem == 8 ? "VecEval kernels take 8-byte columns" : "DECIMAL operands are 40-byte cells");
    if (on_device) { v.data = c->data; v.nulls = c->null_bitmap; return TG_OK; }
    TG_TRY(upload_column(device, st, c->data, c->null_bitmap, c->length, elem, data, nulls, nullptr));
    v.data = data.p;
    if (c->null_bitmap) v.nulls = nulls.as<uint8_t>();
    return TG_OK;
  }
};

extern const char* const kMalformedCell;

// The INT / REAL / DECIMAL items of a tg_vec_filter_ex CNF (the items whose `skip` entry is set are the caller's): checks
// them without a device, marks their operand columns in `needed` and sorts them into d (DECIMAL) and f (the rest).
int check_filter_items(int on_device, const tg_chunk* chk, const int32_t* col_types, const tg_filter_item* items,
                       int32_t n_items, const uint8_t* dec_consts, const std::vector<char>& skip, DecFilter& d,
                       DevFilter& f, std::vector<char>& needed);

}  // namespace tg
