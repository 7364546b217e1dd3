// topn.cu — tg_topn: TopNExec (pkg/executor/sortexec/topn.go:74 TopNExec, :230 executeTopN, :325 processChildChk) on the
// device.  The reference keeps a heap of offset+count rows and compares rows with the ORDER BY items' CompareFuncs
// (chunk.GetCompareFunc: NULL sorts before every value, DESC negates).  Here:
//   1. k_topn_rank   : one 64-bit RANK per row from the FIRST item (order-preserving map of the value, inverted for DESC,
//                      NULL = smallest / largest) — smaller rank = earlier in the output.  A DECIMAL first item takes
//                      k_topn_rank_dec, whose rank (decimal.cuh dec_order_key) is monotone but may tie unequal values
//                      that share their first 16 significant digits: ties only widen step 3's candidates;
//   2. radix select  : 8 histogram passes (k_topn_hist, 8 bits each, most significant first) find the rank of the
//                      (offset+count)-th row without sorting anything;
//   3. k_topn_collect: rows whose rank is <= that threshold (>= offset+count rows; more only on ties of the first item)
//                      are compacted, their columns gathered (k_topn_gather; DECIMAL cells by launch_gather_cells) and
//                      copied to the host;
//   4. host          : the few candidates are sorted with the full multi-item comparator and rows [offset, offset+count)
//                      are returned.  Ties are broken arbitrarily, as by the reference's heap.
// HBM-bound: the rank pass reads 8 B/row + bitmap (40 B/row for DECIMAL), each histogram pass 8 B/row.
#include <algorithm>
#include <vector>
#include "common.cuh"
#include "chunk_io.cuh"
#include "decimal.cuh"

namespace tg {

// ORDER BY kinds: how a column's 8-byte value is compared
enum { KIND_SIGNED = 0, KIND_UNSIGNED = 1, KIND_REAL = 2, KIND_TIME = 3, KIND_DECIMAL = 4 };
// Packed CoreTime (types/time.go:235-251): year..microsecond from bit 63 down to bit 4, then 4 fspTt bits (fsp and
// type).  compareTime (types/core_time.go:256) compares the calendar fields and the microseconds only, which is the
// unsigned order of the word with the fspTt bits cleared.
constexpr unsigned long long kTimeValueMask = ~0xFull;

__device__ __forceinline__ unsigned long long rank_of(unsigned long long raw, bool is_null, int kind, bool desc) {
  unsigned long long o;
  if (is_null) o = 0ull;                         // NULL sorts before every value (chunk.GetCompareFunc -> cmpNull)
  else if (kind == KIND_REAL) { o = (raw >> 63) ? ~raw : (raw | 0x8000000000000000ull); }
  else if (kind == KIND_UNSIGNED) o = raw;
  else if (kind == KIND_TIME) o = raw & kTimeValueMask;
  else o = raw ^ 0x8000000000000000ull;
  // NULL and the smallest value may share rank 0 (and, inverted, the largest): that only widens the candidate set; the
  // final order comes from the exact comparator on the host
  return desc ? ~o : o;
}

__global__ void __launch_bounds__(256)
k_topn_rank(const unsigned long long* __restrict__ data, const uint8_t* __restrict__ nulls, int64_t n, int kind, int desc,
            unsigned long long* __restrict__ rank) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    bool isn = nulls && !bit_not_null(nulls, i);
    unsigned long long raw = __ldcs(data + i);
    if (kind == KIND_REAL && !isn) {
      const double d = __longlong_as_double((long long)raw);
      if (d != d) raw = 0xFFF8000000000000ull;   // every NaN below everything and equal (Go cmp.Compare)
      else if (d == 0.0) raw = 0ull;             // -0 == +0: both zeros share one rank, so a tie on zero is collected whole
    }
    rank[i] = rank_of(raw, isn, kind, desc != 0);
  }
}

// A DECIMAL first item: the rank of k_topn_rank from each 40-byte cell's dec_order_key, each cell read once as five
// 8-byte loads per thread (a warp's 5 loads cover its 1280 contiguous bytes; L1 serves the sectors each load leaves to
// the next).  Staging each warp's 1280 bytes through shared memory with coalesced loads was no faster: 1.66 ms against
// 1.63 ms (2.94 TB/s at 48 B per row) over 100 M DECIMAL(15,2) cells on an H100 80GB HBM3 at 700 W
// (tools/scratch/topn_rank_lab.cu), so the plain loads stay.  *bad = 1 when a non-NULL cell is malformed (decimal.cuh
// dec_cell_ok).  With rank == nullptr the pass only checks the cells: the check of a later DECIMAL item.
__global__ void __launch_bounds__(256)
k_topn_rank_dec(const unsigned long long* __restrict__ cells, const uint8_t* __restrict__ nulls, int64_t n, int desc,
                unsigned long long* __restrict__ rank, unsigned int* __restrict__ bad) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const bool isn = nulls && !bit_not_null(nulls, i);
    uint32_t c[10];
#pragma unroll
    for (int j = 0; j < 5; j++) {
      const unsigned long long v = cells[i * 5 + j];
      c[2 * j] = (uint32_t)v; c[2 * j + 1] = (uint32_t)(v >> 32);
    }
    unsigned long long o = 0ull;   // NULL sorts before every value
    if (!isn) {
      if (!dec_cell_ok(c)) *bad = 1u;
      o = dec_order_key(c);
    }
    if (rank) rank[i] = desc ? ~o : o;
  }
}

// histogram of byte `shift/8` over the rows whose higher bytes equal `prefix`
__global__ void __launch_bounds__(256)
k_topn_hist(const unsigned long long* __restrict__ rank, int64_t n, unsigned long long prefix, int shift, unsigned long long* __restrict__ hist) {
  __shared__ unsigned int s_h[256];
  s_h[threadIdx.x] = 0;
  __syncthreads();
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const unsigned long long himask = shift >= 56 ? 0ull : (~0ull << (shift + 8));
  for (; i < n; i += stride) {
    unsigned long long r = rank[i];
    if ((r & himask) == (prefix & himask)) atomicAdd(&s_h[(r >> shift) & 0xffu], 1u);
  }
  __syncthreads();
  if (s_h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], (unsigned long long)s_h[threadIdx.x]);
}

__global__ void __launch_bounds__(256)
k_topn_collect(const unsigned long long* __restrict__ rank, int64_t n, unsigned long long threshold, unsigned long long cap,
               unsigned long long* __restrict__ cursor, long long* __restrict__ idx) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    if (rank[i] <= threshold) {
      unsigned long long o = atomicAdd(cursor, 1ull);
      if (o < cap) idx[o] = i;
    }
  }
}

__global__ void __launch_bounds__(256)
k_topn_gather(const unsigned long long* __restrict__ data, const uint8_t* __restrict__ nulls, const long long* __restrict__ idx, int64_t m,
              unsigned long long* __restrict__ out, uint8_t* __restrict__ out_valid) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < m; i += stride) {
    const long long r = idx[i];
    if (out) out[i] = data[r];   // NULL: the valid flags of a DECIMAL column, whose cells launch_gather_cells moves
    out_valid[i] = (nulls && !bit_not_null(nulls, r)) ? 0 : 1;
  }
}

static int kind_of(int tp, uint32_t flag) {
  if (tp == TG_TYPE_DOUBLE) return KIND_REAL;
  if (is_int_family(tp)) return (flag & TG_FLAG_UNSIGNED) ? KIND_UNSIGNED : KIND_SIGNED;
  if (tp == TG_TYPE_DATE || tp == TG_TYPE_DATETIME || tp == TG_TYPE_TIMESTAMP) return KIND_TIME;
  return -1;
}

}  // namespace tg

using namespace tg;

extern "C" {

int tg_topn(int device, int on_device, const tg_chunk* chk, const int32_t* col_types, const uint32_t* col_flags,
            const tg_sort_item* items, int32_t n_items, int64_t offset, int64_t count, tg_mut_chunk* out, int64_t* nrows, void* stream) {
  if (!chk || !col_types || !items || !out || !nrows) return fail(TG_ERR_INVALID, "chk / col_types / items / out / nrows is NULL");
  *nrows = 0;
  if (n_items < 1 || n_items > 8) return fail(TG_ERR_UNSUPPORTED, "1..8 ORDER BY items are offloaded");
  if (offset < 0 || count < 0) return fail(TG_ERR_INVALID, "negative offset / count");
  if (chk->sel) return fail(TG_ERR_UNSUPPORTED, "TopN input must not carry a sel vector");
  const int nc = chk->ncols;
  if (nc < 1 || nc > TG_MAX_COLS || out->ncols != nc) return fail(TG_ERR_INVALID, "1..16 columns; the output chunk has the child's schema");
  std::vector<int> kinds(nc), elem(nc);
  for (int c = 0; c < nc; c++) {
    elem[c] = chk->cols[c].elem_len;
    if (elem[c] == TG_DEC_CELL_BYTES) {
      if (col_types[c] != TG_TYPE_NEWDECIMAL) return fail(TG_ERR_UNSUPPORTED, "a 40-byte TopN column must be DECIMAL (MyDecimal cells)");
      if (on_device && (reinterpret_cast<uintptr_t>(chk->cols[c].data) & 7)) return fail(TG_ERR_INVALID, "DECIMAL device columns must be 8-byte aligned");
      kinds[c] = KIND_DECIMAL;
    } else if (elem[c] != 8) {
      return fail(TG_ERR_UNSUPPORTED, "TopN is offloaded for 8-byte columns and 40-byte DECIMAL cells only");
    } else {
      kinds[c] = kind_of(col_types[c], col_flags ? col_flags[c] : 0);
    }
  }
  bool dec_items = false;
  for (int q = 0; q < n_items; q++) {
    if (items[q].col < 0 || items[q].col >= nc) return fail(TG_ERR_INVALID, "ORDER BY column out of range");
    if (kinds[items[q].col] < 0) return fail(TG_ERR_UNSUPPORTED, "ORDER BY column type is not offloaded (int family / double / time / DECIMAL cells)");
    dec_items |= kinds[items[q].col] == KIND_DECIMAL;
  }
  TG_TRY(require_device("TopN"));
  DeviceGuard g(device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = chk->cols[0].length;
  // a malformed DECIMAL cell fails the call whatever offset and count select, so those cells are read even then
  if (n == 0 || ((count == 0 || offset >= n) && !dec_items)) return TG_OK;
  // device-resident columns
  std::vector<DevBuf> hdata(nc), hnulls(nc);
  std::vector<const unsigned long long*> dcol(nc);
  std::vector<const uint8_t*> dnul(nc, nullptr);
  for (int c = 0; c < nc; c++) {
    if (chk->cols[c].length != n) return fail(TG_ERR_INVALID, "chunk columns have different lengths");
    if (on_device) { dcol[c] = reinterpret_cast<const unsigned long long*>(chk->cols[c].data); dnul[c] = chk->cols[c].null_bitmap; continue; }
    TG_TRY(upload_column(device, st, chk->cols[c].data, chk->cols[c].null_bitmap, n, elem[c], hdata[c], hnulls[c], nullptr));
    dcol[c] = hdata[c].as<unsigned long long>();
    if (chk->cols[c].null_bitmap) dnul[c] = hnulls[c].as<uint8_t>();
  }
  const int nsm = device_sm_count(device);
  const int grid = grid_size(nsm, n, 256, 8);
  DevBuf rank, scratch, idx;
  TG_TRY(rank.ensure(device, (size_t)n * 8 + 16));
  TG_TRY(scratch.ensure(device, 258 * 8));
  unsigned int* bad = reinterpret_cast<unsigned int*>(scratch.as<unsigned long long>() + 257);
  const int c0 = items[0].col;
  if (dec_items) {
    // every non-NULL cell of every DECIMAL item is checked: the first item's in its rank pass, each other one in a pass
    // of its own, so the result does not depend on which rows become candidates
    TG_CUDA(cudaMemsetAsync(bad, 0, 4, st));
    for (int q = 1; q < n_items; q++) {
      const int c = items[q].col;
      bool seen = c == c0;
      for (int p = 1; p < q; p++) seen |= items[p].col == c;
      if (kinds[c] == KIND_DECIMAL && !seen) k_topn_rank_dec<<<grid, 256, 0, st>>>(dcol[c], dnul[c], n, 0, nullptr, bad);
    }
  }
  if (kinds[c0] == KIND_DECIMAL) k_topn_rank_dec<<<grid, 256, 0, st>>>(dcol[c0], dnul[c0], n, items[0].desc, rank.as<unsigned long long>(), bad);
  else k_topn_rank<<<grid, 256, 0, st>>>(dcol[c0], dnul[c0], n, kinds[c0], items[0].desc, rank.as<unsigned long long>());
  if (dec_items) {
    unsigned int hbad = 0;
    TG_CUDA(cudaMemcpyAsync(&hbad, bad, 4, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    if (hbad) return fail(TG_ERR_INVALID, "malformed DECIMAL cell in an ORDER BY column (digitsInt / digitsFrac < 0, more than 9 words, or a word >= 10^9)");
    if (count == 0 || offset >= n) return TG_OK;
  }
  const int64_t want = count >= n - offset ? n : offset + count;   // min(n, offset + count) without overflowing int64
  // radix select: the rank of the `want`-th smallest row
  unsigned long long prefix = 0, remaining = (unsigned long long)want;
  unsigned long long hist[256];
  for (int shift = 56; shift >= 0; shift -= 8) {
    TG_CUDA(cudaMemsetAsync(scratch.p, 0, 256 * 8, st));
    k_topn_hist<<<grid, 256, 0, st>>>(rank.as<unsigned long long>(), n, prefix, shift, scratch.as<unsigned long long>());
    TG_CUDA(cudaMemcpyAsync(hist, scratch.p, 256 * 8, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    int b = 0;
    for (; b < 256; b++) { if (hist[b] >= remaining) break; remaining -= hist[b]; }
    if (b == 256) return fail(TG_ERR_CUDA, "internal: TopN radix select ran out of rows");
    prefix |= (unsigned long long)b << shift;
  }
  // candidates: every row at or below the threshold rank
  unsigned long long* cursor = scratch.as<unsigned long long>() + 256;
  unsigned long long cap = (unsigned long long)want + 65536;
  unsigned long long m = 0;
  for (int attempt = 0; attempt < 2; attempt++) {
    TG_TRY(idx.ensure(device, (size_t)cap * 8 + 16));
    TG_CUDA(cudaMemsetAsync(cursor, 0, 8, st));
    k_topn_collect<<<grid, 256, 0, st>>>(rank.as<unsigned long long>(), n, prefix, cap, cursor, idx.as<long long>());
    TG_CUDA(cudaMemcpyAsync(&m, cursor, 8, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    if (m <= cap) break;
    cap = m;   // many rows tie with the threshold on the first item: take them all, the host comparator decides
  }
  // gather the candidates' columns and bring them to the host (w[c] 8-byte words per row: 5 for a DECIMAL cell)
  std::vector<int> w(nc);
  for (int c = 0; c < nc; c++) w[c] = elem[c] / 8;
  std::vector<std::vector<unsigned long long>> hv(nc);
  std::vector<std::vector<uint8_t>> hn(nc, std::vector<uint8_t>((size_t)m));
  DevBuf gcol, gval;
  TG_TRY(gcol.ensure(device, (size_t)m * TG_DEC_CELL_BYTES + 16));
  TG_TRY(gval.ensure(device, (size_t)m + 16));
  const int ggrid = grid_size(nsm, (int64_t)m, 256, 8);
  for (int c = 0; c < nc; c++) {
    hv[c].resize((size_t)m * w[c]);
    const bool cells = kinds[c] == KIND_DECIMAL;
    k_topn_gather<<<ggrid, 256, 0, st>>>(dcol[c], dnul[c], idx.as<long long>(), (int64_t)m, cells ? nullptr : gcol.as<unsigned long long>(), gval.as<uint8_t>());
    if (cells) launch_gather_cells(idx.as<int64_t>(), nullptr, dcol[c], gcol.p, (int64_t)m, nullptr, nsm, st);
    TG_CUDA(cudaMemcpyAsync(hv[c].data(), gcol.p, (size_t)m * elem[c], cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaMemcpyAsync(hn[c].data(), gval.p, (size_t)m, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
  }
  TG_CUDA(cudaGetLastError());
  // exact multi-item comparator (sortexec compareRow: per item CompareFunc, NULL first, DESC negated)
  std::vector<int64_t> order((size_t)m);
  for (size_t i = 0; i < order.size(); i++) order[i] = (int64_t)i;
  auto cmp_item = [&](int q, int64_t a, int64_t b) -> int {
    const int c = items[q].col;
    const bool an = !hn[c][(size_t)a], bn = !hn[c][(size_t)b];
    int r;
    if (an || bn) r = an == bn ? 0 : (an ? -1 : 1);
    else if (kinds[c] == KIND_DECIMAL) {   // cmpMyDecimal -> MyDecimal.Compare
      r = dec_cell_cmp(reinterpret_cast<const uint32_t*>(hv[c].data() + (size_t)a * w[c]),
                       reinterpret_cast<const uint32_t*>(hv[c].data() + (size_t)b * w[c]));
    } else {
      const unsigned long long x = hv[c][(size_t)a], y = hv[c][(size_t)b];
      if (kinds[c] == KIND_REAL) {
        double dx, dy; std::memcpy(&dx, &x, 8); std::memcpy(&dy, &y, 8);
        const bool xn = dx != dx, yn = dy != dy;
        r = xn ? (yn ? 0 : -1) : (yn ? 1 : (dx < dy ? -1 : (dx > dy ? 1 : 0)));
      } else if (kinds[c] == KIND_UNSIGNED) r = x < y ? -1 : (x > y ? 1 : 0);
      else if (kinds[c] == KIND_TIME) {
        const unsigned long long tx = x & kTimeValueMask, ty = y & kTimeValueMask;
        r = tx < ty ? -1 : (tx > ty ? 1 : 0);
      } else r = (long long)x < (long long)y ? -1 : ((long long)x > (long long)y ? 1 : 0);
    }
    return items[q].desc ? -r : r;
  };
  std::sort(order.begin(), order.end(), [&](int64_t a, int64_t b) {
    for (int q = 0; q < n_items; q++) { int r = cmp_item(q, a, b); if (r) return r < 0; }
    return false;
  });
  const int64_t take = std::min<int64_t>(want - offset, std::min<int64_t>(out->capacity_rows, (int64_t)m - offset));
  if (want - offset > out->capacity_rows) return fail(TG_ERR_CAPACITY, "TopN output chunk is smaller than `count`");
  // every output column is checked before the first write: a rejected call leaves `out` as it was
  for (int c = 0; c < nc; c++)
    if (kinds[c] == KIND_DECIMAL && out->cols[c].elem_len != TG_DEC_CELL_BYTES) return fail(TG_ERR_INVALID, "a DECIMAL output column must have elem_len 40");
  for (int c = 0; c < nc; c++) {
    if (out->cols[c].elem_len != elem[c]) return fail(TG_ERR_INVALID, "output column elem_len mismatch");
    if (out->cols[c].null_bitmap) continue;
    for (int64_t i = 0; i < take; i++)
      if (!hn[c][(size_t)order[(size_t)(offset + i)]]) return fail(TG_ERR_INVALID, "output column can be NULL but the caller passed no null bitmap");
  }
  for (int c = 0; c < nc; c++) {
    uint8_t* dst = reinterpret_cast<uint8_t*>(out->cols[c].data);
    uint8_t* nb = out->cols[c].null_bitmap;
    if (nb) std::memset(nb, 0, (size_t)((take + 7) / 8));
    for (int64_t i = 0; i < take; i++) {
      const int64_t r = order[(size_t)(offset + i)];
      const bool valid = hn[c][(size_t)r] != 0;
      // a NULL row's value is zero bytes (a DECIMAL cell: 40 of them, as the join writes)
      if (valid) std::memcpy(dst + i * elem[c], hv[c].data() + (size_t)r * w[c], (size_t)elem[c]);
      else std::memset(dst + i * elem[c], 0, (size_t)elem[c]);
      if (nb && valid) nb[i >> 3] |= (uint8_t)(1u << (i & 7));
    }
  }
  *nrows = take;
  return TG_OK;
}

}  // extern "C"
