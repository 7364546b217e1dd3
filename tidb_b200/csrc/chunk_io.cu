// chunk_io.cu — the host side of the chunk contract shared by the operators (chunk_io.cuh).
#include "chunk_io.cuh"
#include "decimal.cuh"

namespace tg {

int64_t logical_rows(const tg_chunk* chk) { return chk->sel ? chk->nsel : (chk->ncols > 0 ? chk->cols[0].length : 0); }

int validate_chunk(int ncols, const std::vector<char>& needed, const std::vector<int>& elem, const tg_chunk* chk) {
  if (!chk || chk->ncols != ncols) return fail(TG_ERR_INVALID, "chunk column count does not match the child schema");
  int64_t phys = chk->ncols ? chk->cols[0].length : 0;
  for (int c = 0; c < ncols; c++) {
    if (!needed[c]) continue;
    if (chk->cols[c].elem_len != elem[c]) return fail(TG_ERR_INVALID, "chunk column elem_len does not match the schema type");
    if (chk->cols[c].length != phys) return fail(TG_ERR_INVALID, "chunk columns have different lengths");
    if (phys && !chk->cols[c].data) return fail(TG_ERR_INVALID, "chunk column data is NULL");
  }
  return TG_OK;
}

int stage_append(HostStage& st, const std::vector<char>& needed, const std::vector<int>& elem, const tg_chunk* chk) {
  int64_t n = logical_rows(chk);
  if (n == 0) return TG_OK;
  for (size_t c = 0; c < needed.size(); c++) {
    if (!needed[c]) continue;
    const tg_column& col = chk->cols[c];
    int el = elem[c];
    PinBuf& d = *st.data[c];
    if (el < 0) {   // var-length: the rows' bytes appended, their offsets rebased onto the staged bytes
      PinBuf& ob = *st.offs[c];
      TG_TRY(ob.reserve((size_t)(st.rows + n + 1) * 8));
      int64_t* o = reinterpret_cast<int64_t*>(ob.p);
      if (st.rows == 0) o[0] = 0;
      const int64_t at = o[st.rows];
      int64_t add = 0;
      if (!chk->sel) add = col.offsets[n] - col.offsets[0];
      else for (int64_t i = 0; i < n; i++) add += col.offsets[chk->sel[i] + 1] - col.offsets[chk->sel[i]];
      TG_TRY(d.reserve((size_t)(at + add)));
      if (!chk->sel) {
        if (add) std::memcpy(d.p + at, col.data + col.offsets[0], (size_t)add);
        for (int64_t i = 0; i < n; i++) o[st.rows + i + 1] = at + col.offsets[i + 1] - col.offsets[0];
      } else {
        int64_t w = at;
        for (int64_t i = 0; i < n; i++) {
          const int64_t s0 = col.offsets[chk->sel[i]], len = col.offsets[chk->sel[i] + 1] - s0;
          if (len) std::memcpy(d.p + w, col.data + s0, (size_t)len);
          w += len;
          o[st.rows + i + 1] = w;
        }
      }
      d.used = (size_t)(at + add);
      ob.used = (size_t)(st.rows + n + 1) * 8;
    } else {
      TG_TRY(d.reserve((size_t)(st.rows + n) * el));
      uint8_t* dst = d.p + (size_t)st.rows * el;
      if (!chk->sel) std::memcpy(dst, col.data, (size_t)n * el);
      else if (el == 8) { auto* o = reinterpret_cast<uint64_t*>(dst); auto* in = reinterpret_cast<const uint64_t*>(col.data); for (int64_t i = 0; i < n; i++) o[i] = in[chk->sel[i]]; }
      else if (el == 4) { auto* o = reinterpret_cast<uint32_t*>(dst); auto* in = reinterpret_cast<const uint32_t*>(col.data); for (int64_t i = 0; i < n; i++) o[i] = in[chk->sel[i]]; }
      else { auto* in = reinterpret_cast<const uint8_t*>(col.data); for (int64_t i = 0; i < n; i++) std::memcpy(dst + (size_t)i * el, in + (size_t)chk->sel[i] * el, el); }
      d.used = (size_t)(st.rows + n) * el;
    }
    // null bitmap: materialised lazily, the first time a chunk brings one
    PinBuf& nb = *st.nulls[c];
    bool bring = col.null_bitmap != nullptr;
    if (bring || st.has_nulls[c]) {
      size_t need = (size_t)((st.rows + n + 7) / 8) + 1;
      TG_TRY(nb.reserve(need));
      if (!st.has_nulls[c]) { std::memset(nb.p, 0xff, (size_t)((st.rows + 7) / 8) + 1); st.has_nulls[c] = 1; }
      if (bring && !chk->sel) append_bits(nb.p, st.rows, col.null_bitmap, n);
      else {
        for (int64_t i = 0; i < n; i++) {
          bool nn = bring ? bit_not_null(col.null_bitmap, chk->sel ? chk->sel[i] : i) : true;
          int64_t r = st.rows + i;
          if (nn) nb.p[r >> 3] |= (uint8_t)(1u << (r & 7)); else nb.p[r >> 3] &= (uint8_t)~(1u << (r & 7));
        }
      }
      nb.used = need;
    }
  }
  st.rows += n;
  return TG_OK;
}

int upload_column(int device, cudaStream_t s, const void* src, const uint8_t* bitmap, int64_t rows, int elem,
                  DevBuf& data, DevBuf& nulls, int64_t* h2d_bytes) {
  size_t bytes = (size_t)rows * elem;
  TG_TRY(data.ensure(device, bytes + 16));
  if (bytes) TG_CUDA(cudaMemcpyAsync(data.p, src, bytes, cudaMemcpyHostToDevice, s));
  if (bitmap) {
    size_t nb = (size_t)((rows + 7) / 8);
    TG_TRY(nulls.ensure(device, nb + 16));
    if (nb) TG_CUDA(cudaMemcpyAsync(nulls.p, bitmap, nb, cudaMemcpyHostToDevice, s));
    bytes += nb;
  }
  if (h2d_bytes) *h2d_bytes += (int64_t)bytes;
  return TG_OK;
}

int upload_varlen_column(int device, cudaStream_t s, const tg_column& c, DevBuf& offs, DevBuf& data, DevBuf& nulls,
                         int64_t* h2d_bytes) {
  const size_t ob = (size_t)(c.length + 1) * 8;
  const int64_t lo = c.offsets[0];
  const size_t bytes = (size_t)(c.offsets[c.length] - lo);
  TG_TRY(offs.ensure(device, ob + 16));
  TG_CUDA(cudaMemcpyAsync(offs.p, c.offsets, ob, cudaMemcpyHostToDevice, s));
  TG_TRY(data.ensure(device, bytes + 16));
  if (bytes) TG_CUDA(cudaMemcpyAsync(data.p, c.data + lo, bytes, cudaMemcpyHostToDevice, s));
  size_t nb = 0;
  if (c.null_bitmap) {
    nb = (size_t)((c.length + 7) / 8);
    TG_TRY(nulls.ensure(device, nb + 16));
    if (nb) TG_CUDA(cudaMemcpyAsync(nulls.p, c.null_bitmap, nb, cudaMemcpyHostToDevice, s));
  }
  if (h2d_bytes) *h2d_bytes += (int64_t)(ob + bytes + nb);
  return TG_OK;
}

int check_varlen_rows(const tg_column& c, const tg_chunk* chk) {
  if (c.elem_len != -1 || !c.offsets) return fail(TG_ERR_INVALID, "a string column is var-length: elem_len -1 and offsets");
  if (c.length < 0) return fail(TG_ERR_INVALID, "negative column length");
  const int64_t lo = c.offsets[0], hi = c.offsets[c.length];
  if (hi < lo) return fail(TG_ERR_INVALID, "string column offsets[length] < offsets[0]");
  if (hi > lo && !c.data) return fail(TG_ERR_INVALID, "string column without data");
  const int64_t n = logical_rows(chk);
  for (int64_t i = 0; i < n; i++) {
    const int64_t r = chk->sel ? chk->sel[i] : i;
    if (r < 0 || r >= c.length) return fail(TG_ERR_INVALID, "sel entry out of range");
    const int64_t o0 = c.offsets[r], o1 = c.offsets[r + 1];
    if (o0 > o1 || o0 < lo || o1 > hi) return fail(TG_ERR_INVALID, "string column row " + std::to_string(r) + " has bad offsets");
  }
  return TG_OK;
}

int device_view(const tg_chunk* chk, int ncols, const std::vector<char>& needed, const std::vector<int>& elem, DevCols& v) {
  TG_TRY(validate_chunk(ncols, needed, elem, chk));
  if (chk->sel) return fail(TG_ERR_UNSUPPORTED, "device-resident chunks must not carry a sel vector");
  std::memset(&v, 0, sizeof(v));
  for (int c = 0; c < ncols; c++) {
    v.elem_len[c] = elem[c];
    if (!needed[c]) continue;
    v.data[c] = chk->cols[c].data;
    v.nulls[c] = chk->cols[c].null_bitmap;
  }
  return TG_OK;
}

int check_out_columns(const std::vector<std::unique_ptr<DevBuf>>& bitmaps, const std::vector<int>& elem, const tg_mut_chunk* out) {
  for (int c = 0; c < out->ncols; c++) {
    if (out->cols[c].elem_len != elem[c]) return fail(TG_ERR_INVALID, "output column elem_len does not match its result column (a DECIMAL result needs elem_len 40, every other one 8)");
    if (bitmaps[c]->p && !out->cols[c].null_bitmap) return fail(TG_ERR_INVALID, "output column can be NULL but the caller passed no null bitmap");
  }
  return TG_OK;
}

int download_bitmaps(const std::vector<std::unique_ptr<DevBuf>>& bitmaps, tg_mut_chunk* out, int64_t lo, int64_t want,
                     cudaStream_t s, int64_t* copied) {
  const int shift = (int)(lo & 7);
  const size_t nb = (size_t)((want + 7) / 8);
  std::vector<std::vector<uint8_t>> shifted;    // bitmaps that start inside a byte: fetched whole, shifted below
  int64_t bytes = 0;
  for (int c = 0; c < out->ncols; c++) {
    uint8_t* dst = out->cols[c].null_bitmap;
    if (bitmaps[c]->p) {
      if (shift == 0) TG_CUDA(cudaMemcpyAsync(dst, bitmaps[c]->as<uint8_t>() + lo / 8, nb, cudaMemcpyDeviceToHost, s));
      else {
        shifted.emplace_back((size_t)((shift + want + 7) / 8) + 1, (uint8_t)0);
        TG_CUDA(cudaMemcpyAsync(shifted.back().data(), bitmaps[c]->as<uint8_t>() + lo / 8, shifted.back().size() - 1, cudaMemcpyDeviceToHost, s));
      }
      bytes += (int64_t)nb;
    } else if (dst) {
      std::memset(dst, 0xff, nb);
      if (want & 7) dst[nb - 1] = (uint8_t)((1u << (want & 7)) - 1);
    }
  }
  TG_CUDA(cudaStreamSynchronize(s));
  if (copied) *copied = bytes;
  size_t q = 0;
  for (int c = 0; c < out->ncols; c++) {
    if (!bitmaps[c]->p) continue;
    uint8_t* dst = out->cols[c].null_bitmap;
    if (shift) {
      const std::vector<uint8_t>& src = shifted[q++];
      for (size_t b = 0; b < nb; b++) dst[b] = (uint8_t)((src[b] >> shift) | (src[b + 1] << (8 - shift)));
    }
    // mask the tail bits (Column.nullBitmap keeps unused bits zero)
    if (want & 7) dst[want >> 3] &= (uint8_t)((1u << (want & 7)) - 1);
  }
  return TG_OK;
}

// valid bytes (1 = NOT NULL) → Column.nullBitmap bits
__global__ void k_pack_bitmap(const uint8_t* __restrict__ valid, int64_t n, uint8_t* __restrict__ bitmap) {
  int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t nbytes = (n + 7) / 8;
  for (; b < nbytes; b += stride) {
    uint8_t v = 0;
    for (int j = 0; j < 8; j++) { int64_t r = b * 8 + j; if (r < n && valid[r]) v |= (uint8_t)(1u << j); }
    bitmap[b] = v;
  }
}

void launch_pack_bitmap(const uint8_t* valid, int64_t n, uint8_t* bitmap, int nsm, cudaStream_t s) {
  k_pack_bitmap<<<grid_size(nsm, (n + 7) / 8, 256, 8), 256, 0, s>>>(valid, n, bitmap);
}

// five lanes per row, one 8-byte word each: coalesced stores
__global__ void __launch_bounds__(256)
k_gather_cells(const int64_t* __restrict__ ids, const uint8_t* __restrict__ bitmap, const unsigned long long* __restrict__ src,
               unsigned long long* __restrict__ dst, int64_t rows, const unsigned long long* dev_rows) {
  constexpr int W = TG_DEC_CELL_BYTES / 8;
  const int64_t n = (dev_rows ? (int64_t)*dev_rows : rows) * W;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / W;
    unsigned long long v = 0;
    if (!bitmap || bit_not_null(bitmap, r)) v = src[ids[r] * W + (i - r * W)];
    dst[i] = v;
  }
}

void launch_gather_cells(const int64_t* ids, const uint8_t* bitmap, const void* src, void* dst, int64_t rows,
                         const unsigned long long* dev_rows, int nsm, cudaStream_t s) {
  const int grid = dev_rows ? nsm * 8 : grid_size(nsm, rows * (TG_DEC_CELL_BYTES / 8), 256, 8);
  k_gather_cells<<<grid, 256, 0, s>>>(ids, bitmap, reinterpret_cast<const unsigned long long*>(src),
                                      reinterpret_cast<unsigned long long*>(dst), rows, dev_rows);
}

int require_device(const char* what, int* ndev) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return fail(TG_ERR_CUDA, std::string("no CUDA device: ") + what + " has no CPU fallback"); }
  if (ndev) *ndev = n;
  return TG_OK;
}

int DeviceHandle::open(int dev, void* caller_stream) {
  device = dev;
  if (caller_stream) { stream = (cudaStream_t)caller_stream; own_stream = false; }
  else { TG_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)); own_stream = true; }
  TG_CUDA(cudaEventCreate(&ev0));
  TG_CUDA(cudaEventCreate(&ev1));
  nsm = device_sm_count(dev);
  return TG_OK;
}

float DeviceHandle::elapsed_ms() const { float ms = 0; cudaEventElapsedTime(&ms, ev0, ev1); return ms; }

void DeviceHandle::release() {
  if (stream) cudaStreamSynchronize(stream);
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  if (own_stream && stream) cudaStreamDestroy(stream);
}

}  // namespace tg
