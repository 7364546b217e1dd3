// chunk_io.cuh — how the operators read a pushed tg_chunk and fill a caller's tg_mut_chunk: validation, pinned host
// staging (sel gather, lazy NULL bitmaps), host → device column uploads, views of device-resident chunks, the NULL
// bitmaps of *_next and the gather of DECIMAL cells by row id; plus what every operator handle needs of its device: the
// launch grid, the device check, and a stream with two timing events.
#pragma once
#include <algorithm>
#include <memory>
#include "common.cuh"

namespace tg {

static const int64_t kStageBatchRows = 4ll << 20;   // host staging batch: small pushed chunks are flushed at this many rows

// rows a chunk holds for the operator: its sel vector's length when it has one, else its physical rows
int64_t logical_rows(const tg_chunk* chk);

// the chunk has the schema's ncols columns; each needed column has its schema width, the chunk's length and, when the
// chunk has rows, data
int validate_chunk(int ncols, const std::vector<char>& needed, const std::vector<int>& elem, const tg_chunk* chk);

// pinned host staging of pushed chunks, one buffer per column (only needed columns are filled).  A var-length column
// (elem -1) stages its rows' bytes in `data` and rows + 1 offsets into them, starting at 0, in `offs`.
struct HostStage {
  std::vector<std::unique_ptr<PinBuf>> data, nulls, offs;
  std::vector<char> has_nulls;
  int64_t rows = 0;
  void init(int ncols) {
    data.clear(); nulls.clear(); offs.clear();
    for (int i = 0; i < ncols; i++) { data.emplace_back(new PinBuf()); nulls.emplace_back(new PinBuf()); offs.emplace_back(new PinBuf()); }
    has_nulls.assign(ncols, 0);
    rows = 0;
  }
  void reset() {
    rows = 0; std::fill(has_nulls.begin(), has_nulls.end(), 0);
    for (auto& d : data) d->used = 0; for (auto& d : nulls) d->used = 0; for (auto& d : offs) d->used = 0;
  }
};

// append the logical rows of a validated host chunk to the staging (gathers through sel).  A var-length column's
// offsets must already be checked at those rows (check_varlen_rows): its bytes are copied here on the host.
int stage_append(HostStage& st, const std::vector<char>& needed, const std::vector<int>& elem, const tg_chunk* chk);

// `rows` host cells of `elem` bytes → data, and their NULL bitmap (when `bitmap` is set) → nulls, on stream s; each
// buffer gets 16 bytes past what is copied.  A zero-byte range enqueues no copy.  The bytes copied are added to
// *h2d_bytes when it is given.
int upload_column(int device, cudaStream_t s, const void* src, const uint8_t* bitmap, int64_t rows, int elem,
                  DevBuf& data, DevBuf& nulls, int64_t* h2d_bytes);

// A var-length host column (elem_len -1) → device, on stream s: its length + 1 offsets as they are → offs, the bytes
// [offsets[0], offsets[length]) → data (data's byte 0 is the byte at offsets[0], so offsets need not start at 0) and its
// NULL bitmap (when it has one) → nulls; each buffer gets 16 bytes past what is copied.  The caller has checked
// offsets[0] <= offsets[length]; offsets between them are not read here.  The bytes copied are added to *h2d_bytes when
// it is given.
int upload_varlen_column(int device, cudaStream_t s, const tg_column& c, DevBuf& offs, DevBuf& data, DevBuf& nulls,
                         int64_t* h2d_bytes);

// a var-length host column at the rows a chunk holds (its sel rows, else every physical row): offsets present,
// offsets[length] >= offsets[0], data present when there are bytes, and each row r with offsets[r] <= offsets[r+1],
// both within [offsets[0], offsets[length]]; TG_ERR_INVALID otherwise
int check_varlen_rows(const tg_column& c, const tg_chunk* chk);

// borrow a validated device-resident chunk (no sel vector) as a column view of its needed columns; no copy
int device_view(const tg_chunk* chk, int ncols, const std::vector<char>& needed, const std::vector<int>& elem, DevCols& v);

// TG_OK when every output column of `out` can take its result column: elem_len == elem[c], and a bitmap wherever
// bitmaps[c] has memory (the column can be NULL).  A *_next call runs it before it enqueues any copy, so a call it
// rejects writes nothing.
int check_out_columns(const std::vector<std::unique_ptr<DevBuf>>& bitmaps, const std::vector<int>& elem, const tg_mut_chunk* out);

// The NULL bitmaps of result rows [lo, lo + want) into out's columns, which check_out_columns accepted.  bitmaps[c]
// holds column c's bitmap from row 0, or no memory when the column cannot be NULL: out then gets all-valid bits if it
// passed a bitmap.  Copies on s, then synchronises s, re-aligns bitmaps that start inside a byte and zeroes the bits
// past `want`.  *copied (when given) = the bitmap bytes the rows cover.
int download_bitmaps(const std::vector<std::unique_ptr<DevBuf>>& bitmaps, tg_mut_chunk* out, int64_t lo, int64_t want,
                     cudaStream_t s, int64_t* copied);

// blocks for n work items: one per `block` items, at least 1, at most per_sm per SM
inline int grid_size(int nsm, int64_t n, int block, int per_sm) {
  int64_t need = (n + block - 1) / block, cap = (int64_t)nsm * per_sm;
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

// valid bytes (1 = NOT NULL) of n rows → Column.nullBitmap bits, on stream s (k_pack_bitmap)
void launch_pack_bitmap(const uint8_t* valid, int64_t n, uint8_t* bitmap, int nsm, cudaStream_t s);

// 40-byte DECIMAL cells by row id, on stream s (k_gather_cells): dst row r = src row ids[r], 40 zero bytes where `bitmap`
// (indexed by r, may be NULL) says NULL.  The row count is *dev_rows when given (kept on the device), else `rows`.
// src and dst are 8-byte aligned.
void launch_gather_cells(const int64_t* ids, const uint8_t* bitmap, const void* src, void* dst, int64_t rows,
                         const unsigned long long* dev_rows, int nsm, cudaStream_t s);

// TG_OK when the process sees a CUDA device (*ndev = how many); `what` names the operator in the error
int require_device(const char* what, int* ndev = nullptr);

// what an operator handle owns on its device: a stream (its own, or the caller's) and two timing events
struct DeviceHandle {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int nsm = 132;
  int open(int dev, void* caller_stream);   // with dev current
  float elapsed_ms() const;                 // ev0 → ev1, both complete
  void release();                           // synchronises the stream, destroys what open created
};

}  // namespace tg

// Entry-point prologue of a handle (shell `h` with mu / closed / impl): locks the shell and binds `var` to the live
// implementation, with its device current.  A closed handle returns TG_ERR_CANCELLED.
#define TG_LOCK(h, Impl, var)                                                  \
  if (!(h)) return tg::fail(TG_ERR_INVALID, "handle is NULL");                 \
  if ((h)->closed.load()) return tg::fail(TG_ERR_CANCELLED, "handle is closed"); \
  std::lock_guard<std::mutex> lock__((h)->mu);                                 \
  if ((h)->closed.load() || !(h)->impl) return tg::fail(TG_ERR_CANCELLED, "handle is closed"); \
  Impl* var = (h)->impl;                                                       \
  tg::DeviceGuard guard__(var->device);                                        \
  if (!guard__.ok) return tg::fail(TG_ERR_CUDA, "cudaSetDevice failed (no usable CUDA device)")
