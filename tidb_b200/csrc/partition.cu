// partition.cu — key-hash repartition for the multi-GPU exchange.
//
// The reference's analogue is the MPP ExchangeSender with ExchangeType HashPartition
// (pkg/planner/core/operator/physicalop/physical_exchange_sender.go:115; executed by TiFlash) and, in
// process, partitionHashSplitter.split (pkg/executor/shuffle.go:450).  Here: count rows per destination
// (k_partition_count), then one scatter kernel that regroups each 2048-row tile by destination in shared
// memory and writes every destination's rows as one contiguous run — either into local per-partition
// regions (tg_partition_by_key, followed by an NCCL all-to-all) or straight into the peers' receive
// buffers over NVLink (tg_partition_exchange: the repartition step and its all-to-all in ONE kernel; the
// stores to peer memory are 1 KB runs, and the transfer overlaps the regrouping tile by tile).
#include "partition_kernels.cuh"
#include <mutex>

namespace tg {

static int check_parts(int32_t nparts, int32_t ncols) {
  if (nparts < 1 || nparts > TG_MAX_PARTS) return fail(TG_ERR_UNSUPPORTED, "1..16 partitions");
  if (ncols < 1 || ncols > TG_PART_MAX_COLS) return fail(TG_ERR_UNSUPPORTED, "1..8 columns per repartition call");
  return TG_OK;
}

// Per-device scratch of the counted calls (counts | cursors): allocated once, never freed — a DevBuf per call would run
// pool_free's device-wide synchronisation on every exchange step.  The counted calls synchronise their stream before
// returning, so holding the device's mutex for the duration of a call makes the shared scratch safe.
struct PartScratch { std::mutex mu; unsigned long long* p = nullptr; };
static PartScratch& part_scratch(int device) { static PartScratch s[64]; return s[device & 63]; }
static int part_scratch_ensure(PartScratch& ps) {
  if (!ps.p) TG_CUDA(cudaMalloc(&ps.p, (size_t)TG_MAX_PARTS * 8 * 4));
  return TG_OK;
}

}  // namespace tg

using namespace tg;

extern "C" {

int32_t tg_partition_of_key(int64_t key, int32_t nparts) { return (int32_t)part_of(hash64((uint64_t)key), (uint32_t)nparts); }

int tg_partition_count(int device, const int64_t* key_dev, int64_t rows, int32_t nparts, int64_t* part_counts_dev, void* stream) {
  TG_TRY(check_parts(nparts, 1));
  DeviceGuard g(device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed (no usable CUDA device)");
  cudaStream_t st = (cudaStream_t)stream;
  TG_CUDA(cudaMemsetAsync(part_counts_dev, 0, (size_t)nparts * 8, st));
  TG_TRY(launch_partition_count<false>(device, st, reinterpret_cast<const long long*>(key_dev), nullptr, rows, (uint32_t)nparts,
                                       reinterpret_cast<unsigned long long*>(part_counts_dev), nullptr));
  TG_CUDA(cudaGetLastError());
  return TG_OK;
}

int tg_partition_by_key(int device, const int64_t* key_dev, const uint8_t* key_nulls_dev, int64_t rows, int32_t nparts,
                        int32_t ncols, const void* const* src_cols_dev, void* const* dst_cols_dev,
                        int64_t* part_offsets_dev, void* stream) {
  TG_TRY(check_parts(nparts, ncols));
  DeviceGuard g(device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed (no usable CUDA device)");
  cudaStream_t st = (cudaStream_t)stream;
  PartScratch& ps = part_scratch(device);
  std::lock_guard<std::mutex> slk(ps.mu);
  TG_TRY(part_scratch_ensure(ps));
  unsigned long long* counts = ps.p;
  unsigned long long* cursors = counts + TG_MAX_PARTS;
  TG_CUDA(cudaMemsetAsync(counts, 0, (size_t)TG_MAX_PARTS * 16, st));
  const long long* key = reinterpret_cast<const long long*>(key_dev);
  TG_TRY(launch_partition_count<false>(device, st, key, key_nulls_dev, rows, (uint32_t)nparts, counts, nullptr));
  k_partition_offsets<<<1, 32, 0, st>>>(counts, (uint32_t)nparts, reinterpret_cast<long long*>(part_offsets_dev), cursors);
  PartDst d{};
  d.nparts = nparts; d.ncols = ncols;
  for (int c = 0; c < ncols; c++) { d.src[c] = src_cols_dev[c]; for (int p = 0; p < nparts; p++) d.dst[p][c] = dst_cols_dev[c]; }
  d.dst_base = reinterpret_cast<const long long*>(part_offsets_dev);
  TG_TRY(launch_partition_scatter<false>(device, st, key, key_nulls_dev, rows, d, cursors, nullptr));
  TG_CUDA(cudaGetLastError());
  TG_CUDA(cudaStreamSynchronize(st));   // the shared scratch is released with the lock
  return TG_OK;
}

int tg_partition_exchange(int device, const int64_t* key_dev, int64_t rows, int32_t nparts, int32_t ncols,
                          const void* const* src_cols_dev, void* const* recv_cols_peer, const int64_t* part_counts_dev,
                          const int64_t* recv_base_dev, void* stream) {
  (void)part_counts_dev;
  TG_TRY(check_parts(nparts, ncols));
  DeviceGuard g(device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed (no usable CUDA device)");
  cudaStream_t st = (cudaStream_t)stream;
  PartScratch& ps = part_scratch(device);
  std::lock_guard<std::mutex> slk(ps.mu);
  TG_TRY(part_scratch_ensure(ps));
  unsigned long long* cursors = ps.p;
  TG_CUDA(cudaMemsetAsync(cursors, 0, (size_t)TG_MAX_PARTS * 8, st));
  PartDst d{};
  d.nparts = nparts; d.ncols = ncols;
  for (int c = 0; c < ncols; c++) { d.src[c] = src_cols_dev[c]; for (int p = 0; p < nparts; p++) d.dst[p][c] = recv_cols_peer[p * ncols + c]; }
  d.dst_base = reinterpret_cast<const long long*>(recv_base_dev);
  TG_TRY(launch_partition_scatter<false>(device, st, reinterpret_cast<const long long*>(key_dev), nullptr, rows, d, cursors, nullptr));
  TG_CUDA(cudaGetLastError());
  TG_CUDA(cudaStreamSynchronize(st));
  return TG_OK;
}

static __global__ void k_zero_cf(unsigned long long* sent, int nparts) {
  if ((int)threadIdx.x < nparts) sent[threadIdx.x] = 0;
  // the overflow flag is sticky: zeroed once by its owner, so an overflow of ANY step is still visible when the host looks
}

static int exchange_cf_impl(int device, const int64_t* key_dev, int64_t rows, int32_t nparts, int32_t ncols,
                            const void* const* src_cols_dev, void* const* recv_cols_peer, int64_t region_base,
                            int64_t region_cap, int64_t* sent_rows_dev, uint64_t* overflow_dev, int ctas_per_sm, void* stream,
                            void* const* spill_cols_dev = nullptr, int64_t spill_cap = 0, uint64_t* spill_cursor_dev = nullptr) {
  TG_TRY(check_parts(nparts, ncols));
  if (spill_cursor_dev && (!spill_cols_dev || spill_cap <= 0)) return fail(TG_ERR_INVALID, "a spill cursor needs spill columns and a positive spill_cap");
  if (ncols > 4) return fail(TG_ERR_UNSUPPORTED, "count-free exchange moves at most 4 columns per call");
  if (!sent_rows_dev || !overflow_dev || region_cap <= 0) return fail(TG_ERR_INVALID, "sent_rows_dev / overflow_dev / region_cap are required");
  if (src_cols_dev[0] != (const void*)key_dev) return fail(TG_ERR_INVALID, "src_cols_dev[0] must be the key column");
  for (int c = 0; c < ncols; c++) if (!ptr_aligned16(src_cols_dev[c])) return fail(TG_ERR_UNSUPPORTED, "source columns must be 16-byte aligned");
  for (int i = 0; i < nparts * ncols; i++) if (!ptr_aligned16(recv_cols_peer[i])) return fail(TG_ERR_UNSUPPORTED, "receive columns must be 16-byte aligned");
  if (region_base & 1) return fail(TG_ERR_UNSUPPORTED, "region_base must be even (16-byte aligned regions)");
  DeviceGuard g(device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed (no usable CUDA device)");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* cursors = reinterpret_cast<unsigned long long*>(sent_rows_dev);
  k_zero_cf<<<1, 32, 0, st>>>(cursors, nparts);
  PartDst d{};
  d.nparts = nparts; d.ncols = ncols;
  for (int c = 0; c < ncols; c++) { d.src[c] = src_cols_dev[c]; for (int p = 0; p < nparts; p++) d.dst[p][c] = recv_cols_peer[p * ncols + c]; }
  d.dst_base = nullptr; d.base_const = region_base;   // every destination holds this sender's region at the same row offset
  d.capacity = region_cap; d.overflow = reinterpret_cast<unsigned long long*>(overflow_dev);
  if (spill_cursor_dev) {
    for (int c = 0; c < ncols; c++) { if (!spill_cols_dev[c]) return fail(TG_ERR_INVALID, "spill column is NULL"); d.spill[c] = spill_cols_dev[c]; }
    d.spill_cap = spill_cap; d.spill_cursor = reinterpret_cast<unsigned long long*>(spill_cursor_dev);
  }
  const int64_t TILE = 1024;
  const int64_t n_main = rows / TILE * TILE;
  if (n_main > 0) TG_TRY(launch_partition_scatter<false>(device, st, reinterpret_cast<const long long*>(key_dev), nullptr, n_main, d, cursors, nullptr, ctas_per_sm));
  if (n_main < rows) {
    // the last < 1024 rows: LSU kernel, one CTA, same cursors and capacity
    PartDst tail = d;
    for (int c = 0; c < ncols; c++) tail.src[c] = reinterpret_cast<const unsigned long long*>(src_cols_dev[c]) + n_main;
    k_partition_scatter<false><<<1, PT_BLOCK, 0, st>>>(reinterpret_cast<const long long*>(tail.src[0]), nullptr, rows - n_main, tail, cursors);
  }
  TG_CUDA(cudaGetLastError());
  return TG_OK;
}

int tg_partition_exchange_cf(int device, const int64_t* key_dev, int64_t rows, int32_t nparts, int32_t ncols,
                             const void* const* src_cols_dev, void* const* recv_cols_peer, int64_t region_base,
                             int64_t region_cap, int64_t* sent_rows_dev, uint64_t* overflow_dev, void* stream) {
  return exchange_cf_impl(device, key_dev, rows, nparts, ncols, src_cols_dev, recv_cols_peer, region_base, region_cap, sent_rows_dev, overflow_dev, 0, stream);
}

int tg_partition_exchange_cf_ex(int device, const int64_t* key_dev, int64_t rows, int32_t nparts, int32_t ncols,
                                const void* const* src_cols_dev, void* const* recv_cols_peer, int64_t region_base,
                                int64_t region_cap, int64_t* sent_rows_dev, uint64_t* overflow_dev, int32_t ctas_per_sm, void* stream) {
  return exchange_cf_impl(device, key_dev, rows, nparts, ncols, src_cols_dev, recv_cols_peer, region_base, region_cap, sent_rows_dev, overflow_dev, ctas_per_sm, stream);
}

int tg_partition_exchange_cf_spill(int device, const int64_t* key_dev, int64_t rows, int32_t nparts, int32_t ncols,
                                   const void* const* src_cols_dev, void* const* recv_cols_peer, int64_t region_base,
                                   int64_t region_cap, int64_t* sent_rows_dev, uint64_t* overflow_dev, void* const* spill_cols_dev,
                                   int64_t spill_cap, uint64_t* spill_cursor_dev, int32_t ctas_per_sm, void* stream) {
  if (!spill_cursor_dev) return fail(TG_ERR_INVALID, "spill_cursor_dev is required (use tg_partition_exchange_cf_ex without a spill area)");
  return exchange_cf_impl(device, key_dev, rows, nparts, ncols, src_cols_dev, recv_cols_peer, region_base, region_cap, sent_rows_dev, overflow_dev,
                          ctas_per_sm, stream, spill_cols_dev, spill_cap, spill_cursor_dev);
}

// ---- SM-driven region copy over NVLink (the transfer stage of the count-free exchange without copy engines) --------------
// Copies the FILLED part of up to 64 staged regions to their peers with 128-bit loads / stores: no shared memory and at most
// 32 registers per thread, 128 threads per CTA — exactly the 4096 registers an SM has left next to three resident CTAs of
// the persistent probe kernel (3 x 256 x 80), so the copy runs UNDER the probe of the previous step without touching the
// probe's L1 carve-out.  CTA b starts with region b % n, so the CTAs spread over the peers instead of convoying.
struct CopyJob {
  const ulonglong2* src[TG_COPY_MAX_REGIONS];
  ulonglong2* dst[TG_COPY_MAX_REGIONS];
  int32_t cnt_idx[TG_COPY_MAX_REGIONS];
  int32_t n, pad;
  long long cap_rows;
  const unsigned long long* counts;
};
static __global__ void __launch_bounds__(128, 16) k_peer_copy(CopyJob j) {   // 16 CTAs per SM = at most 32 registers per thread
  for (int q = 0; q < j.n; q++) {
    const int r = (q + (int)blockIdx.x) % j.n;
    unsigned long long rows = j.counts[j.cnt_idx[r]];
    if (rows > (unsigned long long)j.cap_rows) rows = (unsigned long long)j.cap_rows;
    const long long n16 = (long long)((rows + 1) >> 1);            // 16-byte units; regions hold an even number of rows
    const ulonglong2* __restrict__ src = j.src[r];
    ulonglong2* __restrict__ dst = j.dst[r];
    for (long long i = (long long)blockIdx.x * 512 + threadIdx.x; i < n16; i += (long long)gridDim.x * 512) {
      ulonglong2 v[4];
#pragma unroll
      for (int u = 0; u < 4; u++) if (i + u * 128 < n16) v[u] = __ldcs(src + i + u * 128);
#pragma unroll
      for (int u = 0; u < 4; u++) if (i + u * 128 < n16) __stcs(dst + i + u * 128, v[u]);
    }
  }
}

int tg_peer_copy_regions(int device, int32_t n_regions, const void* const* src_dev, void* const* dst_peer, const int32_t* count_index,
                         const int64_t* counts_dev, int64_t cap_rows, int32_t ctas, void* stream) {
  if (n_regions < 1 || n_regions > TG_COPY_MAX_REGIONS) return fail(TG_ERR_INVALID, "1..64 regions per call");
  if (!src_dev || !dst_peer || !count_index || !counts_dev || cap_rows <= 0 || (cap_rows & 1)) return fail(TG_ERR_INVALID, "pointers required; cap_rows must be even");
  DeviceGuard g(device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed (no usable CUDA device)");
  CopyJob j{};
  j.n = n_regions; j.cap_rows = cap_rows; j.counts = reinterpret_cast<const unsigned long long*>(counts_dev);
  for (int r = 0; r < n_regions; r++) {
    if (!ptr_aligned16(src_dev[r]) || !ptr_aligned16(dst_peer[r])) return fail(TG_ERR_UNSUPPORTED, "regions must be 16-byte aligned");
    j.src[r] = reinterpret_cast<const ulonglong2*>(src_dev[r]); j.dst[r] = reinterpret_cast<ulonglong2*>(dst_peer[r]); j.cnt_idx[r] = count_index[r];
  }
  int grid = ctas > 0 ? ctas : device_sm_count(device);
  k_peer_copy<<<grid, 128, 0, (cudaStream_t)stream>>>(j);
  TG_CUDA(cudaGetLastError());
  return TG_OK;
}

// ---- cross-GPU mailboxes: the exchange's only synchronisation, peer stores + spinning loads, no NCCL, no host ------
// One 8-byte word per (kind, buffer set, sender): epoch << 40 | value.  A single 64-bit store is atomic, so the word needs
// no second flag.  The signal kernel runs AFTER the kernel whose peer stores it publishes (stream order: kernel
// completion makes them visible system-wide); the wait kernel runs BEFORE the kernel that consumes them.
static __global__ void k_mail_signal(tg_mail_targets t, const unsigned long long* values, unsigned long long epoch) {
  const int p = threadIdx.x;
  if (p >= t.n) return;
  unsigned long long v = values ? values[p] : 0ull;
  if (v >= (1ull << 40)) v = (1ull << 40) - 1;
  __threadfence_system();
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(t.slot[p]), "l"((epoch << 40) | v) : "memory");
}

static __global__ void k_mail_wait(const unsigned long long* mail, int n, unsigned long long epoch, unsigned long long* values_out,
                                   unsigned long long* error_flag, unsigned long long timeout_ns) {
  const int p = threadIdx.x;
  if (p >= n) return;
  unsigned long long t0, now, v;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
  for (;;) {
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(mail + p) : "memory");
    if ((v >> 40) >= epoch) break;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(now));
    if (now - t0 > timeout_ns) { atomicExch(error_flag, 1ull + (unsigned long long)p); v = 0; break; }   // never hang the GPU: report and go on
    __nanosleep(200);
  }
  if (values_out) values_out[p] = v & ((1ull << 40) - 1);
}

int tg_mail_signal(int device, const tg_mail_targets* targets, const int64_t* values_dev, int64_t epoch, void* stream) {
  if (!targets || targets->n < 1 || targets->n > TG_MAIL_MAX_PEERS) return fail(TG_ERR_INVALID, "1..16 mailbox targets");
  DeviceGuard g(device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed (no usable CUDA device)");
  k_mail_signal<<<1, 32, 0, (cudaStream_t)stream>>>(*targets, reinterpret_cast<const unsigned long long*>(values_dev), (unsigned long long)epoch);
  TG_CUDA(cudaGetLastError());
  return TG_OK;
}

int tg_mail_wait(int device, const uint64_t* mail_dev, int32_t n, int64_t epoch, int64_t* values_out_dev, uint64_t* error_flag_dev,
                 int64_t timeout_ms, void* stream) {
  if (!mail_dev || !error_flag_dev || n < 1 || n > TG_MAIL_MAX_PEERS) return fail(TG_ERR_INVALID, "mail_dev / error_flag_dev required, 1..16 senders");
  DeviceGuard g(device);
  if (!g.ok) return fail(TG_ERR_CUDA, "cudaSetDevice failed (no usable CUDA device)");
  k_mail_wait<<<1, 32, 0, (cudaStream_t)stream>>>(reinterpret_cast<const unsigned long long*>(mail_dev), n, (unsigned long long)epoch,
                                                   reinterpret_cast<unsigned long long*>(values_out_dev), reinterpret_cast<unsigned long long*>(error_flag_dev),
                                                   (unsigned long long)(timeout_ms > 0 ? timeout_ms : 10000) * 1000000ull);
  TG_CUDA(cudaGetLastError());
  return TG_OK;
}

}  // extern "C"
