// partition_kernels.cuh — histogram + shared-memory-regrouped scatter by key hash (see partition.cu for the
// reference mapping).  Used twice: across GPUs (low hash bits) and, inside one GPU, to split a large probe side into
// L2-sized partitions (high hash bits) before the fused probe kernel (join.cu).
#pragma once
#include "common.cuh"
#include "tma.cuh"
#include <algorithm>
#include <cstdlib>

namespace tg {

#define TG_MAX_PARTS 16   // destinations of the count kernels (register arrays, k_partition_count4's 8-bit packed counters)
#define TG_MAX_SLICES 32  // destinations of the scatters: up to 32 L2 slices of a join probe (join.cu), TG_MAX_PARTS GPUs
#define TG_PART_MAX_COLS 8
#define PT_BLOCK 256
#define PT_ITEMS 8
#define PT_TILE (PT_BLOCK * PT_ITEMS)

struct PartDst {
  int32_t nparts, ncols;
  const void* src[TG_PART_MAX_COLS];
  void* dst[TG_MAX_SLICES][TG_PART_MAX_COLS];  // column base per destination
  // row offset inside the destination buffers where this launch starts writing, per destination
  const long long* dst_base;                   // device array [nparts]; nullptr = `base_const` for every destination
  long long base_const;
  // capacity > 0: destination p may hold at most `capacity` rows (count-free partitioning into fixed-size segments);
  // rows beyond it are dropped and *overflow is set — the caller then falls back to an unpartitioned pass.
  long long capacity;
  unsigned long long* overflow;
  // segmented INPUT (k_partition_scatter_bulk only): segment s = rows [s*in_cap, s*in_cap + min(in_cnt[s], in_cap)),
  // in_cap a multiple of the scatter tile; nullptr = dense input
  const unsigned long long* in_cnt;
  long long in_cap;
  uint32_t in_tiles_per_seg;
  // spill_cursor != nullptr (count-free mode): rows that do not fit their destination's capacity are not
  // dropped but appended to a LOCAL spill area (column c at spill[c], at most spill_cap rows, one global cursor); the host
  // drains it afterwards through a counted exchange.  *overflow is then raised only when the spill area itself is full.
  // A skewed key distribution makes the exchange slower, never wrong (the reference's exchange queues are unbounded).
  void* spill[TG_PART_MAX_COLS];
  long long spill_cap;
  unsigned long long* spill_cursor;
};

// HIGH = false: destination GPU, low 32 hash bits (disjoint from the slot bits).
// HIGH = true : local L2 partition, the TOP hash bits — the table slot is mulhi(h, nslots), monotone in h, so
//               partition p owns the contiguous slot range [p*nslots/P, (p+1)*nslots/P).
template <bool HIGH>
__device__ __forceinline__ uint32_t row_part(const long long* key, const uint8_t* nulls, int64_t i, uint32_t nparts) {
  uint64_t h = (nulls && !bit_not_null(nulls, i)) ? hash64((uint64_t)i)    // NULL keys never join: spread them
                                                   : hash64((uint64_t)__ldcs(key + i));
  return HIGH ? mulhi32((uint32_t)(h >> 32), nparts) : part_of(h, nparts);
}

template <bool HIGH>
__global__ void __launch_bounds__(256)
k_partition_count(const long long* __restrict__ key, const uint8_t* __restrict__ nulls, int64_t n, uint32_t nparts,
                  unsigned long long* __restrict__ counts) {
  __shared__ unsigned long long s_cnt[TG_MAX_PARTS];
  if (threadIdx.x < TG_MAX_PARTS) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  unsigned int local[TG_MAX_PARTS];
#pragma unroll
  for (int p = 0; p < TG_MAX_PARTS; p++) local[p] = 0;
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    uint32_t p = row_part<HIGH>(key, nulls, i, nparts);
#pragma unroll
    for (int q = 0; q < TG_MAX_PARTS; q++) local[q] += (p == (uint32_t)q);
  }
#pragma unroll
  for (int p = 0; p < TG_MAX_PARTS; p++) {
    unsigned int v = local[p];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(&s_cnt[p], (unsigned long long)v);
  }
  __syncthreads();
  if (threadIdx.x < nparts && s_cnt[threadIdx.x]) atomicAdd(&counts[threadIdx.x], s_cnt[threadIdx.x]);
}

// exclusive prefix of counts → part_offsets[nparts+1]; also seeds the scatter cursors
static __global__ void k_partition_offsets(const unsigned long long* counts, uint32_t nparts, long long* part_offsets,
                                    unsigned long long* cursors) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    long long run = 0;
    for (uint32_t p = 0; p < nparts; p++) { part_offsets[p] = run; cursors[p] = 0; run += (long long)counts[p]; }
    part_offsets[nparts] = run;
  }
}

// count-free partitioning: zero the fill counters and the overflow flag, lay the segments out back to back
static __global__ void k_segment_bases(unsigned long long* cursors, long long* bases, unsigned long long* flag, int nparts, long long cap) {
  if (threadIdx.x < TG_MAX_SLICES) { cursors[threadIdx.x] = 0; bases[threadIdx.x] = (long long)threadIdx.x * cap; }
  if (threadIdx.x == 0) *flag = 0;
  (void)nparts;
}

template <bool HIGH>
__global__ void __launch_bounds__(PT_BLOCK)
k_partition_scatter(const long long* __restrict__ key, const uint8_t* __restrict__ nulls, int64_t n, PartDst d,
                    unsigned long long* __restrict__ cursors) {
  __shared__ unsigned long long s_val[PT_TILE];
  __shared__ uint32_t s_cnt[TG_MAX_SLICES], s_off[TG_MAX_SLICES + 1], s_room[TG_MAX_SLICES];
  __shared__ unsigned long long s_gbase[TG_MAX_SLICES], s_spill[TG_MAX_SLICES];   // s_spill: first spill row of the rows that did not fit, ~0 = dropped
  const int lane = threadIdx.x & 31;
  const uint32_t P = (uint32_t)d.nparts;
  const int64_t ntiles = (n + PT_TILE - 1) / PT_TILE;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t base = tile * PT_TILE;
    if (threadIdx.x < TG_MAX_SLICES) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    // phase 1: destination of every row + rank inside (tile, destination), warp-aggregated
    uint32_t part[PT_ITEMS], rank[PT_ITEMS];
#pragma unroll
    for (int j = 0; j < PT_ITEMS; j++) {
      int64_t i = base + (int64_t)j * PT_BLOCK + threadIdx.x;
      bool in = i < n;
      uint32_t p = in ? row_part<HIGH>(key, nulls, i, P) : 0xffffffffu;
      unsigned peers = __match_any_sync(0xffffffffu, p);
      uint32_t r = 0;
      if (in) {
        int leader = __ffs(peers) - 1;
        uint32_t wbase = 0;
        if (lane == leader) wbase = atomicAdd(&s_cnt[p], (uint32_t)__popc(peers));
        wbase = __shfl_sync(peers, wbase, leader);
        r = wbase + __popc(peers & ((1u << lane) - 1));
      }
      part[j] = p; rank[j] = r;
    }
    __syncthreads();
    // phase 2: reserve a contiguous run per destination in the global cursors
    if (threadIdx.x == 0) {
      uint32_t run = 0;
      for (uint32_t p = 0; p < P; p++) { s_off[p] = run; run += s_cnt[p]; }
      s_off[P] = run;
    }
    if (threadIdx.x < P) {
      uint32_t c = s_cnt[threadIdx.x];
      unsigned long long old = c ? atomicAdd(&cursors[threadIdx.x], (unsigned long long)c) : 0ull;
      s_gbase[threadIdx.x] = old + (unsigned long long)(d.dst_base ? d.dst_base[threadIdx.x] : d.base_const);
      // rows of this tile that still fit the destination's capacity (0 = unbounded)
      unsigned long long room = d.capacity > 0 ? (old < (unsigned long long)d.capacity ? (unsigned long long)d.capacity - old : 0ull) : ~0ull;
      s_room[threadIdx.x] = room > c ? c : (uint32_t)room;
      unsigned long long sp = ~0ull;
      if (d.capacity > 0 && room < c) {
        if (d.spill_cursor) {
          const unsigned long long extra = (unsigned long long)c - room;
          sp = atomicAdd(d.spill_cursor, extra);
          if (sp + extra > (unsigned long long)d.spill_cap) { sp = ~0ull; *d.overflow = 1ull; }
        } else *d.overflow = 1ull;
      }
      s_spill[threadIdx.x] = sp;
    }
    __syncthreads();
    const uint32_t tile_rows = s_off[P];
    // phase 3: per column, regroup through shared memory and write coalesced runs
    for (int c = 0; c < d.ncols; c++) {
      const unsigned long long* src = reinterpret_cast<const unsigned long long*>(d.src[c]);
#pragma unroll
      for (int j = 0; j < PT_ITEMS; j++) {
        int64_t i = base + (int64_t)j * PT_BLOCK + threadIdx.x;
        if (i < n) s_val[s_off[part[j]] + rank[j]] = __ldcs(src + i);
      }
      __syncthreads();
      for (uint32_t sidx = threadIdx.x; sidx < tile_rows; sidx += PT_BLOCK) {
        uint32_t p = 0;
        while (sidx >= s_off[p + 1]) p++;   // ≤ nparts steps
        unsigned long long* dst = reinterpret_cast<unsigned long long*>(d.dst[p][c]);
        if (sidx - s_off[p] < s_room[p]) dst[s_gbase[p] + (sidx - s_off[p])] = s_val[sidx];
        else if (s_spill[p] != ~0ull) reinterpret_cast<unsigned long long*>(d.spill[c])[s_spill[p] + (sidx - s_off[p] - s_room[p])] = s_val[sidx];
      }
      __syncthreads();
    }
  }
}


// shared → global bulk store (cp.async.bulk, bulk_group completion) and its fences
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Scatter with the copy engine on BOTH sides (8-byte columns, no NULL keys): source tiles arrive through a 2-stage
// cp.async.bulk ring; each tile is regrouped by destination inside a shared-memory staging buffer and every
// (destination, column) run leaves as ONE bulk store (SASS UBLKCP ... to global; local HBM or a peer over NVLink).
// The run of destination p is parked at a staging offset whose parity equals the parity of its global row, so the
// 16-byte aligned middle of the run is a legal bulk copy; an odd head / tail element goes out as a scalar store.
// Threads only touch shared memory: per row one LDS + one atomic (rank) and, per column, one LDS + one STS.
// Count-free mode (d.capacity > 0): destinations are fixed-size segments and the global cursor atomics are the only
// bookkeeping — no histogram pass over the keys.  Full TILE-row tiles only; the caller handles the tail.
template <bool HIGH, int NC, int ITEMS, int THREADS = PT_BLOCK>
__global__ void __launch_bounds__(THREADS)
k_partition_scatter_bulk(int64_t ntiles, PartDst d, unsigned long long* __restrict__ cursors) {
  constexpr int STAGES = 2, TILE = THREADS * ITEMS, SROWS = TILE + 2 * TG_MAX_SLICES;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned long long* ring = reinterpret_cast<unsigned long long*>(smem_raw);      // [STAGES][NC][TILE]
  unsigned long long* stage = ring + (size_t)STAGES * NC * TILE;                   // [NC][SROWS]
  uint64_t* full = reinterpret_cast<uint64_t*>(stage + (size_t)NC * SROWS);
  __shared__ uint32_t s_cnt[TG_MAX_SLICES], s_off[TG_MAX_SLICES], s_len[TG_MAX_SLICES];
  __shared__ unsigned long long s_gbase[TG_MAX_SLICES], s_spg[TG_MAX_SLICES];
  __shared__ uint32_t s_spn[TG_MAX_SLICES];    // rows of this tile's run that go to the spill area, starting at spill row s_spg
  const int tid = threadIdx.x, lane = tid & 31;
  const uint32_t P = (uint32_t)d.nparts;
  const unsigned long long pol = l2_policy_evict_first();
  if (tid == 0) {
    for (int s = 0; s < STAGES; s++) mbar_init(&full[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  auto issue = [&](int64_t it) {
    int64_t tile = (int64_t)blockIdx.x + it * gridDim.x;
    if (tile >= ntiles) return;
    int s = (int)(it % STAGES);
    mbar_arrive_expect_tx(&full[s], (uint32_t)(NC * TILE * 8));
#pragma unroll
    for (int c = 0; c < NC; c++)
      bulk_g2s(ring + ((size_t)s * NC + c) * TILE, reinterpret_cast<const unsigned long long*>(d.src[c]) + tile * TILE, TILE * 8, &full[s], pol);
  };
  if (tid == 0) for (int it = 0; it < STAGES; it++) issue(it);
  for (int64_t it = 0;; it++) {
    const int64_t tile = (int64_t)blockIdx.x + it * gridDim.x;
    if (tile >= ntiles) break;
    const int s = (int)(it % STAGES);
    if (tid < TG_MAX_SLICES) s_cnt[tid] = 0;
    mbar_wait(&full[s], (uint32_t)((it / STAGES) & 1));
    __syncthreads();
    const unsigned long long* in = ring + (size_t)s * NC * TILE;
    int valid = TILE;     // rows of this tile that exist (segmented input: the tail of a segment is padding)
    if (d.in_cnt) {
      const uint32_t sg = (uint32_t)tile / d.in_tiles_per_seg;
      const unsigned long long c = d.in_cnt[sg];
      const long long left = (long long)sg * d.in_cap + (long long)(c < (unsigned long long)d.in_cap ? c : (unsigned long long)d.in_cap) - tile * TILE;
      valid = left <= 0 ? 0 : (left < TILE ? (int)left : TILE);
    }
    uint32_t pr[ITEMS];   // destination << 16 | rank inside (tile, destination); 0xffff.... = padding row
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      if (j * THREADS + tid < valid) {
        uint64_t h = hash64(in[j * THREADS + tid]);
        uint32_t p = HIGH ? mulhi32((uint32_t)(h >> 32), P) : part_of(h, P);
        pr[j] = (p << 16) | atomicAdd(&s_cnt[p], 1u);
      } else pr[j] = 0xffffffffu;
    }
    __syncthreads();
    if (tid < 32) {
      uint32_t c = tid < (int)P ? s_cnt[tid] : 0, len = c, spn = 0;
      unsigned long long g = 0, spg = 0;
      if (tid < (int)P) {
        unsigned long long old = c ? atomicAdd(&cursors[tid], (unsigned long long)c) : 0ull;
        if (d.capacity > 0) {
          unsigned long long avail = old < (unsigned long long)d.capacity ? (unsigned long long)d.capacity - old : 0ull;
          if ((unsigned long long)c > avail) {
            len = (uint32_t)avail;
            if (d.spill_cursor) {   // skewed destination: the rest of the run goes to the local spill area
              spn = c - len;
              spg = atomicAdd(d.spill_cursor, (unsigned long long)spn);
              if (spg + spn > (unsigned long long)d.spill_cap) { spn = 0; *d.overflow = 1ull; }
            } else *d.overflow = 1ull;
          }
        }
        g = old + (unsigned long long)(d.dst_base ? d.dst_base[tid] : d.base_const);
      }
      uint32_t w = tid < (int)P ? (((uint32_t)(g & 1) + c + 1) & ~1u) : 0, incl = w;
      for (int o = 1; o < 32; o <<= 1) { uint32_t u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
      if (tid < (int)P) { s_off[tid] = incl - w + (uint32_t)(g & 1); s_gbase[tid] = g; s_len[tid] = len; s_spg[tid] = spg; s_spn[tid] = spn; }
    }
    if (tid < (int)P * NC) bulk_wait_read_all();   // the previous tile's bulk stores have read the staging buffer
    __syncthreads();
#pragma unroll
    for (int c = 0; c < NC; c++) {
#pragma unroll
      for (int j = 0; j < ITEMS; j++)
        if (pr[j] != 0xffffffffu) stage[(size_t)c * SROWS + s_off[pr[j] >> 16] + (pr[j] & 0xffffu)] = in[(size_t)c * TILE + j * THREADS + tid];
    }
    fence_async_smem();              // generic-proxy STS → visible to the async proxy that executes the bulk stores
    __syncthreads();                 // staging complete, ring stage s fully consumed (LDS results fed the STS above)
    if (tid == 0) issue(it + STAGES);
    if (tid < (int)P * NC) {
      const uint32_t p = tid / NC, c = tid % NC;
      const unsigned long long g = s_gbase[p];
      const uint32_t len = s_len[p], so = s_off[p];
      unsigned long long* dst = reinterpret_cast<unsigned long long*>(d.dst[p][c]);
      const unsigned long long* src = stage + (size_t)c * SROWS;
      const uint32_t head = (uint32_t)(g & 1) & (len > 0 ? 1u : 0u);
      const uint32_t mid = (len - head) & ~1u;
      if (mid) bulk_s2g(dst + g + head, src + so + head, mid * 8);
      bulk_commit();
      if (head) dst[g] = src[so];
      if ((len - head) & 1u) dst[g + len - 1] = src[so + len - 1];
      const uint32_t spn = s_spn[p];
      if (spn) {   // rare (skew): scalar stores, the staging buffer is released by the bulk_wait_read_all + barrier of the next tile like the runs above
        unsigned long long* sp = reinterpret_cast<unsigned long long*>(d.spill[c]) + s_spg[p];
        for (uint32_t r = 0; r < spn; r++) sp[r] = src[so + len + r];
      }
    }
  }
  if (tid < (int)P * NC) bulk_wait_read_all();
}

// histogram of destinations: 128-bit loads, 4 in flight per thread, counts packed 8 x 8 bit in two 64-bit registers
template <bool HIGH>
__global__ void __launch_bounds__(256)
k_partition_count4(const long long* __restrict__ key, int64_t n, uint32_t nparts, unsigned long long* __restrict__ counts) {
  __shared__ unsigned long long s_cnt[TG_MAX_PARTS];
  if (threadIdx.x < TG_MAX_PARTS) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  unsigned int local[TG_MAX_PARTS];
#pragma unroll
  for (int p = 0; p < TG_MAX_PARTS; p++) local[p] = 0;
  unsigned long long a0 = 0, a1 = 0;
  int pending = 0;
  auto add = [&](uint64_t k) {
    uint64_t h = hash64(k);
    uint32_t p = HIGH ? mulhi32((uint32_t)(h >> 32), nparts) : part_of(h, nparts);
    unsigned long long inc = 1ull << ((p & 7u) << 3);
    a0 += (p < 8u) ? inc : 0ull;
    a1 += (p < 8u) ? 0ull : inc;
  };
  auto flush = [&]() {
#pragma unroll
    for (int q = 0; q < 8; q++) { local[q] += (unsigned int)((a0 >> (8 * q)) & 0xffu); local[8 + q] += (unsigned int)((a1 >> (8 * q)) & 0xffu); }
    a0 = a1 = 0; pending = 0;
  };
  const int64_t n2 = n >> 1;   // pairs, loaded as 128-bit
  const ulonglong2* k2 = reinterpret_cast<const ulonglong2*>(key);
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n2; i += 4 * stride) {
    ulonglong2 v[4];
    bool ok[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      int64_t q = i + u * stride;
      ok[u] = q < n2;
      v[u] = ok[u] ? __ldcs(k2 + q) : make_ulonglong2(0ull, 0ull);
    }
#pragma unroll
    for (int u = 0; u < 4; u++) if (ok[u]) { add(v[u].x); add(v[u].y); }
    pending += 8;
    if (pending > 240) flush();
  }
  if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) add((uint64_t)key[n - 1]);
  flush();
#pragma unroll
  for (int p = 0; p < TG_MAX_PARTS; p++) {
    unsigned int v = local[p];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(&s_cnt[p], (unsigned long long)v);
  }
  __syncthreads();
  if (threadIdx.x < nparts && s_cnt[threadIdx.x]) atomicAdd(&counts[threadIdx.x], s_cnt[threadIdx.x]);
}


// ---- host launchers shared by partition.cu (across GPUs, low hash bits) and join.cu (L2 partitions, top bits) ----------
inline bool ptr_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <bool HIGH>
inline int launch_partition_count(int device, cudaStream_t st, const long long* key, const uint8_t* nulls, int64_t n, uint32_t nparts,
                                  unsigned long long* counts, int64_t* launches) {
  if (n <= 0) return TG_OK;
  int nsm = device_sm_count(device);
  if (!nulls && ptr_aligned16(key)) {
    int64_t need = ((n + 7) / 8 + 255) / 256;
    int grid = (int)std::min<int64_t>(std::max<int64_t>(need, 1), (int64_t)nsm * 8);
    k_partition_count4<HIGH><<<grid, 256, 0, st>>>(key, n, nparts, counts);
  } else {
    int64_t need = (n + 255) / 256;
    int grid = (int)std::min<int64_t>(std::max<int64_t>(need, 1), (int64_t)nsm * 8);
    k_partition_count<HIGH><<<grid, 256, 0, st>>>(key, nulls, n, nparts, counts);
  }
  if (launches) (*launches)++;
  return TG_OK;
}

// Rows per tile of k_partition_scatter_bulk for `ncols` columns.  The L2 partition pass of a join (HIGH) over dense input
// with at most 2 columns takes 4096-row tiles of 512 threads: a quarter of the per-tile bookkeeping (barriers, cursor
// atomics, the staging drain) per row, at one CTA per SM (193 KiB of shared memory at 2 columns); the pass got faster with
// every doubling of the tile (DESIGN.md §4.1, "4096-row scatter tiles").  Everything else takes 1024-row tiles of 256
// threads: segmented input, whose segment capacities are multiples of 1024 rows; the exchange across GPUs, whose
// mailboxes are sized in 1024-row tiles; and 3–4 columns, whose 4096-row tile does not fit in shared memory.
inline int64_t scatter_tile_rows(bool high, bool segmented, int ncols) {
  return high && !segmented && ncols <= 2 ? 4096 : 1024;
}

template <bool HIGH, int NC, int ITEMS, int THREADS>
inline int launch_scatter_tiles(int device, cudaStream_t st, int64_t n, PartDst& d, unsigned long long* cursors, int64_t* launches, int ctas_per_sm,
                                int32_t* paths) {
  int nsm = device_sm_count(device);
  constexpr int TILE = THREADS * ITEMS;
  int64_t ntiles = n / TILE;
  if (ntiles > 0) {
    size_t smem = (size_t)2 * NC * TILE * 8 + (size_t)NC * (TILE + 2 * TG_MAX_SLICES) * 8 + 2 * 8 + 16;
    TG_CUDA(cudaFuncSetAttribute(k_partition_scatter_bulk<HIGH, NC, ITEMS, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // 4 CTAs per SM with 1024-row tiles of <= 2 columns, 1 with 4096-row tiles
    int per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (size_t)(220 * 1024) / (smem + 1024)));
    // a scatter that runs NEXT TO a probe kernel (exchange of step k+1 under the probe of step k) should leave the SMs'
    // L1 to the probe: TG_SCATTER_CTAS_PER_SM caps the CTAs (and with them the shared-memory carve-out) per SM
    const int cap_env = env_int("TG_SCATTER_CTAS_PER_SM", 0);
    if (!HIGH && cap_env > 0 && per_sm > cap_env) per_sm = cap_env;
    if (ctas_per_sm > 0 && per_sm > ctas_per_sm) per_sm = ctas_per_sm;
    int grid = (int)std::min<int64_t>(ntiles, (int64_t)nsm * per_sm);
    k_partition_scatter_bulk<HIGH, NC, ITEMS, THREADS><<<grid, THREADS, smem, st>>>(ntiles, d, cursors);
    if (launches) (*launches)++;
    if (paths) *paths |= TG_JOIN_PATH_SCATTER_BULK | (TILE == 4096 ? TG_JOIN_SCATTER_TILE_4K : 0);
  }
  int64_t done = ntiles * TILE;
  if (done < n) {
    if (d.capacity > 0) return fail(TG_ERR_CUDA, "internal: capacity-bounded scatter needs a whole number of tiles");
    PartDst tail = d;
    for (int c = 0; c < NC; c++) tail.src[c] = reinterpret_cast<const unsigned long long*>(d.src[c]) + done;
    k_partition_scatter<HIGH><<<1, PT_BLOCK, 0, st>>>(reinterpret_cast<const long long*>(tail.src[0]), nullptr, n - done, tail, cursors);
    if (launches) (*launches)++;
  }
  return TG_OK;
}

template <bool HIGH, int NC>
inline int launch_scatter_nc(int device, cudaStream_t st, int64_t n, PartDst& d, unsigned long long* cursors, int64_t* launches, int ctas_per_sm,
                             int32_t* paths) {
  if constexpr (HIGH && NC <= 2) {
    if (scatter_tile_rows(HIGH, d.in_cnt != nullptr, NC) == 4096)
      return launch_scatter_tiles<HIGH, NC, 8, 512>(device, st, n, d, cursors, launches, ctas_per_sm, paths);
  }
  return launch_scatter_tiles<HIGH, NC, 4, PT_BLOCK>(device, st, n, d, cursors, launches, ctas_per_sm, paths);
}

// d.src[0] must be the key column; falls back to the LSU kernel for NULL-able keys, unaligned sources or > 4 columns.
// `paths` (optional) gains TG_JOIN_PATH_SCATTER_BULK when the bulk kernel ran, TG_JOIN_PATH_SCATTER when the LSU kernel
// scattered the whole input (the < 1-tile remainder behind the bulk kernel is not counted)
template <bool HIGH>
inline int launch_partition_scatter(int device, cudaStream_t st, const long long* key, const uint8_t* nulls, int64_t n, PartDst& d,
                                    unsigned long long* cursors, int64_t* launches, int ctas_per_sm = 0, int32_t* paths = nullptr) {
  if (n <= 0) return TG_OK;
  bool tma_ok = !nulls && d.ncols <= 4 && d.src[0] == (const void*)key;
  for (int c = 0; c < d.ncols && tma_ok; c++) tma_ok = ptr_aligned16(d.src[c]);
  // the bulk stores start at dst + (even row): every destination column base must be 16-byte aligned too
  for (int p = 0; p < d.nparts && tma_ok; p++) for (int c = 0; c < d.ncols && tma_ok; c++) tma_ok = ptr_aligned16(d.dst[p][c]);
  if (tma_ok) {
    switch (d.ncols) {
      case 1: return launch_scatter_nc<HIGH, 1>(device, st, n, d, cursors, launches, ctas_per_sm, paths);
      case 2: return launch_scatter_nc<HIGH, 2>(device, st, n, d, cursors, launches, ctas_per_sm, paths);
      case 3: return launch_scatter_nc<HIGH, 3>(device, st, n, d, cursors, launches, ctas_per_sm, paths);
      default: return launch_scatter_nc<HIGH, 4>(device, st, n, d, cursors, launches, ctas_per_sm, paths);
    }
  }
  int nsm = device_sm_count(device);
  int64_t tiles = (n + PT_TILE - 1) / PT_TILE;
  int grid = (int)std::min<int64_t>(tiles, (int64_t)nsm * 4);
  k_partition_scatter<HIGH><<<grid, PT_BLOCK, 0, st>>>(key, nulls, n, d, cursors);
  if (launches) (*launches)++;
  if (paths) *paths |= TG_JOIN_PATH_SCATTER;
  return TG_OK;
}

}  // namespace tg
