// probe_lab.cu — scratch harness for the fused-probe kernel structure (not part of the library).
// Measures, on the bench workload (100 M probe rows, 10 M build keys, 16-byte slots, load factor 0.4):
//   S*  pure streaming kernels with the probe's traffic shape (16 B in, 32 B out per row), to find the ceiling
//   P*  probe kernels on the unpartitioned input and on the input regrouped by L2 partition
// build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -I include -I tidb_b200/csrc \
//        tools/scratch/probe_lab.cu tidb_b200/csrc/runtime.cu -o tools/scratch/probe_lab
#include "join_kernels.cuh"
#include "partition_kernels.cuh"
#include <thrust/device_ptr.h>
#include <thrust/sort.h>
#include <thrust/sequence.h>
#include <thrust/reduce.h>
#include <thrust/execution_policy.h>
#include <cstdio>
#include <vector>
#include <string>

using namespace tg;
typedef unsigned long long u64;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA %s at line %d\n", cudaGetErrorString(e_), __LINE__); exit(1); } } while (0)

static const u64 ODD = 0x9E3779B97F4A7C15ull;

// ------------------------------------------------------------------ data generation
__global__ void k_gen_build(int64_t* bk, u64* bp, int64_t nb) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < nb) { bk[i] = (int64_t)((u64)(i + 1) * ODD); bp[i] = (u64)i * 3 + 7; }
}
__device__ __forceinline__ u64 rnd64(u64 x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return x; }
__global__ void k_gen_probe(int64_t* pk, u64* pv, int64_t n, int64_t nb, u64 seed) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) { u64 id = rnd64((u64)i + seed) % (u64)nb; pk[i] = (int64_t)((id + 1) * ODD); pv[i] = (u64)i; }
}
__global__ void k_lab_init(Slot* s, u64 n) {
  u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
  if (i < n) { s[i].key = kEmptyKey; s[i].meta = 0; }
}
__global__ void k_lab_insert(const int64_t* bk, const u64* bp, int64_t nb, Slot* slots, u64 nslots, int home_width = 2) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= nb) return;
  int64_t k = bk[i];
  u64 s = home_slot(hash64((uint64_t)k), nslots, home_width);
  for (;;) {
    unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(&slots[s].key), (unsigned long long)kEmptyKey, (unsigned long long)k);
    if (prev == (unsigned long long)kEmptyKey) { slots[s].meta = bp[i]; return; }
    if (++s == nslots) s = 0;
  }
}
__global__ void k_part_of(const int64_t* pk, int64_t n, uint32_t P, uint8_t* part) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) part[i] = (uint8_t)mulhi32((uint32_t)(hash64((uint64_t)pk[i]) >> 32), P);
}
__global__ void k_gather2(const int64_t* pk, const u64* pv, const uint32_t* idx, int64_t n, int64_t* ok, u64* ov) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) { ok[i] = pk[idx[i]]; ov[i] = pv[idx[i]]; }
}
// output check: o0 = probe key, o1 = build key (== probe key), o2 = probe payload (row id), o3 = build payload
__global__ void k_check(const u64* o0, const u64* o1, const u64* o2, const u64* o3, int64_t n, u64* acc) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  u64 bad = 0, s2 = 0, s3 = 0;
  for (; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    u64 k = o0[i];
    bad += (o1[i] != k);
    u64 id = k * 0xf1de83e19937733dull;   // inverse of ODD mod 2^64 → id+1
    bad += (o3[i] != (id - 1) * 3 + 7);
    s2 += o2[i]; s3 += o3[i];
  }
  for (int o = 16; o; o >>= 1) { bad += __shfl_xor_sync(~0u, bad, o); s2 += __shfl_xor_sync(~0u, s2, o); s3 += __shfl_xor_sync(~0u, s3, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(acc, bad); atomicAdd(acc + 1, s2); atomicAdd(acc + 2, s3); }
}

// ------------------------------------------------------------------ S: streaming ceilings (16 B in, 32 B out per row)
template <int R, bool CS>
__global__ void __launch_bounds__(256) k_stream_scalar(const u64* __restrict__ a, const u64* __restrict__ b, int64_t n,
                                                       u64* __restrict__ o0, u64* __restrict__ o1, u64* __restrict__ o2, u64* __restrict__ o3) {
  const int64_t stride = (int64_t)gridDim.x * 256 * R;
  for (int64_t base = (int64_t)blockIdx.x * 256 * R + threadIdx.x; base < n; base += stride) {
    u64 x[R], y[R];
#pragma unroll
    for (int j = 0; j < R; j++) { int64_t i = base + j * 256; if (i < n) { x[j] = CS ? __ldcs(a + i) : a[i]; y[j] = CS ? __ldcs(b + i) : b[i]; } }
#pragma unroll
    for (int j = 0; j < R; j++) {
      int64_t i = base + j * 256;
      if (i < n) {
        if (CS) { __stcs(o0 + i, x[j]); __stcs(o1 + i, x[j] + 1); __stcs(o2 + i, y[j]); __stcs(o3 + i, y[j] + 1); }
        else { o0[i] = x[j]; o1[i] = x[j] + 1; o2[i] = y[j]; o3[i] = y[j] + 1; }
      }
    }
  }
}
template <int R>
__global__ void __launch_bounds__(256) k_stream_vec2(const ulonglong2* __restrict__ a, const ulonglong2* __restrict__ b, int64_t n2,
                                                     ulonglong2* __restrict__ o0, ulonglong2* __restrict__ o1, ulonglong2* __restrict__ o2, ulonglong2* __restrict__ o3) {
  const int64_t stride = (int64_t)gridDim.x * 256 * R;
  for (int64_t base = (int64_t)blockIdx.x * 256 * R + threadIdx.x; base < n2; base += stride) {
    ulonglong2 x[R], y[R];
#pragma unroll
    for (int j = 0; j < R; j++) { int64_t i = base + j * 256; if (i < n2) { x[j] = __ldcs(a + i); y[j] = __ldcs(b + i); } }
#pragma unroll
    for (int j = 0; j < R; j++) {
      int64_t i = base + j * 256;
      if (i < n2) {
        __stcs(o0 + i, x[j]); __stcs(o2 + i, y[j]);
        x[j].x += 1; x[j].y += 1; y[j].x += 1; y[j].y += 1;
        __stcs(o1 + i, x[j]); __stcs(o3 + i, y[j]);
      }
    }
  }
}

template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }

// TMA in (ring of T-row tiles) and TMA out (double-buffered staging): the copy engine moves everything, threads only
// touch shared memory
template <int T, int STAGES>
__global__ void __launch_bounds__(256) k_stream_tma(const u64* __restrict__ a, const u64* __restrict__ b, int64_t ntiles,
                                                    u64* __restrict__ o0, u64* __restrict__ o1, u64* __restrict__ o2, u64* __restrict__ o3) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  u64* ring = reinterpret_cast<u64*>(smem_raw);                       // [STAGES][2][T]
  u64* outb = ring + (size_t)STAGES * 2 * T;                          // [2][4][T]
  uint64_t* full = reinterpret_cast<uint64_t*>(outb + (size_t)2 * 4 * T);
  const int tid = threadIdx.x;
  const u64 pol = l2_policy_evict_first();
  if (tid == 0) { for (int s = 0; s < STAGES; s++) mbar_init(&full[s], 1); mbar_fence_init(); }
  __syncthreads();
  auto issue = [&](int64_t it) {
    int64_t tile = (int64_t)blockIdx.x + it * gridDim.x;
    if (tile >= ntiles) return;
    int s = (int)(it % STAGES);
    u64* st = ring + (size_t)s * 2 * T;
    mbar_arrive_expect_tx(&full[s], 2 * T * 8);
    bulk_g2s(st, a + tile * T, T * 8, &full[s], pol);
    bulk_g2s(st + T, b + tile * T, T * 8, &full[s], pol);
  };
  if (tid == 0) for (int it = 0; it < STAGES; it++) issue(it);
  for (int64_t it = 0;; it++) {
    const int64_t tile = (int64_t)blockIdx.x + it * gridDim.x;
    if (tile >= ntiles) break;
    const int s = (int)(it % STAGES);
    mbar_wait(&full[s], (uint32_t)((it / STAGES) & 1));
    const u64* st = ring + (size_t)s * 2 * T;
    u64* ob = outb + (size_t)(it & 1) * 4 * T;
    if (tid == 0) bulk_wait_read<1>();      // the stores issued from this staging buffer two tiles ago have read it
    __syncthreads();
#pragma unroll
    for (int j = 0; j < T / 256; j++) {
      u64 x = st[j * 256 + tid], y = st[T + j * 256 + tid];
      ob[j * 256 + tid] = x; ob[T + j * 256 + tid] = x + 1; ob[2 * T + j * 256 + tid] = y; ob[3 * T + j * 256 + tid] = y + 1;
    }
    fence_async_smem();
    __syncthreads();
    if (tid == 0) {
      issue(it + STAGES);
      bulk_s2g(o0 + tile * T, ob, T * 8); bulk_s2g(o1 + tile * T, ob + T, T * 8);
      bulk_s2g(o2 + tile * T, ob + 2 * T, T * 8); bulk_s2g(o3 + tile * T, ob + 3 * T, T * 8);
      bulk_commit();
    }
  }
  if (tid == 0) bulk_wait_read<0>();
}

// ------------------------------------------------------------------ P: probe variants
struct Out4 { u64* key_p; u64* key_b; u64* pay_p; u64* pay_b; };

// shared gather+match for R rows of a lane; returns ballots
template <int R>
__device__ __forceinline__ uint32_t gather_match(const int64_t (&k)[R], const TableView& t, u64 (&meta)[R], unsigned (&bal)[R]) {
  Slot v[R], w[R];
#pragma unroll
  for (int j = 0; j < R; j++) {
    u64 sl = home_slot(hash64((uint64_t)k[j]), t.nslots, 2);
    load_pair(t.slots + sl, v[j], w[j]);
  }
  uint32_t total = 0;
#pragma unroll
  for (int j = 0; j < R; j++) {
    bool m;
    if (v[j].key == k[j]) { m = true; meta[j] = v[j].meta; }
    else if (w[j].key == k[j]) { m = true; meta[j] = w[j].meta; }
    else if (v[j].key == kEmptyKey || w[j].key == kEmptyKey) { m = false; meta[j] = 0; }
    else {
      u64 sl = home_slot(hash64((uint64_t)k[j]), t.nslots, 2) + 2;
      if (sl >= t.nslots) sl = 0;
      Slot x = load_slot(t.slots + sl);
      while (x.key != k[j] && x.key != kEmptyKey) { if (++sl == t.nslots) sl = 0; x = load_slot(t.slots + sl); }
      m = x.key == k[j]; meta[j] = x.meta;
    }
    bal[j] = __ballot_sync(0xffffffffu, m);
    total += __popc(bal[j]);
  }
  return total;
}

// P2: warp kernel, each lane owns 2 ADJACENT rows per step (128-bit loads); when the whole warp tile matched and the
// output base is even, the four output columns are written with 128-bit stores
template <int G, int MINB = 1>   // G groups of 64 rows per warp tile
__global__ void __launch_bounds__(256, MINB) k_probe_vec2(const int64_t* __restrict__ pkey, const u64* __restrict__ ppay, int64_t n, TableView t, Out4 o,
                                                    u64* __restrict__ cursor) {
  constexpr int R = 2 * G;
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * 8, warp_id = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int64_t ntiles = n / (64 * G);   // lab: n is a multiple of the tile
  for (int64_t tile = warp_id; tile < ntiles; tile += warps_total) {
    const int64_t base = tile * 64 * G;
    int64_t k[R]; u64 pv[R], meta[R]; unsigned bal[R];
#pragma unroll
    for (int g = 0; g < G; g++) {
      ulonglong2 kk = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + base + g * 64) + lane);
      ulonglong2 pp = __ldcs(reinterpret_cast<const ulonglong2*>(ppay + base + g * 64) + lane);
      k[2 * g] = (int64_t)kk.x; k[2 * g + 1] = (int64_t)kk.y; pv[2 * g] = pp.x; pv[2 * g + 1] = pp.y;
    }
    uint32_t total = gather_match<R>(k, t, meta, bal);
    u64 wbase = 0;
    if (lane == 0 && total) wbase = atomicAdd(cursor, (u64)total);
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (total == 64 * G && (wbase & 1) == 0) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const u64 ob = wbase + g * 64;
        ulonglong2 kk = make_ulonglong2((u64)k[2 * g], (u64)k[2 * g + 1]);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_p + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_b + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_p + ob) + lane, make_ulonglong2(pv[2 * g], pv[2 * g + 1]));
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_b + ob) + lane, make_ulonglong2(meta[2 * g], meta[2 * g + 1]));
      }
    } else {
#pragma unroll
      for (int j = 0; j < R; j++) {
        if ((bal[j] >> lane) & 1u) {
          const u64 q = wbase + __popc(bal[j] & ((1u << lane) - 1));
          __stcs(o.key_p + q, (u64)k[j]); __stcs(o.key_b + q, (u64)k[j]); __stcs(o.pay_p + q, pv[j]); __stcs(o.pay_b + q, meta[j]);
        }
        wbase += __popc(bal[j]);
      }
    }
  }
}

// P4: warp-autonomous, LDG in, output through per-warp shared-memory staging + bulk stores (cp.async.bulk s2g).
// PREFETCH: keep the next tile's key/payload loads in flight while the current tile is gathered.
#define STG_ROWS 132      // 128 + head parity + pad; 132*8 = 1056 bytes = 66 * 16
template <bool PREFETCH>
__global__ void __launch_bounds__(256) k_probe_bulkout(const int64_t* __restrict__ pkey, const u64* __restrict__ ppay, int64_t n, TableView t, Out4 o,
                                                       u64* __restrict__ cursor) {
  constexpr int R = 4;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  u64* stage = reinterpret_cast<u64*>(smem_raw) + (size_t)warp * 2 * 4 * STG_ROWS;   // [2][4][STG_ROWS]
  const int64_t warps_total = (int64_t)gridDim.x * 8, warp_id = (int64_t)blockIdx.x * 8 + warp;
  const int64_t ntiles = n / 128;
  u64* const dst[4] = {o.key_p, o.key_b, o.pay_p, o.pay_b};
  int64_t kn[R]; u64 pn[R];
  int64_t tile = warp_id;
  if (PREFETCH && tile < ntiles) {
#pragma unroll
    for (int j = 0; j < R; j++) { kn[j] = (int64_t)__ldcs(reinterpret_cast<const u64*>(pkey) + tile * 128 + j * 32 + lane); pn[j] = __ldcs(ppay + tile * 128 + j * 32 + lane); }
  }
  for (int it = 0; tile < ntiles; tile += warps_total, it++) {
    int64_t k[R]; u64 pv[R], meta[R]; unsigned bal[R];
    if (PREFETCH) {
#pragma unroll
      for (int j = 0; j < R; j++) { k[j] = kn[j]; pv[j] = pn[j]; }
      const int64_t nt = tile + warps_total;
      if (nt < ntiles) {
#pragma unroll
        for (int j = 0; j < R; j++) { kn[j] = (int64_t)__ldcs(reinterpret_cast<const u64*>(pkey) + nt * 128 + j * 32 + lane); pn[j] = __ldcs(ppay + nt * 128 + j * 32 + lane); }
      }
    } else {
#pragma unroll
      for (int j = 0; j < R; j++) { k[j] = (int64_t)__ldcs(reinterpret_cast<const u64*>(pkey) + tile * 128 + j * 32 + lane); pv[j] = __ldcs(ppay + tile * 128 + j * 32 + lane); }
    }
    uint32_t total = gather_match<R>(k, t, meta, bal);
    u64 wbase = 0;
    if (lane == 0 && total) wbase = atomicAdd(cursor, (u64)total);
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    u64* sb = stage + (size_t)(it & 1) * 4 * STG_ROWS;
    if (lane < 4) bulk_wait_read<1>();      // stores issued from this buffer two tiles ago have finished reading it
    __syncwarp();
    const uint32_t par = (uint32_t)(wbase & 1);
    uint32_t q = par;
#pragma unroll
    for (int j = 0; j < R; j++) {
      if ((bal[j] >> lane) & 1u) {
        const uint32_t r = q + __popc(bal[j] & ((1u << lane) - 1));
        sb[r] = (u64)k[j]; sb[STG_ROWS + r] = (u64)k[j]; sb[2 * STG_ROWS + r] = pv[j]; sb[3 * STG_ROWS + r] = meta[j];
      }
      q += __popc(bal[j]);
    }
    fence_async_smem();
    __syncwarp();
    // staging index q ↔ global row (wbase - par + q); even q is 16-byte aligned on both sides
    const uint32_t q_end = par + total;
    const uint32_t q_lo = par ? 2u : 0u, q_hi = q_end & ~1u;
    const u64 g0 = wbase - par;
    if (lane < 4) {
      if (q_hi > q_lo) bulk_s2g(dst[lane] + g0 + q_lo, sb + lane * STG_ROWS + q_lo, (q_hi - q_lo) * 8);
      bulk_commit();
      if (par && total) dst[lane][g0 + 1] = sb[lane * STG_ROWS + 1];                                   // head
      if ((q_end & 1u) && q_end - 1 >= q_lo && total) dst[lane][g0 + q_end - 1] = sb[lane * STG_ROWS + q_end - 1];   // tail
    }
  }
  if (lane < 4) bulk_wait_read<0>();
}

// P3: per-warp TMA input ring (STAGES x 128 rows x 2 columns) + per-warp bulk output; fully warp-autonomous
template <int STAGES>
__global__ void __launch_bounds__(256) k_probe_tma_io(const int64_t* __restrict__ pkey, const u64* __restrict__ ppay, int64_t n, TableView t, Out4 o,
                                                      u64* __restrict__ cursor) {
  constexpr int R = 4;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr size_t WARP_U64 = (size_t)STAGES * 2 * 128 + 2 * 4 * STG_ROWS + ((STAGES + 1) & ~1);
  u64* wb = reinterpret_cast<u64*>(smem_raw) + (size_t)warp * WARP_U64;
  u64* ring = wb;                                  // [STAGES][2][128]
  u64* stage = wb + (size_t)STAGES * 2 * 128;      // [2][4][STG_ROWS]
  uint64_t* full = reinterpret_cast<uint64_t*>(stage + 2 * 4 * STG_ROWS);
  const int64_t warps_total = (int64_t)gridDim.x * 8, warp_id = (int64_t)blockIdx.x * 8 + warp;
  const int64_t ntiles = n / 128;
  u64* const dst[4] = {o.key_p, o.key_b, o.pay_p, o.pay_b};
  const u64 pol = l2_policy_evict_first();
  if (lane == 0) { for (int s = 0; s < STAGES; s++) mbar_init(&full[s], 1); mbar_fence_init(); }
  __syncwarp();
  auto issue = [&](int64_t it) {
    int64_t tile = warp_id + it * warps_total;
    if (tile >= ntiles) return;
    int s = (int)(it % STAGES);
    mbar_arrive_expect_tx(&full[s], 2 * 128 * 8);
    bulk_g2s(ring + (size_t)s * 256, pkey + tile * 128, 1024, &full[s], pol);
    bulk_g2s(ring + (size_t)s * 256 + 128, ppay + tile * 128, 1024, &full[s], pol);
  };
  if (lane == 0) for (int it = 0; it < STAGES; it++) issue(it);
  for (int64_t it = 0;; it++) {
    const int64_t tile = warp_id + it * warps_total;
    if (tile >= ntiles) break;
    const int s = (int)(it % STAGES);
    mbar_wait(&full[s], (uint32_t)((it / STAGES) & 1));
    int64_t k[R]; u64 pv[R], meta[R]; unsigned bal[R];
    u64 dep = 0;
#pragma unroll
    for (int j = 0; j < R; j++) { k[j] = (int64_t)ring[(size_t)s * 256 + j * 32 + lane]; pv[j] = ring[(size_t)s * 256 + 128 + j * 32 + lane]; dep ^= pv[j] ^ (u64)k[j]; }
    if (dep == 0x9E3779B97F4A7C15ull && n == -5) cursor[1] = dep;   // consume the LDS results before the refill below
    __syncwarp();
    if (lane == 0) issue(it + STAGES);
    uint32_t total = gather_match<R>(k, t, meta, bal);
    u64 wbase = 0;
    if (lane == 0 && total) wbase = atomicAdd(cursor, (u64)total);
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    u64* sb = stage + (size_t)(it & 1) * 4 * STG_ROWS;
    if (lane < 4) bulk_wait_read<1>();
    __syncwarp();
    const uint32_t par = (uint32_t)(wbase & 1);
    uint32_t q = par;
#pragma unroll
    for (int j = 0; j < R; j++) {
      if ((bal[j] >> lane) & 1u) {
        const uint32_t r = q + __popc(bal[j] & ((1u << lane) - 1));
        sb[r] = (u64)k[j]; sb[STG_ROWS + r] = (u64)k[j]; sb[2 * STG_ROWS + r] = pv[j]; sb[3 * STG_ROWS + r] = meta[j];
      }
      q += __popc(bal[j]);
    }
    fence_async_smem();
    __syncwarp();
    const uint32_t q_end = par + total;
    const uint32_t q_lo = par ? 2u : 0u, q_hi = q_end & ~1u;
    const u64 g0 = wbase - par;
    if (lane < 4) {
      if (q_hi > q_lo) bulk_s2g(dst[lane] + g0 + q_lo, sb + lane * STG_ROWS + q_lo, (q_hi - q_lo) * 8);
      bulk_commit();
      if (par && total) dst[lane][g0 + 1] = sb[lane * STG_ROWS + 1];
      if ((q_end & 1u) && q_end - 1 >= q_lo && total) dst[lane][g0 + q_end - 1] = sb[lane * STG_ROWS + q_end - 1];
    }
  }
  if (lane < 4) bulk_wait_read<0>();
}

// P6: vec2 warp kernel + REGISTER prefetch of the next tile's keys/payloads (software pipelining)
template <int G, int MINB, int MODE = 0>
__global__ void __launch_bounds__(256, MINB) k_probe_vec2_pf(const int64_t* __restrict__ pkey, const u64* __restrict__ ppay, int64_t n, TableView t, Out4 o,
                                                            u64* __restrict__ cursor) {
  constexpr int R = 2 * G;
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * 8, warp_id = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int64_t ntiles = n / (64 * G);
  ulonglong2 kn[G], pn[G];
  int64_t tile = warp_id;
  if (tile < ntiles) {
#pragma unroll
    for (int g = 0; g < G; g++) {
      kn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + tile * 64 * G + g * 64) + lane);
      pn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(ppay + tile * 64 * G + g * 64) + lane);
    }
  }
  for (; tile < ntiles; tile += warps_total) {
    int64_t k[R]; u64 pv[R], meta[R]; unsigned bal[R];
#pragma unroll
    for (int g = 0; g < G; g++) { k[2 * g] = (int64_t)kn[g].x; k[2 * g + 1] = (int64_t)kn[g].y; pv[2 * g] = pn[g].x; pv[2 * g + 1] = pn[g].y; }
    const int64_t nt = tile + warps_total;
    if (nt < ntiles) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        kn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + nt * 64 * G + g * 64) + lane);
        pn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(ppay + nt * 64 * G + g * 64) + lane);
      }
    }
    uint32_t total = gather_match<R>(k, t, meta, bal);
    u64 wbase = 0;
    if (MODE == 1) {
      wbase = (u64)tile * 64 * G;                       // diagnostic: no atomic at all (valid only at 100 % match)
      if (lane == 0 && total != 64 * G) cursor[2] = 1;
    } else if (MODE == 2) {
      __shared__ uint32_t s_tot[8];
      __shared__ u64 s_base;
      const int w = threadIdx.x >> 5;
      if (lane == 0) s_tot[w] = total;
      __syncthreads();
      if (threadIdx.x == 0) { uint32_t sum = 0; for (int q = 0; q < 8; q++) sum += s_tot[q]; s_base = sum ? atomicAdd(cursor, (u64)sum) : 0ull; }
      __syncthreads();
      wbase = s_base;
      for (int q = 0; q < w; q++) wbase += s_tot[q];
    } else {
      if (lane == 0 && total) wbase = atomicAdd(cursor, (u64)total);
      wbase = __shfl_sync(0xffffffffu, wbase, 0);
    }
    if (total == 64 * G && (wbase & 1) == 0) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const u64 ob = wbase + g * 64;
        ulonglong2 kk = make_ulonglong2((u64)k[2 * g], (u64)k[2 * g + 1]);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_p + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_b + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_p + ob) + lane, make_ulonglong2(pv[2 * g], pv[2 * g + 1]));
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_b + ob) + lane, make_ulonglong2(meta[2 * g], meta[2 * g + 1]));
      }
    } else {
#pragma unroll
      for (int j = 0; j < R; j++) {
        if ((bal[j] >> lane) & 1u) {
          const u64 q = wbase + __popc(bal[j] & ((1u << lane) - 1));
          __stcs(o.key_p + q, (u64)k[j]); __stcs(o.key_b + q, (u64)k[j]); __stcs(o.pay_p + q, pv[j]); __stcs(o.pay_b + q, meta[j]);
        }
        wbase += __popc(bal[j]);
      }
    }
  }
}

// P14: P6 + software prefetch of the NEXT tile's table sectors into L1 (PF=1) / L2 (PF=2): no destination registers, so the
// gathers of two tiles are in flight per warp
template <int G, int MINB, int PF>
__global__ void __launch_bounds__(256, MINB) k_probe_vec2_tpf(const int64_t* __restrict__ pkey, const u64* __restrict__ ppay, int64_t n, TableView t, Out4 o,
                                                            u64* __restrict__ cursor) {
  constexpr int R = 2 * G;
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * 8, warp_id = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int64_t ntiles = n / (64 * G);
  ulonglong2 kn[G], pn[G];
  int64_t tile = warp_id;
  if (tile < ntiles) {
#pragma unroll
    for (int g = 0; g < G; g++) {
      kn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + tile * 64 * G + g * 64) + lane);
      pn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(ppay + tile * 64 * G + g * 64) + lane);
    }
  }
  for (; tile < ntiles; tile += warps_total) {
    int64_t k[R]; u64 pv[R], meta[R]; unsigned bal[R];
#pragma unroll
    for (int g = 0; g < G; g++) { k[2 * g] = (int64_t)kn[g].x; k[2 * g + 1] = (int64_t)kn[g].y; pv[2 * g] = pn[g].x; pv[2 * g + 1] = pn[g].y; }
    const int64_t nt = tile + warps_total;
    if (nt < ntiles) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        kn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + nt * 64 * G + g * 64) + lane);
        pn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(ppay + nt * 64 * G + g * 64) + lane);
      }
    }
    if (nt < ntiles) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const Slot* a0 = t.slots + home_slot(hash64(kn[g].x), t.nslots, 2);
        const Slot* a1 = t.slots + home_slot(hash64(kn[g].y), t.nslots, 2);
        if (PF == 1) { asm volatile("prefetch.global.L1 [%0];" ::"l"(a0)); asm volatile("prefetch.global.L1 [%0];" ::"l"(a1)); }
        else { asm volatile("prefetch.global.L2 [%0];" ::"l"(a0)); asm volatile("prefetch.global.L2 [%0];" ::"l"(a1)); }
      }
    }
    uint32_t total = gather_match<R>(k, t, meta, bal);
    u64 wbase = 0;
    constexpr int MODE = 0;
    if (MODE == 1) {
      wbase = (u64)tile * 64 * G;                       // diagnostic: no atomic at all (valid only at 100 % match)
      if (lane == 0 && total != 64 * G) cursor[2] = 1;
    } else if (MODE == 2) {
      __shared__ uint32_t s_tot[8];
      __shared__ u64 s_base;
      const int w = threadIdx.x >> 5;
      if (lane == 0) s_tot[w] = total;
      __syncthreads();
      if (threadIdx.x == 0) { uint32_t sum = 0; for (int q = 0; q < 8; q++) sum += s_tot[q]; s_base = sum ? atomicAdd(cursor, (u64)sum) : 0ull; }
      __syncthreads();
      wbase = s_base;
      for (int q = 0; q < w; q++) wbase += s_tot[q];
    } else {
      if (lane == 0 && total) wbase = atomicAdd(cursor, (u64)total);
      wbase = __shfl_sync(0xffffffffu, wbase, 0);
    }
    if (total == 64 * G && (wbase & 1) == 0) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const u64 ob = wbase + g * 64;
        ulonglong2 kk = make_ulonglong2((u64)k[2 * g], (u64)k[2 * g + 1]);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_p + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_b + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_p + ob) + lane, make_ulonglong2(pv[2 * g], pv[2 * g + 1]));
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_b + ob) + lane, make_ulonglong2(meta[2 * g], meta[2 * g + 1]));
      }
    } else {
#pragma unroll
      for (int j = 0; j < R; j++) {
        if ((bal[j] >> lane) & 1u) {
          const u64 q = wbase + __popc(bal[j] & ((1u << lane) - 1));
          __stcs(o.key_p + q, (u64)k[j]); __stcs(o.key_b + q, (u64)k[j]); __stcs(o.pay_p + q, pv[j]); __stcs(o.pay_b + q, meta[j]);
        }
        wbase += __popc(bal[j]);
      }
    }
  }
}

// P8: vec2 warp kernel + cp.async (LDGSTS) prefetch ring in shared memory: every lane copies ITS OWN 16-byte pieces D
// tiles ahead and reads them back itself, so no barrier, fence or register is spent on the data in flight
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, u64 pol) {
  asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int G, int D, int MINB>
__global__ void __launch_bounds__(256, MINB) k_probe_vec2_cpa(const int64_t* __restrict__ pkey, const u64* __restrict__ ppay, int64_t n, TableView t, Out4 o,
                                                             u64* __restrict__ cursor) {
  constexpr int R = 2 * G;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // [warp][D][2 cols][G][32 lanes] x 16 bytes
  ulonglong2* ring = reinterpret_cast<ulonglong2*>(smem_raw) + (size_t)warp * D * 2 * G * 32;
  const int64_t warps_total = (int64_t)gridDim.x * 8, warp_id = (int64_t)blockIdx.x * 8 + warp;
  const int64_t ntiles = n / (64 * G);
  const u64 pol = l2_policy_evict_first();
  auto issue = [&](int64_t it) {
    const int64_t tile = warp_id + it * warps_total;
    if (tile < ntiles) {
      ulonglong2* st = ring + (size_t)(it % D) * 2 * G * 32;
#pragma unroll
      for (int g = 0; g < G; g++) {
        cp_async16(st + g * 32 + lane, reinterpret_cast<const ulonglong2*>(pkey + tile * 64 * G + g * 64) + lane, pol);
        cp_async16(st + (G + g) * 32 + lane, reinterpret_cast<const ulonglong2*>(ppay + tile * 64 * G + g * 64) + lane, pol);
      }
    }
    cp_async_commit();
  };
  for (int it = 0; it < D; it++) issue(it);
  for (int64_t it = 0;; it++) {
    const int64_t tile = warp_id + it * warps_total;
    if (tile >= ntiles) break;
    cp_async_wait<D - 1>();
    const ulonglong2* st = ring + (size_t)(it % D) * 2 * G * 32;
    int64_t k[R]; u64 pv[R], meta[R]; unsigned bal[R];
#pragma unroll
    for (int g = 0; g < G; g++) {
      ulonglong2 kk = st[g * 32 + lane], pp = st[(G + g) * 32 + lane];
      k[2 * g] = (int64_t)kk.x; k[2 * g + 1] = (int64_t)kk.y; pv[2 * g] = pp.x; pv[2 * g + 1] = pp.y;
    }
    issue(it + D);
    uint32_t total = gather_match<R>(k, t, meta, bal);
    u64 wbase = 0;
    if (lane == 0 && total) wbase = atomicAdd(cursor, (u64)total);
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (total == 64 * G && (wbase & 1) == 0) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const u64 ob = wbase + g * 64;
        ulonglong2 kk = make_ulonglong2((u64)k[2 * g], (u64)k[2 * g + 1]);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_p + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_b + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_p + ob) + lane, make_ulonglong2(pv[2 * g], pv[2 * g + 1]));
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_b + ob) + lane, make_ulonglong2(meta[2 * g], meta[2 * g + 1]));
      }
    } else {
#pragma unroll
      for (int j = 0; j < R; j++) {
        if ((bal[j] >> lane) & 1u) {
          const u64 q = wbase + __popc(bal[j] & ((1u << lane) - 1));
          __stcs(o.key_p + q, (u64)k[j]); __stcs(o.key_b + q, (u64)k[j]); __stcs(o.pay_p + q, pv[j]); __stcs(o.pay_b + q, meta[j]);
        }
        wbase += __popc(bal[j]);
      }
    }
  }
  cp_async_wait<0>();
}

// P12: single-slot (16-byte) gathers, R = 2G rows per lane, keys/payloads PARKED in the cp.async ring (re-read from shared
// memory after the gathers return) so that registers hold little besides the gathers in flight
__device__ __forceinline__ ulonglong2 lds128(const ulonglong2* p) {
  ulonglong2 v;
  asm volatile("ld.shared.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "r"(smem_u32(p)));
  return v;
}
template <int G, int D, int MINB>
__global__ void __launch_bounds__(256, MINB) k_probe_v3(const int64_t* __restrict__ pkey, const u64* __restrict__ ppay, int64_t n, TableView t, Out4 o,
                                                       u64* __restrict__ cursor) {
  constexpr int R = 2 * G;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  ulonglong2* ring = reinterpret_cast<ulonglong2*>(smem_raw) + (size_t)warp * D * 2 * G * 32;
  const int64_t warps_total = (int64_t)gridDim.x * 8, warp_id = (int64_t)blockIdx.x * 8 + warp;
  const int64_t ntiles = n / (64 * G);
  const u64 pol = l2_policy_evict_first();
  auto issue = [&](int64_t it) {
    const int64_t tile = warp_id + it * warps_total;
    if (tile < ntiles) {
      ulonglong2* st = ring + (size_t)(it % D) * 2 * G * 32;
#pragma unroll
      for (int g = 0; g < G; g++) {
        cp_async16(st + g * 32 + lane, reinterpret_cast<const ulonglong2*>(pkey + tile * 64 * G + g * 64) + lane, pol);
        cp_async16(st + (G + g) * 32 + lane, reinterpret_cast<const ulonglong2*>(ppay + tile * 64 * G + g * 64) + lane, pol);
      }
    }
    cp_async_commit();
  };
  for (int it = 0; it < D - 1; it++) issue(it);
  for (int64_t it = 0;; it++) {
    const int64_t tile = warp_id + it * warps_total;
    if (tile >= ntiles) break;
    issue(it + D - 1);                      // stage (it-1)%D was fully consumed in the previous iteration
    cp_async_wait<D - 1>();
    const ulonglong2* st = ring + (size_t)(it % D) * 2 * G * 32;
    Slot v[R];
    u64 sl[R];
#pragma unroll
    for (int g = 0; g < G; g++) {
      const ulonglong2 kk = lds128(st + g * 32 + lane);
      sl[2 * g] = home_slot(hash64(kk.x), t.nslots, 1); sl[2 * g + 1] = home_slot(hash64(kk.y), t.nslots, 1);
      v[2 * g] = load_slot(t.slots + sl[2 * g]); v[2 * g + 1] = load_slot(t.slots + sl[2 * g + 1]);
    }
    unsigned bal[R];
    uint32_t total = 0;
#pragma unroll
    for (int g = 0; g < G; g++) {
      const ulonglong2 kk = lds128(st + g * 32 + lane);
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int j = 2 * g + h;
        const int64_t k = (int64_t)(h ? kk.y : kk.x);
        while (v[j].key != k && v[j].key != kEmptyKey) { if (++sl[j] == t.nslots) sl[j] = 0; v[j] = load_slot(t.slots + sl[j]); }
        bal[j] = __ballot_sync(0xffffffffu, v[j].key == k);
        total += __popc(bal[j]);
      }
    }
    u64 wbase = 0;
    if (lane == 0 && total) wbase = atomicAdd(cursor, (u64)total);
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (total == 64 * G && (wbase & 1) == 0) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const u64 ob = wbase + g * 64;
        const ulonglong2 kk = lds128(st + g * 32 + lane), pp = lds128(st + (G + g) * 32 + lane);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_p + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_b + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_p + ob) + lane, pp);
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_b + ob) + lane, make_ulonglong2(v[2 * g].meta, v[2 * g + 1].meta));
      }
    } else {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const ulonglong2 kk = lds128(st + g * 32 + lane), pp = lds128(st + (G + g) * 32 + lane);
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int j = 2 * g + h;
          if ((bal[j] >> lane) & 1u) {
            const u64 q = wbase + __popc(bal[j] & ((1u << lane) - 1));
            const u64 k = h ? kk.y : kk.x;
            __stcs(o.key_p + q, k); __stcs(o.key_b + q, k); __stcs(o.pay_p + q, h ? pp.y : pp.x); __stcs(o.pay_b + q, v[j].meta);
          }
          wbase += __popc(bal[j]);
        }
      }
    }
  }
  cp_async_wait<0>();
}

// P13: P6 + explicit L2 policies: table gathers evict_last (POL & 1), stores with an evict_first cache hint instead of .cs (POL & 2),
// streamed inputs with evict_first hint (POL & 4)
__device__ __forceinline__ void load_pair_pol(const Slot* p, Slot& a, Slot& b, u64 pol) {
  u64 x0, x1, x2, x3;
  asm volatile("ld.global.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;" : "=l"(x0), "=l"(x1) : "l"(p), "l"(pol));
  asm volatile("ld.global.L2::cache_hint.v2.u64 {%0, %1}, [%2+16], %3;" : "=l"(x2), "=l"(x3) : "l"(p), "l"(pol));
  a.key = (int64_t)x0; a.meta = x1; b.key = (int64_t)x2; b.meta = x3;
}
__device__ __forceinline__ void st16_pol(void* p, ulonglong2 v, u64 pol) {
  asm volatile("st.global.L2::cache_hint.v2.u64 [%0], {%1, %2}, %3;" ::"l"(p), "l"(v.x), "l"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ ulonglong2 ld16_pol(const void* p, u64 pol) {
  ulonglong2 v;
  asm volatile("ld.global.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;" : "=l"(v.x), "=l"(v.y) : "l"(p), "l"(pol));
  return v;
}
template <int G, int MINB, int POL>
__global__ void __launch_bounds__(256, MINB) k_probe_pol(const int64_t* __restrict__ pkey, const u64* __restrict__ ppay, int64_t n, TableView t, Out4 o,
                                                        u64* __restrict__ cursor) {
  constexpr int R = 2 * G;
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * 8, warp_id = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int64_t ntiles = n / (64 * G);
  const u64 pol_last = l2_policy_evict_last(), pol_first = l2_policy_evict_first();
  ulonglong2 kn[G], pn[G];
  int64_t tile = warp_id;
  auto ld_in = [&](const void* p) { return (POL & 4) ? ld16_pol(p, pol_first) : __ldcs(reinterpret_cast<const ulonglong2*>(p)); };
  if (tile < ntiles) {
#pragma unroll
    for (int g = 0; g < G; g++) {
      kn[g] = ld_in(reinterpret_cast<const ulonglong2*>(pkey + tile * 64 * G + g * 64) + lane);
      pn[g] = ld_in(reinterpret_cast<const ulonglong2*>(ppay + tile * 64 * G + g * 64) + lane);
    }
  }
  for (; tile < ntiles; tile += warps_total) {
    int64_t k[R]; u64 pv[R], meta[R]; unsigned bal[R];
#pragma unroll
    for (int g = 0; g < G; g++) { k[2 * g] = (int64_t)kn[g].x; k[2 * g + 1] = (int64_t)kn[g].y; pv[2 * g] = pn[g].x; pv[2 * g + 1] = pn[g].y; }
    const int64_t nt = tile + warps_total;
    if (nt < ntiles) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        kn[g] = ld_in(reinterpret_cast<const ulonglong2*>(pkey + nt * 64 * G + g * 64) + lane);
        pn[g] = ld_in(reinterpret_cast<const ulonglong2*>(ppay + nt * 64 * G + g * 64) + lane);
      }
    }
    Slot v[R], w[R];
#pragma unroll
    for (int j = 0; j < R; j++) {
      const u64 sl = home_slot(hash64((uint64_t)k[j]), t.nslots, 2);
      if (POL & 1) load_pair_pol(t.slots + sl, v[j], w[j], pol_last); else load_pair(t.slots + sl, v[j], w[j]);
    }
    uint32_t total = 0;
#pragma unroll
    for (int j = 0; j < R; j++) {
      bool m;
      if (v[j].key == k[j]) { m = true; meta[j] = v[j].meta; }
      else if (w[j].key == k[j]) { m = true; meta[j] = w[j].meta; }
      else if (v[j].key == kEmptyKey || w[j].key == kEmptyKey) { m = false; meta[j] = 0; }
      else {
        u64 sl = home_slot(hash64((uint64_t)k[j]), t.nslots, 2) + 2;
        if (sl >= t.nslots) sl = 0;
        Slot x = load_slot(t.slots + sl);
        while (x.key != k[j] && x.key != kEmptyKey) { if (++sl == t.nslots) sl = 0; x = load_slot(t.slots + sl); }
        m = x.key == k[j]; meta[j] = x.meta;
      }
      bal[j] = __ballot_sync(0xffffffffu, m);
      total += __popc(bal[j]);
    }
    u64 wbase = 0;
    if (lane == 0 && total) wbase = atomicAdd(cursor, (u64)total);
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (total == 64 * G && (wbase & 1) == 0) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const u64 ob = wbase + g * 64;
        ulonglong2 kk = make_ulonglong2((u64)k[2 * g], (u64)k[2 * g + 1]);
        ulonglong2 pp = make_ulonglong2(pv[2 * g], pv[2 * g + 1]), mm = make_ulonglong2(meta[2 * g], meta[2 * g + 1]);
        if (POL & 2) {
          st16_pol(reinterpret_cast<ulonglong2*>(o.key_p + ob) + lane, kk, pol_first); st16_pol(reinterpret_cast<ulonglong2*>(o.key_b + ob) + lane, kk, pol_first);
          st16_pol(reinterpret_cast<ulonglong2*>(o.pay_p + ob) + lane, pp, pol_first); st16_pol(reinterpret_cast<ulonglong2*>(o.pay_b + ob) + lane, mm, pol_first);
        } else {
          __stcs(reinterpret_cast<ulonglong2*>(o.key_p + ob) + lane, kk); __stcs(reinterpret_cast<ulonglong2*>(o.key_b + ob) + lane, kk);
          __stcs(reinterpret_cast<ulonglong2*>(o.pay_p + ob) + lane, pp); __stcs(reinterpret_cast<ulonglong2*>(o.pay_b + ob) + lane, mm);
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < R; j++) {
        if ((bal[j] >> lane) & 1u) {
          const u64 q = wbase + __popc(bal[j] & ((1u << lane) - 1));
          __stcs(o.key_p + q, (u64)k[j]); __stcs(o.key_b + q, (u64)k[j]); __stcs(o.pay_p + q, pv[j]); __stcs(o.pay_b + q, meta[j]);
        }
        wbase += __popc(bal[j]);
      }
    }
  }
}

// ================================================================== pipeline lab: count-free scatter with bulk stores + segment probe
#include "partition_kernels.cuh"
template <bool HIGH, int NC, int ITEMS, int RANKMODE>
__global__ void __launch_bounds__(PT_BLOCK) k_scatter_bulk(int64_t ntiles, PartDst d, u64* __restrict__ cursors, long long capacity, u64* __restrict__ overflow) {
  constexpr int STAGES = 2, TILE = PT_BLOCK * ITEMS, SROWS = TILE + 2 * TG_MAX_PARTS;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  u64* ring = reinterpret_cast<u64*>(smem_raw);                        // [STAGES][NC][TILE]
  u64* stage = ring + (size_t)STAGES * NC * TILE;                   // [NC][SROWS]
  uint64_t* full = reinterpret_cast<uint64_t*>(stage + (size_t)NC * SROWS);
  __shared__ uint32_t s_cnt[TG_MAX_PARTS], s_off[TG_MAX_PARTS], s_len[TG_MAX_PARTS];
  __shared__ u64 s_gbase[TG_MAX_PARTS];
  const int tid = threadIdx.x, lane = tid & 31;
  const uint32_t P = (uint32_t)d.nparts;
  const u64 pol = l2_policy_evict_first();
  if (tid == 0) { for (int s = 0; s < STAGES; s++) mbar_init(&full[s], 1); mbar_fence_init(); }
  __syncthreads();
  auto issue = [&](int64_t it) {
    int64_t tile = (int64_t)blockIdx.x + it * gridDim.x;
    if (tile >= ntiles) return;
    int s = (int)(it % STAGES);
    mbar_arrive_expect_tx(&full[s], (uint32_t)(NC * TILE * 8));
#pragma unroll
    for (int c = 0; c < NC; c++)
      bulk_g2s(ring + ((size_t)s * NC + c) * TILE, reinterpret_cast<const u64*>(d.src[c]) + tile * TILE, TILE * 8, &full[s], pol);
  };
  if (tid == 0) for (int it = 0; it < STAGES; it++) issue(it);
  for (int64_t it = 0;; it++) {
    const int64_t tile = (int64_t)blockIdx.x + it * gridDim.x;
    if (tile >= ntiles) break;
    const int s = (int)(it % STAGES);
    if (tid < TG_MAX_PARTS) s_cnt[tid] = 0;
    mbar_wait(&full[s], (uint32_t)((it / STAGES) & 1));
    __syncthreads();
    const u64* in = ring + (size_t)s * NC * TILE;
    uint32_t pr[ITEMS];   // part << 16 | rank inside (tile, part)
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      uint64_t h = hash64(in[j * PT_BLOCK + tid]);
      uint32_t p = HIGH ? mulhi32((uint32_t)(h >> 32), P) : part_of(h, P);
      if (RANKMODE == 1) {
        pr[j] = (p << 16) | atomicAdd(&s_cnt[p], 1u);
      } else {
        unsigned peers = __match_any_sync(0xffffffffu, p);
        int leader = __ffs(peers) - 1;
        uint32_t wbase = 0;
        if (lane == leader) wbase = atomicAdd(&s_cnt[p], (uint32_t)__popc(peers));
        wbase = __shfl_sync(peers, wbase, leader);
        pr[j] = (p << 16) | (wbase + __popc(peers & ((1u << lane) - 1)));
      }
    }
    __syncthreads();
    if (tid < 32) {
      // one global reservation per destination; the run of destination p is parked in the staging buffer at an offset
      // whose parity equals the parity of its global row, so that the 16-byte aligned middle can go out as ONE bulk store
      uint32_t c = tid < (int)P ? s_cnt[tid] : 0;
      u64 g = 0; uint32_t len = c;
      if (tid < (int)P) {
        u64 old = c ? atomicAdd(&cursors[tid], (u64)c) : 0ull;
        if (capacity > 0) {
          u64 avail = old < (u64)capacity ? (u64)capacity - old : 0ull;
          if ((u64)c > avail) { len = (uint32_t)avail; *overflow = 1ull; }
        }
        g = old + (u64)d.dst_base[tid];
      }
      uint32_t w = tid < (int)P ? (((uint32_t)(g & 1) + c + 1) & ~1u) : 0, incl = w;
      for (int o = 1; o < 32; o <<= 1) { uint32_t u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
      if (tid < (int)P) { s_off[tid] = incl - w + (uint32_t)(g & 1); s_gbase[tid] = g; s_len[tid] = len; }
    }
    if (tid < (int)P * NC) bulk_wait_read<0>();     // the previous tile's bulk stores have read the staging buffer
    __syncthreads();
#pragma unroll
    for (int c = 0; c < NC; c++) {
#pragma unroll
      for (int j = 0; j < ITEMS; j++) stage[(size_t)c * SROWS + s_off[pr[j] >> 16] + (pr[j] & 0xffffu)] = in[(size_t)c * TILE + j * PT_BLOCK + tid];
    }
    fence_async_smem();
    __syncthreads();
    if (tid == 0) issue(it + STAGES);
    if (tid < (int)P * NC) {
      const uint32_t p = tid / NC, c = tid % NC;
      const u64 g = s_gbase[p];
      const uint32_t len = s_len[p], so = s_off[p];
      u64* dst = reinterpret_cast<u64*>(d.dst[p][c]);
      const u64* src = stage + (size_t)c * SROWS;
      const uint32_t head = (uint32_t)(g & 1) & (len > 0 ? 1u : 0u);
      const uint32_t mid = (len - head) & ~1u;
      if (mid) bulk_s2g(dst + g + head, src + so + head, mid * 8);
      bulk_commit();
      if (head) dst[g] = src[so];
      if ((len - head) & 1u) dst[g + len - 1] = src[so + len - 1];
    }
  }
  if (tid < (int)P * NC) bulk_wait_read<0>();
}

// probe over capacity segments: segment p = rows [p*C, p*C + min(cursors[p], C)); C is a multiple of 128
template <int MINB>
__global__ void __launch_bounds__(256, MINB) k_probe_seg(const int64_t* __restrict__ pkey, const u64* __restrict__ ppay, const u64* __restrict__ seg_cnt,
                                                        int P, long long C, const u64* __restrict__ overflow, TableView t, Out4 o, u64* __restrict__ cursor) {
  constexpr int G = 2, R = 4;
  __shared__ long long s_tile0[TG_MAX_PARTS + 1];
  __shared__ long long s_cntp[TG_MAX_PARTS];
  if (*overflow) return;
  if (threadIdx.x == 0) {
    long long run = 0;
    for (int p = 0; p < P; p++) { long long c = (long long)seg_cnt[p]; if (c > C) c = C; s_cntp[p] = c; s_tile0[p] = run; run += (c + 127) / 128; }
    s_tile0[P] = run;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warps_total = (long long)gridDim.x * 8, warp_id = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long ntiles = s_tile0[P];
  int p = 0;
  auto locate = [&](long long g, int& pp, long long& row0, long long& left) {
    while (g >= s_tile0[pp + 1]) pp++;
    const long long lt = g - s_tile0[pp];
    row0 = (long long)pp * C + lt * 128; left = s_cntp[pp] - lt * 128;
  };
  ulonglong2 kn[G], pn[G];
  long long tile = warp_id, row0 = 0, left = 0, nrow0 = 0, nleft = 0;
  int pnx = 0;
  if (tile < ntiles) {
    locate(tile, pnx, nrow0, nleft);
#pragma unroll
    for (int g = 0; g < G; g++) {
      kn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + nrow0 + g * 64) + lane);
      pn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(ppay + nrow0 + g * 64) + lane);
    }
  }
  for (; tile < ntiles; tile += warps_total) {
    int64_t k[R]; u64 pv[R], meta[R]; unsigned bal[R];
    row0 = nrow0; left = nleft; p = pnx;
#pragma unroll
    for (int g = 0; g < G; g++) { k[2 * g] = (int64_t)kn[g].x; k[2 * g + 1] = (int64_t)kn[g].y; pv[2 * g] = pn[g].x; pv[2 * g + 1] = pn[g].y; }
    const long long nt = tile + warps_total;
    if (nt < ntiles) {
      locate(nt, pnx, nrow0, nleft);
#pragma unroll
      for (int g = 0; g < G; g++) {
        kn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + nrow0 + g * 64) + lane);
        pn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(ppay + nrow0 + g * 64) + lane);
      }
    }
    // rows of this lane inside the tile: g*64 + 2*lane + {0,1}
    Slot v[R], w[R];
#pragma unroll
    for (int j = 0; j < R; j++) { const u64 sl = home_slot(hash64((uint64_t)k[j]), t.nslots, 2); load_pair(t.slots + sl, v[j], w[j]); }
    uint32_t total = 0;
    const bool full_tile = left >= 128;
#pragma unroll
    for (int j = 0; j < R; j++) {
      const bool valid = full_tile || (long long)((j >> 1) * 64 + 2 * lane + (j & 1)) < left;
      bool m;
      if (v[j].key == k[j]) { m = true; meta[j] = v[j].meta; }
      else if (w[j].key == k[j]) { m = true; meta[j] = w[j].meta; }
      else if (v[j].key == kEmptyKey || w[j].key == kEmptyKey) { m = false; meta[j] = 0; }
      else {
        m = false; meta[j] = 0;
        if (valid) {
          u64 sl = home_slot(hash64((uint64_t)k[j]), t.nslots, 2) + 2;
          if (sl >= t.nslots) sl = 0;
          Slot x = load_slot(t.slots + sl);
          while (x.key != k[j] && x.key != kEmptyKey) { if (++sl == t.nslots) sl = 0; x = load_slot(t.slots + sl); }
          m = x.key == k[j]; meta[j] = x.meta;
        }
      }
      bal[j] = __ballot_sync(0xffffffffu, m && valid);
      total += __popc(bal[j]);
    }
    u64 wbase = 0;
    if (lane == 0 && total) wbase = atomicAdd(cursor, (u64)total);
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (total == 128 && (wbase & 1) == 0) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const u64 ob = wbase + g * 64;
        ulonglong2 kk = make_ulonglong2((u64)k[2 * g], (u64)k[2 * g + 1]);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_p + ob) + lane, kk); __stcs(reinterpret_cast<ulonglong2*>(o.key_b + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_p + ob) + lane, make_ulonglong2(pv[2 * g], pv[2 * g + 1]));
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_b + ob) + lane, make_ulonglong2(meta[2 * g], meta[2 * g + 1]));
      }
    } else {
      // output order inside the tile = row order: rows are interleaved (2 adjacent rows per lane), rank accordingly
#pragma unroll
      for (int g = 0; g < G; g++) {
        const unsigned b0 = bal[2 * g], b1 = bal[2 * g + 1];
        const unsigned below = (1u << lane) - 1;
        const uint32_t r0 = __popc(b0 & below) + __popc(b1 & below);
        if ((b0 >> lane) & 1u) { const u64 q = wbase + r0; __stcs(o.key_p + q, (u64)k[2 * g]); __stcs(o.key_b + q, (u64)k[2 * g]); __stcs(o.pay_p + q, pv[2 * g]); __stcs(o.pay_b + q, meta[2 * g]); }
        if ((b1 >> lane) & 1u) { const u64 q = wbase + r0 + ((b0 >> lane) & 1u); __stcs(o.key_p + q, (u64)k[2 * g + 1]); __stcs(o.key_b + q, (u64)k[2 * g + 1]); __stcs(o.pay_p + q, pv[2 * g + 1]); __stcs(o.pay_b + q, meta[2 * g + 1]); }
        wbase += __popc(b0) + __popc(b1);
      }
    }
  }
}

// dynamic-ticket variant (tiles handed out by an atomic counter, two tickets ahead): probe over capacity segments: segment p = rows [p*C, p*C + min(cursors[p], C)); C is a multiple of 128
template <int MINB>
__global__ void __launch_bounds__(256, MINB) k_probe_seg_dyn(const int64_t* __restrict__ pkey, const u64* __restrict__ ppay, const u64* __restrict__ seg_cnt,
                                                        int P, long long C, const u64* __restrict__ overflow, TableView t, Out4 o, u64* __restrict__ cursor) {
  constexpr int G = 2, R = 4;
  __shared__ long long s_tile0[TG_MAX_PARTS + 1];
  __shared__ long long s_cntp[TG_MAX_PARTS];
  if (*overflow) return;
  if (threadIdx.x == 0) {
    long long run = 0;
    for (int p = 0; p < P; p++) { long long c = (long long)seg_cnt[p]; if (c > C) c = C; s_cntp[p] = c; s_tile0[p] = run; run += (c + 127) / 128; }
    s_tile0[P] = run;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warps_total = (long long)gridDim.x * 8, warp_id = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long ntiles = s_tile0[P];
  int p = 0;
  auto locate = [&](long long g, int& pp, long long& row0, long long& left) {
    while (g >= s_tile0[pp + 1]) pp++;
    const long long lt = g - s_tile0[pp];
    row0 = (long long)pp * C + lt * 128; left = s_cntp[pp] - lt * 128;
  };
  ulonglong2 kn[G], pn[G];
  u64* ticket = cursor + 1;
  auto take = [&]() { unsigned long long tk = 0; if (lane == 0) tk = atomicAdd(ticket, 1ull); return (long long)__shfl_sync(0xffffffffu, tk, 0); };
  long long tile = take(), tile1 = take(), row0 = 0, left = 0, nrow0 = 0, nleft = 0;
  int pnx = 0;
  (void)warp_id; (void)warps_total;
  if (tile < ntiles) {
    locate(tile, pnx, nrow0, nleft);
#pragma unroll
    for (int g = 0; g < G; g++) {
      kn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + nrow0 + g * 64) + lane);
      pn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(ppay + nrow0 + g * 64) + lane);
    }
  }
  while (tile < ntiles) {
    int64_t k[R]; u64 pv[R], meta[R]; unsigned bal[R];
    row0 = nrow0; left = nleft; p = pnx;
    const long long nt = tile1;
    unsigned long long tk2 = 0;
    if (lane == 0) tk2 = atomicAdd(ticket, 1ull);      // ticket for the tile after next; read at the end of this iteration
#pragma unroll
    for (int g = 0; g < G; g++) { k[2 * g] = (int64_t)kn[g].x; k[2 * g + 1] = (int64_t)kn[g].y; pv[2 * g] = pn[g].x; pv[2 * g + 1] = pn[g].y; }
    if (nt < ntiles) {
      locate(nt, pnx, nrow0, nleft);
#pragma unroll
      for (int g = 0; g < G; g++) {
        kn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + nrow0 + g * 64) + lane);
        pn[g] = __ldcs(reinterpret_cast<const ulonglong2*>(ppay + nrow0 + g * 64) + lane);
      }
    }
    // rows of this lane inside the tile: g*64 + 2*lane + {0,1}
    Slot v[R], w[R];
#pragma unroll
    for (int j = 0; j < R; j++) { const u64 sl = home_slot(hash64((uint64_t)k[j]), t.nslots, 2); load_pair(t.slots + sl, v[j], w[j]); }
    uint32_t total = 0;
    const bool full_tile = left >= 128;
#pragma unroll
    for (int j = 0; j < R; j++) {
      const bool valid = full_tile || (long long)((j >> 1) * 64 + 2 * lane + (j & 1)) < left;
      bool m;
      if (v[j].key == k[j]) { m = true; meta[j] = v[j].meta; }
      else if (w[j].key == k[j]) { m = true; meta[j] = w[j].meta; }
      else if (v[j].key == kEmptyKey || w[j].key == kEmptyKey) { m = false; meta[j] = 0; }
      else {
        m = false; meta[j] = 0;
        if (valid) {
          u64 sl = home_slot(hash64((uint64_t)k[j]), t.nslots, 2) + 2;
          if (sl >= t.nslots) sl = 0;
          Slot x = load_slot(t.slots + sl);
          while (x.key != k[j] && x.key != kEmptyKey) { if (++sl == t.nslots) sl = 0; x = load_slot(t.slots + sl); }
          m = x.key == k[j]; meta[j] = x.meta;
        }
      }
      bal[j] = __ballot_sync(0xffffffffu, m && valid);
      total += __popc(bal[j]);
    }
    u64 wbase = 0;
    if (lane == 0 && total) wbase = atomicAdd(cursor, (u64)total);
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (total == 128 && (wbase & 1) == 0) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const u64 ob = wbase + g * 64;
        ulonglong2 kk = make_ulonglong2((u64)k[2 * g], (u64)k[2 * g + 1]);
        __stcs(reinterpret_cast<ulonglong2*>(o.key_p + ob) + lane, kk); __stcs(reinterpret_cast<ulonglong2*>(o.key_b + ob) + lane, kk);
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_p + ob) + lane, make_ulonglong2(pv[2 * g], pv[2 * g + 1]));
        __stcs(reinterpret_cast<ulonglong2*>(o.pay_b + ob) + lane, make_ulonglong2(meta[2 * g], meta[2 * g + 1]));
      }
    } else {
      // output order inside the tile = row order: rows are interleaved (2 adjacent rows per lane), rank accordingly
#pragma unroll
      for (int g = 0; g < G; g++) {
        const unsigned b0 = bal[2 * g], b1 = bal[2 * g + 1];
        const unsigned below = (1u << lane) - 1;
        const uint32_t r0 = __popc(b0 & below) + __popc(b1 & below);
        if ((b0 >> lane) & 1u) { const u64 q = wbase + r0; __stcs(o.key_p + q, (u64)k[2 * g]); __stcs(o.key_b + q, (u64)k[2 * g]); __stcs(o.pay_p + q, pv[2 * g]); __stcs(o.pay_b + q, meta[2 * g]); }
        if ((b1 >> lane) & 1u) { const u64 q = wbase + r0 + ((b0 >> lane) & 1u); __stcs(o.key_p + q, (u64)k[2 * g + 1]); __stcs(o.key_b + q, (u64)k[2 * g + 1]); __stcs(o.pay_p + q, pv[2 * g + 1]); __stcs(o.pay_b + q, meta[2 * g + 1]); }
        wbase += __popc(b0) + __popc(b1);
      }
    }
    tile = nt;
    tile1 = (long long)__shfl_sync(0xffffffffu, tk2, 0);
  }
}


// ------------------------------------------------------------------ harness
struct Timer {
  cudaEvent_t a, b;
  Timer() { CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b)); }
  bool once = false;
  template <typename F> float run(F f, int reps = 5) {
    f(); CK(cudaDeviceSynchronize()); CK(cudaGetLastError());
    if (once) return 0.f;
    CK(cudaEventRecord(a));
    for (int i = 0; i < reps; i++) f();
    CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b));
    return ms / reps;
  }
};

int main(int argc, char** argv) {
  const int64_t n = 100000000 / 1024 * 1024, nb = 10000000;
  const double load = argc > 1 ? atof(argv[1]) : 0.4;
  const uint32_t P = argc > 2 ? atoi(argv[2]) : 12;
  const bool all = argc > 3 && std::string(argv[3]) == "all";
  int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  u64 nslots = ((u64)(nb / load) + 32) & ~1ull;
  printf("n=%lld nb=%lld nslots=%llu (%.0f MB) P=%u slice=%.1f MB\n", (long long)n, (long long)nb, nslots, nslots * 16 / 1048576.0, P, nslots * 16 / 1048576.0 / P);
  int64_t *bk, *pk, *pk_s; u64 *bp, *pv, *pv_s, *o[4], *cursor, *acc; Slot* slots; uint8_t* part; uint32_t* idx;
  CK(cudaMalloc(&bk, nb * 8)); CK(cudaMalloc(&bp, nb * 8));
  CK(cudaMalloc(&pk, n * 8 + 64)); CK(cudaMalloc(&pv, n * 8 + 64)); CK(cudaMalloc(&pk_s, n * 8 + 64)); CK(cudaMalloc(&pv_s, n * 8 + 64));
  for (int c = 0; c < 4; c++) CK(cudaMalloc(&o[c], n * 8 + 64));
  CK(cudaMalloc(&cursor, 64)); CK(cudaMalloc(&acc, 64)); CK(cudaMalloc(&slots, (nslots + 1) * 16));
  CK(cudaMalloc(&part, n)); CK(cudaMalloc(&idx, n * 4));
  k_gen_build<<<(nb + 255) / 256, 256>>>(bk, bp, nb);
  k_gen_probe<<<(n + 255) / 256, 256>>>(pk, pv, n, nb, 1234);
  k_lab_init<<<(nslots + 1 + 255) / 256, 256>>>(slots, nslots + 1);
  k_lab_insert<<<(nb + 255) / 256, 256>>>(bk, bp, nb, slots, nslots);
  Slot* slots0; CK(cudaMalloc(&slots0, (nslots + 1) * 16));
  k_lab_init<<<(nslots + 1 + 255) / 256, 256>>>(slots0, nslots + 1);
  k_lab_insert<<<(nb + 255) / 256, 256>>>(bk, bp, nb, slots0, nslots, 0);
  k_part_of<<<(n + 255) / 256, 256>>>(pk, n, P, part);
  thrust::sequence(thrust::device, idx, idx + n);
  thrust::stable_sort_by_key(thrust::device, part, part + n, idx);
  k_gather2<<<(n + 255) / 256, 256>>>(pk, pv, idx, n, pk_s, pv_s);
  CK(cudaDeviceSynchronize());
  // expected checksums
  u64 exp_s2 = (u64)n * (u64)(n - 1) / 2;
  TableView tv{slots, nslots, nullptr, 0, -1, TABLE_U1, 1};
  TableView tv0{slots0, nslots, nullptr, 0, -1, TABLE_U1, 0};
  Out4 out{o[0], o[1], o[2], o[3]};
  Timer T;
  T.once = argc > 3 && std::string(argv[3]) == "ncu";
  u64 exp_s3 = 0; bool have_s3 = false;
  auto verify = [&](const char* name) {
    u64 got = 0; CK(cudaMemcpy(&got, cursor, 8, cudaMemcpyDeviceToHost));
    CK(cudaMemset(acc, 0, 64));
    k_check<<<sms * 8, 256>>>(o[0], o[1], o[2], o[3], n, acc);
    u64 h[3]; CK(cudaMemcpy(h, acc, 24, cudaMemcpyDeviceToHost));
    if (!have_s3) { exp_s3 = h[2]; have_s3 = true; }
    bool ok = got == (u64)n && h[0] == 0 && h[1] == exp_s2 && h[2] == exp_s3;
    printf("    verify %-28s rows=%llu bad=%llu s2 %s s3 %s => %s\n", name, got, h[0], h[1] == exp_s2 ? "ok" : "BAD", h[2] == exp_s3 ? "ok" : "BAD", ok ? "OK" : "FAIL");
  };
  auto report = [&](const char* name, float ms) { printf("%-44s %.3f ms  %.1f G rows/s  %.2f TB/s(64B/row)\n", name, ms, n / ms / 1e6, n * 64.0 / ms / 1e9); fflush(stdout); };

  // ---- S: streaming ceilings
  if (all) for (int cps : {4, 8, 16}) {
    char nm[128];
    snprintf(nm, sizeof nm, "S scalar R=4 cs ctas/sm=%d", cps);
    report(nm, T.run([&] { k_stream_scalar<4, true><<<sms * cps, 256>>>((u64*)pk, pv, n, o[0], o[1], o[2], o[3]); }));
    snprintf(nm, sizeof nm, "S scalar R=4 plain ctas/sm=%d", cps);
    report(nm, T.run([&] { k_stream_scalar<4, false><<<sms * cps, 256>>>((u64*)pk, pv, n, o[0], o[1], o[2], o[3]); }));
    snprintf(nm, sizeof nm, "S scalar R=8 cs ctas/sm=%d", cps);
    report(nm, T.run([&] { k_stream_scalar<8, true><<<sms * cps, 256>>>((u64*)pk, pv, n, o[0], o[1], o[2], o[3]); }));
    snprintf(nm, sizeof nm, "S vec2 R=2 ctas/sm=%d", cps);
    report(nm, T.run([&] { k_stream_vec2<2><<<sms * cps, 256>>>((ulonglong2*)pk, (ulonglong2*)pv, n / 2, (ulonglong2*)o[0], (ulonglong2*)o[1], (ulonglong2*)o[2], (ulonglong2*)o[3]); }));
    snprintf(nm, sizeof nm, "S vec2 R=4 ctas/sm=%d", cps);
    report(nm, T.run([&] { k_stream_vec2<4><<<sms * cps, 256>>>((ulonglong2*)pk, (ulonglong2*)pv, n / 2, (ulonglong2*)o[0], (ulonglong2*)o[1], (ulonglong2*)o[2], (ulonglong2*)o[3]); }));
  }
  if (all) {
    auto run_tma = [&](auto kern, int Tt, int stages, int cps, const char* nm) {
      size_t smem = (size_t)stages * 2 * Tt * 8 + 2 * 4 * Tt * 8 + stages * 8 + 16;
      CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      report(nm, T.run([&] { kern<<<sms * cps, 256, smem>>>((u64*)pk, pv, n / Tt, o[0], o[1], o[2], o[3]); }));
    };
    run_tma(k_stream_tma<1024, 2>, 1024, 2, 2, "S tma T=1024 stages=2 ctas/sm=2");
    run_tma(k_stream_tma<1024, 3>, 1024, 3, 2, "S tma T=1024 stages=3 ctas/sm=2");
    run_tma(k_stream_tma<1024, 2>, 1024, 2, 1, "S tma T=1024 stages=2 ctas/sm=1");
    run_tma(k_stream_tma<512, 3>, 512, 3, 4, "S tma T=512 stages=3 ctas/sm=4");
    run_tma(k_stream_tma<2048, 2>, 2048, 2, 1, "S tma T=2048 stages=2 ctas/sm=1");
  }

  // ---- P: probe variants, unpartitioned (u) and partition-ordered (s) input
  FastOut fo{};
  fo.n_pcols = 1; fo.n_key_dst = 2; fo.n_meta_dst = 1;
  fo.pdst[0] = o[2]; fo.key_dst[0] = o[0]; fo.key_dst[1] = o[1]; fo.meta_dst[0] = o[3];
  if (argc > 3 && std::string(argv[3]) == "pipe") {
    report("Z0 P6 flat over stable-sorted, before anything else", T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_vec2_pf<2, 3, 0><<<sms * 3, 256>>>(pk_s, pv_s, n, tv, out, cursor); }));
    // (a) the library's count + offsets + TMA scatter (dense partitions), timed per kernel
    u64* scratch; CK(cudaMalloc(&scratch, TG_MAX_PARTS * 8 * 3 + 64));
    u64* counts = scratch; u64* cursors = counts + TG_MAX_PARTS; long long* offs = (long long*)(cursors + TG_MAX_PARTS);
    const long long C = ((long long)((double)n / P * 1.04) + 8192 + 127) / 128 * 128;
    int64_t* pk_c; u64* pv_c; CK(cudaMalloc(&pk_c, (size_t)P * C * 8 + 64)); CK(cudaMalloc(&pv_c, (size_t)P * C * 8 + 64));
    u64* ovf; CK(cudaMalloc(&ovf, 8)); CK(cudaMemset(ovf, 0, 8));
    CK(cudaMemset(pk_c, 0, (size_t)P * C * 8)); CK(cudaMemset(pv_c, 0, (size_t)P * C * 8));
    PartDst d{}; d.nparts = P; d.ncols = 2; d.src[0] = pk; d.src[1] = pv;
    int64_t* pk_l; u64* pv_l; CK(cudaMalloc(&pk_l, n * 8 + 64)); CK(cudaMalloc(&pv_l, n * 8 + 64));
    for (uint32_t q = 0; q < P; q++) { d.dst[q][0] = pk_l; d.dst[q][1] = pv_l; }
    d.dst_base = offs;
    report("A1 lib count4", T.run([&] { cudaMemsetAsync(scratch, 0, TG_MAX_PARTS * 8 * 3 + 8); launch_partition_count<true>(0, 0, (const long long*)pk, nullptr, n, P, counts, nullptr); }));
    k_partition_offsets<<<1, 32>>>(counts, P, offs, cursors);
    report("A2 lib scatter_tma", T.run([&] { k_partition_offsets<<<1, 32>>>(counts, P, offs, cursors); launch_partition_scatter<true>(0, 0, (const long long*)pk, nullptr, n, d, cursors, nullptr); }));
    // (b) count-free scatter with bulk stores into capacity segments + segment probe
    long long* base_h = new long long[TG_MAX_PARTS]; for (uint32_t q = 0; q < TG_MAX_PARTS; q++) base_h[q] = (long long)q * C;
    long long* base_d; CK(cudaMalloc(&base_d, TG_MAX_PARTS * 8)); CK(cudaMemcpy(base_d, base_h, TG_MAX_PARTS * 8, cudaMemcpyHostToDevice));
    PartDst e = d; for (uint32_t q = 0; q < P; q++) { e.dst[q][0] = pk_c; e.dst[q][1] = pv_c; } e.dst_base = base_d;
    auto run_sc = [&](auto kern, int items, int cps, const char* what) {
      const int tile = PT_BLOCK * items;
      size_t smem = (size_t)2 * 2 * tile * 8 + (size_t)2 * (tile + 2 * TG_MAX_PARTS) * 8 + 2 * 8 + 16;
      CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      char nm[96]; snprintf(nm, sizeof nm, "B1 scatter_bulk %s ctas/sm=%d", what, cps);
      report(nm, T.run([&] { cudaMemsetAsync(cursors, 0, TG_MAX_PARTS * 8); kern<<<sms * cps, PT_BLOCK, smem>>>(n / tile, e, cursors, C, ovf); }));
    };
    run_sc(k_scatter_bulk<true, 2, 8, 1>, 8, 2, "items=8 rank=atomic");
    run_sc(k_scatter_bulk<true, 2, 4, 0>, 4, 4, "items=4 rank=match");
    run_sc(k_scatter_bulk<true, 2, 4, 1>, 4, 4, "items=4 rank=atomic");
    run_sc(k_scatter_bulk<true, 2, 4, 1>, 4, 3, "items=4 rank=atomic");
    run_sc(k_scatter_bulk<true, 2, 2, 1>, 2, 8, "items=2 rank=atomic");
    run_sc(k_scatter_bulk<true, 2, 8, 0>, 8, 2, "items=8 rank=match");
    size_t smem = (size_t)2 * 2 * PT_TILE * 8 + (size_t)2 * (PT_TILE + 2 * TG_MAX_PARTS) * 8 + 2 * 8 + 16;
    u64 hc[TG_MAX_PARTS], ho; CK(cudaMemcpy(hc, cursors, P * 8, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(&ho, ovf, 8, cudaMemcpyDeviceToHost));
    u64 tot = 0, mx = 0; for (uint32_t q = 0; q < P; q++) { tot += hc[q]; if (hc[q] > mx) mx = hc[q]; }
    printf("    segments: total=%llu (n=%lld, tiles cover %lld) max=%llu capacity=%lld overflow=%llu\n", tot, (long long)n, (long long)(n / PT_TILE * PT_TILE), mx, C, ho);
    report("B2 probe_seg minb=3 grid=3x", T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_seg<3><<<sms * 3, 256>>>(pk_c, pv_c, cursors, P, C, ovf, tv, out, cursor); }));
    verify("B pipeline");
    {
      cudaEvent_t ev[4]; for (auto& x : ev) CK(cudaEventCreate(&x));
      float t1 = 0, t2 = 0;
      for (int rep = 0; rep < 5; rep++) {
        cudaMemsetAsync(cursors, 0, TG_MAX_PARTS * 8); cudaMemsetAsync(cursor, 0, 8);
        CK(cudaEventRecord(ev[0]));
        k_scatter_bulk<true, 2, 4, 1><<<sms * 4, PT_BLOCK, (size_t)2 * 2 * 1024 * 8 + (size_t)2 * (1024 + 2 * TG_MAX_PARTS) * 8 + 32>>>(n / 1024, e, cursors, C, ovf);
        CK(cudaEventRecord(ev[1]));
        k_probe_seg<3><<<sms * 3, 256>>>(pk_c, pv_c, cursors, P, C, ovf, tv, out, cursor);
        CK(cudaEventRecord(ev[2])); CK(cudaEventSynchronize(ev[2]));
        float a, b; CK(cudaEventElapsedTime(&a, ev[0], ev[1])); CK(cudaEventElapsedTime(&b, ev[1], ev[2]));
        if (rep) { t1 += a; t2 += b; }
      }
      printf("    in sequence: scatter %.3f ms, probe %.3f ms\n", t1 / 4, t2 / 4);
    }
    CK(cudaMemset(cursor, 0, 8));
    report("B3 P6 flat kernel over the capacity layout", T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_vec2_pf<2, 3, 0><<<sms * 3, 256>>>(pk_c, pv_c, (int64_t)P * C, tv, out, cursor); }));
    verify("B3");
    report("B4 P6 flat kernel over the stable-sorted input", T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_vec2_pf<2, 3, 0><<<sms * 3, 256>>>(pk_s, pv_s, n, tv, out, cursor); }));
    verify("B4");
    report("B5 P0 prod warp kernel over the stable-sorted input", T.run([&] { cudaMemsetAsync(cursor, 0, 8); FastOut f2{}; f2.n_pcols = 1; f2.n_key_dst = 2; f2.n_meta_dst = 1; f2.pdst[0] = o[2]; f2.key_dst[0] = o[0]; f2.key_dst[1] = o[1]; f2.meta_dst[0] = o[3]; f2.psrc[0] = pv_s; k_probe_inner_u1_w<4, 1, 2, 1><<<sms * 3, 256>>>(pk_s, n, tv, f2, cursor, SegSpec{}); }));
    report("B6 P0 prod warp kernel over the lib-scatter output", T.run([&] { cudaMemsetAsync(cursor, 0, 8); FastOut f2{}; f2.n_pcols = 1; f2.n_key_dst = 2; f2.n_meta_dst = 1; f2.pdst[0] = o[2]; f2.key_dst[0] = o[0]; f2.key_dst[1] = o[1]; f2.meta_dst[0] = o[3]; f2.psrc[0] = pv_l; k_probe_inner_u1_w<4, 1, 2, 1><<<sms * 3, 256>>>(pk_l, n, tv, f2, cursor, SegSpec{}); }));
    verify("B6");
    report("B1+B2 back to back", T.run([&] {
      cudaMemsetAsync(cursors, 0, TG_MAX_PARTS * 8); cudaMemsetAsync(cursor, 0, 8);
      k_scatter_bulk<true, 2, 4, 1><<<sms * 4, PT_BLOCK, (size_t)2 * 2 * 1024 * 8 + (size_t)2 * (1024 + 2 * TG_MAX_PARTS) * 8 + 32>>>(n / 1024, e, cursors, C, ovf);
      k_probe_seg<3><<<sms * 3, 256>>>(pk_c, pv_c, cursors, P, C, ovf, tv, out, cursor); }));
    verify("B pipeline (fused timing)");
    report("Z1 P6 flat over stable-sorted, at the end", T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_vec2_pf<2, 3, 0><<<sms * 3, 256>>>(pk_s, pv_s, n, tv, out, cursor); }));
    for (int rep = 0; rep < 4; rep++) {
      const int carve = rep == 0 ? -1 : rep == 1 ? 0 : rep == 2 ? 100 : 0;
      CK(cudaFuncSetAttribute(k_probe_vec2_pf<2, 3, 0>, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
      CK(cudaFuncSetAttribute(k_probe_seg<3>, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
      CK(cudaFuncSetAttribute(k_probe_seg_dyn<3>, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
      printf("  -- preferred shared memory carveout = %d\n", carve);
      report("Z2 P6 flat over capacity layout", T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_vec2_pf<2, 3, 0><<<sms * 3, 256>>>(pk_c, pv_c, (int64_t)P * C, tv, out, cursor); }));
      report("Z3 probe_seg", T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_seg<3><<<sms * 3, 256>>>(pk_c, pv_c, cursors, P, C, ovf, tv, out, cursor); }));
      report("Z5 probe_seg_dyn", T.run([&] { cudaMemsetAsync(cursor, 0, 16); k_probe_seg_dyn<3><<<sms * 3, 256>>>(pk_c, pv_c, cursors, P, C, ovf, tv, out, cursor); }));
      report("Z4 P6 flat over stable-sorted", T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_vec2_pf<2, 3, 0><<<sms * 3, 256>>>(pk_s, pv_s, n, tv, out, cursor); }));
    }
    verify("Z (last = Z4)");
    cudaMemsetAsync(cursor, 0, 16); k_probe_seg_dyn<3><<<sms * 3, 256>>>(pk_c, pv_c, cursors, P, C, ovf, tv, out, cursor);
    verify("Z5 dyn");
    return 0;
  }
  if (argc > 3 && std::string(argv[3]) == "p6") {
    k_probe_vec2_pf<2, 3, 0><<<sms * 3, 256>>>(pk_s, pv_s, n, tv, out, cursor);
    CK(cudaDeviceSynchronize());
    cudaMemset(cursor, 0, 8);
    k_probe_vec2_pf<2, 3, 0><<<sms * 3, 256>>>(pk_s, pv_s, n, tv, out, cursor);
    CK(cudaDeviceSynchronize());
    return 0;
  }
  for (int sorted = all ? 0 : 1; sorted < 2; sorted++) {
    const int64_t* K = sorted ? pk_s : pk; const u64* V = sorted ? pv_s : pv;
    const char* tag = sorted ? "part-ordered" : "unpartitioned";
    char nm[160];
    fo.psrc[0] = V;
    for (int cps : {3, 8}) {
      snprintf(nm, sizeof nm, "P0 prod warp<4,1,2,1> %s grid=%dx", tag, cps);
      report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_inner_u1_w<4, 1, 2, 1><<<sms * cps, 256>>>(K, n, tv, fo, cursor, SegSpec{}); }));
    }
    verify("P0");
    {
      size_t smem = (size_t)4 * 2 * TG_PROBE_TILE * 8 + 4 * 8 + 16;
      CK(cudaFuncSetAttribute(k_probe_inner_u1_tma<1, 2, 1, 4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      snprintf(nm, sizeof nm, "P1 prod tma stages=4 %s grid=3x", tag);
      report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_inner_u1_tma<1, 2, 1, 4, false><<<sms * 3, 256, smem>>>(K, n / TG_PROBE_TILE, tv, fo, cursor); }));
      verify("P1");
    }
    for (int cps : {3, 4, 8}) {
      snprintf(nm, sizeof nm, "P2 vec2 G=2 %s grid=%dx", tag, cps);
      report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_vec2<2><<<sms * cps, 256>>>(K, V, n, tv, out, cursor); }));
    }
    verify("P2 G=2");
    snprintf(nm, sizeof nm, "P2 vec2 G=1 %s grid=8x", tag);
    report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_vec2<1><<<sms * 8, 256>>>(K, V, n, tv, out, cursor); }));
    verify("P2 G=1");
    for (int rep = 0; rep < 2; rep++) {
      snprintf(nm, sizeof nm, "P2b vec2 G=2 minb=3 %s grid=3x", tag);
      report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_vec2<2, 3><<<sms * 3, 256>>>(K, V, n, tv, out, cursor); }));
      snprintf(nm, sizeof nm, "P2b vec2 G=2 minb=4 %s grid=4x", tag);
      report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_vec2<2, 4><<<sms * 4, 256>>>(K, V, n, tv, out, cursor); }));
      snprintf(nm, sizeof nm, "P0 prod warp %s grid=3x", tag);
      report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_inner_u1_w<4, 1, 2, 1><<<sms * 3, 256>>>(K, n, tv, fo, cursor, SegSpec{}); }));
    }
    verify("P2b");
    {
      auto run_tpf = [&](auto kern, const char* what, int cps) {
        snprintf(nm, sizeof nm, "P14 %s %s grid=%dx", what, tag, cps);
        report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); kern<<<sms * cps, 256>>>(K, V, n, tv, out, cursor); }));
      };
      for (int rep = 0; rep < 2; rep++) {
        run_tpf(k_probe_vec2_tpf<2, 3, 1>, "vec2+regpf+L1 table prefetch minb=3", 3);
        run_tpf(k_probe_vec2_tpf<2, 3, 2>, "vec2+regpf+L2 table prefetch minb=3", 3);
        run_tpf(k_probe_vec2_tpf<2, 2, 1>, "vec2+regpf+L1 table prefetch minb=2", 2);
      }
      verify("P14");
    }
    {
      auto run_pf = [&](auto kern, const char* what, int cps) {
        snprintf(nm, sizeof nm, "P6 %s %s grid=%dx", what, tag, cps);
        report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); kern<<<sms * cps, 256>>>(K, V, n, tv, out, cursor); }));
      };
      run_pf(k_probe_vec2_pf<2, 1>, "vec2+regpf G=2 minb=1", 2); run_pf(k_probe_vec2_pf<2, 1>, "vec2+regpf G=2 minb=1", 3);
      run_pf(k_probe_vec2_pf<2, 3>, "vec2+regpf G=2 minb=3", 3);
      verify("P6 G=2 minb=3");
      run_pf(k_probe_vec2_pf<2, 3, 1>, "vec2+regpf G=2 minb=3 NOATOMIC", 3);
      run_pf(k_probe_vec2_pf<2, 3, 2>, "vec2+regpf G=2 minb=3 CTA-AGG", 3);
      run_pf(k_probe_vec2_pf<2, 2, 2>, "vec2+regpf G=2 minb=2 CTA-AGG", 2);
      run_pf(k_probe_vec2_pf<2, 4>, "vec2+regpf G=2 minb=4", 4);
      run_pf(k_probe_vec2_pf<1, 4>, "vec2+regpf G=1 minb=4", 4); run_pf(k_probe_vec2_pf<1, 6>, "vec2+regpf G=1 minb=6", 6);
      verify("P6 G=1 minb=6");
      run_pf(k_probe_vec2_pf<4, 1>, "vec2+regpf G=4 minb=1", 1); run_pf(k_probe_vec2_pf<4, 2>, "vec2+regpf G=4 minb=2", 2);
      verify("P6 G=4 minb=2");
    }
    {
      auto run_cpa = [&](auto kern, int G, int D, const char* what, int cps) {
        size_t smem = (size_t)8 * D * 2 * G * 32 * 16;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        snprintf(nm, sizeof nm, "P8 %s %s grid=%dx", what, tag, cps);
        report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); kern<<<sms * cps, 256, smem>>>(K, V, n, tv, out, cursor); }));
      };
      run_cpa(k_probe_vec2_cpa<2, 2, 3>, 2, 2, "vec2+cpasync G=2 D=2 minb=3", 3);
      run_cpa(k_probe_vec2_cpa<2, 3, 3>, 2, 3, "vec2+cpasync G=2 D=3 minb=3", 3);
      run_cpa(k_probe_vec2_cpa<2, 4, 3>, 2, 4, "vec2+cpasync G=2 D=4 minb=3", 3);
      verify("P8 G=2 D=4");
      run_cpa(k_probe_vec2_cpa<2, 3, 2>, 2, 3, "vec2+cpasync G=2 D=3 minb=2", 2);
      run_cpa(k_probe_vec2_cpa<2, 3, 4>, 2, 3, "vec2+cpasync G=2 D=3 minb=4", 4);
      run_cpa(k_probe_vec2_cpa<4, 2, 2>, 4, 2, "vec2+cpasync G=4 D=2 minb=2", 2);
      run_cpa(k_probe_vec2_cpa<4, 3, 1>, 4, 3, "vec2+cpasync G=4 D=3 minb=1", 1);
      verify("P8 G=4");
    }
    {
      auto run_v3 = [&](auto kern, int G, int D, const char* what, int cps) {
        size_t smem = (size_t)8 * D * 2 * G * 32 * 16;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        snprintf(nm, sizeof nm, "P12 %s %s grid=%dx", what, tag, cps);
        report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); kern<<<sms * cps, 256, smem>>>(K, V, n, tv0, out, cursor); }));
      };
      run_v3(k_probe_v3<2, 2, 4>, 2, 2, "v3 slot16 G=2 D=2 minb=4", 4);
      run_v3(k_probe_v3<2, 2, 5>, 2, 2, "v3 slot16 G=2 D=2 minb=5", 5);
      run_v3(k_probe_v3<2, 2, 6>, 2, 2, "v3 slot16 G=2 D=2 minb=6", 6);
      run_v3(k_probe_v3<2, 3, 4>, 2, 3, "v3 slot16 G=2 D=3 minb=4", 4);
      verify("P12 G=2");
      run_v3(k_probe_v3<4, 2, 3>, 4, 2, "v3 slot16 G=4 D=2 minb=3", 3);
      run_v3(k_probe_v3<4, 2, 2>, 4, 2, "v3 slot16 G=4 D=2 minb=2", 2);
      run_v3(k_probe_v3<4, 3, 2>, 4, 3, "v3 slot16 G=4 D=3 minb=2", 2);
      verify("P12 G=4");
      run_v3(k_probe_v3<8, 2, 1>, 8, 2, "v3 slot16 G=8 D=2 minb=1", 1);
      verify("P12 G=8");
    }
    {
      auto run_pol = [&](auto kern, const char* what, int cps) {
        snprintf(nm, sizeof nm, "P13 %s %s grid=%dx", what, tag, cps);
        report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); kern<<<sms * cps, 256>>>(K, V, n, tv, out, cursor); }));
      };
      run_pol(k_probe_pol<2, 3, 0>, "pol=0 (base)", 3);
      run_pol(k_probe_pol<2, 3, 1>, "pol=1 table evict_last", 3);
      run_pol(k_probe_pol<2, 3, 2>, "pol=2 stores evict_first hint", 3);
      run_pol(k_probe_pol<2, 3, 3>, "pol=3 both", 3);
      run_pol(k_probe_pol<2, 3, 7>, "pol=7 all", 3);
      run_pol(k_probe_pol<2, 3, 5>, "pol=5 table last + in first", 3);
      verify("P13");
      run_pol(k_probe_pol<2, 4, 7>, "pol=7 minb=4", 4);
      run_pol(k_probe_pol<1, 6, 7>, "G=1 pol=7 minb=6", 6);
      run_pol(k_probe_pol<1, 6, 0>, "G=1 pol=0 minb=6", 6);
      verify("P13b");
    }
    if (all) {
      size_t smem = (size_t)8 * 2 * 4 * STG_ROWS * 8;
      CK(cudaFuncSetAttribute(k_probe_bulkout<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      CK(cudaFuncSetAttribute(k_probe_bulkout<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      for (int cps : {2, 3}) {
        snprintf(nm, sizeof nm, "P4 ldg-in bulk-out %s grid=%dx", tag, cps);
        report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_bulkout<false><<<sms * cps, 256, smem>>>(K, V, n, tv, out, cursor); }));
      }
      verify("P4");
      for (int cps : {2, 3}) {
        snprintf(nm, sizeof nm, "P5 ldg-in prefetch bulk-out %s grid=%dx", tag, cps);
        report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); k_probe_bulkout<true><<<sms * cps, 256, smem>>>(K, V, n, tv, out, cursor); }));
      }
      verify("P5");
    }
    if (all) {
      auto run_io = [&](auto kern, int stages, int cps) {
        size_t smem = (size_t)8 * ((size_t)stages * 2 * 128 + 2 * 4 * STG_ROWS + ((stages + 1) & ~1)) * 8;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        snprintf(nm, sizeof nm, "P3 tma-in(%d) bulk-out %s grid=%dx", stages, tag, cps);
        report(nm, T.run([&] { cudaMemsetAsync(cursor, 0, 8); kern<<<sms * cps, 256, smem>>>(K, V, n, tv, out, cursor); }));
      };
      run_io(k_probe_tma_io<2>, 2, 2); run_io(k_probe_tma_io<2>, 2, 1);
      run_io(k_probe_tma_io<3>, 3, 1); run_io(k_probe_tma_io<4>, 4, 1);
      verify("P3");
    }
  }
  return 0;
}
