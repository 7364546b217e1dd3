// pilot_lab.cu — can a per-slice pilot index (hash-and-displace, one 16-byte gather per row) beat the linear-probe table
// in the in-place segment probe at the bench shape?  100 M partition-ordered probe rows, 100 % match, against 10 M unique
// build keys (bench.py's keys: id * ODD), 16 slices.
//
//   (a) k_probe_inner_u1_seg_inplace<1,2,1> from the library against the linear-probe table at load factor 0.5
//   (b) a prototype of the same kernel that reads the key's pilot byte and gathers ONE 16-byte slot of a dense slice table
//       at load factor ALPHA; the pilots come from global memory through L1 (`gl`), or from shared memory, where a CTA
//       loads the pilots of one slice and its warps sweep that slice's tiles together (`sm`)
//
// build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I include -I tidb_b200/csrc \
//          -o tools/scratch/pilot_lab tools/scratch/pilot_lab.cu
// run:   tools/scratch/pilot_lab [ALPHA LAMBDA]...        (GPU: kernel times, median of 30 alternating launches per variant,
//                                                          for each (load factor, mean keys per bucket) pair; default
//                                                          0.9 2  0.8 3  0.75 4)
//        tools/scratch/pilot_lab --host [ALPHA LAMBDA]   (CPU only: placement statistics of the pilot index)
//        tools/scratch/pilot_lab --slices                (GPU: 16 against 32 slices — the index probe and the scatter of the
//                                                         library at the bench shape, DESIGN.md §4.1 "16 against 32")
//        tools/scratch/pilot_lab --scatter               (GPU: the L2 partition pass at 16 and 32 slices — 1024- to 4096-row
//                                                         tiles, 256 to 1024 threads, ballot ranks, two staging buffers, a
//                                                         one-stage ring and a plain copy of the same bytes, DESIGN.md §4.1
//                                                         "4096-row scatter tiles")
//
// The index is built on the host here (sequential, largest bucket first, one byte per pilot, 255 = not placed: such a
// key's tile takes the library's generic path on the linear-probe table).  Results: DESIGN.md §4.1 "Pilot index".
#include "join_kernels.cuh"
#include "partition_kernels.cuh"
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <random>
#include <vector>

using namespace tg;
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e_), __LINE__); exit(1); } } while (0)

static const uint64_t ODD = 0x9E3779B97F4A7C15ull;
static int P = 16;   // slices (--slices sets 16 and 32 in turn)

// slot of a key within its slice under pilot q
__host__ __device__ __forceinline__ uint32_t pilot_slot(uint64_t h, uint32_t q, uint32_t S) {
  return slot32(hash64(h ^ ((uint64_t)(q + 1) * 0xC2B2AE3D27D4EB4Full)), S);
}
__host__ __device__ __forceinline__ uint32_t bucket_of(uint64_t h, uint32_t B) { return mulhi32((uint32_t)h, B); }

struct Index {
  uint32_t S = 0, B = 0;
  std::vector<uint8_t> pilot;   // [P][B]
  std::vector<Slot> slots;      // [P][S]
  long long bad_buckets = 0, bad_keys = 0;
};

// sequential hash-and-displace per slice, largest bucket first; pilot 255 = not placed
static Index build_index(const std::vector<uint64_t>& keys, const std::vector<uint64_t>& payload, double alpha, double lambda,
                         bool fill_slots, bool library_sizing = false) {
  std::vector<std::vector<uint32_t>> part(P);
  for (uint32_t i = 0; i < keys.size(); i++) part[slot32(hash64(keys[i]), P)].push_back(i);
  size_t mx = 0;
  for (auto& v : part) mx = std::max(mx, v.size());
  Index ix;
  ix.S = (uint32_t)std::ceil(mx / alpha);
  ix.B = ((uint32_t)std::ceil(mx / lambda) + 15) & ~15u;   // whole uint4 rows for the shared-memory copy
  if (library_sizing) {   // build_slice_index (join.cu)
    ix.S = (uint32_t)std::ceil((double)mx / alpha) + 1;
    ix.B = ((uint32_t)std::ceil((double)mx / lambda) + 16) & ~15u;
  }
  ix.pilot.assign((size_t)P * ix.B, 255);
  if (fill_slots) ix.slots.assign((size_t)P * ix.S, Slot{kEmptyKey, 0});
  std::vector<uint8_t> taken(ix.S);
  for (int p = 0; p < P; p++) {
    std::fill(taken.begin(), taken.end(), 0);
    std::vector<uint32_t> cnt(ix.B + 1, 0), ord(part[p].size());
    for (uint32_t i : part[p]) cnt[bucket_of(hash64(keys[i]), ix.B) + 1]++;
    std::partial_sum(cnt.begin(), cnt.end(), cnt.begin());
    std::vector<uint32_t> pos(cnt.begin(), cnt.end() - 1);
    for (uint32_t i : part[p]) ord[pos[bucket_of(hash64(keys[i]), ix.B)]++] = i;
    std::vector<uint32_t> bs(ix.B);
    std::iota(bs.begin(), bs.end(), 0);
    std::stable_sort(bs.begin(), bs.end(), [&](uint32_t a, uint32_t b) { return cnt[a + 1] - cnt[a] > cnt[b + 1] - cnt[b]; });
    uint32_t sl[64];
    for (uint32_t b : bs) {
      const uint32_t n = cnt[b + 1] - cnt[b];
      if (!n) break;
      int q = 0;
      for (; q < 255; q++) {
        bool ok = n <= 64;
        for (uint32_t j = 0; ok && j < n; j++) {
          sl[j] = pilot_slot(hash64(keys[ord[cnt[b] + j]]), q, ix.S);
          if (taken[sl[j]]) ok = false;
          for (uint32_t i = 0; ok && i < j; i++) ok = sl[i] != sl[j];
        }
        if (ok) break;
      }
      if (q == 255) { ix.bad_buckets++; ix.bad_keys += n; continue; }
      ix.pilot[(size_t)p * ix.B + b] = (uint8_t)q;
      for (uint32_t j = 0; j < n; j++) {
        taken[sl[j]] = 1;
        if (fill_slots) {
          const uint32_t i = ord[cnt[b] + j];
          ix.slots[(size_t)p * ix.S + sl[j]] = Slot{(int64_t)keys[i], payload[i]};
        }
      }
    }
  }
  return ix;
}

// ---- (b) prototype: pilot → slot → one LDG.128 → compare ---------------------------------------------------------------
struct PilotView {
  const Slot* slots; const uint8_t* pilot; uint32_t S, B, P;
};

template <bool SMEM>
__device__ __forceinline__ void pilot_tile(int64_t base, int64_t limit, const PilotView& ix, const uint8_t* spil, const TableView& t,
                                           const FastOut& out, int lane, uint32_t& m) {
  constexpr int R = 4, G = 2, NPC = 1, NKD = 2, NMD = 1, NP = 1;
  const int64_t* pkey = reinterpret_cast<const int64_t*>(out.key_dst[0]);
  if (limit - base < 128) { m = inplace_tile_generic<NPC, NKD, NMD>(base, limit, t, out, lane); return; }
  int64_t k[R];
#pragma unroll
  for (int g = 0; g < G; g++) {
    const ulonglong2 kk = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + base + g * 64 + 2 * lane));
    k[2 * g] = (int64_t)kk.x; k[2 * g + 1] = (int64_t)kk.y;
  }
  uint32_t q[R];
  bool odd = false;
#pragma unroll
  for (int j = 0; j < R; j++) {
    const uint64_t h = hash64((uint64_t)k[j]);
    const uint32_t p = slot32(h, ix.P), b = bucket_of(h, ix.B);
    q[j] = SMEM ? spil[b] : __ldg(ix.pilot + (size_t)p * ix.B + b);
    odd |= (k[j] == kEmptyKey) | (q[j] == 255u);
  }
  if (__any_sync(0xffffffffu, odd)) { m = inplace_tile_generic<NPC, NKD, NMD>(base, limit, t, out, lane); return; }
  unsigned long long meta[R];
  unsigned hit = 0;
#pragma unroll
  for (int j = 0; j < R; j++) {
    const uint64_t h = hash64((uint64_t)k[j]);
    const Slot v = load_slot(ix.slots + (size_t)slot32(h, ix.P) * ix.S + pilot_slot(h, q[j], ix.S));
    meta[j] = v.meta;
    if (v.key == k[j]) hit |= 1u << j;
  }
  if (__all_sync(0xffffffffu, hit == 0xFu)) {
    m = 128;
#pragma unroll
    for (int g = 0; g < G; g++) {
      const int64_t o = base + g * 64 + 2 * lane;
      const ulonglong2 kk = make_ulonglong2((unsigned long long)k[2 * g], (unsigned long long)k[2 * g + 1]);
#pragma unroll
      for (int d = 1; d < NKD; d++) __stcs(reinterpret_cast<ulonglong2*>(out.key_dst[d] + o), kk);
#pragma unroll
      for (int d = 0; d < NMD; d++) __stcs(reinterpret_cast<ulonglong2*>(out.meta_dst[d] + o), make_ulonglong2(meta[2 * g], meta[2 * g + 1]));
    }
  } else {
    unsigned long long pv[R][NP];
    inplace_load_pv<NPC>(base, out, pv, lane);
    unsigned bal[R];
    m = 0;
#pragma unroll
    for (int j = 0; j < R; j++) { bal[j] = __ballot_sync(0xffffffffu, (hit >> j) & 1u); m += __popc(bal[j]); }
    inplace_store<NPC, NKD, NMD>(base, k, meta, pv, bal, out, lane);
  }
}

// warp-autonomous, pilots through L1
__global__ void __launch_bounds__(256, 3)
k_pilot_gl(int64_t n, TableView t, PilotView ix, FastOut out, unsigned long long* out_cursor, SegSpec seg, uint32_t* tile_cnt) {
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t warp_id = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t ntiles = n / 128;
  unsigned long long kept = 0;
  for (int64_t tile = warp_id; tile < ntiles; tile += warps_total) {
    const int64_t base = tile * 128;
    const uint32_t p = (uint32_t)tile / seg.tiles_per_seg;
    const unsigned long long c = seg.cnt[p];
    const int64_t limit = (int64_t)p * seg.cap + (int64_t)(c < (unsigned long long)seg.cap ? c : (unsigned long long)seg.cap);
    uint32_t m = 0;
    if (limit > base) pilot_tile<false>(base, limit, ix, nullptr, t, out, lane, m);
    if (lane == 0) tile_cnt[tile] = m;
    kept += m;
  }
  if (lane == 0 && kept) atomicAdd(out_cursor, kept);
}

// CTA per slice in turn: the CTA's pilots of slice p in shared memory, its warps stride over slice p's tiles
template <int NT>
__global__ void __launch_bounds__(NT, 1)
k_pilot_sm(int64_t n, TableView t, PilotView ix, FastOut out, unsigned long long* out_cursor, SegSpec seg, uint32_t* tile_cnt) {
  extern __shared__ uint8_t spil[];
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (NT >> 5);
  const int64_t warp_id = (int64_t)blockIdx.x * (NT >> 5) + (threadIdx.x >> 5);
  unsigned long long kept = 0;
  const int nseg = (int)(n / 128 / seg.tiles_per_seg);
  for (int p = 0; p < nseg; p++) {
    __syncthreads();
    const uint4* src = reinterpret_cast<const uint4*>(ix.pilot + (size_t)p * ix.B);
    for (uint32_t i = threadIdx.x; i < ix.B / 16; i += NT) reinterpret_cast<uint4*>(spil)[i] = __ldcs(src + i);
    __syncthreads();
    const unsigned long long c = seg.cnt[p];
    const int64_t limit = (int64_t)p * seg.cap + (int64_t)(c < (unsigned long long)seg.cap ? c : (unsigned long long)seg.cap);
    const int64_t t0 = (int64_t)p * seg.tiles_per_seg, t1 = t0 + seg.tiles_per_seg;
    for (int64_t tile = t0 + warp_id; tile < t1; tile += warps_total) {
      const int64_t base = tile * 128;
      uint32_t m = 0;
      if (limit > base) pilot_tile<true>(base, limit, ix, spil, t, out, lane, m);
      if (lane == 0) tile_cnt[tile] = m;
      kept += m;
    }
  }
  if (lane == 0 && kept) atomicAdd(out_cursor, kept);
}

// linear-probe insert (the library's k_build_insert without its column plumbing): U1, meta = payload
__global__ void k_lp_insert(const unsigned long long* keys, const unsigned long long* pay, int64_t n, Slot* slots, unsigned long long nslots) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t k = (int64_t)keys[i];
  unsigned long long s = home_slot(hash64((uint64_t)k), nslots);
  for (;;) {
    const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(&slots[s].key), (unsigned long long)kEmptyKey, (unsigned long long)k);
    if (old == (unsigned long long)kEmptyKey) { slots[s].meta = pay[i]; return; }
    if (++s == nslots) s = 0;
  }
}

static void host_stats(const std::vector<double>& as, const std::vector<double>& ls) {
  std::vector<uint64_t> keys(10000000), pay(keys.size());
  for (uint64_t i = 0; i < keys.size(); i++) { keys[i] = i * ODD; pay[i] = i * 7; }
  for (double a : as)
    for (double l : ls) {
      Index ix = build_index(keys, pay, a, l, false);
      printf("alpha %.2f lambda %.1f: S %u (%.2f MiB per slice) B %u (%.0f KiB of pilots)  unplaced buckets %lld keys %lld\n", a, l,
             ix.S, ix.S * 16.0 / (1 << 20), ix.B, ix.B / 1024.0, ix.bad_buckets, ix.bad_keys);
      fflush(stdout);
    }
}

// ---- --slices: 16 against 32 slices at the bench shape (DESIGN.md §4.1, "32 slices") -------------------------------
// The library's k_probe_inner_u1_seg_inplace_pidx as it was with 16 slices: one pilot buffer, and every slice behind two
// CTA-wide barriers (the CTA loads the pilots while no gather is in flight).  Variant (a) runs it with half-size slices.
template <int NPC, int NKD, int NMD>
__global__ void __launch_bounds__(1024, 1)
k_pidx_barrier(int64_t n, TableView t, SliceIndex ix, FastOut out, unsigned long long* __restrict__ out_cursor,
                                  SegSpec seg, uint32_t* __restrict__ tile_cnt) {
  static_assert(NKD >= 1, "the probe key is read from the first key destination");
  constexpr int R = 4, G = 2, NP = NPC > 0 ? NPC : 1;
  extern __shared__ __align__(16) uint8_t spil[];
  if (seg.gate && ((*seg.gate != 0ull) != (seg.gate_want != 0))) return;
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (1024 / 32);
  const int64_t warp_id = (int64_t)blockIdx.x * (1024 / 32) + (threadIdx.x >> 5);
  const int64_t* __restrict__ pkey = reinterpret_cast<const int64_t*>(out.key_dst[0]);
  const int nseg = (int)(n / 128 / seg.tiles_per_seg);
  unsigned long long kept = 0;
  for (int p = 0; p < nseg; p++) {
    __syncthreads();   // every warp is done with the previous slice's pilots
    const uint4* src = reinterpret_cast<const uint4*>(ix.pilot + (size_t)p * ix.B);
    for (uint32_t i = threadIdx.x; i < ix.B / 16; i += 1024) reinterpret_cast<uint4*>(spil)[i] = __ldcs(src + i);
    __syncthreads();
    const unsigned long long c = seg.cnt[p];
    const int64_t limit = (int64_t)p * seg.cap + (int64_t)(c < (unsigned long long)seg.cap ? c : (unsigned long long)seg.cap);
    const int64_t t0 = (int64_t)p * seg.tiles_per_seg, t1 = t0 + seg.tiles_per_seg;
    const Slot* __restrict__ islots = ix.slots + (size_t)p * ix.S;
    for (int64_t tile = t0 + warp_id; tile < t1; tile += warps_total) {
      const int64_t base = tile * 128;
      uint32_t m = 0;
      if (limit - base >= 128) {
        int64_t k[R];
#pragma unroll
        for (int g = 0; g < G; g++) {
          const ulonglong2 kk = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + base + g * 64 + 2 * lane));
          k[2 * g] = (int64_t)kk.x; k[2 * g + 1] = (int64_t)kk.y;
        }
        uint32_t q[R];
        bool generic = false;
#pragma unroll
        for (int j = 0; j < R; j++) {
          q[j] = spil[pidx_bucket(hash64((uint64_t)k[j]), ix.B)];
          generic |= (k[j] == kEmptyKey) | (q[j] == kPilotNone);
        }
        if (__any_sync(0xffffffffu, generic)) {
          m = inplace_tile_generic<NPC, NKD, NMD>(base, limit, t, out, lane);
        } else {
          unsigned long long meta[R];
          unsigned hit = 0;
#pragma unroll
          for (int j = 0; j < R; j++) {
            const Slot v = load_slot(islots + pidx_slot(hash64((uint64_t)k[j]), q[j], ix.S));
            meta[j] = v.meta;
            if (v.key == k[j]) hit |= 1u << j;
          }
          if (__all_sync(0xffffffffu, hit == 0xFu)) {
            m = 128;
#pragma unroll
            for (int g = 0; g < G; g++) {
              const int64_t o = base + g * 64 + 2 * lane;
              const ulonglong2 kk = make_ulonglong2((unsigned long long)k[2 * g], (unsigned long long)k[2 * g + 1]);
#pragma unroll
              for (int d = 1; d < NKD; d++) __stcs(reinterpret_cast<ulonglong2*>(out.key_dst[d] + o), kk);
#pragma unroll
              for (int d = 0; d < NMD; d++) __stcs(reinterpret_cast<ulonglong2*>(out.meta_dst[d] + o), make_ulonglong2(meta[2 * g], meta[2 * g + 1]));
            }
          } else {
            unsigned long long pv[R][NP];
            inplace_load_pv<NPC>(base, out, pv, lane);
            unsigned bal[R];
#pragma unroll
            for (int j = 0; j < R; j++) {
              bal[j] = __ballot_sync(0xffffffffu, (hit >> j) & 1u);
              m += __popc(bal[j]);
            }
            inplace_store<NPC, NKD, NMD>(base, k, meta, pv, bal, out, lane);
          }
        }
      } else if (limit > base) {
        m = inplace_tile_generic<NPC, NKD, NMD>(base, limit, t, out, lane);
      }
      if (lane == 0) tile_cnt[tile] = m;
      kept += m;
    }
  }
  if (lane == 0 && kept) atomicAdd(out_cursor, kept);
}


template <int ITEMS>
static void scatter(int sms, int64_t rows, const PartDst& d, unsigned long long* cursors, long long* bases, unsigned long long* flag,
                    int P, long long C) {
  constexpr int NC = 2, TILE = PT_BLOCK * ITEMS;
  const size_t smem = (size_t)2 * NC * TILE * 8 + (size_t)NC * (TILE + 2 * TG_MAX_SLICES) * 8 + 2 * 8 + 16;
  static bool set = false;
  if (!set) { CK(cudaFuncSetAttribute(k_partition_scatter_bulk<true, NC, ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); set = true; }
  const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (size_t)(220 * 1024) / (smem + 1024)));   // launch_scatter_nc
  const int64_t ntiles = rows / TILE;   // whole tiles of this ITEMS only
  k_segment_bases<<<1, 32>>>(cursors, bases, flag, P, C);
  k_partition_scatter_bulk<true, NC, ITEMS><<<(int)std::min<int64_t>(ntiles, (int64_t)sms * per_sm), PT_BLOCK, smem>>>(ntiles, d, cursors);
}

// One configuration: P slices, its segments (scattered from the same probe columns), its index.
struct Cut {
  int P; long long C; unsigned long long *key0, *pv0, *scr; Index ix; Slot* d_ix; uint8_t* d_pil; SliceIndex si;
};

static int slices_gate() {
  const int64_t nb = 10000000, np = 100000000;
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  printf("card %s, %d SMs, L2 %d MiB, shared memory per block (opt-in) %zu B\n", prop.name, sms, prop.l2CacheSize >> 20, prop.sharedMemPerBlockOptin);
  // bench.py's columns: build keys id * ODD (ids a permutation), payload id * 7; probe keys uniform ids * ODD, payload the row
  std::vector<uint64_t> bk(nb), bv(nb), ids(nb), pk(np), pv(np);
  std::iota(ids.begin(), ids.end(), 0);
  std::mt19937_64 rng(42);
  std::shuffle(ids.begin(), ids.end(), rng);
  for (int64_t i = 0; i < nb; i++) { bk[i] = ids[i] * ODD; bv[i] = ids[i] * 7; }
  std::uniform_int_distribution<uint64_t> U(0, nb - 1);
  for (int64_t i = 0; i < np; i++) { pk[i] = U(rng) * ODD; pv[i] = (uint64_t)i; }
  unsigned long long *d_bk, *d_bv, *d_pk, *d_pv, *d_key1, *d_meta, *d_cur;
  uint32_t* d_tc;
  Slot* d_lp;
  const unsigned long long nslots = (unsigned long long)(nb / 0.5 + 32) & ~3ull;
  const long long cmax = (long long)(np / 16 * 1.05) + 16384 + 128;
  CK(cudaMalloc(&d_bk, nb * 8)); CK(cudaMalloc(&d_bv, nb * 8)); CK(cudaMalloc(&d_pk, np * 8)); CK(cudaMalloc(&d_pv, np * 8));
  CK(cudaMalloc(&d_key1, 16 * cmax * 8)); CK(cudaMalloc(&d_meta, 16 * cmax * 8)); CK(cudaMalloc(&d_cur, 8));
  CK(cudaMalloc(&d_tc, 16 * cmax / 128 * 4 + 64)); CK(cudaMalloc(&d_lp, (nslots + 2) * sizeof(Slot)));
  CK(cudaMemcpy(d_bk, bk.data(), nb * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(d_bv, bv.data(), nb * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_pk, pk.data(), np * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(d_pv, pv.data(), np * 8, cudaMemcpyHostToDevice));
  k_table_init<<<(nslots + 256) / 256, 256>>>(d_lp, nslots + 2, nslots);
  k_lp_insert<<<(nb + 255) / 256, 256>>>(d_bk, d_bv, nb, d_lp, nslots);
  CK(cudaDeviceSynchronize());
  const TableView t{d_lp, nslots, nullptr, 0, -1, TABLE_U1, 0};
  const int64_t nrows = np / 2048 * 2048;   // whole scatter tiles at ITEMS 4 and 8: the same rows for both
  Cut cut[2];
  for (int c = 0; c < 2; c++) {
    Cut& k = cut[c];
    P = k.P = 16 << c;
    const long long C0 = ((long long)((double)np / P * 1.05) + 16384 + 127) / 128 * 128;
    CK(cudaMalloc(&k.key0, P * C0 * 8)); CK(cudaMalloc(&k.pv0, P * C0 * 8)); CK(cudaMalloc(&k.scr, (3 * TG_MAX_SLICES + 8) * 8));
    PartDst d{};
    d.nparts = P; d.ncols = 2; d.src[0] = d_pk; d.src[1] = d_pv;
    for (int q = 0; q < P; q++) { d.dst[q][0] = k.key0; d.dst[q][1] = k.pv0; }
    unsigned long long* cursors = k.scr;
    long long* bases = reinterpret_cast<long long*>(k.scr + TG_MAX_SLICES);
    unsigned long long* flag = k.scr + 2 * TG_MAX_SLICES;
    d.dst_base = bases; d.capacity = C0; d.overflow = flag;
    scatter<4>(sms, nrows, d, cursors, bases, flag, P, C0);
    unsigned long long fill[TG_MAX_SLICES];
    CK(cudaMemcpy(fill, cursors, P * 8, cudaMemcpyDeviceToHost));
    const double f = (double)*std::max_element(fill, fill + P);
    k.C = std::min(((long long)(f + 8.0 * std::sqrt(f)) + 4096 + 127) / 128 * 128, C0);   // inplace_seg_cap
    d.capacity = k.C;
    scatter<4>(sms, nrows, d, cursors, bases, flag, P, k.C);
    unsigned long long ov = 0;
    CK(cudaMemcpy(&ov, flag, 8, cudaMemcpyDeviceToHost));
    k.ix = build_index(bk, bv, 0.7, 4.0, true, true);
    CK(cudaMalloc(&k.d_ix, k.ix.slots.size() * sizeof(Slot))); CK(cudaMalloc(&k.d_pil, k.ix.pilot.size()));
    CK(cudaMemcpy(k.d_ix, k.ix.slots.data(), k.ix.slots.size() * sizeof(Slot), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(k.d_pil, k.ix.pilot.data(), k.ix.pilot.size(), cudaMemcpyHostToDevice));
    k.si = SliceIndex{k.d_ix, k.d_pil, (uint32_t)P, k.ix.S, k.ix.B, 1};
    printf("P %d: segment capacity %lld (largest fill %.0f, overflow %llu), S %u (%.2f MiB per slice), B %u (%.1f KiB of pilots), unplaced keys %lld\n",
           P, k.C, f, ov, k.ix.S, k.ix.S * 16.0 / (1 << 20), k.ix.B, k.ix.B / 1024.0, k.ix.bad_keys);
    fflush(stdout);
  }
  auto scatter_run = [&](int v) {   // v: 0 = P16 ITEMS 4, 1 = P32 ITEMS 4, 2 = P32 ITEMS 8, 3 = P16 ITEMS 8
    Cut& k = cut[v == 1 || v == 2];
    PartDst d{};
    d.nparts = k.P; d.ncols = 2; d.src[0] = d_pk; d.src[1] = d_pv;
    for (int q = 0; q < k.P; q++) { d.dst[q][0] = k.key0; d.dst[q][1] = k.pv0; }
    d.dst_base = reinterpret_cast<long long*>(k.scr + TG_MAX_SLICES); d.capacity = k.C; d.overflow = k.scr + 2 * TG_MAX_SLICES;
    if (v == 0 || v == 1) scatter<4>(sms, nrows, d, k.scr, reinterpret_cast<long long*>(k.scr + TG_MAX_SLICES), k.scr + 2 * TG_MAX_SLICES, k.P, k.C);
    else scatter<8>(sms, nrows, d, k.scr, reinterpret_cast<long long*>(k.scr + TG_MAX_SLICES), k.scr + 2 * TG_MAX_SLICES, k.P, k.C);
  };
  // probe variants: 0 = P16 barrier kernel (the library with 16 slices), 1 = (a) P32 barrier kernel, one buffer,
  // 2 = (b) P32 library kernel, two buffers, 3 = P32 library kernel, one buffer, 4 = P16 library kernel, one buffer
  const int NV = 5;
  const char* pname[NV] = {"P16, barriers, 1 buffer (parent)", "(a) P32, barriers, 1 buffer", "(b) P32, library, 2 buffers",
                           "P32, library, 1 buffer", "P16, library, 1 buffer"};
  CK(cudaFuncSetAttribute(k_pidx_barrier<1, 2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 << 10));
  CK(cudaFuncSetAttribute(k_probe_inner_u1_seg_inplace_pidx<1, 2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 << 10));
  auto probe_run = [&](int v) {
    Cut& k = cut[v >= 1 && v <= 3];
    FastOut out{};
    out.n_pcols = 1; out.n_key_dst = 2; out.n_meta_dst = 1;
    out.psrc[0] = k.pv0; out.pdst[0] = k.pv0; out.key_dst[0] = k.key0; out.key_dst[1] = d_key1; out.meta_dst[0] = d_meta;
    const SegSpec sg{k.scr, (uint32_t)(k.C / 128), 0, k.C, nullptr, 0};
    const int64_t n = (int64_t)k.P * k.C;
    CK(cudaMemsetAsync(d_cur, 0, 8));
    SliceIndex si = k.si;
    if (v <= 1) { k_pidx_barrier<1, 2, 1><<<sms, 1024, si.B>>>(n, t, si, out, d_cur, sg, d_tc); return; }
    si.nbuf = v == 2 ? 2 : 1;
    k_probe_inner_u1_seg_inplace_pidx<1, 2, 1><<<sms, 1024, si.nbuf * (si.B + 8)>>>(n, t, si, out, d_cur, sg, d_tc);
  };
  // correctness: every variant matches every probe row and writes the build payload of the key at the row's position
  for (int v = 0; v < NV; v++) {
    Cut& k = cut[v >= 1 && v <= 3];
    CK(cudaMemset(d_meta, 0, 16 * cmax * 8)); CK(cudaMemset(d_key1, 0, 16 * cmax * 8));
    probe_run(v); CK(cudaDeviceSynchronize()); CK(cudaGetLastError());
    unsigned long long cur, fill[TG_MAX_SLICES];
    CK(cudaMemcpy(&cur, d_cur, 8, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(fill, k.scr, k.P * 8, cudaMemcpyDeviceToHost));
    std::vector<uint64_t> m(k.P * k.C), k0(k.P * k.C), k1(k.P * k.C);
    CK(cudaMemcpy(m.data(), d_meta, m.size() * 8, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(k0.data(), k.key0, m.size() * 8, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(k1.data(), d_key1, m.size() * 8, cudaMemcpyDeviceToHost));
    long long bad = 0, rows = 0;
    for (int p = 0; p < k.P; p++)
      for (unsigned long long i = 0; i < fill[p]; i++, rows++) {
        const size_t o = (size_t)p * k.C + i;
        bad += (m[o] * ODD != k0[o] * 7) | (k1[o] != k0[o]);
      }
    printf("%-36s rows %llu (want %lld, segment rows %lld), wrong rows %lld\n", pname[v], cur, (long long)np, rows, bad);
    fflush(stdout);
  }
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  auto timed = [&](auto&& fn, int nv, const char* const* names, const char* what) {
    std::vector<std::vector<float>> ms(nv);
    for (int v = 0; v < nv; v++) { fn(v); fn(v); }
    for (int it = 0; it < 30; it++)
      for (int v = 0; v < nv; v++) {
        CK(cudaEventRecord(e0)); fn(v); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        float x; CK(cudaEventElapsedTime(&x, e0, e1)); ms[v].push_back(x);
      }
    CK(cudaGetLastError());
    printf("\n%s, ms per launch, median of 30 alternating launches (min, max):\n", what);
    for (int v = 0; v < nv; v++) {
      std::sort(ms[v].begin(), ms[v].end());
      printf("  %-36s %.3f  (%.3f, %.3f)  %+.1f %%\n", names[v], ms[v][15], ms[v][0], ms[v][29], 100.0 * (ms[v][15] / ms[0][15] - 1));
    }
    fflush(stdout);
  };
  const char* sname[4] = {"P16, ITEMS 4 (parent)", "P32, ITEMS 4", "P32, ITEMS 8", "P16, ITEMS 8"};
  for (int round = 0; round < 2; round++) {
    timed(scatter_run, 4, sname, "k_partition_scatter_bulk<true,2,ITEMS> (k_segment_bases + scatter, 100 M rows, 2 columns)");
    timed(probe_run, NV, pname, "index probe <1,2,1> (100 M rows, 100 % match)");
  }
  return 0;
}

// ---- --scatter: the per-tile serial work of the L2 partition pass (DESIGN.md §4.1, "2048-row scatter tiles") ----------
// k_scatter_lab restates k_partition_scatter_bulk<true, 2, ITEMS, THREADS> for dense input and a capacity without spill,
// with STAGES input buffers and two switches.  RANK: a row's rank inside (tile, destination) comes from five warp ballots of its destination's bits (the
// lanes of the same destination, and in lane q the warp's rows for destination q, kept in a register) and one CTA scan over
// the per-warp counts, instead of one shared atomicAdd per row; the ranks are deterministic.  DBL: two staging buffers, so
// tile k+1 stages while the bulk stores of tile k still read (cp.async.bulk.wait_group.read 1 instead of 0).
template <int ITEMS, bool RANK, bool DBL, int THREADS = PT_BLOCK, int STAGES = 2>
__global__ void __launch_bounds__(THREADS)
k_scatter_lab(int64_t ntiles, PartDst d, unsigned long long* __restrict__ cursors) {
  constexpr int NC = 2, TILE = THREADS * ITEMS, SROWS = TILE + 2 * TG_MAX_SLICES, NW = THREADS / 32;
  constexpr int NBUF = DBL ? 2 : 1;
  static_assert(!RANK || THREADS == PT_BLOCK, "ballot ranks: 8 warps");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned long long* ring = reinterpret_cast<unsigned long long*>(smem_raw);      // [STAGES][NC][TILE]
  unsigned long long* stage0 = ring + (size_t)STAGES * NC * TILE;                  // [NBUF][NC][SROWS]
  uint64_t* full = reinterpret_cast<uint64_t*>(stage0 + (size_t)NBUF * NC * SROWS);
  __shared__ uint32_t s_cnt[TG_MAX_SLICES], s_off[TG_MAX_SLICES], s_len[TG_MAX_SLICES];
  __shared__ uint32_t s_w[NW][TG_MAX_SLICES];   // RANK: the warp's rows per destination, then the warp's first rank
  __shared__ unsigned long long s_gbase[TG_MAX_SLICES];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
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
    unsigned long long* stage = stage0 + (size_t)(DBL ? (it & 1) : 0) * NC * SROWS;
    if (!RANK && tid < TG_MAX_SLICES) s_cnt[tid] = 0;
    mbar_wait(&full[s], (uint32_t)((it / STAGES) & 1));
    __syncthreads();
    const unsigned long long* in = ring + (size_t)s * NC * TILE;
    uint32_t pr[ITEMS], wcnt = 0;   // wcnt (RANK): in lane q, this warp's rows for destination q so far
#pragma unroll
    for (int j = 0; j < ITEMS; j++) {
      const uint64_t h = hash64(in[j * THREADS + tid]);
      const uint32_t p = mulhi32((uint32_t)(h >> 32), P);
      if constexpr (RANK) {
        unsigned peers = 0xffffffffu, mine = 0xffffffffu;
#pragma unroll
        for (int b = 0; b < 5; b++) {
          const unsigned bal = __ballot_sync(0xffffffffu, (p >> b) & 1u);
          peers &= ((p >> b) & 1u) ? bal : ~bal;
          mine &= ((lane >> b) & 1) ? bal : ~bal;
        }
        const uint32_t before = __shfl_sync(0xffffffffu, wcnt, (int)p);
        pr[j] = (p << 16) | (before + __popc(peers & ((1u << lane) - 1)));
        wcnt += __popc(mine);
      } else {
        pr[j] = (p << 16) | atomicAdd(&s_cnt[p], 1u);
      }
    }
    if (RANK) s_w[warp][lane] = wcnt;
    __syncthreads();
    if (tid < 32) {
      uint32_t c = 0;
      if (tid < (int)P) {
        if constexpr (RANK) {
          for (int w = 0; w < NW; w++) { const uint32_t t = s_w[w][tid]; s_w[w][tid] = c; c += t; }
        } else c = s_cnt[tid];
      }
      uint32_t len = c;
      unsigned long long g = 0;
      if (tid < (int)P) {
        const unsigned long long old = c ? atomicAdd(&cursors[tid], (unsigned long long)c) : 0ull;
        const unsigned long long avail = old < (unsigned long long)d.capacity ? (unsigned long long)d.capacity - old : 0ull;
        if ((unsigned long long)c > avail) { len = (uint32_t)avail; *d.overflow = 1ull; }
        g = old + (unsigned long long)d.dst_base[tid];
      }
      uint32_t w = tid < (int)P ? (((uint32_t)(g & 1) + c + 1) & ~1u) : 0, incl = w;
      for (int o = 1; o < 32; o <<= 1) { uint32_t u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
      if (tid < (int)P) { s_off[tid] = incl - w + (uint32_t)(g & 1); s_gbase[tid] = g; s_len[tid] = len; }
    }
    if (tid < (int)P * NC) {
      if (DBL) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");   // the stores of tile k-2 have read this buffer
      else bulk_wait_read_all();
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < NC; c++) {
#pragma unroll
      for (int j = 0; j < ITEMS; j++) {
        const uint32_t p = pr[j] >> 16;
        stage[(size_t)c * SROWS + s_off[p] + (RANK ? s_w[warp][p] : 0u) + (pr[j] & 0xffffu)] = in[(size_t)c * TILE + j * THREADS + tid];
      }
    }
    fence_async_smem();
    __syncthreads();
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
    }
  }
  if (tid < (int)P * NC) bulk_wait_read_all();
}

// per segment, the sum of a mix of (key, payload) over its filled rows: equal sums = the same rows in every segment
static __global__ void k_seg_sum(const unsigned long long* key, const unsigned long long* pv, const unsigned long long* fill, long long C,
                                 int P, unsigned long long* out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (int64_t)P * C; i += (int64_t)gridDim.x * blockDim.x) {
    const int p = (int)(i / C);
    if (i - (int64_t)p * C < (int64_t)fill[p]) atomicAdd(&out[p], hash64(key[i] ^ (pv[i] * 0xD6E8FEB86659FD93ull)));
  }
}

static int scatter_gate() {
  const int64_t np = 100000000, nb = 10000000;
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  printf("card %s, %d SMs, L2 %d MiB\n", prop.name, sms, prop.l2CacheSize >> 20);
  // bench.py's probe columns: uniform build ids * ODD, payload the row
  std::vector<uint64_t> pk(np), pv(np);
  std::mt19937_64 rng(42);
  std::uniform_int_distribution<uint64_t> U(0, nb - 1);
  for (int64_t i = 0; i < np; i++) { pk[i] = U(rng) * ODD; pv[i] = (uint64_t)i; }
  const int64_t nrows = np / 2048 * 2048;   // whole tiles at ITEMS 4 and 8
  unsigned long long *d_pk, *d_pv, *d_c0, *d_c1, *d_key0, *d_pv0, *scr, *sum;
  const long long cmax = (long long)(np / 16 * 1.05) + 16384 + 128;
  CK(cudaMalloc(&d_pk, np * 8)); CK(cudaMalloc(&d_pv, np * 8)); CK(cudaMalloc(&d_c0, np * 8)); CK(cudaMalloc(&d_c1, np * 8));
  CK(cudaMalloc(&d_key0, 16 * cmax * 8)); CK(cudaMalloc(&d_pv0, 16 * cmax * 8));
  CK(cudaMalloc(&scr, (3 * TG_MAX_SLICES + 8) * 8)); CK(cudaMalloc(&sum, TG_MAX_SLICES * 8));
  CK(cudaMemcpy(d_pk, pk.data(), np * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(d_pv, pv.data(), np * 8, cudaMemcpyHostToDevice));
  unsigned long long* cursors = scr;
  long long* bases = reinterpret_cast<long long*>(scr + TG_MAX_SLICES);
  unsigned long long* flag = scr + 2 * TG_MAX_SLICES;
  const int NV = 13;
  const char* name[NV] = {"library ITEMS 4 (parent)", "library ITEMS 8", "lab ITEMS 8", "(a) ITEMS 8, ballot ranks",
                          "(b) ITEMS 8, 2 staging buffers", "(a)+(b) ITEMS 8", "(b) ITEMS 4, 2 staging buffers", "copy of the same bytes",
                          "(c) 512 threads x 4 (2048 rows)", "(c) 1024 threads x 2 (2048 rows)", "(d) ITEMS 8, 1-stage ring",
                          "(c)+(d) 512 x 4, 1-stage ring", "(c) 512 threads x 8 (4096 rows)"};
  auto lab = [&](auto kernel, int items, int nbuf, const PartDst& d, int threads = PT_BLOCK, int stages = 2) {
    const size_t tile = (size_t)threads * items;
    const size_t smem = (size_t)stages * 2 * tile * 8 + (size_t)nbuf * 2 * (tile + 2 * TG_MAX_SLICES) * 8 + 2 * 8 + 16;
    CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (size_t)(220 * 1024) / (smem + 1024)));   // launch_scatter_nc
    const int64_t ntiles = nrows / (int64_t)tile;
    kernel<<<(int)std::min<int64_t>(ntiles, (int64_t)sms * per_sm), threads, smem>>>(ntiles, d, cursors);
  };
  for (int P : {16, 32}) {
    const long long C0 = ((long long)((double)nrows / P * 1.05) + 16384 + 127) / 128 * 128;
    PartDst d{};
    d.nparts = P; d.ncols = 2; d.src[0] = d_pk; d.src[1] = d_pv;
    for (int q = 0; q < P; q++) { d.dst[q][0] = d_key0; d.dst[q][1] = d_pv0; }
    d.dst_base = bases; d.capacity = C0; d.overflow = flag;
    scatter<4>(sms, nrows, d, cursors, bases, flag, P, C0);
    unsigned long long fill[TG_MAX_SLICES];
    CK(cudaMemcpy(fill, cursors, P * 8, cudaMemcpyDeviceToHost));
    const double f = (double)*std::max_element(fill, fill + P);
    d.capacity = std::min(((long long)(f + 8.0 * std::sqrt(f)) + 4096 + 127) / 128 * 128, C0);   // inplace_seg_cap
    auto run = [&](int v) {
      if (v == 7) {
        CK(cudaMemcpyAsync(d_c0, d_pk, nrows * 8, cudaMemcpyDeviceToDevice)); CK(cudaMemcpyAsync(d_c1, d_pv, nrows * 8, cudaMemcpyDeviceToDevice));
        return;
      }
      if (v < 2) { (v ? scatter<8> : scatter<4>)(sms, nrows, d, cursors, bases, flag, P, d.capacity); return; }
      k_segment_bases<<<1, 32>>>(cursors, bases, flag, P, d.capacity);
      if (v == 2) lab(k_scatter_lab<8, false, false>, 8, 1, d);
      else if (v == 3) lab(k_scatter_lab<8, true, false>, 8, 1, d);
      else if (v == 4) lab(k_scatter_lab<8, false, true>, 8, 2, d);
      else if (v == 5) lab(k_scatter_lab<8, true, true>, 8, 2, d);
      else if (v == 6) lab(k_scatter_lab<4, false, true>, 4, 2, d);
      else if (v == 8) lab(k_scatter_lab<4, false, false, 512>, 4, 1, d, 512);
      else if (v == 9) lab(k_scatter_lab<2, false, false, 1024>, 2, 1, d, 1024);
      else if (v == 10) lab(k_scatter_lab<8, false, false, 256, 1>, 8, 1, d, 256, 1);
      else if (v == 11) lab(k_scatter_lab<4, false, false, 512, 1>, 4, 1, d, 512, 1);
      else lab(k_scatter_lab<8, false, false, 512>, 8, 1, d, 512);
    };
    // correctness: every variant leaves the same rows in every segment as the parent's kernel, and no overflow
    std::vector<unsigned long long> ref(P);
    for (int v = 0; v < NV; v++) {
      if (v == 7) continue;
      run(v);
      CK(cudaMemsetAsync(sum, 0, TG_MAX_SLICES * 8));
      k_seg_sum<<<sms * 8, 256>>>(d_key0, d_pv0, cursors, d.capacity, P, sum);
      CK(cudaDeviceSynchronize()); CK(cudaGetLastError());
      std::vector<unsigned long long> got(P), fl(P);
      unsigned long long ov = 0;
      CK(cudaMemcpy(got.data(), sum, P * 8, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(fl.data(), cursors, P * 8, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(&ov, flag, 8, cudaMemcpyDeviceToHost));
      if (v == 0) ref = got;
      unsigned long long rows = 0;
      for (int p = 0; p < P; p++) rows += fl[p];
      printf("P %d %-32s rows %llu (want %lld), overflow %llu, segments %s\n", P, name[v], rows, (long long)nrows, ov, got == ref ? "same" : "DIFFERENT");
    }
    fflush(stdout);
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    for (int round = 0; round < 2; round++) {
      std::vector<std::vector<float>> ms(NV);
      for (int v = 0; v < NV; v++) { run(v); run(v); }
      for (int it = 0; it < 30; it++)
        for (int v = 0; v < NV; v++) {
          CK(cudaEventRecord(e0)); run(v); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
          float x; CK(cudaEventElapsedTime(&x, e0, e1)); ms[v].push_back(x);
        }
      CK(cudaGetLastError());
      printf("\nP %d, round %d: %lld rows x 2 columns, ms per launch, median of 30 alternating launches (min, max), TB/s of 32 B/row:\n",
             P, round, (long long)nrows);
      for (int v = 0; v < NV; v++) {
        std::sort(ms[v].begin(), ms[v].end());
        printf("  %-32s %.3f  (%.3f, %.3f)  %.2f TB/s  %+.1f %%\n", name[v], ms[v][15], ms[v][0], ms[v][29],
               32.0 * nrows / (ms[v][15] * 1e-3) / 1e12, 100.0 * (ms[v][15] / ms[0][15] - 1));
      }
      fflush(stdout);
    }
  }
  return 0;
}

int main(int argc, char** argv) {
  if (argc > 1 && !strcmp(argv[1], "--slices")) return slices_gate();
  if (argc > 1 && !strcmp(argv[1], "--scatter")) return scatter_gate();
  if (argc > 1 && !strcmp(argv[1], "--host")) {
    if (argc == 4) host_stats({atof(argv[2])}, {atof(argv[3])});
    else host_stats({0.8, 0.85, 0.9}, {4.0, 5.0, 6.0});
    return 0;
  }
  std::vector<std::pair<double, double>> cfg;   // (ALPHA, LAMBDA) pairs from the command line
  for (int i = 1; i + 1 < argc; i += 2) cfg.push_back({atof(argv[i]), atof(argv[i + 1])});
  if (cfg.empty()) cfg = {{0.9, 2.0}, {0.8, 3.0}, {0.75, 4.0}};
  const int64_t nb = 10000000, np = 100000000;
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  printf("card %s, %d SMs, L2 %d MiB\n", prop.name, prop.multiProcessorCount, prop.l2CacheSize >> 20);
  std::vector<uint64_t> bk(nb), bv(nb);
  std::vector<uint64_t> ids(nb);
  std::iota(ids.begin(), ids.end(), 0);
  std::mt19937_64 rng(42);
  std::shuffle(ids.begin(), ids.end(), rng);
  for (int64_t i = 0; i < nb; i++) { bk[i] = ids[i] * ODD; bv[i] = ids[i] * 7; }
  // probe side: uniform ids, partition-ordered into P segments of capacity cap (learned-capacity slack)
  std::vector<std::vector<uint64_t>> seg(P);
  std::uniform_int_distribution<uint64_t> U(0, nb - 1);
  for (int64_t i = 0; i < np; i++) { const uint64_t k = U(rng) * ODD; seg[slot32(hash64(k), P)].push_back(k); }
  size_t mx = 0;
  for (auto& s : seg) mx = std::max(mx, s.size());
  const long long cap = ((long long)(mx + 8 * std::sqrt((double)mx)) + 4096 + 127) / 128 * 128;   // whole 128-row tiles
  const int64_t ntot = cap * P;
  std::vector<uint64_t> hk(ntot, 0), hcnt(P), hpv(ntot, 0);
  for (int p = 0; p < P; p++) {
    std::copy(seg[p].begin(), seg[p].end(), hk.begin() + p * cap);
    for (size_t i = 0; i < seg[p].size(); i++) hpv[p * cap + i] = p * cap + i;
    hcnt[p] = seg[p].size();
  }
  unsigned long long *d_bk, *d_bv, *d_key0, *d_key1, *d_meta, *d_pv, *d_cnt, *d_cur;
  uint32_t* d_tc;
  Slot *d_lp, *d_ix;
  uint8_t* d_pil;
  const unsigned long long nslots = (unsigned long long)(nb / 0.5 + 32) & ~3ull;
  CK(cudaMalloc(&d_bk, nb * 8)); CK(cudaMalloc(&d_bv, nb * 8));
  CK(cudaMalloc(&d_key0, ntot * 8)); CK(cudaMalloc(&d_key1, ntot * 8)); CK(cudaMalloc(&d_meta, ntot * 8)); CK(cudaMalloc(&d_pv, ntot * 8));
  CK(cudaMalloc(&d_cnt, P * 8)); CK(cudaMalloc(&d_cur, 8)); CK(cudaMalloc(&d_tc, ntot / 128 * 4));
  CK(cudaMalloc(&d_lp, (nslots + 2) * sizeof(Slot)));
  CK(cudaMemcpy(d_bk, bk.data(), nb * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(d_bv, bv.data(), nb * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_key0, hk.data(), ntot * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(d_pv, hpv.data(), ntot * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_cnt, hcnt.data(), P * 8, cudaMemcpyHostToDevice));
  k_table_init<<<(nslots + 256) / 256, 256>>>(d_lp, nslots + 2, nslots);
  k_lp_insert<<<(nb + 255) / 256, 256>>>(d_bk, d_bv, nb, d_lp, nslots);
  CK(cudaDeviceSynchronize());
  TableView t{d_lp, nslots, nullptr, 0, -1, TABLE_U1, 0};
  FastOut out{};
  out.n_pcols = 1; out.n_key_dst = 2; out.n_meta_dst = 1;
  out.psrc[0] = d_pv; out.pdst[0] = d_pv; out.key_dst[0] = d_key0; out.key_dst[1] = d_key1; out.meta_dst[0] = d_meta;
  SegSpec sg{d_cnt, (uint32_t)(cap / 128), 0, cap, nullptr, 0};
  int occ_a = 0, occ_g = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_a, k_probe_inner_u1_seg_inplace<1, 2, 1>, 256, 0));
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_g, k_pilot_gl, 256, 0));
  const int sms = prop.multiProcessorCount;
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (auto [alpha, lambda] : cfg) {
    Index ix = build_index(bk, bv, alpha, lambda, true);
    printf("\nindex: alpha %.2f lambda %.1f  S %u (%.2f MiB per slice)  B %u  unplaced buckets %lld keys %lld\n", alpha, lambda, ix.S,
           ix.S * 16.0 / (1 << 20), ix.B, ix.bad_buckets, ix.bad_keys);
    CK(cudaMalloc(&d_ix, ix.slots.size() * sizeof(Slot))); CK(cudaMalloc(&d_pil, ix.pilot.size()));
    CK(cudaMemcpy(d_ix, ix.slots.data(), ix.slots.size() * sizeof(Slot), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_pil, ix.pilot.data(), ix.pilot.size(), cudaMemcpyHostToDevice));
    PilotView pv{d_ix, d_pil, ix.S, ix.B, (uint32_t)P};
    const size_t smem = ix.B;
    const int nv = smem <= prop.sharedMemPerBlockOptin ? 3 : 2;   // the shared-memory variant needs the slice's pilots in one CTA
    if (nv == 3) CK(cudaFuncSetAttribute(k_pilot_sm<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    printf("resident CTAs per SM: (a) %d, (b/gl) %d, (b/sm) %s, %zu B of pilots per slice\n", occ_a, occ_g, nv == 3 ? "1 x 1024 threads" : "n/a", smem);
    auto run = [&](int v) {
      CK(cudaMemsetAsync(d_cur, 0, 8));
      if (v == 0) k_probe_inner_u1_seg_inplace<1, 2, 1><<<occ_a * sms, 256>>>(ntot, t, out, d_cur, sg, d_tc);
      else if (v == 1) k_pilot_gl<<<occ_g * sms, 256>>>(ntot, t, pv, out, d_cur, sg, d_tc);
      else k_pilot_sm<1024><<<sms, 1024, smem>>>(ntot, t, pv, out, d_cur, sg, d_tc);
    };
    const char* name[3] = {"(a) seg_inplace, linear probe, alpha 0.5", "(b) pilot index, pilots via L1", "(b) pilot index, pilots in smem"};
    // correctness: every variant matches every row and writes the same build payload
    for (int v = 0; v < nv; v++) {
      CK(cudaMemset(d_meta, 0, ntot * 8));
      CK(cudaMemcpy(d_key0, hk.data(), ntot * 8, cudaMemcpyHostToDevice));   // a variant with misses compacts the keys in place
      run(v); CK(cudaDeviceSynchronize()); CK(cudaGetLastError());
      unsigned long long cur; CK(cudaMemcpy(&cur, d_cur, 8, cudaMemcpyDeviceToHost));
      // a tile that takes the generic path is compacted in lane order, so rows may move within their tile: check each output
      // row's build payload against the key at the same position, and the keys as a multiset (sum and xor)
      std::vector<uint64_t> m(ntot), ko(ntot);
      CK(cudaMemcpy(m.data(), d_meta, ntot * 8, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(ko.data(), d_key0, ntot * 8, cudaMemcpyDeviceToHost));
      long long bad = 0;
      uint64_t s0 = 0, x0 = 0, s1 = 0, x1 = 0;
      for (int p = 0; p < P; p++)
        for (size_t i = 0; i < seg[p].size(); i++) {
          bad += m[p * cap + i] * ODD != ko[p * cap + i] * 7;
          s0 += seg[p][i]; x0 ^= seg[p][i] * 0x2545F4914F6CDD1Dull; s1 += ko[p * cap + i]; x1 ^= ko[p * cap + i] * 0x2545F4914F6CDD1Dull;
        }
      printf("%s: rows %llu (want %lld), wrong payloads %lld, keys %s\n", name[v], cur, (long long)np, bad,
             s0 == s1 && x0 == x1 ? "kept" : "CHANGED");
    }
    std::vector<float> ms[3];
    for (int r = 0; r < nv; r++) run(r);
    for (int it = 0; it < 30; it++)
      for (int v = 0; v < nv; v++) {
        CK(cudaEventRecord(e0)); run(v); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        float x; CK(cudaEventElapsedTime(&x, e0, e1)); ms[v].push_back(x);
      }
    for (int v = 0; v < nv; v++) {
      std::sort(ms[v].begin(), ms[v].end());
      printf("%-44s median %.3f ms  (min %.3f, max %.3f, 30 launches)", name[v], ms[v][15], ms[v][0], ms[v][29]);
      if (v) printf("  %+.1f %% against (a)", 100.0 * (ms[v][15] / ms[0][15] - 1));
      printf("\n");
    }
    fflush(stdout);
    CK(cudaFree(d_ix)); CK(cudaFree(d_pil));
  }
  return 0;
}
