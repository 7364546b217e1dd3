// str_dict.cu — the device string dictionaries of the hash aggregation (str_dict.cuh): the encode pass that turns a
// string GROUP BY column into ids, the growth of a dictionary, the copy of new entries' bytes into its arena, and the
// gather of a string result column from ids.
//
// Grouping key (codec.go HashGroupKey, collator.ImmutableKey): the bytes under binary (63) and utf8mb4_0900_bin (309),
// the bytes with trailing 0x20 cut under the PAD collations (46, 83, 65, 47).  Keys are equal only when their bytes
// are: the hash picks the slot, a byte comparison decides.
#include "str_dict.cuh"
#include "string.cuh"
#include "chunk_io.cuh"

namespace tg {

// 64-bit hash of a key: FNV-1a over the bytes, then a strong mix (the table takes its slot from the top bits)
__device__ __forceinline__ unsigned long long str_hash(const uint8_t* p, int64_t n) {
  unsigned long long h = 0xcbf29ce484222325ull;
  for (int64_t i = 0; i < n; i++) h = (h ^ p[i]) * 0x100000001b3ull;
  return mix64(h ^ (unsigned long long)n);
}

__device__ __forceinline__ bool bytes_eq(const uint8_t* a, const uint8_t* b, int64_t n) {
  for (int64_t i = 0; i < n; i++) if (a[i] != b[i]) return false;
  return true;
}

struct DictDev {
  unsigned long long* tbl;     // records {tag, id}
  unsigned long long nslots;
  unsigned long long* kptr;    // per id: key bytes (a batch buffer while the batch runs, then the arena)
  long long* klen;             // per id: key length
  long long* rlen;             // per id: raw length of the earliest row
  unsigned long long* first;   // per id: ordinal of the earliest row
  unsigned long long* ctr;
  unsigned long long id_cap;   // entries the per-id arrays hold
};
static DictDev dict_dev(StrDict& d) {
  return DictDev{d.tbl.as<unsigned long long>(), d.nslots, d.kptr.as<unsigned long long>(), d.klen.as<long long>(),
                 d.rlen.as<long long>(), d.first.as<unsigned long long>(), d.ctr.as<unsigned long long>(), (unsigned long long)d.id_cap};
}

// an ordered load through L2: a record's fields are written by other SMs during the pass, and a plain load may be
// hoisted above the wait for the record's tag
template <class T> __device__ __forceinline__ T vld(const T* p) { return *reinterpret_cast<const volatile T*>(p); }

// find-or-insert key (p, len) with hash h; returns its id, -1 when the probe runs past max_probe, -2 when a new entry
// finds the per-id arrays full (ctr[4] counts the entries taken or being taken; the host grows the arrays).  A found
// entry's earliest ordinal is lowered with atomicMin only when `ord` is below the value read.
__device__ long long dict_find_or_insert(const DictDev& d, const uint8_t* p, int64_t len, unsigned long long h,
                                         unsigned long long ord, uint32_t max_probe) {
  const unsigned long long ready = h | 3ull, busy = (h & ~3ull) | 1ull;
  uint32_t s = slot32(h, (uint32_t)d.nslots), steps = 0;
  for (;;) {
    unsigned long long* rec = d.tbl + 2 * (size_t)s;
    unsigned long long cur = vld(rec);
    if (cur == 0) {
      if (atomicAdd(&d.ctr[4], 1ull) >= d.id_cap) { atomicAdd(&d.ctr[4], ~0ull); return -2; }
      cur = atomicCAS(rec, 0ull, busy);
      if (cur != 0) atomicAdd(&d.ctr[4], ~0ull);   // another key took the slot: release the reservation
      if (cur == 0) {
        const unsigned long long id = atomicAdd(&d.ctr[0], 1ull);
        d.kptr[id] = (unsigned long long)p;
        d.klen[id] = len;
        d.first[id] = ord;
        rec[1] = id;
        __threadfence();
        *reinterpret_cast<volatile unsigned long long*>(rec) = ready;   // publish
        return (long long)id;
      }
    }
    if ((cur | 2ull) == ready) {
      while (cur != ready) cur = *reinterpret_cast<volatile unsigned long long*>(rec);
      const unsigned long long id = vld(rec + 1);
      if (vld(d.klen + id) == len && bytes_eq(p, reinterpret_cast<const uint8_t*>(vld(d.kptr + id)), len)) {
        if (ord < vld(d.first + id)) atomicMin(&d.first[id], ord);
        return (long long)id;
      }
    }
    if (++steps > max_probe) return -1;
    if (++s == (uint32_t)d.nslots) s = 0;
  }
}

// One lane per logical row, warps over 32 consecutive rows.  tails (when given): per row (ordinal << kTailBits) | the
// number of trailing 0x20 bytes the key cut (PAD only), the value a group's MIN keeps to find its earliest row's raw
// bytes; a count that does not fit kTailBits raises ctr[6].  __match_any_sync on the hash elects one lookup per distinct
// key per warp (the lowest lane, which has the warp's earliest row of that key); the other lanes of the key compare
// their bytes with the leader's and take its id, or look up on their own after a hash collision.
template <bool PAD>
__global__ void __launch_bounds__(256)
k_str_dict_encode(StrColDev c, int64_t n, unsigned long long ord0, DictDev d, uint32_t max_probe, long long* __restrict__ ids,
                  uint32_t* deferred, const uint32_t* only, unsigned long long* __restrict__ tails) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long my_deferred = 0, my_probe = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i - lane < n; i += stride) {
    const bool row = i < n && (!only || ((only[i >> 5] >> (i & 31)) & 1u));
    const bool want = row && (!c.nulls || bit_not_null(c.nulls, i));
    if (row && !want) ids[i] = 0;
    if (row && !want && tails) tails[i] = (ord0 + (unsigned long long)i) << kTailBits;
    const uint8_t* p = nullptr;
    int64_t len = 0;
    unsigned long long h = 0;
    if (want) {
      const int64_t o0 = c.offs[i];
      p = c.data - c.base + o0;
      len = c.offs[i + 1] - o0;
      const int64_t raw = len;
      if (PAD) len = str_trim_len(p, len);
      h = str_hash(p, len);
      if (tails) {
        const unsigned long long cut = (unsigned long long)(raw - len);
        if (cut >> kTailBits) atomicExch(&d.ctr[6], 1ull);
        tails[i] = ((ord0 + (unsigned long long)i) << kTailBits) | (cut & ((1ull << kTailBits) - 1));
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, h) & __ballot_sync(0xffffffffu, want);
    const int leader = want ? __ffs(peers) - 1 : lane;
    long long id = -1;
    if (want && lane == leader) id = dict_find_or_insert(d, p, len, h, ord0 + (unsigned long long)i, max_probe);
    const long long lid = __shfl_sync(0xffffffffu, id, leader);
    const unsigned long long lp = __shfl_sync(0xffffffffu, (unsigned long long)p, leader);
    const long long llen = __shfl_sync(0xffffffffu, (long long)len, leader);
    if (want && lane != leader) {
      if (llen == len && bytes_eq(p, reinterpret_cast<const uint8_t*>(lp), len)) id = lid;   // the leader's row is earlier
      else id = dict_find_or_insert(d, p, len, h, ord0 + (unsigned long long)i, max_probe);
    }
    if (want) {
      if (id < 0) { atomicOr(&deferred[i >> 5], 1u << (i & 31)); my_deferred++; my_probe += id == -1; }
      else ids[i] = id;
    }
  }
  for (int o = 16; o; o >>= 1) {
    my_deferred += __shfl_xor_sync(0xffffffffu, my_deferred, o);
    my_probe += __shfl_xor_sync(0xffffffffu, my_probe, o);
  }
  if (lane == 0 && my_deferred) atomicAdd(&d.ctr[1], my_deferred);
  if (lane == 0 && my_probe) atomicAdd(&d.ctr[5], my_probe);
}

// re-insert every record of an old table into a bigger one (tags are distinct keys: claim with the published tag)
__global__ void k_str_dict_rehash(const unsigned long long* __restrict__ oldt, unsigned long long old_slots, unsigned long long* newt,
                                  unsigned long long new_slots) {
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < old_slots; i += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long tag = oldt[2 * i];
    if (tag == 0) continue;
    uint32_t s = slot32(tag, (uint32_t)new_slots);
    while (atomicCAS(&newt[2 * (size_t)s], 0ull, tag) != 0ull) if (++s == (uint32_t)new_slots) s = 0;
    newt[2 * (size_t)s + 1] = oldt[2 * i + 1];
  }
}

// the row whose ordinal is its new entry's earliest (exactly one per entry) points the entry at its raw bytes and adds
// their length to ctr[2]
__global__ void k_str_dict_claim(StrColDev c, int64_t n, unsigned long long ord0, long long e0, DictDev d, const long long* __restrict__ ids) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (c.nulls && !bit_not_null(c.nulls, i)) continue;
    const long long id = ids[i];
    if (id < e0 || d.first[id] != ord0 + (unsigned long long)i) continue;
    const int64_t o0 = c.offs[i], raw = c.offs[i + 1] - o0;
    d.kptr[id] = (unsigned long long)(c.data - c.base + o0);
    d.rlen[id] = raw;
    atomicAdd(&d.ctr[2], (unsigned long long)raw);
  }
}

// a warp per new entry: its raw bytes → the arena at a cursor position, and the entry repointed there
__global__ void k_str_dict_copy(DictDev d, long long e0, long long e1, uint8_t* arena) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t id = e0 + ((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5); id < e1; id += nw) {
    const int64_t len = d.rlen[id];
    unsigned long long pos = 0;
    if (lane == 0) pos = atomicAdd(&d.ctr[3], (unsigned long long)len);
    pos = __shfl_sync(0xffffffffu, pos, 0);
    const uint8_t* src = reinterpret_cast<const uint8_t*>(d.kptr[id]);
    for (int64_t b = lane; b < len; b += 32) arena[pos + b] = src[b];
    __syncwarp();
    if (lane == 0) d.kptr[id] = (unsigned long long)(arena + pos);
  }
}

// entries [0, e) of a moved arena: pointers rebased
__global__ void k_str_dict_rebase(unsigned long long* kptr, long long e, unsigned long long old_base, unsigned long long new_base) {
  for (int64_t id = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; id < e; id += (int64_t)gridDim.x * blockDim.x)
    kptr[id] = kptr[id] - old_base + new_base;
}

// no_data: the column has no data pointer, so every row must be empty
__global__ void k_str_check_offsets(const int64_t* __restrict__ offs, int64_t n, bool no_data, unsigned int* flag) {
  const int64_t lo = offs[0], hi = offs[n];
  bool bad = false;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o0 = offs[r], o1 = offs[r + 1];
    bad |= o0 > o1 || o0 < lo || o1 > hi || (no_data && o1 > o0);
  }
  if (bad) *flag = 1u;
}

void str_check_offsets(const int64_t* offs, const uint8_t* data, int64_t n, unsigned int* flag, int nsm, cudaStream_t s) {
  k_str_check_offsets<<<grid_size(nsm, n, 256, 8), 256, 0, s>>>(offs, n, data == nullptr, flag);
}

// ---- result column: lengths, an exclusive scan in blocks of kScanItems, bytes ----------------------------------------
static constexpr int kScanItems = 1024;   // 256 threads x 4 items

// a result row's length: its entry's raw bytes, or with tails the key bytes plus the group's own trailing spaces
__device__ __forceinline__ int64_t result_len(const DictDev& d, long long id, const unsigned long long* tails, int64_t r) {
  return tails ? d.klen[id] + (int64_t)(tails[r] & ((1ull << kTailBits) - 1)) : d.rlen[id];
}

__global__ void __launch_bounds__(256) k_str_lens(DictDev d, const long long* __restrict__ ids, const uint8_t* __restrict__ valid,
                                                  const unsigned long long* __restrict__ tails, int64_t rows, long long* lens) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x)
    lens[r] = (!valid || valid[r]) ? result_len(d, ids[r], tails, r) : 0;
}

// exclusive scan of the 256 threads' values of a block; *total = the block's sum
__device__ __forceinline__ long long block_exclusive(long long v, long long* total) {
  __shared__ long long s_w[8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  long long x = v;
  for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) s_w[w] = x;
  __syncthreads();
  long long before = 0, all = 0;
  for (int j = 0; j < 8; j++) { if (j < w) before += s_w[j]; all += s_w[j]; }
  __syncthreads();
  *total = all;
  return before + x - v;
}

__global__ void __launch_bounds__(256) k_scan_sums(const long long* __restrict__ lens, int64_t rows, long long* bsum) {
  const int64_t b0 = (int64_t)blockIdx.x * kScanItems + threadIdx.x * 4;
  long long s = 0;
  for (int j = 0; j < 4; j++) if (b0 + j < rows) s += lens[b0 + j];
  long long total;
  block_exclusive(s, &total);
  if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

// one block: bsum → its exclusive scan, in place, carried across passes of 256 entries
__global__ void __launch_bounds__(256) k_scan_carry(long long* bsum, int64_t nb) {
  long long carry = 0;
  for (int64_t b0 = 0; b0 < nb; b0 += 256) {
    const int64_t b = b0 + threadIdx.x;
    const long long v = b < nb ? bsum[b] : 0;
    long long total;
    const long long ex = block_exclusive(v, &total);
    if (b < nb) bsum[b] = carry + ex;
    carry += total;
  }
}

__global__ void __launch_bounds__(256) k_scan_out(const long long* __restrict__ lens, int64_t rows, const long long* __restrict__ bsum, long long* offs) {
  const int64_t b0 = (int64_t)blockIdx.x * kScanItems + threadIdx.x * 4;
  long long v[4], s = 0;
  for (int j = 0; j < 4; j++) { v[j] = b0 + j < rows ? lens[b0 + j] : 0; s += v[j]; }
  long long total;
  long long at = bsum[blockIdx.x] + block_exclusive(s, &total);
  if (blockIdx.x == 0 && threadIdx.x == 0) offs[0] = 0;
  for (int j = 0; j < 4; j++) { at += v[j]; if (b0 + j < rows) offs[b0 + j + 1] = at; }
}

// a warp per result row: its entry's raw bytes at offs[r]
__global__ void k_str_gather(DictDev d, const long long* __restrict__ ids, const uint8_t* __restrict__ valid,
                             const unsigned long long* __restrict__ tails, int64_t rows, const long long* __restrict__ offs, uint8_t* out) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < rows; r += nw) {
    if (valid && !valid[r]) continue;
    const long long id = ids[r];
    const uint8_t* src = reinterpret_cast<const uint8_t*>(d.kptr[id]);
    const int64_t at = offs[r], len = offs[r + 1] - at, keep = tails ? d.klen[id] : len;   // then the group's own spaces
    for (int64_t b = lane; b < len; b += 32) out[at + b] = b < keep ? src[b] : (uint8_t)0x20;
  }
}

// ---- host side -------------------------------------------------------------------------------------------------------
static int read_counters(StrDict& d, unsigned long long (&back)[8], cudaStream_t s) {
  TG_CUDA(cudaMemcpyAsync(back, d.ctr.p, 64, cudaMemcpyDeviceToHost, s));
  TG_CUDA(cudaStreamSynchronize(s));
  return TG_OK;
}

static int alloc_dict_table(StrDict& d, DevBuf& mem, unsigned long long nslots, int device, cudaStream_t s) {
  if (nslots >= (1ull << 32)) return fail(TG_ERR_OOM, "a string dictionary would need 2^32 slots or more");
  TG_TRY(mem.ensure(device, (size_t)nslots * 16));
  TG_CUDA(cudaMemsetAsync(mem.p, 0, (size_t)nslots * 16, s));
  return TG_OK;
}

// the per-id arrays with room for `cap` entries, the first `used` kept
static int grow_ids(StrDict& d, size_t cap, size_t used, int device, cudaStream_t s) {
  if (cap <= d.id_cap) return TG_OK;
  TG_TRY(d.kptr.ensure_preserve(device, cap * 8, used * 8, s));
  TG_TRY(d.klen.ensure_preserve(device, cap * 8, used * 8, s));
  TG_TRY(d.rlen.ensure_preserve(device, cap * 8, used * 8, s));
  TG_TRY(d.first.ensure_preserve(device, cap * 8, used * 8, s));
  d.id_cap = cap;
  return TG_OK;
}

int str_dict_prepare(StrDict& d, int device, int64_t n, int64_t expected_groups, cudaStream_t s) {
  if (d.nslots == 0) {
    unsigned long long want = std::max<unsigned long long>(1024, (unsigned long long)std::min<int64_t>(n, 1ll << 22) * 2);
    if (expected_groups > 0) want = std::min<unsigned long long>(want, std::max<unsigned long long>(1024, (unsigned long long)expected_groups * 2));
    TG_TRY(alloc_dict_table(d, d.tbl, want, device, s));
    d.nslots = want;
    TG_TRY(d.ctr.ensure(device, 64));
    TG_CUDA(cudaMemsetAsync(d.ctr.p, 0, 64, s));
  }
  // the per-id arrays start at half the table's slots and grow when a round defers new entries for want of room
  // (str_dict_grow), so they follow the number of entries, not the rows pushed
  if (d.id_cap < (size_t)d.entries + 1024) TG_TRY(grow_ids(d, std::max<size_t>((size_t)d.nslots / 2, (size_t)d.entries + 1024), d.entries, device, s));
  TG_CUDA(cudaMemsetAsync(d.ctr.as<unsigned long long>() + 6, 0, 8, s));
  return TG_OK;
}

int str_dict_round(StrDict& d, const StrColDev& c, int64_t n, int64_t ord0, uint32_t max_probe, long long* ids, uint32_t* deferred,
                   const uint32_t* only, unsigned long long& nd, unsigned long long* tails, int nsm, cudaStream_t s) {
  TG_CUDA(cudaMemsetAsync(d.ctr.as<unsigned long long>() + 1, 0, 8, s));
  TG_CUDA(cudaMemsetAsync(d.ctr.as<unsigned long long>() + 5, 0, 8, s));
  const int grid = grid_size(nsm, n, 256, 8);
  if (d.coll == COLL_PAD_BIN) k_str_dict_encode<true><<<grid, 256, 0, s>>>(c, n, (unsigned long long)ord0, dict_dev(d), max_probe, ids, deferred, only, tails);
  else k_str_dict_encode<false><<<grid, 256, 0, s>>>(c, n, (unsigned long long)ord0, dict_dev(d), max_probe, ids, deferred, only, tails);
  d.launches++;
  unsigned long long back[8];
  TG_TRY(read_counters(d, back, s));
  nd = back[1];
  return TG_OK;
}

int str_dict_tail_overflow(StrDict& d, bool& overflow, cudaStream_t s) {
  unsigned long long back[8];
  TG_TRY(read_counters(d, back, s));
  overflow = back[6] != 0;
  return TG_OK;
}

int str_dict_used(StrDict& d, unsigned long long& used, cudaStream_t s) {
  unsigned long long back[8];
  TG_TRY(read_counters(d, back, s));
  used = back[0];
  return TG_OK;
}

int str_dict_grow(StrDict& d, unsigned long long more, bool room, int device, int nsm, cudaStream_t s) {
  unsigned long long back[8];
  TG_TRY(read_counters(d, back, s));
  // entries deferred for want of per-id room: x4 arrays (the new entries of this batch, ctr[0], are kept)
  if (back[1] > back[5]) TG_TRY(grow_ids(d, std::max<size_t>(d.id_cap * 4, (size_t)back[0] + 1024), (size_t)back[0], device, s));
  if (back[5] == 0 || room) return TG_OK;   // no probe ran past its limit, or one did in a table with room
  // x4, or more: at most half full once `more` new entries join
  const unsigned long long want = std::max<unsigned long long>(d.nslots * 4, (back[0] + more) * 2);
  DevBuf nm;
  TG_TRY(alloc_dict_table(d, nm, want, device, s));
  k_str_dict_rehash<<<grid_size(nsm, (int64_t)d.nslots, 256, 8), 256, 0, s>>>(d.tbl.as<unsigned long long>(), d.nslots, nm.as<unsigned long long>(), want);
  d.launches++;
  TG_CUDA(cudaStreamSynchronize(s));
  std::swap(d.tbl.p, nm.p); std::swap(d.tbl.cap, nm.cap); std::swap(d.tbl.device, nm.device);
  d.nslots = want;
  d.grows++;
  return TG_OK;
}

int str_dict_commit(StrDict& d, const StrColDev& c, const long long* ids, int64_t n, int64_t ord0, int device, int nsm, cudaStream_t s) {
  unsigned long long* ctr = d.ctr.as<unsigned long long>();
  unsigned long long back[8];
  TG_TRY(read_counters(d, back, s));
  const long long e0 = d.entries, e1 = (long long)back[0];
  if (e1 == e0) return TG_OK;
  TG_CUDA(cudaMemsetAsync(ctr + 2, 0, 8, s));
  k_str_dict_claim<<<grid_size(nsm, n, 256, 8), 256, 0, s>>>(c, n, (unsigned long long)ord0, e0, dict_dev(d), ids);
  d.launches++;
  TG_TRY(read_counters(d, back, s));
  const size_t add = (size_t)back[2];
  if (d.arena_used + add + 16 > d.arena.cap) {
    const unsigned long long old_base = (unsigned long long)d.arena.p;
    TG_TRY(d.arena.ensure_preserve(device, d.arena_used + add + 16, d.arena_used, s));
    if (e0 && old_base) {
      k_str_dict_rebase<<<grid_size(nsm, e0, 256, 8), 256, 0, s>>>(d.kptr.as<unsigned long long>(), e0, old_base, (unsigned long long)d.arena.p);
      d.launches++;
    }
  }
  const unsigned long long cursor = d.arena_used;
  TG_CUDA(cudaMemcpyAsync(ctr + 3, &cursor, 8, cudaMemcpyHostToDevice, s));
  k_str_dict_copy<<<grid_size(nsm, (e1 - e0) * 32, 256, 8), 256, 0, s>>>(dict_dev(d), e0, e1, d.arena.as<uint8_t>());
  d.launches++;
  TG_CUDA(cudaStreamSynchronize(s));
  d.arena_used += add;
  d.entries = e1;
  return TG_OK;
}

int str_dict_gather(const StrDict& d, const long long* ids, const uint8_t* valid, const unsigned long long* tails, int64_t rows, DevBuf& offs, DevBuf& bytes,
                    int64_t* total, int device, int nsm, cudaStream_t s) {
  const DictDev dd = dict_dev(const_cast<StrDict&>(d));
  TG_TRY(offs.ensure(device, (size_t)(rows + 1) * 8 + 16));
  *total = 0;
  if (rows == 0) {
    TG_CUDA(cudaMemsetAsync(offs.p, 0, 8, s));
    TG_TRY(bytes.ensure(device, 16));
    return TG_OK;
  }
  const int64_t nb = (rows + kScanItems - 1) / kScanItems;
  DevBuf lens, bsum;
  TG_TRY(lens.ensure(device, (size_t)rows * 8 + 16));
  TG_TRY(bsum.ensure(device, (size_t)nb * 8 + 16));
  k_str_lens<<<grid_size(nsm, rows, 256, 8), 256, 0, s>>>(dd, ids, valid, tails, rows, lens.as<long long>());
  k_scan_sums<<<(unsigned)nb, 256, 0, s>>>(lens.as<long long>(), rows, bsum.as<long long>());
  k_scan_carry<<<1, 256, 0, s>>>(bsum.as<long long>(), nb);
  k_scan_out<<<(unsigned)nb, 256, 0, s>>>(lens.as<long long>(), rows, bsum.as<long long>(), offs.as<long long>());
  TG_CUDA(cudaMemcpyAsync(total, offs.as<long long>() + rows, 8, cudaMemcpyDeviceToHost, s));
  TG_CUDA(cudaStreamSynchronize(s));
  TG_TRY(bytes.ensure(device, (size_t)*total + 16));
  k_str_gather<<<grid_size(nsm, rows * 32, 256, 8), 256, 0, s>>>(dd, ids, valid, tails, rows, offs.as<long long>(), bytes.as<uint8_t>());
  TG_CUDA(cudaStreamSynchronize(s));
  TG_CUDA(cudaGetLastError());
  return TG_OK;
}

}  // namespace tg
