// join_kernels.cuh — hash-join build / probe kernels for sm_90a.
//
// What they replace in the reference (pkg/executor/join):
//   build : rowTableBuilder.processOneChunk (row_table_builder.go:138) + subTable.build
//           (hash_table_v2.go:107)                                   → k_table_init, k_build_insert,
//                                                                      k_table_stats, k_table_assign,
//                                                                      k_build_scatter_u1 / _rows
//   probe : baseJoinProbe.SetChunkForProbe (base_join_probe.go:179) + innerJoinProbe.Probe
//           (inner_join_probe.go:27) + append{Build,Probe}RowToChunkInternal (:589/:677)
//                                                                    → k_probe_inner_u1_seg_lean / k_probe_inner_u1_w
//                                                                      (fused fast path), k_probe_inner_uq (unique
//                                                                      keys, one pass), k_probe_count / k_probe_write
//
// Data layout in HBM (GPU-first, not the reference's chained row pointers):
//   * open-addressing table of 16-byte slots {int64 key, u64 meta}, linear probing, one slot per
//     DISTINCT key; any table size (multiply-high range reduction), one extra slot at index nslots
//     for the key whose value equals the empty sentinel.
//   * mode U1 (unique build keys, ≤1 eight-byte NOT NULL build payload): meta = payload.  A probe is ONE
//     16-byte gather — no dependent pointer chase.
//   * mode G  (anything else): meta = (offset << 28) | count into a row-major "row store" where the
//     rows of one key are contiguous (count-then-place build, O(n) for any duplicate skew).
#pragma once
#include "common.cuh"
#include "tma.cuh"

namespace tg {

struct __align__(16) Slot { int64_t key; unsigned long long meta; };

static const uint32_t kInvalidSlot = 0xFFFFFFFFu;
static const unsigned long long kCntMask = (1ull << 28) - 1;

enum { TABLE_NONE = 0, TABLE_U1 = 1, TABLE_G = 2 };
enum { KEY_I64 = 0, KEY_F64 = 1, KEY_F32 = 2, KEY_TIME = 3 };
enum { SRC_PROBE_COL = 0, SRC_BUILD_KEY = 1, SRC_BUILD_META = 2, SRC_BUILD_WORD = 3, SRC_FLAG = 4 };

struct KeySpec {
  const void* data;
  const uint8_t* nulls;      // bitmap, nullptr = no NULLs
  int32_t kind;              // KEY_*
  int32_t reject_negative;   // mixed signed/unsigned key pair, this side is the signed one: a negative
                             // value carries intFlag and can never match (codec.go:647-653)
};

struct TableView {
  Slot* slots;
  unsigned long long nslots;        // regular slots; slot[nslots] belongs to key == kEmptyKey
  const unsigned long long* rows;   // row store (mode G)
  int32_t row_words;
  int32_t null_word;                // index of the per-row NULL mask word in the row store, -1 = none
  int32_t mode;
  int32_t pad;
};

// A key's home is the first slot of an aligned group of kHomeWidth slots (nslots is a multiple of it), so its first two
// 32-byte pairs lie in one 64-byte half-line.  4 beat homes of one 32-byte pair at every load factor measured (DESIGN.md §4.1).
static constexpr int kHomeWidth = 4;

// home slot of a hash value: slot32(h, nslots / w) * w, which equals slot32(h, nslots) rounded down to a multiple of w
// because nslots is one.  Linear probing runs on from there one slot at a time.
__device__ __forceinline__ uint32_t home_slot(unsigned long long h, unsigned long long nslots) {
  return slot32(h, (uint32_t)nslots) & ~(uint32_t)(kHomeWidth - 1);
}

#define TG_MAX_OUT 24
struct OutSpec {
  int32_t src;        // SRC_*
  int32_t idx;        // probe column index | row-store word
  int32_t elem_len;   // 4 or 8
  int32_t null_bit;   // SRC_BUILD_WORD: bit in the null word, -1 = never NULL
};
struct OutCols {
  int32_t n;
  int32_t pad;
  OutSpec spec[TG_MAX_OUT];
  void* data[TG_MAX_OUT];
  uint8_t* valid[TG_MAX_OUT];   // one byte per output row (1 = NOT NULL), nullptr when the column cannot be NULL
};

// row store build description
struct RowSpec {
  int32_t nwords;
  int32_t null_word;            // -1 = none
  int32_t col[TG_MAX_COLS];     // build column feeding word w
  int32_t elem_len[TG_MAX_COLS];
  int32_t null_bit[TG_MAX_COLS];
};

// OtherCondition compiled for the probe kernels: operands are probe columns, words of the build row store, or a constant
enum { OSRC_PROBE = 0, OSRC_BUILD = 1, OSRC_CONST = 2 };
#define TG_MAX_OTHER 8
struct OtherItemDev {
  int32_t op, is_real;
  int32_t l_src, l_idx, l_null_bit, l_unsigned;
  int32_t r_src, r_idx, r_null_bit, r_unsigned;
  int64_t const_i64;
  double const_f64;
};
struct DevOther { int32_t n, pad; OtherItemDev it[TG_MAX_OTHER]; };

// join kinds as the probe kernels see them
enum {
  PK_INNER = 0,            // emit cnt rows per probe row (also outer join whose OUTER side is the build side)
  PK_PROBE_OUTER = 1,      // emit max(cnt,1) rows, NULL-padded build side when unmatched
  PK_SEMI = 2,             // probe is the left side: emit 1 row iff matched
  PK_ANTI = 3,             // emit 1 row iff not matched
  PK_LEFT_OUTER_SEMI = 4,  // emit 1 row + flag
  PK_ANTI_LEFT_OUTER_SEMI = 5,
  PK_MARK_ONLY = 6         // build is the left side of a semi/anti join: only mark used slots
};

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool load_key(const KeySpec& ks, int64_t row, int64_t& k) {
  if (ks.nulls && !bit_not_null(ks.nulls, row)) return false;
  if (ks.kind == KEY_I64) {
    k = reinterpret_cast<const int64_t*>(ks.data)[row];
    if (ks.reject_negative && k < 0) return false;
  } else if (ks.kind == KEY_TIME) {
    // DATE / DATETIME / TIMESTAMP keys are serialized as Time.ToPackedUint (codec.go:697-707, types/time.go:646): a function
    // of the calendar fields only.  The CoreTime bit fields above the 4 fspTt bits (types/time.go:235-251) carry exactly those
    // fields, so equal packed values <=> equal masked words; the type / fsp bits never take part in a key comparison.
    k = reinterpret_cast<const int64_t*>(ks.data)[row] & ~(int64_t)0xF;
  } else {
    double d = ks.kind == KEY_F64 ? reinterpret_cast<const double*>(ks.data)[row]
                                  : (double)reinterpret_cast<const float*>(ks.data)[row];
    if (d == 0) d = 0;   // -0 → +0 (codec.go:663-667, :676-682)
    k = __double_as_longlong(d);
  }
  return true;
}

__device__ __forceinline__ Slot load_slot(const Slot* p) {
  // one 128-bit gather
  const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(p);
  Slot s; s.key = (int64_t)v.x; s.meta = v.y;
  return s;
}

// both slots of a 32-byte home pair: two back-to-back 128-bit loads (128 bits is the widest load sm_90 has) of the same
// 32-byte sector, so the pair still costs one sector fetch; p must be 32-byte aligned
__device__ __forceinline__ void load_pair(const Slot* p, Slot& a, Slot& b) {
  unsigned long long x0, x1, x2, x3;
  asm volatile("ld.global.v2.u64 {%0, %1}, [%2];" : "=l"(x0), "=l"(x1) : "l"(p));
  asm volatile("ld.global.v2.u64 {%0, %1}, [%2+16];" : "=l"(x2), "=l"(x3) : "l"(p));
  a.key = (int64_t)x0; a.meta = x1; b.key = (int64_t)x2; b.meta = x3;
}

// continue the linear probe for key k (not the sentinel) at slot s: one slot if s is odd, then by aligned 32-byte pairs
// (nslots is even, so pairs wrap exactly at the end), until the slot holding k or the first empty slot.  true iff found.
__device__ __forceinline__ bool probe_run(const Slot* __restrict__ slots, unsigned long long nslots, int64_t k, unsigned long long s,
                                       unsigned long long& meta) {
  if (s >= nslots) s = 0;
  if (s & 1) {
    const Slot x = load_slot(slots + s);
    if (x.key == k) { meta = x.meta; return true; }
    if (x.key == kEmptyKey) return false;
    if (++s == nslots) s = 0;
  }
  for (;;) {
    Slot a, b;
    load_pair(slots + s, a, b);
    if (a.key == k) { meta = a.meta; return true; }
    if (a.key == kEmptyKey) return false;
    if (b.key == k) { meta = b.meta; return true; }
    if (b.key == kEmptyKey) return false;
    s += 2;
    if (s == nslots) s = 0;
  }
}

// lookup without insertion: returns slot index or kInvalidSlot; meta of the found slot in *meta
__device__ __forceinline__ uint32_t table_find(const TableView& t, int64_t k, unsigned long long* meta) {
  if (k == kEmptyKey) {
    Slot s = load_slot(t.slots + t.nslots);
    *meta = s.meta;
    // the side slot is "occupied" iff a build row carried this key: mode U1 marks that in key
    return s.key == 0 ? kInvalidSlot : (uint32_t)t.nslots;
  }
  unsigned long long s = home_slot(hash64((uint64_t)k), t.nslots);
  for (;;) {
    Slot v = load_slot(t.slots + s);
    if (v.key == k) { *meta = v.meta; return (uint32_t)s; }
    if (v.key == kEmptyKey) return kInvalidSlot;
    if (++s == t.nslots) s = 0;
  }
}

// ---------------------------------------------------------------------------------------------
// several equal conditions (join keys): FixedSerializedKey mode of the reference (join_table_meta.go:174-178: every key
// column fixed width → codec.SerializeKeys codec.go:822 concatenates them; a row with a NULL in ANY key column has no key,
// hash_join_v2.go / preAllocForSerializedKeyBuffer :429-447).  Here the serialized key is replaced by ONE 64-bit candidate
// key = a mix of the key column values, written with its own NOT-NULL bitmap by this pre-pass; the table and every probe
// kernel then run unchanged on that synthetic int64 column, and the exact equality of every key column is re-checked on each
// candidate pair by residual `left_key_i = right_key_i` items the host appends to OtherCondition (a 64-bit collision can
// create a candidate pair, never a result row).  reject[c]: mixed signed / unsigned pair and this side is the signed one —
// a negative value can never equal an unsigned one (NeedSignFlag, join_table_meta.go:296-303), the row has no key.
// ---------------------------------------------------------------------------------------------
#define TG_MAX_JOIN_KEYS 4
struct MultiKeySrc {
  int32_t nk, pad;
  const int64_t* data[TG_MAX_JOIN_KEYS];
  const uint8_t* nulls[TG_MAX_JOIN_KEYS];
  int32_t reject[TG_MAX_JOIN_KEYS];
};
__global__ void __launch_bounds__(256)
k_composite_key(MultiKeySrc src, int64_t n, int64_t* __restrict__ out_key, uint32_t* __restrict__ out_not_null) {
  // whole warps stride over 32-row groups; lane 0 stores the group's 32 NOT-NULL bits (LSB = first row, chunk.Column layout)
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t groups = (n + 31) >> 5;
  for (int64_t g = warp; g < groups; g += nwarps) {
    const int64_t i = (g << 5) + lane;
    bool valid = i < n;
    uint64_t h = 0;
    if (valid) {
      for (int c = 0; c < src.nk; c++) {
        if (src.nulls[c] && !bit_not_null(src.nulls[c], i)) { valid = false; break; }
        const int64_t v = src.data[c][i];
        if (src.reject[c] && v < 0) { valid = false; break; }
        if (c == 0) h = (uint64_t)v;
        else {   // splitmix-style finalizer of the running value (a bijection), then the next column folded in by an odd multiply
          h ^= h >> 30; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 27; h *= 0x94D049BB133111EBull; h ^= h >> 31;
          h += (uint64_t)v * 0x9E3779B97F4A7C15ull + (uint64_t)c;
        }
      }
      if (valid) out_key[i] = (int64_t)h; else out_key[i] = 0;
    }
    const unsigned bits = __ballot_sync(0xffffffffu, valid);
    if (lane == 0) out_not_null[g] = bits;
  }
}

// ---------------------------------------------------------------------------------------------
// build
// ---------------------------------------------------------------------------------------------
__global__ void k_table_init(Slot* slots, unsigned long long n_total, unsigned long long nslots) {
  unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (; i < n_total; i += stride) {
    Slot s; s.key = (i == nslots) ? 0 : kEmptyKey; s.meta = 0;   // side slot: key field = occupied flag
    *reinterpret_cast<ulonglong2*>(slots + i) = make_ulonglong2((unsigned long long)s.key, 0ull);
  }
}

// pass 1: claim one slot per distinct key, count multiplicities, remember (slot, rank) per build row
__global__ void __launch_bounds__(256)
k_build_insert(KeySpec key, DevCols cols, DevFilter filt, int64_t n, Slot* slots, unsigned long long nslots,
               uint32_t* __restrict__ row_slot, uint32_t* __restrict__ row_rank) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    int64_t k;
    bool valid = load_key(key, i, k);
    if (valid && filt.n) valid = eval_filter(filt, cols, i);
    if (!valid) { row_slot[i] = kInvalidSlot; row_rank[i] = 0; continue; }
    unsigned long long s;
    if (k == kEmptyKey) {
      s = nslots;
      slots[s].key = 1;   // occupied flag (benign race: every writer stores 1)
    } else {
      s = home_slot(hash64((uint64_t)k), nslots);
      for (;;) {
        int64_t cur = *reinterpret_cast<volatile int64_t*>(&slots[s].key);
        if (cur == k) break;
        if (cur == kEmptyKey) {
          unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(&slots[s].key),
                                             (unsigned long long)kEmptyKey, (unsigned long long)k);
          if (old == (unsigned long long)kEmptyKey || old == (unsigned long long)k) break;
        }
        if (++s == nslots) s = 0;
      }
    }
    unsigned long long rank = atomicAdd(&slots[s].meta, 1ull);
    row_slot[i] = (uint32_t)s;
    row_rank[i] = (uint32_t)rank;
  }
}

// pass 2: distinct keys, largest multiplicity
__global__ void k_table_stats(const Slot* slots, unsigned long long n_total, unsigned long long* distinct,
                              unsigned long long* maxcnt) {
  unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  unsigned long long d = 0, m = 0;
  for (; i < n_total; i += stride) {
    unsigned long long c = slots[i].meta;
    d += c != 0;
    m = c > m ? c : m;
  }
  for (int o = 16; o; o >>= 1) {
    d += __shfl_xor_sync(0xffffffffu, d, o);
    unsigned long long mo = __shfl_xor_sync(0xffffffffu, m, o);
    m = mo > m ? mo : m;
  }
  if ((threadIdx.x & 31) == 0) {
    if (d) atomicAdd(distinct, d);
    if (m) atomicMax(maxcnt, m);
  }
}

// pass 3 (mode G): give every occupied slot a contiguous range of the row store
__global__ void k_table_assign(Slot* slots, unsigned long long n_total, unsigned long long* cursor) {
  unsigned long long base = blockIdx.x * (unsigned long long)blockDim.x;
  unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  for (; base < n_total; base += stride) {   // warp-uniform trip count
    unsigned long long i = base + threadIdx.x;
    unsigned long long c = i < n_total ? slots[i].meta : 0;
    unsigned long long incl = c;
    for (int o = 1; o < 32; o <<= 1) {
      unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);
    unsigned long long wbase = 0;
    if (lane == 31 && total) wbase = atomicAdd(cursor, total);
    wbase = __shfl_sync(0xffffffffu, wbase, 31);
    if (c) slots[i].meta = ((wbase + incl - c) << 28) | c;
  }
}

// pass 4a (mode U1): meta = the single payload of the key
__global__ void k_build_scatter_u1(const uint32_t* __restrict__ row_slot, const unsigned long long* __restrict__ payload,
                                   int64_t n, Slot* slots) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    uint32_t s = row_slot[i];
    if (s != kInvalidSlot) slots[s].meta = payload ? payload[i] : 0ull;
  }
}

// pass 4b (mode G): column → row conversion into the key-grouped row store
__global__ void k_build_scatter_rows(const uint32_t* __restrict__ row_slot, const uint32_t* __restrict__ row_rank,
                                     int64_t n, const Slot* slots, DevCols cols, RowSpec rs,
                                     unsigned long long* __restrict__ rows) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    uint32_t s = row_slot[i];
    if (s == kInvalidSlot) continue;
    unsigned long long pos = (slots[s].meta >> 28) + row_rank[i];
    unsigned long long* dst = rows + pos * rs.nwords;
    unsigned long long nullmask = 0;
    int nw = rs.null_word >= 0 ? rs.nwords - 1 : rs.nwords;
    for (int w = 0; w < nw; w++) {
      int c = rs.col[w];
      unsigned long long v;
      if (rs.elem_len[w] == 8) v = reinterpret_cast<const unsigned long long*>(cols.data[c])[i];
      else v = reinterpret_cast<const uint32_t*>(cols.data[c])[i];
      if (rs.null_bit[w] >= 0 && cols.nulls[c] && !bit_not_null(cols.nulls[c], i)) nullmask |= 1ull << rs.null_bit[w];
      dst[w] = v;
    }
    if (rs.null_word >= 0) dst[rs.null_word] = nullmask;
  }
}

// ---------------------------------------------------------------------------------------------
// probe — fused fast path: unique build keys (mode U1), inner join, NOT NULL 8-byte columns.
// One pass: stream probe key (+ payload columns) with coalesced loads, one gather of the home slot pair per row,
// warp-ballot compaction, one output-cursor atomic per warp tile, coalesced column stores.
// The output shape is a template parameter (NPC probe payload columns, NKD outputs fed by the join key, NMD outputs
// fed by the build payload): with run-time destination counts ptxas unrolled the store loops into ~360 predicated
// STG + 350 LDC per kernel.
// ---------------------------------------------------------------------------------------------
#define TG_FAST_MAX_PCOLS 3
#define TG_FAST_MAX_KEYDST 2
#define TG_FAST_MAX_METADST 1
struct FastOut {
  int32_t n_pcols, n_key_dst, n_meta_dst, pad;
  const unsigned long long* psrc[TG_FAST_MAX_PCOLS];
  unsigned long long* pdst[TG_FAST_MAX_PCOLS];       // exactly one destination per probe payload column
  unsigned long long* key_dst[TG_FAST_MAX_KEYDST];   // outputs that carry the join key (probe key and/or build key)
  unsigned long long* meta_dst[TG_FAST_MAX_METADST]; // output that carries the build payload
};

// Warp-tile output stores at the rows the warp reserved from wbase on.  Paired: the whole tile matched and wbase is even;
// rows 2g, 2g+1 of a lane are adjacent input rows, so the input order is kept and a lane writes 16 bytes per column (half
// the store instructions of the compacting store).
template <int R, int NPC, int NKD, int NMD>
__device__ __forceinline__ void store_tile_paired(unsigned long long wbase, const int64_t (&k)[R], const unsigned long long (&meta)[R],
                                                  const unsigned long long (&pv)[R][NPC > 0 ? NPC : 1], const FastOut& out, int lane) {
#pragma unroll
  for (int g = 0; g < R / 2; g++) {
    const unsigned long long o = wbase + (unsigned long long)(g * 64 + 2 * lane);
    const ulonglong2 kk = make_ulonglong2((unsigned long long)k[2 * g], (unsigned long long)k[2 * g + 1]);
#pragma unroll
    for (int d = 0; d < NKD; d++) __stcs(reinterpret_cast<ulonglong2*>(out.key_dst[d] + o), kk);
#pragma unroll
    for (int d = 0; d < NMD; d++) __stcs(reinterpret_cast<ulonglong2*>(out.meta_dst[d] + o), make_ulonglong2(meta[2 * g], meta[2 * g + 1]));
#pragma unroll
    for (int c = 0; c < NPC; c++) __stcs(reinterpret_cast<ulonglong2*>(out.pdst[c] + o), make_ulonglong2(pv[2 * g][c], pv[2 * g + 1][c]));
  }
}

// compacting: row j of a lane goes to its rank among the warp's matched rows j (bal[j]), behind the matched rows before j
template <int R, int NPC, int NKD, int NMD>
__device__ __forceinline__ void store_tile_compact(unsigned long long wbase, const int64_t (&k)[R], const unsigned long long (&meta)[R],
                                                   const unsigned long long (&pv)[R][NPC > 0 ? NPC : 1], const unsigned (&bal)[R],
                                                   const FastOut& out, int lane) {
#pragma unroll
  for (int j = 0; j < R; j++) {
    if ((bal[j] >> lane) & 1u) {
      const unsigned long long o = wbase + __popc(bal[j] & ((1u << lane) - 1));
#pragma unroll
      for (int d = 0; d < NKD; d++) __stcs(out.key_dst[d] + o, (unsigned long long)k[j]);
#pragma unroll
      for (int d = 0; d < NMD; d++) __stcs(out.meta_dst[d] + o, meta[j]);
#pragma unroll
      for (int c = 0; c < NPC; c++) __stcs(out.pdst[c] + o, pv[j][c]);
    }
    wbase += __popc(bal[j]);
  }
}

// R rows per lane, keys and payloads already in registers: gather, resolve, compact, store.
// `in[j]` = row j of this lane exists (tail tiles).
template <int R, int NPC, int NKD, int NMD, bool PAIRED = false>
__device__ __forceinline__ void probe_rows_u1(const int64_t (&k)[R], const unsigned long long (&pv)[R][NPC > 0 ? NPC : 1],
                                              const unsigned long long (&sl0)[R], const bool (&in)[R], const TableView& t,
                                              const FastOut& out, unsigned long long* __restrict__ out_cursor, int lane) {
  Slot v[R], w[R];
  // the home is the first slot of an aligned pair: load both.  The side slot of the sentinel key is loaded as a pair too
  // (the table holds one spare slot behind it); only its first slot counts.
#pragma unroll
  for (int j = 0; j < R; j++) load_pair(t.slots + sl0[j], v[j], w[j]);
  unsigned long long meta[R];
  unsigned bal[R];
  uint32_t total = 0;
#pragma unroll
  for (int j = 0; j < R; j++) {
    bool m;
    if (k[j] == kEmptyKey) m = in[j] && v[j].key != 0;
    else if (v[j].key == k[j]) m = true;
    else if (w[j].key == k[j]) { v[j] = w[j]; m = true; }
    else if (v[j].key == kEmptyKey || w[j].key == kEmptyKey) m = false;
    else m = probe_run(t.slots, t.nslots, k[j], sl0[j] + 2, v[j].meta);   // the home slots hold other keys
    meta[j] = v[j].meta;
    bal[j] = __ballot_sync(0xffffffffu, m);
    total += __popc(bal[j]);
  }
  unsigned long long wbase = 0;
  if (lane == 0 && total) wbase = atomicAdd(out_cursor, (unsigned long long)total);
  wbase = __shfl_sync(0xffffffffu, wbase, 0);
  if (PAIRED && total == 32u * R && (wbase & 1ull) == 0) store_tile_paired<R, NPC, NKD, NMD>(wbase, k, meta, pv, out, lane);
  else store_tile_compact<R, NPC, NKD, NMD>(wbase, k, meta, pv, bal, out, lane);
}

// Optional input shape of the warp kernel: the probe rows regrouped by L2 partition into fixed-capacity segments
// (k_partition_scatter_bulk, count-free): segment p = rows [p*cap, p*cap + min(cnt[p], cap)), cap a multiple of the
// 128-row warp tile, so a tile never straddles two segments.  `gate` makes a launch conditional on a device flag, so the
// host can enqueue "partitioned probe if the scatter fitted, else direct probe" without a round trip.
struct SegSpec {
  const unsigned long long* cnt;     // nullptr = plain dense input of n rows
  uint32_t tiles_per_seg;            // cap / (32*R)
  int32_t gate_want;                 // run iff (*gate != 0) == gate_want
  long long cap;
  const unsigned long long* gate;    // nullptr = unconditional
  long long ungated_from;            // k_probe_inner_u1_w, dense input: when the gate says "do not run", rows >= ungated_from
                                     // (a multiple of 128) are probed all the same — the < 1 scatter tile the partition pass
                                     // leaves behind rides on the gated fallback launch instead of costing a launch of its own
};

// true when the launch's gate says "do not run"
__device__ __forceinline__ bool gated_off(const SegSpec& seg) {
  return seg.gate && ((*seg.gate != 0ull) != (seg.gate_want != 0));
}

// one past the last row of segment p: p·cap + min(cnt[p], cap).  p keeps the caller's integer type, and with it the
// caller's address arithmetic.
template <typename I>
__device__ __forceinline__ int64_t seg_end(const SegSpec& seg, I p) {
  const unsigned long long c = seg.cnt[p];
  return (int64_t)p * seg.cap + (int64_t)(c < (unsigned long long)seg.cap ? c : (unsigned long long)seg.cap);
}

// warp-autonomous: no shared memory, no block barrier; each warp owns tiles of 32×R rows.
// Launch with exactly the resident CTA count (occupancy × SMs): every extra wave of a persistent grid-stride kernel
// re-sweeps all partitions of a partition-ordered input and re-fetches the table slices.
template <int R, int NPC, int NKD, int NMD>
__global__ void __launch_bounds__(256)
k_probe_inner_u1_w(const int64_t* __restrict__ pkey, int64_t n, TableView t, FastOut out,
                   unsigned long long* __restrict__ out_cursor, SegSpec seg) {
  const int64_t tile_rows = 32 * R;
  int64_t first_tile = 0;
  if (gated_off(seg)) {
    if (seg.ungated_from <= 0 || seg.cnt) return;
    first_tile = seg.ungated_from / tile_rows;
  }
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t warp_id = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t ntiles = (n + tile_rows - 1) / tile_rows;
  for (int64_t tile = first_tile + warp_id; tile < ntiles; tile += warps_total) {
    const int64_t base = tile * tile_rows;
    int64_t limit = n;
    if (seg.cnt) {
      limit = seg_end(seg, (uint32_t)tile / seg.tiles_per_seg);
      if (base >= limit) continue;
    }
    int64_t k[R];
    unsigned long long pv[R][NPC > 0 ? NPC : 1];
    unsigned long long sl[R];
    bool in[R];
#pragma unroll
    for (int j = 0; j < R; j++) {
      int64_t i = base + j * 32 + lane;
      in[j] = i < limit;
      k[j] = in[j] ? __ldcs(pkey + i) : kEmptyKey;
    }
#pragma unroll
    for (int j = 0; j < R; j++) {
      int64_t i = base + j * 32 + lane;
      sl[j] = (k[j] == kEmptyKey) ? t.nslots : home_slot(hash64((uint64_t)k[j]), t.nslots);
#pragma unroll
      for (int c = 0; c < NPC; c++) pv[j][c] = in[j] ? __ldcs(out.psrc[c] + i) : 0ull;
    }
    probe_rows_u1<R, NPC, NKD, NMD>(k, pv, sl, in, t, out, out_cursor, lane);
  }
}

// ---------------------------------------------------------------------------------------------
// Segment-ordered input (SegSpec.cnt != nullptr), 128-bit accesses: a lane owns 2 ADJACENT rows of each 64-row group, so
// keys and payloads are read with LDG.128 and — when the whole tile matched — written with STG.128.  Segment bases are
// 1 KB aligned and the capacity is allocated in full, so a tile is always loaded whole; rows past the fill count are
// masked.  A full tile takes a lean path — no per-row `in` flags, no slot array, sentinel-valued keys detected once per
// tile (then the tile takes the generic path).  3 CTAs per SM (80 registers): launch exactly the resident CTA count.
// ---------------------------------------------------------------------------------------------

// the keys of the 128-row tile at `base`: lane owns rows 2·lane, 2·lane+1 of each 64-row group, one 128-bit load per group
__device__ __forceinline__ void load_tile_keys(const int64_t* __restrict__ pkey, int64_t base, int lane, int64_t (&k)[4]) {
#pragma unroll
  for (int g = 0; g < 2; g++) {
    const ulonglong2 kk = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + base + g * 64 + 2 * lane));
    k[2 * g] = (int64_t)kk.x; k[2 * g + 1] = (int64_t)kk.y;
  }
}

// the same for a tile that may end early: in[j] = row j lies below `limit`; a row past it gets the sentinel key
__device__ __forceinline__ void load_tile_keys(const int64_t* __restrict__ pkey, int64_t base, int64_t limit, int lane, int64_t (&k)[4],
                                               bool (&in)[4]) {
#pragma unroll
  for (int g = 0; g < 2; g++) {
    const int64_t i = base + g * 64 + 2 * lane;
    const ulonglong2 kk = __ldcs(reinterpret_cast<const ulonglong2*>(pkey + i));
    in[2 * g] = i < limit; in[2 * g + 1] = i + 1 < limit;
    k[2 * g] = in[2 * g] ? (int64_t)kk.x : kEmptyKey;
    k[2 * g + 1] = in[2 * g + 1] ? (int64_t)kk.y : kEmptyKey;
  }
}

template <int NPC, int NKD, int NMD>
__device__ __forceinline__ void probe_tile_generic(const int64_t* __restrict__ pkey, int64_t base, int64_t limit, const TableView& t,
                                                   const FastOut& out, unsigned long long* __restrict__ out_cursor, int lane) {
  constexpr int R = 4;
  int64_t k[R];
  unsigned long long pv[R][NPC > 0 ? NPC : 1];
  unsigned long long sl[R];
  bool in[R];
  load_tile_keys(pkey, base, limit, lane, k, in);
#pragma unroll
  for (int g = 0; g < R / 2; g++) {
    const int64_t i = base + g * 64 + 2 * lane;
    sl[2 * g] = (k[2 * g] == kEmptyKey) ? t.nslots : home_slot(hash64((uint64_t)k[2 * g]), t.nslots);
    sl[2 * g + 1] = (k[2 * g + 1] == kEmptyKey) ? t.nslots : home_slot(hash64((uint64_t)k[2 * g + 1]), t.nslots);
#pragma unroll
    for (int cc = 0; cc < NPC; cc++) {
      const ulonglong2 pp = __ldcs(reinterpret_cast<const ulonglong2*>(out.psrc[cc] + i));
      pv[2 * g][cc] = pp.x; pv[2 * g + 1][cc] = pp.y;
    }
  }
  probe_rows_u1<R, NPC, NKD, NMD, true>(k, pv, sl, in, t, out, out_cursor, lane);
}

// A full tile without the sentinel key: gather each row's home pair, then continue the linear probe of every row whose home
// pair holds two other keys, one aligned pair per row and step.  The rows of a lane walk their runs side by side, so a step
// costs one L2 round trip however many rows are still walking (dense tables: one of the 128 rows of a tile nearly always
// has a run).  Bit j of the result: row j matched, its build payload in meta[j].
__device__ __forceinline__ unsigned gather_walk(const int64_t (&k)[4], const TableView& t, unsigned long long (&meta)[4]) {
  constexpr int R = 4;
  Slot v[R], w[R];
#pragma unroll
  for (int j = 0; j < R; j++) load_pair(t.slots + home_slot(hash64((uint64_t)k[j]), t.nslots), v[j], w[j]);
  unsigned run = 0, hit = 0;   // bit j: row j's home pair holds two other keys / row j matched
#pragma unroll
  for (int j = 0; j < R; j++) {
    meta[j] = 0;
    if (v[j].key == k[j]) { hit |= 1u << j; meta[j] = v[j].meta; }
    else if (w[j].key == k[j]) { hit |= 1u << j; meta[j] = w[j].meta; }
    else if (v[j].key != kEmptyKey && w[j].key != kEmptyKey) run |= 1u << j;
  }
  if (run) {
    uint32_t sl[R];
#pragma unroll
    for (int j = 0; j < R; j++) {
      const unsigned long long s = home_slot(hash64((uint64_t)k[j]), t.nslots) + 2;
      sl[j] = s == t.nslots ? 0u : (uint32_t)s;
    }
    do {
#pragma unroll
      for (int j = 0; j < R; j++) if ((run >> j) & 1u) load_pair(t.slots + sl[j], v[j], w[j]);
#pragma unroll
      for (int j = 0; j < R; j++) {
        if (!((run >> j) & 1u)) continue;
        if (v[j].key == k[j]) { hit |= 1u << j; meta[j] = v[j].meta; run &= ~(1u << j); }
        else if (v[j].key == kEmptyKey) run &= ~(1u << j);
        else if (w[j].key == k[j]) { hit |= 1u << j; meta[j] = w[j].meta; run &= ~(1u << j); }
        else if (w[j].key == kEmptyKey) run &= ~(1u << j);
        else { sl[j] += 2; if (sl[j] == t.nslots) sl[j] = 0; }
      }
    } while (run);
  }
  return hit;
}

template <int NPC, int NKD, int NMD>
__global__ void __launch_bounds__(256, 3)
k_probe_inner_u1_seg_lean(const int64_t* __restrict__ pkey, int64_t n, TableView t, FastOut out,
                          unsigned long long* __restrict__ out_cursor, SegSpec seg) {
  constexpr int R = 4, G = 2, NP = NPC > 0 ? NPC : 1;
  if (gated_off(seg)) return;
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t warp_id = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t ntiles = n / 128;
  // Pass 1 sweeps the FULL tiles, pass 2 the (at most one per segment) partial tile at the end of each segment: a partial
  // tile adds an odd row count to the output cursor about half the time, and from then on every 128-row reservation
  // would start at an odd row — misaligned for the 128-bit stores of the all-matched path.
  // Pass 1: the capacity of every segment is allocated in full, so a tile can always be loaded
  for (int64_t tile = warp_id; tile < ntiles; tile += warps_total) {
    int64_t k[R];
    unsigned long long pv[R][NP];
    load_tile_keys(pkey, tile * 128, lane, k);
#pragma unroll
    for (int g = 0; g < G; g++) {
      const int64_t i = tile * 128 + g * 64 + 2 * lane;
#pragma unroll
      for (int c = 0; c < NPC; c++) {
        const ulonglong2 pp = __ldcs(reinterpret_cast<const ulonglong2*>(out.psrc[c] + i));
        pv[2 * g][c] = pp.x; pv[2 * g + 1][c] = pp.y;
      }
    }
    const int64_t base = tile * 128;
    const int64_t limit = seg_end(seg, (uint32_t)tile / seg.tiles_per_seg);
    if (limit - base < 128) continue;                       // empty or partial tile: pass 2
    const bool sentinel = (k[0] == kEmptyKey) | (k[1] == kEmptyKey) | (k[2] == kEmptyKey) | (k[3] == kEmptyKey);
    if (__any_sync(0xffffffffu, sentinel)) {                // the key value used as the empty marker: generic path for this tile
      probe_tile_generic<NPC, NKD, NMD>(pkey, base, limit, t, out, out_cursor, lane);
      continue;
    }
    unsigned long long meta[R];
    const unsigned hit = gather_walk(k, t, meta);
    unsigned bal[R];
    uint32_t total = 0;
#pragma unroll
    for (int j = 0; j < R; j++) {
      bal[j] = __ballot_sync(0xffffffffu, (hit >> j) & 1u);
      total += __popc(bal[j]);
    }
    unsigned long long wbase = 0;
    if (lane == 0 && total) wbase = atomicAdd(out_cursor, (unsigned long long)total);
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (total == 128u && (wbase & 1ull) == 0) store_tile_paired<R, NPC, NKD, NMD>(wbase, k, meta, pv, out, lane);
    else store_tile_compact<R, NPC, NKD, NMD>(wbase, k, meta, pv, bal, out, lane);
  }
  // pass 2: the partial tile of each segment
  const int64_t nseg = ntiles / seg.tiles_per_seg;
  for (int64_t sp = warp_id; sp < nseg; sp += warps_total) {
    const unsigned long long cc = seg.cnt[sp];
    const int64_t fill = (int64_t)(cc < (unsigned long long)seg.cap ? cc : (unsigned long long)seg.cap);
    if ((fill & 127) == 0) continue;
    const int64_t base = (sp * seg.tiles_per_seg + fill / 128) * 128;
    probe_tile_generic<NPC, NKD, NMD>(pkey, base, sp * seg.cap + fill, t, out, out_cursor, lane);
  }
}

// (There is no TMA-fed variant of this kernel — keys/payloads through a cp.async.bulk ring: the segment probe is bound by
// L1 gather issue, every KB of shared memory such a ring holds costs L1, and it would add 96 instantiations to the library.
// tools/scratch/probe_lab.cu keeps the experiment.)

// ---------------------------------------------------------------------------------------------
// In-place segment probe (dense input, fresh output batch, at least one output fed by the join key): the partition pass
// has scattered the probe key into out.key_dst[0] and the probe payloads into out.pdst[c], in segment layout.  A warp owns
// 128-row tiles, as in k_probe_inner_u1_seg_lean.  A tile whose 128 rows all match stays where it is: the kernel reads its
// keys and writes only key_dst[1..NKD) and the build payload, 8 + 8·(NKD-1+NMD) bytes per row instead of the lean kernel's
// 8·(1+NPC) read and 8·(NKD+NMD+NPC) written.  Any other tile (misses, a segment's partial last tile, sentinel-valued
// keys) is compacted to its front; the warp holds the whole tile in registers before the __syncwarp that precedes its
// stores, so it may overwrite its own rows.  tile_cnt[t] = rows tile t keeps (every tile is written); the warp adds its
// total to the output cursor once.  The output is dense in [0, *out_cursor) after k_inplace_holes + scan + k_inplace_fill.
// ---------------------------------------------------------------------------------------------
template <int NPC, int NKD, int NMD>
__device__ __forceinline__ void inplace_store(int64_t base, const int64_t (&k)[4], const unsigned long long (&meta)[4],
                                              const unsigned long long (&pv)[4][NPC > 0 ? NPC : 1], const unsigned (&bal)[4],
                                              const FastOut& out, int lane) {
  __syncwarp();   // every lane's loads of this tile precede any store into it
  int64_t o = base;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    if ((bal[j] >> lane) & 1u) {
      const int64_t r = o + __popc(bal[j] & ((1u << lane) - 1));
#pragma unroll
      for (int d = 0; d < NKD; d++) __stcs(out.key_dst[d] + r, (unsigned long long)k[j]);
#pragma unroll
      for (int d = 0; d < NMD; d++) __stcs(out.meta_dst[d] + r, meta[j]);
#pragma unroll
      for (int c = 0; c < NPC; c++) __stcs(out.pdst[c] + r, pv[j][c]);
    }
    o += __popc(bal[j]);
  }
}

// the probe payloads of a tile's rows (lane owns rows 2·lane, 2·lane+1 of each 64-row group)
template <int NPC>
__device__ __forceinline__ void inplace_load_pv(int64_t base, const FastOut& out, unsigned long long (&pv)[4][NPC > 0 ? NPC : 1], int lane) {
#pragma unroll
  for (int g = 0; g < 2; g++) {
    const int64_t i = base + g * 64 + 2 * lane;
#pragma unroll
    for (int c = 0; c < NPC; c++) {
      const ulonglong2 pp = __ldcs(reinterpret_cast<const ulonglong2*>(out.pdst[c] + i));
      pv[2 * g][c] = pp.x; pv[2 * g + 1][c] = pp.y;
    }
  }
}

// a tile with rows past the segment's fill count or sentinel-valued keys: per-row `in` flags, side slot, compaction
template <int NPC, int NKD, int NMD>
__device__ __forceinline__ uint32_t inplace_tile_generic(int64_t base, int64_t limit, const TableView& t, const FastOut& out, int lane) {
  constexpr int R = 4;
  int64_t k[R];
  unsigned long long pv[R][NPC > 0 ? NPC : 1], meta[R];
  bool in[R];
  load_tile_keys(reinterpret_cast<const int64_t*>(out.key_dst[0]), base, limit, lane, k, in);
  inplace_load_pv<NPC>(base, out, pv, lane);
  unsigned bal[R];
  uint32_t total = 0;
#pragma unroll
  for (int j = 0; j < R; j++) {
    const unsigned long long sl = (k[j] == kEmptyKey) ? t.nslots : home_slot(hash64((uint64_t)k[j]), t.nslots);
    Slot v, w;
    load_pair(t.slots + sl, v, w);
    bool m;
    meta[j] = v.meta;
    if (k[j] == kEmptyKey) m = in[j] && v.key != 0;
    else if (v.key == k[j]) m = true;
    else if (w.key == k[j]) { meta[j] = w.meta; m = true; }
    else if (v.key == kEmptyKey || w.key == kEmptyKey) m = false;
    else m = probe_run(t.slots, t.nslots, k[j], sl + 2, meta[j]);
    bal[j] = __ballot_sync(0xffffffffu, m);
    total += __popc(bal[j]);
  }
  inplace_store<NPC, NKD, NMD>(base, k, meta, pv, bal, out, lane);
  return total;
}

// The end of a full in-place tile whose rows are resolved (bit j of hit: row j matched, its build payload in meta[j]).  When
// all 128 rows matched, the probe columns are already in place: only the extra key copies and the build payload are written.
// Else the tile is compacted to its front.  Returns the rows the tile keeps.
template <int NPC, int NKD, int NMD>
__device__ __forceinline__ uint32_t inplace_finish(int64_t base, const int64_t (&k)[4], const unsigned long long (&meta)[4], unsigned hit,
                                                   const FastOut& out, int lane) {
  if (__all_sync(0xffffffffu, hit == 0xFu)) {
#pragma unroll
    for (int g = 0; g < 2; g++) {
      const int64_t o = base + g * 64 + 2 * lane;
      const ulonglong2 kk = make_ulonglong2((unsigned long long)k[2 * g], (unsigned long long)k[2 * g + 1]);
#pragma unroll
      for (int d = 1; d < NKD; d++) __stcs(reinterpret_cast<ulonglong2*>(out.key_dst[d] + o), kk);
#pragma unroll
      for (int d = 0; d < NMD; d++) __stcs(reinterpret_cast<ulonglong2*>(out.meta_dst[d] + o), make_ulonglong2(meta[2 * g], meta[2 * g + 1]));
    }
    return 128;
  }
  unsigned long long pv[4][NPC > 0 ? NPC : 1];
  inplace_load_pv<NPC>(base, out, pv, lane);
  unsigned bal[4];
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    bal[j] = __ballot_sync(0xffffffffu, (hit >> j) & 1u);
    m += __popc(bal[j]);
  }
  inplace_store<NPC, NKD, NMD>(base, k, meta, pv, bal, out, lane);
  return m;
}

template <int NPC, int NKD, int NMD>
__global__ void __launch_bounds__(256, 3)
k_probe_inner_u1_seg_inplace(int64_t n, TableView t, FastOut out, unsigned long long* __restrict__ out_cursor, SegSpec seg,
                             uint32_t* __restrict__ tile_cnt) {
  static_assert(NKD >= 1, "the probe key is read from the first key destination");
  constexpr int R = 4;
  if (gated_off(seg)) return;
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t warp_id = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t ntiles = n / 128;
  const int64_t* __restrict__ pkey = reinterpret_cast<const int64_t*>(out.key_dst[0]);
  unsigned long long kept = 0;
  for (int64_t tile = warp_id; tile < ntiles; tile += warps_total) {
    const int64_t base = tile * 128;
    const int64_t limit = seg_end(seg, (uint32_t)tile / seg.tiles_per_seg);
    uint32_t m = 0;
    if (limit - base >= 128) {
      int64_t k[R];
      load_tile_keys(pkey, base, lane, k);
      const bool sentinel = (k[0] == kEmptyKey) | (k[1] == kEmptyKey) | (k[2] == kEmptyKey) | (k[3] == kEmptyKey);
      if (__any_sync(0xffffffffu, sentinel)) {
        m = inplace_tile_generic<NPC, NKD, NMD>(base, limit, t, out, lane);
      } else {
        unsigned long long meta[R];
        const unsigned hit = gather_walk(k, t, meta);
        m = inplace_finish<NPC, NKD, NMD>(base, k, meta, hit, out, lane);
      }
    } else if (limit > base) {
      m = inplace_tile_generic<NPC, NKD, NMD>(base, limit, t, out, lane);
    }
    if (lane == 0) tile_cnt[tile] = m;
    kept += m;
  }
  if (lane == 0 && kept) atomicAdd(out_cursor, kept);
}

// ---------------------------------------------------------------------------------------------
// Slice index of a U1 table the partitioned probe slices (hash-and-displace, PTHash style): slice p holds the keys of
// partition mulhi32(hi32(h), P) in S slots of 16 bytes; a key's bucket is mulhi32(lo32(h), B), bits the partition does not
// use; its slot is p·S + pidx_slot(h, pilot[p·B + bucket], S).  A probe row costs one pilot byte and ONE 16-byte gather,
// no linear-probe run.  Pilot kPilotNone = the bucket found no placement: its keys are looked up in the linear-probe
// table, which keeps every key.  DESIGN.md §4.1.
// ---------------------------------------------------------------------------------------------
static constexpr uint32_t kPilotNone = 255;
static constexpr int kPidxMaxBucket = 32;   // a bigger bucket is never placed (Poisson(4) tail: none at 10 M keys)
static constexpr int kPidxThreads = 1024;   // CTA of the index probe: the CTA's warps share one slice's pilots

struct SliceIndex {
  const Slot* slots;        // [P][S]
  const uint8_t* pilot;     // [P][B], B a multiple of 16
  uint32_t P, S, B;
  uint32_t nbuf;            // pilot buffers of the index probe: 2 when 2·B fits kPidxMaxPilotBytes (join.cu), else 1
};

__host__ __device__ __forceinline__ uint32_t pidx_slot(uint64_t h, uint32_t q, uint32_t S) {
  return slot32(hash64(h ^ ((uint64_t)(q + 1) * 0xC2B2AE3D27D4EB4Full)), S);
}
__host__ __device__ __forceinline__ uint32_t pidx_bucket(uint64_t h, uint32_t B) { return mulhi32((uint32_t)h, B); }

// keys per partition (block-aggregated in shared memory)
__global__ void __launch_bounds__(256) k_pidx_part_count(const Slot* __restrict__ slots, unsigned long long nslots, uint32_t P,
                                                         unsigned long long* __restrict__ pcnt) {
  __shared__ unsigned int c[64];   // P <= TG_MAX_SLICES (partition_kernels.cuh: 32)
  for (int i = threadIdx.x; i < 64; i += blockDim.x) c[i] = 0;
  __syncthreads();
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nslots; i += (unsigned long long)gridDim.x * blockDim.x) {
    const int64_t k = slots[i].key;
    if (k != kEmptyKey) atomicAdd(&c[slot32(hash64((uint64_t)k), P)], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < (int)P; i += blockDim.x) if (c[i]) atomicAdd(&pcnt[i], (unsigned long long)c[i]);
}

// keys per bucket (global bucket id p·B + b)
__global__ void __launch_bounds__(256) k_pidx_bucket_count(const Slot* __restrict__ slots, unsigned long long nslots, SliceIndex ix,
                                                           uint32_t* __restrict__ bcnt) {
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nslots; i += (unsigned long long)gridDim.x * blockDim.x) {
    const int64_t k = slots[i].key;
    if (k == kEmptyKey) continue;
    const uint64_t h = hash64((uint64_t)k);
    atomicAdd(&bcnt[(size_t)slot32(h, ix.P) * ix.B + pidx_bucket(h, ix.B)], 1u);
  }
}

// the table slots of each bucket's keys, at off[bucket] (exclusive scan of the counts); bcnt counts back down to 0
__global__ void __launch_bounds__(256) k_pidx_lists(const Slot* __restrict__ slots, unsigned long long nslots, SliceIndex ix,
                                                    const unsigned long long* __restrict__ off, uint32_t* __restrict__ bcnt,
                                                    uint32_t* __restrict__ list) {
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nslots; i += (unsigned long long)gridDim.x * blockDim.x) {
    const int64_t k = slots[i].key;
    if (k == kEmptyKey) continue;
    const uint64_t h = hash64((uint64_t)k);
    const size_t b = (size_t)slot32(h, ix.P) * ix.B + pidx_bucket(h, ix.B);
    list[off[b] + atomicSub(&bcnt[b], 1u) - 1] = (uint32_t)i;
  }
}

// place every bucket of exactly `size` keys (launched largest size first): try pilots 0, 1, ...; a try claims each key's
// slot with atomicCAS from empty to the bucket id, and a bucket that loses any claim (to another bucket or to one of its own
// keys) releases the claims it won and tries its next pilot.  No placement within kPilotNone pilots leaves kPilotNone.
__global__ void __launch_bounds__(256) k_pidx_place(const Slot* __restrict__ slots, SliceIndex ix, const unsigned long long* __restrict__ off,
                                                    const uint32_t* __restrict__ list, uint32_t size, uint32_t* __restrict__ owner,
                                                    uint8_t* __restrict__ pilot) {
  const size_t nb = (size_t)ix.P * ix.B;
  for (size_t b = blockIdx.x * (size_t)blockDim.x + threadIdx.x; b < nb; b += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long o = off[b];
    if (off[b + 1] - o != size) continue;
    uint64_t h[kPidxMaxBucket];
    for (uint32_t j = 0; j < size; j++) h[j] = hash64((uint64_t)slots[list[o + j]].key);
    uint32_t* const base = owner + (b / ix.B) * ix.S;
    for (uint32_t q = 0; q < kPilotNone; q++) {
      uint32_t won = 0;
      for (; won < size; won++)
        if (atomicCAS(base + pidx_slot(h[won], q, ix.S), 0xFFFFFFFFu, (uint32_t)b) != 0xFFFFFFFFu) break;
      if (won == size) { pilot[b] = (uint8_t)q; break; }
      for (uint32_t j = 0; j < won; j++) atomicExch(base + pidx_slot(h[j], q, ix.S), 0xFFFFFFFFu);
    }
  }
}

// write each placed key's {key, payload} into its index slot, then (second launch, check = 1) verify that every placed key
// is at its computed slot; *bad != 0 drops the index
__global__ void __launch_bounds__(256) k_pidx_write(const Slot* __restrict__ slots, unsigned long long nslots, SliceIndex ix,
                                                    Slot* __restrict__ islots, int check, unsigned long long* __restrict__ bad) {
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nslots; i += (unsigned long long)gridDim.x * blockDim.x) {
    const Slot s = slots[i];
    if (s.key == kEmptyKey) continue;
    const uint64_t h = hash64((uint64_t)s.key);
    const uint32_t p = slot32(h, ix.P);
    const uint32_t q = ix.pilot[(size_t)p * ix.B + pidx_bucket(h, ix.B)];
    if (q == kPilotNone) continue;
    Slot* d = islots + (size_t)p * ix.S + pidx_slot(h, q, ix.S);
    if (!check) *d = s;
    else if (d->key != s.key || d->meta != s.meta) atomicAdd(bad, 1ull);
  }
}

// In-place segment probe through the slice index: the contract of k_probe_inner_u1_seg_inplace (tile_cnt, one cursor
// atomic per warp, compaction of partly matched tiles), but CTA-cooperative: one CTA of kPidxThreads per SM holds slice
// pilots in shared memory, in ix.nbuf buffers (2 when two slices' pilots fit kPidxMaxPilotBytes, else 1).  Buffer b is
// filled by one cp.async.bulk that completes on full[b]; a warp waits for slice p's pilots, sweeps its own tiles of segment
// p and moves on to slice p + 1 at once; the last warp done with a buffer refills it with slice p + nbuf.  So with two
// buffers no barrier spans the CTA: the next slice's pilots land while slow warps finish the current one.  Tile i of
// segment p goes to warp (p·tiles_per_seg + i) mod warps: the warps that take one tile more than the others differ from
// slice to slice.  A full tile reads its keys, one pilot byte and ONE 16-byte slot per row; a tile with a sentinel-valued
// key or a key whose bucket has no pilot, and a segment's partial last tile, take inplace_tile_generic on the
// linear-probe table.
template <int NPC, int NKD, int NMD>
__global__ void __launch_bounds__(kPidxThreads, 1)
k_probe_inner_u1_seg_inplace_pidx(int64_t n, TableView t, SliceIndex ix, FastOut out, unsigned long long* __restrict__ out_cursor,
                                  SegSpec seg, uint32_t* __restrict__ tile_cnt) {
  static_assert(NKD >= 1, "the probe key is read from the first key destination");
  constexpr int R = 4, NW = kPidxThreads / 32;
  extern __shared__ __align__(16) uint8_t spil[];   // [nbuf][B] pilots, then nbuf "full" mbarriers
  __shared__ uint32_t s_done[2];                     // warps done with buffer b, summed over the sweep
  if (gated_off(seg)) return;
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * NW;
  const int64_t warp_id = (int64_t)blockIdx.x * NW + (threadIdx.x >> 5);
  const int64_t* __restrict__ pkey = reinterpret_cast<const int64_t*>(out.key_dst[0]);
  const int nseg = (int)(n / 128 / seg.tiles_per_seg);
  const int nbuf = (int)ix.nbuf;
  uint64_t* full = reinterpret_cast<uint64_t*>(spil + (size_t)nbuf * ix.B);
  auto load = [&](int p) {   // one thread: slice p's pilots into buffer p % nbuf
    const int b = p % nbuf;
    mbar_arrive_expect_tx(&full[b], ix.B);
    bulk_g2s(spil + (size_t)b * ix.B, ix.pilot + (size_t)p * ix.B, ix.B, &full[b], l2_policy_evict_normal());
  };
  if (threadIdx.x == 0) {
    s_done[0] = s_done[1] = 0;
    for (int b = 0; b < nbuf; b++) mbar_init(&full[b], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int p = 0; p < nbuf && p < nseg; p++) load(p);
  unsigned long long kept = 0;
  for (int p = 0; p < nseg; p++) {
    const int b = p % nbuf;
    const uint32_t use = (uint32_t)(p / nbuf);   // how many slices buffer b held before this one
    mbar_wait(&full[b], use & 1u);
    const uint8_t* __restrict__ pil = spil + (size_t)b * ix.B;
    const int64_t limit = seg_end(seg, p);
    const int64_t t0 = (int64_t)p * seg.tiles_per_seg, t1 = t0 + seg.tiles_per_seg;
    const int64_t r = t0 % warps_total;
    const Slot* __restrict__ islots = ix.slots + (size_t)p * ix.S;
    for (int64_t tile = t0 + (warp_id >= r ? warp_id - r : warp_id - r + warps_total); tile < t1; tile += warps_total) {
      const int64_t base = tile * 128;
      uint32_t m = 0;
      if (limit - base >= 128) {
        int64_t k[R];
        load_tile_keys(pkey, base, lane, k);
        uint32_t q[R];
        bool generic = false;
#pragma unroll
        for (int j = 0; j < R; j++) {
          q[j] = pil[pidx_bucket(hash64((uint64_t)k[j]), ix.B)];
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
          m = inplace_finish<NPC, NKD, NMD>(base, k, meta, hit, out, lane);
        }
      } else if (limit > base) {
        m = inplace_tile_generic<NPC, NKD, NMD>(base, limit, t, out, lane);
      }
      if (lane == 0) tile_cnt[tile] = m;
      kept += m;
    }
    // this warp's pilot reads of buffer b are done (their values fed its gathers); the last of the NW warps refills it
    __syncwarp();
    if (lane == 0 && atomicAdd(&s_done[b], 1u) == (use + 1) * NW - 1 && p + nbuf < nseg) load(p + nbuf);
  }
  if (lane == 0 && kept) atomicAdd(out_cursor, kept);
}

// Hole fill behind k_probe_inner_u1_seg_inplace, R = *out_cursor: tile t keeps rows [128t, 128t + m_t).  cnt[t] = its holes
// below R, [128t + m_t, min(128t + 128, R)); cnt[ntiles + t] = its kept rows at or beyond R.  Both sum to the same total;
// one exclusive scan over the 2·ntiles counts numbers the holes and the rows that fill them.
__global__ void __launch_bounds__(256)
k_inplace_holes(const uint32_t* __restrict__ tile_cnt, int64_t ntiles, const unsigned long long* out_cursor,
                const unsigned long long* gate, uint32_t* __restrict__ cnt) {
  if (*gate) return;
  const int64_t R = (int64_t)*out_cursor;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < ntiles; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t s = t * 128, e = s + tile_cnt[t];
    cnt[t] = e < R ? (uint32_t)((s + 128 < R ? s + 128 : R) - e) : 0u;
    cnt[ntiles + t] = e > R ? (uint32_t)(e - (s > R ? s : R)) : 0u;
  }
}

// largest u in [lo, hi] with off[u] <= k (off non-decreasing, off[lo] <= k)
__device__ __forceinline__ int64_t last_le(const unsigned long long* __restrict__ off, int64_t lo, int64_t hi, unsigned long long k) {
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (off[mid] <= k) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// the k-th kept row at or beyond R moves into the k-th hole below R, every output column; a warp takes one tile's rows
__global__ void __launch_bounds__(256)
k_inplace_fill(const uint32_t* __restrict__ tile_cnt, int64_t ntiles, const unsigned long long* __restrict__ off,
               const unsigned long long* out_cursor, const unsigned long long* gate, FastOut out) {
  if (*gate) return;
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t warp_id = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t R = (int64_t)*out_cursor;
  const unsigned long long holes = off[ntiles];
  if (!holes) return;
  for (int64_t t = R / 128 + warp_id; t < ntiles; t += warps_total) {
    const uint32_t c = (uint32_t)(off[ntiles + t + 1] - off[ntiles + t]);
    if (!c) continue;
    const unsigned long long k0 = off[ntiles + t] - holes;
    const int64_t first = t * 128 > R ? t * 128 : R;
    const int64_t lo = last_le(off, 0, ntiles - 1, k0), hi = last_le(off, lo, ntiles - 1, k0 + c - 1);
    for (uint32_t r = lane; r < c; r += 32) {
      const unsigned long long k = k0 + r;
      const int64_t u = last_le(off, lo, hi, k);
      const int64_t dst = u * 128 + tile_cnt[u] + (int64_t)(k - off[u]), src = first + r;
      for (int d = 0; d < out.n_key_dst; d++) out.key_dst[d][dst] = out.key_dst[d][src];
      for (int d = 0; d < out.n_meta_dst; d++) out.meta_dst[d][dst] = out.meta_dst[d][src];
      for (int c2 = 0; c2 < out.n_pcols; c2++) out.pdst[c2][dst] = out.pdst[c2][src];
    }
  }
}

// OtherCondition on ONE candidate pair (probe row i, build row `brow` of the row store): true iff every CNF item is
// non-NULL true (expression.VectorizedFilter over the joined chunk, inner_join_probe.go:72-79)
__device__ __forceinline__ bool other_operand(const OtherItemDev& it, bool lhs, const DevCols& pcols, int64_t i, const unsigned long long* brow,
                                              int null_word, unsigned long long& raw) {
  const int src = lhs ? it.l_src : it.r_src, idx = lhs ? it.l_idx : it.r_idx, nbit = lhs ? it.l_null_bit : it.r_null_bit;
  if (src == OSRC_PROBE) {
    const uint8_t* nb = pcols.nulls[idx];
    if (nb && !bit_not_null(nb, i)) return false;
    raw = reinterpret_cast<const unsigned long long*>(pcols.data[idx])[i];
    return true;
  }
  if (src == OSRC_BUILD) {
    if (nbit >= 0 && ((brow[null_word] >> nbit) & 1ull)) return false;
    raw = brow[idx];
    return true;
  }
  raw = it.is_real ? (unsigned long long)__double_as_longlong(it.const_f64) : (unsigned long long)it.const_i64;
  return true;
}
__device__ __forceinline__ bool eval_other(const DevOther& o, const DevCols& pcols, int64_t i, const unsigned long long* brow, int null_word) {
  for (int q = 0; q < o.n; q++) {
    const OtherItemDev& it = o.it[q];
    unsigned long long a, b;
    if (!other_operand(it, true, pcols, i, brow, null_word, a) || !other_operand(it, false, pcols, i, brow, null_word, b)) return false;
    int r = it.is_real ? cmp_real(__longlong_as_double((long long)a), __longlong_as_double((long long)b))
                       : cmp_int((int64_t)a, it.l_unsigned != 0, (int64_t)b, it.r_unsigned != 0);
    if (!apply_cmp(it.op, r)) return false;
  }
  return true;
}

// ---------------------------------------------------------------------------------------------
// probe — general path (any join type, NULLs, filters, duplicates): count → scan → write
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_probe_count(KeySpec key, DevCols pcols, DevFilter filt, DevOther oth, int64_t n, TableView t, int kind,
              uint32_t* __restrict__ row_cnt, uint32_t* __restrict__ row_slot, uint8_t* slot_used) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    int64_t k;
    bool valid = load_key(key, i, k);
    if (valid && filt.n) valid = eval_filter(filt, pcols, i);
    uint32_t s = kInvalidSlot;
    unsigned long long meta = 0;
    if (valid) s = table_find(t, k, &meta);
    uint32_t cnt = 0;
    if (s != kInvalidSlot) cnt = t.mode == TABLE_U1 ? 1u : (uint32_t)(meta & kCntMask);
    if (oth.n && cnt) {   // OtherCondition: only the candidate pairs that pass it count (host forces mode G when it is present)
      const unsigned long long roff = meta >> 28;
      uint32_t pass = 0;
      for (uint32_t r = 0; r < cnt; r++) pass += eval_other(oth, pcols, i, t.rows + (roff + r) * t.row_words, t.null_word) ? 1u : 0u;
      cnt = pass;
    }
    bool matched = cnt > 0;
    if (slot_used && matched) slot_used[s] = 1;
    uint32_t c;
    switch (kind) {
      case PK_INNER: c = cnt; break;
      case PK_PROBE_OUTER: c = matched ? cnt : 1u; break;
      case PK_SEMI: c = matched ? 1u : 0u; break;
      case PK_ANTI: c = matched ? 0u : 1u; break;
      case PK_LEFT_OUTER_SEMI: case PK_ANTI_LEFT_OUTER_SEMI: c = 1u; break;
      default: c = 0u; break;
    }
    row_cnt[i] = c;
    row_slot[i] = matched ? s : kInvalidSlot;
  }
}

// exclusive scan of u32 counts into u64 offsets (n+1 entries): block sums → scan of sums → rescan
#define TG_SCAN_BLOCK 256
#define TG_SCAN_ITEMS 8
__global__ void __launch_bounds__(TG_SCAN_BLOCK)
k_scan_block_sums(const uint32_t* __restrict__ in, int64_t n, unsigned long long* __restrict__ block_sums) {
  __shared__ unsigned long long s[TG_SCAN_BLOCK / 32];
  int64_t base = (int64_t)blockIdx.x * TG_SCAN_BLOCK * TG_SCAN_ITEMS;
  unsigned long long sum = 0;
#pragma unroll
  for (int j = 0; j < TG_SCAN_ITEMS; j++) {
    int64_t i = base + (int64_t)j * TG_SCAN_BLOCK + threadIdx.x;
    if (i < n) sum += in[i];
  }
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long tot = 0;
    for (int w = 0; w < TG_SCAN_BLOCK / 32; w++) tot += s[w];
    block_sums[blockIdx.x] = tot;
  }
}
// single block: exclusive scan of block_sums in place; total written to block_sums[nblocks]
__global__ void __launch_bounds__(1024) k_scan_sums(unsigned long long* block_sums, int64_t nblocks) {
  __shared__ unsigned long long s_warp[32];
  __shared__ unsigned long long s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t base = 0; base < nblocks; base += 1024) {
    int64_t i = base + threadIdx.x;
    unsigned long long v = i < nblocks ? block_sums[i] : 0, incl = v;
    for (int o = 1; o < 32; o <<= 1) { unsigned long long u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      unsigned long long w = s_warp[lane], wi = w;
      for (int o = 1; o < 32; o <<= 1) { unsigned long long u = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += u; }
      s_warp[lane] = wi - w;
    }
    __syncthreads();
    unsigned long long carry = s_carry;
    if (i < nblocks) block_sums[i] = carry + s_warp[warp] + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + s_warp[31] + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) block_sums[nblocks] = s_carry;
}
__global__ void __launch_bounds__(TG_SCAN_BLOCK)
k_scan_write(const uint32_t* __restrict__ in, int64_t n, const unsigned long long* __restrict__ block_sums,
             unsigned long long* __restrict__ out_off) {
  // thread t owns TG_SCAN_ITEMS consecutive elements → serial scan per thread + block scan of thread sums
  __shared__ unsigned long long s_warp[TG_SCAN_BLOCK / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t base = (int64_t)blockIdx.x * TG_SCAN_BLOCK * TG_SCAN_ITEMS + (int64_t)threadIdx.x * TG_SCAN_ITEMS;
  uint32_t v[TG_SCAN_ITEMS];
  unsigned long long tsum = 0;
#pragma unroll
  for (int j = 0; j < TG_SCAN_ITEMS; j++) { v[j] = (base + j) < n ? in[base + j] : 0u; tsum += v[j]; }
  unsigned long long incl = tsum;
  for (int o = 1; o < 32; o <<= 1) { unsigned long long u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  unsigned long long wpre = 0;
  for (int w = 0; w < warp; w++) wpre += s_warp[w];
  unsigned long long run = block_sums[blockIdx.x] + wpre + incl - tsum;
#pragma unroll
  for (int j = 0; j < TG_SCAN_ITEMS; j++) { if (base + j < n) out_off[base + j] = run; run += v[j]; }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) out_off[n] = block_sums[gridDim.x];
}

__device__ __forceinline__ void store_out(const OutCols& out, int c, unsigned long long o, unsigned long long val, bool not_null) {
  if (out.spec[c].elem_len == 8) reinterpret_cast<unsigned long long*>(out.data[c])[o] = not_null ? val : 0ull;
  else reinterpret_cast<uint32_t*>(out.data[c])[o] = not_null ? (uint32_t)val : 0u;
  if (out.valid[c]) out.valid[c][o] = not_null ? 1 : 0;
}

__global__ void __launch_bounds__(256)
k_probe_write(int64_t n, const unsigned long long* __restrict__ off, const uint32_t* __restrict__ row_slot,
              const int64_t* __restrict__ pkey_i64, KeySpec key, TableView t, DevCols pcols, OutCols out, int kind,
              unsigned long long out_base, DevOther oth) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    unsigned long long o0 = off[i], c = off[i + 1] - o0;
    if (c == 0) continue;
    o0 += out_base;
    uint32_t s = row_slot[i];
    bool matched = s != kInvalidSlot;
    unsigned long long meta = matched ? t.slots[s].meta : 0ull;
    unsigned long long roff = meta >> 28;
    int64_t k = 0;
    if (matched) load_key(key, i, k);
    // with an OtherCondition the c emitted rows are the PASSING ones among the key's (meta & kCntMask) candidates
    unsigned long long cand = 0;
    for (unsigned long long r = 0; r < c; r++) {
      unsigned long long o = o0 + r;
      if (oth.n && matched) { while (!eval_other(oth, pcols, i, t.rows + (roff + cand) * t.row_words, t.null_word)) cand++; }
      const unsigned long long* brow = (matched && t.mode == TABLE_G) ? t.rows + (roff + (oth.n ? cand : r)) * t.row_words : nullptr;
      cand++;
      for (int cc = 0; cc < out.n; cc++) {
        const OutSpec sp = out.spec[cc];
        unsigned long long val = 0;
        bool nn = true;
        switch (sp.src) {
          case SRC_PROBE_COL: {
            const uint8_t* nb = pcols.nulls[sp.idx];
            nn = !(nb && !bit_not_null(nb, i));
            if (sp.elem_len == 8) val = reinterpret_cast<const unsigned long long*>(pcols.data[sp.idx])[i];
            else val = reinterpret_cast<const uint32_t*>(pcols.data[sp.idx])[i];
            break;
          }
          case SRC_BUILD_KEY: nn = matched; val = (unsigned long long)k; break;
          case SRC_BUILD_META: nn = matched; val = meta; break;
          case SRC_BUILD_WORD:
            nn = matched;
            if (matched) {
              val = brow[sp.idx];
              if (sp.null_bit >= 0 && ((brow[t.null_word] >> sp.null_bit) & 1ull)) nn = false;
            }
            break;
          default:   // SRC_FLAG: LeftOuterSemi 1/0, AntiLeftOuterSemi 0/1
            val = (kind == PK_ANTI_LEFT_OUTER_SEMI) ? (matched ? 0ull : 1ull) : (matched ? 1ull : 0ull);
            break;
        }
        store_out(out, cc, o, val, nn);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// probe — single pass for inner joins on UNIQUE build keys (any number of NOT NULL build payload columns, probe
// filters, NULL-able keys): SetChunkForProbe's filter + innerJoinProbe.Probe (base_join_probe.go:179, inner_join_probe.go:27)
// fused.  The general path costs three passes (count, scan, write) and two table gathers per matching row; with at most
// one match per probe row the output position is a warp ballot + one cursor atomic per warp row-group, so one pass does
// it: R rows per thread, all first-slot gathers of a tile in flight before the first compare.  Output order is arrival
// order (unspecified in the reference too).  Q3-shape: lineitem (600 M rows, l_shipdate filter) against the filtered
// orders runs here instead of count -> scan -> write.
// ---------------------------------------------------------------------------------------------
#define UQ_R 4
__global__ void __launch_bounds__(256)
k_probe_inner_uq(KeySpec key, DevCols pcols, DevFilter filt, int64_t n, TableView t, OutCols out, unsigned long long* __restrict__ out_cursor) {
  // ONE output-cursor atomic per 1024-row CTA tile: a per-warp reservation (600 M rows -> 19 M atomics on one address)
  // serialises in L2; per tile it is 0.6 M
  __shared__ uint32_t s_cnt[2][UQ_R][8];          // double-buffered by tile parity: two CTA barriers per tile, not three
  __shared__ unsigned long long s_base[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t tile = 256 * UQ_R;
  int par = 0;
  for (int64_t base = (int64_t)blockIdx.x * tile; base < n; base += (int64_t)gridDim.x * tile, par ^= 1) {
    int64_t k[UQ_R];
    unsigned long long sl[UQ_R];
    Slot v[UQ_R];
    bool valid[UQ_R];
    // the key loads do not depend on the filter: issue them first so that key and filter columns stream in together
    // (otherwise the kernel is bound by three dependent DRAM round trips per tile)
#pragma unroll
    for (int r = 0; r < UQ_R; r++) {
      const int64_t i = base + (int64_t)r * 256 + threadIdx.x;
      valid[r] = i < n;
      k[r] = (valid[r] && key.kind == KEY_I64) ? __ldcs(reinterpret_cast<const int64_t*>(key.data) + i) : 0;
    }
#pragma unroll
    for (int r = 0; r < UQ_R; r++) {
      const int64_t i = base + (int64_t)r * 256 + threadIdx.x;
      if (valid[r] && filt.n) valid[r] = eval_filter(filt, pcols, i);
      if (valid[r]) {
        if (key.kind == KEY_I64) valid[r] = !(key.nulls && !bit_not_null(key.nulls, i)) && !(key.reject_negative && k[r] < 0);
        else valid[r] = load_key(key, i, k[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < UQ_R; r++) {
      sl[r] = t.nslots; v[r].key = kEmptyKey; v[r].meta = 0;
      if (valid[r]) {
        if (k[r] != kEmptyKey) sl[r] = home_slot(hash64((uint64_t)k[r]), t.nslots);
        v[r] = load_slot(t.slots + sl[r]);
      }
    }
    unsigned bal[UQ_R];
#pragma unroll
    for (int r = 0; r < UQ_R; r++) {
      bool m = false;
      if (valid[r]) {
        if (k[r] == kEmptyKey) m = v[r].key != 0;                       // the side slot is occupied iff a build row carried this key
        else if (v[r].key == k[r]) m = true;
        else if (v[r].key != kEmptyKey) m = probe_run(t.slots, t.nslots, k[r], sl[r] + 1, v[r].meta);   // run on behind the home slot
      }
      bal[r] = __ballot_sync(0xffffffffu, m);
      if (lane == 0) s_cnt[par][r][warp] = __popc(bal[r]);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t tot = 0;
#pragma unroll
      for (int r = 0; r < UQ_R; r++) for (int w = 0; w < 8; w++) tot += s_cnt[par][r][w];
      s_base[par] = tot ? atomicAdd(out_cursor, (unsigned long long)tot) : 0ull;
    }
    __syncthreads();
    unsigned long long run = s_base[par];
#pragma unroll
    for (int r = 0; r < UQ_R; r++) {
      unsigned long long wb = run;
      for (int w = 0; w < 8; w++) { if (w < warp) wb += s_cnt[par][r][w]; run += s_cnt[par][r][w]; }
      if (!((bal[r] >> lane) & 1u)) continue;
      const int64_t i = base + (int64_t)r * 256 + threadIdx.x;
      const unsigned long long o = wb + __popc(bal[r] & ((1u << lane) - 1));
      const unsigned long long* brow = t.mode == TABLE_G ? t.rows + (v[r].meta >> 28) * t.row_words : nullptr;
      for (int c = 0; c < out.n; c++) {
        const OutSpec sp = out.spec[c];
        unsigned long long val;
        switch (sp.src) {
          case SRC_PROBE_COL: val = reinterpret_cast<const unsigned long long*>(pcols.data[sp.idx])[i]; break;
          case SRC_BUILD_KEY: val = (unsigned long long)k[r]; break;
          case SRC_BUILD_META: val = v[r].meta; break;
          default: val = brow[sp.idx]; break;   // SRC_BUILD_WORD
        }
        reinterpret_cast<unsigned long long*>(out.data[c])[o] = val;
      }
    }
    // no third barrier: the next tile writes the OTHER parity of s_cnt / s_base, and the tile after that is two barriers away
  }
}

// ScanRowTable (outer_join_probe.go:117, semi_join_probe.go:72): rows of the BUILD side that are
// (un)matched, taken from the device-resident build columns; probe-side output columns become NULL.
//   mode 0: emit build rows whose key was never matched (outer join, anti semi) — invalid-key rows included
//   mode 1: emit build rows whose key was matched (semi join)
__global__ void __launch_bounds__(256)
k_build_scan_count(const uint32_t* __restrict__ row_slot, const uint8_t* __restrict__ slot_used, int64_t n, int mode,
                   uint32_t* __restrict__ row_cnt) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    uint32_t s = row_slot[i];
    bool used = s != kInvalidSlot && slot_used[s];
    row_cnt[i] = (mode == 0 ? !used : used) ? 1u : 0u;
  }
}
// OutSpec.src here: SRC_BUILD_WORD.idx = build column index (read from the columns), SRC_PROBE_COL → NULL
__global__ void __launch_bounds__(256)
k_build_scan_write(int64_t n, const unsigned long long* __restrict__ off, DevCols bcols, OutCols out,
                   unsigned long long out_base) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    if (off[i + 1] == off[i]) continue;
    unsigned long long o = out_base + off[i];
    for (int cc = 0; cc < out.n; cc++) {
      const OutSpec sp = out.spec[cc];
      if (sp.src == SRC_PROBE_COL) { store_out(out, cc, o, 0, false); continue; }
      const uint8_t* nb = bcols.nulls[sp.idx];
      bool nn = !(nb && !bit_not_null(nb, i));
      unsigned long long val = sp.elem_len == 8 ? reinterpret_cast<const unsigned long long*>(bcols.data[sp.idx])[i]
                                                : reinterpret_cast<const uint32_t*>(bcols.data[sp.idx])[i];
      store_out(out, cc, o, val, nn);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// DECIMAL payload (late materialisation, join.cu kernel_view / gather_cells): the kernels above move a used DECIMAL column
// as 8-byte row ids; k_iota makes the ids and launch_gather_cells (chunk_io.cuh) turns them back into cells.  A cell is
// copied as 40 raw bytes, as the reference copies a fixed-length column's bytes into its row table and back
// (row_table_builder.go fillRowData).
// ---------------------------------------------------------------------------------------------
static constexpr int kCellBytes = 40;   // one MyDecimal cell in a chunk column

__global__ void k_iota(int64_t* __restrict__ out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = i;
}

}  // namespace tg
