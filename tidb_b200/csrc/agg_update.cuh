// agg_update.cuh — the round-2 grouped-aggregation update kernels (included by agg.cu after its table structs).
//
// What bounds a grouped aggregation (tools/scratch/agg_lab.cu measures the primitives; 100 M rows): while the table stays
// in L2 the cost is L2 OPERATIONS, not HBM bytes — one key gather and two 64-bit REDs per row, and their costs add up.  A
// table that does not fit L2 (1 M groups = 48 MB on an H100's 50 MB L2) adds random HBM sector traffic on top and takes
// about twice as long (DESIGN.md §4.2).  Packing a group's words into one 32-byte sector is slower (same-sector atomics serialise), so the table stays
// structure-of-arrays.  Shared-memory atomics are not free either (f64 is a CAS loop), so a CTA-local table pays only
// while most rows hit it.  Hence ONE kernel with two levels (the reference's partial/final split, agg_hash_partial_worker.go:256 /
// agg_hash_final_worker.go:73, with a CTA as the partial worker):
//   level 1 (LOCAL): a small shared-memory table per CTA absorbs the rows of the keys it holds; a CTA that sees a low
//                    hit rate after its first tiles switches it off for the rest of its rows (high-cardinality input);
//   level 2        : everything else goes straight to the global table — R rows per thread, all slot gathers of a
//                    tile issued before the first compare (memory-level parallelism instead of a dependent chain);
//   at the end the CTA folds its local groups into the global table (MergePartialResult semantics).
// Rows / local groups that cannot be inserted within `max_probe` steps (table overfull) are deferred (bitmap) / spilled
// (tuple buffer); the host grows the table and re-runs just those.
#pragma once

namespace tg {

#define AGG2_BLOCK 256
#define AGG2_R 4
#define AGG2_TILE (AGG2_BLOCK * AGG2_R)

// ---- shared-memory atomics on 32-bit shared addresses (generic-address atomics on shared memory are slower) ----------
__device__ __forceinline__ void sred_add_u64(uint32_t a, unsigned long long v) { asm volatile("red.shared.add.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
// +1 on the LOW word of a 64-bit counter: a native 32-bit shared atomic (ATOMS.ADD) instead of the 64-bit CAS loop every
// 64-bit shared atomic compiles to (ATOMS.CAST.SPIN).  Exact while the counter stays below
// 2^32, which a CTA's share of one launch (< 2^31 rows) guarantees.
__device__ __forceinline__ void sred_inc_lo32(uint32_t a) { asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(a) : "memory"); }
__device__ __forceinline__ void sred_add_f64(uint32_t a, double v) { asm volatile("red.shared.add.f64 [%0], %1;" ::"r"(a), "d"(v) : "memory"); }
__device__ __forceinline__ void sred_min_u64(uint32_t a, unsigned long long v) { asm volatile("red.shared.min.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ void sred_max_u64(uint32_t a, unsigned long long v) { asm volatile("red.shared.max.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ unsigned long long scas_u64(uint32_t a, unsigned long long cmp, unsigned long long v) {
  unsigned long long old;
  asm volatile("atom.shared.cas.b64 %0, [%1], %2, %3;" : "=l"(old) : "r"(a), "l"(cmp), "l"(v) : "memory");
  return old;
}
__device__ __forceinline__ unsigned long long satom_add_u64(uint32_t a, unsigned long long v) {
  unsigned long long old;
  asm volatile("atom.shared.add.u64 %0, [%1], %2;" : "=l"(old) : "r"(a), "l"(v) : "memory");
  return old;
}
// dec_add (agg.cu) on the shared-memory table: the same carry rule
__device__ __forceinline__ void sdec_add(uint32_t lo, uint32_t hi, unsigned long long v, unsigned long long ext) {
  const unsigned long long old = satom_add_u64(lo, v);
  const unsigned long long add = ext + (old + v < old ? 1ull : 0ull);
  if (add) sred_add_u64(hi, add);
}
// one row of a DECIMAL SUM / AVG: the 128-bit add and the non-NULL count (count: nullptr / has_cnt false = NOT NULL argument)
__device__ __noinline__ void dec_apply(unsigned long long* lo, unsigned long long* hi, unsigned long long* cnt, unsigned long long v, unsigned long long ext) {
  dec_add(lo, hi, v, ext);
  if (cnt) atomicAdd(cnt, 1ull);
}
__device__ __noinline__ void sdec_apply(uint32_t lo, uint32_t hi, bool has_cnt, uint32_t cnt, unsigned long long v, unsigned long long ext) {
  sdec_add(lo, hi, v, ext);
  if (has_cnt) sred_inc_lo32(cnt);
}
// dec3_add / dec3_apply (agg.cu) on the shared-memory table: the same carry rule
__device__ __forceinline__ void sdec3_add(uint32_t w0, uint32_t w1, uint32_t w2, unsigned long long v0, unsigned long long v1, unsigned long long v2) {
  const unsigned long long old0 = satom_add_u64(w0, v0);
  const unsigned long long x1 = v1 + (old0 + v0 < old0 ? 1ull : 0ull);
  unsigned long long x2 = v2 + (x1 < v1 ? 1ull : 0ull);
  if (x1) { const unsigned long long old1 = satom_add_u64(w1, x1); x2 += old1 + x1 < old1 ? 1ull : 0ull; }
  if (x2) sred_add_u64(w2, x2);
}
__device__ __noinline__ void sdec3_apply(uint32_t w0, uint32_t step, bool has_cnt, uint32_t cnt, long long a, long long t) {
  unsigned long long lo, mid, top;
  dec_mul(a, t, lo, mid, top);
  sdec3_add(w0, w0 + step, w0 + 2 * step, lo, mid, top);
  if (has_cnt) sred_inc_lo32(cnt);
}
__device__ __forceinline__ unsigned long long sld_u64(uint32_t a) {
  unsigned long long v;
  asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory");
  return v;
}

// local (shared-memory) table: [keys | rows | state0 | state1 ...], each LS + 2 words; slot LS = NULL group, LS + 1 = the
// group whose key equals the empty sentinel
struct LocalTable { uint32_t base, stride_bytes, ls; };
__device__ __forceinline__ uint32_t lt_key(const LocalTable& l, uint32_t s) { return l.base + s * 8u; }
__device__ __forceinline__ uint32_t lt_rows(const LocalTable& l, uint32_t s) { return l.base + l.stride_bytes + s * 8u; }
__device__ __forceinline__ uint32_t lt_state(const LocalTable& l, int k, uint32_t s) { return l.base + l.stride_bytes * (2u + (uint32_t)k) + s * 8u; }

// value of aggregate argument column as raw 8 bytes
__device__ __forceinline__ unsigned long long arg_raw(const DevCols& cols, int col, int64_t row) {
  return __ldcs(reinterpret_cast<const unsigned long long*>(cols.data[col]) + row);
}

// per-row update of one group's states; SH = shared-memory table at 32-bit addresses, else the global table
template <bool SH, bool WIDE>
__device__ __forceinline__ void agg_apply2(const AggTable& t, const LocalTable& lt, const AggSpec& spec, const DevCols& cols, int64_t row, unsigned long long s) {
  if (SH) sred_inc_lo32(lt_rows(lt, (uint32_t)s)); else atomicAdd(&t.rows[s], 1ull);
#pragma unroll 1
  for (int k = 0; k < spec.n; k++) {
    const AggFuncDev& f = spec.f[k];
    if (f.arg_col < 0 || f.s0 < 0) continue;   // COUNT(*) and NOT NULL COUNT(x) read rows[]; FIRSTROW reads the key
    const uint8_t* nb = cols.nulls[f.arg_col];
    if (nb && !bit_not_null(nb, row)) continue;
    if (WIDE && f.s3 >= 0) {   // DECIMAL SUM / AVG of a product: exact 192-bit sum (out of line, like dec_apply)
      long long x, y;
      if (!dec_expr_operands(f, cols, row, x, y)) continue;
      if (SH) sdec3_apply(lt_state(lt, f.s0, (uint32_t)s), lt.stride_bytes, f.s1 >= 0, lt_state(lt, f.s1 >= 0 ? f.s1 : 0, (uint32_t)s), x, y);
      else dec3_apply(&t.state[f.s0][s], t.state[f.s2] - t.state[f.s0], f.s1 >= 0 ? &t.state[f.s1][s] : nullptr, x, y);
      continue;
    }
    switch (f.name) {
      case TG_AGG_COUNT: {
        unsigned long long v = f.final_mode ? arg_raw(cols, f.arg_col, row) : 1ull;
        if (!SH) atomicAdd(&t.state[f.s0][s], v);
        else if (f.final_mode) sred_add_u64(lt_state(lt, f.s0, (uint32_t)s), v);
        else sred_inc_lo32(lt_state(lt, f.s0, (uint32_t)s));
        break;
      }
      case TG_AGG_SUM: case TG_AGG_AVG: {
        if (f.s2 >= 0) {   // DECIMAL: exact 128-bit sum of the integer argument (out of line: keeps the DOUBLE path's registers)
          const unsigned long long v = arg_raw(cols, f.arg_col, row), ext = dec_ext(f, v);
          if (SH) sdec_apply(lt_state(lt, f.s0, (uint32_t)s), lt_state(lt, f.s2, (uint32_t)s), f.s1 >= 0, lt_state(lt, f.s1 >= 0 ? f.s1 : 0, (uint32_t)s), v, ext);
          else dec_apply(&t.state[f.s0][s], &t.state[f.s2][s], f.s1 >= 0 ? &t.state[f.s1][s] : nullptr, v, ext);
          break;
        }
        unsigned long long cnt = 1ull;
        int vcol = f.arg_col;
        if (f.name == TG_AGG_AVG && f.final_mode) {   // args: count column, sum column (func_avg.go:405)
          const uint8_t* nb2 = cols.nulls[f.arg_col2];
          if (nb2 && !bit_not_null(nb2, row)) break;
          cnt = arg_raw(cols, f.arg_col, row);
          vcol = f.arg_col2;
        }
        double v;
        if (f.arg_expr) { if (!agg_arg_real(spec, f, cols, row, v)) break; }
        else v = __longlong_as_double((long long)arg_raw(cols, vcol, row));
        if (SH) sred_add_f64(lt_state(lt, f.s0, (uint32_t)s), v); else atomicAdd(reinterpret_cast<double*>(&t.state[f.s0][s]), v);
        if (f.s1 >= 0) {
          if (!SH) atomicAdd(&t.state[f.s1][s], cnt);
          else if (f.name == TG_AGG_AVG && f.final_mode) sred_add_u64(lt_state(lt, f.s1, (uint32_t)s), cnt);   // partial counts: any 64-bit value
          else sred_inc_lo32(lt_state(lt, f.s1, (uint32_t)s));
        }
        break;
      }
      case TG_AGG_MIN: case TG_AGG_MAX: {
        unsigned long long raw = arg_raw(cols, f.arg_col, row), v;
        if (f.is_real) v = f64_to_ordered(__longlong_as_double((long long)raw));
        else if (f.is_unsigned) v = raw;
        else v = i64_to_ordered((long long)raw);
        if (f.name == TG_AGG_MIN) { if (SH) sred_min_u64(lt_state(lt, f.s0, (uint32_t)s), v); else atomicMin(&t.state[f.s0][s], v); }
        else { if (SH) sred_max_u64(lt_state(lt, f.s0, (uint32_t)s), v); else atomicMax(&t.state[f.s0][s], v); }
        if (f.s1 >= 0) { if (SH) sred_inc_lo32(lt_state(lt, f.s1, (uint32_t)s)); else atomicAdd(&t.state[f.s1][s], 1ull); }
        break;
      }
      default: break;
    }
  }
}

struct Agg2Params {
  GroupKey gk;
  int64_t n;
  uint32_t max_probe;
  int32_t nstates;
  int32_t local_slots;           // 0: no CTA-local level
  uint32_t* deferred;            // bitmap of rows that could not be inserted (table overfull)
  const uint32_t* only;          // re-run: restrict to these rows
  unsigned long long* n_deferred;
  unsigned long long* local_rows;   // statistics: rows absorbed by the CTA-local level
  AggPartials spill;             // local groups that could not be folded into the global table
  unsigned long long spill_cap;
};

template <bool LOCAL, bool WIDE>
__global__ void __launch_bounds__(AGG2_BLOCK)
k_agg_update2(Agg2Params p, DevCols cols, AggTable t, AggSpec spec) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ unsigned int s_fill, s_seen, s_hit, s_use_local;
  const int tid = threadIdx.x;
  LocalTable lt{0, 0, 0};
  if (LOCAL) {
    lt.base = smem_u32(smem_raw); lt.ls = (uint32_t)p.local_slots; lt.stride_bytes = (lt.ls + 2u) * 8u;
    unsigned long long* w = reinterpret_cast<unsigned long long*>(smem_raw);
    const uint32_t NT = lt.ls + 2u;
    for (uint32_t i = tid; i < NT; i += AGG2_BLOCK) {
      w[i] = (unsigned long long)kEmptyKey; w[NT + i] = 0;
      for (int k = 0; k < spec.n; k++) {
        const AggFuncDev& f = spec.f[k];
        if (f.s0 >= 0) w[(size_t)NT * (2 + f.s0) + i] = f.name == TG_AGG_MIN ? ~0ull : 0ull;
        if (f.s1 >= 0) w[(size_t)NT * (2 + f.s1) + i] = 0;
        if (f.s2 >= 0) w[(size_t)NT * (2 + f.s2) + i] = 0;
        if (f.s3 >= 0) w[(size_t)NT * (2 + f.s3) + i] = 0;
      }
    }
    if (tid == 0) { s_fill = 0; s_seen = 0; s_hit = 0; s_use_local = 1; }
    __syncthreads();
  }
  const uint32_t S = (uint32_t)t.nslots;
  const uint32_t max_local_fill = LOCAL ? lt.ls / 2u : 0u;
  unsigned long long my_deferred = 0, my_local = 0;
  int iter = 0;
  for (int64_t base = (int64_t)blockIdx.x * AGG2_TILE; base < p.n; base += (int64_t)gridDim.x * AGG2_TILE, iter++) {
    long long key[AGG2_R];
    uint32_t slot[AGG2_R];
    unsigned char kind[AGG2_R];   // 0 regular key, 1 NULL group, 2 sentinel-valued key, 3 no row, 4 done (local level)
#pragma unroll
    for (int r = 0; r < AGG2_R; r++) {
      const int64_t i = base + (int64_t)r * AGG2_BLOCK + tid;
      bool in = i < p.n;
      if (in && p.only) in = (p.only[i >> 5] >> (i & 31)) & 1u;
      kind[r] = 3; key[r] = 0; slot[r] = 0;
      if (!in) continue;
      if (p.gk.nulls && !bit_not_null(p.gk.nulls, i)) { kind[r] = 1; continue; }
      long long k = __ldcs(reinterpret_cast<const long long*>(p.gk.data) + i);
      if (p.gk.kind == GK_F64) { double d = __longlong_as_double(k); if (d == 0) d = 0; k = __double_as_longlong(d); }   // -0 groups with +0 (codec float.go:23)
      key[r] = k;
      kind[r] = k == kEmptyKey ? 2 : 0;
    }
    // ---- level 1: CTA-local table ---------------------------------------------------------------------------------
    if (LOCAL && *reinterpret_cast<volatile unsigned int*>(&s_use_local)) {
      unsigned int seen = 0, hit = 0;
#pragma unroll
      for (int r = 0; r < AGG2_R; r++) {
        if (kind[r] == 3) continue;
        const int64_t i = base + (int64_t)r * AGG2_BLOCK + tid;
        seen++;
        uint32_t ls;
        bool ok = true;
        if (kind[r] == 1) ls = lt.ls;
        else if (kind[r] == 2) ls = lt.ls + 1;
        else {
          const unsigned long long k = (unsigned long long)key[r];
          ls = slot32(hash64(k) * 0xD6E8FEB86659FD93ull, lt.ls);   // a second multiply: the global slot uses hash64's top bits too
          for (;;) {
            unsigned long long cur = sld_u64(lt_key(lt, ls));
            if (cur == k) break;
            if (cur == (unsigned long long)kEmptyKey) {
              if (*reinterpret_cast<volatile unsigned int*>(&s_fill) >= max_local_fill) { ok = false; break; }
              unsigned long long old = scas_u64(lt_key(lt, ls), (unsigned long long)kEmptyKey, k);
              if (old == (unsigned long long)kEmptyKey) { atomicAdd(&s_fill, 1u); break; }
              if (old == k) break;
            }
            if (++ls == lt.ls) ls = 0;
          }
        }
        if (ok) { agg_apply2<true, WIDE>(t, lt, spec, cols, i, ls); kind[r] = 4; hit++; }
      }
      my_local += hit;
      // hit-rate statistics of the CTA's first tiles decide whether the local level stays on
      if (iter < 4) { atomicAdd(&s_seen, seen); atomicAdd(&s_hit, hit); }
      else if (iter == 4 && tid == 0) {
        unsigned int a = *reinterpret_cast<volatile unsigned int*>(&s_seen), b = *reinterpret_cast<volatile unsigned int*>(&s_hit);
        if (b * 2u < a) s_use_local = 0;
      }
    }
    // ---- level 2: global table: issue every slot gather of the tile, then resolve ----------------------------------
    long long cur[AGG2_R];
#pragma unroll
    for (int r = 0; r < AGG2_R; r++) {
      cur[r] = 0;
      if (kind[r] == 0) { slot[r] = agg_home(key[r], S); cur[r] = *reinterpret_cast<volatile long long*>(&t.keys[slot[r]]); }
    }
#pragma unroll
    for (int r = 0; r < AGG2_R; r++) {
      if (kind[r] >= 3) continue;
      const int64_t i = base + (int64_t)r * AGG2_BLOCK + tid;
      unsigned long long s;
      if (kind[r] == 1) s = t.nslots;
      else if (kind[r] == 2) s = t.nslots + 1;
      else {
        uint32_t sl = slot[r];
        if (!global_find_or_insert(t, key[r], sl, cur[r], p.max_probe)) {
          atomicOr(&p.deferred[i >> 5], 1u << (i & 31));
          my_deferred++;
          continue;
        }
        s = sl;
      }
      agg_apply2<false, WIDE>(t, lt, spec, cols, i, s);
    }
  }
  for (int o = 16; o; o >>= 1) { my_deferred += __shfl_xor_sync(0xffffffffu, my_deferred, o); my_local += __shfl_xor_sync(0xffffffffu, my_local, o); }
  if ((tid & 31) == 0) { if (my_deferred) atomicAdd(p.n_deferred, my_deferred); if (my_local) atomicAdd(p.local_rows, my_local); }
  if (!LOCAL) return;
  __syncthreads();
  // ---- fold the CTA's local groups into the global table ---------------------------------------------------------------
  const unsigned long long* w = reinterpret_cast<const unsigned long long*>(smem_raw);
  const uint32_t NT = lt.ls + 2u;
  for (uint32_t i = tid; i < NT; i += AGG2_BLOCK) {
    const unsigned long long rows = w[NT + i];
    const long long k = (long long)w[i];
    const bool occ = i < lt.ls ? k != kEmptyKey : rows != 0;
    if (!occ) continue;
    unsigned long long st[AGG_LOCAL_MAX_STATES];
    for (int a = 0; a < p.nstates; a++) st[a] = w[(size_t)NT * (2 + a) + i];
    unsigned long long s;
    bool ok = true;
    if (i == lt.ls) s = t.nslots;
    else if (i == lt.ls + 1) s = t.nslots + 1;
    else {
      uint32_t sl = agg_home(k, S);
      long long c0 = *reinterpret_cast<volatile long long*>(&t.keys[sl]);
      ok = global_find_or_insert(t, k, sl, c0, p.max_probe);
      s = sl;
    }
    if (ok) { agg_merge_into<WIDE>(t, spec, s, rows, st); continue; }
    unsigned long long o = atomicAdd(p.spill.count, 1ull);   // overfull table: hand the group to the host's grow-and-merge loop
    if (o < p.spill_cap) {
      p.spill.keys[o] = k; p.spill.kind[o] = 0; p.spill.rows[o] = rows;
      for (int a = 0; a < p.nstates; a++) p.spill.state[a][o] = st[a];
    }
  }
}

}  // namespace tg
