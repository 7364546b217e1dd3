// agg_lab.cu — what bounds a 100 M-row / 1 M-group SUM+COUNT aggregation on an H100?
// Scratch tool (round 2): rates of the primitive operations a grouped aggregation can be built from — L2 atomics by
// width / layout, shared-memory atomics, L2-resident gathers — and of whole-kernel candidates.  Numbers guide agg.cu.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/scratch/agg_lab tools/scratch/agg_lab.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint64_t h64(uint64_t k) { return (k ^ (k >> 32)) * 0x9E3779B97F4A7C15ull; }
__device__ __forceinline__ uint64_t mix(uint64_t k) { k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; return k; }

// ---- primitive rates: every thread does R independent ops per iteration on "group" g = keys[i] -------------------
enum { OP_RED_U64, OP_RED_F64, OP_RED_U32, OP_LD64, OP_AOS32, OP_SOA3, OP_AOS_F64_U32, OP_RED_F64_X2 };

template <int OP>
__global__ void __launch_bounds__(256) k_prim(const long long* __restrict__ keys, const double* __restrict__ x, int64_t n, uint64_t G,
                                              unsigned long long* a0, unsigned long long* a1, unsigned long long* a2, unsigned long long* sink) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long acc = 0;
  for (; i < n; i += stride) {
    uint64_t g = (uint64_t)__ldcs(keys + i);
    if (OP == OP_RED_U64) atomicAdd(a0 + g, 1ull);
    if (OP == OP_RED_F64) atomicAdd(reinterpret_cast<double*>(a0) + g, __ldcs(x + i));
    if (OP == OP_RED_U32) atomicAdd(reinterpret_cast<unsigned int*>(a0) + g, 1u);
    if (OP == OP_LD64) acc += *reinterpret_cast<volatile unsigned long long*>(a0 + g);
    if (OP == OP_RED_F64_X2) { atomicAdd(reinterpret_cast<double*>(a0) + g, __ldcs(x + i)); atomicAdd(a1 + g, 1ull); }
    if (OP == OP_SOA3) {   // the round-1 kernel's traffic: key check + rows++ + sum, three arrays
      acc += *reinterpret_cast<volatile unsigned long long*>(a0 + g);
      atomicAdd(a1 + g, 1ull);
      atomicAdd(reinterpret_cast<double*>(a2) + g, __ldcs(x + i));
    }
    if (OP == OP_AOS32) {  // one 32-byte record per group: key | sum | count | pad
      unsigned long long* r = a0 + 4 * g;
      acc += *reinterpret_cast<volatile unsigned long long*>(r);
      atomicAdd(reinterpret_cast<double*>(r + 1), __ldcs(x + i));
      atomicAdd(r + 2, 1ull);
    }
    if (OP == OP_AOS_F64_U32) {
      unsigned long long* r = a0 + 4 * g;
      acc += *reinterpret_cast<volatile unsigned long long*>(r);
      atomicAdd(reinterpret_cast<double*>(r + 1), __ldcs(x + i));
      atomicAdd(reinterpret_cast<unsigned int*>(r + 2), 1u);
    }
  }
  if (acc == 0x123456789ull) *sink = acc;
}

// ---- shared-memory atomics: each CTA hammers a private table of S slots with random adds --------------------------
enum { SM_U32, SM_U64, SM_F64, SM_F64_U32, SM_LOOKUP_F64_U32 };
template <int OP>
__global__ void __launch_bounds__(256) k_smem(const long long* __restrict__ keys, const double* __restrict__ x, int64_t n, uint32_t S, unsigned long long* sink) {
  extern __shared__ __align__(16) unsigned char sm[];
  unsigned long long* t64 = reinterpret_cast<unsigned long long*>(sm);
  unsigned int* t32 = reinterpret_cast<unsigned int*>(sm + (size_t)S * 8);
  unsigned long long* tk = reinterpret_cast<unsigned long long*>(sm + (size_t)S * 12);
  for (uint32_t i = threadIdx.x; i < S; i += blockDim.x) { t64[i] = 0; t32[i] = 0; if (OP == SM_LOOKUP_F64_U32) tk[i] = ~0ull; }
  __syncthreads();
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    uint64_t k = (uint64_t)__ldcs(keys + i);
    uint32_t s = __umulhi((uint32_t)(h64(k) >> 32), S);
    if (OP == SM_U32) atomicAdd(t32 + s, 1u);
    if (OP == SM_U64) atomicAdd(t64 + s, 1ull);
    if (OP == SM_F64) atomicAdd(reinterpret_cast<double*>(t64) + s, __ldcs(x + i));
    if (OP == SM_F64_U32) { atomicAdd(reinterpret_cast<double*>(t64) + s, __ldcs(x + i)); atomicAdd(t32 + s, 1u); }
    if (OP == SM_LOOKUP_F64_U32) {
      uint64_t kk = k % (S / 2);   // keep the table half full
      s = __umulhi((uint32_t)(h64(kk) >> 32), S);
      for (;;) {
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(tk + s);
        if (cur == kk) break;
        if (cur == ~0ull) { unsigned long long old = atomicCAS(tk + s, ~0ull, (unsigned long long)kk); if (old == ~0ull || old == kk) break; }
        if (++s == S) s = 0;
      }
      atomicAdd(reinterpret_cast<double*>(t64) + s, __ldcs(x + i)); atomicAdd(t32 + s, 1u);
    }
  }
  __syncthreads();
  unsigned long long a = 0;
  for (uint32_t j = threadIdx.x; j < S; j += blockDim.x) a += t64[j] + t32[j];
  if (a == 0x123456789ull) *sink = a;
}

// ---- candidate A: full hash aggregation with AoS 32-byte records in L2 (open addressing, keys arbitrary int64) ----------
struct alignas(32) Rec { unsigned long long key; double sum; unsigned long long cnt; unsigned long long pad; };
__global__ void k_rec_init(Rec* t, uint64_t S) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < S) { t[i].key = ~0ull; t[i].sum = 0; t[i].cnt = 0; t[i].pad = 0; }
}
template <int R>
__global__ void __launch_bounds__(256) k_agg_aos(const long long* __restrict__ keys, const double* __restrict__ x, int64_t n, Rec* t, uint32_t S) {
  int64_t stride = (int64_t)gridDim.x * blockDim.x * R;
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x * R + threadIdx.x; base < n; base += stride) {
    uint64_t k[R]; double v[R]; uint32_t s[R];
#pragma unroll
    for (int r = 0; r < R; r++) { int64_t i = base + (int64_t)r * blockDim.x; bool in = i < n; k[r] = in ? (uint64_t)__ldcs(keys + i) : ~0ull; v[r] = in ? __ldcs(x + i) : 0.0; s[r] = __umulhi((uint32_t)(h64(k[r]) >> 32), S); }
    unsigned long long cur[R];
#pragma unroll
    for (int r = 0; r < R; r++) cur[r] = *reinterpret_cast<volatile unsigned long long*>(&t[s[r]].key);
#pragma unroll
    for (int r = 0; r < R; r++) {
      if (k[r] == ~0ull) continue;
      uint32_t sl = s[r]; unsigned long long c = cur[r];
      for (;;) {
        if (c == k[r]) break;
        if (c == ~0ull) { unsigned long long old = atomicCAS(&t[sl].key, ~0ull, (unsigned long long)k[r]); if (old == ~0ull || old == k[r]) break; }
        if (++sl == S) sl = 0;
        c = *reinterpret_cast<volatile unsigned long long*>(&t[sl].key);
      }
      atomicAdd(&t[sl].sum, v[r]);
      atomicAdd(&t[sl].cnt, 1ull);
    }
  }
}

// ---- candidate B: warp-level duplicate merging before the atomics (pays only when groups repeat inside a warp) -------
// ---- candidate C: one-pass 512-way LSU scatter + per-partition shared-memory aggregation --------------------------
#define LP_BLOCK 256
#define LP_ITEMS 16
#define LP_TILE (LP_BLOCK * LP_ITEMS)
template <int P>
__global__ void __launch_bounds__(LP_BLOCK) k_scatter_wide(const long long* __restrict__ keys, const double* __restrict__ x, int64_t ntiles,
                                                           long long* __restrict__ okeys, double* __restrict__ ox, unsigned long long* __restrict__ cursors, uint64_t cap) {
  extern __shared__ __align__(16) unsigned char dyn[];
  unsigned long long* s_val = reinterpret_cast<unsigned long long*>(dyn);
  unsigned short* s_part = reinterpret_cast<unsigned short*>(dyn + LP_TILE * 8);
  __shared__ uint32_t s_cnt[P], s_off[P];
  __shared__ unsigned long long s_gbase[P];
  __shared__ uint32_t s_warp[LP_BLOCK / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t base = tile * LP_TILE;
    for (int p = tid; p < P; p += LP_BLOCK) s_cnt[p] = 0;
    __syncthreads();
    unsigned long long k[LP_ITEMS]; uint32_t pr[LP_ITEMS];
#pragma unroll
    for (int j = 0; j < LP_ITEMS; j++) k[j] = (unsigned long long)__ldcs(keys + base + j * LP_BLOCK + tid);
#pragma unroll
    for (int j = 0; j < LP_ITEMS; j++) { uint32_t p = __umulhi((uint32_t)(h64(k[j]) >> 32), (uint32_t)P); pr[j] = (p << 16) | atomicAdd(&s_cnt[p], 1u); }
    __syncthreads();
    // block exclusive scan of P counts (P / LP_BLOCK per thread) + one global reservation per non-empty partition
    {
      constexpr int PER = P / LP_BLOCK > 0 ? P / LP_BLOCK : 1;
      uint32_t c[PER], sum = 0;
#pragma unroll
      for (int q = 0; q < PER; q++) { int p = tid * PER + q; c[q] = p < P ? s_cnt[p] : 0; sum += c[q]; }
      uint32_t incl = sum;
      for (int o = 1; o < 32; o <<= 1) { uint32_t u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
      if (lane == 31) s_warp[wid] = incl;
      __syncthreads();
      uint32_t wbase = 0;
      for (int w = 0; w < wid; w++) wbase += s_warp[w];
      uint32_t run = wbase + incl - sum;
#pragma unroll
      for (int q = 0; q < PER; q++) {
        int p = tid * PER + q;
        if (p < P) {
          s_off[p] = run; run += c[q];
          unsigned long long old = c[q] ? atomicAdd(&cursors[p], (unsigned long long)c[q]) : 0ull;
          s_gbase[p] = (unsigned long long)p * cap + old;
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < LP_ITEMS; j++) { uint32_t p = pr[j] >> 16; uint32_t slot = s_off[p] + (pr[j] & 0xffffu); pr[j] = slot; s_val[slot] = k[j]; s_part[slot] = (unsigned short)p; }
    // second column: load now (overlaps with the key write-out below)
    double v[LP_ITEMS];
#pragma unroll
    for (int j = 0; j < LP_ITEMS; j++) v[j] = __ldcs(x + base + j * LP_BLOCK + tid);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < LP_ITEMS; j++) { int sidx = j * LP_BLOCK + tid; uint32_t p = s_part[sidx]; okeys[s_gbase[p] + (sidx - s_off[p])] = (long long)s_val[sidx]; }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < LP_ITEMS; j++) s_val[pr[j]] = (unsigned long long)__double_as_longlong(v[j]);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < LP_ITEMS; j++) { int sidx = j * LP_BLOCK + tid; uint32_t p = s_part[sidx]; ox[s_gbase[p] + (sidx - s_off[p])] = __longlong_as_double((long long)s_val[sidx]); }
    __syncthreads();
  }
}

// per-partition aggregation in shared memory: CTA b handles partitions b, b+grid, ...; table S slots {key, sum, cnt32}
__global__ void __launch_bounds__(512) k_agg_part(const long long* __restrict__ pk, const double* __restrict__ px, const unsigned long long* __restrict__ cursors,
                                                  uint64_t cap, int P, uint32_t S, unsigned long long* out_groups, long long* ok, double* os, unsigned long long* oc) {
  extern __shared__ __align__(16) unsigned char sm[];
  unsigned long long* tk = reinterpret_cast<unsigned long long*>(sm);
  double* ts = reinterpret_cast<double*>(sm + (size_t)S * 8);
  unsigned int* tc = reinterpret_cast<unsigned int*>(sm + (size_t)S * 16);
  for (int p = blockIdx.x; p < P; p += gridDim.x) {
    for (uint32_t i = threadIdx.x; i < S; i += blockDim.x) { tk[i] = ~0ull; ts[i] = 0; tc[i] = 0; }
    __syncthreads();
    const int64_t n = (int64_t)cursors[p];
    const long long* k = pk + (uint64_t)p * cap; const double* x = px + (uint64_t)p * cap;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      unsigned long long kk = (unsigned long long)__ldcs(k + i);
      uint32_t s = __umulhi((uint32_t)(mix(kk) >> 32), S);
      for (;;) {
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(tk + s);
        if (cur == kk) break;
        if (cur == ~0ull) { unsigned long long old = atomicCAS(tk + s, ~0ull, kk); if (old == ~0ull || old == kk) break; }
        if (++s == S) s = 0;
      }
      atomicAdd(ts + s, __ldcs(x + i)); atomicAdd(tc + s, 1u);
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < S; i += blockDim.x) if (tk[i] != ~0ull) { unsigned long long o = atomicAdd(out_groups, 1ull); ok[o] = (long long)tk[i]; os[o] = ts[i]; oc[o] = tc[i]; }
    __syncthreads();
  }
}

int main(int argc, char** argv) {
  int64_t n = argc > 1 ? atoll(argv[1]) : 100000000;
  uint64_t G = argc > 2 ? strtoull(argv[2], 0, 10) : 1000000;
  int nsm = 0; CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0));
  long long* keys; double* x;
  CK(cudaMalloc(&keys, n * 8)); CK(cudaMalloc(&x, n * 8));
  {
    long long* hk = (long long*)malloc(n * 8); double* hx = (double*)malloc(n * 8);
    uint64_t s = 44;
    for (int64_t i = 0; i < n; i++) { s += 0x9E3779B97F4A7C15ull; uint64_t z = s; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; z ^= z >> 31; hk[i] = (long long)(z % G); hx[i] = (double)((z >> 20) % 10000000); }
    CK(cudaMemcpy(keys, hk, n * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(x, hx, n * 8, cudaMemcpyHostToDevice));
    free(hk); free(hx);
  }
  unsigned long long *a0, *a1, *a2, *sink;
  CK(cudaMalloc(&a0, G * 32 + 64)); CK(cudaMalloc(&a1, G * 8 + 64)); CK(cudaMalloc(&a2, G * 8 + 64)); CK(cudaMalloc(&sink, 8));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  auto timeit = [&](const char* name, auto fn, int reps = 3) {
    fn(); CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(e0)); for (int r = 0; r < reps; r++) fn(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); ms /= reps;
    printf("%-64s %8.3f ms  %7.1f G rows/s\n", name, ms, n / ms / 1e6); fflush(stdout);
  };
  printf("# n=%lld G=%llu SMs=%d\n", (long long)n, (unsigned long long)G, nsm);
  for (int per_sm : {8}) {
    int grid = nsm * per_sm;
    CK(cudaMemset(a0, 0, G * 32)); CK(cudaMemset(a1, 0, G * 8)); CK(cudaMemset(a2, 0, G * 8));
    timeit("prim: 8 B volatile load (L2 gather)", [&] { k_prim<OP_LD64><<<grid, 256>>>(keys, x, n, G, a0, a1, a2, sink); });
    timeit("prim: red.u64", [&] { k_prim<OP_RED_U64><<<grid, 256>>>(keys, x, n, G, a0, a1, a2, sink); });
    timeit("prim: red.f64", [&] { k_prim<OP_RED_F64><<<grid, 256>>>(keys, x, n, G, a0, a1, a2, sink); });
    timeit("prim: red.u32", [&] { k_prim<OP_RED_U32><<<grid, 256>>>(keys, x, n, G, a0, a1, a2, sink); });
    timeit("prim: red.f64 + red.u64, two arrays", [&] { k_prim<OP_RED_F64_X2><<<grid, 256>>>(keys, x, n, G, a0, a1, a2, sink); });
    timeit("prim: SoA ld + red.u64 + red.f64, three arrays (round-1 traffic)", [&] { k_prim<OP_SOA3><<<grid, 256>>>(keys, x, n, G, a0, a1, a2, sink); });
    timeit("prim: AoS 32 B record: ld + red.f64 + red.u64 in one sector", [&] { k_prim<OP_AOS32><<<grid, 256>>>(keys, x, n, G, a0, a1, a2, sink); });
    timeit("prim: AoS 32 B record: ld + red.f64 + red.u32", [&] { k_prim<OP_AOS_F64_U32><<<grid, 256>>>(keys, x, n, G, a0, a1, a2, sink); });
  }
  for (uint32_t S : {2048u, 4096u}) {
    size_t sm = (size_t)S * 20 + 64;
    int grid = nsm * 4;
    char nm[128];
    CK(cudaFuncSetAttribute(k_smem<SM_U32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    CK(cudaFuncSetAttribute(k_smem<SM_U64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    CK(cudaFuncSetAttribute(k_smem<SM_F64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    CK(cudaFuncSetAttribute(k_smem<SM_F64_U32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    CK(cudaFuncSetAttribute(k_smem<SM_LOOKUP_F64_U32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    snprintf(nm, sizeof nm, "smem S=%u: atomicAdd u32", S); timeit(nm, [&] { k_smem<SM_U32><<<grid, 256, sm>>>(keys, x, n, S, sink); });
    snprintf(nm, sizeof nm, "smem S=%u: atomicAdd u64", S); timeit(nm, [&] { k_smem<SM_U64><<<grid, 256, sm>>>(keys, x, n, S, sink); });
    snprintf(nm, sizeof nm, "smem S=%u: atomicAdd f64", S); timeit(nm, [&] { k_smem<SM_F64><<<grid, 256, sm>>>(keys, x, n, S, sink); });
    snprintf(nm, sizeof nm, "smem S=%u: atomicAdd f64 + u32", S); timeit(nm, [&] { k_smem<SM_F64_U32><<<grid, 256, sm>>>(keys, x, n, S, sink); });
    snprintf(nm, sizeof nm, "smem S=%u: lookup + f64 + u32 (half-full table)", S); timeit(nm, [&] { k_smem<SM_LOOKUP_F64_U32><<<grid, 256, sm>>>(keys, x, n, S, sink); });
  }
  {  // candidate A
    uint32_t S = (uint32_t)(G * 2);
    Rec* t; CK(cudaMalloc(&t, (size_t)S * 32));
    for (int per_sm : {4, 8}) {
      char nm[128];
      snprintf(nm, sizeof nm, "A: AoS-record hash agg in L2, R=4, %d CTAs/SM (incl. table init)", per_sm);
      timeit(nm, [&] { k_rec_init<<<(S + 255) / 256, 256>>>(t, S); k_agg_aos<4><<<nsm * per_sm, 256>>>(keys, x, n, t, S); });
      snprintf(nm, sizeof nm, "A: AoS-record hash agg in L2, R=8, %d CTAs/SM (incl. table init)", per_sm);
      timeit(nm, [&] { k_rec_init<<<(S + 255) / 256, 256>>>(t, S); k_agg_aos<8><<<nsm * per_sm, 256>>>(keys, x, n, t, S); });
    }
    CK(cudaFree(t));
  }
  {  // candidate C
    constexpr int P = 512;
    uint64_t cap = (uint64_t)(n / P * 1.1) + 4096;
    long long* pk; double* px; unsigned long long* cur; unsigned long long* ng; long long* ok; double* os; unsigned long long* oc;
    CK(cudaMalloc(&pk, cap * P * 8)); CK(cudaMalloc(&px, cap * P * 8)); CK(cudaMalloc(&cur, P * 8)); CK(cudaMalloc(&ng, 8));
    CK(cudaMalloc(&ok, G * 8 * 2)); CK(cudaMalloc(&os, G * 8 * 2)); CK(cudaMalloc(&oc, G * 8 * 2));
    int64_t ntiles = n / LP_TILE;
    CK(cudaFuncSetAttribute(k_scatter_wide<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, LP_TILE * 10));
    for (int per_sm : {2, 3, 4}) {
      char nm[128]; snprintf(nm, sizeof nm, "C1: one-pass %d-way LSU scatter (4096-row tiles), %d CTAs/SM", P, per_sm);
      timeit(nm, [&] { CK(cudaMemsetAsync(cur, 0, P * 8)); k_scatter_wide<P><<<nsm * per_sm, LP_BLOCK, LP_TILE * 10>>>(keys, x, ntiles, pk, px, cur, cap); });
    }
    uint32_t S = 4096;
    size_t sm = (size_t)S * 20;
    CK(cudaFuncSetAttribute(k_agg_part, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    timeit("C2: per-partition shared-memory aggregation (512 threads, S=4096)", [&] { CK(cudaMemsetAsync(ng, 0, 8)); k_agg_part<<<P, 512, sm>>>(pk, px, cur, cap, P, S, ng, ok, os, oc); });
    unsigned long long h = 0; CK(cudaMemcpy(&h, ng, 8, cudaMemcpyDeviceToHost));
    printf("# C groups found: %llu (expect %llu)\n", h, (unsigned long long)G);
  }
  return 0;
}
