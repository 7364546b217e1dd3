// gather_bench.cu — how many random 32-byte gathers per second can an H100 sustain, as a function of table size,
// loads in flight per thread, L2 fetch granularity and the mechanism (LDG into registers vs cp.async into shared memory)?
// Scratch tool: numbers guide the probe kernel's structure.
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint64_t h64(uint64_t k) { return (k ^ (k >> 32)) * 0x9E3779B97F4A7C15ull; }
__device__ __forceinline__ uint32_t slot_of(uint64_t i, uint32_t npairs) { return __umulhi((uint32_t)(h64(i * 0xD6E8FEB86659FD93ull + 12345) >> 32), npairs); }

struct alignas(32) Pair { uint64_t a, b, c, d; };

__device__ __forceinline__ Pair ldg256(const Pair* p) {
  Pair r;
  // two 128-bit loads of one 32-byte sector (sm_90 has no 256-bit load)
  asm volatile("ld.global.v2.u64 {%0,%1}, [%2];" : "=l"(r.a), "=l"(r.b) : "l"(p));
  asm volatile("ld.global.v2.u64 {%0,%1}, [%2+16];" : "=l"(r.c), "=l"(r.d) : "l"(p));
  return r;
}

template <int R>
__global__ void __launch_bounds__(256) k_ldg(const Pair* __restrict__ t, uint32_t npairs, int64_t n, unsigned long long* out) {
  uint64_t acc = 0;
  int64_t stride = (int64_t)gridDim.x * blockDim.x * R;
  for (int64_t base = ((int64_t)blockIdx.x * blockDim.x) * R + threadIdx.x; base < n; base += stride) {
    Pair v[R];
#pragma unroll
    for (int r = 0; r < R; r++) { int64_t i = base + (int64_t)r * blockDim.x; v[r] = ldg256(t + slot_of(i < n ? i : 0, npairs)); }
#pragma unroll
    for (int r = 0; r < R; r++) acc += v[r].a ^ v[r].d;
  }
  if (acc == 0x1234567) atomicAdd(out, acc);
}

// cp.async variant: each thread keeps D gathers of 32 bytes in flight in shared memory (2 x 16-byte LDGSTS)
template <int D>
__global__ void __launch_bounds__(256) k_cpasync(const Pair* __restrict__ t, uint32_t npairs, int64_t n, unsigned long long* out) {
  extern __shared__ __align__(32) unsigned char smem[];
  Pair* buf = reinterpret_cast<Pair*>(smem);     // [D][256]
  uint64_t acc = 0;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int issued = 0, done = 0;
  int64_t total = (n - i0 + stride - 1) / stride; if (i0 >= n) total = 0;
  // prologue
  for (; issued < D && issued < total; issued++) {
    const Pair* g = t + slot_of(i0 + (int64_t)issued * stride, npairs);
    uint32_t s = (uint32_t)__cvta_generic_to_shared(buf + (issued % D) * 256 + threadIdx.x);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(g));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s + 16), "l"((const char*)g + 16));
    asm volatile("cp.async.commit_group;");
  }
  while (done < total) {
    asm volatile("cp.async.wait_group %0;" ::"n"(D - 1));
    if (total - done < D) asm volatile("cp.async.wait_group 0;");
    Pair v = buf[(done % D) * 256 + threadIdx.x];
    acc += v.a ^ v.d;
    done++;
    if (issued < total) {
      const Pair* g = t + slot_of(i0 + (int64_t)issued * stride, npairs);
      uint32_t s = (uint32_t)__cvta_generic_to_shared(buf + (issued % D) * 256 + threadIdx.x);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(g));
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s + 16), "l"((const char*)g + 16));
      issued++;
    }
    asm volatile("cp.async.commit_group;");
  }
  if (acc == 0x1234567) atomicAdd(out, acc);
}

// 16-byte gathers (one slot, not a pair) for comparison
template <int R>
__global__ void __launch_bounds__(256) k_ldg128(const ulonglong2* __restrict__ t, uint32_t nslots, int64_t n, unsigned long long* out) {
  uint64_t acc = 0;
  int64_t stride = (int64_t)gridDim.x * blockDim.x * R;
  for (int64_t base = ((int64_t)blockIdx.x * blockDim.x) * R + threadIdx.x; base < n; base += stride) {
    ulonglong2 v[R];
#pragma unroll
    for (int r = 0; r < R; r++) { int64_t i = base + (int64_t)r * blockDim.x; v[r] = __ldg(t + slot_of(i < n ? i : 0, nslots)); }
#pragma unroll
    for (int r = 0; r < R; r++) acc += v[r].x ^ v[r].y;
  }
  if (acc == 0x1234567) atomicAdd(out, acc);
}

template <typename F>
static float time_ms(F f, int reps = 5) {
  cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  f(); CK(cudaDeviceSynchronize());
  CK(cudaEventRecord(a));
  for (int i = 0; i < reps; i++) f();
  CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
  float ms; CK(cudaEventElapsedTime(&ms, a, b));
  CK(cudaGetLastError());
  return ms / reps;
}

int main() {
  const int64_t n = 100000000;
  unsigned long long* out; CK(cudaMalloc(&out, 8));
  int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  size_t gran_default = 0; cudaDeviceGetLimit(&gran_default, cudaLimitMaxL2FetchGranularity);
  printf("SMs %d, default L2 fetch granularity %zu\n", sms, gran_default);
  const size_t table_mb[] = {16, 32, 64, 128, 400};
  for (size_t mb : table_mb) {
    size_t bytes = mb << 20;
    Pair* t; CK(cudaMalloc(&t, bytes)); CK(cudaMemset(t, 1, bytes));
    uint32_t npairs = (uint32_t)(bytes / 32);
    for (size_t gran : {(size_t)0, (size_t)32}) {
      if (gran) CK(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran)); else CK(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran_default));
#define RUN_LDG(R, CPS) { float ms = time_ms([&] { k_ldg<R><<<sms * CPS, 256>>>(t, npairs, n, out); }); \
        printf("table %4zu MB gran %3zu ldg256 R=%-2d ctas/sm=%d : %.3f ms  %.1f G/s\n", mb, gran ? gran : gran_default, R, CPS, ms, n / ms / 1e6); }
      RUN_LDG(1, 8) RUN_LDG(2, 8) RUN_LDG(4, 8) RUN_LDG(8, 8) RUN_LDG(8, 4) RUN_LDG(16, 4) RUN_LDG(16, 2)
#define RUN_L128(R, CPS) { float ms = time_ms([&] { k_ldg128<R><<<sms * CPS, 256>>>((const ulonglong2*)t, npairs * 2, n, out); }); \
        printf("table %4zu MB gran %3zu ldg128 R=%-2d ctas/sm=%d : %.3f ms  %.1f G/s\n", mb, gran ? gran : gran_default, R, CPS, ms, n / ms / 1e6); }
      RUN_L128(4, 8) RUN_L128(8, 8) RUN_L128(16, 4)
#define RUN_CPA(D, CPS) { CK(cudaFuncSetAttribute(k_cpasync<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, D * 256 * 32)); \
        float ms = time_ms([&] { k_cpasync<D><<<sms * CPS, 256, D * 256 * 32>>>(t, npairs, n, out); }); \
        printf("table %4zu MB gran %3zu cpasync D=%-2d ctas/sm=%d : %.3f ms  %.1f G/s\n", mb, gran ? gran : gran_default, D, CPS, ms, n / ms / 1e6); }
      RUN_CPA(4, 6) RUN_CPA(8, 3) RUN_CPA(16, 1) RUN_CPA(8, 2) RUN_CPA(4, 4)
    }
    CK(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran_default));
    CK(cudaFree(t));
  }
  return 0;
}
