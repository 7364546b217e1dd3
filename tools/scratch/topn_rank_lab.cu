// topn_rank_lab.cu — how should k_topn_rank_dec (csrc/topn.cu) read its 40-byte DECIMAL cells?  Two versions of the same
// pass (dec_cell_ok + dec_order_key of decimal.cuh, one 8-byte rank out per row) over n cells in HBM:
//   plain : each thread loads its own cell as five 8-byte words (a warp's 5 loads cover its 1280 contiguous bytes; each
//           load touches 40 sectors and leaves the rest of them to the next loads through L1);
//   staged: each warp copies its 1280 bytes to shared memory with 5 fully coalesced 8-byte loads per lane, then every
//           lane reads its cell from shared memory (lane stride 40 B: no bank conflicts for 8-byte reads).
// Prints the median time of each (CUDA events, alternating) and the bandwidth at 48 B per row, and checks that both write
// the same ranks.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/scratch/topn_rank_lab tools/scratch/topn_rank_lab.cu
//   tools/scratch/topn_rank_lab 100000000
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
#include "../../tidb_b200/csrc/decimal.cuh"

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)
using namespace tg;

__device__ __forceinline__ unsigned long long rank_of_cell(const uint32_t (&c)[10], unsigned int* bad) {
  if (!dec_cell_ok(c)) *bad = 1u;
  return ~dec_order_key(c);   // DESC
}

__global__ void __launch_bounds__(256) k_plain(const unsigned long long* __restrict__ cells, int64_t n, unsigned long long* __restrict__ rank, unsigned int* bad) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint32_t c[10];
#pragma unroll
    for (int j = 0; j < 5; j++) { const unsigned long long v = cells[i * 5 + j]; c[2 * j] = (uint32_t)v; c[2 * j + 1] = (uint32_t)(v >> 32); }
    rank[i] = rank_of_cell(c, bad);
  }
}

__global__ void __launch_bounds__(256) k_staged(const unsigned long long* __restrict__ cells, int64_t n, unsigned long long* __restrict__ rank, unsigned int* bad) {
  __shared__ unsigned long long s[8][160];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int64_t nw = (n + 31) / 32;
  for (int64_t t = blockIdx.x * 8ll + wp; t < nw; t += gridDim.x * 8ll) {
    const int64_t r0 = t * 32, words = (n - r0 < 32 ? n - r0 : 32) * 5;
#pragma unroll
    for (int k = 0; k < 5; k++) if (lane + 32 * k < words) s[wp][lane + 32 * k] = cells[r0 * 5 + lane + 32 * k];
    __syncwarp();
    if (r0 + lane < n) {
      uint32_t c[10];
#pragma unroll
      for (int j = 0; j < 5; j++) { const unsigned long long v = s[wp][lane * 5 + j]; c[2 * j] = (uint32_t)v; c[2 * j + 1] = (uint32_t)(v >> 32); }
      rank[r0 + lane] = rank_of_cell(c, bad);
    }
    __syncwarp();
  }
}

int main(int argc, char** argv) {
  const int64_t n = argc > 1 ? atoll(argv[1]) : 100000000;
  // DECIMAL(15,2) cells in FromBin's form: digitsInt 13 (2 integer words), 1 fraction word
  std::vector<uint32_t> h((size_t)n * 10, 0);
  uint64_t x = 88172645463325252ull;
  for (int64_t i = 0; i < n; i++) {
    x ^= x << 13; x ^= x >> 7; x ^= x << 17;
    const uint64_t v = x % 1000000000000000ull;   // < 10^15, 2 fraction digits
    uint32_t* c = &h[(size_t)i * 10];
    c[0] = 13u | (2u << 8) | ((uint32_t)(x >> 60 & 1) << 24);
    c[1] = (uint32_t)(v / 100 / 1000000000ull); c[2] = (uint32_t)(v / 100 % 1000000000ull); c[3] = (uint32_t)(v % 100) * 10000000u;
  }
  unsigned long long *d, *r1, *r2; unsigned int* bad;
  CK(cudaMalloc(&d, (size_t)n * 40)); CK(cudaMalloc(&r1, (size_t)n * 8)); CK(cudaMalloc(&r2, (size_t)n * 8)); CK(cudaMalloc(&bad, 4));
  CK(cudaMemcpy(d, h.data(), (size_t)n * 40, cudaMemcpyHostToDevice));
  CK(cudaMemset(bad, 0, 4));
  int nsm; CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0));
  const int gp = (int)std::min<int64_t>((n + 255) / 256, nsm * 8), gs = (int)std::min<int64_t>((n + 255) / 256, nsm * 8);
  cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  std::vector<float> tp, ts;
  for (int it = 0; it < 22; it++) {
    for (int v = 0; v < 2; v++) {
      const bool plain = (v == 0) == (it % 2 == 0);
      CK(cudaEventRecord(a));
      if (plain) k_plain<<<gp, 256>>>(d, n, r1, bad); else k_staged<<<gs, 256>>>(d, n, r2, bad);
      CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
      float ms; CK(cudaEventElapsedTime(&ms, a, b));
      if (it >= 2) (plain ? tp : ts).push_back(ms);   // the first two rounds warm up
    }
  }
  std::vector<unsigned long long> o1((size_t)n), o2((size_t)n); unsigned int hb;
  CK(cudaMemcpy(o1.data(), r1, (size_t)n * 8, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(o2.data(), r2, (size_t)n * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(&hb, bad, 4, cudaMemcpyDeviceToHost));
  std::sort(tp.begin(), tp.end()); std::sort(ts.begin(), ts.end());
  const double mp = tp[tp.size() / 2], msd = ts[ts.size() / 2];
  printf("{\"rows\": %lld, \"plain_ms\": %.4f, \"staged_ms\": %.4f, \"plain_min_ms\": %.4f, \"staged_min_ms\": %.4f, "
         "\"plain_TBps\": %.3f, \"staged_TBps\": %.3f, \"same_ranks\": %s, \"bad\": %u}\n",
         (long long)n, mp, msd, tp[0], ts[0], 48.0 * n / mp / 1e9, 48.0 * n / msd / 1e9, o1 == o2 ? "true" : "false", hb);
  return 0;
}
