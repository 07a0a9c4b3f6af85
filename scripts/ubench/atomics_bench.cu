// Micro-benchmark (not part of the product): throughput of L2 atomics for direct-address
// aggregation  sum[k] += v / cnt[k] += 1  with uniformly random 32-bit keys in [0, K).
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__global__ void gen(uint32_t* k, double* v, size_t n, uint32_t K) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x, st = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += st) {
    uint64_t x = i * 0x9E3779B97F4A7C15ull; x ^= x >> 29; x *= 0xBF58476D1CE4E5B9ull; x ^= x >> 32;
    k[i] = (uint32_t)(x % K); v[i] = (double)(x & 0xffff) / 65536.0;
  }
}
template <int MODE>
__global__ void agg(const uint32_t* __restrict__ k, const double* __restrict__ v, size_t n, double* sum, unsigned* cnt) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x, st = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += st) {
    uint32_t kk = k[i];
    if (MODE & 1) atomicAdd(&sum[kk], v[i]);
    if (MODE & 2) atomicAdd(&cnt[kk], 1u);
    if (MODE == 0) { if (kk == 0xffffffffu) sum[0] = v[i]; }
  }
}
int main(int argc, char** argv) {
  size_t n = argc > 1 ? atoll(argv[1]) : 1000000000ull;
  uint32_t K = argc > 2 ? atoi(argv[2]) : 1000000;
  uint32_t* k; double* v; double* sum; unsigned* cnt;
  cudaMalloc(&k, n * 4); cudaMalloc(&v, n * 8); cudaMalloc(&sum, (size_t)K * 8); cudaMalloc(&cnt, (size_t)K * 4);
  gen<<<132 * 8, 256>>>(k, v, n, K);
  cudaMemset(sum, 0, (size_t)K * 8); cudaMemset(cnt, 0, (size_t)K * 4);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  const char* names[4] = {"read-only k,v", "f64 sum atomics", "u32 count atomics", "sum + count"};
  for (int mode = 0; mode < 4; mode++) {
    for (int rep = 0; rep < 3; rep++) {
      cudaEventRecord(a);
      if (mode == 0) agg<0><<<132 * 16, 512>>>(k, v, n, sum, cnt);
      if (mode == 1) agg<1><<<132 * 16, 512>>>(k, v, n, sum, cnt);
      if (mode == 2) agg<2><<<132 * 16, 512>>>(k, v, n, sum, cnt);
      if (mode == 3) agg<3><<<132 * 16, 512>>>(k, v, n, sum, cnt);
      cudaEventRecord(b); cudaEventSynchronize(b);
      float ms; cudaEventElapsedTime(&ms, a, b);
      if (rep == 2) printf("K=%u n=%zu %-20s %.3f ms  %.1f Grows/s\n", K, n, names[mode], ms, n / ms / 1e6);
    }
  }
  printf("err=%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
