// Micro-benchmark (not part of the product): cost of finding the lanes of a warp that hold the
// same 7/8-bit digit -- MATCH.ANY vs a ballot per digit bit vs shared-memory atomicOr.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ unsigned peers_ballot(unsigned d, int bits) {
  unsigned peers = 0xffffffffu;
#pragma unroll
  for (int b = 0; b < 8; b++) {
    if (b < bits) {
      const bool p = (d >> b) & 1;
      const unsigned m = __ballot_sync(0xffffffffu, p);
      peers &= p ? m : ~m;
    }
  }
  return peers;
}

template <int MODE>
__global__ void __launch_bounds__(256, 4) k(unsigned* out, int iters, int bits) {
  __shared__ unsigned masks[8][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < 8 * 256; i += 256) (&masks[0][0])[i] = 0;
  __syncthreads();
  unsigned x = threadIdx.x * 2654435761u + blockIdx.x * 40503u, acc = 0;
  const unsigned mask = (1u << bits) - 1;
  for (int it = 0; it < iters; it++) {
    x = x * 1664525u + 1013904223u;
    const unsigned d = (x >> 13) & mask;
    unsigned peers;
    if (MODE == 0) peers = __match_any_sync(0xffffffffu, d);
    else if (MODE == 1) peers = peers_ballot(d, bits);
    else {
      atomicOr(&masks[warp][d], 1u << lane);
      __syncwarp();
      peers = masks[warp][d];
      __syncwarp();
      if ((peers & ((1u << lane) - 1)) == 0) masks[warp][d] = 0;
      __syncwarp();
    }
    acc += __popc(peers & ((1u << lane) - 1)) + (peers >> 31);
  }
  out[blockIdx.x * 256 + threadIdx.x] = acc;
}

int main() {
  unsigned* out; cudaMalloc(&out, 132 * 4 * 256 * 4);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  const int iters = 20000;
  const char* names[3] = {"match.any", "ballot x bits", "smem atomicOr"};
  for (int bits = 7; bits <= 8; bits++)
    for (int mode = 0; mode < 3; mode++) {
      for (int rep = 0; rep < 2; rep++) {
        cudaEventRecord(a);
        if (mode == 0) k<0><<<132 * 4, 256>>>(out, iters, bits);
        if (mode == 1) k<1><<<132 * 4, 256>>>(out, iters, bits);
        if (mode == 2) k<2><<<132 * 4, 256>>>(out, iters, bits);
        cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b);
        // warp-level operations per second over the chip, and SM cycles per warp-op at 1.965 GHz
        double wops = 132.0 * 4 * 8 * iters;
        if (rep == 1) printf("bits=%d %-14s %.3f ms  %.1f G warp-ops/s  %.1f SM-cycles per warp-op (32 warps/SM resident)\n",
                             bits, names[mode], ms, wops / ms / 1e6, ms * 1e-3 * 1.98e9 / (wops / 132));
      }
    }
  printf("err=%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
