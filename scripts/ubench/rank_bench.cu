// Micro-benchmark (not part of the product): cost of the stable in-warp ranking step of a radix
// scatter pass, per 32-row round, for digit widths 6..11 bits.
//   mode 0  "ballot"      : one vote.ballot per digit bit (round-1 kernel), running count in smem (u16)
//   mode 1  "atomic"      : r = atomicAdd(&cnt[d], 1); after = cnt[d]; rounds in which two lanes hold the
//                           same digit (after - r != 1 somewhere) are repaired with one ballot per
//                           colliding digit value; running count lives in the same smem word
// Both produce rank = rows of the same digit at an earlier (round, lane) position of the warp.
// A check kernel compares the two on the same digit stream.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ unsigned lanemask_lt() { unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }

template <int NB>
__device__ __forceinline__ unsigned rank_ballot(unsigned d, unsigned short* hist, unsigned lt) {
  unsigned peers = 0xffffffffu;
#pragma unroll
  for (int b = 0; b < NB; b++) {
    asm("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\t"
        "and.b32 t, %1, %2;\n\t"
        "setp.ne.u32 p, t, 0;\n\t"
        "vote.sync.ballot.b32 t, p, 0xffffffff;\n\t"
        "@!p not.b32 t, t;\n\t"
        "and.b32 %0, %0, t;\n\t}"
        : "+r"(peers) : "r"(d), "r"(1u << b));
  }
  const unsigned short cnt = hist[d];
  const unsigned before = peers & lt;
  const unsigned r = (unsigned)cnt + __popc(before);
  __syncwarp();
  if (before == 0) hist[d] = cnt + (unsigned short)__popc(peers);
  __syncwarp();
  return r;
}

// mode 2 "redux": the same peer masks from redux.sync.or of one-hot lane bits (does REDUX run beside VOTE?)
// mode 3 "mixed": low half of the bits by vote.ballot, high half by redux.sync.or
template <int NB, int NVOTE>
__device__ __forceinline__ unsigned rank_mixed(unsigned d, unsigned short* hist, unsigned lt, unsigned lanebit) {
  unsigned peers = 0xffffffffu;
#pragma unroll
  for (int b = 0; b < NB; b++) {
    const bool p = (d >> b) & 1;
    unsigned m;
    if (b < NVOTE) m = __ballot_sync(0xffffffffu, p);
    else m = __reduce_or_sync(0xffffffffu, p ? lanebit : 0u);
    peers &= p ? m : ~m;
  }
  const unsigned short cnt = hist[d];
  const unsigned before = peers & lt;
  const unsigned r = (unsigned)cnt + __popc(before);
  __syncwarp();
  if (before == 0) hist[d] = cnt + (unsigned short)__popc(peers);
  __syncwarp();
  return r;
}

__device__ __forceinline__ unsigned rank_atomic(unsigned d, unsigned* cnt, unsigned lt) {
  unsigned r = atomicAdd(&cnt[d], 1u);
  __syncwarp();
  const unsigned after = cnt[d];
  unsigned pending = __ballot_sync(0xffffffffu, after - r != 1u);
  while (pending) {                                   // warp-uniform
    const int leader = __ffs(pending) - 1;
    const unsigned dl = __shfl_sync(0xffffffffu, d, leader);
    const unsigned m = __ballot_sync(0xffffffffu, d == dl);
    if (d == dl) r = after - __popc(m) + __popc(m & lt);
    pending &= ~m;
  }
  __syncwarp();
  return r;
}

template <int MODE, int NB>
__global__ void __launch_bounds__(256, 4) k(unsigned* out, int iters) {
  constexpr int NBINS = 1 << NB;
  extern __shared__ unsigned tab[];                   // 8 * NBINS words; mode 0 uses it as u16
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = lanemask_lt();
  unsigned x = threadIdx.x * 2654435761u + blockIdx.x * 40503u, acc = 0;
  for (int it = 0; it < iters; it++) {
    if ((it & 15) == 0) {                             // new "tile": clear the warp's table
      __syncwarp();
      for (int i = lane; i < NBINS; i += 32) tab[warp * NBINS + i] = 0;
      __syncwarp();
    }
    x = x * 1664525u + 1013904223u;
    const unsigned d = (x >> 13) & (NBINS - 1);
    unsigned r;
    if (MODE == 0) r = rank_ballot<NB>(d, reinterpret_cast<unsigned short*>(tab + warp * NBINS), lt);
    else if (MODE == 2) r = rank_mixed<NB, 0>(d, reinterpret_cast<unsigned short*>(tab + warp * NBINS), lt, 1u << lane);
    else if (MODE == 3) r = rank_mixed<NB, (NB + 1) / 2>(d, reinterpret_cast<unsigned short*>(tab + warp * NBINS), lt, 1u << lane);
    else           r = rank_atomic(d, tab + warp * NBINS, lt);
    acc += r;
  }
  out[blockIdx.x * 256 + threadIdx.x] = acc;
}

template <int NB>
__global__ void __launch_bounds__(256) check(unsigned* bad, int iters) {
  constexpr int NBINS = 1 << NB;
  extern __shared__ unsigned ta[];
  unsigned* tb = ta + 8 * NBINS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = lanemask_lt();
  for (int i = lane; i < NBINS; i += 32) { ta[warp * NBINS + i] = 0; tb[warp * NBINS + i] = 0; }
  __syncwarp();
  unsigned x = threadIdx.x * 2654435761u + blockIdx.x * 40503u;
  for (int it = 0; it < iters; it++) {
    x = x * 1664525u + 1013904223u;
    // skewed every other block: few distinct digits
    const unsigned d = (blockIdx.x & 1) ? ((x >> 13) & 3u) : ((x >> 13) & (NBINS - 1));
    const unsigned ra = rank_ballot<NB>(d, reinterpret_cast<unsigned short*>(ta + warp * NBINS), lt);
    const unsigned rb = rank_atomic(d, tb + warp * NBINS, lt);
    if (ra != rb) atomicAdd(bad, 1u);
  }
}

template <int NB> void run(unsigned* out, unsigned* bad) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  const int iters = 20000;
  cudaMemset(bad, 0, 4);
  const int smem = 8 * (1 << NB) * 4;
  cudaFuncSetAttribute(check<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * smem);
  cudaFuncSetAttribute(k<0, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaFuncSetAttribute(k<1, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaFuncSetAttribute(k<2, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaFuncSetAttribute(k<3, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  check<NB><<<132, 256, 2 * smem>>>(bad, 400);
  unsigned hbad = 0; cudaMemcpy(&hbad, bad, 4, cudaMemcpyDeviceToHost);
  for (int mode = 0; mode < 4; mode++) {
    float ms = 0;
    for (int rep = 0; rep < 2; rep++) {
      cudaEventRecord(a);
      if (mode == 0) k<0, NB><<<132 * 4, 256, smem>>>(out, iters);
      else if (mode == 1) k<1, NB><<<132 * 4, 256, smem>>>(out, iters);
      else if (mode == 2) k<2, NB><<<132 * 4, 256, smem>>>(out, iters);
      else           k<3, NB><<<132 * 4, 256, smem>>>(out, iters);
      cudaEventRecord(b); cudaEventSynchronize(b);
      cudaEventElapsedTime(&ms, a, b);
    }
    const double wops = 132.0 * 4 * 8 * iters;
    printf("bits=%2d %-7s %8.3f ms  %6.1f SM-cycles per 32-row round (32 warps/SM)  mismatches=%u\n", NB,
           mode == 0 ? "ballot" : mode == 1 ? "atomic" : mode == 2 ? "redux" : "mixed", ms, ms * 1e-3 * 1.98e9 / (wops / 132), hbad);
  }
}

int main() {
  unsigned* out; cudaMalloc(&out, 132 * 4 * 256 * 4);
  unsigned* bad; cudaMalloc(&bad, 4);
  run<6>(out, bad); run<7>(out, bad); run<8>(out, bad);
  printf("err=%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
