// dtb_stats.cu -- per-column min / max / NA count / varying-bit masks in one
// streaming read.  Replaces NumericStats<T>::compute_minmax (stats.cc:601-634),
// which feeds the integer key normalisation (sort.cc:729-740).
//
// HBM-bound: 1 read of the column, 16-byte vector loads, grid = 132 SMs x 8.
// Algorithmic bytes per row: sizeof(T).
// Single-column keys take col_stats_hist_kernel: the same statistics plus the first radix pass's histogram
// (per 4096-row tile, low 8 bits of u) from the same read -- the pass then needs no count kernel.
#include "dtb_common.cuh"

namespace dtb {

// Per-thread accumulator.  Columns of at most 32 bits accumulate in 32-bit registers (the 64-bit
// form costs twice the ALU work and kept the kernel below the HBM rate).
template <typename T, bool IS_FLOAT, bool NARROW = Raw32<T>::ok>
struct StatAcc;

template <typename T, bool IS_FLOAT>
struct StatAcc<T, IS_FLOAT, false> {
  u64 lo, hi, bor, band, nna, nvalid;
  __device__ __forceinline__ void init() {
    if (IS_FLOAT) { lo = ~0ull; hi = 0ull; }
    else { lo = (u64)INT64_MAX; hi = (u64)INT64_MIN; }
    bor = 0; band = ~0ull; nna = 0; nvalid = 0;
  }
  __device__ __forceinline__ void add(typename RawKey<T>::load_t raw) {
    u64 u; bool valid = RawKey<T>::get(raw, u);
    if (!valid) { nna++; return; }
    nvalid++;
    bor |= u; band &= u;
    if (IS_FLOAT) { lo = u < lo ? u : lo; hi = u > hi ? u : hi; }
    else {
      int64_t s = (int64_t)u;
      if (s < (int64_t)lo) lo = u;
      if (s > (int64_t)hi) hi = u;
    }
  }
  __device__ __forceinline__ void widen() {}
  __device__ __forceinline__ void merge(u64 lo2, u64 hi2, u64 or2, u64 and2, u64 na2, u64 nv2) {
    if (IS_FLOAT) { lo = lo2 < lo ? lo2 : lo; hi = hi2 > hi ? hi2 : hi; }
    else {
      if ((int64_t)lo2 < (int64_t)lo) lo = lo2;
      if ((int64_t)hi2 > (int64_t)hi) hi = hi2;
    }
    bor |= or2; band &= and2; nna += na2; nvalid += nv2;
  }
};

template <typename T, bool IS_FLOAT>
struct StatAcc<T, IS_FLOAT, true> {
  u32 lo32, hi32, or32, and32, na32, nv32;       // a thread sees far fewer than 2^32 rows
  u64 lo, hi, bor, band, nna, nvalid;            // filled by widen()
  __device__ __forceinline__ void init() {
    if (IS_FLOAT) { lo32 = ~0u; hi32 = 0u; }
    else { lo32 = (u32)INT32_MAX; hi32 = (u32)INT32_MIN; }
    or32 = 0; and32 = ~0u; na32 = 0; nv32 = 0;
  }
  __device__ __forceinline__ void add(typename RawKey<T>::load_t raw) {
    u32 u; const bool valid = Raw32<T>::get(raw, u);
    if (!valid) { na32++; return; }
    nv32++;
    or32 |= u; and32 &= u;
    if (IS_FLOAT) { lo32 = u < lo32 ? u : lo32; hi32 = u > hi32 ? u : hi32; }
    else {
      lo32 = ((int32_t)u < (int32_t)lo32) ? u : lo32;
      hi32 = ((int32_t)u > (int32_t)hi32) ? u : hi32;
    }
  }
  __device__ __forceinline__ void widen() {
    if (IS_FLOAT) { lo = nv32 ? (u64)lo32 : ~0ull; hi = (u64)hi32; bor = or32; band = nv32 ? (u64)and32 : ~0ull; }
    else {
      lo = nv32 ? (u64)(int64_t)(int32_t)lo32 : (u64)INT64_MAX;
      hi = nv32 ? (u64)(int64_t)(int32_t)hi32 : (u64)INT64_MIN;
      bor = nv32 ? (u64)(int64_t)(int32_t)or32 : 0ull;          // sign-extended images, like the 64-bit form
      band = nv32 ? (u64)(int64_t)(int32_t)and32 : ~0ull;
    }
    nna = na32; nvalid = nv32;
  }
  __device__ __forceinline__ void merge(u64 lo2, u64 hi2, u64 or2, u64 and2, u64 na2, u64 nv2) {
    if (IS_FLOAT) { lo = lo2 < lo ? lo2 : lo; hi = hi2 > hi ? hi2 : hi; }
    else {
      if ((int64_t)lo2 < (int64_t)lo) lo = lo2;
      if ((int64_t)hi2 > (int64_t)hi) hi = hi2;
    }
    bor |= or2; band &= and2; nna += na2; nvalid += nv2;
  }
};

// block reduction of the per-thread accumulators and the commit to the global ColStats
template <typename T, bool IS_FLOAT>
__device__ __forceinline__ void stats_commit(StatAcc<T, IS_FLOAT>& acc, ColStats* out)
{
  acc.widen();
  // warp reduce
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    u64 lo2 = __shfl_xor_sync(0xffffffffu, acc.lo, d);
    u64 hi2 = __shfl_xor_sync(0xffffffffu, acc.hi, d);
    u64 or2 = __shfl_xor_sync(0xffffffffu, acc.bor, d);
    u64 an2 = __shfl_xor_sync(0xffffffffu, acc.band, d);
    u64 na2 = __shfl_xor_sync(0xffffffffu, acc.nna, d);
    u64 nv2 = __shfl_xor_sync(0xffffffffu, acc.nvalid, d);
    acc.merge(lo2, hi2, or2, an2, na2, nv2);
  }
  __shared__ u64 sm[16][6];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    sm[warp][0] = acc.lo; sm[warp][1] = acc.hi; sm[warp][2] = acc.bor;
    sm[warp][3] = acc.band; sm[warp][4] = acc.nna; sm[warp][5] = acc.nvalid;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int nw = blockDim.x >> 5;
    for (int w = 1; w < nw; w++)
      acc.merge(sm[w][0], sm[w][1], sm[w][2], sm[w][3], sm[w][4], sm[w][5]);
    if (acc.nvalid) {
      if (IS_FLOAT) { atomicMin(&out->lo, acc.lo); atomicMax(&out->hi, acc.hi); }
      else {
        atomicMin(reinterpret_cast<long long*>(&out->lo), (long long)acc.lo);
        atomicMax(reinterpret_cast<long long*>(&out->hi), (long long)acc.hi);
      }
      atomicOr(&out->bits_or, acc.bor);
      atomicAnd(&out->bits_and, acc.band);
      atomicAdd(&out->nvalid, acc.nvalid);
    }
    if (acc.nna) atomicAdd(&out->nacount, acc.nna);
  }
}

template <typename T, bool IS_FLOAT>
__global__ void __launch_bounds__(512)
col_stats_kernel(const typename RawKey<T>::load_t* __restrict__ data, int64_t n, ColStats* out)
{
  typedef typename RawKey<T>::load_t L;
  constexpr int VEC = 16 / sizeof(L);
  StatAcc<T, IS_FLOAT> acc; acc.init();

  // 16-byte vector loads need a 16-byte aligned base: peel the (rare) unaligned head.
  int64_t head = (int64_t)(((16 - (reinterpret_cast<uintptr_t>(data) & 15)) & 15) / sizeof(L));
  if (head > n) head = n;
  const int64_t nvec = (n - head) / VEC;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint4* v4 = reinterpret_cast<const uint4*>(data + head);
  for (int64_t i = tid0; i < nvec; i += stride) {
    uint4 q = __ldg(v4 + i);
    L e[VEC];
    *reinterpret_cast<uint4*>(e) = q;
#pragma unroll
    for (int j = 0; j < VEC; j++) acc.add(e[j]);
  }
  for (int64_t i = head + nvec * VEC + tid0; i < n; i += stride) acc.add(data[i]);   // tail
  for (int64_t i = tid0; i < head; i += stride) acc.add(data[i]);                    // head

  stats_commit<T, IS_FLOAT>(acc, out);
}

// ---- statistics + per-tile histogram of the low 8 bits of u, one read of the column ------------------------
// The tiles are the radix passes' (4096 rows, 16 per CTA): the first pass turns the histogram into its digit
// counts (fold_counts_kernel, dtb_radix.cu) instead of reading the keys again in a count kernel.
template <typename T, bool IS_FLOAT>
__global__ void __launch_bounds__(PASS_THREADS)
col_stats_hist_kernel(const typename RawKey<T>::load_t* __restrict__ data, int64_t n, ColStats* out,
                      unsigned short* __restrict__ tile_hist, unsigned short* __restrict__ tile_na)
{
  typedef typename RawKey<T>::load_t L;
  __shared__ u32 h[256 + 1];                                   // [256]: NA rows of the tile
  StatAcc<T, IS_FLOAT> acc; acc.init();
  const int64_t cbase = (int64_t)blockIdx.x * CHUNK_ROWS;
  const int64_t cend = (cbase + CHUNK_ROWS < n) ? cbase + CHUNK_ROWS : n;
  for (int64_t base = cbase; base < cend; base += PASS_TILE) {
    h[threadIdx.x] = 0;
    if (threadIdx.x == 0) h[256] = 0;
    __syncthreads();
    const int64_t end = (base + PASS_TILE < cend) ? base + PASS_TILE : cend;
    if (end - base == PASS_TILE) {
      L raw[PASS_IPT];                                         // 16 independent coalesced loads in flight
#pragma unroll
      for (int j = 0; j < PASS_IPT; j++) raw[j] = data[base + threadIdx.x + j * PASS_THREADS];
#pragma unroll
      for (int j = 0; j < PASS_IPT; j++) {
        u64 u; const bool valid = RawKey<T>::get(raw[j], u);
        acc.add(raw[j]);
        atomicAdd(&h[valid ? (u32)u & 255u : 256u], 1u);
      }
    } else {
      for (int64_t i = base + threadIdx.x; i < end; i += PASS_THREADS) {
        const L raw = data[i];
        u64 u; const bool valid = RawKey<T>::get(raw, u);
        acc.add(raw);
        atomicAdd(&h[valid ? (u32)u & 255u : 256u], 1u);
      }
    }
    __syncthreads();
    const int64_t tile = base / PASS_TILE;
    tile_hist[(size_t)tile * 256 + threadIdx.x] = (unsigned short)h[threadIdx.x];     // a tile holds 4096 rows: fits
    if (threadIdx.x == 0) tile_na[tile] = (unsigned short)h[256];
    __syncthreads();
  }
  stats_commit<T, IS_FLOAT>(acc, out);
}

// ---- statistics of the column seen through a RowIndex (cut over selected rows) -------------------------------
// Position p reads data[order[p]]; an index outside [0, nrows) is an NA row.  Each thread issues GATHER_IPT index
// loads, then GATHER_IPT value loads, before it folds any of them.
constexpr int GATHER_IPT = 8;

template <typename T, bool IS_FLOAT, typename OrdT>
__global__ void __launch_bounds__(512)
col_stats_gather_kernel(const typename RawKey<T>::load_t* __restrict__ data, int64_t nrows,
                        const OrdT* __restrict__ order, int64_t n, ColStats* out)
{
  typedef typename RawKey<T>::load_t L;
  StatAcc<T, IS_FLOAT> acc; acc.init();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * GATHER_IPT;
  for (int64_t p0 = (int64_t)blockIdx.x * blockDim.x * GATHER_IPT + threadIdx.x; p0 < n; p0 += stride) {
    int64_t j[GATHER_IPT];
#pragma unroll
    for (int k = 0; k < GATHER_IPT; k++) {
      const int64_t p = p0 + (int64_t)k * blockDim.x;
      j[k] = p < n ? (int64_t)order[p] : -1;
    }
    L raw[GATHER_IPT];
#pragma unroll
    for (int k = 0; k < GATHER_IPT; k++) raw[k] = (j[k] >= 0 && j[k] < nrows) ? data[j[k]] : raw_na<T>();
#pragma unroll
    for (int k = 0; k < GATHER_IPT; k++) if (p0 + (int64_t)k * blockDim.x < n) acc.add(raw[k]);   // every position, NA rows included
  }
  stats_commit<T, IS_FLOAT>(acc, out);
}

template <bool IS_FLOAT>
static int stats_init(ColStats* d_stats, cudaStream_t s) {
  ColStats init;
  if (IS_FLOAT) { init.lo = ~0ull; init.hi = 0ull; }
  else { init.lo = (u64)INT64_MAX; init.hi = (u64)INT64_MIN; }
  init.bits_or = 0; init.bits_and = ~0ull; init.nacount = 0; init.nvalid = 0;
  DTB_CUDA_CHECK(cudaMemcpyAsync(d_stats, &init, sizeof(init), cudaMemcpyHostToDevice, s));
  return DTB_OK;
}

int launch_col_stats_gather(const void* data, int stype, int64_t nrows, const void* order, int order_is64, int64_t n,
                            ColStats* d_stats, cudaStream_t s) {
  return with_stype(stype, "Unable to compute statistics of a Column of stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    constexpr bool F = std::is_floating_point<T>::value;
    DTB_TRY(stats_init<F>(d_stats, s));
    if (n == 0) return DTB_OK;
    const int threads = 512;
    with_order(order, order_is64, [&](auto o) {
      col_stats_gather_kernel<T, F><<<grid_for((n + threads * GATHER_IPT - 1) / (threads * GATHER_IPT), 4), threads, 0,
                                      s>>>(reinterpret_cast<const typename RawKey<T>::load_t*>(data), nrows, o, n,
                                           d_stats);
    });
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  });
}

template <typename T, bool IS_FLOAT>
static int run_stats(const void* data, int64_t n, ColStats* d_stats, cudaStream_t s,
                     unsigned short* tile_hist, unsigned short* tile_na) {
  DTB_TRY(stats_init<IS_FLOAT>(d_stats, s));
  if (n > 0 && tile_hist) {
    const int64_t nchunks = (n + CHUNK_ROWS - 1) / CHUNK_ROWS;
    col_stats_hist_kernel<T, IS_FLOAT><<<(unsigned)nchunks, PASS_THREADS, 0, s>>>(
        reinterpret_cast<const typename RawKey<T>::load_t*>(data), n, d_stats, tile_hist, tile_na);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
  } else if (n > 0) {
    const int threads = 512;
    const int64_t want = (n / (16 / (int)sizeof(T)) + threads - 1) / threads;
    col_stats_kernel<T, IS_FLOAT><<<grid_for(want, 8), threads, 0, s>>>(
        reinterpret_cast<const typename RawKey<T>::load_t*>(data), n, d_stats);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
  }
  return DTB_OK;
}

int launch_col_stats(const void* data, int stype, int64_t n, ColStats* d_stats, cudaStream_t s) {
  return launch_col_stats_hist(data, stype, n, d_stats, nullptr, nullptr, s);
}

size_t stats_hist_bytes(int64_t n) { return sizeof(unsigned short) * 256 * (size_t)((n + PASS_TILE - 1) / PASS_TILE) + 256; }
size_t stats_na_bytes(int64_t n) { return sizeof(unsigned short) * (size_t)((n + PASS_TILE - 1) / PASS_TILE) + 256; }

int launch_col_stats_hist(const void* data, int stype, int64_t n, ColStats* d_stats, unsigned short* tile_hist,
                          unsigned short* tile_na, cudaStream_t s) {
  return with_stype(stype, "Unable to sort Column of stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    return run_stats<T, std::is_floating_point<T>::value>(data, n, d_stats, s, tile_hist, tile_na);
  });
}

}  // namespace dtb
