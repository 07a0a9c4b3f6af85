// dtb_groups.cu -- the Groupby group-offset scan.
//
// Replaces GroupGatherer (sort.h:119-148, sort_groups.cc:34-117): the
// reference collects cumulative group ends serially per radix range and
// memmove-compacts them.  Here the sorted composite keys are read once, rows
// whose group key (key >> group_shift) differs from their predecessor are
// flagged as group heads, and the head positions are compacted into
// offsets[] with a single-pass block scan + decoupled look-back over tiles.
//
// Output layout == Groupby::offsets_ (groupby.h:41-47): int32[ng+1],
// offsets[0] = 0, strictly increasing, offsets[ng] = nrows.
//
// Bound: HBM, 1 read of the sorted keys (sizeof(KeyT) B/row) + 4 B/group.
#include "dtb_common.cuh"

namespace dtb {

constexpr int OFF_THREADS = 512;
constexpr u64 OST_AGG  = 1ull << 62;
constexpr u64 OST_INCL = 2ull << 62;
constexpr u64 OST_MASK = (1ull << 62) - 1;

template <typename KeyT, bool FLAGS>
__global__ void __launch_bounds__(OFF_THREADS)
group_offsets_kernel(const KeyT* __restrict__ keys, int gshift, int64_t n,
                     int32_t* __restrict__ offsets, u64* d_ngroups, u64* scratch /*[0]=ticket, [1..]=status*/)
{
  constexpr int IPT = FLAGS ? 32 : 128 / sizeof(KeyT);         // consecutive rows per thread (<= 32)
  constexpr int NV = IPT * sizeof(KeyT) / 16;                   // 16-byte vector loads per thread
  constexpr int TILE = OFF_THREADS * IPT;
  constexpr int WARPS = OFF_THREADS / 32;
  __shared__ u64 s_tile;
  __shared__ u32 s_wsum[WARPS];
  __shared__ u64 s_prefix;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(&scratch[0], 1ull);
  __syncthreads();
  const int64_t tile = (int64_t)s_tile;
  const int64_t ntiles = (n + TILE - 1) / TILE;
  u64* status = scratch + 1;

  const int64_t p0 = tile * TILE + (int64_t)tid * IPT;
  KeyT k[IPT];
  KeyT prev = 0;
  if (p0 + IPT <= n) {
    const uint4* v = reinterpret_cast<const uint4*>(keys + p0);
    uint4 q[NV];
#pragma unroll
    for (int j = 0; j < NV; j++) q[j] = __ldg(v + j);
#pragma unroll
    for (int j = 0; j < NV; j++) *reinterpret_cast<uint4*>(&k[j * (IPT / NV)]) = q[j];
  } else {
#pragma unroll
    for (int i = 0; i < IPT; i++) k[i] = (p0 + i < n) ? keys[p0 + i] : (KeyT)0;
  }
  if (!FLAGS && p0 > 0 && p0 < n) prev = keys[p0 - 1];

  unsigned heads = 0; int c = 0;
#pragma unroll
  for (int i = 0; i < IPT; i++) {
    const int64_t p = p0 + i;
    bool h = false;
    if (p < n) {
      if (FLAGS) h = (p == 0) || (k[i] != 0);
      else {
        const KeyT before = (i == 0) ? prev : k[i - 1];
        h = (p == 0) || ((k[i] >> gshift) != (before >> gshift));
      }
    }
    heads |= (h ? 1u : 0u) << i;
    c += h;
  }

  // block exclusive scan of c
  u32 incl = (u32)c;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    u32 o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) s_wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    u32 w = lane < WARPS ? s_wsum[lane] : 0;
    u32 wi = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      u32 o = __shfl_up_sync(0xffffffffu, wi, d);
      if (lane >= d) wi += o;
    }
    if (lane < WARPS) s_wsum[lane] = wi - w;
    // warp 0 resolves the tile's exclusive prefix: publish the tile total, then inspect the
    // 32 preceding tiles per step (one status word per lane) until an inclusive prefix appears
    const u64 total = __shfl_sync(0xffffffffu, wi, WARPS - 1);
    if (lane == 0) st_relaxed_u64(&status[tile], (tile == 0 ? OST_INCL : OST_AGG) | total);
    u64 excl = 0;
    int64_t t = tile - 1;
    while (tile > 0) {
      const int64_t j = t - lane;
      const u64 sv = (j >= 0) ? ld_relaxed_u64(&status[j]) : OST_INCL;
      const u64 flag = sv & ~OST_MASK;
      const unsigned incl_m = __ballot_sync(0xffffffffu, flag == OST_INCL);
      const unsigned zero_m = __ballot_sync(0xffffffffu, flag == 0);
      const int first = incl_m ? (__ffs(incl_m) - 1) : 32;
      const unsigned relevant = (first < 31) ? ((2u << first) - 1u) : 0xffffffffu;
      if (zero_m & relevant) continue;                         // a needed predecessor has not published yet
      u64 c = (lane <= first) ? (sv & OST_MASK) : 0ull;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
      excl += c;
      if (first < 32) break;
      t -= 32;
    }
    if (lane == 0) {
      if (tile > 0) st_relaxed_u64(&status[tile], OST_INCL | (excl + total));
      s_prefix = excl;
      if (tile == ntiles - 1) {
        const u64 ng = excl + total;
        *d_ngroups = ng;
        offsets[ng] = (int32_t)n;
      }
    }
  }
  __syncthreads();
  u64 out = s_prefix + s_wsum[warp] + (incl - (u32)c);
#pragma unroll
  for (int i = 0; i < IPT; i++) {
    if (heads & (1u << i)) offsets[out++] = (int32_t)(p0 + i);
  }
}

template <typename KeyT>
__global__ void __launch_bounds__(256)
mark_heads_kernel(const KeyT* __restrict__ keys, int gshift, int64_t n, uint8_t* __restrict__ flags)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i > 0 && ((keys[i] >> gshift) != (keys[i - 1] >> gshift))) flags[i] = 1;
  }
}

int launch_mark_heads(const void* sorted_keys, int key_bytes, int group_shift, int64_t n,
                      uint8_t* flags, cudaStream_t s)
{
  if (n == 0) return DTB_OK;
  int64_t want = (n + 255) / 256;
  int grid = (int)(want > NUM_SMS * 16 ? NUM_SMS * 16 : want);
  if (key_bytes == 4) mark_heads_kernel<u32><<<grid, 256, 0, s>>>((const u32*)sorted_keys, group_shift, n, flags);
  else                mark_heads_kernel<u64><<<grid, 256, 0, s>>>((const u64*)sorted_keys, group_shift, n, flags);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// Offsets from a count table (small key domains)
// ===========================================================================
// count[x] = rows whose group key is x (filled by the last radix pass).  Three tiny kernels over the
// table (<= 4M entries): block sums, scan of the block sums, local scan + compaction.
constexpr int CT_BLOCK = 1024;                 // table entries per block (256 threads x 4)

__global__ void __launch_bounds__(256)
count_block_sums_kernel(const u32* __restrict__ count, u64* __restrict__ bsum /*[nb][2]*/)
{
  __shared__ u64 wr[8], wg[8];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint4 c = reinterpret_cast<const uint4*>(count)[(size_t)blockIdx.x * 256 + t];
  u64 rows = (u64)c.x + c.y + c.z + c.w;
  u64 grp = (c.x != 0) + (c.y != 0) + (c.z != 0) + (c.w != 0);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { rows += __shfl_xor_sync(0xffffffffu, rows, d); grp += __shfl_xor_sync(0xffffffffu, grp, d); }
  if (lane == 0) { wr[warp] = rows; wg[warp] = grp; }
  __syncthreads();
  if (t == 0) {
    u64 r = 0, g = 0;
    for (int w = 0; w < 8; w++) { r += wr[w]; g += wg[w]; }
    bsum[2 * (size_t)blockIdx.x] = r; bsum[2 * (size_t)blockIdx.x + 1] = g;
  }
}

__global__ void __launch_bounds__(1024)
count_scan_sums_kernel(u64* bsum, int nb)          // in place: exclusive prefixes; nb <= 4096
{
  __shared__ u64 sr[1024], sg[1024];
  const int t = threadIdx.x;
  u64 r[4], g[4], tr = 0, tg = 0;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int b = t * 4 + j;
    r[j] = b < nb ? bsum[2 * b] : 0; g[j] = b < nb ? bsum[2 * b + 1] : 0;
    tr += r[j]; tg += g[j];
  }
  sr[t] = tr; sg[t] = tg;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    u64 ar = 0, ag = 0;
    if (t >= d) { ar = sr[t - d]; ag = sg[t - d]; }
    __syncthreads();
    sr[t] += ar; sg[t] += ag;
    __syncthreads();
  }
  u64 er = sr[t] - tr, eg = sg[t] - tg;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int b = t * 4 + j;
    if (b < nb) { bsum[2 * b] = er; bsum[2 * b + 1] = eg; }
    er += r[j]; eg += g[j];
  }
}

__global__ void __launch_bounds__(256)
count_compact_kernel(const u32* __restrict__ count, const u64* __restrict__ bsum, int64_t n, int nb,
                     int32_t* __restrict__ offsets, u32* __restrict__ gkeys, u64* d_ngroups)
{
  __shared__ u64 wr[8], wg[8];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint4 cv = reinterpret_cast<const uint4*>(count)[(size_t)blockIdx.x * 256 + t];
  const u32 c[4] = {cv.x, cv.y, cv.z, cv.w};
  u64 rows = (u64)c[0] + c[1] + c[2] + c[3];
  u64 grp = (c[0] != 0) + (c[1] != 0) + (c[2] != 0) + (c[3] != 0);
  u64 ir = rows, ig = grp;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u64 a = __shfl_up_sync(0xffffffffu, ir, d), b = __shfl_up_sync(0xffffffffu, ig, d);
    if (lane >= d) { ir += a; ig += b; }
  }
  if (lane == 31) { wr[warp] = ir; wg[warp] = ig; }
  __syncthreads();
  u64 pr = 0, pg = 0;
#pragma unroll
  for (int w = 0; w < 8; w++) if (w < warp) { pr += wr[w]; pg += wg[w]; }
  u64 r = bsum[2 * (size_t)blockIdx.x] + pr + ir - rows;          // rows before this thread's entries
  u64 g = bsum[2 * (size_t)blockIdx.x + 1] + pg + ig - grp;       // groups before this thread's entries
#pragma unroll
  for (int j = 0; j < 4; j++) {
    if (c[j]) {
      offsets[g] = (int32_t)r;
      gkeys[g] = (u32)(((size_t)blockIdx.x * 256 + t) * 4 + j);
      g++; r += c[j];
    }
  }
  if (blockIdx.x == nb - 1 && t == 255) { *d_ngroups = g; offsets[g] = (int32_t)n; }
  // d_ngroups[1] = rows of the largest group (the reducers pick their streaming mode from it)
  u32 m = c[0] > c[1] ? c[0] : c[1];
  m = c[2] > m ? c[2] : m; m = c[3] > m ? c[3] : m;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { const u32 o = __shfl_xor_sync(0xffffffffu, m, d); m = o > m ? o : m; }
  if (lane == 0 && m) atomicMax(&d_ngroups[1], (u64)m);
}

int launch_offsets_from_counts(const uint32_t* count, int64_t table, int64_t n, int32_t* offsets,
                               uint32_t* gkeys, unsigned long long* d_ngroups, unsigned long long* scratch,
                               cudaStream_t s)
{
  const int nb = (int)(table / CT_BLOCK);
  if (nb < 1 || nb > 4096 || table % CT_BLOCK) { set_error("internal: bad count table size"); return DTB_EINVAL; }
  count_block_sums_kernel<<<nb, 256, 0, s>>>(count, scratch);
  count_scan_sums_kernel<<<1, 1024, 0, s>>>(scratch, nb);
  count_compact_kernel<<<nb, 256, 0, s>>>(count, scratch, n, nb, offsets, gkeys, d_ngroups);
  count_launch(3);
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int64_t offsets_num_tiles(int64_t n) {
  // the smallest tile (8-byte keys: 16 rows/thread) bounds the status array
  const int64_t tile = OFF_THREADS * 16;
  return (n + tile - 1) / tile;
}

int launch_group_offsets(const void* sorted_keys, int key_bytes, int group_shift, int64_t n,
                         int32_t* offsets_out, unsigned long long* d_ngroups,
                         unsigned long long* scratch, cudaStream_t s)
{
  if (n == 0) return DTB_OK;
  if (reinterpret_cast<uintptr_t>(sorted_keys) & 15) {
    set_error("internal: sorted key buffer must be 16-byte aligned"); return DTB_EINVAL;
  }
  if (key_bytes == 1) {
    const int64_t tile = OFF_THREADS * 32;
    group_offsets_kernel<uint8_t, true><<<(unsigned)((n + tile - 1) / tile), OFF_THREADS, 0, s>>>(
        (const uint8_t*)sorted_keys, 0, n, offsets_out, d_ngroups, scratch);
  } else if (key_bytes == 4) {
    const int64_t tile = OFF_THREADS * 32;
    group_offsets_kernel<u32, false><<<(unsigned)((n + tile - 1) / tile), OFF_THREADS, 0, s>>>(
        (const u32*)sorted_keys, group_shift, n, offsets_out, d_ngroups, scratch);
  } else {
    const int64_t tile = OFF_THREADS * 16;
    group_offsets_kernel<u64, false><<<(unsigned)((n + tile - 1) / tile), OFF_THREADS, 0, s>>>(
        (const u64*)sorted_keys, group_shift, n, offsets_out, d_ngroups, scratch);
  }
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// Dense per-key tables for the multi-GPU merge of per-group partials (SURVEY.md 8e: "a final NCCL
// reduce of per-group partials").  Every rank scatters its (group key, partial) list into a table
// indexed by key - kmin; the tables are all-reduced in place over NVLink (NCCL, by the caller) and
// compacted back into (key, value) lists with the count-table kernels above.  No re-sort, no host
// round trip between the kernels.
// ===========================================================================
template <typename KT>
__global__ void dense_scatter_kernel(const KT* __restrict__ keys, const u64* __restrict__ vals, int64_t n,
                                     int64_t kmin, int64_t size, u64* __restrict__ table, u32* __restrict__ present)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t x = (int64_t)keys[i] - kmin;
    if (x >= 0 && x < size) { table[x] = vals[i]; present[x] = 1u; }
  }
}

template <typename KT>
__global__ void dense_emit_kernel(const u32* __restrict__ gidx, const u64* __restrict__ table, int64_t ng, int64_t kmin,
                                  KT* __restrict__ out_keys, u64* __restrict__ out_vals)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const u32 x = gidx[g];
    out_keys[g] = (KT)(kmin + (int64_t)x);
    out_vals[g] = table[x];
  }
}

int launch_dense_scatter(const void* keys, int key_bytes, const void* vals, int64_t n, int64_t kmin, int64_t size,
                         void* table, uint32_t* present, cudaStream_t s)
{
  if (n == 0) return DTB_OK;
  const int grid = (int)((n + 255) / 256 > NUM_SMS * 8 ? NUM_SMS * 8 : (n + 255) / 256);
  if (key_bytes == 4) dense_scatter_kernel<int32_t><<<grid, 256, 0, s>>>((const int32_t*)keys, (const u64*)vals, n, kmin, size, (u64*)table, present);
  else                dense_scatter_kernel<int64_t><<<grid, 256, 0, s>>>((const int64_t*)keys, (const u64*)vals, n, kmin, size, (u64*)table, present);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int launch_dense_emit(const uint32_t* gidx, const void* table, int64_t ng, int64_t kmin, int key_bytes,
                      void* out_keys, void* out_vals, cudaStream_t s)
{
  if (ng == 0) return DTB_OK;
  const int grid = (int)((ng + 255) / 256 > NUM_SMS * 8 ? NUM_SMS * 8 : (ng + 255) / 256);
  if (key_bytes == 4) dense_emit_kernel<int32_t><<<grid, 256, 0, s>>>(gidx, (const u64*)table, ng, kmin, (int32_t*)out_keys, (u64*)out_vals);
  else                dense_emit_kernel<int64_t><<<grid, 256, 0, s>>>(gidx, (const u64*)table, ng, kmin, (int64_t*)out_keys, (u64*)out_vals);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

}  // namespace dtb
