// dtb_bucket.cu -- bucketed multi-reducer: every reducer of one value column in ONE sweep, with
// shared-memory accumulators instead of one L2 atomic per row and reducer.
//
// Replaces, for DT[:, {mean(v), min(v), max(v), count(v), ...}, by(k...)], the reference's one full
// pass per reducer per column (column/latent.cc:103-135 materialising sumprod.h / mean.h / minmax.h /
// count.h one after the other: 12 passes for BASELINE config C4) -- and this engine's own first
// version, which streamed the rows once per reducer and folded them with L2 atomics (1-2 per row and
// reducer: 15e9 atomics for C4 at 1e9 rows).
//
// When the normalised group key x spans 2^12 .. 2^20 values and no key is hot:
//   count    : rows per bucket, bucket = x >> 11 (<= 512 buckets of 2048 consecutive keys)      [once per call]
//   scatter  : the rows of up to BK_MAXCOLS value columns are partitioned by bucket -- x & 2047 as uint16
//              once, the raw values per column -- tile by tile: shared-memory counters hand out the slots of a tile (order inside a bucket does
//              not matter to a reducer), one global atomic per (tile, bucket) reserves the output range,
//              the tile is staged in shared memory and written out in bucket runs
//   aggregate: a CTA walks a fixed-size chunk of the partitioned rows bucket by bucket; every 8192-row tile is
//              counting-sorted by key in shared memory and the thread that owns a key folds its rows into
//              registers -- every requested word (int sum, float sum, count, min, max, NA count) at once --
//              and flushes them once per (chunk, bucket)
// Bytes per row: read 4 (x) + sum V, write 2 + sum V, read (2 + V) per column  (V = value bytes) -- against
// (4 + V) per reducer before; L2 atomics: ~2048 * words per 262144 rows instead of 1-2 per row.
//
// Bound: LSU wavefronts (scattered shared-memory stores, ~3-way bank conflicts) and HBM, about evenly.
#include <type_traits>
#include "dtb_common.cuh"

namespace dtb {

constexpr int BK_BITS = 11;                       // keys per bucket = 2048
constexpr int BK_KEYS = 1 << BK_BITS;
constexpr int BK_MAXB = 512;                      // buckets: group key domain <= 2^20
constexpr int BK_THREADS = 512;                   // = BK_MAXB: thread t owns bucket t in the tile scan
constexpr int BK_IPT = 8;                         // (16 rows x 256 threads ran at 24 % occupancy: 48 registers of row
constexpr int BK_TILE = BK_THREADS * BK_IPT;      //  state per thread) 4096 rows per tile
constexpr int64_t BK_CHUNK = 262144;              // rows per aggregate CTA

static inline int bk_grid(int64_t n, int threads) {
  const int64_t want = (n + threads - 1) / threads;
  return (int)(want > NUM_SMS * 16 ? NUM_SMS * 16 : (want < 1 ? 1 : want));
}

// ---- rows per (slab, bucket) -> start[slab][bucket] ------------------------------------------------
// A slab is a contiguous range of tiles.  Every slab gets its own output range inside every bucket
// (buckets stay contiguous: slab 0's rows, then slab 1's, ...), so that the scatter tiles of one slab
// reserve their runs from a cursor only they share: with ONE cursor per bucket the 244 k tiles of a 1e9-row
// column issued 244 k same-address L2 atomics-with-return per bucket (the LSUs sat half idle).
__global__ void __launch_bounds__(512)
bucket_count_kernel(const u32* __restrict__ xkeys, int gshift, int64_t n, int64_t slab_rows, u32* __restrict__ hist /*[nslabs][BK_MAXB]*/)
{
  __shared__ u32 h[BK_MAXB];
  for (int i = threadIdx.x; i < BK_MAXB; i += blockDim.x) h[i] = 0;
  __syncthreads();
  const int64_t r0 = (int64_t)blockIdx.x * slab_rows;
  const int64_t r1 = (r0 + slab_rows < n) ? r0 + slab_rows : n;
  for (int64_t i = r0 + threadIdx.x; i < r1; i += blockDim.x)
    atomicAdd(&h[(xkeys[i] >> gshift) >> BK_BITS], 1u);
  __syncthreads();
  for (int i = threadIdx.x; i < BK_MAXB; i += blockDim.x) hist[(size_t)blockIdx.x * BK_MAXB + i] = h[i];
}

// start[slab][b] = rows of buckets < b (all slabs) + rows of bucket b in slabs < slab; bstart[b] = start[0][b], bstart[nb] = n
__global__ void __launch_bounds__(BK_MAXB)
bucket_scan_kernel(u32* __restrict__ hist /*in: counts, out: starts*/, int nslabs, int nb, u32* __restrict__ bstart /*[nb+1]*/)
{
  __shared__ u32 s[BK_MAXB];
  const int t = threadIdx.x;
  u32 tot = 0;
  if (t < nb) for (int c = 0; c < nslabs; c++) tot += hist[(size_t)c * BK_MAXB + t];
  s[t] = tot;
  __syncthreads();
  for (int d = 1; d < BK_MAXB; d <<= 1) {
    const u32 a = t >= d ? s[t - d] : 0;
    __syncthreads();
    s[t] += a;
    __syncthreads();
  }
  if (t < nb) {
    u32 run = s[t] - tot;
    bstart[t] = run;
    for (int c = 0; c < nslabs; c++) { const u32 v = hist[(size_t)c * BK_MAXB + t]; hist[(size_t)c * BK_MAXB + t] = run; run += v; }
    if (t == nb - 1) bstart[nb] = s[t];
  }
}

int64_t bucket_slab_rows(int64_t n) {
  // ~4 slabs per SM, whole tiles per slab
  int64_t r = (n + NUM_SMS * 4 - 1) / (NUM_SMS * 4);
  r = (r + BK_TILE - 1) / BK_TILE * BK_TILE;
  return r < BK_TILE ? BK_TILE : r;
}
int bucket_num_slabs(int64_t n) { const int64_t r = bucket_slab_rows(n); return (int)((n + r - 1) / r); }

// hist: u32[nslabs * 512] (becomes the per-slab cursors' initial values), bstart: u32[nb + 1]
int launch_bucket_starts(const u32* xkeys, int gshift, int64_t n, int nb, u32* hist, u32* bstart, cudaStream_t s)
{
  const int nslabs = bucket_num_slabs(n);
  prof_begin("bucket_count", s);
  bucket_count_kernel<<<nslabs, 512, 0, s>>>(xkeys, gshift, n, bucket_slab_rows(n), hist);
  prof_end(s);
  bucket_scan_kernel<<<1, BK_MAXB, 0, s>>>(hist, nslabs, nb, bstart);
  count_launch(2);
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ---- partition value columns by bucket ---------------------------------------------------------------
// All the value columns of a sweep share one rank: the rows' tile slots are computed once (shared-memory
// counters, one reservation per (tile, bucket)), xlow is written once, and every column is then staged
// through the same shared-memory buffer and written out in bucket runs.  (One launch per column repeated the
// rank for every column.)
struct BucketCols {
  int ncols;
  int esz[BK_MAXCOLS];
  const void* in[BK_MAXCOLS];
  void* out[BK_MAXCOLS];
};

template <typename L, int TH, int IP>
__device__ __forceinline__ void bucket_load_column(const void* v, u64 (&val)[IP], int64_t base, int tile_n) {
#pragma unroll
  for (int i = 0; i < IP; i++) {
    const int p = threadIdx.x + i * TH;
    val[i] = p < tile_n ? (u64)reinterpret_cast<const L*>(v)[base + p] : 0ull;
  }
}
template <int TH, int IP>
__device__ __forceinline__ void bucket_load_column(int esz, const void* v, u64 (&val)[IP], int64_t base, int tile_n) {
  switch (esz) {
    case 1:  bucket_load_column<uint8_t, TH, IP>(v, val, base, tile_n); break;
    case 2:  bucket_load_column<uint16_t, TH, IP>(v, val, base, tile_n); break;
    case 4:  bucket_load_column<u32, TH, IP>(v, val, base, tile_n); break;
    default: bucket_load_column<u64, TH, IP>(v, val, base, tile_n); break;
  }
}
template <typename L, int TH, int IP>
__device__ __forceinline__ void bucket_stage_column(unsigned char* stage, const u64 (&val)[IP], const unsigned short (&slot)[IP], int tile_n) {
  L* sv = reinterpret_cast<L*>(stage);
#pragma unroll
  for (int i = 0; i < IP; i++) {
    const int p = threadIdx.x + i * TH;
    if (p < tile_n) sv[slot[i]] = (L)val[i];
  }
}
template <typename L, int TH>
__device__ __forceinline__ void bucket_write_column(void* v_out, const unsigned char* stage, const u32* sx, const u32* gbase, int tile_n) {
  const L* sv = reinterpret_cast<const L*>(stage);
  for (int p = threadIdx.x; p < tile_n; p += TH) reinterpret_cast<L*>(v_out)[gbase[sx[p] >> BK_BITS] + (u32)p] = sv[p];
}

// The next column's values are loaded into registers before the staged column is written out, and the
// columns alternate between two staging buffers: one barrier per column (2 CTAs and 2 x 80 KB per SM;
// 3 CTAs of 40 registers without the prefetch measured slower).
template <int TH, int IP>
__global__ void __launch_bounds__(TH, 2048 / TH > 2 ? 2 : 2048 / TH)
bucket_scatter_kernel(const u32* __restrict__ xkeys, int gshift, int64_t n, int64_t slab_rows,
                      u32* __restrict__ cursors /*[nslabs][BK_MAXB]*/, unsigned short* __restrict__ xlow_out,
                      const __grid_constant__ BucketCols cols, int stage_bytes)
{
  __shared__ u32 cnt[BK_MAXB];                 // rows of the bucket in this tile; then: tile slot of its first row
  __shared__ u32 gbase[BK_MAXB];               // (reserved global slot) - (tile slot) of the bucket
  __shared__ u32 wsum[TH / 32];
  static_assert(TH * IP == BK_TILE && TH >= BK_MAXB, "one tile, thread t owns bucket t in the scan");
  extern __shared__ __align__(16) unsigned char bk_stage[];      // group keys of the staged tile, then two value buffers
  u32* sx = reinterpret_cast<u32*>(bk_stage);
  unsigned char* stage0 = bk_stage + sizeof(u32) * BK_TILE;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t base = (int64_t)blockIdx.x * BK_TILE;
  u32* cursor = cursors + (size_t)(base / slab_rows) * BK_MAXB;       // the slab's own reservation cursors
  const int tile_n = (int)((n - base) < (int64_t)BK_TILE ? (n - base) : (int64_t)BK_TILE);
  for (int i = tid; i < BK_MAXB; i += TH) cnt[i] = 0;
  __syncthreads();

  u32 x[IP]; unsigned short slot[IP]; u64 val[IP];
#pragma unroll
  for (int i = 0; i < IP; i++) {
    const int p = tid + i * TH;
    x[i] = p < tile_n ? (xkeys[base + p] >> gshift) : 0xffffffffu;
  }
  bucket_load_column<TH, IP>(cols.esz[0], cols.in[0], val, base, tile_n);
#pragma unroll
  for (int i = 0; i < IP; i++)
    slot[i] = (x[i] != 0xffffffffu) ? (unsigned short)atomicAdd(&cnt[x[i] >> BK_BITS], 1u) : (unsigned short)0;
  __syncthreads();

  // exclusive scan of cnt[] over the buckets (one per thread), one global reservation per non-empty bucket
  const u32 c0 = tid < BK_MAXB ? cnt[tid] : 0u;
  u32 incl = c0;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const u32 o = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += o; }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  u32 wpre = 0;
#pragma unroll
  for (int w = 0; w < TH / 32; w++) if (w < warp) wpre += wsum[w];
  const u32 e0 = wpre + incl - c0;
  __syncthreads();
  if (tid < BK_MAXB) cnt[tid] = e0;
  if (c0) gbase[tid] = atomicAdd(&cursor[tid], c0) - e0;
  __syncthreads();

#pragma unroll
  for (int i = 0; i < IP; i++) {
    if (x[i] != 0xffffffffu) {
      slot[i] = (unsigned short)(cnt[x[i] >> BK_BITS] + slot[i]);
      sx[slot[i]] = x[i];
    }
  }
  __syncthreads();
  for (int p = tid; p < tile_n; p += TH) {
    const u32 xx = sx[p];
    xlow_out[gbase[xx >> BK_BITS] + (u32)p] = (unsigned short)(xx & (BK_KEYS - 1));
  }
  for (int c = 0; c < cols.ncols; c++) {
    const int esz = cols.esz[c];
    unsigned char* stage = stage0 + (size_t)(c & 1) * stage_bytes;
    switch (esz) {
      case 1:  bucket_stage_column<uint8_t, TH, IP>(stage, val, slot, tile_n); break;
      case 2:  bucket_stage_column<uint16_t, TH, IP>(stage, val, slot, tile_n); break;
      case 4:  bucket_stage_column<u32, TH, IP>(stage, val, slot, tile_n); break;
      default: bucket_stage_column<u64, TH, IP>(stage, val, slot, tile_n); break;
    }
    __syncthreads();       // also: every thread is done reading the other buffer (column c - 1)
    if (c + 1 < cols.ncols) bucket_load_column<TH, IP>(cols.esz[c + 1], cols.in[c + 1], val, base, tile_n);
    switch (esz) {
      case 1:  bucket_write_column<uint8_t, TH>(cols.out[c], stage, sx, gbase, tile_n); break;
      case 2:  bucket_write_column<uint16_t, TH>(cols.out[c], stage, sx, gbase, tile_n); break;
      case 4:  bucket_write_column<u32, TH>(cols.out[c], stage, sx, gbase, tile_n); break;
      default: bucket_write_column<u64, TH>(cols.out[c], stage, sx, gbase, tile_n); break;
    }
  }
}

// ---- aggregate ---------------------------------------------------------------------------------------
// A CTA walks a fixed-size chunk of one partitioned column bucket by bucket, tile by tile.  Inside a tile the
// rows are counting-sorted by their 11-bit key in shared memory (one native 32-bit shared-memory atomic per
// row hands out the rank, one scattered store places the value); thread t then owns keys 4t..4t+3, whose rows
// are now contiguous, and folds them into REGISTER accumulators: every requested word (int sum, float sum,
// count, min, max, NA count) at once, no 64-bit shared-memory atomics (they compile to CAS loops:
// ATOMS.CAST.SPIN -- the first version of this kernel spent 1.85 LSU wavefronts per row in them), and the
// valid-row count falls out of the walk.  The registers are flushed once per (chunk, bucket).
struct BucketAcc { u64* w[BK_NWORDS]; };        // global accumulator tables, indexed by group key x (NULL = not requested)

constexpr int BK_KPT = BK_KEYS / BK_THREADS;                  // 4 keys per thread

constexpr int BK_AIPT = 16;                                   // rows per thread and tile (8 rows, and re-reading
constexpr int BK_ATILE = BK_THREADS * BK_AIPT;                //  the keys in the place phase to save registers,
                                                              //  both measured slower)
template <typename T>
__global__ void __launch_bounds__(BK_THREADS, 2)
bucket_aggregate_kernel(const unsigned short* __restrict__ xlow, const typename RawKey<T>::load_t* __restrict__ v,
                        const u32* __restrict__ start, int nb, int64_t n, const __grid_constant__ BucketAcc acc)
{
  constexpr bool ISF = std::is_floating_point<T>::value;
  typedef typename RawKey<T>::load_t L;
  static_assert(BK_KPT == 4, "thread t owns keys 4t..4t+3 (one uint4 of counters)");
  extern __shared__ __align__(16) unsigned char ag_smem[];
  L* sval = reinterpret_cast<L*>(ag_smem);                                  // the tile's values, sorted by key
  u32* cnt = reinterpret_cast<u32*>(ag_smem + sizeof(L) * BK_ATILE);        // rows per key; then first slot of the key
  __shared__ u32 wsum[BK_THREADS / 32];
  __shared__ int s_b;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool want_sumf = acc.w[BK_SUMF] != nullptr;

  const int64_t c0 = (int64_t)blockIdx.x * BK_CHUNK;
  const int64_t c1 = (c0 + BK_CHUNK < n) ? c0 + BK_CHUNK : n;
  if (tid == 0) {                               // bucket that holds row c0: largest b with start[b] <= c0
    int lo = 0, hi = nb;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if ((int64_t)start[mid] <= c0) lo = mid; else hi = mid; }
    s_b = lo;
  }
  __syncthreads();
  for (int b = s_b; b < nb; b++) {
    const int64_t bs = start[b], be = start[b + 1];
    if (bs >= c1) break;
    const int64_t lo = bs > c0 ? bs : c0, hi = be < c1 ? be : c1;
    if (lo >= hi) continue;
    u64 sum_i[BK_KPT], kmin[BK_KPT], kmax[BK_KPT]; double sum_f[BK_KPT]; u32 nvalid[BK_KPT], nrows[BK_KPT];
#pragma unroll
    for (int j = 0; j < BK_KPT; j++) { sum_i[j] = 0; sum_f[j] = 0.0; kmin[j] = ~0ull; kmax[j] = 0; nvalid[j] = 0; nrows[j] = 0; }

    for (int64_t t0 = lo; t0 < hi; t0 += BK_ATILE) {
      const int tile_n = (int)((hi - t0) < (int64_t)BK_ATILE ? (hi - t0) : (int64_t)BK_ATILE);
      reinterpret_cast<uint4*>(cnt)[tid] = make_uint4(0, 0, 0, 0);
      __syncthreads();
      u32 kr[BK_AIPT];                                             // key | rank << 11
#pragma unroll
      for (int i = 0; i < BK_AIPT; i++) {
        const int p = tid + i * BK_THREADS;
        kr[i] = p < tile_n ? (u32)xlow[t0 + p] : 0xffffffffu;
      }
#pragma unroll
      for (int i = 0; i < BK_AIPT; i++)
        if (kr[i] != 0xffffffffu) kr[i] |= atomicAdd(&cnt[kr[i]], 1u) << BK_BITS;
      __syncthreads();
      // exclusive scan over the 2048 keys: thread t owns keys 4t..4t+3
      const uint4 c = reinterpret_cast<const uint4*>(cnt)[tid];
      const u32 tsum = c.x + c.y + c.z + c.w;
      u32 incl = tsum;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const u32 o = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += o; }
      if (lane == 31) wsum[warp] = incl;
      __syncthreads();
      u32 wpre = 0;
#pragma unroll
      for (int w = 0; w < BK_THREADS / 32; w++) if (w < warp) wpre += wsum[w];
      const u32 e = wpre + incl - tsum;
      reinterpret_cast<uint4*>(cnt)[tid] = make_uint4(e, e + c.x, e + c.x + c.y, e + c.x + c.y + c.z);
      __syncthreads();
      // place: eight loads in flight per thread, then the scattered stores
#pragma unroll
      for (int h = 0; h < BK_AIPT; h += 8) {
        L raw[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
          const int p = tid + (h + i) * BK_THREADS;
          raw[i] = p < tile_n ? v[t0 + p] : (L)0;
        }
#pragma unroll
        for (int i = 0; i < 8; i++)
          if (kr[h + i] != 0xffffffffu) sval[cnt[kr[h + i] & (BK_KEYS - 1)] + (kr[h + i] >> BK_BITS)] = raw[i];
      }
      __syncthreads();
      // walk the thread's four keys
      u32 pos = e;
      const u32 cj[BK_KPT] = {c.x, c.y, c.z, c.w};
#pragma unroll
      for (int j = 0; j < BK_KPT; j++) {
        nrows[j] += cj[j];
        for (u32 q = 0; q < cj[j]; q++, pos++) {
          const L raw = sval[pos];
          u64 u; const bool valid = RawKey<T>::get(raw, u);       // u: sign-extended int or float image
          if (!valid) continue;
          nvalid[j]++;
          if constexpr (ISF) {
            double d;
            if constexpr (std::is_same<T, float>::value) d = (double)__uint_as_float((u32)raw);
            else d = __longlong_as_double((long long)raw);
            sum_f[j] += d;
          } else {
            sum_i[j] += u;
            if (want_sumf) sum_f[j] += (double)(int64_t)u;
          }
          const u64 key = ISF ? u : (u ^ 0x8000000000000000ull);    // same encodings as dtb_reduce.cu:p_add
          const u64 km = ISF ? key : key - 1;
          kmin[j] = km < kmin[j] ? km : kmin[j];
          kmax[j] = key > kmax[j] ? key : kmax[j];
        }
      }
      // no barrier here: the next tile's stores into sval sit behind two of its barriers
    }
    const u64 xb = ((u64)b << BK_BITS) + (u64)tid * BK_KPT;
#pragma unroll
    for (int j = 0; j < BK_KPT; j++) {
      if (nrows[j] == 0) continue;
      if (acc.w[BK_CNT] && nvalid[j])              atomicAdd(&acc.w[BK_CNT][xb + j], (u64)nvalid[j]);
      if (acc.w[BK_CNTNA] && nrows[j] != nvalid[j]) atomicAdd(&acc.w[BK_CNTNA][xb + j], (u64)(nrows[j] - nvalid[j]));
      if (acc.w[BK_SUMI] && sum_i[j])              atomicAdd(&acc.w[BK_SUMI][xb + j], sum_i[j]);
      if (acc.w[BK_SUMF] && sum_f[j] != 0.0)       atomicAdd(reinterpret_cast<double*>(acc.w[BK_SUMF]) + xb + j, sum_f[j]);
      if (acc.w[BK_MIN] && kmin[j] != ~0ull)       atomicMin(&acc.w[BK_MIN][xb + j], kmin[j]);
      if (acc.w[BK_MAX] && kmax[j] != 0ull)        atomicMax(&acc.w[BK_MAX][xb + j], kmax[j]);
    }
  }
}

static inline size_t bk_align(size_t b) { return (b + 255) / 256 * 256; }
// scratch of one sweep: xlow u16[n] | the partitioned columns (sum_value_bytes per row) | the slabs' cursors
size_t bucket_scratch_bytes(int64_t n, int sum_value_bytes, int ncols) {
  return bk_align((size_t)n * 2) + (size_t)n * sum_value_bytes + 256 * (size_t)(ncols + 1) + bucket_starts_bytes(n);
}
size_t bucket_starts_bytes(int64_t n) { return sizeof(u32) * ((size_t)bucket_num_slabs(n) * BK_MAXB + 8); }

// One sweep over ncols <= BK_MAXCOLS value columns: partition them by bucket (one rank for all), then fold each
// into its accumulator tables.  acc_w[c][w]: global table of (1 << dbits) u64 for every requested word of
// column c (NULL otherwise), already set to the word's identity (~0 for BK_MIN, 0 otherwise).
// slab_starts / start: from launch_bucket_starts.
int launch_bucketed_reduce(const u32* xkeys, int gshift, int dbits, int ncols, const void* const* values, const int* stypes,
                           int64_t n, const u32* slab_starts, const u32* start, unsigned long long* const (*acc_w)[BK_NWORDS],
                           void* scratch, cudaStream_t s)
{
  if (n == 0 || ncols == 0) return DTB_OK;
  if (ncols > BK_MAXCOLS) { set_error("internal: too many columns in one bucket sweep"); return DTB_EINVAL; }
  const int nb = 1 << (dbits > BK_BITS ? dbits - BK_BITS : 0);
  if (nb > BK_MAXB) { set_error("internal: bucketed reducer needs a group key domain of at most 2^20"); return DTB_EINVAL; }
  unsigned short* xlow = (unsigned short*)scratch;
  char* at = (char*)scratch + bk_align((size_t)n * 2);
  BucketCols cols; cols.ncols = ncols;
  int maxb = 1;
  for (int c = 0; c < ncols; c++) {
    const int esz = stype_bytes(stypes[c]);
    if (!esz) { set_error("unsupported stype"); return DTB_ENOTIMPL; }
    cols.esz[c] = esz; cols.in[c] = values[c]; cols.out[c] = at;
    at += bk_align((size_t)n * esz);
    maxb = esz > maxb ? esz : maxb;
  }
  u32* cursor = (u32*)at;
  const int64_t slab_rows = bucket_slab_rows(n);
  DTB_CUDA_CHECK(cudaMemcpyAsync(cursor, slab_starts, sizeof(u32) * (size_t)bucket_num_slabs(n) * BK_MAXB, cudaMemcpyDeviceToDevice, s));
  const unsigned tiles = (unsigned)((n + BK_TILE - 1) / BK_TILE);
  const int stage_bytes = maxb * BK_TILE;
  const size_t sm_scatter = (size_t)4 * BK_TILE + (size_t)stage_bytes * (ncols > 1 ? 2 : 1);
  // 1024 threads x 4 rows: 32 registers, two CTAs = every warp slot of the SM (512 x 8 at 64 registers measured slower)
  DTB_CUDA_CHECK(cudaFuncSetAttribute(bucket_scatter_kernel<1024, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 20 * BK_TILE));
  prof_begin("bucket_scatter", s);
  bucket_scatter_kernel<1024, 4><<<tiles, 1024, sm_scatter, s>>>(xkeys, gshift, n, slab_rows, cursor, xlow, cols, stage_bytes);
  prof_end(s);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());

  const unsigned chunks = (unsigned)((n + BK_CHUNK - 1) / BK_CHUNK);
  for (int c = 0; c < ncols; c++) {
    BucketAcc acc;
    for (int w = 0; w < BK_NWORDS; w++) acc.w[w] = acc_w[c][w];
    prof_begin("bucket_aggregate", s);
    const size_t smem = (size_t)cols.esz[c] * BK_ATILE + sizeof(u32) * BK_KEYS;
#define DTB_AGG(T) { DTB_CUDA_CHECK(cudaFuncSetAttribute(bucket_aggregate_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
                     bucket_aggregate_kernel<T><<<chunks, BK_THREADS, smem, s>>>(xlow, (const typename RawKey<T>::load_t*)cols.out[c], start, nb, n, acc); }
    switch (stypes[c]) {
      case DTB_STYPE_BOOL: case DTB_STYPE_INT8:    DTB_AGG(int8_t)  break;
      case DTB_STYPE_INT16:                        DTB_AGG(int16_t) break;
      case DTB_STYPE_INT32: case DTB_STYPE_DATE32: DTB_AGG(int32_t) break;
      case DTB_STYPE_INT64: case DTB_STYPE_TIME64: DTB_AGG(int64_t) break;
      case DTB_STYPE_FLOAT32:                      DTB_AGG(float)   break;
      case DTB_STYPE_FLOAT64:                      DTB_AGG(double)  break;
      default: set_error("unsupported stype"); return DTB_ENOTIMPL;
    }
#undef DTB_AGG
    prof_end(s);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
  }
  return DTB_OK;
}

}  // namespace dtb
