// dtb_radix.cu -- stable LSD radix sort passes over normalised composite keys.
//
// Replaces SortContext::build_histogram / reorder_data / radix_psort /
// _radix_recurse (sort.cc:950-1353).  The reference is an MSD recursion over
// a chunk x radix size_t histogram with insertion-sort leaves -- a CPU idiom.
// Here every digit is one pass of three kernels:
//
//   count   : every CTA owns a contiguous CHUNK of 65536 rows and counts its digits
//             (shared-memory histogram) -> counts[chunk][digit]
//   scan    : per digit, exclusive prefix over the chunks; exclusive prefix over the digit
//             totals -> every (chunk, digit) knows its first output slot
//   scatter : the CTA walks its chunk tile by tile (4096 rows), ranks the rows of a tile with
//             warp-level peer masks in shared memory, reorders the tile in shared memory and
//             writes digit runs out coalesced, keeping the running digit offsets in registers.
//
// No look-back, no status words, no spinning: a first version used single-sweep tiles with
// a decoupled look-back; with ~600 tiles in flight the look-back walk was 40 % of the stall
// samples and 31 % of the instructions of the pass.  The price
// is one extra read of the keys per pass (K of 2(K+4) bytes per row).
//
// Stability (ties keep ascending row index, sort.cc:27-33): chunks and tiles are in row
// order and rows of a tile are ranked in (item, lane) = position order.
//
// Key normalisation (sort.cc:690-845) is evaluated on the fly in the first pass (count and
// scatter): no separate `x` array is materialised for single-column keys.
//
// Bound: HBM.  Algorithmic bytes per row per pass = read (key + idx) + write (key + idx);
// first pass reads the raw column only, last pass of a sort-only call writes idx only.
#include "dtb_common.cuh"

namespace dtb {

// ===========================================================================
// Composite key materialisation (multi-column keys)
// ===========================================================================
// Four rows per thread and column: the stype switch is taken once per four rows and the four loads of a
// column are in flight together (one row per thread cost 104 instructions per row).
template <typename T>
__device__ __forceinline__ void compose_col4(const KeyNorm& k, const int64_t (&row)[4], const bool (&in)[4], u64 (&x)[4]) {
  typedef typename RawKey<T>::load_t L;
  L raw[4];
#pragma unroll
  for (int r = 0; r < 4; r++) raw[r] = in[r] ? ((const L*)k.data)[row[r]] : (L)0;
#pragma unroll
  for (int r = 0; r < 4; r++) {
    u64 u; const bool valid = RawKey<T>::get(raw[r], u);
    x[r] |= norm_apply(valid, u, k) << k.lshift;
  }
}

template <typename KeyT>
__global__ void __launch_bounds__(256)
compose_keys_kernel(KeyPlan kp, int64_t n, const int32_t* __restrict__ idx, KeyT* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x * 4 + threadIdx.x; i0 < n; i0 += stride) {
    int64_t row[4]; bool in[4]; u64 x[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int64_t i = i0 + (int64_t)r * blockDim.x;           // consecutive threads, consecutive rows
      in[r] = i < n;
      row[r] = !in[r] ? 0 : (idx ? (int64_t)(u32)idx[i] : i);   // later rounds see the rows in the current order (ids are 32-bit patterns)
      x[r] = 0;
    }
    for (int c = 0; c < kp.nkeys; c++) {
      const KeyNorm& k = kp.k[c];
      switch (k.stype) {
        case DTB_STYPE_BOOL: case DTB_STYPE_INT8:    compose_col4<int8_t>(k, row, in, x); break;
        case DTB_STYPE_INT16:                        compose_col4<int16_t>(k, row, in, x); break;
        case DTB_STYPE_INT32: case DTB_STYPE_DATE32: compose_col4<int32_t>(k, row, in, x); break;
        case DTB_STYPE_INT64: case DTB_STYPE_TIME64: compose_col4<int64_t>(k, row, in, x); break;
        case DTB_STYPE_FLOAT32:                      compose_col4<float>(k, row, in, x); break;
        default:                                     compose_col4<double>(k, row, in, x); break;
      }
    }
#pragma unroll
    for (int r = 0; r < 4; r++) if (in[r]) out[i0 + (int64_t)r * blockDim.x] = (KeyT)x[r];
  }
}

int launch_compose_keys(const KeyPlan& kp, int64_t n, const int32_t* idx, void* keys_out, int key_bytes,
                        cudaStream_t s)
{
  if (n == 0) return DTB_OK;
  int64_t want = (n + 1023) / 1024;
  int grid = (int)(want > NUM_SMS * 16 ? NUM_SMS * 16 : want);
  if (key_bytes == 4) compose_keys_kernel<u32><<<grid, 256, 0, s>>>(kp, n, idx, (u32*)keys_out);
  else                compose_keys_kernel<u64><<<grid, 256, 0, s>>>(kp, n, idx, (u64*)keys_out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// Pass geometry
// ===========================================================================
// Digits are at most 8 bits (256 bins).  Wider digits were built and measured twice and removed: round 1, two
// 10-bit ballot-ranked passes over 1024 bins, slower than three 7/7/6-bit passes on 20-bit keys; round 2,
// 1024/2048 bins ranked with shared-memory atomics, slower scatter -- 16-byte output runs and 16-32 KB of per-warp tables cost more LSU
// wavefronts than the pass they save.
// PASS_THREADS / PASS_IPT / PASS_TILE (4096 rows) / CHUNK_TILES / CHUNK_ROWS (65536 rows per count CTA): dtb_common.cuh

int64_t radix_num_chunks(int64_t n) { return (n + CHUNK_ROWS - 1) / CHUNK_ROWS; }

// ===========================================================================
// count: tile_pre[tile][digit] (u16, rows of the digit in the earlier tiles of the chunk) and counts[chunk][digit]
// ===========================================================================
template <typename KeyT, typename Src, int NBINS>
__global__ void __launch_bounds__(PASS_THREADS)
count_kernel(const __grid_constant__ Src src, int64_t n, int shift, u32 mask, u32* __restrict__ counts,
             unsigned short* __restrict__ tile_pre, KeyT* __restrict__ keys_out)
{
  // keys_out (first pass over a raw column): also store the normalised keys, so that the scatter
  // kernel of this pass streams 32/64-bit keys like every later pass instead of re-normalising.
  constexpr int BPT = NBINS / PASS_THREADS;
  __shared__ u32 h[NBINS];
  const int64_t cbase = (int64_t)blockIdx.x * CHUNK_ROWS;
  const int64_t cend = (cbase + CHUNK_ROWS < n) ? cbase + CHUNK_ROWS : n;
  u32 total[BPT];                                          // rows of digit tid + j*THREADS in this chunk
#pragma unroll
  for (int j = 0; j < BPT; j++) total[j] = 0;
  for (int64_t base = cbase; base < cend; base += PASS_TILE) {
#pragma unroll
    for (int j = 0; j < BPT; j++) h[threadIdx.x + j * PASS_THREADS] = 0;
    __syncthreads();
    const int64_t end = (base + PASS_TILE < cend) ? base + PASS_TILE : cend;
    if (end - base == PASS_TILE) {
      // coalesced: consecutive threads read consecutive rows; 16 independent loads in flight per thread
      KeyT k[PASS_IPT];
#pragma unroll
      for (int j = 0; j < PASS_IPT; j++) k[j] = src.load(base + threadIdx.x + j * PASS_THREADS);
      if (keys_out) {
#pragma unroll
        for (int j = 0; j < PASS_IPT; j++) keys_out[base + threadIdx.x + j * PASS_THREADS] = k[j];
      }
#pragma unroll
      for (int j = 0; j < PASS_IPT; j++) atomicAdd(&h[(u32)(k[j] >> shift) & mask], 1u);
    } else {
      for (int64_t i = base + threadIdx.x; i < end; i += PASS_THREADS) {
        const KeyT kk = src.load(i);
        if (keys_out) keys_out[i] = kk;
        atomicAdd(&h[(u32)(kk >> shift) & mask], 1u);
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < BPT; j++) {
      const u32 c = h[threadIdx.x + j * PASS_THREADS];
      // rows of this digit in the EARLIER tiles of the chunk (<= 15 * 4096, fits 16 bits): the scatter
      // kernel adds it to the digit base and the chunk offset without walking the chunk's tiles
      tile_pre[(size_t)(base / PASS_TILE) * NBINS + threadIdx.x + j * PASS_THREADS] = (unsigned short)total[j];
      total[j] += c;
    }
  }
#pragma unroll
  for (int j = 0; j < BPT; j++) counts[(size_t)blockIdx.x * NBINS + threadIdx.x + j * PASS_THREADS] = total[j];
}

// First pass over a raw column, counts from the statistics kernel's histogram of the low 8 bits of u
// (launch_col_stats_hist): x = +-(u - edge) + inc keeps a function of those bits in its low 8 bits when no
// constant low bits are dropped, so raw bin b lands in digit (+-(b - edge) + inc) & mask, the NA rows in
// na_value & mask.  Same outputs as count_kernel; reads 512 bytes per tile instead of the tile's keys.
__global__ void __launch_bounds__(256)
fold_counts_kernel(const unsigned short* __restrict__ tile_hist, const unsigned short* __restrict__ tile_na, int64_t ntiles,
                   u32 edge8, u32 inc8, int desc, u32 na_digit, u32 mask, u32* __restrict__ counts,
                   unsigned short* __restrict__ tile_pre)
{
  __shared__ u32 dg[256];
  const int t = threadIdx.x;
  const int64_t t0 = (int64_t)blockIdx.x * CHUNK_TILES;
  const int64_t t1 = (t0 + CHUNK_TILES < ntiles) ? t0 + CHUNK_TILES : ntiles;
  const u32 d = (desc ? (edge8 - (u32)t + inc8) : ((u32)t - edge8 + inc8)) & mask;     // digit of raw bin t
  u32 total = 0;
  for (int64_t tile = t0; tile < t1; tile++) {
    dg[t] = 0;
    __syncthreads();
    const u32 c = tile_hist[(size_t)tile * 256 + t];
    if (c) atomicAdd(&dg[d], c);
    if (t == 0) { const u32 na = tile_na[tile]; if (na) atomicAdd(&dg[na_digit], na); }
    __syncthreads();
    tile_pre[(size_t)tile * 256 + t] = (unsigned short)total;
    total += dg[t];
    __syncthreads();
  }
  counts[(size_t)blockIdx.x * 256 + t] = total;
}

// ===========================================================================
// scan: offs[chunk][digit] = sum over earlier chunks (in place); total[digit]
// then base[digit] = exclusive scan of total[]; hmax = largest total (skew detector)
// ===========================================================================
__global__ void __launch_bounds__(256)
chunk_scan_kernel(u32* __restrict__ counts, int64_t nchunks, int nbins, u32* __restrict__ total)
{
  // one CTA per digit walks the chunks, 1024 per round: every thread owns four consecutive chunks (four strided
  // loads in flight; one chunk per thread and round took 60 dependent rounds for 1e9 rows)
  __shared__ u32 wsum[8];
  __shared__ u32 s_carry;
  const int d = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (t == 0) s_carry = 0;
  __syncthreads();
  for (int64_t c0 = 0; c0 < nchunks; c0 += 1024) {
    const int64_t c = c0 + (int64_t)t * 4;
    u32 v[4];
#pragma unroll
    for (int j = 0; j < 4; j++) v[j] = (c + j < nchunks) ? counts[(size_t)(c + j) * nbins + d] : 0;
    const u32 tsum = v[0] + v[1] + v[2] + v[3];
    u32 incl = tsum;
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) { const u32 o = __shfl_up_sync(0xffffffffu, incl, k); if (lane >= k) incl += o; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    u32 wpre = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) if (w < warp) wpre += wsum[w];
    const u32 carry = s_carry;
    u32 e = carry + wpre + incl - tsum;
#pragma unroll
    for (int j = 0; j < 4; j++) { if (c + j < nchunks) counts[(size_t)(c + j) * nbins + d] = e; e += v[j]; }
    __syncthreads();
    if (t == 255) s_carry = carry + wpre + incl;
    __syncthreads();
  }
  if (t == 0) total[d] = s_carry;
}

template <int NBINS>
__global__ void __launch_bounds__(256)
digit_base_kernel(const u32* __restrict__ total, u32* __restrict__ base, u32* __restrict__ hmax)
{
  constexpr int BPT = NBINS / 256;                        // thread t owns digits t*BPT .. t*BPT+BPT-1
  __shared__ u32 wsum[8];
  __shared__ u32 wmax[8];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  u32 v[BPT], tsum = 0, m = 0;
#pragma unroll
  for (int j = 0; j < BPT; j++) { v[j] = total[t * BPT + j]; tsum += v[j]; m = v[j] > m ? v[j] : m; }
  u32 incl = tsum;
#pragma unroll
  for (int k = 1; k < 32; k <<= 1) { const u32 o = __shfl_up_sync(0xffffffffu, incl, k); if (lane >= k) incl += o; }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) { const u32 o = __shfl_xor_sync(0xffffffffu, m, k); m = o > m ? o : m; }
  if (lane == 31) wsum[warp] = incl;
  if (lane == 0) wmax[warp] = m;
  __syncthreads();
  u32 wpre = 0;
#pragma unroll
  for (int w = 0; w < 8; w++) if (w < warp) wpre += wsum[w];
  u32 e = wpre + incl - tsum;
#pragma unroll
  for (int j = 0; j < BPT; j++) { base[t * BPT + j] = e; e += v[j]; }
  if (t == 0 && hmax) {
    u32 mm = 0;
    for (int w = 0; w < 8; w++) mm = wmax[w] > mm ? wmax[w] : mm;
    *hmax = mm;
  }
}

// ===========================================================================
// scatter
// ===========================================================================
template <typename KeyT, typename Src>
struct PassArgs {
  Src            src;
  const int32_t* idx_in;        // NULL = identity
  KeyT*          keys_out;      // NULL = do not write keys
  int32_t*       idx_out;
  int64_t        n;
  int            shift;
  u32            mask;
  const u32*     chunk_offs;    // [nchunks][NBINS] rows of this digit in earlier chunks
  const u32*     digit_base;    // [NBINS] first output slot of every digit
  const unsigned short* tile_pre;      // [ntiles][NBINS] rows of this digit in the earlier tiles of the chunk
  u32*           group_count;   // optional (last pass, small key domains): rows per group key
  int            group_shift;
  int            narrow;        // 64-bit keys only, > 0: write (key >> narrow) as uint32 -- the low bits are consumed
};

// ---- TMA 1-D bulk copy (cp.async.bulk, SASS UBLKCP) completing on an mbarrier -----------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, u32 count) {
  const u32 a = (u32)__cvta_generic_to_shared(bar);
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(a), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");      // visible to the async proxy
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, u32 bytes, uint64_t* bar) {
  const u32 d = (u32)__cvta_generic_to_shared(smem_dst), b = (u32)__cvta_generic_to_shared(bar);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(b), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(d), "l"(gsrc), "r"(bytes), "r"(b) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, u32 parity) {
  const u32 b = (u32)__cvta_generic_to_shared(bar);
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" :: "r"(b), "r"(parity) : "memory");
}

template <typename KeyT, int NBINS> struct PassCfg {
  static constexpr int WARPS = PASS_THREADS / 32;
  // the incoming row ids of the tile are staged in shared memory by one TMA bulk copy
  static constexpr bool USE_RIDX = true;
  static constexpr int MINB = (sizeof(KeyT) == 4) ? 4 : 3;
  static constexpr size_t SMEM = sizeof(unsigned short) * WARPS * NBINS + sizeof(u32) * (NBINS + 4)
                               + (sizeof(KeyT) + sizeof(int32_t)) * PASS_TILE
                               + (USE_RIDX ? sizeof(int32_t) * PASS_TILE : 0);
};

// One tile per CTA.
// Shared memory: whist[WARPS][NBINS] u16 | bin_dst[NBINS] u32 | skey[TILE] | sidx[TILE] | ridx[TILE]
// (the per-warp peer-mask table of the rank phase aliases skey/sidx, idle until the reorder phase).
// With 32-bit keys the sorted tile is staged as interleaved (key, row id) pairs so that the
// scattered shared-memory write of the reorder phase is ONE 8-byte store per row, not two
// 4-byte stores: shared-memory wavefronts, not HBM, bound this kernel.
// Thread t owns the BPT = NBINS/256 consecutive digits t*BPT.. in the scan phase.
template <typename KeyT, typename Src, int NBINS, bool FULL, int NB>
__device__ __forceinline__ void scatter_tile(const PassArgs<KeyT, Src>& a, unsigned char* smem_raw, u32* s_wsum,
                                             uint64_t* s_bar, const int64_t base, const int tile_n,
                                             const u32 (&bin_run)[NBINS / PASS_THREADS])
{
  constexpr int THREADS = PASS_THREADS, IPT = PASS_IPT, TILE = PASS_TILE;
  constexpr int WARPS = THREADS / 32;
  constexpr int BPT = NBINS / THREADS;
  constexpr bool USE_RIDX = PassCfg<KeyT, NBINS>::USE_RIDX;
  unsigned short* whist = reinterpret_cast<unsigned short*>(smem_raw);
  u32* bin_dst    = reinterpret_cast<u32*>(smem_raw + sizeof(unsigned short) * WARPS * NBINS);
  KeyT* skey      = reinterpret_cast<KeyT*>(bin_dst + NBINS + 4);
  int32_t* sidx   = reinterpret_cast<int32_t*>(skey + TILE);
  int32_t* ridx   = sidx + TILE;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool have_idx = a.idx_in != nullptr;

  // ---- clear the per-warp digit counters and peer masks; prefetch the row ids ----
  {
    u32* z = reinterpret_cast<u32*>(whist);
#pragma unroll
    for (int j = 0; j < WARPS * NBINS / 2 / THREADS; j++) z[tid + j * THREADS] = 0;
    if (USE_RIDX && have_idx) {
      const int32_t* g = a.idx_in + base;
      if (FULL) {
        // the whole 16 KB row-id tile is one TMA bulk copy issued by one thread; it lands in shared
        // memory while the tile is being ranked and is awaited (mbarrier) before the reorder phase
        if (tid == 0) { mbar_init(s_bar, 1); tma_load_1d(ridx, g, (u32)(TILE * sizeof(int32_t)), s_bar); }
      } else {
        for (int p = tid; p < tile_n; p += THREADS) ridx[p] = g[p];
      }
    }
  }

  // ---- load keys (warp-striped: item i of lane l sits at warp_base + i*32 + l) ----
  KeyT key[IPT];
  const int wbase = warp * 32 * IPT;
  {
    typename Src::raw_t raw[IPT];                                // every load of the tile in flight first ...
#pragma unroll
    for (int i = 0; i < IPT; i++) {
      const int lp = wbase + i * 32 + lane;
      raw[i] = (FULL || lp < tile_n) ? a.src.load_raw(base + lp) : (typename Src::raw_t)0;
    }
#pragma unroll
    for (int i = 0; i < IPT; i++) {                              // ... then normalised (identity for packed keys)
      const int lp = wbase + i * 32 + lane;
      key[i] = (FULL || lp < tile_n) ? a.src.norm(raw[i]) : (KeyT)0;
    }
  }
  // first output slot of the thread's digits (loaded by the caller before the keys, parked here until
  // the scan phase: the store waits for those loads only after the key loads are in flight)
#pragma unroll
  for (int j = 0; j < BPT; j++) bin_dst[tid * BPT + j] = bin_run[j];
  __syncthreads();

  // ---- rank inside the warp: rows with equal digits keep (item, lane) order ----
  // The lanes holding the same digit ("peers") are found with one __ballot_sync per digit bit
  // (peers = AND over the bits of "lanes whose bit equals mine"), NB = digit width of the pass: no
  // shared-memory traffic, and the cost does not depend on how the digits are distributed.
  // Measured against a shared-memory atomicOr on a per-warp mask table (one word per digit): C2 scatter
  // passes and the float64 sort got faster; a hot digit made the atomicOr form serialise on one word.
  // Never MATCH.ANY: it issues far more slowly than a ballot and would bound the whole kernel
  // (scripts/ubench/match_bench.cu measures it).
  u32 rank2[IPT / 2];                                         // two 16-bit ranks per register
  unsigned short* myhist = whist + warp * NBINS;
  const unsigned lt = lanemask_lt();
#pragma unroll
  for (int i = 0; i < IPT; i++) {
    const bool valid = FULL || (wbase + i * 32 + lane) < tile_n;
    const u32 d = (u32)(key[i] >> a.shift) & a.mask;
    unsigned peers = FULL ? 0xffffffffu : __ballot_sync(0xffffffffu, valid);
#pragma unroll
    for (int b = 0; b < NB; b++) {
      // peers &= (lanes whose bit b equals mine): 4 instructions per bit (LOP3->P, VOTE, @!P NOT, AND)
      asm("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\t"
          "and.b32 t, %1, %2;\n\t"
          "setp.ne.u32 p, t, 0;\n\t"
          "vote.sync.ballot.b32 t, p, 0xffffffff;\n\t"
          "@!p not.b32 t, t;\n\t"
          "and.b32 %0, %0, t;\n\t}"
          : "+r"(peers) : "r"(d), "r"(1u << b));
    }
    const unsigned short cnt = valid ? myhist[d] : (unsigned short)0;
    const unsigned before = peers & lt;
    const u32 r = (u32)cnt + (u32)__popc(before);
    if (i & 1) rank2[i >> 1] |= r << 16; else rank2[i >> 1] = r;
    __syncwarp();                                               // all reads of this round precede the update
    if (valid && before == 0) myhist[d] = cnt + (unsigned short)__popc(peers);
    __syncwarp();
  }
  __syncthreads();

  // ---- per digit: prefix over warps, scan over digits, output offsets ----
  const int b0 = tid * BPT;                                     // first of the thread's BPT consecutive digits
  u32 run[BPT];
#pragma unroll
  for (int j = 0; j < BPT; j++) run[j] = 0;
#pragma unroll
  for (int w = 0; w < WARPS; w++) {
#pragma unroll
    for (int j = 0; j < BPT; j++) run[j] += whist[w * NBINS + b0 + j];
  }
  u32 tsum = 0;
#pragma unroll
  for (int j = 0; j < BPT; j++) tsum += run[j];
  u32 incl = tsum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u32 o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) s_wsum[warp] = incl;
  __syncthreads();
  u32 wpre = 0;
#pragma unroll
  for (int w = 0; w < WARPS; w++) if (w < warp) wpre += s_wsum[w];
  u32 tstart = incl - tsum + wpre;                               // first tile slot of digit b0
#pragma unroll
  for (int j = 0; j < BPT; j++) {
    u32 pre = tstart;                                            // tile slot of warp w's first row of digit b0+j
#pragma unroll
    for (int w = 0; w < WARPS; w++) {
      const u32 c = whist[w * NBINS + b0 + j];
      whist[w * NBINS + b0 + j] = (unsigned short)pre;
      pre += c;
    }
    bin_dst[b0 + j] -= tstart;                                   // was: the digit's first output slot (set by the caller)
    tstart += run[j];
  }
  if (USE_RIDX && have_idx && FULL) mbar_wait(s_bar, 0);
  __syncthreads();

  // ---- reorder the tile in shared memory ----
#pragma unroll
  for (int i = 0; i < IPT; i++) {
    const int pos = wbase + i * 32 + lane;
    if (FULL || pos < tile_n) {
      const u32 d = (u32)(key[i] >> a.shift) & a.mask;
      const u32 lp = (u32)myhist[d] + ((rank2[i >> 1] >> (16 * (i & 1))) & 0xffffu);
      const int32_t r = !have_idx ? (int32_t)(base + pos) : (USE_RIDX ? ridx[pos] : a.idx_in[base + pos]);
      if constexpr (sizeof(KeyT) == 4) {
        reinterpret_cast<uint2*>(skey)[lp] = make_uint2((u32)key[i], (u32)r);      // pairs span skey+sidx
      } else {
        skey[lp] = key[i];
        sidx[lp] = r;
      }
    }
  }
  __syncthreads();
}

// key of the sorted tile's slot q (32-bit keys are staged as (key, row id) pairs)
// (Staging the first pass of keys below 2^20 as one word per row, key << 12 | tile position -- a 4-byte
// scattered store instead of an 8-byte one -- was measured slower on EVERY pass for the extra uniform
// branch and registers, no gain on the first.)
template <typename KeyT>
__device__ __forceinline__ KeyT staged_key(const KeyT* skey, int q) {
  if constexpr (sizeof(KeyT) == 4) return (KeyT)reinterpret_cast<const uint2*>(skey)[q].x;
  else return skey[q];
}

template <typename KeyT, typename Src, int NBINS, int MINB, int NB>
__global__ void __launch_bounds__(PASS_THREADS, MINB)
scatter_kernel(const __grid_constant__ PassArgs<KeyT, Src> a)
{
  constexpr int THREADS = PASS_THREADS, TILE = PASS_TILE;
  constexpr int WARPS = THREADS / 32;
  constexpr int BPT = NBINS / THREADS;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ u32 s_wsum[WARPS];
  __shared__ __align__(8) uint64_t s_bar;                       // mbarrier of the row-id TMA copy
  u32* bin_dst    = reinterpret_cast<u32*>(smem_raw + sizeof(unsigned short) * WARPS * NBINS);
  KeyT* skey      = reinterpret_cast<KeyT*>(bin_dst + NBINS + 4);
  int32_t* sidx   = reinterpret_cast<int32_t*>(skey + TILE);

  // One tile per CTA: neighbouring tiles run at the same time on different SMs, so the partial
  // sectors at the ends of their digit runs meet in L2 before they are evicted.
  const int tid = threadIdx.x;
  const int64_t tile = blockIdx.x;
  const int64_t base = tile * TILE;
  const int tile_n = (int)((a.n - base) < (int64_t)TILE ? (a.n - base) : (int64_t)TILE);
  const int64_t chunk = tile / CHUNK_TILES;

  // first output slot of the thread's digits for this tile: digit base + earlier chunks + earlier
  // tiles of the chunk (three independent loads, issued ahead of the key loads)
  u32 bin_run[BPT];
#pragma unroll
  for (int j = 0; j < BPT; j++) {
    const int b = tid * BPT + j;
    bin_run[j] = a.digit_base[b] + a.chunk_offs[(size_t)chunk * NBINS + b] + (u32)a.tile_pre[(size_t)tile * NBINS + b];
  }

  if (tile_n == TILE) scatter_tile<KeyT, Src, NBINS, true,  NB>(a, smem_raw, s_wsum, &s_bar, base, tile_n, bin_run);
  else                scatter_tile<KeyT, Src, NBINS, false, NB>(a, smem_raw, s_wsum, &s_bar, base, tile_n, bin_run);

  // ---- coalesced scatter: consecutive threads write consecutive slots of a digit run ----
  const int lane = tid & 31;
#pragma unroll 4
  for (int p0 = 0; p0 < tile_n; p0 += THREADS) {
    const int p = p0 + tid;
    const bool valid = p < tile_n;
    KeyT k = 0; int32_t rid = 0;
    if (valid) {
      if constexpr (sizeof(KeyT) == 4) {
        const uint2 kv = reinterpret_cast<const uint2*>(skey)[p];
        k = (KeyT)kv.x; rid = (int32_t)kv.y;
      } else {
        k = skey[p]; rid = sidx[p];
      }
    }
    if (a.group_count) {
      // Last pass: the tile is sorted by the full composite key (its rows arrive sorted by the lower
      // digits), so equal group keys are adjacent.  Every run of equal group keys adds its length to
      // count[group key]; the Groupby offsets are then a scan over that L2-resident table instead of a
      // pass over 4n bytes of sorted keys.  Only the run HEADS act: the row at tile slot p > 0 whose
      // predecessor holds another key closes that run (+p) and opens its own (-p, mod 2^32); the tile's
      // last row adds the tile length.  Two atomics per run however many warps it spans -- one atomic
      // per warp and run made few-key inputs serialise on a handful of L2 addresses.
      const u32 x = valid ? (u32)(k >> a.group_shift) : 0xffffffffu;
      u32 xprev = __shfl_up_sync(0xffffffffu, x, 1);
      // lane 0 reads its predecessor from the staged tile; every lane loads (slot 0 when it needs nothing:
      // a broadcast) so that no branch is needed
      const int q = (lane == 0 && p > 0) ? p - 1 : 0;
      const u32 xb = (u32)(staged_key<KeyT>(skey, q) >> a.group_shift);
      xprev = (lane == 0) ? (p > 0 ? xb : x) : xprev;
      if (valid) {
        if (xprev != x) { atomicAdd(&a.group_count[x], 0u - (u32)p); atomicAdd(&a.group_count[xprev], (u32)p); }
        if (p == tile_n - 1) atomicAdd(&a.group_count[x], (u32)tile_n);
      }
    }
    if (valid) {
      const u32 d = (u32)(k >> a.shift) & a.mask;
      const u32 dst = bin_dst[d] + (u32)p;
      if (a.keys_out) {
        if constexpr (sizeof(KeyT) == 8) {
          if (a.narrow) reinterpret_cast<u32*>(a.keys_out)[dst] = (u32)(k >> a.narrow);
          else a.keys_out[dst] = k;
        } else a.keys_out[dst] = k;
      }
      a.idx_out[dst] = rid;
    }
  }
}

template <typename KeyT, typename Src, int NBINS>
static int run_scatter(Src src, const PassIO& io, int64_t n, int shift, u32 mask, int64_t ntiles,
                       const u32* counts, const u32* base, const unsigned short* tile_counts,
                       u32* group_count, int group_shift, cudaStream_t s)
{
  constexpr int MINB = PassCfg<KeyT, NBINS>::MINB;
  PassArgs<KeyT, Src> a;
  a.src = src; a.idx_in = io.idx_in; a.keys_out = (KeyT*)io.keys_out; a.idx_out = io.idx_out;
  a.n = n; a.shift = shift; a.mask = mask; a.chunk_offs = counts; a.digit_base = base;
  a.tile_pre = tile_counts; a.group_count = group_count; a.group_shift = group_shift;
  a.narrow = io.narrow_out;
  constexpr size_t smem = PassCfg<KeyT, NBINS>::SMEM;
  // NB = ballots per row in the rank phase = digit width, rounded up to a built variant
  const int bits = __builtin_popcount(mask);
  void (*kern)(const PassArgs<KeyT, Src>) =
      bits <= 6 ? scatter_kernel<KeyT, Src, NBINS, MINB, 6>
    : bits == 7 ? scatter_kernel<KeyT, Src, NBINS, MINB, 7> : scatter_kernel<KeyT, Src, NBINS, MINB, 8>;
  DTB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  prof_begin("radix_scatter", s);
  kern<<<(unsigned)ntiles, PASS_THREADS, smem, s>>>(a);
  prof_end(s);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

template <typename KeyT, typename Src, int NBINS>
static int run_pass_nb(Src src, const PassIO& io, int64_t n, int shift, int bits, u32* work, u32* hmax,
                       cudaStream_t s, cudaEvent_t after_counts, u32* group_count, int group_shift)
{
  const int64_t nchunks = radix_num_chunks(n);
  const int64_t ntiles = (n + PASS_TILE - 1) / PASS_TILE;
  u32* counts = work;                                   // [nchunks][NBINS], becomes chunk_offs in place
  u32* total  = work + (size_t)nchunks * NBINS;         // [NBINS]
  u32* base   = total + NBINS;                          // [NBINS]
  unsigned short* tile_counts = reinterpret_cast<unsigned short*>(base + NBINS);   // [ntiles][NBINS]
  const u32 mask = (1u << bits) - 1;

  prof_begin("radix_count", s);
  if (io.raw_hist && (shift != 0 || io.keys_stage)) { set_error("internal: a folded histogram needs shift 0 and no key staging"); return DTB_EINVAL; }
  if (io.raw_hist) {
    static_assert(NBINS == 256, "the statistics kernel counts 256 bins per tile");
    const KeyNorm& k = src.key_norm();
    fold_counts_kernel<<<(unsigned)nchunks, 256, 0, s>>>(io.raw_hist, io.raw_na, ntiles, (u32)k.edge & 255u, (u32)k.inc & 255u,
                                                       k.desc, (u32)k.na_value & mask, mask, counts, tile_counts);
  } else {
    count_kernel<KeyT, Src, NBINS><<<(unsigned)nchunks, PASS_THREADS, 0, s>>>(src, n, shift, mask, counts, tile_counts,
                                                                               (KeyT*)io.keys_stage);
  }
  prof_end(s);
  chunk_scan_kernel<<<NBINS, 256, 0, s>>>(counts, nchunks, NBINS, total);
  digit_base_kernel<NBINS><<<1, 256, 0, s>>>(total, base, hmax);
  count_launch(3);
  if (after_counts) DTB_CUDA_CHECK(cudaEventRecord(after_counts, s));

  if (io.keys_stage) {
    // the count kernel materialised the normalised keys: scatter from them
    PassIO io2 = io; io2.src_kind = 0; io2.keys_in = io.keys_stage; io2.keys_stage = nullptr;
    PackedSrc<KeyT> psrc{(const KeyT*)io.keys_stage};
    return run_scatter<KeyT, PackedSrc<KeyT>, NBINS>(psrc, io2, n, shift, mask, ntiles, counts, base, tile_counts,
                                                     group_count, group_shift, s);
  }
  return run_scatter<KeyT, Src, NBINS>(src, io, n, shift, mask, ntiles, counts, base, tile_counts,
                                       group_count, group_shift, s);
}

template <typename KeyT, typename Src>
static int run_pass(Src src, const PassIO& io, int64_t n, int shift, int bits, u32* work, u32* hmax, cudaStream_t s,
                    cudaEvent_t after_counts, u32* group_count, int group_shift)
{
  if (n == 0) return DTB_OK;
  if (io.idx_in && (reinterpret_cast<uintptr_t>(io.idx_in) & 15)) {
    set_error("internal: row-id buffer must be 16-byte aligned"); return DTB_EINVAL;
  }
  return run_pass_nb<KeyT, Src, 256>(src, io, n, shift, bits, work, hmax, s, after_counts, group_count, group_shift);
}

template <typename KeyT>
static int run_pass_raw(const PassIO& io, const KeyPlan& kp, int64_t n, int shift, int bits,
                        u32* work, u32* hmax, cudaStream_t s, cudaEvent_t after_counts,
                        u32* group_count, int group_shift)
{
  const KeyNorm& k = kp.k[0];
#define DTB_CASE(T)                                                                          \
  { RawSrc<T, KeyT> src; src.init(k);                                                        \
    return run_pass<KeyT>(src, io, n, shift, bits, work, hmax, s, after_counts, group_count, group_shift); }
  switch (k.stype) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8:    DTB_CASE(int8_t)
    case DTB_STYPE_INT16:                        DTB_CASE(int16_t)
    case DTB_STYPE_INT32: case DTB_STYPE_DATE32: DTB_CASE(int32_t)
    case DTB_STYPE_INT64: case DTB_STYPE_TIME64: DTB_CASE(int64_t)
    case DTB_STYPE_FLOAT32:                      DTB_CASE(float)
    case DTB_STYPE_FLOAT64:                      DTB_CASE(double)
  }
#undef DTB_CASE
  set_error("internal: bad stype in radix pass"); return DTB_EINVAL;
}

size_t radix_pass_work_bytes(int64_t n) {
  const size_t ntiles = (size_t)((n + PASS_TILE - 1) / PASS_TILE);
  const size_t nbins = 256;
  return sizeof(u32) * ((size_t)radix_num_chunks(n) * nbins + 2 * nbins)
       + sizeof(unsigned short) * (ntiles + CHUNK_TILES) * nbins;
}

int launch_radix_pass(const PassIO& io, const KeyPlan& kp, int key_bytes, int64_t n,
                      int shift, int bits, uint32_t* work, uint32_t* hmax, cudaStream_t s,
                      cudaEvent_t after_counts, uint32_t* group_count, int group_shift)
{
  if (bits < 1 || bits > 8) { set_error("internal: digit width must be 1..8 bits"); return DTB_EINVAL; }
  if (io.src_kind == 0) {
    if (key_bytes == 4) { PackedSrc<u32> src{(const u32*)io.keys_in};
      return run_pass<u32>(src, io, n, shift, bits, work, hmax, s, after_counts, group_count, group_shift); }
    else { PackedSrc<u64> src{(const u64*)io.keys_in};
      return run_pass<u64>(src, io, n, shift, bits, work, hmax, s, after_counts, group_count, group_shift); }
  }
  return key_bytes == 4 ? run_pass_raw<u32>(io, kp, n, shift, bits, work, hmax, s, after_counts, group_count, group_shift)
                        : run_pass_raw<u64>(io, kp, n, shift, bits, work, hmax, s, after_counts, group_count, group_shift);
}

__global__ void widen_u32_kernel(const u32* __restrict__ in, int64_t n, int64_t* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (int64_t)in[i];
}

int launch_widen_u32(const uint32_t* in, int64_t n, int64_t* out, cudaStream_t s) {
  if (n == 0) return DTB_OK;
  int64_t want = (n + 255) / 256;
  int grid = (int)(want > NUM_SMS * 16 ? NUM_SMS * 16 : want);
  widen_u32_kernel<<<grid, 256, 0, s>>>(in, n, out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

__global__ void iota32_kernel(int32_t* out, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (int32_t)i;
}

int launch_iota32(int32_t* out, int64_t n, cudaStream_t s) {
  if (n == 0) return DTB_OK;
  int64_t want = (n + 255) / 256;
  int grid = (int)(want > NUM_SMS * 16 ? NUM_SMS * 16 : want);
  iota32_kernel<<<grid, 256, 0, s>>>(out, n);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

}  // namespace dtb
