// dtb_reduce.cu -- per-group reducers and the RowIndex gather.
//
// Replaces the reference's reducer columns, which are evaluated one group per
// virtual get_element() call with two more virtual calls per row
// (column/sumprod.h:34-59, mean.h:33-51, minmax.h:33-60, count.h:35-89, driven
// by column/column_impl.cc:78-103), and ArrayView_ColumnImpl's gather
// (column/view.cc:138-155).
//
// Design: rows, not groups, are the unit of parallelism, so skewed group
// sizes cannot unbalance the grid (the reference partitions groups statically,
// column_impl.h:106).  A tile of consecutive sorted positions finds the groups
// it intersects from `offsets`, every thread folds its 8 consecutive rows
// (gathered through the RowIndex), partials of the same group are combined
// across the warp with a segmented shuffle scan, and one atomic per
// (warp, group) lands in an L2-resident accumulator table.  A finalize kernel
// turns accumulators into the reference's output stype and NA sentinels.
//
// Bound: HBM (random 8-byte gathers: one 32-byte sector per row).
// Algorithmic bytes per row: sizeof(order elem) + sizeof(value elem).
#include <type_traits>
#include "dtb_common.cuh"

namespace dtb {

enum { CAT_SUMI = 0, CAT_SUMF = 1, CAT_MEAN = 2, CAT_MINMAX = 3, CAT_COUNT = 4, CAT_PRODI = 5, CAT_PRODF = 6 };

constexpr int RT = 256;          // threads per tile
constexpr int RIPT = 8;          // consecutive rows per thread
constexpr int RTILE = RT * RIPT;

template <int CAT> struct Partial;
template <> struct Partial<CAT_SUMI> { u64 s; };
template <> struct Partial<CAT_SUMF> { double s; };
template <> struct Partial<CAT_MEAN> { double s; u32 c; };
template <> struct Partial<CAT_MINMAX> { u64 key; };
template <> struct Partial<CAT_COUNT> { u32 c; };
template <> struct Partial<CAT_PRODI> { u64 p; };                    // wraps modulo 2^64
// A float product kept as |prod| = m * 2^e, m in [1, 2): no intermediate product overflows or underflows.  f: bit 0
// a zero was seen, bit 1 an infinity was seen, bit 2 the sign parity.
template <> struct Partial<CAT_PRODF> { double m; int64_t e; u32 f; };

// In the accumulators a float product is two words: acc0 = f << 52 | the 52 fraction bits of m, acc1 = e.
constexpr u64 PRODF_FRAC = (1ull << 52) - 1;
__device__ __forceinline__ double prodf_sig(u64 w) {
  return __longlong_as_double((long long)((w & PRODF_FRAC) | 0x3FF0000000000000ull));
}
__device__ __forceinline__ void prodf_mul(Partial<CAT_PRODF>& a, double m, int64_t e, u32 f) {
  const double r = a.m * m;                                       // [1, 4): one rounding
  const bool carry = r >= 2.0;
  a.m = carry ? r * 0.5 : r;                                      // exact
  a.e += e + (carry ? 1 : 0);
  a.f = ((a.f | f) & 3u) | ((a.f ^ f) & 4u);
}

// The value of a float product: zero and infinity together give NA (0 * inf, valid = false), otherwise a zero or an
// infinity with the sign parity, otherwise m * 2^e rounded once to float64.
__device__ __forceinline__ double prodf_value(const Partial<CAT_PRODF>& p, bool& valid) {
  const bool neg = (p.f & 4u) != 0;
  double r;
  if (p.f & 1u) r = neg ? -0.0 : 0.0;
  else if (p.f & 2u) r = neg ? -INFINITY : INFINITY;
  else r = ldexp(neg ? -p.m : p.m, (int)(p.e < -4000 ? -4000 : (p.e > 4000 ? 4000 : p.e)));
  valid = (p.f & 3u) != 3u;
  return r;
}

template <int CAT>
__device__ __forceinline__ void p_init(Partial<CAT>& p, int flag) {
  if constexpr (CAT == CAT_SUMI) p.s = 0;
  else if constexpr (CAT == CAT_SUMF) p.s = 0.0;
  else if constexpr (CAT == CAT_MEAN) { p.s = 0.0; p.c = 0; }
  else if constexpr (CAT == CAT_MINMAX) p.key = flag ? ~0ull : 0ull;   // flag: 1 = MIN
  else if constexpr (CAT == CAT_PRODI) p.p = 1;
  else if constexpr (CAT == CAT_PRODF) { p.m = 1.0; p.e = 0; p.f = 0; }
  else p.c = 0;
}

template <int CAT>
__device__ __forceinline__ void p_merge(Partial<CAT>& a, const Partial<CAT>& b, int flag) {
  if constexpr (CAT == CAT_SUMI) a.s += b.s;
  else if constexpr (CAT == CAT_SUMF) a.s += b.s;
  else if constexpr (CAT == CAT_MEAN) { a.s += b.s; a.c += b.c; }
  else if constexpr (CAT == CAT_MINMAX) a.key = flag ? (b.key < a.key ? b.key : a.key) : (b.key > a.key ? b.key : a.key);
  else if constexpr (CAT == CAT_PRODI) a.p *= b.p;
  else if constexpr (CAT == CAT_PRODF) prodf_mul(a, b.m, b.e, b.f);
  else a.c += b.c;
}

template <int CAT>
__device__ __forceinline__ Partial<CAT> p_shfl_up(const Partial<CAT>& a, int d) {
  Partial<CAT> r;
  if constexpr (CAT == CAT_SUMI) r.s = __shfl_up_sync(0xffffffffu, a.s, d);
  else if constexpr (CAT == CAT_SUMF) r.s = __shfl_up_sync(0xffffffffu, a.s, d);
  else if constexpr (CAT == CAT_MEAN) { r.s = __shfl_up_sync(0xffffffffu, a.s, d); r.c = __shfl_up_sync(0xffffffffu, a.c, d); }
  else if constexpr (CAT == CAT_MINMAX) r.key = __shfl_up_sync(0xffffffffu, a.key, d);
  else if constexpr (CAT == CAT_PRODI) r.p = __shfl_up_sync(0xffffffffu, a.p, d);
  else if constexpr (CAT == CAT_PRODF) {
    r.m = __shfl_up_sync(0xffffffffu, a.m, d); r.e = __shfl_up_sync(0xffffffffu, a.e, d); r.f = __shfl_up_sync(0xffffffffu, a.f, d);
  }
  else r.c = __shfl_up_sync(0xffffffffu, a.c, d);
  return r;
}

template <int CAT>
__device__ __forceinline__ void p_flush(const Partial<CAT>& p, int64_t g, u64* acc0, u64* acc1, int flag) {
  if constexpr (CAT == CAT_SUMI) { if (p.s) atomicAdd(&acc0[g], p.s); }
  else if constexpr (CAT == CAT_SUMF) { if (p.s != 0.0) atomicAdd(reinterpret_cast<double*>(acc0) + g, p.s); }
  else if constexpr (CAT == CAT_MEAN) {
    if (p.c) { atomicAdd(reinterpret_cast<double*>(acc0) + g, p.s); atomicAdd(&acc1[g], (u64)p.c); }
  }
  else if constexpr (CAT == CAT_MINMAX) {
    if (flag) { if (p.key != ~0ull) atomicMin(&acc0[g], p.key); }
    else      { if (p.key != 0ull)  atomicMax(&acc0[g], p.key); }
  }
  else if constexpr (CAT == CAT_PRODI) {                         // no atomic multiply: a CAS loop
    if (p.p != 1) { u64 old = acc0[g], seen; do { seen = old; old = atomicCAS(&acc0[g], seen, seen * p.p); } while (old != seen); }
  }
  else if constexpr (CAT == CAT_PRODF) {
    if (p.m == 1.0 && p.e == 0 && p.f == 0) return;
    // the significand and the flags by CAS; the exponent, with the significand's carry, by one atomicAdd
    Partial<CAT_PRODF> q;
    u64 old = acc0[g], seen;
    do {
      seen = old;
      q.m = prodf_sig(seen); q.e = 0; q.f = (u32)(seen >> 52);
      prodf_mul(q, p.m, 0, p.f);
      old = atomicCAS(&acc0[g], seen, ((u64)q.f << 52) | ((u64)__double_as_longlong(q.m) & PRODF_FRAC));
    } while (old != seen);
    if (p.e + q.e) atomicAdd(&acc1[g], (u64)(p.e + q.e));
  }
  else { if (p.c) atomicAdd(&acc0[g], (u64)p.c); }
}

// PROD: a tile's first and last groups may go on in other tiles, and a group of 1e9 rows would have every warp of
// the grid retry its CAS on one word.  So the runs of those two groups fold into two slots in shared memory, each
// tile writes its slots out, and prod_finalize_kernel multiplies them into the group's result.  Only the groups
// strictly inside a tile are flushed to the accumulators directly.  slot: u64[4] = word 0 of slots 0 / 1, then
// word 1 of slots 0 / 1.
template <int CAT>
__device__ __forceinline__ void flush_run(const Partial<CAT>& p, int64_t g, int64_t g_lo, int64_t g_hi, u64* slot,
                                          u64* acc0, u64* acc1, int flag) {
  if constexpr (CAT == CAT_PRODI || CAT == CAT_PRODF) {
    if (g == g_lo || g == g_hi) { p_flush(p, (int64_t)(g == g_lo ? 0 : 1), slot, slot + 2, flag); return; }
  }
  p_flush(p, g, acc0, acc1, flag);
}

// fold one (possibly NA) raw element into a partial
template <typename T, int CAT>
__device__ __forceinline__ void p_add(Partial<CAT>& p, typename RawKey<T>::load_t raw, bool row_valid, int flag) {
  constexpr bool ISF = std::is_floating_point<T>::value;
  u64 u; bool valid = RawKey<T>::get(raw, u) && row_valid;   // u: sign-extended int or float image
  if constexpr (CAT == CAT_COUNT) { p.c += (flag ? !valid : valid); return; }
  if (!valid) return;
  if constexpr (CAT == CAT_SUMI) p.s += u;
  else if constexpr (CAT == CAT_SUMF || CAT == CAT_MEAN) {
    double x;
    if constexpr (std::is_same<T, float>::value) x = (double)__uint_as_float((u32)raw);
    else if constexpr (std::is_same<T, double>::value) x = __longlong_as_double((long long)raw);
    else x = (double)(int64_t)u;
    p.s += x;
    if constexpr (CAT == CAT_MEAN) p.c += 1;
  }
  else if constexpr (CAT == CAT_PRODI) p.p *= u;
  else if constexpr (CAT == CAT_PRODF) {
    // |x| = m * 2^e exactly, from the bits (a float32 is widened first; a float64 subnormal is scaled up by 2^64)
    u64 b = std::is_same<T, float>::value ? (u64)__double_as_longlong((double)__uint_as_float((u32)raw)) : (u64)raw;
    const u32 sign = (u32)(b >> 63) << 2;
    b &= ~0x8000000000000000ull;
    if (b == 0) { p.f = (p.f | 1u) ^ sign; return; }
    if (b == 0x7FF0000000000000ull) { p.f = (p.f | 2u) ^ sign; return; }
    int64_t ex = (int64_t)(b >> 52);
    if (ex == 0) { b = (u64)__double_as_longlong(__longlong_as_double((long long)b) * 0x1p64); ex = (int64_t)(b >> 52) - 64; }
    prodf_mul(p, __longlong_as_double((long long)((b & PRODF_FRAC) | 0x3FF0000000000000ull)), ex - 1023, sign);
  }
  else if constexpr (CAT == CAT_MINMAX) {
    u64 key = ISF ? u : (u ^ 0x8000000000000000ull);      // order-preserving unsigned key, never 0 for ints
    if (flag) { if (!ISF) key -= 1; p.key = key < p.key ? key : p.key; }
    else p.key = key > p.key ? key : p.key;
  }
}

// The head bitmap of the tile of positions [t0, t1): bit p of s_bits is set where a group starts at t0 + p, p >= 1
// (s_bits zeroed by the caller).  g_lo / g_hi: the groups of the tile's first and last positions.  REV: positions
// are mirrored (p -> n - 1 - p), so group g starts at n - offsets[ng - g].
template <bool REV>
__device__ __forceinline__ int64_t head_offset(const int32_t* __restrict__ offsets, int64_t ng, int64_t n, int64_t g) {
  return REV ? n - (int64_t)offsets[ng - g] : (int64_t)offsets[g];
}

template <bool REV>
__device__ __forceinline__ void tile_heads(const int32_t* __restrict__ offsets, int64_t ng, int64_t n, int64_t t0,
                                           int64_t t1, int tid, int64_t* s_g, u32* s_bits, int64_t& g_lo, int64_t& g_hi) {
  if (tid == 0 || tid == 32) {
    // largest g with offsets[g] <= pos
    const int64_t pos = (tid == 0) ? t0 : (t1 - 1);
    int64_t lo = 0, hi = ng;             // offsets[0] = 0 <= pos < offsets[ng] = n
    while (hi - lo > 1) {
      int64_t mid = (lo + hi) >> 1;
      if (head_offset<REV>(offsets, ng, n, mid) <= pos) lo = mid; else hi = mid;
    }
    s_g[tid ? 1 : 0] = lo;
  }
  __syncthreads();
  g_lo = s_g[0]; g_hi = s_g[1];
  for (int64_t g = g_lo + 1 + tid; g <= g_hi; g += RT) {
    const int p = (int)(head_offset<REV>(offsets, ng, n, g) - t0);    // 1 .. RTILE-1
    atomicOr(&s_bits[p >> 5], 1u << (p & 31));
  }
  __syncthreads();
}

template <typename T, int CAT, typename OrdT>
__global__ void __launch_bounds__(RT)
reduce_kernel(const typename RawKey<T>::load_t* __restrict__ v, int64_t nv,
              const OrdT* __restrict__ order, const int32_t* __restrict__ offsets,
              int64_t ng, int64_t n, u64* acc0, u64* acc1, int flag)
{
  typedef typename RawKey<T>::load_t L;
  __shared__ int64_t s_g[2];
  __shared__ u32 s_bits[RTILE / 32];
  __shared__ u32 s_wpre[RTILE / 32];

  const int tid = threadIdx.x, lane = tid & 31;
  const int64_t t0 = (int64_t)blockIdx.x * RTILE;
  const int64_t t1 = (t0 + RTILE < n) ? t0 + RTILE : n;

  if (tid < RTILE / 32) s_bits[tid] = 0;
  u64* s_slot = nullptr;                                       // PROD: the tile's two slots (flush_run)
  if constexpr (CAT == CAT_PRODI || CAT == CAT_PRODF) {
    __shared__ u64 s_prod[4];
    s_slot = s_prod;
    if (tid < 4) s_prod[tid] = (CAT == CAT_PRODI && tid < 2) ? 1ull : 0ull;
  }
  int64_t g_lo, g_hi;
  tile_heads<false>(offsets, ng, n, t0, t1, tid, s_g, s_bits, g_lo, g_hi);
  if (tid < 32) {
    // exclusive prefix of popcounts over the RTILE/32 = 64 bitmap words (2 per lane)
    u32 a = __popc(s_bits[2 * lane]), b = __popc(s_bits[2 * lane + 1]);
    u32 incl = a + b;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      u32 o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += o;
    }
    s_wpre[2 * lane] = incl - a - b;
    s_wpre[2 * lane + 1] = incl - b;
  }
  __syncthreads();

  const int c0 = tid * RIPT;                                   // RIPT = 8 rows: one byte of the bitmap
  const u32 word = s_bits[c0 >> 5];
  const u32 mybits = (word >> (c0 & 31)) & 0xffu;
  int64_t g_cur = g_lo + s_wpre[c0 >> 5] + __popc(word & ((1u << (c0 & 31)) - 1u));

  // gather: all index loads first, then all value loads
  const int64_t p0 = t0 + c0;
  int64_t row[RIPT];
#pragma unroll
  for (int i = 0; i < RIPT; i++) {
    const int64_t p = p0 + i;
    row[i] = (p < n) ? (order ? (int64_t)order[p] : p) : -2;
  }
  L val[RIPT];
#pragma unroll
  for (int i = 0; i < RIPT; i++) val[i] = (row[i] >= 0 && row[i] < nv) ? v[row[i]] : (L)0;

  Partial<CAT> part; p_init(part, flag);
#pragma unroll
  for (int i = 0; i < RIPT; i++) {
    if (mybits & (1u << i)) {                 // a new group starts at this row: close the previous run
      flush_run(part, g_cur, g_lo, g_hi, s_slot, acc0, acc1, flag);
      p_init(part, flag);
      g_cur++;
    }
    if (p0 + i < n) p_add<T, CAT>(part, val[i], row[i] >= 0 && row[i] < nv, flag);
  }

  // segmented combine of the open partials across the warp (keys ascend with the lane)
  const int64_t key = (p0 < n) ? g_cur : (int64_t)-1 - lane;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    Partial<CAT> o = p_shfl_up(part, d);
    int64_t ok = __shfl_up_sync(0xffffffffu, key, d);
    if (lane >= d && ok == key) p_merge(part, o, flag);
  }
  const int64_t nkey = __shfl_down_sync(0xffffffffu, key, 1);
  if (key >= 0 && (lane == 31 || nkey != key)) flush_run(part, key, g_lo, g_hi, s_slot, acc0, acc1, flag);
  if constexpr (CAT == CAT_PRODI || CAT == CAT_PRODF) {
    // tile t's slots go to acc1[ng + 2t + slot] (word 0) and acc1[ng + 2 * ntiles + 2t + slot] (word 1)
    __syncthreads();
    u64* c = acc1 + ng + (tid >> 1) * 2 * (int64_t)gridDim.x;
    if (tid < 4) c[2 * (int64_t)blockIdx.x + (tid & 1)] = s_slot[tid];
  }
}

// ---- accumulator init / finalize ------------------------------------------------
__global__ void fill_u64_kernel(u64* p, int64_t n, u64 v) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}

void fill_u64(unsigned long long* p, int64_t n, unsigned long long v, cudaStream_t s) {
  if (n <= 0) return;
  fill_u64_kernel<<<grid_for((n + 255) / 256, 8), 256, 0, s>>>(p, n, v);
  count_launch();
}

__global__ void nrows_kernel(const int32_t* __restrict__ offsets, int64_t ng, int64_t* out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride)
    out[g] = (int64_t)offsets[g + 1] - (int64_t)offsets[g];
}

__device__ __forceinline__ bool is_float_zero(int stype, u64 bits) {
  return ((stype == DTB_STYPE_FLOAT32) ? (bits << 33) : (bits << 1)) == 0;     // float32 bits sit in the low word
}

// bits: a float min / max result of group g that is a zero.  Its sign is that of the group's first valid zero in
// RowIndex order: reducers fed piecewise have recorded it (first_zero); otherwise the group is marked for the
// row-parallel lookup that follows the finalize (launch_zero_minmax_fix), and the word after the marks says so.
__device__ __forceinline__ u64 zero_minmax_bits(const GroupRows& gr, int stype, int64_t g, int64_t ng, u64 bits) {
  if (gr.first_zero) {
    const u64 sign = (stype == DTB_STYPE_FLOAT32) ? 0x80000000ull : 0x8000000000000000ull;
    const u64 f = gr.first_zero[g];
    return f == ~0ull ? bits : ((f & 1) ? sign : 0ull);
  }
  if (gr.zpos) { gr.zpos[g] = ~0ull; *reinterpret_cast<volatile u64*>(gr.zpos + ng) = 1ull; }
  return bits;
}

// out[g] = the group's first valid zero, for the groups marked by the finalize (zpos[g]: its RowIndex position,
// found by launch_first_zero_pos).  Returns at once when the finalize marked no group.
__global__ void zero_fix_kernel(int stype, const GroupRows gr, int64_t ng, void* out) {
  if (gr.zpos[ng] == 0) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const u64 bits = (stype == DTB_STYPE_FLOAT32) ? (u64)((const u32*)out)[g] : ((const u64*)out)[g];
    const u64 p = gr.zpos[g];
    if (!is_float_zero(stype, bits) || p == ~0ull) continue;     // not marked (its word is not a position then)
    const int64_t j = gr.order ? (gr.order_is64 ? ((const int64_t*)gr.order)[p] : (int64_t)((const int32_t*)gr.order)[p])
                               : (int64_t)p;
    if (stype == DTB_STYPE_FLOAT32) ((u32*)out)[g] = ((const u32*)gr.v)[j];
    else                            ((u64*)out)[g] = ((const u64*)gr.v)[j];
  }
}

size_t zero_fix_bytes(int64_t ng) { return sizeof(u64) * (size_t)((ng > 0 ? ng : 0) + 1); }

bool minmax_zero_sign(int op, int stype) {
  return (op == DTB_OP_MIN || op == DTB_OP_MAX) && (stype == DTB_STYPE_FLOAT32 || stype == DTB_STYPE_FLOAT64);
}

static bool wants_zero_fix(int op, int stype, const GroupRows& gr) { return gr.zpos && minmax_zero_sign(op, stype); }

// before the finalize: no group marked yet
static int zero_fix_begin(int op, int stype, const GroupRows& gr, int64_t ng, cudaStream_t s) {
  if (wants_zero_fix(op, stype, gr)) DTB_CUDA_CHECK(cudaMemsetAsync(gr.zpos + ng, 0, sizeof(u64), s));
  return DTB_OK;
}

// after the finalize: one pass over the rows (it returns at once when no group was marked) finds the first valid
// zero of every group, and the marked groups take its bits
static int zero_fix_end(int op, int stype, const GroupRows& gr, int64_t ng, void* out, cudaStream_t s) {
  if (!wants_zero_fix(op, stype, gr) || ng == 0) return DTB_OK;
  DTB_TRY(launch_first_zero_pos(gr.v, stype, gr.nv, gr.order, gr.order_is64, gr.offsets, ng, gr.n, gr.zpos + ng,
                                gr.zpos, s));
  zero_fix_kernel<<<grid_for((ng + 255) / 256, 8), 256, 0, s>>>(stype, gr, ng, out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// out[g] = the result of the accumulators of group key gkeys[g] (direct-address reducers), or of group g (gkeys NULL)
__global__ void finalize_kernel(int op, int in_stype, int out_stype, const u64* __restrict__ acc0,
                                const u64* __restrict__ acc1, const u32* __restrict__ gkeys,
                                int64_t ng, void* out, const GroupRows gr)
{
  const bool in_float = (in_stype == DTB_STYPE_FLOAT32 || in_stype == DTB_STYPE_FLOAT64);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const u32 x = gkeys ? gkeys[g] : (u32)g;
    const u64 a = acc0[x];
    bool valid = true; u64 bits = a;
    switch (op) {
      case DTB_OP_SUM:
        if (out_stype == DTB_STYPE_FLOAT32) bits = __float_as_uint((float)__longlong_as_double((long long)a));
        break;                                            // int64 / float64: accumulator bits are the result
      case DTB_OP_MEAN: {
        const u64 c = acc1[x];
        valid = c != 0;
        const double m = __longlong_as_double((long long)a) / (double)c;
        bits = (out_stype == DTB_STYPE_FLOAT32) ? (u64)__float_as_uint((float)m) : (u64)__double_as_longlong(m);
        break; }
      case DTB_OP_MIN: case DTB_OP_MAX: {
        const bool is_min = (op == DTB_OP_MIN);
        valid = is_min ? (a != ~0ull) : (a != 0ull);
        if (in_float) bits = (in_stype == DTB_STYPE_FLOAT32) ? (u64)f32_unimage((u32)a) : f64_unimage(a);
        else bits = (is_min ? a + 1 : a) ^ 0x8000000000000000ull;
        if (in_float && valid && is_float_zero(in_stype, bits)) bits = zero_minmax_bits(gr, in_stype, g, ng, bits);
        break; }
      default: break;                                     // COUNT / COUNTNA: as is
    }
    store_result(out, out_stype, g, valid, bits);
  }
}

static int reduce_out_stype(int op, int st) {
  const bool isint = (st == DTB_STYPE_BOOL || st == DTB_STYPE_INT8 || st == DTB_STYPE_INT16 ||
                      st == DTB_STYPE_INT32 || st == DTB_STYPE_INT64);
  const bool isflt = (st == DTB_STYPE_FLOAT32 || st == DTB_STYPE_FLOAT64);
  switch (op) {
    case DTB_OP_NROWS: return DTB_STYPE_INT64;
    case DTB_OP_COUNT: case DTB_OP_COUNTNA: return (isint || isflt) ? DTB_STYPE_INT64 : 0;
    case DTB_OP_SUM:  return isint ? DTB_STYPE_INT64 : (isflt ? st : 0);           // fexpr_sumprod.cc:50-66
    case DTB_OP_MEAN: return isint ? DTB_STYPE_FLOAT64 : (isflt ? st : 0);         // fexpr_mean.cc:49-78
    case DTB_OP_MIN: case DTB_OP_MAX:
      return (isint || isflt) ? st : 0;      // fexpr_minmax.cc:50-72: the column's own stype (bool8 stays bool8)
    case DTB_OP_FIRST: case DTB_OP_LAST: return stype_bytes(st) ? st : 0;          // head_reduce_unary.cc:126-128
    case DTB_OP_SD: case DTB_OP_MEDIAN:                                           // head_reduce_unary.cc:224-245, 480-506
      return isint ? DTB_STYPE_FLOAT64 : (isflt ? st : 0);
    case DTB_OP_NUNIQUE: return stype_bytes(st) ? DTB_STYPE_INT64 : 0;            // head_reduce_unary.cc:398-415
    case DTB_OP_PROD: return isint ? DTB_STYPE_INT64 : (isflt ? st : 0);          // fexpr_sumprod.cc:47-67
  }
  return 0;
}

// out[g] = finalize_kernel's result for every group, with the sign lookup of a zero float min / max (gr.zpos)
static int finalize(int op, int stype, const u64* acc0, const u64* acc1, const u32* gkeys, int64_t ng, void* out,
                    const GroupRows& gr, cudaStream_t s)
{
  const int out_st = reduce_out_stype(op, stype);
  if (!out_st) { set_error("Invalid column type in reducer"); return DTB_EINVAL; }
  if (ng == 0) return DTB_OK;
  DTB_TRY(zero_fix_begin(op, stype, gr, ng, s));
  finalize_kernel<<<grid_for((ng + 255) / 256, 8), 256, 0, s>>>(op, stype, out_st, acc0, acc1, gkeys, ng, out, gr);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return zero_fix_end(op, stype, gr, ng, out, s);
}

size_t reduce_extra_bytes(int op, int stype, int64_t ng, int64_t n) {
  if (op == DTB_OP_SD) return 2 * sizeof(double) * (size_t)(ng > 0 ? ng : 1);      // sq, pivot (MomentWords)
  if (op == DTB_OP_PROD)                                                          // acc1, then the tiles' slots
    return sizeof(u64) * (size_t)((ng > 0 ? ng : 1) + 4 * ((n + RTILE - 1) / RTILE));
  if (minmax_zero_sign(op, stype)) return zero_fix_bytes(ng);
  if (op == DTB_OP_NUNIQUE) return (size_t)n + 16;
  return 0;
}

template <typename T, int CAT>
static int run_reduce(const void* v, int64_t nv, const void* order, int order_is64,
                      const int32_t* offsets, int64_t ng, int64_t n, u64* acc0, u64* acc1,
                      int flag, cudaStream_t s)
{
  typedef typename RawKey<T>::load_t L;
  const unsigned grid = (unsigned)((n + RTILE - 1) / RTILE);
  with_order(order, order_is64, [&](auto o) {
    reduce_kernel<T, CAT><<<grid, RT, 0, s>>>((const L*)v, nv, o, offsets, ng, n, acc0, acc1, flag);
  });
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

template <int CAT>
__device__ __forceinline__ Partial<CAT> prod_word(const u64* w0, const u64* w1, int64_t i) {
  Partial<CAT> p;
  if constexpr (CAT == CAT_PRODI) p.p = w0[i];
  else { const u64 w = w0[i]; p.m = prodf_sig(w); p.e = (int64_t)w1[i]; p.f = (u32)(w >> 52); }
  return p;
}

template <int CAT>
__device__ __forceinline__ Partial<CAT> p_shfl_xor(const Partial<CAT>& a, int d) {
  Partial<CAT> r;
  if constexpr (CAT == CAT_PRODI) r.p = __shfl_xor_sync(0xffffffffu, a.p, d);
  else {
    r.m = __shfl_xor_sync(0xffffffffu, a.m, d); r.e = __shfl_xor_sync(0xffffffffu, a.e, d); r.f = __shfl_xor_sync(0xffffffffu, a.f, d);
  }
  return r;
}

// out[g] = the product of group g: its accumulators (the runs strictly inside a tile) times the slots of the tiles it
// reaches into.  Group g covers positions [a, b), tiles ta .. tb: in tile ta it is slot 0 (it starts the tile) or
// slot 1 (it ends the tile) or neither; in every later tile it is slot 0.  A group that reaches into more than 32
// tiles is folded by its whole warp, 32 tiles at a time.  The slots are assigned from the offsets alone, which relies on
// the Groupby invariant that no group is empty (an empty group at a tile start would take the next group's slot 0):
// group() never makes one, and caller-supplied offsets are checked first (offsets_check_kernel).  Float results: zero and infinity together give NA
// (0 * inf), otherwise a zero or an infinity with the sign parity, otherwise m * 2^e rounded once.
template <int CAT>
__global__ void prod_finalize_kernel(const int32_t* __restrict__ offsets, int64_t ng, int64_t n, const u64* __restrict__ acc0,
                                     const u64* __restrict__ acc1, int64_t ntiles, int out_stype, void* out)
{
  const u64* c0 = acc1 + ng;
  const u64* c1 = c0 + 2 * ntiles;
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t gend = (ng + 31) & ~(int64_t)31;             // whole warps stay in the loop
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < gend; g += stride) {
    Partial<CAT> p; p_init(p, 0);
    int64_t t1 = 0, t2 = -1;                                   // the later tiles: slot 0 of t1 .. t2
    if (g < ng) {
      p = prod_word<CAT>(acc0, acc1, g);
      const int64_t a = offsets[g], b = offsets[g + 1];
      if (a < b) {                                             // the empty group of zero rows has no tile
        const int64_t ta = a / RTILE, tend = (ta + 1) * RTILE < n ? (ta + 1) * RTILE : n;
        if (a == ta * RTILE) p_merge(p, prod_word<CAT>(c0, c1, 2 * ta), 0);
        else if (b >= tend)  p_merge(p, prod_word<CAT>(c0, c1, 2 * ta + 1), 0);
        t1 = ta + 1; t2 = (b - 1) / RTILE;
      }
    }
    const bool wide = t2 - t1 >= 32;
    if (!wide) for (int64_t t = t1; t <= t2; t++) p_merge(p, prod_word<CAT>(c0, c1, 2 * t), 0);
    for (unsigned todo = __ballot_sync(0xffffffffu, wide); todo; todo &= todo - 1) {
      const int src = __ffs(todo) - 1;
      const int64_t s1 = __shfl_sync(0xffffffffu, t1, src), s2 = __shfl_sync(0xffffffffu, t2, src);
      Partial<CAT> q; p_init(q, 0);
      for (int64_t t = s1 + lane; t <= s2; t += 32) p_merge(q, prod_word<CAT>(c0, c1, 2 * t), 0);
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) p_merge(q, p_shfl_xor(q, d), 0);
      if (lane == src) p_merge(p, q, 0);
    }
    if (g >= ng) continue;
    if constexpr (CAT == CAT_PRODI) {
      ((int64_t*)out)[g] = (int64_t)p.p;
    } else {
      bool valid;
      const double r = prodf_value(p, valid);
      // float32: the float64 r is exact wherever a float32 result is not 0, so this rounds once
      store_float(out, out_stype, g, valid, r);
    }
  }
}

// PROD (column/sumprod.h:34-59): integers wrap modulo 2^64, bit-exact in any order; floats are exponent-tracked (see
// Partial<CAT_PRODF>) and rounded once.  acc1 = extra (reduce_extra_bytes): the exponents, then the tiles' slots.
static int launch_prod(const void* value, int stype, int64_t nv, const void* order, int order_is64,
                       const int32_t* offsets, int64_t ng, int64_t n, u64* acc0, u64* acc1, int out_st, void* out,
                       cudaStream_t s)
{
  return with_stype(stype, "internal: product of stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    constexpr bool ISF = std::is_floating_point<T>::value;
    constexpr int CAT = ISF ? CAT_PRODF : CAT_PRODI;
    const int64_t ntiles = (n + RTILE - 1) / RTILE;          // every tile writes both its slots
    fill_u64(acc0, ng, ISF ? 0ull : 1ull, s);
    fill_u64(acc1, ng, 0ull, s);
    DTB_CUDA_CHECK(cudaGetLastError());
    if (n > 0) DTB_TRY((run_reduce<T, CAT>(value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 0, s)));
    prod_finalize_kernel<CAT><<<grid_for((ng + 255) / 256, 8), 256, 0, s>>>(offsets, ng, n, acc0, acc1, ntiles, out_st, out);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  });
}

// acc0/acc1: device scratch of ng u64 each (allocated by the caller in dtb_api.cu)
int launch_reduce_impl(int op, const void* value, int stype, int64_t nv, const void* order, int order_is64,
                       const int32_t* offsets, int64_t ng, int64_t n, u64* acc0, u64* acc1,
                       void* out, cudaStream_t s, void* extra)
{
  const int out_st = reduce_out_stype(op, stype);
  if (!out_st) { set_error("Invalid column type in reducer"); return DTB_EINVAL; }
  if (ng == 0) return DTB_OK;
  const int fgrid = grid_for((ng + 255) / 256, 8);
  if (op >= DTB_OP_FIRST && op <= DTB_OP_NUNIQUE) {
    // within-group ordered reducers (dtb_next.cu): they walk the ARR32 RowIndex
    if (order_is64) { set_error("first/last/sd/median/nunique take an int32 RowIndex"); return DTB_ENOTIMPL; }
    const int32_t* o32 = (const int32_t*)order;
    if (op == DTB_OP_FIRST || op == DTB_OP_LAST) return launch_firstlast(value, stype, nv, o32, offsets, ng, op == DTB_OP_LAST, out, s);
    if (op == DTB_OP_MEDIAN) return launch_median(value, stype, nv, o32, offsets, ng, out, s);
    if (!extra) { set_error("internal: reducer scratch missing"); return DTB_EINVAL; }
    if (op == DTB_OP_SD) {                         // sum, cnt: acc0, acc1; sq, pivot: extra
      double* sq = (double*)extra;
      const MomentWords w = {{(double*)acc0}, acc1, {sq}, nullptr, {sq + ng}};
      return launch_moments(op, value, stype, nullptr, 0, nv, o32, 0, offsets, ng, n, w, out_st, out, s);
    }
    // NUNIQUE: flag the rows that start a new distinct value, then count the flags per group
    int8_t* flag = (int8_t*)extra;
    DTB_TRY(launch_distinct_flags(value, stype, nv, o32, offsets, ng, n, flag, s));
    fill_u64_kernel<<<fgrid, 256, 0, s>>>(acc0, ng, 0ull);
    count_launch();
    if (n > 0) DTB_TRY((run_reduce<int8_t, CAT_COUNT>(flag, n, nullptr, 0, offsets, ng, n, acc0, acc1, 0, s)));
    return finalize(DTB_OP_COUNT, DTB_STYPE_INT8, acc0, acc1, nullptr, ng, out, GroupRows(), s);
  }
  if (op == DTB_OP_NROWS) return launch_nrows(offsets, ng, out, s);
  if (op == DTB_OP_PROD) {
    if (!extra) { set_error("internal: reducer scratch missing"); return DTB_EINVAL; }
    return launch_prod(value, stype, nv, order, order_is64, offsets, ng, n, acc0, (u64*)extra, out_st, out, s);
  }
  u64 init0 = (op == DTB_OP_MIN) ? ~0ull : 0ull;          // 0.0 == 0 bits for float sums
  fill_u64_kernel<<<fgrid, 256, 0, s>>>(acc0, ng, init0);
  count_launch();
  if (op == DTB_OP_MEAN) { fill_u64_kernel<<<fgrid, 256, 0, s>>>(acc1, ng, 0ull); count_launch(); }
  DTB_CUDA_CHECK(cudaGetLastError());
  if (n > 0) {
    DTB_TRY(with_stype(stype, "internal: reducer of stype ", [&](auto t) {
      typedef typename decltype(t)::type T;
      constexpr int SUM = std::is_floating_point<T>::value ? CAT_SUMF : CAT_SUMI;
      switch (op) {
        case DTB_OP_SUM:     return run_reduce<T, SUM>(value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 0, s);
        case DTB_OP_MEAN:    return run_reduce<T, CAT_MEAN>(value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 0, s);
        case DTB_OP_MIN:     return run_reduce<T, CAT_MINMAX>(value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 1, s);
        case DTB_OP_MAX:     return run_reduce<T, CAT_MINMAX>(value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 0, s);
        case DTB_OP_COUNT:   return run_reduce<T, CAT_COUNT>(value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 0, s);
        case DTB_OP_COUNTNA: return run_reduce<T, CAT_COUNT>(value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 1, s);
      }
      set_error("unknown reducer"); return DTB_EINVAL;
    }));
  }
  GroupRows gr;                                 // extra: the zero lookup's marks, float min / max (reduce_extra_bytes)
  gr.v = value; gr.nv = nv; gr.order = order; gr.order_is64 = order_is64; gr.offsets = offsets; gr.n = n;
  gr.zpos = (u64*)extra;
  return finalize(op, stype, acc0, acc1, nullptr, ng, out, gr, s);
}

int reduce_out_stype_host(int op, int st) { return reduce_out_stype(op, st); }

// Groupby invariants (groupby.h:41-47): offsets[0] = 0 and strictly increasing.  reduce_kernel marks
// group starts in a one-bit-per-row bitmap, so an empty group would silently shift every later group of
// the tile: caller-supplied offsets are checked first.  The one exception is the single group of zero rows,
// offsets [0, 0] (Groupby::single_group(0), groupby.cc:60-68), which no row-parallel kernel sees.  *bad
// receives the index of a violating group + 1.
__global__ void offsets_check_kernel(const int32_t* __restrict__ offsets, int64_t ng, int* bad) {
  const bool single_empty = ng == 1 && offsets[1] == 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    if ((offsets[g] >= offsets[g + 1] && !single_empty) || (g == 0 && offsets[0] != 0))
      atomicMax(bad, (int)(g < INT32_MAX ? g + 1 : INT32_MAX));
  }
}

int launch_offsets_check(const int32_t* offsets, int64_t ng, int* d_bad, cudaStream_t s) {
  if (ng == 0) return DTB_OK;
  const int fgrid = grid_for((ng + 255) / 256, 8);
  offsets_check_kernel<<<fgrid, 256, 0, s>>>(offsets, ng, d_bad);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int launch_nrows(const int32_t* offsets, int64_t ng, void* out, cudaStream_t s) {
  if (ng == 0) return DTB_OK;
  const int fgrid = grid_for((ng + 255) / 256, 8);
  nrows_kernel<<<fgrid, 256, 0, s>>>(offsets, ng, (int64_t*)out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// Cumulative functions per group: cumsum / cumprod / cummin / cummax (dtb_cumulative)
// ===========================================================================
// Replaces CumSumProd_ColumnImpl (column/cumsumprod.h) and CumMinMax_ColumnImpl (column/cumminmax.h), which scan
// every group sequentially.  Here it is a segmented scan over the RowIndex positions in fixed tiles of RTILE, so a
// single long group does not serialise it, and the combining order is fixed (two calls give the same bytes):
//   cum_tile_kernel   gathers every position's value through the RowIndex once, writes its contribution to the
//                     scan into out[p] (every output type holds its input type), and the tile's segmented aggregate
//                     (the fold since its last group head) with a flag "the tile holds a head";
//   cum_carry_kernel  one CTA: segmented scan of the tiles' aggregates into every tile's carry-in;
//   cum_emit_kernel   reads the contributions back in order and writes the prefixes, carry-in included.
// REV (reverse=True) mirrors the positions, p -> n - 1 - p, and the offsets with them.
// Bound: HBM (one random gather per row, like dtb_gather, plus one sequential read and write of out).

// One cumulative function over input type T: the scan state S, the element type O of out, the contribution of one
// row (what the tile kernel writes into out), the fold, the merge (a = a then b) and the result of a state.
enum { CUM_SUMI, CUM_SUMF, CUM_PRODI, CUM_PRODF, CUM_MIN, CUM_MAX, CUM_FILL };

template <typename T> struct CumMM { typename RawKey<T>::load_t b; };   // the latest extreme, or T's NA = none

template <int K, typename T> struct Cum;

template <typename T> struct Cum<CUM_SUMI, T> {            // wraps modulo 2^64; an NA row adds 0
  typedef Partial<CAT_SUMI> S; typedef u64 O;
  static __device__ __forceinline__ O contrib(typename RawKey<T>::load_t raw, bool row_valid) {
    u64 u; return (RawKey<T>::get(raw, u) && row_valid) ? u : 0ull;
  }
  static __device__ __forceinline__ void init(S& a) { p_init(a, 0); }
  static __device__ __forceinline__ void add(S& a, O c) { a.s += c; }
  static __device__ __forceinline__ void merge(S& a, const S& b) { p_merge(a, b, 0); }
  static __device__ __forceinline__ S shfl_up(const S& a, int d) { return p_shfl_up(a, d); }
  static __device__ __forceinline__ O result(const S& a) { return a.s; }
};

// Float sums run in float64 and each prefix is rounded once.  An NA row adds +0.0 and the scan starts at -0.0, the
// identity, so a prefix of zeros is -0.0 exactly when every row so far is -0.0, as in the reference's loop.
template <typename T> struct Cum<CUM_SUMF, T> {
  typedef Partial<CAT_SUMF> S; typedef typename RawKey<T>::load_t O;
  static __device__ __forceinline__ O contrib(O raw, bool row_valid) {
    u64 u; return (RawKey<T>::get(raw, u) && row_valid) ? raw : (O)0;
  }
  static __device__ __forceinline__ void init(S& a) { a.s = -0.0; }
  static __device__ __forceinline__ void add(S& a, O c) {
    if constexpr (std::is_same<T, float>::value) a.s += (double)__uint_as_float((u32)c);
    else a.s += __longlong_as_double((long long)c);
  }
  static __device__ __forceinline__ void merge(S& a, const S& b) { p_merge(a, b, 0); }
  static __device__ __forceinline__ S shfl_up(const S& a, int d) { return p_shfl_up(a, d); }
  static __device__ __forceinline__ O result(const S& a) {
    if constexpr (std::is_same<T, float>::value) return (O)__float_as_uint((float)a.s);
    else return (O)__double_as_longlong(a.s);
  }
};

template <typename T> struct Cum<CUM_PRODI, T> {           // wraps modulo 2^64; an NA row multiplies by 1
  typedef Partial<CAT_PRODI> S; typedef u64 O;
  static __device__ __forceinline__ O contrib(typename RawKey<T>::load_t raw, bool row_valid) {
    u64 u; return (RawKey<T>::get(raw, u) && row_valid) ? u : 1ull;
  }
  static __device__ __forceinline__ void init(S& a) { p_init(a, 0); }
  static __device__ __forceinline__ void add(S& a, O c) { a.p *= c; }
  static __device__ __forceinline__ void merge(S& a, const S& b) { p_merge(a, b, 0); }
  static __device__ __forceinline__ S shfl_up(const S& a, int d) { return p_shfl_up(a, d); }
  static __device__ __forceinline__ O result(const S& a) { return a.p; }
};

// Float products keep the significand and the exponent apart (Partial<CAT_PRODF>); an NA row multiplies by 1.0.
template <typename T> struct Cum<CUM_PRODF, T> {
  typedef Partial<CAT_PRODF> S; typedef typename RawKey<T>::load_t O;
  static constexpr O ONE = std::is_same<T, float>::value ? (O)0x3F800000u : (O)0x3FF0000000000000ull;
  static __device__ __forceinline__ O contrib(O raw, bool row_valid) {
    u64 u; return (RawKey<T>::get(raw, u) && row_valid) ? raw : ONE;
  }
  static __device__ __forceinline__ void init(S& a) { p_init(a, 0); }
  static __device__ __forceinline__ void add(S& a, O c) { p_add<T, CAT_PRODF>(a, c, true, 0); }
  static __device__ __forceinline__ void merge(S& a, const S& b) { p_merge(a, b, 0); }
  static __device__ __forceinline__ S shfl_up(const S& a, int d) { return p_shfl_up(a, d); }
  static __device__ __forceinline__ O result(const S& a) {
    bool valid;
    const double r = prodf_value(a, valid);
    if constexpr (std::is_same<T, float>::value) return valid ? (O)__float_as_uint((float)r) : raw_na<T>();
    else return valid ? (O)__double_as_longlong(r) : raw_na<T>();
  }
};

// cummin / cummax: the state is the latest row holding the extreme so far, compared in T (prev < val ? prev : val
// for min, > for max), so of equal values -- -0.0 and +0.0 included -- the later one wins.  "Latest among the
// extremes" is associative.  An NA row leaves the state as it is; before the first valid row the state is NA.
// CUM_FILL (fillna without a value) is the same state with every valid row winning: the latest valid value.
template <int K, typename T> struct CumMinMax {
  typedef CumMM<T> S; typedef typename RawKey<T>::load_t O;
  static __device__ __forceinline__ O contrib(O raw, bool row_valid) { return row_valid ? raw : na(); }
  static __device__ __forceinline__ O na() { return raw_na<T>(); }
  static __device__ __forceinline__ bool valid(O b) { u64 u; return RawKey<T>::get(b, u); }
  static __device__ __forceinline__ T val(O b) {
    if constexpr (std::is_same<T, float>::value) return __uint_as_float((u32)b);
    else if constexpr (std::is_same<T, double>::value) return __longlong_as_double((long long)b);
    else return b;
  }
  static __device__ __forceinline__ void init(S& a) { a.b = na(); }
  static __device__ __forceinline__ void add(S& a, O c) {
    if (!valid(c)) return;
    if (K != CUM_FILL && valid(a.b) && (K == CUM_MIN ? val(a.b) < val(c) : val(a.b) > val(c))) return;
    a.b = c;
  }
  static __device__ __forceinline__ void merge(S& a, const S& b) { add(a, b.b); }
  static __device__ __forceinline__ S shfl_up(const S& a, int d) { S r; r.b = __shfl_up_sync(0xffffffffu, a.b, d); return r; }
  static __device__ __forceinline__ O result(const S& a) { return a.b; }
};
template <typename T> struct Cum<CUM_MIN, T> : CumMinMax<CUM_MIN, T> {};
template <typename T> struct Cum<CUM_MAX, T> : CumMinMax<CUM_MAX, T> {};
template <typename T> struct Cum<CUM_FILL, T> : CumMinMax<CUM_FILL, T> {};

// (a, f) = (pa, pf) then (a, f): a segment state is the fold since the last head, f = a head was seen
template <class C>
__device__ __forceinline__ void seg_after(typename C::S& a, u32& f, const typename C::S& pa, u32 pf) {
  if (!f) { typename C::S t = pa; C::merge(t, a); a = t; }
  f |= pf;
}

// Segmented scan over the CTA's threads in thread order (NW warps).  In: the thread's own (a, f).  Out: (a, f) =
// the exclusive prefix of the threads before it, and (ta, tf) = the CTA's total.  s_a / s_f: NW + 1 slots.
template <class C, int NW>
__device__ __forceinline__ void block_seg_scan(typename C::S& a, u32& f, typename C::S* s_a, u32* s_f,
                                               typename C::S& ta, u32& tf) {
  typedef typename C::S S;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const S o = C::shfl_up(a, d);
    const u32 of = __shfl_up_sync(0xffffffffu, f, d);
    if (lane >= d) seg_after<C>(a, f, o, of);
  }
  if (lane == 31) { s_a[w] = a; s_f[w] = f; }
  S e = C::shfl_up(a, 1);
  u32 ef = __shfl_up_sync(0xffffffffu, f, 1);
  if (lane == 0) { C::init(e); ef = 0; }
  __syncthreads();
  if (threadIdx.x == 0) {
    S run; C::init(run); u32 rf = 0;
    for (int i = 0; i < NW; i++) {
      S x = s_a[i]; u32 xf = s_f[i];
      s_a[i] = run; s_f[i] = rf;
      seg_after<C>(x, xf, run, rf);
      run = x; rf = xf;
    }
    s_a[NW] = run; s_f[NW] = rf;
  }
  __syncthreads();
  seg_after<C>(e, ef, s_a[w], s_f[w]);
  a = e; f = ef;
  ta = s_a[NW]; tf = s_f[NW];
}

// The tile's head bits of this thread's RIPT positions; bit 0 of thread 0 is set when a group starts at the tile's
// first position (tile_heads leaves that one out).
template <bool REV>
__device__ __forceinline__ u32 cum_heads(const int32_t* __restrict__ offsets, int64_t ng, int64_t n, int64_t t0,
                                         int64_t t1, int64_t* s_g, u32* s_bits) {
  const int tid = threadIdx.x;
  if (tid < RTILE / 32) s_bits[tid] = 0;
  int64_t g_lo, g_hi;
  tile_heads<REV>(offsets, ng, n, t0, t1, tid, s_g, s_bits, g_lo, g_hi);
  const int c0 = tid * RIPT;
  u32 bits = (s_bits[c0 >> 5] >> (c0 & 31)) & 0xffu;
  if (tid == 0 && head_offset<REV>(offsets, ng, n, g_lo) == t0) bits |= 1u;
  return bits;
}

template <int K, typename T, bool REV, typename OrdT>
__global__ void __launch_bounds__(RT, 1)
cum_tile_kernel(const typename RawKey<T>::load_t* __restrict__ v, int64_t nv, const OrdT* __restrict__ order,
                const int32_t* __restrict__ offsets, int64_t ng, int64_t n, typename Cum<K, T>::O* __restrict__ out,
                typename Cum<K, T>::S* __restrict__ tagg, u32* __restrict__ thead)
{
  typedef Cum<K, T> C;
  typedef typename C::S S;
  typedef typename RawKey<T>::load_t L;
  __shared__ int64_t s_g[2];
  __shared__ u32 s_bits[RTILE / 32];
  __shared__ S s_a[RT / 32 + 1];
  __shared__ u32 s_f[RT / 32 + 1];
  const int64_t t0 = (int64_t)blockIdx.x * RTILE;
  const int64_t t1 = (t0 + RTILE < n) ? t0 + RTILE : n;
  const u32 bits = cum_heads<REV>(offsets, ng, n, t0, t1, s_g, s_bits);

  // gather: all index loads first, then all value loads
  const int64_t q0 = t0 + threadIdx.x * RIPT, p0 = REV ? n - 1 - q0 : q0;   // position q is p0 -+ (q - q0)
  int64_t row[RIPT];
#pragma unroll
  for (int i = 0; i < RIPT; i++) {
    const int64_t p = REV ? p0 - i : p0 + i;
    row[i] = (q0 + i < n) ? (order ? (int64_t)order[p] : p) : -2;
  }
  L val[RIPT];
#pragma unroll
  for (int i = 0; i < RIPT; i++) val[i] = (row[i] >= 0 && row[i] < nv) ? v[row[i]] : (L)0;

  S a; C::init(a);
  u32 f = 0;
#pragma unroll
  for (int i = 0; i < RIPT; i++) {
    if (q0 + i < n) {
      const typename C::O c = C::contrib(val[i], row[i] >= 0 && row[i] < nv);
      out[REV ? p0 - i : p0 + i] = c;
      if (bits & (1u << i)) { C::init(a); f = 1; }
      C::add(a, c);
    }
  }
  S ta; u32 tf;
  block_seg_scan<C, RT / 32>(a, f, s_a, s_f, ta, tf);
  if (threadIdx.x == 0) { tagg[blockIdx.x] = ta; thead[blockIdx.x] = tf; }
}

// tagg[t] <- the state of the group open at tile t's first position, before it (the carry-in); one CTA of CARRY_T
// threads, each over a run of consecutive tiles
constexpr int CARRY_T = 1024;

template <int K, typename T>
__global__ void __launch_bounds__(CARRY_T)
cum_carry_kernel(typename Cum<K, T>::S* __restrict__ tagg, const u32* __restrict__ thead, int64_t ntiles)
{
  typedef Cum<K, T> C;
  typedef typename C::S S;
  __shared__ S s_a[CARRY_T / 32 + 1];
  __shared__ u32 s_f[CARRY_T / 32 + 1];
  const int64_t per = (ntiles + CARRY_T - 1) / CARRY_T;
  const int64_t b = (int64_t)threadIdx.x * per, e = (b + per < ntiles) ? b + per : ntiles;
  S a; C::init(a);
  u32 f = 0;
  for (int64_t t = b; t < e; t++) {
    S x = tagg[t]; u32 xf = thead[t];
    seg_after<C>(x, xf, a, f);
    a = x; f = xf;
  }
  S ta; u32 tf;
  block_seg_scan<C, CARRY_T / 32>(a, f, s_a, s_f, ta, tf);
  for (int64_t t = b; t < e; t++) {
    const S x = tagg[t];
    const u32 xf = thead[t];
    tagg[t] = a;
    if (xf) a = x; else C::merge(a, x);
  }
}

template <int K, typename T, bool REV>
__global__ void __launch_bounds__(RT)
cum_emit_kernel(const int32_t* __restrict__ offsets, int64_t ng, int64_t n, typename Cum<K, T>::O* __restrict__ out,
                const typename Cum<K, T>::S* __restrict__ tcarry)
{
  typedef Cum<K, T> C;
  typedef typename C::S S;
  typedef typename C::O O;
  __shared__ int64_t s_g[2];
  __shared__ u32 s_bits[RTILE / 32];
  __shared__ S s_a[RT / 32 + 1];
  __shared__ u32 s_f[RT / 32 + 1];
  const int64_t t0 = (int64_t)blockIdx.x * RTILE;
  const int64_t t1 = (t0 + RTILE < n) ? t0 + RTILE : n;
  const u32 bits = cum_heads<REV>(offsets, ng, n, t0, t1, s_g, s_bits);

  const int64_t q0 = t0 + threadIdx.x * RIPT, p0 = REV ? n - 1 - q0 : q0;
  O c[RIPT];
#pragma unroll
  for (int i = 0; i < RIPT; i++) c[i] = (q0 + i < n) ? out[REV ? p0 - i : p0 + i] : (O)0;
  S a; C::init(a);
  u32 f = 0;
#pragma unroll
  for (int i = 0; i < RIPT; i++) {
    if (q0 + i < n) {
      if (bits & (1u << i)) { C::init(a); f = 1; }
      C::add(a, c[i]);
    }
  }
  S ta; u32 tf;
  block_seg_scan<C, RT / 32>(a, f, s_a, s_f, ta, tf);
  seg_after<C>(a, f, tcarry[blockIdx.x], 0);              // the running state before this thread's first position
#pragma unroll
  for (int i = 0; i < RIPT; i++) {
    if (q0 + i < n) {
      if (bits & (1u << i)) C::init(a);
      C::add(a, c[i]);
      out[REV ? p0 - i : p0 + i] = C::result(a);
    }
  }
}

int cumulative_out_stype(int op, int st) {
  const bool isint = (st == DTB_STYPE_BOOL || st == DTB_STYPE_INT8 || st == DTB_STYPE_INT16 ||
                      st == DTB_STYPE_INT32 || st == DTB_STYPE_INT64);
  const bool isflt = (st == DTB_STYPE_FLOAT32 || st == DTB_STYPE_FLOAT64);
  switch (op) {
    case DTB_OP_SUM: case DTB_OP_PROD:                        // fexpr_cumsumprod.cc: evaluate1
      return isint ? DTB_STYPE_INT64 : (isflt ? st : 0);
    case DTB_OP_MIN: case DTB_OP_MAX:                         // fexpr_cumminmax.cc: the column's own stype
      return (isint || isflt || st == DTB_STYPE_DATE32 || st == DTB_STYPE_TIME64) ? st : 0;
  }
  return 0;
}

// tagg: the largest scan state (Partial<CAT_PRODF>) per tile, then the tiles' head flags
size_t cumulative_scratch_bytes(int64_t n) {
  const size_t ntiles = (size_t)((n + RTILE - 1) / RTILE);
  return ntiles * (sizeof(Partial<CAT_PRODF>) + sizeof(u32));
}

template <int K, typename T, bool REV>
static int run_cumulative(const void* v, int64_t nv, const void* order, int order_is64, const int32_t* offsets,
                          int64_t ng, int64_t n, void* scratch, void* out, cudaStream_t s)
{
  typedef Cum<K, T> C;
  typedef typename RawKey<T>::load_t L;
  const int64_t ntiles = (n + RTILE - 1) / RTILE;
  typename C::S* tagg = (typename C::S*)scratch;
  u32* thead = (u32*)((char*)scratch + (size_t)ntiles * sizeof(Partial<CAT_PRODF>));
  typename C::O* o = (typename C::O*)out;
  with_order(order, order_is64, [&](auto ord) {
    cum_tile_kernel<K, T, REV><<<(unsigned)ntiles, RT, 0, s>>>((const L*)v, nv, ord, offsets, ng, n, o, tagg, thead);
  });
  cum_carry_kernel<K, T><<<1, CARRY_T, 0, s>>>(tagg, thead, ntiles);
  cum_emit_kernel<K, T, REV><<<(unsigned)ntiles, RT, 0, s>>>(offsets, ng, n, o, tagg);
  count_launch(3);
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

template <int K, typename T>
static int run_cumulative_dir(int reverse, const void* v, int64_t nv, const void* order, int order_is64,
                              const int32_t* offsets, int64_t ng, int64_t n, void* scratch, void* out, cudaStream_t s)
{
  return reverse ? run_cumulative<K, T, true>(v, nv, order, order_is64, offsets, ng, n, scratch, out, s)
                 : run_cumulative<K, T, false>(v, nv, order, order_is64, offsets, ng, n, scratch, out, s);
}

// out: n elements of cumulative_out_stype(op, stype), out[p] for RowIndex position p; scratch:
// cumulative_scratch_bytes(n) of device memory.  The stype is checked by the caller.
int launch_cumulative(int op, int reverse, const void* v, int stype, int64_t nv, const void* order, int order_is64,
                      const int32_t* offsets, int64_t ng, int64_t n, void* scratch, void* out, cudaStream_t s)
{
  if (n <= 0) return DTB_OK;
  return with_stype(stype, "internal: cumulative function of stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    constexpr bool ISF = std::is_floating_point<T>::value;
    switch (op) {
      case DTB_OP_SUM:
        return run_cumulative_dir<ISF ? CUM_SUMF : CUM_SUMI, T>(reverse, v, nv, order, order_is64, offsets, ng, n, scratch, out, s);
      case DTB_OP_PROD:
        return run_cumulative_dir<ISF ? CUM_PRODF : CUM_PRODI, T>(reverse, v, nv, order, order_is64, offsets, ng, n, scratch, out, s);
      case DTB_OP_MIN: return run_cumulative_dir<CUM_MIN, T>(reverse, v, nv, order, order_is64, offsets, ng, n, scratch, out, s);
      case DTB_OP_MAX: return run_cumulative_dir<CUM_MAX, T>(reverse, v, nv, order, order_is64, offsets, ng, n, scratch, out, s);
    }
    set_error("internal: cumulative function / stype combination"); return DTB_EINVAL;
  });
}

// ===========================================================================
// Row functions per group: fillna, shift, cumcount, ngroup (dtb_fillna, dtb_shift, dtb_group_index)
// ===========================================================================
// fillna without a value replaces fill_rowindex (expr/fexpr_fillna.cc:66-118) and the apply_rowindex after it: it is
// CUM_FILL of the cumulative scan above, the latest valid value of the group so far (REV: the earliest at or after).
//
// shift, cumcount and ngroup need no scan: a position's result depends only on its group's bounds.  One row-parallel
// kernel over tiles of RTILE positions does them; the group of every position comes from the tile's head bitmap and
// its popcount prefix, as in reduce_kernel.  Position q of the tile is t0 + i * RT + tid, so order is read and out
// is written coalesced.
//   ROW_SHIFT     out[p] = value[order[p - shift]] where p - shift lies in p's group [start, end), else NA: replaces
//                 compute_lag_rowindex (expr/head_func_shift.cc:40-64) and the apply_rowindex after it in one pass;
//                 no RowIndex of source positions is built.  Bound: the random value reads of a gather.
//   ROW_CUMCOUNT  out[p] = p - start, reverse: end - 1 - p        (column/cumcountngroup.h:48-66)
//   ROW_NGROUP    out[p] = g, reverse: ng - 1 - g                  Bound: the 8-byte write per row.
enum { ROW_SHIFT, ROW_CUMCOUNT, ROW_NGROUP };

template <int KIND, typename T, typename OrdT>
__global__ void __launch_bounds__(RT, 1)
group_row_kernel(const typename RawKey<T>::load_t* __restrict__ v, int64_t nv, const OrdT* __restrict__ order,
                 const int32_t* __restrict__ offsets, int64_t ng, int64_t n, int64_t shift, int reverse,
                 typename RawKey<T>::load_t* __restrict__ out)
{
  typedef typename RawKey<T>::load_t L;
  __shared__ int64_t s_g[2];
  __shared__ u32 s_bits[RTILE / 32];
  __shared__ u32 s_wpre[RTILE / 32];
  const int tid = threadIdx.x, lane = tid & 31;
  const int64_t t0 = (int64_t)blockIdx.x * RTILE;
  const int64_t t1 = (t0 + RTILE < n) ? t0 + RTILE : n;
  if (tid < RTILE / 32) s_bits[tid] = 0;
  int64_t g_lo, g_hi;
  tile_heads<false>(offsets, ng, n, t0, t1, tid, s_g, s_bits, g_lo, g_hi);
  if (tid < 32) {
    // exclusive prefix of popcounts over the RTILE/32 = 64 bitmap words (2 per lane)
    const u32 a = __popc(s_bits[2 * lane]), b = __popc(s_bits[2 * lane + 1]);
    u32 incl = a + b;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const u32 o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += o;
    }
    s_wpre[2 * lane] = incl - a - b;
    s_wpre[2 * lane + 1] = incl - b;
  }
  __syncthreads();
  // the group of tile position c is g_lo + heads(c), the number of heads at positions 1 .. c
  auto heads = [&](int c) -> u32 { return s_wpre[c >> 5] + __popc(s_bits[c >> 5] & ((2u << (c & 31)) - 1u)); };

  if constexpr (KIND == ROW_SHIFT) {
    // all index loads first, then all value loads
    int64_t row[RIPT];
#pragma unroll
    for (int i = 0; i < RIPT; i++) {
      const int c = i * RT + tid;
      const int64_t p = t0 + c, src = p - shift;               // |shift| <= 2^32: no overflow
      row[i] = -1;
      if (p < n) {
        const int64_t g = g_lo + heads(c);
        if (src >= (int64_t)offsets[g] && src < (int64_t)offsets[g + 1]) row[i] = order ? (int64_t)order[src] : src;
      }
    }
    L val[RIPT];
#pragma unroll
    for (int i = 0; i < RIPT; i++) val[i] = (row[i] >= 0 && row[i] < nv) ? v[row[i]] : raw_na<T>();
#pragma unroll
    for (int i = 0; i < RIPT; i++) {
      const int64_t p = t0 + i * RT + tid;
      u64 u;
      if (p < n) out[p] = RawKey<T>::get(val[i], u) ? val[i] : raw_na<T>();    // every NA as the stype's NA
    }
  } else if constexpr (KIND == ROW_CUMCOUNT) {
#pragma unroll
    for (int i = 0; i < RIPT; i++) {
      const int c = i * RT + tid;
      const int64_t p = t0 + c, g = g_lo + heads(c);
      if (p < n) out[p] = reverse ? (int64_t)offsets[g + 1] - 1 - p : p - (int64_t)offsets[g];
    }
  } else {
    const int64_t base = reverse ? ng - 1 - g_lo : g_lo;       // ngroup: base -+ heads(c)
#pragma unroll
    for (int i = 0; i < RIPT; i++) {
      const int c = i * RT + tid;
      const int64_t p = t0 + c, k = heads(c);
      if (p < n) out[p] = reverse ? base - k : base + k;
    }
  }
}

template <typename T>
static int run_shift(const void* v, int64_t nv, const void* order, int order_is64, const int32_t* offsets, int64_t ng,
                     int64_t n, int64_t shift, void* out, cudaStream_t s)
{
  typedef typename RawKey<T>::load_t L;
  const unsigned grid = (unsigned)((n + RTILE - 1) / RTILE);
  with_order(order, order_is64, [&](auto o) {
    group_row_kernel<ROW_SHIFT, T><<<grid, RT, 0, s>>>((const L*)v, nv, o, offsets, ng, n, shift, 0, (L*)out);
  });
  count_launch(1);
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// out: n elements of the value's stype, out[p] for RowIndex position p.  The stype is checked by the caller.
int launch_shift(const void* v, int stype, int64_t nv, const void* order, int order_is64, const int32_t* offsets,
                 int64_t ng, int64_t n, int64_t shift, void* out, cudaStream_t s)
{
  if (n <= 0) return DTB_OK;
  // positions are below 2^31, so every |shift| beyond that puts each source outside its group
  const int64_t lim = (int64_t)1 << 32;
  shift = shift > lim ? lim : (shift < -lim ? -lim : shift);
  return with_stype(stype, "internal: shift of stype ", [&](auto t) {
    return run_shift<typename decltype(t)::type>(v, nv, order, order_is64, offsets, ng, n, shift, out, s);
  });
}

// out: n elements of the value's stype; scratch: cumulative_scratch_bytes(n) of device memory.
int launch_fillna(int reverse, const void* v, int stype, int64_t nv, const void* order, int order_is64,
                  const int32_t* offsets, int64_t ng, int64_t n, void* scratch, void* out, cudaStream_t s)
{
  if (n <= 0) return DTB_OK;
  return with_stype(stype, "internal: fillna of stype ", [&](auto t) {
    return run_cumulative_dir<CUM_FILL, typename decltype(t)::type>(reverse, v, nv, order, order_is64, offsets, ng, n,
                                                                    scratch, out, s);
  });
}

// kind: DTB_GROUP_CUMCOUNT or DTB_GROUP_NGROUP (checked by the caller); out: n int64 values.
int launch_group_index(int kind, int reverse, const int32_t* offsets, int64_t ng, int64_t n, int64_t* out,
                       cudaStream_t s)
{
  if (n <= 0) return DTB_OK;
  const unsigned grid = (unsigned)((n + RTILE - 1) / RTILE);
  if (kind == DTB_GROUP_CUMCOUNT)
    group_row_kernel<ROW_CUMCOUNT, int64_t, int32_t><<<grid, RT, 0, s>>>(nullptr, 0, nullptr, offsets, ng, n, 0,
                                                                          reverse, out);
  else
    group_row_kernel<ROW_NGROUP, int64_t, int32_t><<<grid, RT, 0, s>>>(nullptr, 0, nullptr, offsets, ng, n, 0,
                                                                        reverse, out);
  count_launch(1);
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// Direct-address reducers (small key domains)
// ===========================================================================
// When the group key of a row can be computed from the key columns alone -- the normalised
// composite key x = X(row) >> group_shift spans at most 2^22 values -- the reducers do not
// need the RowIndex at all: rows are streamed in storage order (coalesced, no gather), and
// each row folds its value into acc[x] with one L2 atomic.  One table (<= 32 MB) fits the
// 50 MB L2 of an H100.  Few keys and skewed group sizes, where one atomic per row would
// serialise on a handful of addresses, take the kernels further down (plan_direct chooses).
// A finalize kernel maps group g -> acc[gkeys[g]] and applies the reference's output stype /
// NA rules.
//
// Bound: L2 atomic throughput, then HBM.
// Algorithmic bytes per row: key column(s) + value column, read once.
template <typename T, int CAT, typename KSrc>
__global__ void __launch_bounds__(512)
direct_reduce_kernel(KSrc ksrc, int gshift, const typename RawKey<T>::load_t* __restrict__ v,
                     int64_t n, u64* acc0, u64* acc1, int flag)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const u32 x = (u32)(ksrc.load(i) >> gshift);
    // keeps the key load next to the value load: otherwise the compiler sinks it under p_flush's test of the
    // value, the two loads of a row serialise, and C2's accumulation measured slower
    asm volatile("" :: "r"(x));
    Partial<CAT> part; p_init(part, flag);
    p_add<T, CAT>(part, v[i], true, flag);
    p_flush(part, (int64_t)x, acc0, acc1, flag);
  }
}

// key sources: one raw column normalised on the fly, or the general multi-column composite
template <typename TK>
struct DirectRawKey {
  RawSrc<TK, u32> src;                       // the direct path only exists for keys of <= 22 bits
  __device__ __forceinline__ u64 load(int64_t i) const { return (u64)src.load(i); }
};
struct DirectComposite {
  KeyPlan kp;
  __device__ __forceinline__ u64 load(int64_t i) const {
    u64 x = 0;
    for (int c = 0; c < kp.nkeys; c++) x |= norm_load_dynamic(kp.k[c], i) << kp.k[c].lshift;
    return x;
  }
};

// One shared-memory accumulator slot (the words a CTA-local table keeps per key) -> the global table.
template <int CAT>
__device__ __forceinline__ void slot_flush(u64 a0, u64 a1, int64_t g, u64* acc0, u64* acc1, int flag) {
  if constexpr (CAT == CAT_SUMI) { if (a0) atomicAdd(&acc0[g], a0); }
  else if constexpr (CAT == CAT_SUMF) {
    const double d = __longlong_as_double((long long)a0);
    if (d != 0.0) atomicAdd(reinterpret_cast<double*>(acc0) + g, d);
  }
  else if constexpr (CAT == CAT_MEAN) {
    if (a1) { atomicAdd(reinterpret_cast<double*>(acc0) + g, __longlong_as_double((long long)a0)); atomicAdd(&acc1[g], a1); }
  }
  else if constexpr (CAT == CAT_MINMAX) {
    if (flag) { if (a0 != ~0ull) atomicMin(&acc0[g], a0); }
    else      { if (a0 != 0ull)  atomicMax(&acc0[g], a0); }
  }
  else { if (a0) atomicAdd(&acc0[g], a0); }
}

// Few distinct group keys (<= 2048): every CTA folds its rows into a shared-memory copy of the
// accumulator table and flushes it once, so the L2 sees gridDim x groups atomics instead of one per row
// (100 keys at 2e8 rows = 1.6e8 same-address L2 atomics; low-cardinality by() is the common case).  SMALL_TABLE:
// dtb_internal.h.

template <typename T, int CAT, typename KSrc>
__global__ void __launch_bounds__(512)
direct_reduce_small_kernel(KSrc ksrc, int gshift, const typename RawKey<T>::load_t* __restrict__ v,
                           int64_t n, int table, const uint16_t* __restrict__ dense,
                           u64* acc0, u64* acc1, int flag)
{
  __shared__ u64 s0[SMALL_TABLE];
  __shared__ u64 s1[SMALL_TABLE];
  const u64 ident = (CAT == CAT_MINMAX && flag) ? ~0ull : 0ull;
  // very few keys (<= 128): one private copy of the table per warp, so that the 16 warps of the CTA do
  // not serialise on the same handful of shared-memory addresses
  const int copies = (table * 16 <= SMALL_TABLE) ? 16 : 1;
  const int wofs = (copies > 1) ? (int)(threadIdx.x >> 5) * table : 0;
  for (int i = threadIdx.x; i < table * copies; i += blockDim.x) { s0[i] = ident; s1[i] = 0; }
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    u32 x = (u32)(ksrc.load(i) >> gshift);
    if (dense) x = dense[x];                                   // sparse key domain, few groups: x -> group
    Partial<CAT> part; p_init(part, flag);
    p_add<T, CAT>(part, v[i], true, flag);
    p_flush(part, (int64_t)(wofs + x), s0, s1, flag);          // shared-memory atomics
  }
  __syncthreads();
  if (copies > 1) {                                             // fold the warps' copies into copy 0
    for (int i = threadIdx.x; i < table; i += blockDim.x) {
      for (int w = 1; w < copies; w++) {
        const u64 a = s0[w * table + i], b = s1[w * table + i];
        if constexpr (CAT == CAT_SUMF || CAT == CAT_MEAN)
          s0[i] = (u64)__double_as_longlong(__longlong_as_double((long long)s0[i]) + __longlong_as_double((long long)a));
        else if constexpr (CAT == CAT_MINMAX) s0[i] = flag ? (a < s0[i] ? a : s0[i]) : (a > s0[i] ? a : s0[i]);
        else s0[i] += a;
        s1[i] += b;
      }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < table; i += blockDim.x) slot_flush<CAT>(s0[i], s1[i], (int64_t)i, acc0, acc1, flag);
}

// Skewed group sizes (some key owns more than ~0.1 % of the rows): one L2 atomic per row would
// serialise on the hot accumulators (same-address L2 atomics retire one at a time).  `hot[x]` (built from the group sizes, see plan_direct) marks the
// keys above the threshold; their rows are folded inside the warp (MATCH.ANY, only in warps that hold
// a hot row) and then inside the CTA in a small open-addressed shared-memory table that is flushed
// once per CTA; every other row takes the plain one-atomic path.
constexpr int HOT_SLOTS = 2048;
constexpr u32 HOT_EMPTY = 0xffffffffu;

template <typename T, int CAT, typename KSrc>
__global__ void __launch_bounds__(512)
direct_reduce_hot_kernel(KSrc ksrc, int gshift, const typename RawKey<T>::load_t* __restrict__ v,
                         int64_t n, const uint8_t* __restrict__ hot, u64* acc0, u64* acc1, int flag)
{
  __shared__ u32 hkey[HOT_SLOTS];
  __shared__ u64 h0[HOT_SLOTS];
  __shared__ u64 h1[HOT_SLOTS];
  const u64 ident = (CAT == CAT_MINMAX && flag) ? ~0ull : 0ull;
  for (int i = threadIdx.x; i < HOT_SLOTS; i += blockDim.x) { hkey[i] = HOT_EMPTY; h0[i] = ident; h1[i] = 0; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t nround = ((n + 31) / 32) * 32;                // keep whole warps in the loop
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nround; i += stride) {
    const bool in = i < n;
    u32 x = 0;
    Partial<CAT> part; p_init(part, flag);
    bool is_hot = false;
    if (in) {
      x = (u32)(ksrc.load(i) >> gshift);
      p_add<T, CAT>(part, v[i], true, flag);
      is_hot = hot[x] != 0;
    }
    if (__any_sync(0xffffffffu, is_hot)) {                      // warp-uniform: the body shuffles
      // cold lanes match nobody (their tag is unique in the warp; x < 2^22)
      const unsigned peers = __match_any_sync(0xffffffffu, is_hot ? x : (0x80000000u | (u32)lane));
      const int leader = __ffs(peers) - 1;
      unsigned rest = peers & ~(1u << leader);
      Partial<CAT> tot = part;
      while (__any_sync(0xffffffffu, rest != 0)) {
        const int src = rest ? (__ffs(rest) - 1) : lane;
        Partial<CAT> o;
        if constexpr (CAT == CAT_SUMI) o.s = __shfl_sync(0xffffffffu, part.s, src);
        else if constexpr (CAT == CAT_SUMF) o.s = __shfl_sync(0xffffffffu, part.s, src);
        else if constexpr (CAT == CAT_MEAN) { o.s = __shfl_sync(0xffffffffu, part.s, src); o.c = __shfl_sync(0xffffffffu, part.c, src); }
        else if constexpr (CAT == CAT_MINMAX) o.key = __shfl_sync(0xffffffffu, part.key, src);
        else o.c = __shfl_sync(0xffffffffu, part.c, src);
        if (rest && lane == leader) p_merge(tot, o, flag);
        rest &= rest - 1;
      }
      if (is_hot) {
        if (lane == leader) {
          bool done = false;
          const u32 h = (x * 2654435761u) >> 21;                // 11 bits
#pragma unroll 1
          for (int t = 0; t < 8 && !done; t++) {
            const u32 slot = (h + (u32)t) & (HOT_SLOTS - 1);
            const u32 old = atomicCAS(&hkey[slot], HOT_EMPTY, x);
            if (old == HOT_EMPTY || old == x) { p_flush(tot, (int64_t)slot, h0, h1, flag); done = true; }
          }
          if (!done) p_flush(tot, (int64_t)x, acc0, acc1, flag);
        }
      }
    }
    if (in && !is_hot) p_flush(part, (int64_t)x, acc0, acc1, flag);   // hot rows never touch L2 directly
  }
  __syncthreads();
  for (int i = threadIdx.x; i < HOT_SLOTS; i += blockDim.x)
    if (hkey[i] != HOT_EMPTY) slot_flush<CAT>(h0[i], h1[i], (int64_t)hkey[i], acc0, acc1, flag);
}

template <typename T, int CAT, typename KSrc>
static int run_direct(const DirectPlan& dp, const KSrc& ks, int gshift, const void* v, int64_t n, u64* acc0, u64* acc1,
                      int flag, cudaStream_t s)
{
  typedef typename RawKey<T>::load_t L;
  const int64_t want = (n + 511) / 512;
  if (dp.kind == DIRECT_SMALL)
    direct_reduce_small_kernel<T, CAT, KSrc><<<grid_for(want, 4), 512, 0, s>>>(ks, gshift, (const L*)v, n, (int)dp.nslots,
                                                                               (const uint16_t*)dp.map, acc0, acc1, flag);
  else if (dp.kind == DIRECT_HOT)
    direct_reduce_hot_kernel<T, CAT, KSrc><<<grid_for(want, 4), 512, 0, s>>>(ks, gshift, (const L*)v, n,
                                                                             (const uint8_t*)dp.map, acc0, acc1, flag);
  else
    direct_reduce_kernel<T, CAT, KSrc><<<grid_for(want, 16), 512, 0, s>>>(ks, gshift, (const L*)v, n, acc0, acc1, flag);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

template <typename T, typename KSrc>
static int direct_op(const DirectPlan& dp, int op, const KSrc& ks, int gshift, const void* v, int64_t n,
                     u64* acc0, u64* acc1, cudaStream_t s)
{
  constexpr int SUM = std::is_floating_point<T>::value ? CAT_SUMF : CAT_SUMI;
  switch (op) {
    case DTB_OP_SUM:     return run_direct<T, SUM>(dp, ks, gshift, v, n, acc0, acc1, 0, s);
    case DTB_OP_MEAN:    return run_direct<T, CAT_MEAN>(dp, ks, gshift, v, n, acc0, acc1, 0, s);
    case DTB_OP_MIN:     return run_direct<T, CAT_MINMAX>(dp, ks, gshift, v, n, acc0, acc1, 1, s);
    case DTB_OP_MAX:     return run_direct<T, CAT_MINMAX>(dp, ks, gshift, v, n, acc0, acc1, 0, s);
    case DTB_OP_COUNT:   return run_direct<T, CAT_COUNT>(dp, ks, gshift, v, n, acc0, acc1, 0, s);
    case DTB_OP_COUNTNA: return run_direct<T, CAT_COUNT>(dp, ks, gshift, v, n, acc0, acc1, 1, s);
  }
  set_error("unknown reducer"); return DTB_EINVAL;
}

// ---- how the rows are streamed: decided on the host once the groups are known ----------------
__global__ void dense_map_kernel(const u32* __restrict__ gkeys, int64_t ng, uint16_t* __restrict__ dense) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < ng) dense[gkeys[g]] = (uint16_t)g;
}
__global__ void hot_map_kernel(const u32* __restrict__ gkeys, const int32_t* __restrict__ offsets, int64_t ng,
                               u32 thresh, uint8_t* __restrict__ hot) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride)
    if ((u32)(offsets[g + 1] - offsets[g]) > thresh) hot[gkeys[g]] = 1;
}

size_t direct_map_bytes(int64_t table) { return (size_t)table * sizeof(uint16_t); }

int plan_direct(int64_t table, const uint32_t* gkeys, const int32_t* offsets, int64_t ng, int64_t n,
                int64_t gmax, void* map_scratch, cudaStream_t s, DirectPlan& dp)
{
  dp.kind = DIRECT_PLAIN; dp.map = nullptr; dp.nslots = table;
  if (ng <= 0) return DTB_OK;
  if (table <= SMALL_TABLE) { dp.kind = DIRECT_SMALL; return DTB_OK; }
  if (ng <= SMALL_TABLE) {
    // few groups in a sparse key domain: x -> group through an L2-resident map (only the entries of
    // keys that occur are ever read, so the map needs no initialisation)
    dense_map_kernel<<<(unsigned)((ng + 255) / 256), 256, 0, s>>>(gkeys, ng, (uint16_t*)map_scratch);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    dp.kind = DIRECT_SMALL; dp.map = map_scratch; dp.nslots = ng;
    return DTB_OK;
  }
  const int64_t hot_at = (n / 1024 > 8192) ? n / 1024 : 8192;      // a key this large makes the call "skewed"
  if (gmax > hot_at) {
    const int64_t key_thresh = (n / 2048 > 1024) ? n / 2048 : 1024;  // at most 2048 keys can exceed it
    DTB_CUDA_CHECK(cudaMemsetAsync(map_scratch, 0, (size_t)table, s));
    const int grid = grid_for((ng + 255) / 256, 8);
    hot_map_kernel<<<grid, 256, 0, s>>>(gkeys, offsets, ng, (u32)key_thresh, (uint8_t*)map_scratch);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    dp.kind = DIRECT_HOT; dp.map = map_scratch;
  }
  return DTB_OK;
}

// Stage 1: stream every row into acc[x] (acc[group] for a dense-mapped small table).  acc0/acc1: device
// scratch of `table` u64 each.  First the accumulator tables' identities (once per reducer; the rows may then
// arrive in pieces):
int launch_direct_init(int op, const DirectPlan& dp, int64_t table, u64* acc0, u64* acc1, cudaStream_t s)
{
  if (dp.kind == DIRECT_SMALL) table = dp.nslots;                // only the used accumulators are initialised
  const int tgrid = grid_for((table + 255) / 256, 8);
  fill_u64_kernel<<<tgrid, 256, 0, s>>>(acc0, table, (op == DTB_OP_MIN) ? ~0ull : 0ull);
  count_launch();
  if (op == DTB_OP_MEAN) { fill_u64_kernel<<<tgrid, 256, 0, s>>>(acc1, table, 0ull); count_launch(); }
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// folds n rows (kp's key columns and `value`, both starting at the piece's first row) into the tables
int launch_direct_accumulate_rows(int op, const KeyPlan& kp, const DirectPlan& dp,
                                  const void* value, int stype, int64_t n, u64* acc0, u64* acc1, cudaStream_t s)
{
  const int out_st = reduce_out_stype(op, stype);
  if (!out_st) { set_error("Invalid column type in reducer"); return DTB_EINVAL; }
  if (n <= 0) return DTB_OK;
  auto accumulate = [&](const auto& ks) {
    return with_stype(stype, "internal: reducer of stype ", [&](auto t) {
      return direct_op<typename decltype(t)::type>(dp, op, ks, kp.group_shift, value, n, acc0, acc1, s);
    });
  };
  if (kp.nkeys != 1) { DirectComposite ks; ks.kp = kp; return accumulate(ks); }
  return with_stype(kp.k[0].stype, "internal: key of stype ", [&](auto t) {
    DirectRawKey<typename decltype(t)::type> ks; ks.src.init(kp.k[0]);
    return accumulate(ks);
  });
}

// Sum over spread-out group keys from the first radix pass's digit regions (GroupPlan::region_sum; the layout is in
// dtb_internal.h).  One L2 atomic per row runs at the L2's atomic rate: measured on an H100 80GB HBM3 (700 W,
// scripts/ubench/atomics_bench.cu), 77.5 G float64 atomics/s into an 8 MB table, which is C2's 12.9 ms for 1e9 rows.
// Here a CTA takes a contiguous range of slots, folds every region piece of it into a shared-memory table of
// 2^lbits accumulators (64 KB at 13 bits) and flushes each touched entry with one L2 atomic: (CTAs + regions) x
// 2^lbits atomics in all.  Within a region the rows keep their row order, and the shared-memory add of a u64 or a
// float64 is a CAS loop (ATOMS.CAST.SPIN.64): lanes of a warp that add to one key retry one after another, 32 deep
// in a warp of one key.  So the lanes whose key repeats in the warp -- the left neighbour holds it (sorted or
// clustered input), or it is hot (DIRECT_HOT's map) -- are summed key by key with a warp butterfly first
// (warp_key_sums), and only the other lanes add on their own.
// The fold waits on its shared-memory adds more than on HBM: each row's CAS loop is a chain of a shared load, a
// float add and the CAS, and a warp cannot start the next row's loop before this one ends.  So the kernel runs as
// many warps as the 64 KB tables allow: two 1024-thread CTAs per SM (64 warps, at most 32 registers), two rows per
// thread, and the next two rows' loads issued before the current ones are folded.  On C2 (H100 80GB HBM3, 700 W)
// the sum took 5.11 ms with 256 threads and 8 rows per thread (3 CTAs, 24 warps per SM), 5.02 ms with the loads
// issued one batch ahead, 4.69 ms with 512 threads and 4 rows (48 warps) and 4.03 ms as here.  The hot-key variant
// keeps 256 threads and 8 rows per thread: there the warps' joined sums of a hot key meet on one table entry, and
// 64 warps per SM made the power-law head of scripts/skew_check.py (2e8 rows) take 3.5 ms instead of 2.4 ms.
template <bool HOT> struct RegionCfg {
  static constexpr int THREADS = HOT ? 256 : 1024;
  static constexpr int IPT = HOT ? 8 : 2;        // rows per thread and batch
  static constexpr int CTAS = HOT ? 3 : 2;       // per SM, with a 64 KB table each
};

// The lanes with `join` add their partials to tab[] once per distinct key among them: per key, one butterfly over the
// warp (the other lanes give zero) and one shared-memory add by the key's lowest lane.  Every lane calls it.
template <int CAT>
__device__ __forceinline__ void warp_key_sums(const Partial<CAT>& part, u32 key, bool join, int lane, u64* tab) {
  for (unsigned m = __ballot_sync(0xffffffffu, join); m; m = __ballot_sync(0xffffffffu, join)) {
    const int src = __ffs(m) - 1;
    const u32 kk = __shfl_sync(0xffffffffu, key, src);
    const bool mine = join && key == kk;
    Partial<CAT> t; p_init(t, 0);
    if (mine) t = part;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t.s += __shfl_xor_sync(0xffffffffu, t.s, o);
    if (lane == src) p_flush(t, (int64_t)kk, tab, nullptr, 0);
    join = join && !mine;
  }
}

template <typename T, int CAT, typename KW, bool HOT>
__global__ void __launch_bounds__(RegionCfg<HOT>::THREADS, RegionCfg<HOT>::CTAS)
region_sum_kernel(const KW* __restrict__ lkey, const typename RawKey<T>::load_t* __restrict__ v,
                  const u32* __restrict__ bases, int rbits, int lbits, int64_t n, int64_t per,
                  const uint8_t* __restrict__ hot, u64* acc0)
{
  typedef typename RawKey<T>::load_t L;
  constexpr int REGION_THREADS = RegionCfg<HOT>::THREADS, REGION_IPT = RegionCfg<HOT>::IPT;
  extern __shared__ u64 tab[];                                // 2^lbits accumulators of the current region
  __shared__ u32 rb[256];
  const int tid = threadIdx.x, lane = tid & 31;
  const int nl = 1 << lbits;
  if (tid < 256) rb[tid] = bases[tid];
  const int64_t s_end = ((int64_t)blockIdx.x + 1) * per < n ? ((int64_t)blockIdx.x + 1) * per : n;
  for (int i = tid; i < nl; i += REGION_THREADS) tab[i] = 0;
  __syncthreads();
  for (int64_t s0 = (int64_t)blockIdx.x * per; s0 < s_end;) {
    const u32 d = slot_owner(rb, 0, 255, (u32)s0);
    const int64_t rend = d < 255 ? (int64_t)rb[d + 1] : n;
    const int64_t e = rend < s_end ? rend : s_end;
    // the next batch is loaded before the current one is folded: a warp's loads stay in flight while it adds
    KW kn[REGION_IPT]; L wn[REGION_IPT];
    auto fetch = [&](int64_t b) {
#pragma unroll
      for (int j = 0; j < REGION_IPT; j++) {
        const int64_t i = b + j * REGION_THREADS + tid;
        kn[j] = i < e ? lkey[i] : (KW)0;
        wn[j] = i < e ? v[i] : (L)0;
      }
    };
    fetch(s0);
    for (int64_t i0 = s0; i0 < e; i0 += REGION_THREADS * REGION_IPT) {
      KW k[REGION_IPT]; L w[REGION_IPT];
#pragma unroll
      for (int j = 0; j < REGION_IPT; j++) { k[j] = kn[j]; w[j] = wn[j]; }
      if (i0 + REGION_THREADS * REGION_IPT < e) fetch(i0 + REGION_THREADS * REGION_IPT);
      // lanes that repeat their left neighbour's key (runs) or hold a hot key join the warp's per-key sums; one vote
      // per batch tells whether any lane of the warp joins at all (spread-out keys: none)
      Partial<CAT> part[REGION_IPT];
      u32 jm = 0;                                              // bit j: row j joins
#pragma unroll
      for (int j = 0; j < REGION_IPT; j++) {
        const bool in = i0 + j * REGION_THREADS + tid < e;
        p_init(part[j], 0);
        p_add<T, CAT>(part[j], w[j], in, 0);
        const u32 x = (u32)k[j], up = __shfl_up_sync(0xffffffffu, x, 1);
        bool join = in && lane > 0 && up == x;
        if constexpr (HOT) join = join || (in && hot[(x << rbits) | d]);
        jm |= (u32)join << j;
      }
      if (__any_sync(0xffffffffu, jm != 0)) {
#pragma unroll
        for (int j = 0; j < REGION_IPT; j++)
          if (__any_sync(0xffffffffu, (jm >> j) & 1u)) warp_key_sums(part[j], (u32)k[j], (jm >> j) & 1u, lane, tab);
      }
#pragma unroll
      for (int j = 0; j < REGION_IPT; j++)
        if (!((jm >> j) & 1u)) p_flush(part[j], (int64_t)k[j], tab, nullptr, 0);         // shared-memory atomics
    }
    __syncthreads();
    for (int i = tid; i < nl; i += REGION_THREADS) {
      slot_flush<CAT>(tab[i], 0, ((int64_t)i << rbits) | d, acc0, nullptr, 0);
      tab[i] = 0;
    }
    __syncthreads();
    s0 = e;
  }
}

template <typename T, typename KW, bool HOT>
static void run_region_sum(const void* lkey, int rbits, int lbits, const uint32_t* bases, const void* vperm, int64_t n,
                           const uint8_t* hot, u64* acc0, cudaStream_t s, cudaError_t& err)
{
  constexpr int CAT = std::is_floating_point<T>::value ? CAT_SUMF : CAT_SUMI;
  typedef typename RawKey<T>::load_t L;
  auto kern = region_sum_kernel<T, CAT, KW, HOT>;
  const int smem = (int)sizeof(u64) << lbits;
  err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (err != cudaSuccess) return;
  const int grid = grid_for((n + 65535) / 65536, RegionCfg<HOT>::CTAS);
  const int64_t per = (n + grid - 1) / grid;
  kern<<<grid, RegionCfg<HOT>::THREADS, smem, s>>>((const KW*)lkey, (const L*)vperm, bases, rbits, lbits, n, per, hot, acc0);
  err = cudaGetLastError();
}

int launch_region_sum(const void* lkey, int key_bytes, int rbits, int lbits, const uint32_t* bases, const void* vperm,
                      int stype, int64_t n, const uint8_t* hot, u64* acc0, cudaStream_t s)
{
  if ((key_bytes != 1 && key_bytes != 2) || lbits < 1 || lbits > REGION_MAX_LBITS || lbits > 8 * key_bytes ||
      rbits < 1 || rbits > 8 || rbits + lbits > 22) {
    set_error("internal: bad region sum layout"); return DTB_EINVAL;
  }
  if (n <= 0) return DTB_OK;
  cudaError_t err = cudaSuccess;
  const int rc = with_stype(stype, "internal: region sum of stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    if (key_bytes == 1) { if (hot) run_region_sum<T, uint8_t, true>(lkey, rbits, lbits, bases, vperm, n, hot, acc0, s, err);
                          else     run_region_sum<T, uint8_t, false>(lkey, rbits, lbits, bases, vperm, n, hot, acc0, s, err); }
    else                { if (hot) run_region_sum<T, uint16_t, true>(lkey, rbits, lbits, bases, vperm, n, hot, acc0, s, err);
                          else     run_region_sum<T, uint16_t, false>(lkey, rbits, lbits, bases, vperm, n, hot, acc0, s, err); }
    return DTB_OK;
  });
  DTB_TRY(rc);
  count_launch();
  DTB_CUDA_CHECK(err);
  return DTB_OK;
}

// Stage 2: out[g] = finalize(acc[gkeys[g]]) in the reference's output stype / NA rules; a dense-mapped small table
// holds acc[g] already.
int launch_direct_finalize(int op, int stype, const u64* acc0, const u64* acc1, const DirectPlan& dp,
                           const uint32_t* gkeys, int64_t ng, void* out, const GroupRows& rows, cudaStream_t s)
{
  return finalize(op, stype, acc0, acc1, (dp.kind == DIRECT_SMALL && dp.map) ? nullptr : gkeys, ng, out, rows, s);
}

// ---- reducers fed piecewise: the first valid zero of every group, for float min / max ----------------
__global__ void inverse_order_kernel(const int32_t* __restrict__ order, int64_t n, int32_t* __restrict__ inv) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += stride) inv[order[p]] = (int32_t)p;
}

int launch_inverse_order(const int32_t* order, int64_t n, int32_t* inv, cudaStream_t s) {
  if (n == 0) return DTB_OK;
  const int grid = grid_for((n + 255) / 256, 8);
  inverse_order_kernel<<<grid, 256, 0, s>>>(order, n, inv);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// first_zero[g] = min over the piece's valid zeros of (RowIndex position << 1 | sign bit); g by bisection of offsets
template <typename T>
__global__ void first_zero_rows_kernel(const typename RawKey<T>::load_t* __restrict__ v, int64_t row0, int64_t nrows,
                                       const int32_t* __restrict__ inv, const int32_t* __restrict__ offsets, int64_t ng,
                                       u64* __restrict__ first_zero) {
  constexpr int SIGN_SHIFT = sizeof(typename RawKey<T>::load_t) * 8 - 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += stride) {
    const typename RawKey<T>::load_t r = v[i];
    if ((typename RawKey<T>::load_t)(r << 1) != 0) continue;        // not a zero (NaN never is)
    const int64_t p = inv[row0 + i];
    atomicMin(&first_zero[group_of(offsets, ng, p)], ((u64)p << 1) | (u64)(r >> SIGN_SHIFT));
  }
}

int launch_first_zero_rows(const void* value_rows, int stype, int64_t row0, int64_t nrows, const int32_t* inv,
                           const int32_t* offsets, int64_t ng, u64* first_zero, cudaStream_t s) {
  if (nrows == 0 || ng == 0) return DTB_OK;
  const int grid = grid_for((nrows + 255) / 256, 8);
  if (stype == DTB_STYPE_FLOAT32)
    first_zero_rows_kernel<float><<<grid, 256, 0, s>>>((const u32*)value_rows, row0, nrows, inv, offsets, ng, first_zero);
  else
    first_zero_rows_kernel<double><<<grid, 256, 0, s>>>((const u64*)value_rows, row0, nrows, inv, offsets, ng, first_zero);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// gkeys[g] = sorted_keys[offsets[g]] >> gshift  (the normalised key of every group)
template <typename KeyT>
__global__ void group_keys_kernel(const KeyT* __restrict__ sorted, const int32_t* __restrict__ offsets,
                                  int gshift, int64_t ng, u32* __restrict__ gkeys)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride)
    gkeys[g] = (u32)(sorted[offsets[g]] >> gshift);
}

int launch_group_keys(const void* sorted_keys, int key_bytes, const int32_t* offsets, int gshift,
                      int64_t ng, uint32_t* gkeys, cudaStream_t s)
{
  if (ng == 0) return DTB_OK;
  const int grid = grid_for((ng + 255) / 256, 8);
  if (key_bytes == 4) group_keys_kernel<u32><<<grid, 256, 0, s>>>((const u32*)sorted_keys, offsets, gshift, ng, gkeys);
  else                group_keys_kernel<u64><<<grid, 256, 0, s>>>((const u64*)sorted_keys, offsets, gshift, ng, gkeys);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// RowIndex gather (ArrayView materialisation)
// ===========================================================================
template <typename E, typename OrdT>
__global__ void __launch_bounds__(256)
gather_kernel(const E* __restrict__ src, int64_t nsrc, const OrdT* __restrict__ order, int64_t n,
              E* __restrict__ out, E na)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i0 < n; i0 += stride) {
    int64_t j[4];
#pragma unroll
    for (int k = 0; k < 4; k++) j[k] = (i0 + k < n) ? (int64_t)order[i0 + k] : -1;
    E e[4];
#pragma unroll
    for (int k = 0; k < 4; k++) e[k] = (j[k] >= 0 && j[k] < nsrc) ? src[j[k]] : na;
#pragma unroll
    for (int k = 0; k < 4; k++) if (i0 + k < n) out[i0 + k] = e[k];
  }
}

int launch_gather(const void* src, int stype, int64_t nrows_src, const void* order,
                  int order_is64, int64_t n, void* out, cudaStream_t s)
{
  return with_stype(stype, "Unable to gather Column of stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    typedef bits_t<T> E;
    if (n == 0) return DTB_OK;
    with_order(order, order_is64, [&](auto o) {
      gather_kernel<E><<<grid_for((n + 1023) / 1024, 16), 256, 0, s>>>((const E*)src, nrows_src, o, n, (E*)out,
                                                                       (E)raw_na<T>());
    });
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  });
}

}  // namespace dtb
