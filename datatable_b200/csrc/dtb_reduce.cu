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

enum { CAT_SUMI = 0, CAT_SUMF = 1, CAT_MEAN = 2, CAT_MINMAX = 3, CAT_COUNT = 4 };

constexpr int RT = 256;          // threads per tile
constexpr int RIPT = 8;          // consecutive rows per thread
constexpr int RTILE = RT * RIPT;

template <int CAT> struct Partial;
template <> struct Partial<CAT_SUMI> { u64 s; };
template <> struct Partial<CAT_SUMF> { double s; };
template <> struct Partial<CAT_MEAN> { double s; u32 c; };
template <> struct Partial<CAT_MINMAX> { u64 key; };
template <> struct Partial<CAT_COUNT> { u32 c; };

template <int CAT>
__device__ __forceinline__ void p_init(Partial<CAT>& p, int flag) {
  if constexpr (CAT == CAT_SUMI) p.s = 0;
  else if constexpr (CAT == CAT_SUMF) p.s = 0.0;
  else if constexpr (CAT == CAT_MEAN) { p.s = 0.0; p.c = 0; }
  else if constexpr (CAT == CAT_MINMAX) p.key = flag ? ~0ull : 0ull;   // flag: 1 = MIN
  else p.c = 0;
}

template <int CAT>
__device__ __forceinline__ void p_merge(Partial<CAT>& a, const Partial<CAT>& b, int flag) {
  if constexpr (CAT == CAT_SUMI) a.s += b.s;
  else if constexpr (CAT == CAT_SUMF) a.s += b.s;
  else if constexpr (CAT == CAT_MEAN) { a.s += b.s; a.c += b.c; }
  else if constexpr (CAT == CAT_MINMAX) a.key = flag ? (b.key < a.key ? b.key : a.key) : (b.key > a.key ? b.key : a.key);
  else a.c += b.c;
}

template <int CAT>
__device__ __forceinline__ Partial<CAT> p_shfl_up(const Partial<CAT>& a, int d) {
  Partial<CAT> r;
  if constexpr (CAT == CAT_SUMI) r.s = __shfl_up_sync(0xffffffffu, a.s, d);
  else if constexpr (CAT == CAT_SUMF) r.s = __shfl_up_sync(0xffffffffu, a.s, d);
  else if constexpr (CAT == CAT_MEAN) { r.s = __shfl_up_sync(0xffffffffu, a.s, d); r.c = __shfl_up_sync(0xffffffffu, a.c, d); }
  else if constexpr (CAT == CAT_MINMAX) r.key = __shfl_up_sync(0xffffffffu, a.key, d);
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
  else { if (p.c) atomicAdd(&acc0[g], (u64)p.c); }
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
  else if constexpr (CAT == CAT_MINMAX) {
    u64 key = ISF ? u : (u ^ 0x8000000000000000ull);      // order-preserving unsigned key, never 0 for ints
    if (flag) { if (!ISF) key -= 1; p.key = key < p.key ? key : p.key; }
    else p.key = key > p.key ? key : p.key;
  }
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
  if (tid == 0 || tid == 32) {
    // largest g with offsets[g] <= pos
    const int64_t pos = (tid == 0) ? t0 : (t1 - 1);
    int64_t lo = 0, hi = ng;             // offsets[0] = 0 <= pos < offsets[ng] = n
    while (hi - lo > 1) {
      int64_t mid = (lo + hi) >> 1;
      if ((int64_t)offsets[mid] <= pos) lo = mid; else hi = mid;
    }
    s_g[tid ? 1 : 0] = lo;
  }
  __syncthreads();
  const int64_t g_lo = s_g[0], g_hi = s_g[1];
  for (int64_t g = g_lo + 1 + tid; g <= g_hi; g += RT) {
    const int p = (int)((int64_t)offsets[g] - t0);          // 1 .. RTILE-1
    atomicOr(&s_bits[p >> 5], 1u << (p & 31));
  }
  __syncthreads();
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
      p_flush(part, g_cur, acc0, acc1, flag);
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
  if (key >= 0 && (lane == 31 || nkey != key)) p_flush(part, key, acc0, acc1, flag);
}

// ---- accumulator init / finalize ------------------------------------------------
__global__ void fill_u64_kernel(u64* p, int64_t n, u64 v) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}

void fill_u64(unsigned long long* p, int64_t n, unsigned long long v, cudaStream_t s) {
  if (n <= 0) return;
  const int g = (int)((n + 255) / 256 > NUM_SMS * 8 ? NUM_SMS * 8 : (n + 255) / 256);
  fill_u64_kernel<<<g, 256, 0, s>>>(p, n, v);
  count_launch();
}

__global__ void nrows_kernel(const int32_t* __restrict__ offsets, int64_t ng, int64_t* out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride)
    out[g] = (int64_t)offsets[g + 1] - (int64_t)offsets[g];
}

// NA bit patterns (stype.h:186-197)
__device__ __forceinline__ void store_result(void* out, int out_stype, int64_t g, bool valid, u64 bits) {
  switch (out_stype) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8:
      ((int8_t*)out)[g] = valid ? (int8_t)bits : INT8_MIN; break;
    case DTB_STYPE_INT16: ((int16_t*)out)[g] = valid ? (int16_t)bits : INT16_MIN; break;
    case DTB_STYPE_INT32: case DTB_STYPE_DATE32:
      ((int32_t*)out)[g] = valid ? (int32_t)bits : INT32_MIN; break;
    case DTB_STYPE_INT64: case DTB_STYPE_TIME64:
      ((int64_t*)out)[g] = valid ? (int64_t)bits : INT64_MIN; break;
    case DTB_STYPE_FLOAT32: ((u32*)out)[g] = valid ? (u32)bits : 0x7FC00000u; break;
    case DTB_STYPE_FLOAT64: ((u64*)out)[g] = valid ? bits : 0x7FF8000000000000ull; break;
  }
}

__global__ void finalize_kernel(int op, int in_stype, int out_stype, const u64* __restrict__ acc0,
                                const u64* __restrict__ acc1, int64_t ng, void* out)
{
  const bool in_float = (in_stype == DTB_STYPE_FLOAT32 || in_stype == DTB_STYPE_FLOAT64);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const u64 a = acc0[g];
    bool valid = true; u64 bits = a;
    switch (op) {
      case DTB_OP_SUM:
        if (out_stype == DTB_STYPE_FLOAT32) bits = __float_as_uint((float)__longlong_as_double((long long)a));
        break;                                            // int64 / float64: accumulator bits are the result
      case DTB_OP_MEAN: {
        const u64 c = acc1[g];
        valid = c != 0;
        const double m = __longlong_as_double((long long)a) / (double)c;
        bits = (out_stype == DTB_STYPE_FLOAT32) ? (u64)__float_as_uint((float)m)
                                                : (u64)__double_as_longlong(m);
        break; }
      case DTB_OP_MIN: case DTB_OP_MAX: {
        const bool is_min = (op == DTB_OP_MIN);
        valid = is_min ? (a != ~0ull) : (a != 0ull);
        if (in_float) bits = (in_stype == DTB_STYPE_FLOAT32) ? (u64)f32_unimage((u32)a) : f64_unimage(a);
        else bits = (is_min ? a + 1 : a) ^ 0x8000000000000000ull;
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
  }
  return 0;
}

size_t reduce_extra_bytes(int op, int64_t ng, int64_t n) {
  if (op == DTB_OP_SD) return sizeof(double) * (size_t)(ng > 0 ? ng : 1);
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
  if (order_is64)
    reduce_kernel<T, CAT, int64_t><<<grid, RT, 0, s>>>((const L*)v, nv, (const int64_t*)order, offsets, ng, n, acc0, acc1, flag);
  else
    reduce_kernel<T, CAT, int32_t><<<grid, RT, 0, s>>>((const L*)v, nv, (const int32_t*)order, offsets, ng, n, acc0, acc1, flag);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

template <int CAT>
static int dispatch_T(int st, const void* v, int64_t nv, const void* order, int order_is64,
                      const int32_t* offsets, int64_t ng, int64_t n, u64* acc0, u64* acc1,
                      int flag, cudaStream_t s)
{
  switch (st) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8:
      if constexpr (CAT != CAT_SUMF) return run_reduce<int8_t, CAT>(v, nv, order, order_is64, offsets, ng, n, acc0, acc1, flag, s);
      break;
    case DTB_STYPE_INT16:
      if constexpr (CAT != CAT_SUMF) return run_reduce<int16_t, CAT>(v, nv, order, order_is64, offsets, ng, n, acc0, acc1, flag, s);
      break;
    case DTB_STYPE_INT32:
      if constexpr (CAT != CAT_SUMF) return run_reduce<int32_t, CAT>(v, nv, order, order_is64, offsets, ng, n, acc0, acc1, flag, s);
      break;
    case DTB_STYPE_INT64:
      if constexpr (CAT != CAT_SUMF) return run_reduce<int64_t, CAT>(v, nv, order, order_is64, offsets, ng, n, acc0, acc1, flag, s);
      break;
    case DTB_STYPE_FLOAT32:
      if constexpr (CAT != CAT_SUMI) return run_reduce<float, CAT>(v, nv, order, order_is64, offsets, ng, n, acc0, acc1, flag, s);
      break;
    case DTB_STYPE_FLOAT64:
      if constexpr (CAT != CAT_SUMI) return run_reduce<double, CAT>(v, nv, order, order_is64, offsets, ng, n, acc0, acc1, flag, s);
      break;
  }
  set_error("internal: reducer/stype combination"); return DTB_EINVAL;
}

// acc0/acc1: device scratch of ng u64 each (allocated by the caller in dtb_api.cu)
int launch_reduce_impl(int op, const void* value, int stype, int64_t nv, const void* order, int order_is64,
                       const int32_t* offsets, int64_t ng, int64_t n, u64* acc0, u64* acc1,
                       void* out, cudaStream_t s, void* extra)
{
  const int out_st = reduce_out_stype(op, stype);
  if (!out_st) { set_error("Invalid column type in reducer"); return DTB_EINVAL; }
  if (ng == 0) return DTB_OK;
  const int fgrid = (int)((ng + 255) / 256 > NUM_SMS * 8 ? NUM_SMS * 8 : (ng + 255) / 256);
  if (op >= DTB_OP_FIRST && op <= DTB_OP_NUNIQUE) {
    // within-group ordered reducers (dtb_next.cu): they walk the ARR32 RowIndex
    if (order_is64) { set_error("first/last/sd/median/nunique take an int32 RowIndex"); return DTB_ENOTIMPL; }
    const int32_t* o32 = (const int32_t*)order;
    if (op == DTB_OP_FIRST || op == DTB_OP_LAST) return launch_firstlast(value, stype, nv, o32, offsets, ng, op == DTB_OP_LAST, out, s);
    if (op == DTB_OP_MEDIAN) return launch_median(value, stype, nv, o32, offsets, ng, out, s);
    if (!extra) { set_error("internal: reducer scratch missing"); return DTB_EINVAL; }
    if (op == DTB_OP_SD) {
      fill_u64_kernel<<<fgrid, 256, 0, s>>>(acc0, ng, 0ull);
      fill_u64_kernel<<<fgrid, 256, 0, s>>>(acc1, ng, 0ull);
      fill_u64_kernel<<<fgrid, 256, 0, s>>>((u64*)extra, ng, 0ull);
      count_launch(3);
      if (n > 0) DTB_TRY(dispatch_T<CAT_MEAN>(stype, value, nv, order, 0, offsets, ng, n, acc0, acc1, 0, s));
      return launch_sd(value, stype, nv, o32, offsets, ng, n, acc0, acc1, (double*)extra, out, s);
    }
    // NUNIQUE: flag the rows that start a new distinct value, then count the flags per group
    int8_t* flag = (int8_t*)extra;
    DTB_TRY(launch_distinct_flags(value, stype, nv, o32, offsets, ng, n, flag, s));
    fill_u64_kernel<<<fgrid, 256, 0, s>>>(acc0, ng, 0ull);
    count_launch();
    if (n > 0) DTB_TRY(dispatch_T<CAT_COUNT>(DTB_STYPE_INT8, flag, n, nullptr, 0, offsets, ng, n, acc0, acc1, 0, s));
    finalize_kernel<<<fgrid, 256, 0, s>>>(DTB_OP_COUNT, DTB_STYPE_INT8, DTB_STYPE_INT64, acc0, acc1, ng, out);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  }
  if (op == DTB_OP_NROWS) {
    nrows_kernel<<<fgrid, 256, 0, s>>>(offsets, ng, (int64_t*)out);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  }
  const bool isflt = (stype == DTB_STYPE_FLOAT32 || stype == DTB_STYPE_FLOAT64);
  u64 init0 = (op == DTB_OP_MIN) ? ~0ull : 0ull;          // 0.0 == 0 bits for float sums
  fill_u64_kernel<<<fgrid, 256, 0, s>>>(acc0, ng, init0);
  count_launch();
  if (op == DTB_OP_MEAN) { fill_u64_kernel<<<fgrid, 256, 0, s>>>(acc1, ng, 0ull); count_launch(); }
  DTB_CUDA_CHECK(cudaGetLastError());
  if (n > 0) {
    int rc = DTB_OK;
    switch (op) {
      case DTB_OP_SUM:
        rc = isflt ? dispatch_T<CAT_SUMF>(stype, value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 0, s)
                   : dispatch_T<CAT_SUMI>(stype, value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 0, s);
        break;
      case DTB_OP_MEAN: rc = dispatch_T<CAT_MEAN>(stype, value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 0, s); break;
      case DTB_OP_MIN:  rc = dispatch_T<CAT_MINMAX>(stype, value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 1, s); break;
      case DTB_OP_MAX:  rc = dispatch_T<CAT_MINMAX>(stype, value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 0, s); break;
      case DTB_OP_COUNT:   rc = dispatch_T<CAT_COUNT>(stype, value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 0, s); break;
      case DTB_OP_COUNTNA: rc = dispatch_T<CAT_COUNT>(stype, value, nv, order, order_is64, offsets, ng, n, acc0, acc1, 1, s); break;
      default: set_error("unknown reducer"); return DTB_EINVAL;
    }
    if (rc != DTB_OK) return rc;
  }
  finalize_kernel<<<fgrid, 256, 0, s>>>(op, stype, out_st, acc0, acc1, ng, out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int reduce_out_stype_host(int op, int st) { return reduce_out_stype(op, st); }

// Groupby invariants (groupby.h:41-47): offsets[0] = 0 and strictly increasing.  reduce_kernel marks
// group starts in a one-bit-per-row bitmap, so an empty group would silently shift every later group of
// the tile: caller-supplied offsets are checked first.  *bad receives the index of a violating group + 1.
__global__ void offsets_check_kernel(const int32_t* __restrict__ offsets, int64_t ng, int* bad) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    if (offsets[g] >= offsets[g + 1] || (g == 0 && offsets[0] != 0)) atomicMax(bad, (int)(g < INT32_MAX ? g + 1 : INT32_MAX));
  }
}

int launch_offsets_check(const int32_t* offsets, int64_t ng, int* d_bad, cudaStream_t s) {
  if (ng == 0) return DTB_OK;
  const int fgrid = (int)((ng + 255) / 256 > NUM_SMS * 8 ? NUM_SMS * 8 : (ng + 255) / 256);
  offsets_check_kernel<<<fgrid, 256, 0, s>>>(offsets, ng, d_bad);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int launch_nrows(const int32_t* offsets, int64_t ng, void* out, cudaStream_t s) {
  if (ng == 0) return DTB_OK;
  const int fgrid = (int)((ng + 255) / 256 > NUM_SMS * 8 ? NUM_SMS * 8 : (ng + 255) / 256);
  nrows_kernel<<<fgrid, 256, 0, s>>>(offsets, ng, (int64_t*)out);
  count_launch();
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
// 50 MB L2 of an H100.  Rows of a warp that share x are combined first
// (__match_any_sync) so that hot keys do not serialise on one address.  A finalize kernel
// maps group g -> acc[gkeys[g]] and applies the reference's output stype / NA rules.
//
// Bound: L2 atomic throughput, then HBM.
// Algorithmic bytes per row: key column(s) + value column, read once.
struct HotSpec {            // "may one key own a large share of the rows?"
  const u32* count;         // device: largest digit count of the first pass (NULL = use `value`)
  u32 thresh;
  int value;
};

template <typename T, int CAT, typename KSrc>
__global__ void __launch_bounds__(512)
direct_reduce_kernel(KSrc ksrc, int gshift, const typename RawKey<T>::load_t* __restrict__ v,
                     int64_t n, u64* acc0, u64* acc1, int flag, HotSpec hs)
{
  const bool HOT = hs.count ? (*hs.count > hs.thresh) : (hs.value != 0);      // warp-uniform
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t nround = ((n + 31) / 32) * 32;                // keep whole warps in the loop
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nround; i += stride) {
    const bool in = i < n;
    u32 x = 0xffffffffu;
    Partial<CAT> part; p_init(part, flag);
    if (in) {
      x = (u32)(ksrc.load(i) >> gshift);
      p_add<T, CAT>(part, v[i], true, flag);
    }
    // HOT: a key may own a large share of the rows (skewed digit histograms): fold equal keys of the
    // warp before touching L2.  MATCH.ANY is a slow, multi-cycle warp instruction, so the
    // common spread-out case skips it entirely.
    const unsigned peers = HOT ? __match_any_sync(0xffffffffu, x) : (1u << lane);
    if (HOT && __any_sync(0xffffffffu, peers != (1u << lane))) {  // warp-uniform: the body shuffles
      // rare for spread-out keys: fold the partials of equal keys into the lowest lane
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
      if (lane == leader) part = tot; else p_init(part, flag);
    }
    if (in) p_flush(part, (int64_t)x, acc0, acc1, flag);
  }
}

__global__ void finalize_direct_kernel(int op, int in_stype, int out_stype, const u64* __restrict__ acc0,
                                       const u64* __restrict__ acc1, const u32* __restrict__ gkeys,
                                       int64_t ng, void* out)
{
  const bool in_float = (in_stype == DTB_STYPE_FLOAT32 || in_stype == DTB_STYPE_FLOAT64);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const u32 x = gkeys ? gkeys[g] : (u32)g;          // NULL: the accumulators are indexed by group
    const u64 a = acc0[x];
    bool valid = true; u64 bits = a;
    switch (op) {
      case DTB_OP_SUM:
        if (out_stype == DTB_STYPE_FLOAT32) bits = __float_as_uint((float)__longlong_as_double((long long)a));
        break;
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
        break; }
      default: break;
    }
    store_result(out, out_stype, g, valid, bits);
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
// (100 keys at 2e8 rows = 1.6e8 same-address L2 atomics; low-cardinality by() is the common case).
constexpr int SMALL_TABLE = 2048;

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

static thread_local DirectPlan t_dp = {DIRECT_PLAIN, nullptr, 0, nullptr, 0};

template <typename T, int CAT, typename KSrc>
static int run_direct(const KSrc& ks, int gshift, const void* v, int64_t n, u64* acc0, u64* acc1, int flag,
                      cudaStream_t s)
{
  typedef typename RawKey<T>::load_t L;
  int64_t want = (n + 511) / 512;
  if (t_dp.kind == DIRECT_SMALL) {
    int grid = (int)(want > NUM_SMS * 4 ? NUM_SMS * 4 : want);
    direct_reduce_small_kernel<T, CAT, KSrc><<<grid, 512, 0, s>>>(ks, gshift, (const L*)v, n, (int)t_dp.nslots,
                                                                  (const uint16_t*)t_dp.map, acc0, acc1, flag);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  }
  if (t_dp.kind == DIRECT_HOT) {
    int grid = (int)(want > NUM_SMS * 4 ? NUM_SMS * 4 : want);
    direct_reduce_hot_kernel<T, CAT, KSrc><<<grid, 512, 0, s>>>(ks, gshift, (const L*)v, n, (const uint8_t*)t_dp.map,
                                                                acc0, acc1, flag);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  }
  HotSpec hs = {nullptr, 0, 0};
  if (t_dp.kind == DIRECT_DEVICE_HOT) { hs.count = t_dp.hot_count; hs.thresh = t_dp.hot_thresh; }
  int grid = (int)(want > NUM_SMS * 16 ? NUM_SMS * 16 : want);
  direct_reduce_kernel<T, CAT, KSrc><<<grid, 512, 0, s>>>(ks, gshift, (const L*)v, n, acc0, acc1, flag, hs);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

template <int CAT, typename KSrc>
static int direct_T(int st, const KSrc& ks, int gshift, const void* v, int64_t n, u64* acc0, u64* acc1,
                    int flag, cudaStream_t s)
{
  switch (st) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8:
      if constexpr (CAT != CAT_SUMF) return run_direct<int8_t, CAT>(ks, gshift, v, n, acc0, acc1, flag, s); break;
    case DTB_STYPE_INT16:
      if constexpr (CAT != CAT_SUMF) return run_direct<int16_t, CAT>(ks, gshift, v, n, acc0, acc1, flag, s); break;
    case DTB_STYPE_INT32:
      if constexpr (CAT != CAT_SUMF) return run_direct<int32_t, CAT>(ks, gshift, v, n, acc0, acc1, flag, s); break;
    case DTB_STYPE_INT64:
      if constexpr (CAT != CAT_SUMF) return run_direct<int64_t, CAT>(ks, gshift, v, n, acc0, acc1, flag, s); break;
    case DTB_STYPE_FLOAT32:
      if constexpr (CAT != CAT_SUMI) return run_direct<float, CAT>(ks, gshift, v, n, acc0, acc1, flag, s); break;
    case DTB_STYPE_FLOAT64:
      if constexpr (CAT != CAT_SUMI) return run_direct<double, CAT>(ks, gshift, v, n, acc0, acc1, flag, s); break;
  }
  set_error("internal: reducer/stype combination"); return DTB_EINVAL;
}

template <typename KSrc>
static int direct_op(int op, int st, const KSrc& ks, int gshift, const void* v, int64_t n, u64* acc0,
                     u64* acc1, cudaStream_t s)
{
  const bool isflt = (st == DTB_STYPE_FLOAT32 || st == DTB_STYPE_FLOAT64);
  switch (op) {
    case DTB_OP_SUM:
      return isflt ? direct_T<CAT_SUMF>(st, ks, gshift, v, n, acc0, acc1, 0, s)
                   : direct_T<CAT_SUMI>(st, ks, gshift, v, n, acc0, acc1, 0, s);
    case DTB_OP_MEAN:    return direct_T<CAT_MEAN>(st, ks, gshift, v, n, acc0, acc1, 0, s);
    case DTB_OP_MIN:     return direct_T<CAT_MINMAX>(st, ks, gshift, v, n, acc0, acc1, 1, s);
    case DTB_OP_MAX:     return direct_T<CAT_MINMAX>(st, ks, gshift, v, n, acc0, acc1, 0, s);
    case DTB_OP_COUNT:   return direct_T<CAT_COUNT>(st, ks, gshift, v, n, acc0, acc1, 0, s);
    case DTB_OP_COUNTNA: return direct_T<CAT_COUNT>(st, ks, gshift, v, n, acc0, acc1, 1, s);
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
  dp.kind = DIRECT_PLAIN; dp.map = nullptr; dp.nslots = table; dp.hot_count = nullptr; dp.hot_thresh = 0;
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
    const int grid = (int)((ng + 255) / 256 > NUM_SMS * 8 ? NUM_SMS * 8 : (ng + 255) / 256);
    hot_map_kernel<<<grid, 256, 0, s>>>(gkeys, offsets, ng, (u32)key_thresh, (uint8_t*)map_scratch);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    dp.kind = DIRECT_HOT; dp.map = map_scratch;
  }
  return DTB_OK;
}

// Stage 1: stream every row into acc[x] (acc[group] for a dense-mapped small table).  acc0/acc1: device
// scratch of `table` u64 each.  DIRECT_DEVICE_HOT (reducers overlapped with the sort, before the groups
// exist): dp.hot_count is the largest digit count of the first radix pass; more than dp.hot_thresh rows
// in one bin switches on the intra-warp pre-aggregation, decided on the device.
int launch_direct_accumulate(int op, const KeyPlan& kp, const DirectPlan& dp,
                             const void* value, int stype, int64_t n, int64_t table,
                             u64* acc0, u64* acc1, cudaStream_t s)
{
  DTB_TRY(launch_direct_init(op, dp, table, acc0, acc1, s));
  return launch_direct_accumulate_rows(op, kp, dp, value, stype, n, table, acc0, acc1, s);
}

// the accumulator tables' identities (once per reducer; the rows may then arrive in pieces)
int launch_direct_init(int op, const DirectPlan& dp, int64_t table, u64* acc0, u64* acc1, cudaStream_t s)
{
  if (dp.kind == DIRECT_SMALL) table = dp.nslots;                // only the used accumulators are initialised
  const int tgrid = (int)((table + 255) / 256 > NUM_SMS * 8 ? NUM_SMS * 8 : (table + 255) / 256);
  fill_u64_kernel<<<tgrid, 256, 0, s>>>(acc0, table, (op == DTB_OP_MIN) ? ~0ull : 0ull);
  count_launch();
  if (op == DTB_OP_MEAN) { fill_u64_kernel<<<tgrid, 256, 0, s>>>(acc1, table, 0ull); count_launch(); }
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// folds n rows (kp's key columns and `value`, both starting at the piece's first row) into the tables
int launch_direct_accumulate_rows(int op, const KeyPlan& kp, const DirectPlan& dp,
                                  const void* value, int stype, int64_t n, int64_t table,
                                  u64* acc0, u64* acc1, cudaStream_t s)
{
  const int out_st = reduce_out_stype(op, stype);
  if (!out_st) { set_error("Invalid column type in reducer"); return DTB_EINVAL; }
  t_dp = dp;
  (void)table;
  if (n > 0) {
    int rc;
    if (kp.nkeys == 1) {
      const KeyNorm& k = kp.k[0];
#define DTB_CASE(TK) { DirectRawKey<TK> ks; ks.src.init(k); \
                       rc = direct_op(op, stype, ks, kp.group_shift, value, n, acc0, acc1, s); break; }
      switch (k.stype) {
        case DTB_STYPE_BOOL: case DTB_STYPE_INT8:    DTB_CASE(int8_t)
        case DTB_STYPE_INT16:                        DTB_CASE(int16_t)
        case DTB_STYPE_INT32: case DTB_STYPE_DATE32: DTB_CASE(int32_t)
        case DTB_STYPE_INT64: case DTB_STYPE_TIME64: DTB_CASE(int64_t)
        case DTB_STYPE_FLOAT32:                      DTB_CASE(float)
        case DTB_STYPE_FLOAT64:                      DTB_CASE(double)
        default: set_error("internal: bad key stype"); return DTB_EINVAL;
      }
#undef DTB_CASE
    } else {
      DirectComposite ks; ks.kp = kp;
      rc = direct_op(op, stype, ks, kp.group_shift, value, n, acc0, acc1, s);
    }
    if (rc != DTB_OK) return rc;
  }
  return DTB_OK;
}

// Stage 2: out[g] = finalize(acc[gkeys[g]]) in the reference's output stype / NA rules.
int launch_direct_finalize(int op, int stype, const u64* acc0, const u64* acc1, const uint32_t* gkeys,
                           int64_t ng, void* out, cudaStream_t s)
{
  const int out_st = reduce_out_stype(op, stype);
  if (!out_st) { set_error("Invalid column type in reducer"); return DTB_EINVAL; }
  if (ng == 0) return DTB_OK;
  const int fgrid = (int)((ng + 255) / 256 > NUM_SMS * 8 ? NUM_SMS * 8 : (ng + 255) / 256);
  finalize_direct_kernel<<<fgrid, 256, 0, s>>>(op, stype, out_st, acc0, acc1, gkeys, ng, out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int launch_reduce_direct(int op, const KeyPlan& kp, const DirectPlan& dp, const void* value, int stype, int64_t n,
                         int64_t table, const uint32_t* gkeys, int64_t ng, u64* acc0, u64* acc1,
                         void* out, cudaStream_t s)
{
  if (ng == 0) return DTB_OK;
  DTB_TRY(launch_direct_accumulate(op, kp, dp, value, stype, n, table, acc0, acc1, s));
  return launch_direct_finalize(op, stype, acc0, acc1, (dp.kind == DIRECT_SMALL && dp.map) ? nullptr : gkeys,
                                ng, out, s);
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
  const int grid = (int)((ng + 255) / 256 > NUM_SMS * 8 ? NUM_SMS * 8 : (ng + 255) / 256);
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

template <typename E>
static int run_gather(const void* src, int64_t nsrc, const void* order, int order_is64, int64_t n,
                      void* out, E na, cudaStream_t s)
{
  if (n == 0) return DTB_OK;
  int64_t want = (n + 1023) / 1024;
  int grid = (int)(want > NUM_SMS * 16 ? NUM_SMS * 16 : want);
  if (order_is64) gather_kernel<E, int64_t><<<grid, 256, 0, s>>>((const E*)src, nsrc, (const int64_t*)order, n, (E*)out, na);
  else            gather_kernel<E, int32_t><<<grid, 256, 0, s>>>((const E*)src, nsrc, (const int32_t*)order, n, (E*)out, na);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int launch_gather(const void* src, int stype, int64_t nrows_src, const void* order,
                  int order_is64, int64_t n, void* out, cudaStream_t s)
{
  switch (stype) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8:
      return run_gather<uint8_t>(src, nrows_src, order, order_is64, n, out, (uint8_t)0x80, s);
    case DTB_STYPE_INT16:
      return run_gather<uint16_t>(src, nrows_src, order, order_is64, n, out, (uint16_t)0x8000, s);
    case DTB_STYPE_INT32: case DTB_STYPE_DATE32:
      return run_gather<u32>(src, nrows_src, order, order_is64, n, out, 0x80000000u, s);
    case DTB_STYPE_FLOAT32:
      return run_gather<u32>(src, nrows_src, order, order_is64, n, out, 0x7FC00000u, s);
    case DTB_STYPE_INT64: case DTB_STYPE_TIME64:
      return run_gather<u64>(src, nrows_src, order, order_is64, n, out, 0x8000000000000000ull, s);
    case DTB_STYPE_FLOAT64:
      return run_gather<u64>(src, nrows_src, order, order_is64, n, out, 0x7FF8000000000000ull, s);
  }
  set_error("Unable to gather Column of stype " + std::to_string(stype));
  return DTB_ENOTIMPL;
}

}  // namespace dtb
