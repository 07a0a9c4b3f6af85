// dtb_next.cu -- the callers either side of the hot path (SURVEY.md 8f): within-group ordered
// reducers, set operations, mode, keyed join.  All of them are consumers of group()'s
// RowIndex / Groupby pair; the kernels here are the per-group / per-row selection steps that the
// reference runs as serial host loops over `indices[goffsets[i]]`.
//
//   first / last          expr/head_reduce_unary.cc:120-190   value of the first / last row of a group
//   sd                    expr/head_reduce_unary.cc:197-245   sample standard deviation (Welford there;
//                                                             here: mean, then sum of squared deviations)
//   median                expr/head_reduce_unary.cc:421-468   over rows sorted inside their group
//                                                             (Column::sort_grouped, sort.cc:1499-1530)
//   nunique               expr/head_reduce_unary.cc:383-415   distinct valid values per group
//   union / intersect / setdiff / symdiff   set_funcs.cc:126-456
//   mode / nmodal         stats.cc:955-1003
//   natural join          frame/join.cc:392-470               binary search of every X row in the sorted keys of J
//
// Bound: none of these is a bandwidth kernel except the row-parallel ones (group ids, distinct
// flags, join), which are random-gather bound like reduce_kernel.
#include <type_traits>
#include "dtb_common.cuh"

namespace dtb {

static inline int grid_for(int64_t n, int threads = 256) {
  const int64_t want = (n + threads - 1) / threads;
  return (int)(want > NUM_SMS * 16 ? NUM_SMS * 16 : (want < 1 ? 1 : want));
}

// raw element -> (valid, double) / (valid, order-preserving u64 image) ------------------------
template <typename T> __device__ __forceinline__ bool elem_valid(const void* v, int64_t i) {
  typedef typename RawKey<T>::load_t L;
  u64 u; return RawKey<T>::get(((const L*)v)[i], u);
}
template <typename T> __device__ __forceinline__ double elem_double(const void* v, int64_t i) {
  if constexpr (std::is_same<T, float>::value) return (double)((const float*)v)[i];
  else if constexpr (std::is_same<T, double>::value) return ((const double*)v)[i];
  else return (double)((const T*)v)[i];
}

#define DTB_DISPATCH_STYPE(st, CALL)                                   \
  switch (st) {                                                        \
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8:    { CALL(int8_t);  break; }   \
    case DTB_STYPE_INT16:                        { CALL(int16_t); break; }   \
    case DTB_STYPE_INT32: case DTB_STYPE_DATE32: { CALL(int32_t); break; }   \
    case DTB_STYPE_INT64: case DTB_STYPE_TIME64: { CALL(int64_t); break; }   \
    case DTB_STYPE_FLOAT32:                      { CALL(float);   break; }   \
    case DTB_STYPE_FLOAT64:                      { CALL(double);  break; }   \
    default: set_error("unsupported stype"); return DTB_ENOTIMPL;      \
  }

// ===========================================================================
// first / last: out[g] = v[order[offsets[g]]] or v[order[offsets[g+1]-1]] (NA stays NA)
// ===========================================================================
template <typename E>
__global__ void firstlast_kernel(const E* __restrict__ v, int64_t nv, const int32_t* __restrict__ order,
                                 const int32_t* __restrict__ offsets, int64_t ng, int last, E na, E* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const int64_t p = last ? (int64_t)offsets[g + 1] - 1 : (int64_t)offsets[g];
    const int64_t j = order ? (int64_t)order[p] : p;
    out[g] = (j >= 0 && j < nv) ? v[j] : na;
  }
}

int launch_firstlast(const void* v, int stype, int64_t nv, const int32_t* order, const int32_t* offsets,
                     int64_t ng, int last, void* out, cudaStream_t s)
{
  if (ng == 0) return DTB_OK;
  const int grid = grid_for(ng);
  switch (stype_bytes(stype)) {
    case 1: firstlast_kernel<uint8_t><<<grid, 256, 0, s>>>((const uint8_t*)v, nv, order, offsets, ng, last, (uint8_t)0x80, (uint8_t*)out); break;
    case 2: firstlast_kernel<uint16_t><<<grid, 256, 0, s>>>((const uint16_t*)v, nv, order, offsets, ng, last, (uint16_t)0x8000, (uint16_t*)out); break;
    case 4: firstlast_kernel<u32><<<grid, 256, 0, s>>>((const u32*)v, nv, order, offsets, ng, last,
                                                       stype == DTB_STYPE_FLOAT32 ? 0x7FC00000u : 0x80000000u, (u32*)out); break;
    case 8: firstlast_kernel<u64><<<grid, 256, 0, s>>>((const u64*)v, nv, order, offsets, ng, last,
                                                       stype == DTB_STYPE_FLOAT64 ? 0x7FF8000000000000ull : 0x8000000000000000ull, (u64*)out); break;
    default: set_error("unsupported stype"); return DTB_ENOTIMPL;
  }
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// group id of every sorted position: gid[p] = g for offsets[g] <= p < offsets[g+1]
// (each thread owns 8 consecutive positions: one binary search, then a walk)
// ===========================================================================
__global__ void expand_gid_kernel(const int32_t* __restrict__ offsets, int64_t ng, int64_t n, int32_t* __restrict__ gid)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 8;
  for (int64_t p0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; p0 < n; p0 += stride) {
    int64_t lo = 0, hi = ng;                       // largest g with offsets[g] <= p0
    while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if ((int64_t)offsets[mid] <= p0) lo = mid; else hi = mid; }
    int64_t g = lo, next = offsets[g + 1];
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int64_t p = p0 + i;
      if (p >= n) break;
      while (p >= next) { g++; next = offsets[g + 1]; }
      gid[p] = (int32_t)g;
    }
  }
}

int launch_expand_gid(const int32_t* offsets, int64_t ng, int64_t n, int32_t* gid, cudaStream_t s) {
  if (n == 0) return DTB_OK;
  expand_gid_kernel<<<grid_for((n + 7) / 8), 256, 0, s>>>(offsets, ng, n, gid);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// sd, pass 2: acc[g] += (x - mean[g])^2 over the valid rows.  The mean comes from the MEAN accumulators
// (sum, count); squared deviations from the group's own mean do not cancel the way sum(x^2) - n mean^2
// does, so the result agrees with the reference's Welford recurrence to ~1e-15 relative.
// ===========================================================================
template <typename T>
__global__ void sqdev_kernel(const void* __restrict__ v, int64_t nv, const int32_t* __restrict__ order,
                             const int32_t* __restrict__ offsets, int64_t ng, int64_t n,
                             const u64* __restrict__ sum, const u64* __restrict__ cnt, double* __restrict__ acc)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 8;
  for (int64_t p0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; p0 < n; p0 += stride) {
    int64_t lo = 0, hi = ng;
    while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if ((int64_t)offsets[mid] <= p0) lo = mid; else hi = mid; }
    int64_t g = lo, next = offsets[g + 1];
    double mean = __longlong_as_double((long long)sum[g]) / (double)cnt[g];
    double part = 0.0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int64_t p = p0 + i;
      if (p >= n) break;
      if (p >= next) {
        if (part != 0.0) atomicAdd(&acc[g], part);
        part = 0.0;
        while (p >= next) { g++; next = offsets[g + 1]; }
        mean = __longlong_as_double((long long)sum[g]) / (double)cnt[g];
      }
      const int64_t j = order ? (int64_t)order[p] : p;
      if (j >= 0 && j < nv && elem_valid<T>(v, j)) { const double d = elem_double<T>(v, j) - mean; part += d * d; }
    }
    if (part != 0.0) atomicAdd(&acc[g], part);
  }
}

__global__ void sd_finalize_kernel(const double* __restrict__ m2, const u64* __restrict__ cnt, int64_t ng, int out_f32, void* out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const u64 c = cnt[g];
    const double q = m2[g];
    const bool valid = c > 1 && !isnan(q);                     // head_reduce_unary.cc:213
    const double sd = q >= 0 ? sqrt(q / (double)(c - 1)) : 0.0;
    if (out_f32) ((u32*)out)[g] = valid ? __float_as_uint((float)sd) : 0x7FC00000u;
    else         ((u64*)out)[g] = valid ? (u64)__double_as_longlong(sd) : 0x7FF8000000000000ull;
  }
}

int launch_sd(const void* v, int stype, int64_t nv, const int32_t* order, const int32_t* offsets, int64_t ng, int64_t n,
              const u64* sum, const u64* cnt, double* m2 /*zeroed*/, void* out, cudaStream_t s)
{
  if (ng == 0) return DTB_OK;
  if (n > 0) {
    const int grid = grid_for((n + 7) / 8);
#define CALL(T) sqdev_kernel<T><<<grid, 256, 0, s>>>(v, nv, order, offsets, ng, n, sum, cnt, m2)
    DTB_DISPATCH_STYPE(stype, CALL)
#undef CALL
    count_launch();
  }
  sd_finalize_kernel<<<grid_for(ng), 256, 0, s>>>(m2, cnt, ng, stype == DTB_STYPE_FLOAT32, out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// median over rows already sorted inside their group (NA first): one thread per group
// ===========================================================================
template <typename T>
__global__ void median_kernel(const void* __restrict__ v, int64_t nv, const int32_t* __restrict__ order,
                              const int32_t* __restrict__ offsets, int64_t ng, void* out)
{
  constexpr bool F32 = std::is_same<T, float>::value;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    int64_t i0 = offsets[g], i1 = offsets[g + 1];
    // skip the NA rows at the front of the group (they sort first): first valid position by bisection
    int64_t lo = i0, hi = i1;                     // invariant: rows < lo are NA, rows >= hi are valid
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      const int64_t j = order ? (int64_t)order[mid] : mid;
      if (j >= 0 && j < nv && elem_valid<T>(v, j)) hi = mid; else lo = mid + 1;
    }
    i0 = lo;
    bool valid = i0 < i1;
    double m = 0.0;
    if (valid) {
      const int64_t jm = (i0 + i1) / 2;                          // head_reduce_unary.cc:456-463
      const int64_t r1 = order ? (int64_t)order[jm] : jm;
      if ((i1 - i0) & 1) {
        m = F32 ? (double)(float)elem_double<T>(v, r1) : elem_double<T>(v, r1);
      } else {
        const int64_t r2 = order ? (int64_t)order[jm - 1] : jm - 1;
        if (F32) m = (double)(((float)elem_double<T>(v, r1) + (float)elem_double<T>(v, r2)) / 2.0f);
        else m = (elem_double<T>(v, r1) + elem_double<T>(v, r2)) / 2;
      }
    }
    if (F32) ((u32*)out)[g] = valid ? __float_as_uint((float)m) : 0x7FC00000u;
    else     ((u64*)out)[g] = valid ? (u64)__double_as_longlong(m) : 0x7FF8000000000000ull;
  }
}

int launch_median(const void* v, int stype, int64_t nv, const int32_t* order, const int32_t* offsets,
                  int64_t ng, void* out, cudaStream_t s)
{
  if (ng == 0) return DTB_OK;
  const int grid = grid_for(ng);
#define CALL(T) median_kernel<T><<<grid, 256, 0, s>>>(v, nv, order, offsets, ng, out)
  DTB_DISPATCH_STYPE(stype, CALL)
#undef CALL
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// nunique over rows sorted inside their group: flag[p] = 1 where a valid value differs from the row
// before it (std::set<T> semantics, head_reduce_unary.cc:383-394: -0.0 and +0.0 are one value);
// group starts are corrected by a per-group kernel; the flags are then counted per group.
// ===========================================================================
template <typename T>
__device__ __forceinline__ bool same_value(const void* v, int64_t a, int64_t b) {
  if constexpr (std::is_floating_point<T>::value) return elem_double<T>(v, a) == elem_double<T>(v, b);
  else return ((const T*)v)[a] == ((const T*)v)[b];
}

template <typename T>
__global__ void distinct_flags_kernel(const void* __restrict__ v, int64_t nv, const int32_t* __restrict__ order,
                                      int64_t n, int8_t* __restrict__ flag)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += stride) {
    const int64_t j = order ? (int64_t)order[p] : p;
    bool isnew = false;
    if (j >= 0 && j < nv && elem_valid<T>(v, j)) {
      isnew = true;
      if (p > 0) {
        const int64_t q = order ? (int64_t)order[p - 1] : p - 1;
        if (q >= 0 && q < nv && elem_valid<T>(v, q) && same_value<T>(v, j, q)) isnew = false;
      }
    }
    flag[p] = isnew ? 1 : INT8_MIN;               // int8 column: 1 = counted, NA = not counted
  }
}

template <typename T>
__global__ void distinct_starts_kernel(const void* __restrict__ v, int64_t nv, const int32_t* __restrict__ order,
                                       const int32_t* __restrict__ offsets, int64_t ng, int8_t* __restrict__ flag)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const int64_t p = offsets[g];
    if (p >= offsets[g + 1]) continue;
    const int64_t j = order ? (int64_t)order[p] : p;
    if (j >= 0 && j < nv && elem_valid<T>(v, j)) flag[p] = 1;   // the first valid row of a group always counts
  }
}

int launch_distinct_flags(const void* v, int stype, int64_t nv, const int32_t* order, const int32_t* offsets,
                          int64_t ng, int64_t n, int8_t* flag, cudaStream_t s)
{
  if (n == 0) return DTB_OK;
#define CALL(T) { distinct_flags_kernel<T><<<grid_for(n), 256, 0, s>>>(v, nv, order, n, flag); \
                  distinct_starts_kernel<T><<<grid_for(ng), 256, 0, s>>>(v, nv, order, offsets, ng, flag); }
  DTB_DISPATCH_STYPE(stype, CALL)
#undef CALL
  count_launch(2);
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// Set operations (set_funcs.cc): the K input columns were concatenated (column k holds the rows
// sizes[k-1] .. sizes[k]-1) and grouped; a group is kept depending on which inputs its rows come from.
// Inside a group the RowIndex ascends, so the rows of input k are contiguous.
// flags[1 + g] = keep group g (flags[0] is a sentinel for the compaction by group_offsets_kernel)
// ===========================================================================
__global__ void set_select_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ offsets, int64_t ng,
                                  const int64_t* __restrict__ sizes, int K, int mode, uint8_t* __restrict__ flags)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const int64_t i0 = offsets[g], i1 = offsets[g + 1];
    bool keep = true;
    if (mode != DTB_SET_UNION && K >= 2) {
      const int64_t n1 = sizes[0];
      const int64_t x = order[i0], y = order[i1 - 1];
      if (mode == DTB_SET_SETDIFF) keep = x < n1 && y < n1;                        // set_funcs.cc:342-349
      else if (K == 2) keep = (mode == DTB_SET_INTERSECT) ? (x < n1 && y >= n1)     // :264-272
                                                          : ((x < n1) == (y < n1)); // :401-407
      else {
        // number of inputs with a row in the group: jump from input to input by bisection
        int present = 0;
        int64_t ii = i0;
        for (int k = 0; k < K && ii < i1; k++) {
          const int64_t nk = sizes[k];
          if ((int64_t)order[ii] >= nk) continue;
          present++;
          int64_t lo = ii, hi = i1;                // first position whose row index is >= nk
          while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if ((int64_t)order[mid] < nk) lo = mid + 1; else hi = mid; }
          ii = lo;
        }
        keep = (mode == DTB_SET_INTERSECT) ? (present == K) : ((present & 1) != 0);  // :277-296, :413-427
      }
    }
    flags[1 + g] = keep ? 1 : 0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) flags[0] = 1;
}

__global__ void set_emit_kernel(const int32_t* __restrict__ pos, int64_t nsel, const int32_t* __restrict__ order,
                                const int32_t* __restrict__ offsets, int32_t* __restrict__ out_rows)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nsel; i += stride)
    out_rows[i] = order[offsets[pos[i + 1] - 1]];        // pos[0] is the sentinel; group = position - 1
}

int launch_set_select(const int32_t* order, const int32_t* offsets, int64_t ng, const int64_t* d_sizes, int K,
                      int mode, uint8_t* flags, cudaStream_t s)
{
  set_select_kernel<<<grid_for(ng), 256, 0, s>>>(order, offsets, ng, d_sizes, K, mode, flags);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int launch_set_emit(const int32_t* pos, int64_t nsel, const int32_t* order, const int32_t* offsets, int32_t* out_rows,
                    cudaStream_t s)
{
  if (nsel == 0) return DTB_OK;
  set_emit_kernel<<<grid_for(nsel), 256, 0, s>>>(pos, nsel, order, offsets, out_rows);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// mode: the first largest group among groups [skip, ng)  (stats.cc:984-991)
// result[0] = (size << 32) | (0xffffffff - index)  maximised  ->  largest size, smallest index
// ===========================================================================
__global__ void largest_group_kernel(const int32_t* __restrict__ offsets, int64_t ng, int64_t skip, u64* result)
{
  u64 best = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = skip + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const u64 sz = (u64)(offsets[g + 1] - offsets[g]);
    const u64 cand = (sz << 32) | (u64)(0xffffffffu - (u32)g);
    best = cand > best ? cand : best;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { const u64 o = __shfl_xor_sync(0xffffffffu, best, d); best = o > best ? o : best; }
  if ((threadIdx.x & 31) == 0 && best) atomicMax(result, best);
}

int launch_largest_group(const int32_t* offsets, int64_t ng, int64_t skip, unsigned long long* d_result, cudaStream_t s)
{
  if (ng <= skip) return DTB_OK;
  largest_group_kernel<<<grid_for(ng - skip), 256, 0, s>>>(offsets, ng, skip, d_result);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// Natural join (frame/join.cc:392-470): for every row of X the row of J (sorted by its key columns,
// unique keys, NA first) whose key columns all compare equal, or NA.  Comparison per column follows
// FwCmp (join.cc:199-232): NA == NA, NA < valid, values compared in J's type; an X value that J's
// integer type cannot represent (out of range, or a fraction) matches nothing.
// ===========================================================================
struct JoinCol { const void* x; const void* j; int32_t xst, jst; };
struct JoinPlan { int nkeys; JoinCol c[MAX_KEYS]; };

__device__ __forceinline__ bool load_any(const void* p, int st, int64_t i, long long& iv, double& dv, bool& isf) {
  switch (st) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8:  { const int8_t t = ((const int8_t*)p)[i]; iv = t; isf = false; return t != INT8_MIN; }
    case DTB_STYPE_INT16: { const int16_t t = ((const int16_t*)p)[i]; iv = t; isf = false; return t != INT16_MIN; }
    case DTB_STYPE_INT32: case DTB_STYPE_DATE32: { const int32_t t = ((const int32_t*)p)[i]; iv = t; isf = false; return t != INT32_MIN; }
    case DTB_STYPE_INT64: case DTB_STYPE_TIME64: { const long long t = ((const long long*)p)[i]; iv = t; isf = false; return t != INT64_MIN; }
    case DTB_STYPE_FLOAT32: { const float t = ((const float*)p)[i]; dv = (double)t; isf = true; return !isnan(t); }
    default: { const double t = ((const double*)p)[i]; dv = t; isf = true; return !isnan(t); }
  }
}

__device__ __forceinline__ void int_range(int st, long long& lo, long long& hi) {
  switch (st) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8: lo = INT8_MIN; hi = INT8_MAX; break;
    case DTB_STYPE_INT16: lo = INT16_MIN; hi = INT16_MAX; break;
    case DTB_STYPE_INT32: case DTB_STYPE_DATE32: lo = INT32_MIN; hi = INT32_MAX; break;
    default: lo = INT64_MIN; hi = INT64_MAX; break;
  }
}

__global__ void join_kernel(JoinPlan jp, int64_t nx, int64_t nj, int32_t* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nx; r += stride) {
    // set_xrow: the X values of this row, converted to J's types
    bool xvalid[MAX_KEYS]; long long xi[MAX_KEYS]; double xd[MAX_KEYS];
    bool impossible = false;
    for (int c = 0; c < jp.nkeys; c++) {
      long long iv = 0; double dv = 0; bool isf = false;
      xvalid[c] = load_any(jp.c[c].x, jp.c[c].xst, r, iv, dv, isf);
      const bool jf = jp.c[c].jst == DTB_STYPE_FLOAT32 || jp.c[c].jst == DTB_STYPE_FLOAT64;
      if (jf) {
        xd[c] = isf ? dv : (double)iv;
        if (jp.c[c].jst == DTB_STYPE_FLOAT32) xd[c] = (double)(float)xd[c];    // static_cast<TJ>(newval)
      } else if (xvalid[c]) {
        long long lo, hi; int_range(jp.c[c].jst, lo, hi);
        if (isf) {
          const double t = trunc(dv);
          if (t != dv || dv < -9.2233720368547758e18 || dv >= 9.2233720368547758e18) impossible = true;
          else { iv = (long long)dv; }
        }
        if (iv < lo || iv > hi) impossible = true;
        xi[c] = iv;
      }
    }
    int32_t res = INT32_MIN;
    if (!impossible && nj > 0) {
      int64_t start = 0, end = nj - 1;
      bool found = false;
      int64_t at = 0;
      while (true) {
        const int64_t mid = (start < end) ? ((start + end) >> 1) : start;
        int cmp = 0;                                   // sign of (J row) - (X row), column by column
        for (int c = 0; c < jp.nkeys && cmp == 0; c++) {
          long long jv = 0; double jd = 0; bool isf = false;
          const bool jvalid = load_any(jp.c[c].j, jp.c[c].jst, mid, jv, jd, isf);
          if (jvalid && xvalid[c]) {
            if (isf) cmp = (jd > xd[c]) - (jd < xd[c]);
            else     cmp = (jv > xi[c]) - (jv < xi[c]);
          } else cmp = (int)jvalid - (int)xvalid[c];
        }
        if (start >= end) { found = (cmp == 0); at = mid; break; }
        if (cmp > 0) end = mid;
        else if (cmp < 0) start = mid + 1;
        else { found = true; at = mid; break; }
      }
      if (found) res = (int32_t)at;
    }
    out[r] = res;
  }
}

int launch_join(int nkeys, const void* const* xcols, const int* xst, const void* const* jcols, const int* jst,
                int64_t nx, int64_t nj, int32_t* out, cudaStream_t s)
{
  if (nx == 0) return DTB_OK;
  JoinPlan jp; jp.nkeys = nkeys;
  for (int c = 0; c < nkeys; c++) { jp.c[c].x = xcols[c]; jp.c[c].j = jcols[c]; jp.c[c].xst = xst[c]; jp.c[c].jst = jst[c]; }
  join_kernel<<<grid_for(nx), 256, 0, s>>>(jp, nx, nj, out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// lower bound: out[i] = number of rows of the ascending column `sorted` that are < values[i]
// (the cut points of a key-range exchange between GPUs, datatable_b200/dist.py)
// ===========================================================================
template <typename T>
__global__ void lower_bound_kernel(const T* __restrict__ sorted, int64_t n, const T* __restrict__ values, int64_t m,
                                   int64_t* __restrict__ out)
{
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const T x = values[i];
  int64_t lo = 0, hi = n;
  while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (sorted[mid] < x) lo = mid + 1; else hi = mid; }
  out[i] = lo;
}

int launch_lower_bound(const void* sorted, int stype, int64_t n, const void* values, int64_t m, int64_t* out, cudaStream_t s)
{
  if (m == 0) return DTB_OK;
  const int grid = grid_for(m);
#define CALL(T) lower_bound_kernel<T><<<grid, 256, 0, s>>>((const T*)sorted, n, (const T*)values, m, out)
  DTB_DISPATCH_STYPE(stype, CALL)
#undef CALL
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// i = integer slice under by() / sort(): the slice applied inside every group
// (FExpr_Literal_SliceInt::evaluate_iby, expr/fexpr_literal_sliceint.cc:82-170; an integer i is the
// slice [i, i+1), fexpr_literal_int.cc:146-192).  The reference walks the groups one after the other and
// appends; here: rows per group (one thread per group), a two-level scan that also drops the groups
// which select nothing, and a row-parallel emit.
// ===========================================================================
// first position, signed step and number of selected rows of the group [off0, off1); restates
// fexpr_literal_sliceint.cc:101-165 including its int32 casts
__device__ __forceinline__ void slice_of_group(const SliceParams& p, int32_t off0, int32_t off1, int32_t& first,
                                               int32_t& step, u32& count)
{
  const int32_t n = off1 - off0;
  step = (int32_t)p.step; count = 0; first = off0;
  if (step > 0) {
    int32_t a = p.has_start ? (int32_t)p.start : 0;
    int32_t b = p.has_stop ? (int32_t)p.stop : (int32_t)p.nrows;
    if (a < 0) a += n;
    if (a < 0) a = 0;
    if (b < 0) b += n;
    if (b > n) b = n;                                          // (stop > off1 -> off1, relative to the group)
    if (a < b) { first = off0 + a; count = (u32)(((long long)b - a + step - 1) / step); }
  } else if (step < 0) {
    int32_t a = (!p.has_start || p.start >= (long long)n) ? n - 1 : (int32_t)p.start;
    if (a < 0) a += n;
    int32_t b;
    if (!p.has_stop) b = -1;
    else { b = (int32_t)p.stop; if (b < 0) b += n; if (b < 0) b = -1; }
    if (a > b) { first = off0 + a; count = (u32)(((long long)a - b - (long long)step - 1) / -(long long)step); }
  } else {                                                     // step 0: `stop` copies of row `start`
    int32_t a = (int32_t)p.start;
    if (a < 0) a += n;
    if (a >= 0 && a < n) { first = off0 + a; count = (u32)p.stop; }
  }
}

constexpr int SL_BLOCK = 1024;                                 // groups per scan block (256 threads x 4)

__global__ void __launch_bounds__(256)
slice_count_kernel(const int32_t* __restrict__ offsets, int64_t ng, SliceParams p, u32* __restrict__ cnt,
                   u64* __restrict__ bsum /*[2 * nblocks]: rows, non-empty groups*/)
{
  __shared__ u64 wr[8], wg[8];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  u64 rows = 0, grp = 0;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int64_t g = ((int64_t)blockIdx.x * 256 + t) * 4 + j;
    u32 c = 0;
    if (g < ng) { int32_t f, st; slice_of_group(p, offsets[g], offsets[g + 1], f, st, c); cnt[g] = c; }
    rows += c; grp += c != 0;
  }
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

// exclusive scan of the block sums in place (one CTA walks them); totals[0] = rows, totals[1] = groups
__global__ void __launch_bounds__(1024)
slice_scan_kernel(u64* __restrict__ bsum, int64_t nb, u64* __restrict__ totals)
{
  __shared__ u64 sr[32], sg[32];
  __shared__ u64 carry_r, carry_g;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (t == 0) { carry_r = 0; carry_g = 0; }
  __syncthreads();
  for (int64_t b0 = 0; b0 < nb; b0 += 1024) {
    const int64_t b = b0 + t;
    const u64 r = b < nb ? bsum[2 * b] : 0, g = b < nb ? bsum[2 * b + 1] : 0;
    u64 ir = r, ig = g;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const u64 a = __shfl_up_sync(0xffffffffu, ir, d), c = __shfl_up_sync(0xffffffffu, ig, d);
      if (lane >= d) { ir += a; ig += c; }
    }
    if (lane == 31) { sr[warp] = ir; sg[warp] = ig; }
    __syncthreads();
    u64 pr = 0, pg = 0;
    for (int w = 0; w < warp; w++) { pr += sr[w]; pg += sg[w]; }
    const u64 cr = carry_r, cg = carry_g;
    if (b < nb) { bsum[2 * b] = cr + pr + ir - r; bsum[2 * b + 1] = cg + pg + ig - g; }
    __syncthreads();
    if (t == 1023) { carry_r = cr + pr + ir; carry_g = cg + pg + ig; }
    __syncthreads();
  }
  if (t == 0) { totals[0] = carry_r; totals[1] = carry_g; }
}

// offsets_out[k] = rows selected before the k-th non-empty group, gsel[k] = its index
__global__ void __launch_bounds__(256)
slice_compact_kernel(const u32* __restrict__ cnt, const u64* __restrict__ bsum, int64_t ng,
                     int32_t* __restrict__ offsets_out, int32_t* __restrict__ gsel)
{
  __shared__ u64 wr[8], wg[8];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  u32 c[4]; u64 rows = 0, grp = 0;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int64_t g = ((int64_t)blockIdx.x * 256 + t) * 4 + j;
    c[j] = g < ng ? cnt[g] : 0;
    rows += c[j]; grp += c[j] != 0;
  }
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
  u64 r = bsum[2 * (size_t)blockIdx.x] + pr + ir - rows;
  u64 k = bsum[2 * (size_t)blockIdx.x + 1] + pg + ig - grp;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    if (c[j]) {
      offsets_out[k] = (int32_t)r;
      gsel[k] = (int32_t)(((int64_t)blockIdx.x * 256 + t) * 4 + j);
      k++; r += c[j];
    }
  }
}

// rows_out[j] = first(g) + (j - offsets_out[k]) * step for the k-th remaining group g = gsel[k]
__global__ void slice_emit_kernel(const int32_t* __restrict__ offsets, SliceParams p, const int32_t* __restrict__ offsets_out,
                                  const int32_t* __restrict__ gsel, const int32_t* __restrict__ gid, int64_t nout,
                                  int32_t* __restrict__ rows_out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nout; j += stride) {
    const int32_t k = gid[j], g = gsel[k];
    int32_t first, step; u32 c;
    slice_of_group(p, offsets[g], offsets[g + 1], first, step, c);
    rows_out[j] = first + (int32_t)(j - offsets_out[k]) * step;
  }
}

size_t slice_scratch_bytes(int64_t ng) {
  const size_t nb = (size_t)((ng + SL_BLOCK - 1) / SL_BLOCK);
  return sizeof(u32) * (size_t)(ng + 4) + sizeof(u64) * (2 * nb + 4);
}

// phase 1: counts, scan, compaction.  totals (device u64[2]) receives {rows selected, groups left};
// offsets_out needs ng + 1 entries, gsel ng.  The caller reads totals, terminates offsets_out and runs phase 2.
int launch_slice_groups_plan(const int32_t* offsets, int64_t ng, const SliceParams& p, void* scratch, int32_t* offsets_out,
                             int32_t* gsel, unsigned long long* totals, cudaStream_t s)
{
  if (ng == 0) { DTB_CUDA_CHECK(cudaMemsetAsync(totals, 0, 2 * sizeof(u64), s)); return DTB_OK; }
  const int64_t nb = (ng + SL_BLOCK - 1) / SL_BLOCK;
  u32* cnt = (u32*)scratch;
  u64* bsum = (u64*)((char*)scratch + ((sizeof(u32) * (size_t)(ng + 4) + 7) / 8) * 8);
  slice_count_kernel<<<(unsigned)nb, 256, 0, s>>>(offsets, ng, p, cnt, bsum);
  slice_scan_kernel<<<1, 1024, 0, s>>>(bsum, nb, totals);
  slice_compact_kernel<<<(unsigned)nb, 256, 0, s>>>(cnt, bsum, ng, offsets_out, gsel);
  count_launch(3);
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// phase 2: gid scratch int32[nout]
int launch_slice_groups_emit(const int32_t* offsets, const SliceParams& p, const int32_t* offsets_out, const int32_t* gsel,
                             int64_t ng_out, int64_t nout, int32_t* gid, int32_t* rows_out, cudaStream_t s)
{
  if (nout == 0) return DTB_OK;
  DTB_TRY(launch_expand_gid(offsets_out, ng_out, nout, gid, s));
  slice_emit_kernel<<<grid_for(nout), 256, 0, s>>>(offsets, p, offsets_out, gsel, gid, nout, rows_out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

}  // namespace dtb
