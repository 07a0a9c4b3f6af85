// dtb_next.cu -- the callers either side of the hot path (SURVEY.md 8f): within-group ordered
// reducers, set operations, mode, keyed join.  All of them are consumers of group()'s
// RowIndex / Groupby pair; the kernels here are the per-group / per-row selection steps that the
// reference runs as serial host loops over `indices[goffsets[i]]`.
//
//   first / last          expr/head_reduce_unary.cc:120-190   value of the first / last row of a group
//   sd, cov / corr        expr/head_reduce_unary.cc:197-245,  sample standard deviation, covariance and correlation
//                         head_reduce_binary.cc:114-221       (Welford there; here: one set of moment kernels, two
//                                                             passes over the values shifted by the group's first
//                                                             valid value or pair)
//   median                expr/head_reduce_unary.cc:421-468   over rows sorted inside their group
//                                                             (Column::sort_grouped, sort.cc:1499-1530)
//   nunique               expr/head_reduce_unary.cc:383-415   distinct valid values per group
//   union / intersect / setdiff / symdiff   set_funcs.cc:126-456
//   mode / nmodal         stats.cc:955-1003
//   natural join          frame/join.cc:392-470               binary search of every X row in the sorted keys of J
//   boolean / integer i   rowindex_array.cc:63-203            the rows a bool8 column selects (two passes over the
//                                                             mask, no look-back); an integer column as an int32
//                                                             RowIndex
//
// Bound: none of these is a bandwidth kernel except the row-parallel ones (group ids, distinct
// flags, join), which are random-gather bound like reduce_kernel.
#include <limits>
#include <type_traits>
#include "dtb_common.cuh"

namespace dtb {

// raw element -> valid / float64: elem_valid<T> and to_f64<T> (of a loaded word) for a column of C++ type T; load_f64
// for a column of runtime stype st, which also says whether the element is valid
template <typename T> __device__ __forceinline__ bool elem_valid(const void* v, int64_t i) {
  typedef typename RawKey<T>::load_t L;
  u64 u; return RawKey<T>::get(((const L*)v)[i], u);
}
template <typename T> __device__ __forceinline__ double to_f64(typename RawKey<T>::load_t r) {
  if constexpr (std::is_same<T, float>::value) return (double)__uint_as_float(r);
  else if constexpr (std::is_same<T, double>::value) return __longlong_as_double((long long)r);
  else return (double)r;
}
__device__ __forceinline__ bool load_f64(const void* v, int st, int64_t j, double& x) {
  switch (st) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8: { const int8_t t = ((const int8_t*)v)[j]; x = (double)t; return t != INT8_MIN; }
    case DTB_STYPE_INT16: { const int16_t t = ((const int16_t*)v)[j]; x = (double)t; return t != INT16_MIN; }
    case DTB_STYPE_INT32: { const int32_t t = ((const int32_t*)v)[j]; x = (double)t; return t != INT32_MIN; }
    case DTB_STYPE_INT64: { const int64_t t = ((const int64_t*)v)[j]; x = (double)t; return t != INT64_MIN; }
    case DTB_STYPE_FLOAT32: { const float t = ((const float*)v)[j]; x = (double)t; return !isnan(t); }
    case DTB_STYPE_FLOAT64: { x = ((const double*)v)[j]; return !isnan(x); }
  }
  return false;
}

// ===========================================================================
// first / last: out[g] = v[order[offsets[g]]] or v[order[offsets[g+1]-1]] (NA stays NA); the empty group of zero
// rows, offsets [0, 0], is NA and reads no position
// ===========================================================================
template <typename E>
__global__ void firstlast_kernel(const E* __restrict__ v, int64_t nv, const int32_t* __restrict__ order,
                                 const int32_t* __restrict__ offsets, int64_t ng, int last, E na, E* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const int64_t a = offsets[g], b = offsets[g + 1];
    if (a >= b) { out[g] = na; continue; }
    const int64_t p = last ? b - 1 : a;
    const int64_t j = order ? (int64_t)order[p] : p;
    out[g] = (j >= 0 && j < nv) ? v[j] : na;
  }
}

int launch_firstlast(const void* v, int stype, int64_t nv, const int32_t* order, const int32_t* offsets,
                     int64_t ng, int last, void* out, cudaStream_t s)
{
  if (ng == 0) return DTB_OK;
  return with_stype(stype, "unsupported stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    typedef bits_t<T> E;
    firstlast_kernel<E><<<grid_for((ng + 255) / 256, 16), 256, 0, s>>>((const E*)v, nv, order, offsets, ng, last,
                                                                       (E)raw_na<T>(), (E*)out);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  });
}

// CTAs of a row-parallel kernel whose threads own 8 consecutive positions each
static int rows8_grid(int64_t n) { return grid_for(((n + 7) / 8 + 255) / 256, 16); }

// ===========================================================================
// group id of every sorted position: gid[p] = g for offsets[g] <= p < offsets[g+1]
// (each thread owns 8 consecutive positions: group_of, then a walk)
// ===========================================================================
__global__ void expand_gid_kernel(const int32_t* __restrict__ offsets, int64_t ng, int64_t n, int32_t* __restrict__ gid)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 8;
  for (int64_t p0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; p0 < n; p0 += stride) {
    int64_t g = group_of(offsets, ng, p0), next = offsets[g + 1];
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
  expand_gid_kernel<<<rows8_grid(n), 256, 0, s>>>(offsets, ng, n, gid);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// Column policies of the row-parallel per-group kernels below: at(j, x) says whether row j exists and qualifies, and
// widens its values to float64 in x[0 .. K).
// ===========================================================================
template <typename T> struct OneCol {             // sd: a valid value of one column of C++ type T
  static constexpr int K = 1;
  const typename RawKey<T>::load_t* v; int64_t nv;
  __device__ __forceinline__ bool at(int64_t j, double* x) const {
    if (j < 0 || j >= nv) return false;
    const typename RawKey<T>::load_t r = v[j];
    u64 u; x[0] = to_f64<T>(r);
    return RawKey<T>::get(r, u);
  }
};

struct PairCols {                                  // cov / corr: two columns of any numeric stype, both values valid
  static constexpr int K = 2;
  const void* x; const void* y; int sx, sy; int64_t nv;
  __device__ __forceinline__ bool at(int64_t j, double* v) const {
    if (j < 0 || j >= nv) return false;
    const bool vx = load_f64(x, sx, j, v[0]);
    const bool vy = load_f64(y, sy, j, v[1]);
    return vx && vy;
  }
};

template <typename T> struct ZeroCol {            // the sign of a zero float min / max: a zero of T, +0.0 or -0.0
  static constexpr int K = 1;
  const typename RawKey<T>::load_t* v; int64_t nv;
  __device__ __forceinline__ bool at(int64_t j, double* x) const {
    x[0] = 0.0;
    return j >= 0 && j < nv && (typename RawKey<T>::load_t)(v[j] << 1) == 0;
  }
};

// ===========================================================================
// first qualifying position of every group (the moments' pivot, the sign of a zero min / max): row-parallel, in the
// shape of the moment passes -- each thread owns 8 consecutive positions, finds its first group by bisection, and
// keeps the first position of each of its groups that qualifies; one atomicMin per (thread, group).  A serial walk
// per group would read a long NA prefix (or a late zero) one row at a time on one thread.
// ===========================================================================
template <typename Cols, typename OrdT>
__global__ void first_valid_pos_kernel(const Cols c, const OrdT* __restrict__ order, const int32_t* __restrict__ offsets,
                                       int64_t ng, int64_t n, const u64* __restrict__ gate, u64* __restrict__ pos)
{
  if (gate && *gate == 0) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 8;
  for (int64_t p0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; p0 < n; p0 += stride) {
    int64_t g = group_of(offsets, ng, p0), next = offsets[g + 1];
    u64 best = ~0ull;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int64_t p = p0 + i;
      if (p >= n) break;
      if (p >= next) {
        if (best != ~0ull) atomicMin(&pos[g], best);
        best = ~0ull;
        while (p >= next) { g++; next = offsets[g + 1]; }
      }
      double x[Cols::K];
      if (best == ~0ull && c.at(order ? (int64_t)order[p] : p, x)) best = (u64)p;
    }
    if (best != ~0ull) atomicMin(&pos[g], best);
  }
}

int launch_first_zero_pos(const void* v, int stype, int64_t nv, const void* order, int order_is64, const int32_t* offsets,
                          int64_t ng, int64_t n, const u64* gate, u64* pos, cudaStream_t s)
{
  if (ng == 0 || n == 0) return DTB_OK;
  with_order(order, order_is64, [&](auto o) {
    if (stype == DTB_STYPE_FLOAT32)
      first_valid_pos_kernel<<<rows8_grid(n), 256, 0, s>>>(ZeroCol<float>{(const u32*)v, nv}, o, offsets, ng, n, gate, pos);
    else
      first_valid_pos_kernel<<<rows8_grid(n), 256, 0, s>>>(ZeroCol<double>{(const u64*)v, nv}, o, offsets, ng, n, gate, pos);
  });
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// sd (OneCol) and cov / corr (PairCols, expr/head_reduce_binary.cc:114-221): the rows that qualify -- for cov / corr
// the rows where both values are valid, both widened to float64 (the reference casts to float32 when both columns
// are float32, else to float64) -- are shifted by a pivot p, the value at the group's first such row in RowIndex
// order, and then folded in two passes:
//   pass 1: sum += x - p, cnt += 1                 (mean' = sum / cnt, the mean of the shifted values)
//   pass 2: with dx = (x - p) - mean':  sd: sq += dx^2;  cov: sxy += dx dy;  corr: sxy, and sq += dx^2 per column
// A group whose valid values are all equal has x - p = 0 on every row, so its sd and cov are exactly 0 (corr NA), as
// the reference's Welford recurrence gives (a mean computed from the rounded sum is not the value itself: three rows
// of 0.1 gave 1.7e-17).  Squared deviations from the group's own mean do not cancel the way sum(x^2) - n mean^2 does,
// and the shift keeps them accurate when |mean| is much larger than the sd.
// One atomic per (thread, group) and word: pass 1 adds its words when the thread saw a row of the group, pass 2 each
// word that is not 0 (adding 0 to a word that starts at +0 never changes it).
// ===========================================================================

// per group: on entry pivot[0] holds, as u64, the group's first qualifying position (~0: none, so cnt stays 0 and the
// result is NA); on exit the pivot, and the words the passes add to are 0
template <int OP, typename Cols, typename OrdT>
__global__ void moment_pivot_kernel(const Cols c, const OrdT* __restrict__ order, int64_t ng, const MomentWords w)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const u64 p = reinterpret_cast<const u64*>(w.pivot[0])[g];
    double x[Cols::K] = {};
    if (p != ~0ull) c.at(order ? (int64_t)order[p] : (int64_t)p, x);
#pragma unroll
    for (int k = 0; k < Cols::K; k++) {
      w.pivot[k][g] = x[k];
      w.sum[k][g] = 0.0;
      if (OP != DTB_OP_COV) w.sq[k][g] = 0.0;
    }
    w.cnt[g] = 0;
    if (OP != DTB_OP_SD) w.sxy[g] = 0.0;
  }
}

template <int OP, bool PASS2, bool ORDERED, typename Cols, typename OrdT>
__device__ __forceinline__ void moment_rows(const Cols& c, const OrdT* __restrict__ order,
                                            const int32_t* __restrict__ offsets, int64_t ng, int64_t n,
                                            const MomentWords& w)
{
  constexpr int K = Cols::K;
  constexpr bool SQ = OP != DTB_OP_COV, XY = OP != DTB_OP_SD;      // what pass 2 adds up
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 8;
  for (int64_t p0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; p0 < n; p0 += stride) {
    int64_t g = group_of(offsets, ng, p0), next = offsets[g + 1];
    double piv[K], mean[K], a[K], axy;
    u32 cnt;
    auto enter = [&]() {                           // group g's pivot and mean' (read-only in this pass), nothing added yet
#pragma unroll
      for (int k = 0; k < K; k++) {
        piv[k] = __ldg(&w.pivot[k][g]);
        mean[k] = PASS2 ? __ldg(&w.sum[k][g]) / (double)__ldg(&w.cnt[g]) : 0.0;
        a[k] = 0.0;
      }
      axy = 0.0; cnt = 0;
    };
    auto flush = [&]() {
      if (!PASS2) {
        if (cnt) {
#pragma unroll
          for (int k = 0; k < K; k++) atomicAdd(&w.sum[k][g], a[k]);
          atomicAdd(&w.cnt[g], (u64)cnt);
        }
      } else {
        if (XY && axy != 0.0) atomicAdd(w.sxy + g, axy);
#pragma unroll
        for (int k = 0; k < K; k++) if (SQ && a[k] != 0.0) atomicAdd(&w.sq[k][g], a[k]);
      }
    };
    enter();
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int64_t p = p0 + i;
      if (p >= n) break;
      if (p >= next) {
        flush();
        while (p >= next) { g++; next = offsets[g + 1]; }
        enter();
      }
      double x[K];
      if (!c.at((ORDERED || order) ? (int64_t)order[p] : p, x)) continue;
      double d[K];
#pragma unroll
      for (int k = 0; k < K; k++) {
        d[k] = (x[k] - piv[k]) - mean[k];
        if (!PASS2) a[k] += d[k];
        else if (SQ) a[k] += d[k] * d[k];
      }
      if constexpr (PASS2 && XY) axy += d[0] * d[1];
      cnt++;
    }
    flush();
  }
}

template <int OP, bool PASS2, typename Cols, typename OrdT>
__global__ void moment_pass_kernel(const Cols c, const OrdT* __restrict__ order, const int32_t* __restrict__ offsets,
                                   int64_t ng, int64_t n, const MomentWords w)
{
  // ORDERED: order is known to be set.  Pass 1 runs a copy of the loop specialised to it: without one its pair instance
  // compiles to 40 registers instead of 64 and is 4-5 % slower on C4 keys.  Pass 2 keeps one loop: specialised, it
  // would need 66-68 registers instead of 44.
  if (!PASS2 && order) moment_rows<OP, PASS2, true>(c, order, offsets, ng, n, w);
  else                 moment_rows<OP, PASS2, false>(c, order, offsets, ng, n, w);
}

// sd: NA unless cnt > 1 and sq is not NaN (head_reduce_unary.cc:213), else sqrt(sq / (cnt - 1)); cov: NA when
// cnt <= 1, else sxy / (cnt - 1); corr: NA unless cnt > 1 and sq_x * sq_y > 0, else sxy / sqrt(sq_x * sq_y)
// (head_reduce_binary.cc:134-136, 196-200; no clamping)
template <int OP>
__global__ void moment_finalize_kernel(const MomentWords w, int64_t ng, int out_stype, void* out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const u64 c = w.cnt[g];
    bool valid; double r;
    if constexpr (OP == DTB_OP_SD) {
      const double q = w.sq[0][g];
      valid = c > 1 && !isnan(q);
      r = q >= 0 ? sqrt(q / (double)(c - 1)) : 0.0;
    } else if constexpr (OP == DTB_OP_COV) {
      valid = c > 1;
      r = w.sxy[g] / (double)(c - 1);
    } else {
      const double vv = w.sq[0][g] * w.sq[1][g];
      valid = c > 1 && vv > 0;
      r = w.sxy[g] / sqrt(vv);
    }
    store_float(out, out_stype, g, valid, r);
  }
}

template <int OP, typename Cols, typename OrdT>
static int run_moments(const Cols& c, const OrdT* order, const int32_t* offsets, int64_t ng, int64_t n,
                       const MomentWords& w, int out_stype, void* out, cudaStream_t s)
{
  const int grid = rows8_grid(n), ggrid = grid_for((ng + 255) / 256, 16);
  fill_u64(reinterpret_cast<u64*>(w.pivot[0]), ng, ~0ull, s);
  if (n > 0) {
    first_valid_pos_kernel<<<grid, 256, 0, s>>>(c, order, offsets, ng, n, nullptr, reinterpret_cast<u64*>(w.pivot[0]));
    count_launch();
  }
  moment_pivot_kernel<OP><<<ggrid, 256, 0, s>>>(c, order, ng, w);         // with no rows: every group NA
  if (n > 0) {
    moment_pass_kernel<OP, false><<<grid, 256, 0, s>>>(c, order, offsets, ng, n, w);
    moment_pass_kernel<OP, true><<<grid, 256, 0, s>>>(c, order, offsets, ng, n, w);
    count_launch(2);
  }
  moment_finalize_kernel<OP><<<ggrid, 256, 0, s>>>(w, ng, out_stype, out);
  count_launch(2);
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int launch_moments(int op, const void* x, int sx, const void* y, int sy, int64_t nv, const void* order, int order_is64,
                   const int32_t* offsets, int64_t ng, int64_t n, const MomentWords& w, int out_stype, void* out,
                   cudaStream_t s)
{
  if (ng == 0) return DTB_OK;
  if (op == DTB_OP_SD)
    return with_stype(sx, "unsupported stype ", [&](auto t) {
      typedef typename decltype(t)::type T;
      const OneCol<T> c = {(const typename RawKey<T>::load_t*)x, nv};
      return run_moments<DTB_OP_SD>(c, (const int32_t*)order, offsets, ng, n, w, out_stype, out, s);
    });
  const PairCols c = {x, y, sx, sy, nv};
  int rc = DTB_OK;
  with_order(order, order_is64, [&](auto o) {
    rc = (op == DTB_OP_CORR) ? run_moments<DTB_OP_CORR>(c, o, offsets, ng, n, w, out_stype, out, s)
                             : run_moments<DTB_OP_COV>(c, o, offsets, ng, n, w, out_stype, out, s);
  });
  return rc;
}

int reduce2_out_stype_host(int op, int sx, int sy) {
  auto num = [](int st) { return st == DTB_STYPE_BOOL || st == DTB_STYPE_INT8 || st == DTB_STYPE_INT16 || st == DTB_STYPE_INT32 ||
                                 st == DTB_STYPE_INT64 || st == DTB_STYPE_FLOAT32 || st == DTB_STYPE_FLOAT64; };
  if ((op != DTB_OP_COV && op != DTB_OP_CORR) || !num(sx) || !num(sy)) return 0;
  return (sx == DTB_STYPE_FLOAT32 && sy == DTB_STYPE_FLOAT32) ? DTB_STYPE_FLOAT32 : DTB_STYPE_FLOAT64;   // :154-159
}

size_t reduce2_scratch_bytes(int64_t ng) { return sizeof(u64) * 8 * (size_t)(ng > 0 ? ng : 1); }

int launch_reduce2(int op, const void* x, int sx, const void* y, int sy, int64_t nv, const void* order, int order_is64,
                   const int32_t* offsets, int64_t ng, int64_t n, u64* scratch, int out_f32, void* out, cudaStream_t s)
{
  double* d = reinterpret_cast<double*>(scratch);             // sx, sy, cnt, sxy, sxx, syy, px, py
  const MomentWords w = {{d, d + ng}, scratch + 2 * ng, {d + 4 * ng, d + 5 * ng}, d + 3 * ng, {d + 6 * ng, d + 7 * ng}};
  return launch_moments(op, x, sx, y, sy, nv, order, order_is64, offsets, ng, n, w,
                        out_f32 ? DTB_STYPE_FLOAT32 : DTB_STYPE_FLOAT64, out, s);
}

// ===========================================================================
// median over rows already sorted inside their group (NA first): one thread per group
// ===========================================================================
template <typename T>
__global__ void median_kernel(const void* __restrict__ v, int64_t nv, const int32_t* __restrict__ order,
                              const int32_t* __restrict__ offsets, int64_t ng, void* out)
{
  constexpr bool F32 = std::is_same<T, float>::value;
  const typename RawKey<T>::load_t* w = (const typename RawKey<T>::load_t*)v;
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
        m = to_f64<T>(w[r1]);
      } else {
        const int64_t r2 = order ? (int64_t)order[jm - 1] : jm - 1;
        if (F32) m = (double)(((float)to_f64<T>(w[r1]) + (float)to_f64<T>(w[r2])) / 2.0f);
        else m = (to_f64<T>(w[r1]) + to_f64<T>(w[r2])) / 2;
      }
    }
    store_float(out, F32 ? DTB_STYPE_FLOAT32 : DTB_STYPE_FLOAT64, g, valid, m);
  }
}

int launch_median(const void* v, int stype, int64_t nv, const int32_t* order, const int32_t* offsets,
                  int64_t ng, void* out, cudaStream_t s)
{
  if (ng == 0) return DTB_OK;
  return with_stype(stype, "unsupported stype ", [&](auto t) {
    median_kernel<typename decltype(t)::type><<<grid_for((ng + 255) / 256, 16), 256, 0, s>>>(v, nv, order, offsets, ng, out);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  });
}

// ===========================================================================
// nunique over rows sorted inside their group: flag[p] = 1 where a valid value differs from the row
// before it (std::set<T> semantics, head_reduce_unary.cc:383-394: -0.0 and +0.0 are one value);
// group starts are corrected by a per-group kernel; the flags are then counted per group.
// ===========================================================================
template <typename T>
__device__ __forceinline__ bool same_value(const void* v, int64_t a, int64_t b) {
  typedef typename RawKey<T>::load_t L;
  if constexpr (std::is_floating_point<T>::value) return to_f64<T>(((const L*)v)[a]) == to_f64<T>(((const L*)v)[b]);
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
  return with_stype(stype, "unsupported stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    distinct_flags_kernel<T><<<grid_for((n + 255) / 256, 16), 256, 0, s>>>(v, nv, order, n, flag);
    distinct_starts_kernel<T><<<grid_for((ng + 255) / 256, 16), 256, 0, s>>>(v, nv, order, offsets, ng, flag);
    count_launch(2);
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  });
}

// ===========================================================================
// qcut (column/qcut.h:78-155) inside every group, over group() of the composite key (group id, value): cord / coff
// are that group()'s RowIndex (sorted position -> RowIndex position of the outer Groupby) and offsets.  The group id
// leads the key, so the composite groups of one outer group are contiguous; inside it they are its distinct values by
// group()'s identity (bit patterns: -0.0 and +0.0 differ, every NaN is NA), NA first.
//   qcut_starts_kernel  per composite group c: cog[c] = its outer group, cstart[og] = first composite group of og
//   qcut_coef_kernel    per outer group: G, has_na and the coefficients a, b of Qcut_ColumnImpl::materialize
//   qcut_emit_kernel    per sorted position (a single value may hold most rows): out[pos] = int32(a * i + b) with
//                       i = c - cstart[og], NA for the NA group
// a * i + b is a multiply and an add, each rounded (__dmul_rn / __dadd_rn), as the reference computes it: a
// contracted FMA could round differently.
// ===========================================================================
__global__ void qcut_starts_kernel(const int32_t* __restrict__ cord, const int32_t* __restrict__ coff, int64_t nc,
                                   const int32_t* __restrict__ gid, int64_t ng, int32_t* __restrict__ cog,
                                   int32_t* __restrict__ cstart)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += stride) {
    const int32_t og = gid[cord[coff[c]]];
    cog[c] = og;
    if (c == 0 || gid[cord[coff[c - 1]]] != og) cstart[og] = (int32_t)c;
    if (c == nc - 1) cstart[ng] = (int32_t)nc;
  }
}

template <typename T>
__global__ void qcut_coef_kernel(const void* __restrict__ vg, const int32_t* __restrict__ cord,
                                 const int32_t* __restrict__ coff, const int32_t* __restrict__ cstart, int64_t ng,
                                 int q, double2* __restrict__ coef, uint8_t* __restrict__ has_na)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += stride) {
    const int64_t c0 = cstart[g];
    const int64_t G = (int64_t)cstart[g + 1] - c0;
    const bool na = !elem_valid<T>(vg, cord[coff[c0]]);      // NA first: the group's first value
    const int64_t V = G - (na ? 1 : 0);
    double a, b;
    if (V <= 1) {                                              // one valid value (or none: only the NA group)
      a = 0.0;
      b = (double)((q - 1) / 2);
    } else {                                                   // q * (1 - FLT_EPSILON) / (V - 1), b = -a * has_na
      a = __ddiv_rn(__dmul_rn((double)q, 1.0 - 1.0 / 8388608.0), (double)(V - 1));     // FLT_EPSILON = 2^-23
      b = __dmul_rn(-a, na ? 1.0 : 0.0);
    }
    coef[g] = make_double2(a, b);
    has_na[g] = na ? 1 : 0;
  }
}

__global__ void qcut_emit_kernel(const int32_t* __restrict__ cord, const int32_t* __restrict__ coff, int64_t nc,
                                 int64_t n, const int32_t* __restrict__ cog, const int32_t* __restrict__ cstart,
                                 const double2* __restrict__ coef, const uint8_t* __restrict__ has_na,
                                 int32_t* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 8;
  for (int64_t k0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; k0 < n; k0 += stride) {
    int64_t c = group_of(coff, nc, k0), next = coff[c + 1];
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const int64_t k = k0 + j;
      if (k >= n) break;
      while (k >= next) { c++; next = coff[c + 1]; }
      const int32_t og = cog[c];
      const int64_t i = c - cstart[og];
      int32_t bin = INT32_MIN;
      if (i > 0 || !has_na[og]) {
        const double2 ab = coef[og];
        bin = (int32_t)__dadd_rn(__dmul_rn(ab.x, (double)i), ab.y);
      }
      out[cord[k]] = bin;
    }
  }
}

size_t qcut_scratch_bytes(int64_t nc, int64_t ng) {
  return sizeof(double2) * (size_t)ng + sizeof(int32_t) * (size_t)(ng + 1 + nc) + (size_t)ng;
}

int launch_qcut(const void* vg, int stype, const int32_t* cord, const int32_t* coff, int64_t nc, const int32_t* gid,
                int64_t ng, int64_t n, int q, void* scratch, int32_t* out, cudaStream_t s)
{
  if (n == 0 || ng == 0) return DTB_OK;
  double2* coef = (double2*)scratch;
  int32_t* cstart = (int32_t*)(coef + ng);
  int32_t* cog = cstart + ng + 1;
  uint8_t* has_na = (uint8_t*)(cog + nc);
  {
    ProfScope ps("qcut_coef", s);
    qcut_starts_kernel<<<grid_for((nc + 255) / 256, 16), 256, 0, s>>>(cord, coff, nc, gid, ng, cog, cstart);
    DTB_TRY(with_stype(stype, "unsupported stype ", [&](auto t) {
      qcut_coef_kernel<typename decltype(t)::type><<<grid_for((ng + 255) / 256, 16), 256, 0, s>>>(vg, cord, coff, cstart,
                                                                                                 ng, q, coef, has_na);
      return DTB_OK;
    }));
    count_launch(2);
    DTB_CUDA_CHECK(cudaGetLastError());
  }
  ProfScope ps("qcut_emit", s);
  qcut_emit_kernel<<<rows8_grid(n), 256, 0, s>>>(cord, coff, nc, n, cog, cstart, coef, has_na, out);
  count_launch();
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
  set_select_kernel<<<grid_for((ng + 255) / 256, 16), 256, 0, s>>>(order, offsets, ng, d_sizes, K, mode, flags);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int launch_set_emit(const int32_t* pos, int64_t nsel, const int32_t* order, const int32_t* offsets, int32_t* out_rows,
                    cudaStream_t s)
{
  if (nsel == 0) return DTB_OK;
  set_emit_kernel<<<grid_for((nsel + 255) / 256, 16), 256, 0, s>>>(pos, nsel, order, offsets, out_rows);
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
  largest_group_kernel<<<grid_for((ng - skip + 255) / 256, 16), 256, 0, s>>>(offsets, ng, skip, d_result);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// Natural join (frame/join.cc:392-470): for every row of X the row of J (sorted by its key columns,
// unique keys, NA first) whose key columns all compare equal, or NA.  Comparison per column follows
// FwCmp (join.cc:199-232): NA == NA, NA < valid, values compared in J's type; an X value that J's
// integer type cannot represent (out of range, or a fraction) matches nothing.
// At the row found, the kernel also writes J's value columns in X's row order (NA where nothing matches), so a
// query that reads J's columns through the join never materialises the index.
// Lookup: a single integer / date32 / time64 key column of J whose valid keys are consecutive (J is keyed: sorted,
// unique, NA first, so jkey[last] - jkey[first valid] == nvalid - 1 decides it from two reads) is addressed
// directly, row = x - kmin + (J has an NA row); every other J takes the binary search.
// ===========================================================================
struct JoinCol { const void* x; const void* j; int32_t xst, jst; };
struct JoinVal { const void* src; void* out; u64 na; int32_t bytes; };
struct JoinPlan { int nkeys, nvals; int32_t* index; JoinCol c[MAX_KEYS]; JoinVal v[JOIN_MAX_VALS]; };

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

__device__ __forceinline__ bool is_float_stype(int st) { return st == DTB_STYPE_FLOAT32 || st == DTB_STYPE_FLOAT64; }

__global__ void join_kernel(JoinPlan jp, int64_t nx, int64_t nj)
{
  // direct address: one integer key column whose valid keys are kmin .. kmin + nvalid - 1
  bool direct = false;
  long long kmin = 0;
  int64_t jna = 0, nvalid = 0;
  if (jp.nkeys == 1 && nj > 0 && !is_float_stype(jp.c[0].jst)) {
    long long k0 = 0, kl = 0; double d; bool f;
    jna = load_any(jp.c[0].j, jp.c[0].jst, 0, k0, d, f) ? 0 : 1;
    nvalid = nj - jna;
    if (nvalid > 0) {
      load_any(jp.c[0].j, jp.c[0].jst, jna, k0, d, f);
      load_any(jp.c[0].j, jp.c[0].jst, nj - 1, kl, d, f);
      direct = (unsigned long long)kl - (unsigned long long)k0 == (unsigned long long)(nvalid - 1);
      kmin = k0;
    }
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nx; r += stride) {
    // set_xrow: the X values of this row, converted to J's types
    bool xvalid[MAX_KEYS]; long long xi[MAX_KEYS]; double xd[MAX_KEYS];
    bool impossible = false;
    for (int c = 0; c < jp.nkeys; c++) {
      long long iv = 0; double dv = 0; bool isf = false;
      xvalid[c] = load_any(jp.c[c].x, jp.c[c].xst, r, iv, dv, isf);
      const bool jf = jp.c[c].jst == DTB_STYPE_FLOAT32 || jp.c[c].jst == DTB_STYPE_FLOAT64;
      if (jf) {                                        // static_cast<TJ>(newval): one rounding, from X's own type
        if (jp.c[c].jst == DTB_STYPE_FLOAT32) xd[c] = isf ? (double)(float)dv : (double)(float)iv;
        else                                  xd[c] = isf ? dv : (double)iv;
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
    if (!impossible && direct) {
      if (!xvalid[0]) { if (jna) res = 0; }
      else {
        const unsigned long long off = (unsigned long long)xi[0] - (unsigned long long)kmin;
        if (off < (unsigned long long)nvalid) res = (int32_t)(off + jna);
      }
    } else if (!impossible && nj > 0) {
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
    if (jp.index) jp.index[r] = res;
    for (int v = 0; v < jp.nvals; v++) {
      const JoinVal& c = jp.v[v];
      switch (c.bytes) {
        case 1: ((uint8_t*)c.out)[r]  = res >= 0 ? ((const uint8_t*)c.src)[res]  : (uint8_t)c.na;  break;
        case 2: ((uint16_t*)c.out)[r] = res >= 0 ? ((const uint16_t*)c.src)[res] : (uint16_t)c.na; break;
        case 4: ((u32*)c.out)[r]      = res >= 0 ? ((const u32*)c.src)[res]      : (u32)c.na;      break;
        default: ((u64*)c.out)[r]     = res >= 0 ? ((const u64*)c.src)[res]      : c.na;           break;
      }
    }
  }
}

int launch_join(int nkeys, const void* const* xcols, const int* xst, const void* const* jcols, const int* jst,
                int64_t nx, int64_t nj, int32_t* index, int nvals, const void* const* vals, const int* vst,
                void* const* vout, cudaStream_t s)
{
  if (nx == 0) return DTB_OK;
  JoinPlan jp; jp.nkeys = nkeys; jp.index = index;
  for (int c = 0; c < nkeys; c++) { jp.c[c].x = xcols[c]; jp.c[c].j = jcols[c]; jp.c[c].xst = xst[c]; jp.c[c].jst = jst[c]; }
  // at most JOIN_MAX_VALS value columns per launch; every further batch repeats the lookup (J stays in L2)
  int v0 = 0;
  do {
    jp.nvals = nvals - v0 < JOIN_MAX_VALS ? nvals - v0 : JOIN_MAX_VALS;
    for (int v = 0; v < jp.nvals; v++) {
      JoinVal& c = jp.v[v];
      c.src = vals[v0 + v]; c.out = vout[v0 + v]; c.bytes = stype_bytes(vst[v0 + v]);
      DTB_TRY(with_stype(vst[v0 + v], "Unable to join a column of stype ", [&](auto t) {
        typedef typename decltype(t)::type T;
        c.na = (u64)raw_na<T>();
        return DTB_OK;
      }));
    }
    join_kernel<<<grid_for((nx + 255) / 256, 16), 256, 0, s>>>(jp, nx, nj);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    jp.index = nullptr;
    v0 += jp.nvals;
  } while (v0 < nvals);
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
  return with_stype(stype, "unsupported stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    lower_bound_kernel<T><<<grid_for((m + 255) / 256, 16), 256, 0, s>>>((const T*)sorted, n, (const T*)values, m, out);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  });
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

// exclusive scan of K interleaved block sums in place (one CTA walks them): bsum[K * b + k] becomes the sum of
// component k over the blocks before b, totals[k] its sum over all blocks.  The slices scan K = 2 (rows, groups),
// the boolean compaction K = 1 (selected rows per tile).
template <int K>
__global__ void __launch_bounds__(1024)
block_sums_scan_kernel(u64* __restrict__ bsum, int64_t nb, u64* __restrict__ totals)
{
  __shared__ u64 sw[K][32];
  __shared__ u64 carry[K];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (t < K) carry[t] = 0;
  __syncthreads();
  for (int64_t b0 = 0; b0 < nb; b0 += 1024) {
    const int64_t b = b0 + t;
    u64 v[K], in[K];
#pragma unroll
    for (int k = 0; k < K; k++) { v[k] = b < nb ? bsum[K * b + k] : 0; in[k] = v[k]; }
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
#pragma unroll
      for (int k = 0; k < K; k++) {
        const u64 a = __shfl_up_sync(0xffffffffu, in[k], d);
        if (lane >= d) in[k] += a;
      }
    }
    if (lane == 31) {
#pragma unroll
      for (int k = 0; k < K; k++) sw[k][warp] = in[k];
    }
    __syncthreads();
    u64 pre[K];
#pragma unroll
    for (int k = 0; k < K; k++) {
      pre[k] = carry[k];
      for (int w = 0; w < warp; w++) pre[k] += sw[k][w];
      if (b < nb) bsum[K * b + k] = pre[k] + in[k] - v[k];
    }
    __syncthreads();
    if (t == 1023) {
#pragma unroll
      for (int k = 0; k < K; k++) carry[k] = pre[k] + in[k];
    }
    __syncthreads();
  }
  if (t < K) totals[t] = carry[t];
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
  block_sums_scan_kernel<2><<<1, 1024, 0, s>>>(bsum, nb, totals);
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
  slice_emit_kernel<<<grid_for((nout + 255) / 256, 16), 256, 0, s>>>(offsets, p, offsets_out, gsel, gid, nout, rows_out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// i = a boolean column: the ascending positions of its selected rows (ArrayRowIndexImpl::init_from_boolean_column,
// rowindex_array.cc:130-170, a serial loop there).  A row is selected when its byte is neither 0 nor the NA -128,
// i.e. when its low 7 bits are not all zero.  Two passes over the mask, no look-back: mask_count_kernel writes the
// selected rows of every MASK_TILE-row tile, block_sums_scan_kernel<1> turns them into each tile's first output
// position, and mask_emit_kernel reads its tile again and writes the tile's positions as one contiguous run.
// ===========================================================================
constexpr int MASK_THREADS = 256;
constexpr int MASK_VECS = 8;                                   // 16-byte loads per thread and tile
constexpr int MASK_CHUNK = MASK_THREADS * 16;                  // rows of one round of loads: 4096
constexpr int MASK_TILE = MASK_CHUNK * MASK_VECS;              // 32768 rows per tile

// 16 bytes of the mask: rows [16 v, 16 v + 16) of the column; rows at or past n read as 0.  aligned: the column's
// base is 16-byte aligned, so that whole vectors are read with one load.
__device__ __forceinline__ uint4 mask_vec(const int8_t* __restrict__ m, int64_t n, int64_t v, bool aligned)
{
  const int64_t r0 = v * 16;
  if (aligned && r0 + 16 <= n) return __ldg(reinterpret_cast<const uint4*>(m) + v);
  u32 w[4] = {0, 0, 0, 0};
  for (int b = 0; b < 16; b++)
    if (r0 + b < n) w[b >> 2] |= (u32)(uint8_t)m[r0 + b] << (8 * (b & 3));
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// bit b (0..3) set when byte b of w is selected
__device__ __forceinline__ u32 mask_bits4(u32 w)
{
  const u32 s = ((w & 0x7f7f7f7fu) + 0x7f7f7f7fu) & 0x80808080u;   // high bit of a byte: its low 7 bits are not 0
  return ((s >> 7) & 1u) | ((s >> 14) & 2u) | ((s >> 21) & 4u) | ((s >> 28) & 8u);
}

// bit b (0..15) set when row 16 v + b is selected
__device__ __forceinline__ u32 mask_bits16(uint4 q)
{
  return mask_bits4(q.x) | (mask_bits4(q.y) << 4) | (mask_bits4(q.z) << 8) | (mask_bits4(q.w) << 12);
}

__global__ void __launch_bounds__(MASK_THREADS)
mask_count_kernel(const int8_t* __restrict__ mask, int64_t n, bool aligned, u64* __restrict__ tile_count)
{
  __shared__ u32 ws[MASK_THREADS / 32];
  const int t = threadIdx.x;
  const int64_t v0 = (int64_t)blockIdx.x * (MASK_TILE / 16) + t;
  uint4 q[MASK_VECS];
#pragma unroll
  for (int j = 0; j < MASK_VECS; j++) q[j] = mask_vec(mask, n, v0 + j * MASK_THREADS, aligned);
  u32 c = 0;
#pragma unroll
  for (int j = 0; j < MASK_VECS; j++) c += __popc(mask_bits16(q[j]));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
  if ((t & 31) == 0) ws[t >> 5] = c;
  __syncthreads();
  if (t == 0) {
    u32 sum = 0;
#pragma unroll
    for (int w = 0; w < MASK_THREADS / 32; w++) sum += ws[w];
    tile_count[blockIdx.x] = sum;
  }
}

// One CTA per tile.  Every round of loads covers MASK_CHUNK consecutive rows, 16 per thread in thread order: a
// thread's rank is the popcount of its 16 bits plus a warp scan of the counts plus the counts of the warps before
// it.  The positions go to shared memory at their rank, then out as one coalesced run after the tile's start.
__global__ void __launch_bounds__(MASK_THREADS)
mask_emit_kernel(const int8_t* __restrict__ mask, int64_t n, bool aligned, const u64* __restrict__ tile_start,
                 int32_t* __restrict__ rows_out)
{
  __shared__ int32_t pos[MASK_CHUNK];
  __shared__ u32 ws[MASK_THREADS / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t v0 = (int64_t)blockIdx.x * (MASK_TILE / 16) + t;
  uint4 q[MASK_VECS];
#pragma unroll
  for (int j = 0; j < MASK_VECS; j++) q[j] = mask_vec(mask, n, v0 + j * MASK_THREADS, aligned);
  int32_t* out = rows_out + tile_start[blockIdx.x];
#pragma unroll
  for (int j = 0; j < MASK_VECS; j++) {
    u32 bits = mask_bits16(q[j]);
    const u32 c = __popc(bits);
    u32 inc = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const u32 a = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += a;
    }
    if (lane == 31) ws[warp] = inc;
    __syncthreads();
    u32 rank = inc - c, total = 0;
#pragma unroll
    for (int w = 0; w < MASK_THREADS / 32; w++) {
      const u32 x = ws[w];
      rank += w < warp ? x : 0;
      total += x;
    }
    const int32_t row0 = (int32_t)((v0 + j * MASK_THREADS) * 16);
    while (bits) {
      pos[rank++] = row0 + (__ffs(bits) - 1);
      bits &= bits - 1;
    }
    __syncthreads();
    for (u32 i = t; i < total; i += MASK_THREADS) out[i] = pos[i];
    out += total;
    __syncthreads();                                           // pos and ws are reused by the next round
  }
}

int64_t mask_num_tiles(int64_t n) { return (n + MASK_TILE - 1) / MASK_TILE; }

int launch_mask_count(const int8_t* mask, int64_t n, u64* tile_count, u64* total, cudaStream_t s)
{
  const int64_t nt = mask_num_tiles(n);
  if (nt == 0) { DTB_CUDA_CHECK(cudaMemsetAsync(total, 0, sizeof(u64), s)); return DTB_OK; }
  const bool aligned = (reinterpret_cast<uintptr_t>(mask) & 15) == 0;
  mask_count_kernel<<<(unsigned)nt, MASK_THREADS, 0, s>>>(mask, n, aligned, tile_count);
  block_sums_scan_kernel<1><<<1, 1024, 0, s>>>(tile_count, nt, total);
  count_launch(2);
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

int launch_mask_emit(const int8_t* mask, int64_t n, const u64* tile_start, int32_t* rows_out, cudaStream_t s)
{
  const int64_t nt = mask_num_tiles(n);
  if (nt == 0) return DTB_OK;
  const bool aligned = (reinterpret_cast<uintptr_t>(mask) & 15) == 0;
  mask_emit_kernel<<<(unsigned)nt, MASK_THREADS, 0, s>>>(mask, n, aligned, tile_start, rows_out);
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

// ===========================================================================
// i = an int8 / int16 / int64 column: its values as an int32 RowIndex, NA -> INT32_MIN (the NA row).  The caller
// has checked the valid values against the frame's rows, so they fit.  16-byte loads of the selector.
// ===========================================================================
template <typename T>
__global__ void __launch_bounds__(256)
narrow_rows_kernel(const T* __restrict__ sel, int64_t n, int32_t* __restrict__ out)
{
  constexpr int VEC = 16 / sizeof(T);
  constexpr T NA = std::numeric_limits<T>::min();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const bool aligned = (reinterpret_cast<uintptr_t>(sel) & 15) == 0;
  const int64_t nvec = aligned ? n / VEC : 0;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    const uint4 q = __ldg(reinterpret_cast<const uint4*>(sel) + v);
    const T* e = reinterpret_cast<const T*>(&q);
#pragma unroll
    for (int k = 0; k < VEC; k++) out[v * VEC + k] = e[k] == NA ? INT32_MIN : (int32_t)e[k];
  }
  for (int64_t i = nvec * VEC + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = sel[i] == NA ? INT32_MIN : (int32_t)sel[i];
}

int launch_narrow_rows(const void* sel, int stype, int64_t n, int32_t* out, cudaStream_t s)
{
  if (n == 0) return DTB_OK;
  auto run = [&](auto tag) {
    typedef decltype(tag) T;
    constexpr int VEC = 16 / sizeof(T);
    narrow_rows_kernel<T><<<grid_for((n / VEC + 255) / 256 + 1, 8), 256, 0, s>>>((const T*)sel, n, out);
    return DTB_OK;
  };
  switch (stype) {
    case DTB_STYPE_INT8:  run(int8_t()); break;
    case DTB_STYPE_INT16: run(int16_t()); break;
    case DTB_STYPE_INT64: run(int64_t()); break;
    default: set_error("narrow_rows takes int8, int16 or int64, not stype " + std::to_string(stype)); return DTB_EINVAL;
  }
  count_launch();
  DTB_CUDA_CHECK(cudaGetLastError());
  return DTB_OK;
}

}  // namespace dtb
