// dtb_cut.cu -- dt.cut over the positions of a RowIndex: replaces CutNbins_ColumnImpl and CutBins_ColumnImpl
// (column/cut.h:91-281) as FExpr_Cut::evaluate_n runs them (expr/fexpr_cut.cc:88-170).
//
//   nbins  cut_stats  min / max / valid count of the column seen through the RowIndex (launch_col_stats or
//                     launch_col_stats_gather, dtb_stats.cu), then cut_coef_kernel turns them into a, b, shift on the
//                     device: the call never waits for them.
//          cut_emit   out[p] = int32(trunc(a * v + b)) + shift, v = value[order[p]] as float64.
//   edges  cut_bins   out[p] = the bin of v by a branch-free bound search over the edges (no statistics pass).
//
// Every multiply and add is rounded on its own (__dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn), as the reference
// computes them: a contracted FMA could round differently.  Row-parallel and bound by HBM: per row the emit reads the
// index (4 or 8 bytes, none for the identity), the value (sizeof(T)) and writes 4 bytes; nbins adds one more read of
// the index and the value for the statistics.
#include "dtb_common.cuh"

namespace dtb {

constexpr int CUT_THREADS = 256;
constexpr int CUT_IPT = 4;                 // positions per thread per step: independent loads in flight
constexpr int CUT_SMEM_EDGES = 4096;       // edges staged in shared memory (32 KB); above it, every k-th edge

// value[j] as float64 (int64 rounded to nearest, as cast_inplace(FLOAT64) does); false for NA, or j outside [0, nv)
template <typename T>
__device__ __forceinline__ bool cut_load(const T* __restrict__ v, int64_t nv, int64_t j, double& x) {
  if (j < 0 || j >= nv) return false;
  const T t = v[j];
  if constexpr (std::is_floating_point<T>::value) {
    x = (double)t;
    return t == t;
  } else if constexpr (sizeof(T) == 8) {
    x = __ll2double_rn((long long)t);
    return t != NaOf<T>::v();
  } else {
    x = (double)t;
    return t != NaOf<T>::v();
  }
}

// static_cast<int32_t>(r) as x86-64 executes it (cvttsd2si): truncation, and INT32_MIN for NaN or a value outside the
// int32 range (where __double2int_rz would saturate)
__device__ __forceinline__ int32_t trunc_i32(double r) {
  return (r > -2147483649.0 && r < 2147483648.0) ? __double2int_rz(r) : INT32_MIN;
}

// ---- coefficients (CutNbins_ColumnImpl::make / compute_cut_coeffs, cut.h:91-182) ----------------------------------
template <typename T>
__global__ void cut_coef_kernel(const ColStats* __restrict__ st, int nbins, int right_closed, CutCoef* __restrict__ coef)
{
  double mn, mx;
  if constexpr (std::is_same<T, double>::value) {
    mn = __longlong_as_double((long long)f64_unimage(st->lo));
    mx = __longlong_as_double((long long)f64_unimage(st->hi));
  } else if constexpr (std::is_same<T, float>::value) {
    mn = (double)__uint_as_float(f32_unimage((u32)st->lo));
    mx = (double)__uint_as_float(f32_unimage((u32)st->hi));
  } else {
    mn = __ll2double_rn((long long)st->lo);
    mx = __ll2double_rn((long long)st->hi);
  }
  CutCoef c{0.0, 0.0, 0, 0};
  if (st->nvalid == 0 || isinf(mn) || isinf(mx)) {
    c.na = 1;                                                  // no valid value, or an infinite one: all NA
  } else if (mn == mx) {
    c.b = (double)((nbins - right_closed) / 2);
  } else {
    // (1 - FLT_EPSILON) * nbins / (max - min); max - min may overflow to inf, and then a = 0
    c.a = __ddiv_rn(__dmul_rn(1.0 - 1.0 / 8388608.0, (double)nbins), __dsub_rn(mx, mn));
    if (right_closed) {
      c.b = __dmul_rn(-c.a, mn);
    } else {
      c.b = __dmul_rn(-c.a, mx);
      c.shift = nbins - 1;
    }
  }
  *coef = c;
}

int launch_cut_coef(const ColStats* d_stats, int stype, int nbins, int right_closed, CutCoef* coef, cudaStream_t s)
{
  return with_stype(stype, "cut() cannot be applied to columns of stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    cut_coef_kernel<T><<<1, 1, 0, s>>>(d_stats, nbins, right_closed, coef);
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  });
}

// ---- equal-width bins ----------------------------------------------------------------------------------------------
template <typename T, typename OrdT, bool GATHER>
__global__ void __launch_bounds__(CUT_THREADS)
cut_emit_kernel(const T* __restrict__ v, int64_t nv, const OrdT* __restrict__ order, int64_t n,
                const CutCoef* __restrict__ coef, int32_t* __restrict__ out)
{
  const CutCoef c = *coef;
  const int64_t stride = (int64_t)gridDim.x * CUT_THREADS * CUT_IPT;
  for (int64_t p0 = (int64_t)blockIdx.x * CUT_THREADS * CUT_IPT + threadIdx.x; p0 < n; p0 += stride) {
    int64_t j[CUT_IPT];
#pragma unroll
    for (int k = 0; k < CUT_IPT; k++) {
      const int64_t p = p0 + k * CUT_THREADS;
      j[k] = p < n ? (GATHER ? (int64_t)order[p] : p) : -1;
    }
    double x[CUT_IPT];
    bool ok[CUT_IPT];
#pragma unroll
    for (int k = 0; k < CUT_IPT; k++) ok[k] = cut_load<T>(v, nv, j[k], x[k]);
#pragma unroll
    for (int k = 0; k < CUT_IPT; k++) {
      const int64_t p = p0 + k * CUT_THREADS;
      if (p >= n) break;
      int32_t bin = INT32_MIN;
      if (ok[k] && !c.na)       // int32 + shift wraps, as the reference's add does on x86-64
        bin = (int32_t)((u32)trunc_i32(__dadd_rn(__dmul_rn(c.a, x[k]), c.b)) + (u32)c.shift);
      out[p] = bin;
    }
  }
}

int launch_cut_emit(const void* v, int stype, int64_t nv, const void* order, int order_is64, int64_t n,
                    const CutCoef* coef, int32_t* out, cudaStream_t s)
{
  return with_stype(stype, "cut() cannot be applied to columns of stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    if (n == 0) return DTB_OK;
    const int grid = grid_for((n + CUT_THREADS * CUT_IPT - 1) / (CUT_THREADS * CUT_IPT), 8);
    if (!order) {
      cut_emit_kernel<T, int32_t, false><<<grid, CUT_THREADS, 0, s>>>((const T*)v, nv, nullptr, n, coef, out);
    } else {
      with_order(order, order_is64, [&](auto o) {
        typedef typename std::remove_cv<typename std::remove_pointer<decltype(o)>::type>::type OrdT;
        cut_emit_kernel<T, OrdT, true><<<grid, CUT_THREADS, 0, s>>>((const T*)v, nv, o, n, coef, out);
      });
    }
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  });
}

// ---- explicit edges (CutBins_ColumnImpl<RIGHT_CLOSED>, cut.h:199-281) ---------------------------------------------
// The reference bisects with v > e (right-closed) or v >= e; the edges strictly increase, so its bin is
// c - 1 with c = #{k : e[k] < v} (right-closed) or #{k : e[k] <= v}, and the value is valid iff 1 <= c <= m - 1.
// c is the partition point of a predicate that holds on a prefix of the edges.  The CTA stages every k-th edge in
// shared memory (ns <= CUT_SMEM_EDGES of them; k = 1 while the edges fit); the sample gives c to within one window
// of k - 1 edges, searched in global memory (the edges stay in L2).  Each search halves a length that depends on
// the edge count only, so a warp's lanes take the same number of steps.
template <bool RC>
__device__ __forceinline__ bool edge_pred(double e, double x) { return RC ? (e < x) : (e <= x); }

template <bool RC>
__device__ __forceinline__ int64_t partition_point(const double* e, int64_t lo, int64_t len, double x) {
  while (len > 1) {
    const int64_t half = len >> 1;
    lo = edge_pred<RC>(e[lo + half], x) ? lo + half : lo;
    len -= half;
  }
  return lo + (edge_pred<RC>(e[lo], x) ? 1 : 0);
}

template <typename T, typename OrdT, bool GATHER, bool RC>
__global__ void __launch_bounds__(CUT_THREADS)
cut_bins_kernel(const T* __restrict__ v, int64_t nv, const OrdT* __restrict__ order, int64_t n,
                const double* __restrict__ edges, int64_t m, int64_t k, int ns, int32_t* __restrict__ out)
{
  extern __shared__ double sample[];
  for (int i = threadIdx.x; i < ns; i += CUT_THREADS) sample[i] = edges[(int64_t)i * k];
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * CUT_THREADS * CUT_IPT;
  for (int64_t p0 = (int64_t)blockIdx.x * CUT_THREADS * CUT_IPT + threadIdx.x; p0 < n; p0 += stride) {
    int64_t j[CUT_IPT];
#pragma unroll
    for (int q = 0; q < CUT_IPT; q++) {
      const int64_t p = p0 + q * CUT_THREADS;
      j[q] = p < n ? (GATHER ? (int64_t)order[p] : p) : -1;
    }
    double x[CUT_IPT];
    bool ok[CUT_IPT];
#pragma unroll
    for (int q = 0; q < CUT_IPT; q++) ok[q] = cut_load<T>(v, nv, j[q], x[q]);
#pragma unroll
    for (int q = 0; q < CUT_IPT; q++) {
      const int64_t p = p0 + q * CUT_THREADS;
      if (p >= n) break;
      int32_t bin = INT32_MIN;
      if (ok[q]) {
        const int64_t cs = partition_point<RC>(sample, 0, ns, x[q]);
        int64_t c = 0;
        if (cs > 0) {                          // sample[cs - 1] = e[(cs - 1) k] holds; e[cs k] (if any) does not
          const int64_t lo = (cs - 1) * k + 1, hi = cs * k < m ? cs * k : m;
          c = hi > lo ? partition_point<RC>(edges, lo, hi - lo, x[q]) : lo;
        }
        if (c >= 1 && c <= m - 1) bin = (int32_t)(c - 1);
      }
      out[p] = bin;
    }
  }
}

int launch_cut_bins(const void* v, int stype, int64_t nv, const void* order, int order_is64, int64_t n,
                    const double* d_edges, int64_t nedges, int right_closed, int32_t* out, cudaStream_t s)
{
  return with_stype(stype, "cut() cannot be applied to columns of stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    if (n == 0) return DTB_OK;
    const int64_t k = (nedges + CUT_SMEM_EDGES - 1) / CUT_SMEM_EDGES;
    const int ns = (int)((nedges + k - 1) / k);
    const size_t smem = sizeof(double) * (size_t)ns;
    const int grid = grid_for((n + CUT_THREADS * CUT_IPT - 1) / (CUT_THREADS * CUT_IPT), 8);
    auto run = [&](auto o, auto gather, auto rc) {
      typedef typename std::remove_cv<typename std::remove_pointer<decltype(o)>::type>::type OrdT;
      cut_bins_kernel<T, OrdT, decltype(gather)::value, decltype(rc)::value><<<grid, CUT_THREADS, smem, s>>>(
          (const T*)v, nv, o, n, d_edges, nedges, k, ns, out);
    };
    auto by_rc = [&](auto o, auto gather) {
      if (right_closed) run(o, gather, std::true_type());
      else              run(o, gather, std::false_type());
    };
    if (!order) by_rc((const int32_t*)nullptr, std::false_type());
    else with_order(order, order_is64, [&](auto o) { by_rc(o, std::true_type()); });
    count_launch();
    DTB_CUDA_CHECK(cudaGetLastError());
    return DTB_OK;
  });
}

}  // namespace dtb
