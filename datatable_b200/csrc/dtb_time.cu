// dtb_time.cu -- the calendar and clock parts of a date32 / time64 column over the positions of a RowIndex: replaces
// YearMonthDay_ColumnImpl, DayOfWeek_ColumnImpl and HourMinSec_ColumnImpl (expr/time/fexpr_year_month_day.cc,
// fexpr_day_of_week.cc, fexpr_hour_min_sec.cc) as dt.time.year() .. nanosecond() evaluate them.
//
//   date32 (int32 days since 1970-01-01)          year, month, day: the proleptic-Gregorian days-to-civil conversion
//                                                  (H. Hinnant, "chrono-Compatible Low-Level Date Algorithms");
//                                                  day_of_week: ISO, Monday = 1 .. Sunday = 7
//   time64 (int64 ns since 1970-01-01T00:00)      the same four through the time64 -> date32 cast (floor division by
//                                                  a day); hour / minute / second / nanosecond: (v mod DAY) / SCALE %
//                                                  MODULO with the floor modulo
//
// The reference computes in int32 / int64 and lets an add wrap where it overflows (days near the ends of the int32
// range, instants near INT64_MIN): every such add here is done on the unsigned word, which wraps the same way.  Every
// divisor is a compile-time constant, so the divisions compile to multiplies.  Row-parallel and bound by HBM: per
// position one index (none for the identity), one value and one int32 out.
#include "dtb_common.cuh"

namespace dtb {

constexpr int TIME_THREADS = 256;
constexpr int TIME_VEC = 4;                // positions per thread per step; the identity path loads them as one vector
constexpr int64_t NS_PER_DAY = 86400ll * 1000000000ll;

__device__ __forceinline__ int32_t add32(int32_t a, int32_t b) { return (int32_t)((u32)a + (u32)b); }
__device__ __forceinline__ int32_t sub32(int32_t a, int32_t b) { return (int32_t)((u32)a - (u32)b); }
__device__ __forceinline__ int32_t mul32(int32_t a, int32_t b) { return (int32_t)((u32)a * (u32)b); }

// CastTime64ToDate32: the day of an instant, rounded toward -inf (value - (DAY - 1) wraps near INT64_MIN), as int32
__device__ __forceinline__ int32_t days_of_time64(int64_t v) {
  if (v < 0) v = (int64_t)((u64)v - (u64)(NS_PER_DAY - 1));
  return (int32_t)(v / NS_PER_DAY);
}

// year (PART 1), month (2) or day (3) of day number z
template <int PART>
__device__ __forceinline__ int32_t civil_part(int32_t z) {
  z = add32(z, 719468);                                        // days since 0000-03-01
  const int32_t era = (z >= 0 ? z : add32(z, -146096)) / 146097;
  const int32_t doe = sub32(z, mul32(era, 146097));          // day of the 400-year era, [0, 146096]
  // doe leaves [0, 146096] only where z wrapped; the arithmetic below wraps there as the reference's does
  const int32_t yoe = sub32(add32(sub32(doe, doe / 1460), doe / 36524), doe / 146096) / 365;
  const int32_t doy = sub32(doe, sub32(add32(mul32(365, yoe), yoe / 4), yoe / 100));
  const int32_t mp = add32(mul32(5, doy), 2) / 153;           // month from March, [0, 11]
  const int32_t m = add32(mp, mp < 10 ? 3 : -9);
  if constexpr (PART == DTB_TIME_YEAR) return add32(add32(yoe, mul32(era, 400)), m <= 2 ? 1 : 0);
  else if constexpr (PART == DTB_TIME_MONTH) return m;
  else return add32(sub32(doy, add32(mul32(153, mp), 2) / 5), 1);
}

// ISO day of the week of day number z.  For z >= -3 the reference's compiled code takes z + 3 as unsigned (it is
// non-negative unless it wraps), so the remainder is the unsigned one.
__device__ __forceinline__ int32_t iso_weekday(int32_t z) {
  return z >= -3 ? (int32_t)(((u32)z + 3u) % 7u) + 1 : (z + 4) % 7 + 7;
}

// PART of a valid element of type T (int32: date32, int64: time64)
template <typename T, int PART>
__device__ __forceinline__ int32_t time_part_of(T v) {
  if constexpr (PART <= DTB_TIME_DAY_OF_WEEK) {
    int32_t z;
    if constexpr (sizeof(T) == 8) z = days_of_time64((int64_t)v);
    else z = (int32_t)v;
    if constexpr (PART == DTB_TIME_DAY_OF_WEEK) return iso_weekday(z);
    else return civil_part<PART>(z);
  } else {
    constexpr int64_t SCALE = PART == DTB_TIME_HOUR ? 3600000000000ll : PART == DTB_TIME_MINUTE ? 60000000000ll :
                              PART == DTB_TIME_SECOND ? 1000000000ll : 1;
    constexpr int64_t MODULO = PART == DTB_TIME_HOUR ? 24 : PART == DTB_TIME_MINUTE || PART == DTB_TIME_SECOND ? 60 :
                               1000000000ll;
    int64_t r = (int64_t)v % NS_PER_DAY;
    if (r < 0) r += NS_PER_DAY;
    return (int32_t)((r / SCALE) % MODULO);
  }
}

template <typename T, int PART>
__device__ __forceinline__ int32_t time_part_or_na(T v) {
  return v == NaOf<T>::v() ? INT32_MIN : time_part_of<T, PART>(v);
}

// Identity: TIME_VEC consecutive elements per thread and step, one vector load and one int4 store when v and out are
// 16-byte aligned (VEC), else element by element.
template <typename T, int PART, bool VEC>
__global__ void __launch_bounds__(TIME_THREADS)
time_part_kernel(const T* __restrict__ v, int64_t n, int32_t* __restrict__ out)
{
  const int64_t nvec = n / TIME_VEC;
  const int64_t stride = (int64_t)gridDim.x * TIME_THREADS;
#pragma unroll 1          // else the compiler derives a trip count with a 64-bit division
  for (int64_t q = (int64_t)blockIdx.x * TIME_THREADS + threadIdx.x; q < nvec; q += stride) {
    T x[TIME_VEC];
    if constexpr (VEC && sizeof(T) == 4) {
      const int4 a = ((const int4*)v)[q];
      x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w;
    } else if constexpr (VEC) {
      const longlong2 a = ((const longlong2*)v)[2 * q], b = ((const longlong2*)v)[2 * q + 1];
      x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y;
    } else {
#pragma unroll
      for (int k = 0; k < TIME_VEC; k++) x[k] = v[q * TIME_VEC + k];
    }
    int32_t r[TIME_VEC];
#pragma unroll
    for (int k = 0; k < TIME_VEC; k++) r[k] = time_part_or_na<T, PART>(x[k]);
    if constexpr (VEC) {
      ((int4*)out)[q] = make_int4(r[0], r[1], r[2], r[3]);
    } else {
#pragma unroll
      for (int k = 0; k < TIME_VEC; k++) out[q * TIME_VEC + k] = r[k];
    }
  }
  const int64_t tail = nvec * TIME_VEC + (int64_t)blockIdx.x * TIME_THREADS + threadIdx.x;
  if (tail < n) out[tail] = time_part_or_na<T, PART>(v[tail]);
}

// Through a RowIndex: an index outside [0, nv) is an NA row, as in dtb_gather.
template <typename T, int PART, typename OrdT>
__global__ void __launch_bounds__(TIME_THREADS)
time_part_gather_kernel(const T* __restrict__ v, int64_t nv, const OrdT* __restrict__ order, int64_t n,
                        int32_t* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * TIME_THREADS * TIME_VEC;
  for (int64_t p0 = (int64_t)blockIdx.x * TIME_THREADS * TIME_VEC + threadIdx.x; p0 < n; p0 += stride) {
    int64_t j[TIME_VEC];
#pragma unroll
    for (int k = 0; k < TIME_VEC; k++) {
      const int64_t p = p0 + k * TIME_THREADS;
      j[k] = p < n ? (int64_t)order[p] : -1;
    }
    T x[TIME_VEC];
#pragma unroll
    for (int k = 0; k < TIME_VEC; k++) x[k] = (j[k] >= 0 && j[k] < nv) ? v[j[k]] : NaOf<T>::v();
#pragma unroll
    for (int k = 0; k < TIME_VEC; k++) {
      const int64_t p = p0 + k * TIME_THREADS;
      if (p < n) out[p] = time_part_or_na<T, PART>(x[k]);
    }
  }
}

template <typename F>
static inline int with_time_part(int part, F&& f) {
  switch (part) {
    case DTB_TIME_YEAR:        return f(std::integral_constant<int, DTB_TIME_YEAR>());
    case DTB_TIME_MONTH:       return f(std::integral_constant<int, DTB_TIME_MONTH>());
    case DTB_TIME_DAY:         return f(std::integral_constant<int, DTB_TIME_DAY>());
    case DTB_TIME_DAY_OF_WEEK: return f(std::integral_constant<int, DTB_TIME_DAY_OF_WEEK>());
    case DTB_TIME_HOUR:        return f(std::integral_constant<int, DTB_TIME_HOUR>());
    case DTB_TIME_MINUTE:      return f(std::integral_constant<int, DTB_TIME_MINUTE>());
    case DTB_TIME_SECOND:      return f(std::integral_constant<int, DTB_TIME_SECOND>());
    case DTB_TIME_NANOSECOND:  return f(std::integral_constant<int, DTB_TIME_NANOSECOND>());
  }
  set_error("unknown time part " + std::to_string(part));
  return DTB_EINVAL;
}

int launch_time_part(int part, const void* v, int stype, int64_t nv, const void* order, int order_is64, int64_t n,
                     int32_t* out, cudaStream_t s)
{
  return with_stype(stype, "time functions cannot be applied to columns of stype ", [&](auto t) {
    typedef typename decltype(t)::type T;
    // date32 runs as int32 and time64 as int64; the caller refuses every other stype, and the clock parts of date32
    if constexpr (std::is_same<T, int32_t>::value || std::is_same<T, int64_t>::value) {
      return with_time_part(part, [&](auto pc) {
        constexpr int P = decltype(pc)::value;
        if constexpr (sizeof(T) == 4 && P > DTB_TIME_DAY_OF_WEEK) {
          set_error("the clock parts need a time64 column");
          return (int)DTB_EINVAL;
        } else {
          if (n == 0) return (int)DTB_OK;
          if (!order) {
            const int grid = grid_for((n / TIME_VEC + TIME_THREADS - 1) / TIME_THREADS, 8);
            if ((((uintptr_t)v | (uintptr_t)out) & 15) == 0)
              time_part_kernel<T, P, true><<<grid, TIME_THREADS, 0, s>>>((const T*)v, n, out);
            else
              time_part_kernel<T, P, false><<<grid, TIME_THREADS, 0, s>>>((const T*)v, n, out);
          } else {
            const int grid = grid_for((n + TIME_THREADS * TIME_VEC - 1) / (TIME_THREADS * TIME_VEC), 8);
            with_order(order, order_is64, [&](auto o) {
              typedef typename std::remove_cv<typename std::remove_pointer<decltype(o)>::type>::type OrdT;
              time_part_gather_kernel<T, P, OrdT><<<grid, TIME_THREADS, 0, s>>>((const T*)v, nv, o, n, out);
            });
          }
          count_launch();
          DTB_CUDA_CHECK(cudaGetLastError());
          return (int)DTB_OK;
        }
      });
    } else {
      set_error("time functions need a date32 or time64 column, got stype " + std::to_string(stype));
      return (int)DTB_EINVAL;
    }
  });
}

}  // namespace dtb
