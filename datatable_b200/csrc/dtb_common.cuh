// dtb_common.cuh -- device-side helpers shared by all kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <type_traits>
#include "dtb_internal.h"

namespace dtb {

constexpr int NUM_SMS = 132;                  // H100 SXM

// radix pass geometry (dtb_radix.cu; the fused statistics kernel of dtb_stats.cu counts by the same tiles)
constexpr int PASS_THREADS = 256;
constexpr int PASS_IPT = 16;
constexpr int PASS_TILE = PASS_THREADS * PASS_IPT;            // 4096 rows
constexpr int CHUNK_TILES = 16;
constexpr int CHUNK_ROWS = PASS_TILE * CHUNK_TILES;           // 65536 rows per count CTA

typedef unsigned long long u64;
typedef unsigned int u32;

// ---- NA sentinels (stype.h:186-197) ---------------------------------------
template <typename T> struct NaOf;
template <> struct NaOf<int8_t>  { static __host__ __device__ int8_t  v() { return INT8_MIN;  } };
template <> struct NaOf<int16_t> { static __host__ __device__ int16_t v() { return INT16_MIN; } };
template <> struct NaOf<int32_t> { static __host__ __device__ int32_t v() { return INT32_MIN; } };
template <> struct NaOf<int64_t> { static __host__ __device__ int64_t v() { return INT64_MIN; } };

// ---- order-preserving unsigned image of a float (sort.cc:778-845, ASC form) ----
__device__ __forceinline__ bool f32_image(u32 t, u64& img) {
  const u32 EXP = 0x7F800000u, SIG = 0x007FFFFFu, SBT = 0x80000000u;
  if ((t & EXP) == EXP && (t & SIG) != 0) return false;          // NaN == NA
  img = (u32)(t ^ (SBT | (0u - (t >> 31))));
  return true;
}
__device__ __forceinline__ bool f64_image(u64 t, u64& img) {
  const u64 EXP = 0x7FF0000000000000ull, SIG = 0x000FFFFFFFFFFFFFull, SBT = 0x8000000000000000ull;
  if ((t & EXP) == EXP && (t & SIG) != 0) return false;
  img = t ^ (SBT | (0ull - (t >> 63)));
  return true;
}
__device__ __forceinline__ u32 f32_unimage(u32 img) {
  return (img & 0x80000000u) ? (img ^ 0x80000000u) : ~img;
}
__device__ __forceinline__ u64 f64_unimage(u64 img) {
  return (img & 0x8000000000000000ull) ? (img ^ 0x8000000000000000ull) : ~img;
}

// Raw element -> (valid, u) where u is the sign-extended integer or the float image.
template <typename T> struct RawKey;
#define DTB_RAWKEY_INT(T)                                                        \
  template <> struct RawKey<T> {                                                 \
    typedef T load_t;                                                            \
    static __device__ __forceinline__ bool get(T t, u64& u) {                    \
      u = (u64)(int64_t)t; return t != NaOf<T>::v(); }                           \
  };
DTB_RAWKEY_INT(int8_t) DTB_RAWKEY_INT(int16_t) DTB_RAWKEY_INT(int32_t) DTB_RAWKEY_INT(int64_t)
#undef DTB_RAWKEY_INT
template <> struct RawKey<float> {
  typedef u32 load_t;
  static __device__ __forceinline__ bool get(u32 t, u64& u) { return f32_image(t, u); }
};
template <> struct RawKey<double> {
  typedef u64 load_t;
  static __device__ __forceinline__ bool get(u64 t, u64& u) { return f64_image(t, u); }
};

// T's NA as stored: the integer sentinel, or the quiet NaN every kernel writes for a float NA
template <typename T> __host__ __device__ __forceinline__ typename RawKey<T>::load_t raw_na() {
  typedef typename RawKey<T>::load_t O;
  if constexpr (std::is_same<T, float>::value) return (O)0x7FC00000u;
  else if constexpr (std::is_same<T, double>::value) return (O)0x7FF8000000000000ull;
  else return NaOf<T>::v();
}

// The unsigned word of T's width: kernels that only move elements (gather, first / last) run one instance per width
template <typename T>
using bits_t = typename std::conditional<sizeof(T) == 1, uint8_t, typename std::conditional<sizeof(T) == 2, uint16_t,
               typename std::conditional<sizeof(T) == 4, u32, u64>::type>::type>::type;

// x = NA ? na_value : (((desc ? edge - u : u - edge) >> cshift) + inc)
__device__ __forceinline__ u64 norm_apply(bool valid, u64 u, const KeyNorm& k) {
  if (!valid) return k.na_value;
  u64 d = k.desc ? (k.edge - u) : (u - k.edge);
  return (d >> k.cshift) + k.inc;
}

// Runtime-typed load used by the multi-column compose kernel.
__device__ __forceinline__ u64 norm_load_dynamic(const KeyNorm& k, int64_t i) {
  u64 u = 0; bool valid = true;
  switch (k.stype) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8:
      valid = RawKey<int8_t>::get(((const int8_t*)k.data)[i], u); break;
    case DTB_STYPE_INT16:
      valid = RawKey<int16_t>::get(((const int16_t*)k.data)[i], u); break;
    case DTB_STYPE_INT32: case DTB_STYPE_DATE32:
      valid = RawKey<int32_t>::get(((const int32_t*)k.data)[i], u); break;
    case DTB_STYPE_INT64: case DTB_STYPE_TIME64:
      valid = RawKey<int64_t>::get(((const int64_t*)k.data)[i], u); break;
    case DTB_STYPE_FLOAT32:
      valid = RawKey<float>::get(((const u32*)k.data)[i], u); break;
    case DTB_STYPE_FLOAT64:
      valid = RawKey<double>::get(((const u64*)k.data)[i], u); break;
  }
  return norm_apply(valid, u, k);
}

// ---- key sources for the radix kernels ---------------------------------------
// load_raw / norm are split so that a kernel can issue all the loads of a tile before it touches any of
// them (with load() alone ptxas reused one register for the raw element and serialised the 16 loads of
// the scatter pass behind one another).
// Packed keys of InT (1, 2, 4 or 8 bytes: the radix passes store only the key bits later passes read, in the
// narrowest word that holds them), widened to the pass's KeyT.
template <typename InT, typename KeyT = InT>
struct PackedSrc {
  typedef InT raw_t;
  static constexpr bool packed = true;
  const InT* p;
  __device__ __forceinline__ KeyT load(int64_t i) const { return (KeyT)p[i]; }
  __device__ __forceinline__ raw_t load_raw(int64_t i) const { return p[i]; }
  __device__ __forceinline__ KeyT norm(raw_t r) const { return (KeyT)r; }
  __host__ KeyNorm key_norm() const { KeyNorm z; memset(&z, 0, sizeof(z)); return z; }   // packed keys carry no normalisation
};

// Raw column normalised on the fly.  Columns of at most 32 bits producing 32-bit keys take an
// all-32-bit path (the u64 arithmetic of the general form costs ~10 extra instructions per row).
template <typename T> struct Raw32;        // (valid, u32 image) for <= 32-bit raw types
#define DTB_RAW32_INT(T)                                                          \
  template <> struct Raw32<T> {                                                   \
    static constexpr bool ok = true;                                              \
    static __device__ __forceinline__ bool get(T t, u32& u) { u = (u32)(int32_t)t; return t != NaOf<T>::v(); } };
DTB_RAW32_INT(int8_t) DTB_RAW32_INT(int16_t) DTB_RAW32_INT(int32_t)
#undef DTB_RAW32_INT
template <> struct Raw32<float> {
  static constexpr bool ok = true;
  static __device__ __forceinline__ bool get(u32 t, u32& u) {
    const u32 EXP = 0x7F800000u, SIG = 0x007FFFFFu, SBT = 0x80000000u;
    u = t ^ (SBT | (0u - (t >> 31)));
    return !((t & EXP) == EXP && (t & SIG) != 0);
  } };
template <> struct Raw32<int64_t> { static constexpr bool ok = false; static __device__ bool get(int64_t, u32&) { return false; } };
template <> struct Raw32<double>  { static constexpr bool ok = false; static __device__ bool get(u64, u32&) { return false; } };

template <typename T, typename KeyT>
struct RawSrc {
  const typename RawKey<T>::load_t* p;
  KeyNorm k;
  u32 edge32, na32, inc32;
  __host__ void init(const KeyNorm& kn) {
    p = (const typename RawKey<T>::load_t*)kn.data; k = kn;
    edge32 = (u32)kn.edge; na32 = (u32)kn.na_value; inc32 = (u32)kn.inc;
  }
  typedef typename RawKey<T>::load_t raw_t;
  static constexpr bool packed = false;
  __host__ const KeyNorm& key_norm() const { return k; }
  __device__ __forceinline__ raw_t load_raw(int64_t i) const { return p[i]; }
  __device__ __forceinline__ KeyT norm(raw_t r) const {
    if constexpr (Raw32<T>::ok && sizeof(KeyT) == 4) {
      u32 u; const bool valid = Raw32<T>::get(r, u);
      const u32 d = k.desc ? (edge32 - u) : (u - edge32);
      return valid ? ((d >> k.cshift) + inc32) : na32;
    } else {
      u64 u; const bool valid = RawKey<T>::get(r, u);
      return (KeyT)norm_apply(valid, u, k);
    }
  }
  __device__ __forceinline__ KeyT load(int64_t i) const { return norm(load_raw(i)); }
};

// ---- relaxed gpu-scope accesses for look-back status words ---------------------
__device__ __forceinline__ u64 ld_relaxed_u64(const u64* p) {
  u64 v; asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_relaxed_u64(u64* p, u64 v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

// The v in [lo, hi] whose rows occupy slot s: the last v with b[v] <= s (b = exclusive scan of the rows per v, so
// b[lo] <= s; an empty v shares its b with the next one and is never the last).
__device__ __forceinline__ u32 slot_owner(const u32* b, u32 lo, u32 hi, u32 s) {
  while (lo < hi) { const u32 mid = (lo + hi + 1) >> 1; if (b[mid] <= s) lo = mid; else hi = mid - 1; }
  return lo;
}

// The group that holds sorted position p: the last g in [0, ng) with offsets[g] <= p (offsets[0] <= p).
__device__ __forceinline__ int64_t group_of(const int32_t* offsets, int64_t ng, int64_t p) {
  int64_t lo = 0, hi = ng;
  while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if ((int64_t)offsets[mid] <= p) lo = mid; else hi = mid; }
  return lo;
}

// out[g] = a result of stype out_stype (bits: its bit pattern, a float32's in the low word), or that stype's NA
// (stype.h:186-197)
__device__ __forceinline__ void store_result(void* out, int out_stype, int64_t g, bool valid, u64 bits) {
  switch (out_stype) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8:
      ((int8_t*)out)[g] = valid ? (int8_t)bits : INT8_MIN; break;
    case DTB_STYPE_INT16: ((int16_t*)out)[g] = valid ? (int16_t)bits : INT16_MIN; break;
    case DTB_STYPE_INT32: case DTB_STYPE_DATE32:
      ((int32_t*)out)[g] = valid ? (int32_t)bits : INT32_MIN; break;
    case DTB_STYPE_INT64: case DTB_STYPE_TIME64:
      ((int64_t*)out)[g] = valid ? (int64_t)bits : INT64_MIN; break;
    case DTB_STYPE_FLOAT32: ((u32*)out)[g] = valid ? (u32)bits : raw_na<float>(); break;
    case DTB_STYPE_FLOAT64: ((u64*)out)[g] = valid ? bits : raw_na<double>(); break;
  }
}

// out[g] = r rounded to out_stype (float32 or float64), or NA
__device__ __forceinline__ void store_float(void* out, int out_stype, int64_t g, bool valid, double r) {
  store_result(out, out_stype, g, valid,
               out_stype == DTB_STYPE_FLOAT32 ? (u64)__float_as_uint((float)r) : (u64)__double_as_longlong(r));
}

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m;
}

static inline int stype_bytes(int st) {
  switch (st) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8: return 1;
    case DTB_STYPE_INT16: return 2;
    case DTB_STYPE_INT32: case DTB_STYPE_FLOAT32: case DTB_STYPE_DATE32: return 4;
    case DTB_STYPE_INT64: case DTB_STYPE_FLOAT64: case DTB_STYPE_TIME64: return 8;
    default: return 0;
  }
}

// ---- host-side launch helpers --------------------------------------------------
// CTAs of a grid-stride loop that wants `blocks` of them: at least 1, at most per_sm per SM
static inline int grid_for(int64_t blocks, int per_sm) {
  return (int)(blocks > NUM_SMS * per_sm ? NUM_SMS * per_sm : (blocks < 1 ? 1 : blocks));
}

template <typename T> struct TypeTag { typedef T type; };

// f(TypeTag<T>()) with T the C++ type of an element of stype st: BOOL runs as INT8, DATE32 as INT32 and TIME64 as
// INT64.  Any other stype fails with DTB_ENOTIMPL and the error `what` followed by the stype's number.
template <typename F>
static inline int with_stype(int st, const char* what, F&& f) {
  switch (st) {
    case DTB_STYPE_BOOL: case DTB_STYPE_INT8:    return f(TypeTag<int8_t>());
    case DTB_STYPE_INT16:                        return f(TypeTag<int16_t>());
    case DTB_STYPE_INT32: case DTB_STYPE_DATE32: return f(TypeTag<int32_t>());
    case DTB_STYPE_INT64: case DTB_STYPE_TIME64: return f(TypeTag<int64_t>());
    case DTB_STYPE_FLOAT32:                      return f(TypeTag<float>());
    case DTB_STYPE_FLOAT64:                      return f(TypeTag<double>());
  }
  set_error(what + std::to_string(st));
  return DTB_ENOTIMPL;
}

// f(order) with the RowIndex typed by its width: const int32_t* or const int64_t*
template <typename F>
static inline void with_order(const void* order, int order_is64, F&& f) {
  if (order_is64) f((const int64_t*)order);
  else            f((const int32_t*)order);
}

}  // namespace dtb
