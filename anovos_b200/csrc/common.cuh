// Shared device helpers for libanovos_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <limits.h>
#include <float.h>

#include "../../include/anovos_b200.h"

#define ANV_BLOCK 256           // threads per CTA in the streaming kernels
#define ANV_WARPS (ANV_BLOCK / 32)
#define ANV_FULL 0xffffffffu

namespace anv {

// ---- error plumbing (host) ---------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
#define ANV_CUDA(call)                                   \
  do {                                                   \
    cudaError_t _e = (call);                             \
    if (_e != cudaSuccess) return anv::cuda_fail(_e, #call); \
  } while (0)

// ---- per-dtype traits --------------------------------------------------------------
template <typename T> struct Traits;
template <> struct Traits<float> {
  static constexpr int VEC = 4;
  using Vec = float4;
  __device__ static float lowest() { return -INFINITY; }
  __device__ static float highest() { return INFINITY; }
  __device__ static float first_slot() { return __int_as_float(0x7fc00000); }
  __device__ static double to_double(float v) { return (double)v; }
  __device__ static bool is_nan(float v) { return v != v; }
};
template <> struct Traits<double> {
  static constexpr int VEC = 2;
  using Vec = double2;
  __device__ static double lowest() { return -INFINITY; }
  __device__ static double highest() { return INFINITY; }
  __device__ static double first_slot() { return __longlong_as_double(0x7ff8000000000000ll); }
  __device__ static double to_double(double v) { return v; }
  __device__ static bool is_nan(double v) { return v != v; }
};
template <> struct Traits<int32_t> {
  static constexpr int VEC = 4;
  using Vec = int4;
  __device__ static int32_t first_slot() { return INT_MIN; }
  __device__ static int32_t lowest() { return INT_MIN; }
  __device__ static int32_t highest() { return INT_MAX; }
  __device__ static double to_double(int32_t v) { return (double)v; }
  __device__ static bool is_nan(int32_t) { return false; }
};
template <> struct Traits<int64_t> {
  static constexpr int VEC = 2;
  using Vec = longlong2;
  __device__ static int64_t first_slot() { return LLONG_MIN; }
  __device__ static int64_t lowest() { return LLONG_MIN; }
  __device__ static int64_t highest() { return LLONG_MAX; }
  __device__ static double to_double(int64_t v) { return (double)v; }
  __device__ static bool is_nan(int64_t) { return false; }
};

// 128-bit streaming load: read-only path, do not allocate in L1 (data is touched once).
__device__ __forceinline__ uint4 ldg_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::128B.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

template <typename T> __device__ __forceinline__ void unpack(const uint4& q, T (&e)[Traits<T>::VEC]);
template <> __device__ __forceinline__ void unpack<float>(const uint4& q, float (&e)[4]) {
  e[0] = __uint_as_float(q.x); e[1] = __uint_as_float(q.y);
  e[2] = __uint_as_float(q.z); e[3] = __uint_as_float(q.w);
}
template <> __device__ __forceinline__ void unpack<int32_t>(const uint4& q, int32_t (&e)[4]) {
  e[0] = (int32_t)q.x; e[1] = (int32_t)q.y; e[2] = (int32_t)q.z; e[3] = (int32_t)q.w;
}
template <> __device__ __forceinline__ void unpack<double>(const uint4& q, double (&e)[2]) {
  e[0] = __hiloint2double((int)q.y, (int)q.x);
  e[1] = __hiloint2double((int)q.w, (int)q.z);
}
template <> __device__ __forceinline__ void unpack<int64_t>(const uint4& q, int64_t (&e)[2]) {
  e[0] = (int64_t)(((uint64_t)q.y << 32) | q.x);
  e[1] = (int64_t)(((uint64_t)q.w << 32) | q.z);
}

__device__ __forceinline__ double shfl_down_d(double v, int d) {
  int lo = __double2loint(v), hi = __double2hiint(v);
  lo = __shfl_down_sync(ANV_FULL, lo, d);
  hi = __shfl_down_sync(ANV_FULL, hi, d);
  return __hiloint2double(hi, lo);
}
__device__ __forceinline__ int64_t shfl_down_ll(int64_t v, int d) {
  return (int64_t)__shfl_down_sync(ANV_FULL, (unsigned long long)v, d);
}

// Pebay / Chan pairwise merge of (n, mean, M2, M3, M4): the algebra Spark's
// CentralMomentAgg.merge uses.  Deterministic given the merge order.
struct Central {
  double n, mean, m2, m3, m4;
};
__host__ __device__ __forceinline__ Central merge_central(const Central& a, const Central& b) {
  if (b.n == 0.0) return a;
  if (a.n == 0.0) return b;
  Central r;
  const double n = a.n + b.n;
  const double d = b.mean - a.mean;
  const double dn = d / n;
  const double dn2 = dn * dn;
  r.n = n;
  r.mean = a.mean + dn * b.n;
  const double ab = a.n * b.n;
  r.m2 = a.m2 + b.m2 + d * dn * ab;
  r.m3 = a.m3 + b.m3 + d * dn2 * ab * (a.n - b.n) + 3.0 * dn * (a.n * b.m2 - b.n * a.m2);
  r.m4 = a.m4 + b.m4 + d * dn * dn2 * ab * (a.n * a.n - ab + b.n * b.n) +
         6.0 * dn2 * (a.n * a.n * b.m2 + b.n * b.n * a.m2) + 4.0 * dn * (a.n * b.m3 - b.n * a.m3);
  return r;
}

}  // namespace anv
