// Four-rows-per-lane streaming helpers of the per-column transform passes (impute.cu, scale.cu, encode.cu, transform.cu,
// invalid.cu).
//
// A warp covers 128 consecutive rows per step, four per lane, so every lane moves its values with 128-bit loads and
// stores (two for 8-byte types).  The validity word of 32 rows is loaded once, by one of the first four lanes, and
// handed to the eight lanes that cover its rows by a shuffle.
#pragma once
#include "common.cuh"

namespace anv {

constexpr int QUAD_ROWS_PER_LANE = 4;
constexpr int QUAD_ROWS_PER_WARP = 32 * QUAD_ROWS_PER_LANE;
constexpr int QUAD_ROWS_PER_CTA = ANV_BLOCK * QUAD_ROWS_PER_LANE;

// Four consecutive values from row r (r % 4 == 0) as 128-bit loads; a quad that crosses n_rows reads its live rows only.
template <typename T> __device__ __forceinline__ void load_quad(const T* __restrict__ p, int64_t r, int64_t n_rows, T (&e)[4]) {
  if (r + 4 <= n_rows) {
    if constexpr (sizeof(T) == 4) {
      unpack<T>(ldg_stream(p + r), e);
    } else {
      T a[2], b[2];
      unpack<T>(ldg_stream(p + r), a);
      unpack<T>(ldg_stream(p + r + 2), b);
      e[0] = a[0]; e[1] = a[1]; e[2] = b[0]; e[3] = b[1];
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) e[k] = (r + k < n_rows) ? p[r + k] : T(0);
  }
}

// Four values to row r of an output padded to a multiple of 4 rows: always whole 128-bit stores.
template <typename U> __device__ __forceinline__ void store_quad(U* __restrict__ p, int64_t r, const U (&e)[4]) {
  if constexpr (sizeof(U) == 4) {
    uint4 q;
    q.x = reinterpret_cast<const uint32_t&>(e[0]); q.y = reinterpret_cast<const uint32_t&>(e[1]);
    q.z = reinterpret_cast<const uint32_t&>(e[2]); q.w = reinterpret_cast<const uint32_t&>(e[3]);
    __stcs(reinterpret_cast<uint4*>(p + r), q);
  } else {
    ulonglong2 a, b;
    a.x = reinterpret_cast<const unsigned long long&>(e[0]); a.y = reinterpret_cast<const unsigned long long&>(e[1]);
    b.x = reinterpret_cast<const unsigned long long&>(e[2]); b.y = reinterpret_cast<const unsigned long long&>(e[3]);
    __stcs(reinterpret_cast<ulonglong2*>(p + r), a);
    __stcs(reinterpret_cast<ulonglong2*>(p + r + 2), b);
  }
}

// The 4 validity bits of the lane's quad: the warp's 128 rows span 4 bitmap words, loaded by lanes 0-3 and shuffled to
// the 8 lanes each word covers.  NULL bitmap: every row valid.  Called by the whole warp (r0 is warp-uniform).
__device__ __forceinline__ uint32_t quad_valid_bits(const uint32_t* __restrict__ validity, int64_t r0, int64_t n_rows, int lane) {
  if (!validity) return 0xFu;
  const int64_t w = r0 / 32 + lane;
  const int64_t n_words = (n_rows + 31) / 32;
  uint32_t word = (lane < 4 && w < n_words) ? __ldg(validity + w) : 0u;
  word = __shfl_sync(ANV_FULL, word, lane >> 3);
  return (word >> (4 * (lane & 7))) & 0xFu;
}

// The inverse of quad_valid_bits: the 8 lanes of each 32-row word OR their 4 keep bits together and the word's first
// lane stores it to the output bitmap.  Called by the whole warp (r0 is warp-uniform).
__device__ __forceinline__ void store_quad_valid_bits(uint32_t* __restrict__ out, uint32_t keep, int64_t r0, int64_t n_rows, int lane) {
  uint32_t word = keep << (4 * (lane & 7));
  word |= __shfl_xor_sync(ANV_FULL, word, 1);
  word |= __shfl_xor_sync(ANV_FULL, word, 2);
  word |= __shfl_xor_sync(ANV_FULL, word, 4);
  const int64_t w = r0 / 32 + (lane >> 3);
  if ((lane & 7) == 0 && w * 32 < n_rows) out[w] = word;
}

// Adds the warp's sum of n to *counter with one atomic from lane 0, none when the sum is 0.  Called by the whole warp.
__device__ __forceinline__ void warp_add_count(unsigned long long* __restrict__ counter, unsigned long long n, int lane) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_down_sync(ANV_FULL, n, o);
  if (lane == 0 && n) atomicAdd(counter, n);
}

// Row tiles per column of a (row tiles, columns) grid: enough CTAs for ~16 per SM across the launch, never more than
// the rows need.
inline unsigned quad_grid_x(int64_t n_rows, int n_cols) {
  int sms = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t need = (n_rows + QUAD_ROWS_PER_CTA - 1) / QUAD_ROWS_PER_CTA;
  int64_t want = ((int64_t)sms * 16 + n_cols - 1) / n_cols;
  if (want < 1) want = 1;
  return (unsigned)(need < want ? need : want);
}

}  // namespace anv
