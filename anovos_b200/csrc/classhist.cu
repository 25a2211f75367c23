// monotonic_binning (reference data_transformer/transformers.py:294-425) tries every bin count n = 20 .. 3 of a column and
// groups the rows of each try by bin and label class.  All 18 candidate models of a column are runs of consecutive slots
// of ONE sorted union of their native thresholds (the host maps slots to bins per model), so this pass counts the rows of
// each (union slot, label class) in one read of the column, its validity and the two class bitmaps.
//
// Grid (row tiles, columns), four rows per lane with 128-bit loads (quad.cuh).  For a valid, non-NaN value x the slot is
// 1 + #(theta < x), found by a branch-free binary search in the column's thresholds staged in shared memory; a NaN value
// has its own slot n_thr + 2 and a null value slot 0.  The class is event / non-event / null label.  Valid -inf and +inf
// values are also counted per column, whatever their class: the host needs them to tell which bins average to NaN.
//
// Every warp bumps its own shared-memory copy of the counters; the copies are summed and added to the uint64 counts once
// per CTA (and every CH_FLUSH_TILES row tiles, so a uint32 counter never wraps).  The counts are integers, so the result
// does not depend on the order the CTAs run in.
#include "quad.cuh"

namespace anv {

constexpr int CH_MAX_THR = 256;                                  // largest threshold union of one column
constexpr int CH_MAX_COUNTERS = 3 * (CH_MAX_THR + 3) + 2;        // ANV_CLASS_HIST_COUNTERS(CH_MAX_THR)
constexpr int CH_WARPS = ANV_BLOCK / 32;
constexpr int64_t CH_FLUSH_TILES = 1 << 20;                      // tiles of 1024 rows: a warp adds < 2^28 per counter

template <typename T> struct ChTraits;
template <> struct ChTraits<float> {
  using Bits = uint32_t;
  __device__ static bool nan(float x) { return x != x; }
  __device__ static int inf(float x) { return x == -INFINITY ? 1 : (x == INFINITY ? 2 : 0); }
};
template <> struct ChTraits<double> {
  using Bits = unsigned long long;
  __device__ static bool nan(double x) { return x != x; }
  __device__ static int inf(double x) { return x == -(double)INFINITY ? 1 : (x == (double)INFINITY ? 2 : 0); }
};
template <> struct ChTraits<int32_t> {
  using Bits = uint32_t;
  __device__ static bool nan(int32_t) { return false; }
  __device__ static int inf(int32_t) { return 0; }
};
template <> struct ChTraits<int64_t> {
  using Bits = unsigned long long;
  __device__ static bool nan(int64_t) { return false; }
  __device__ static int inf(int64_t) { return 0; }
};

__device__ __forceinline__ void ch_flush(uint32_t (*s_cnt)[CH_MAX_COUNTERS], int n_counters, unsigned long long* counts) {
  __syncthreads();
  for (int i = threadIdx.x; i < n_counters; i += blockDim.x) {
    uint32_t s = 0;
#pragma unroll
    for (int w = 0; w < CH_WARPS; ++w) {
      s += s_cnt[w][i];
      s_cnt[w][i] = 0;
    }
    if (s) atomicAdd(counts + i, (unsigned long long)s);
  }
  __syncthreads();
}

template <typename T>
__device__ __forceinline__ void class_hist_column(const anv_column_t& col, const anv_class_hist_spec_t& sp,
                                                  const uint32_t* __restrict__ ev_words, const uint32_t* __restrict__ nev_words,
                                                  int64_t n_rows, T* s_thr, uint32_t (*s_cnt)[CH_MAX_COUNTERS]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n_thr = sp.n_thr;
  const int n_slots = n_thr + 3;                       // null, n_thr + 1 value slots, NaN
  const int n_counters = ANV_CLASS_HIST_COUNTERS(n_thr);
  for (int i = threadIdx.x; i < n_thr; i += blockDim.x) s_thr[i] = __ldg((const T*)sp.thresholds + i);
  for (int i = threadIdx.x; i < n_counters; i += blockDim.x)
#pragma unroll
    for (int w = 0; w < CH_WARPS; ++w) s_cnt[w][i] = 0;
  __syncthreads();
  uint32_t* __restrict__ cnt = s_cnt[warp];
  const T* __restrict__ data = (const T*)col.data;
  const int64_t step = (int64_t)gridDim.x * QUAD_ROWS_PER_CTA;
  int64_t tiles = 0;
  // the trip count is uniform per CTA, so the periodic flush may synchronise the block
  for (int64_t t0 = (int64_t)blockIdx.x * QUAD_ROWS_PER_CTA; t0 < n_rows; t0 += step) {
    const int64_t r0 = t0 + (int64_t)warp * QUAD_ROWS_PER_WARP;
    if (r0 < n_rows) {                                   // warp-uniform
      const uint32_t vb = quad_valid_bits(col.validity, r0, n_rows, lane);
      const uint32_t eb = quad_valid_bits(ev_words, r0, n_rows, lane);
      const uint32_t nb = quad_valid_bits(nev_words, r0, n_rows, lane);
      const int64_t r = r0 + lane * QUAD_ROWS_PER_LANE;
      if (r < n_rows) {
        T e[4];
        load_quad<T>(data, r, n_rows, e);
        int base[4] = {0, 0, 0, 0};
        for (int len = n_thr; len > 1;) {              // #(theta < x) as a lower bound; trip count depends on n_thr only
          const int half = len >> 1;
#pragma unroll
          for (int k = 0; k < 4; ++k) base[k] = s_thr[base[k] + half] < e[k] ? base[k] + half : base[k];
          len -= half;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (r + k >= n_rows) continue;
          const int below = n_thr > 0 ? base[k] + (s_thr[base[k]] < e[k] ? 1 : 0) : 0;
          const bool valid = (vb >> k) & 1u;
          const int slot = !valid ? 0 : (ChTraits<T>::nan(e[k]) ? n_thr + 2 : 1 + below);
          const int cls = ((eb >> k) & 1u) ? 0 : (((nb >> k) & 1u) ? 1 : 2);
          atomicAdd(cnt + cls * n_slots + slot, 1u);
          const int inf = valid ? ChTraits<T>::inf(e[k]) : 0;
          if (inf) atomicAdd(cnt + 3 * n_slots + inf - 1, 1u);
        }
      }
    }
    if (++tiles == CH_FLUSH_TILES) {
      tiles = 0;
      ch_flush(s_cnt, n_counters, sp.counts);
    }
  }
  ch_flush(s_cnt, n_counters, sp.counts);
}

__global__ void __launch_bounds__(ANV_BLOCK) class_hist_kernel(const anv_column_t* __restrict__ cols,
                                                               const anv_class_hist_spec_t* __restrict__ specs,
                                                               const uint32_t* __restrict__ ev_words,
                                                               const uint32_t* __restrict__ nev_words, int64_t n_rows) {
  __shared__ __align__(16) unsigned long long s_thr[CH_MAX_THR];
  __shared__ uint32_t s_cnt[CH_WARPS][CH_MAX_COUNTERS];
  const int c = blockIdx.y;
  const anv_column_t col = cols[c];
  const anv_class_hist_spec_t sp = specs[c];
  // the branches are uniform per CTA
  if (sp.n_thr < 0 || sp.n_thr > CH_MAX_THR || (sp.n_thr > 0 && !sp.thresholds) || !sp.counts) return;
  switch (col.dtype) {
    case ANV_F32: class_hist_column<float>(col, sp, ev_words, nev_words, n_rows, reinterpret_cast<float*>(s_thr), s_cnt); break;
    case ANV_F64: class_hist_column<double>(col, sp, ev_words, nev_words, n_rows, reinterpret_cast<double*>(s_thr), s_cnt); break;
    case ANV_I32: class_hist_column<int32_t>(col, sp, ev_words, nev_words, n_rows, reinterpret_cast<int32_t*>(s_thr), s_cnt); break;
    case ANV_I64: class_hist_column<int64_t>(col, sp, ev_words, nev_words, n_rows, reinterpret_cast<int64_t*>(s_thr), s_cnt); break;
    default: break;
  }
}

int check_common(const void* cols, int n_cols, int64_t n_rows);

}  // namespace anv

using namespace anv;

extern "C" int anv_class_hist_max_thresholds() { return CH_MAX_THR; }

extern "C" int anv_class_hist(const anv_column_t* cols, const anv_class_hist_spec_t* specs, const uint32_t* event_words,
                              const uint32_t* nonevent_words, int n_cols, int64_t n_rows, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0 || n_rows == 0) return ANV_OK;
  if (!specs || !event_words || !nonevent_words) {
    set_error("anv_class_hist: specs and both class bitmaps are required");
    return ANV_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(quad_grid_x(n_rows, n_cols), (unsigned)n_cols);
  class_hist_kernel<<<grid, ANV_BLOCK, 0, st>>>(cols, specs, event_words, nonevent_words, n_rows);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}
