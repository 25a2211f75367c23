// The scaling transformers z_standardization, IQR_standardization and normalization (reference
// data_transformer/transformers.py:965-1366): one streaming pass per column writes the scaled column.
//
// Grid (row tiles, columns), four rows per lane with 128-bit loads and stores (quad.cuh).  Per row, in IEEE double with
// every operation rounded on its own (no FMA contraction, no reciprocal multiply), so the output is bit-identical to the
// same formula evaluated in NumPy:
//   DIV     out = (double(x) - a) / b            z_standardization (a, b) = (mean, stddev); IQR (p50, p75 - p25)
//   AFFINE  out = (double(x) - a) * b + c        MinMaxScalerModel (min, (max - min) scale, lo)
//   CONST   out = c                              MinMaxScalerModel of a zero scale: (hi + lo) / 2
// then rounded to nearest float for an F32 output.  NAN_TO_NULL (normalization: MinMaxScalerModel keeps NaN, and the
// reference then turns NaN results into null) makes a row null where its input or its result is NaN.  Null rows are
// written as 0, so every output byte is deterministic.
//
// NAN_TO_NULL also writes the output bitmap: each lane tests its quad, the 8 lanes of a word OR their nibbles together
// and the word's first lane writes it.  Null counts of the output: one atomic per warp.
#include "quad.cuh"

namespace anv {

__device__ __forceinline__ double scale_value(double x, int mode, double a, double b, double c) {
  if (mode == ANV_SCALE_DIV) return __ddiv_rn(__dsub_rn(x, a), b);
  if (mode == ANV_SCALE_AFFINE) return __dadd_rn(__dmul_rn(__dsub_rn(x, a), b), c);
  return c;
}

template <typename U> __device__ __forceinline__ U narrow(double v);
template <> __device__ __forceinline__ double narrow<double>(double v) { return v; }
template <> __device__ __forceinline__ float narrow<float>(double v) { return __double2float_rn(v); }

template <typename T, typename U, bool NAN_TO_NULL>
__device__ __forceinline__ void scale_column(const T* __restrict__ src, const uint32_t* __restrict__ validity, U* __restrict__ dst,
                                             uint32_t* __restrict__ out_valid, unsigned long long* __restrict__ n_null,
                                             const anv_scale_spec_t& sp, int64_t n_rows) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t step = (int64_t)gridDim.x * QUAD_ROWS_PER_CTA;
  unsigned long long nulls = 0;
  for (int64_t r0 = (int64_t)blockIdx.x * QUAD_ROWS_PER_CTA + (int64_t)warp * QUAD_ROWS_PER_WARP; r0 < n_rows; r0 += step) {
    const uint32_t vb = quad_valid_bits(validity, r0, n_rows, lane);
    const int64_t r = r0 + lane * QUAD_ROWS_PER_LANE;
    uint32_t keep = 0;
    if (r < n_rows) {
      T e[4];
      load_quad<T>(src, r, n_rows, e);
      U o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const bool live = r + k < n_rows;
        const double v = scale_value((double)e[k], sp.mode, sp.a, sp.b, sp.c);
        const bool ok = live && ((vb >> k) & 1u) && !(NAN_TO_NULL && (Traits<T>::is_nan(e[k]) || v != v));
        keep |= (uint32_t)ok << k;
        nulls += (unsigned long long)(live && !ok);
        o[k] = ok ? narrow<U>(v) : U(0);
      }
      store_quad<U>(dst, r, o);
    }
    if constexpr (NAN_TO_NULL) store_quad_valid_bits(out_valid, keep, r0, n_rows, lane);
  }
  warp_add_count(n_null, nulls, lane);
}

template <typename T, typename U>
__device__ __forceinline__ void scale_column_of(const anv_column_t& col, void* dst, uint32_t* out_valid, unsigned long long* n_null,
                                                const anv_scale_spec_t& sp, int64_t n_rows) {
  if (sp.flags & ANV_SCALE_NAN_TO_NULL)
    scale_column<T, U, true>((const T*)col.data, col.validity, (U*)dst, out_valid, n_null, sp, n_rows);
  else
    scale_column<T, U, false>((const T*)col.data, col.validity, (U*)dst, out_valid, n_null, sp, n_rows);
}

template <typename U>
__device__ __forceinline__ void scale_dispatch(const anv_column_t& col, void* dst, uint32_t* out_valid, unsigned long long* n_null,
                                               const anv_scale_spec_t& sp, int64_t n_rows) {
  switch (col.dtype) {
    case ANV_F32: scale_column_of<float, U>(col, dst, out_valid, n_null, sp, n_rows); break;
    case ANV_F64: scale_column_of<double, U>(col, dst, out_valid, n_null, sp, n_rows); break;
    case ANV_I32: scale_column_of<int32_t, U>(col, dst, out_valid, n_null, sp, n_rows); break;
    default: scale_column_of<int64_t, U>(col, dst, out_valid, n_null, sp, n_rows); break;
  }
}

__global__ void __launch_bounds__(ANV_BLOCK) scale_kernel(const anv_column_t* __restrict__ cols,
                                                          const anv_scale_spec_t* __restrict__ specs,
                                                          void* const* __restrict__ out_ptrs, uint32_t* __restrict__ out_validity,
                                                          unsigned long long* __restrict__ null_counts, int64_t n_rows) {
  const int c = blockIdx.y;
  const anv_column_t col = cols[c];
  const anv_scale_spec_t sp = specs[c];
  if (sp.mode < ANV_SCALE_DIV || sp.mode > ANV_SCALE_CONST) return;     // not a mode of the header: left unwritten
  if ((sp.flags & ANV_SCALE_NAN_TO_NULL) && !out_validity) return;
  const int64_t n_words = (n_rows + 31) / 32;
  uint32_t* out_valid = out_validity ? out_validity + (size_t)c * n_words : nullptr;
  // the branches are uniform per CTA
  if (sp.out_dtype == ANV_F64)
    scale_dispatch<double>(col, out_ptrs[c], out_valid, null_counts + c, sp, n_rows);
  else if (sp.out_dtype == ANV_F32)
    scale_dispatch<float>(col, out_ptrs[c], out_valid, null_counts + c, sp, n_rows);
}

int check_common(const void* cols, int n_cols, int64_t n_rows);

}  // namespace anv

using namespace anv;

extern "C" int anv_scale_columns(const anv_column_t* cols, const anv_scale_spec_t* specs, void* const* out_ptrs,
                                 uint32_t* out_validity, int64_t* null_counts, int n_cols, int64_t n_rows, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0) return ANV_OK;
  if (!specs || !out_ptrs || !null_counts) { set_error("anv_scale_columns: specs / out_ptrs / null_counts is NULL"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  ANV_CUDA(cudaMemsetAsync(null_counts, 0, (size_t)n_cols * sizeof(int64_t), st));
  if (n_rows == 0) return ANV_OK;
  dim3 grid(quad_grid_x(n_rows, n_cols), (unsigned)n_cols);
  scale_kernel<<<grid, ANV_BLOCK, 0, st>>>(cols, specs, out_ptrs, out_validity, reinterpret_cast<unsigned long long*>(null_counts),
                                           n_rows);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}
