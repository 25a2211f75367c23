// Mean / median / mode imputation of missing values (imputation_MMM, reference data_transformer/transformers.py:
// 1369-1676): the fill pass that writes the imputed columns, and the "non-null and not NaN" bitmap the Imputer's
// statistics are taken over.
//
// Both passes stream each column once.  Grid (row tiles, columns); a warp covers 128 consecutive rows per step, four
// per lane, so every lane moves its values with 128-bit loads and stores (two for 8-byte types).  The validity word of
// 32 rows is loaded once, by one of the first four lanes, and handed to the eight lanes that cover its rows by a shuffle.
//
// Fill: out = (valid && !(nan_missing && isnan(x))) ? convert(x) : fill, dense, with no bitmap.  convert is the
// identity, int -> double (numeric mode imputation keeps numbers in the recast type) or, for bigint under mean / median,
// the round trip (long)(double)x of Spark's recast (cvt saturates like Java's d2l: 2^63-1 comes back as 2^63-1).  The
// fill value arrives already converted to the output type: the kernel does no per-column double work.
#include "common.cuh"

namespace anv {

constexpr int IMP_ROWS_PER_LANE = 4;
constexpr int IMP_ROWS_PER_WARP = 32 * IMP_ROWS_PER_LANE;
constexpr int IMP_ROWS_PER_CTA = ANV_BLOCK * IMP_ROWS_PER_LANE;

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

template <typename T, typename U, bool ROUND> __device__ __forceinline__ U convert(T x) {
  if constexpr (ROUND) return (U)(double)x;                  // bigint under mean / median: Spark's recast round trip
  else return (U)x;
}

template <typename T, typename U, bool ROUND>
__device__ __forceinline__ void fill_column(const T* __restrict__ src, const uint32_t* __restrict__ validity, U* __restrict__ dst,
                                            U fill, bool nan_missing, int64_t n_rows) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t step = (int64_t)gridDim.x * IMP_ROWS_PER_CTA;
  for (int64_t r0 = (int64_t)blockIdx.x * IMP_ROWS_PER_CTA + (int64_t)warp * IMP_ROWS_PER_WARP; r0 < n_rows; r0 += step) {
    const uint32_t vb = quad_valid_bits(validity, r0, n_rows, lane);
    const int64_t r = r0 + lane * IMP_ROWS_PER_LANE;
    if (r >= n_rows) continue;
    T e[4];
    load_quad<T>(src, r, n_rows, e);
    U o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const bool keep = ((vb >> k) & 1u) && !(nan_missing && Traits<T>::is_nan(e[k]));
      o[k] = keep ? convert<T, U, ROUND>(e[k]) : fill;
    }
    store_quad<U>(dst, r, o);
  }
}

template <typename U> __device__ __forceinline__ U fill_of(uint64_t bits) {
  if constexpr (sizeof(U) == 4) { const uint32_t b = (uint32_t)bits; return reinterpret_cast<const U&>(b); }
  else return reinterpret_cast<const U&>(bits);
}

__global__ void __launch_bounds__(ANV_BLOCK) impute_fill_kernel(const anv_column_t* __restrict__ cols,
                                                                const anv_impute_spec_t* __restrict__ specs,
                                                                void* const* __restrict__ out_ptrs, int64_t n_rows) {
  const int c = blockIdx.y;
  const anv_column_t col = cols[c];
  const anv_impute_spec_t sp = specs[c];
  void* dst = out_ptrs[c];
  const bool nan_missing = (sp.flags & ANV_IMPUTE_NAN_MISSING) != 0;
  const bool round = (sp.flags & ANV_IMPUTE_ROUND_DOUBLE) != 0;
  // the (input, output) pairs of the header; the branch is uniform per CTA
  switch (col.dtype * 4 + sp.out_dtype) {
    case ANV_F32 * 4 + ANV_F32:
      fill_column<float, float, false>((const float*)col.data, col.validity, (float*)dst, fill_of<float>(sp.fill), nan_missing, n_rows);
      break;
    case ANV_F64 * 4 + ANV_F64:
      fill_column<double, double, false>((const double*)col.data, col.validity, (double*)dst, fill_of<double>(sp.fill), nan_missing, n_rows);
      break;
    case ANV_I32 * 4 + ANV_I32:    // int under mean / median (the round trip is the identity) and dictionary codes
      fill_column<int32_t, int32_t, false>((const int32_t*)col.data, col.validity, (int32_t*)dst, fill_of<int32_t>(sp.fill), false, n_rows);
      break;
    case ANV_I64 * 4 + ANV_I64:
      if (round)
        fill_column<int64_t, int64_t, true>((const int64_t*)col.data, col.validity, (int64_t*)dst, fill_of<int64_t>(sp.fill), false, n_rows);
      else
        fill_column<int64_t, int64_t, false>((const int64_t*)col.data, col.validity, (int64_t*)dst, fill_of<int64_t>(sp.fill), false, n_rows);
      break;
    case ANV_I32 * 4 + ANV_F64:
      fill_column<int32_t, double, false>((const int32_t*)col.data, col.validity, (double*)dst, fill_of<double>(sp.fill), false, n_rows);
      break;
    case ANV_I64 * 4 + ANV_F64:
      fill_column<int64_t, double, false>((const int64_t*)col.data, col.validity, (double*)dst, fill_of<double>(sp.fill), false, n_rows);
      break;
    default:   // not a pair of the header's list: the column is left unwritten
      break;
  }
}

// "non-null and not NaN" bitmap of a float column: each lane tests its quad, the 8 lanes of a word OR their nibbles
// together, the word's first lane writes it.  NaN count: one atomic per warp at the end.
template <typename T>
__device__ __forceinline__ void valid_not_nan_column(const T* __restrict__ src, const uint32_t* __restrict__ validity,
                                                     uint32_t* __restrict__ out, unsigned long long* __restrict__ n_nan,
                                                     int64_t n_rows) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t step = (int64_t)gridDim.x * IMP_ROWS_PER_CTA;
  unsigned long long nan_count = 0;
  for (int64_t r0 = (int64_t)blockIdx.x * IMP_ROWS_PER_CTA + (int64_t)warp * IMP_ROWS_PER_WARP; r0 < n_rows; r0 += step) {
    const uint32_t vb = quad_valid_bits(validity, r0, n_rows, lane);
    const int64_t r = r0 + lane * IMP_ROWS_PER_LANE;
    uint32_t keep = 0, nan = 0;
    if (r < n_rows) {
      T e[4];
      load_quad<T>(src, r, n_rows, e);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const bool live = r + k < n_rows && ((vb >> k) & 1u);
        const bool isn = Traits<T>::is_nan(e[k]);
        keep |= (uint32_t)(live && !isn) << k;
        nan |= (uint32_t)(live && isn) << k;
      }
    }
    nan_count += __popc(nan);
    uint32_t word = keep << (4 * (lane & 7));
    word |= __shfl_xor_sync(ANV_FULL, word, 1);
    word |= __shfl_xor_sync(ANV_FULL, word, 2);
    word |= __shfl_xor_sync(ANV_FULL, word, 4);
    const int64_t w = r0 / 32 + (lane >> 3);
    if ((lane & 7) == 0 && w * 32 < n_rows) out[w] = word;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nan_count += __shfl_down_sync(ANV_FULL, nan_count, o);
  if (lane == 0 && nan_count) atomicAdd(n_nan, nan_count);
}

__global__ void __launch_bounds__(ANV_BLOCK) valid_not_nan_kernel(const anv_column_t* __restrict__ cols, int64_t n_rows,
                                                                  uint32_t* __restrict__ out_validity,
                                                                  unsigned long long* __restrict__ n_nan) {
  const int c = blockIdx.y;
  const anv_column_t col = cols[c];
  const int64_t n_words = (n_rows + 31) / 32;
  uint32_t* out = out_validity + (size_t)c * n_words;
  switch (col.dtype) {   // integer columns hold no NaN: their bitmap is the validity itself
    case ANV_F32: valid_not_nan_column<float>((const float*)col.data, col.validity, out, n_nan + c, n_rows); break;
    case ANV_F64: valid_not_nan_column<double>((const double*)col.data, col.validity, out, n_nan + c, n_rows); break;
    case ANV_I32: valid_not_nan_column<int32_t>((const int32_t*)col.data, col.validity, out, n_nan + c, n_rows); break;
    default: valid_not_nan_column<int64_t>((const int64_t*)col.data, col.validity, out, n_nan + c, n_rows); break;
  }
}

// Row tiles per column: enough CTAs for ~16 per SM across the launch, never more than the rows need.
static unsigned impute_grid_x(int64_t n_rows, int n_cols) {
  int sms = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t need = (n_rows + IMP_ROWS_PER_CTA - 1) / IMP_ROWS_PER_CTA;
  int64_t want = ((int64_t)sms * 16 + n_cols - 1) / n_cols;
  if (want < 1) want = 1;
  return (unsigned)(need < want ? need : want);
}

int check_common(const void* cols, int n_cols, int64_t n_rows);

}  // namespace anv

using namespace anv;

extern "C" int anv_impute_fill(const anv_column_t* cols, const anv_impute_spec_t* specs, void* const* out_ptrs, int n_cols,
                               int64_t n_rows, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0 || n_rows == 0) return ANV_OK;
  if (!specs || !out_ptrs) { set_error("anv_impute_fill: specs / out_ptrs is NULL"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(impute_grid_x(n_rows, n_cols), (unsigned)n_cols);
  impute_fill_kernel<<<grid, ANV_BLOCK, 0, st>>>(cols, specs, out_ptrs, n_rows);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

extern "C" int anv_valid_not_nan(const anv_column_t* cols, int n_cols, int64_t n_rows, uint32_t* out_validity,
                                 int64_t* n_nan, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0) return ANV_OK;
  if (!n_nan || (n_rows > 0 && !out_validity)) { set_error("anv_valid_not_nan: out_validity / n_nan is NULL"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  ANV_CUDA(cudaMemsetAsync(n_nan, 0, (size_t)n_cols * sizeof(int64_t), st));
  if (n_rows == 0) return ANV_OK;
  dim3 grid(impute_grid_x(n_rows, n_cols), (unsigned)n_cols);
  valid_not_nan_kernel<<<grid, ANV_BLOCK, 0, st>>>(cols, n_rows, out_validity, reinterpret_cast<unsigned long long*>(n_nan));
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}
