// The categorical encoders cat_to_num_unsupervised, cat_to_num_supervised and outlier_categories (reference
// data_transformer/transformers.py:506-962, 3489-3671): every row's dictionary code is looked up in a small per-column
// table.
//
// Grid (row tiles, columns), four rows per lane with 128-bit loads and stores (quad.cuh).  A row's table slot is
//   slot = valid(r) ? min((uint32)code, size) : size
// where size is the column's dictionary size: the table has size + 1 entries and the last one is what null rows read.
// The unsigned min sends a negative code or one past the dictionary to the null slot, so no code reads outside the table.
// Tables are tiny next to the columns (51 entries for a default one-hot, 10 001 for a 10 000-key column): they are read
// through the read-only cache.
//
// code_map_kernel:  out[r] = table[slot] (int32 or double).  With a per-entry bitmap of the table, the row is null where
//                   its entry is; the kernel writes the output bitmap (the 8 lanes of a word OR their nibbles together)
//                   and counts the null rows, one atomic per warp.  Null rows are written as 0.
// one_hot_kernel:   out[j * stride + r] = (index[slot] == j) for j < k, dense int32.  Every lane loads its four codes
//                   once and then stores one int4 per output column: each warp store is a coalesced 512-byte run.
//                   Rows past n_rows up to the next multiple of 4 are written as 0.
#include "quad.cuh"

namespace anv {

__device__ __forceinline__ uint32_t code_slot(int32_t code, bool valid, uint32_t size) {
  return valid ? min((uint32_t)code, size) : size;
}

template <typename U, bool ENTRY_VALID>
__device__ __forceinline__ void map_column(const int32_t* __restrict__ codes, const uint32_t* __restrict__ validity,
                                           const anv_code_map_spec_t& sp, unsigned long long* __restrict__ n_null,
                                           int64_t n_rows) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t step = (int64_t)gridDim.x * QUAD_ROWS_PER_CTA;
  const U* __restrict__ table = (const U*)sp.table;
  const uint32_t* __restrict__ tvalid = sp.table_valid;
  U* __restrict__ dst = (U*)sp.out;
  const uint32_t size = (uint32_t)sp.size;
  unsigned long long nulls = 0;
  for (int64_t r0 = (int64_t)blockIdx.x * QUAD_ROWS_PER_CTA + (int64_t)warp * QUAD_ROWS_PER_WARP; r0 < n_rows; r0 += step) {
    const uint32_t vb = quad_valid_bits(validity, r0, n_rows, lane);
    const int64_t r = r0 + lane * QUAD_ROWS_PER_LANE;
    uint32_t keep = 0;
    if (r < n_rows) {
      int32_t e[4];
      load_quad<int32_t>(codes, r, n_rows, e);
      U o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t s = code_slot(e[k], (vb >> k) & 1u, size);
        o[k] = __ldg(table + s);
        if constexpr (ENTRY_VALID) {
          const bool live = r + k < n_rows;
          const bool ok = live && ((__ldg(tvalid + (s >> 5)) >> (s & 31)) & 1u);
          keep |= (uint32_t)ok << k;
          nulls += (unsigned long long)(live && !ok);
          if (!ok) o[k] = U(0);
        }
      }
      store_quad<U>(dst, r, o);
    }
    if constexpr (ENTRY_VALID) store_quad_valid_bits(sp.out_valid, keep, r0, n_rows, lane);
  }
  if constexpr (ENTRY_VALID) warp_add_count(n_null, nulls, lane);
}

template <typename U>
__device__ __forceinline__ void map_column_of(const anv_column_t& col, const anv_code_map_spec_t& sp,
                                              unsigned long long* n_null, int64_t n_rows) {
  if (sp.table_valid)
    map_column<U, true>((const int32_t*)col.data, col.validity, sp, n_null, n_rows);
  else
    map_column<U, false>((const int32_t*)col.data, col.validity, sp, n_null, n_rows);
}

__global__ void __launch_bounds__(ANV_BLOCK) code_map_kernel(const anv_column_t* __restrict__ cols,
                                                             const anv_code_map_spec_t* __restrict__ specs,
                                                             unsigned long long* __restrict__ null_counts, int64_t n_rows) {
  const int c = blockIdx.y;
  const anv_column_t col = cols[c];
  const anv_code_map_spec_t sp = specs[c];
  // the branches are uniform per CTA
  if (col.dtype != ANV_I32 || sp.size < 0 || !sp.table || !sp.out || (sp.table_valid && !sp.out_valid)) return;
  if (sp.out_dtype == ANV_I32)
    map_column_of<int32_t>(col, sp, null_counts + c, n_rows);
  else if (sp.out_dtype == ANV_F64)
    map_column_of<double>(col, sp, null_counts + c, n_rows);
}

__global__ void __launch_bounds__(ANV_BLOCK) one_hot_kernel(const anv_column_t* __restrict__ cols,
                                                            const anv_one_hot_spec_t* __restrict__ specs, int64_t n_rows) {
  const int c = blockIdx.y;
  const anv_column_t col = cols[c];
  const anv_one_hot_spec_t sp = specs[c];
  if (col.dtype != ANV_I32 || sp.size < 0 || sp.k < 1 || !sp.index || !sp.out || sp.stride < n_rows || (sp.stride & 3)) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t step = (int64_t)gridDim.x * QUAD_ROWS_PER_CTA;
  const int32_t* __restrict__ codes = (const int32_t*)col.data;
  const uint32_t size = (uint32_t)sp.size;
  for (int64_t r0 = (int64_t)blockIdx.x * QUAD_ROWS_PER_CTA + (int64_t)warp * QUAD_ROWS_PER_WARP; r0 < n_rows; r0 += step) {
    const uint32_t vb = quad_valid_bits(col.validity, r0, n_rows, lane);
    const int64_t r = r0 + lane * QUAD_ROWS_PER_LANE;
    if (r < n_rows) {
      int32_t e[4], idx[4];
      load_quad<int32_t>(codes, r, n_rows, e);
#pragma unroll
      for (int k = 0; k < 4; ++k) idx[k] = r + k < n_rows ? __ldg(sp.index + code_slot(e[k], (vb >> k) & 1u, size)) : -1;
      int32_t* __restrict__ dst = sp.out + r;
      for (int j = 0; j < sp.k; ++j) {
        const int4 q = make_int4(idx[0] == j, idx[1] == j, idx[2] == j, idx[3] == j);
        __stcs(reinterpret_cast<int4*>(dst + (int64_t)j * sp.stride), q);
      }
    }
  }
}

int check_common(const void* cols, int n_cols, int64_t n_rows);

}  // namespace anv

using namespace anv;

extern "C" int anv_code_map(const anv_column_t* cols, const anv_code_map_spec_t* specs, int64_t* null_counts, int n_cols,
                            int64_t n_rows, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0) return ANV_OK;
  if (!specs || !null_counts) { set_error("anv_code_map: specs / null_counts is NULL"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  ANV_CUDA(cudaMemsetAsync(null_counts, 0, (size_t)n_cols * sizeof(int64_t), st));
  if (n_rows == 0) return ANV_OK;
  dim3 grid(quad_grid_x(n_rows, n_cols), (unsigned)n_cols);
  code_map_kernel<<<grid, ANV_BLOCK, 0, st>>>(cols, specs, reinterpret_cast<unsigned long long*>(null_counts), n_rows);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

extern "C" int anv_one_hot(const anv_column_t* cols, const anv_one_hot_spec_t* specs, int n_cols, int64_t n_rows,
                           void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0 || n_rows == 0) return ANV_OK;
  if (!specs) { set_error("anv_one_hot: specs is NULL"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(quad_grid_x(n_rows, n_cols), (unsigned)n_cols);
  one_hot_kernel<<<grid, ANV_BLOCK, 0, st>>>(cols, specs, n_rows);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}
