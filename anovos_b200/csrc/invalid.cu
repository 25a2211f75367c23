// invalidEntries_detection (reference data_analyzer/quality_checker.py:1342-1711): the host decides which distinct values
// of a column are invalid (shared/invalid_rules.py); this pass counts the rows holding each of them and, for the
// null-replacement treatment, writes the column's new validity bitmap.
//
// Grid (row tiles, columns), four rows per lane with 128-bit loads (quad.cuh).  Every row's value becomes an unsigned key
// whose order is numeric order:
//   int32 / int64 (dictionary codes included): the bits with the sign bit flipped;
//   float32 / float64: every NaN payload first becomes the one quiet NaN, then the bits flip entirely when the sign is
//   set and only the sign bit otherwise (so -0.0 and 0.0 stay two keys and NaN sorts above +inf).
// The key is looked up by binary search in the column's sorted table.  A valid row that hits adds one to its entry's
// count and, with an output bitmap, its bit is valid & !hit (the 8 lanes of a word OR their nibbles together, as
// code_map_kernel does).  Null rows never hit.
//
// Tables of at most FLAG_SMEM_KEYS entries are staged in shared memory with per-CTA uint32 counters, flushed to the
// uint64 counts once per CTA (and every FLAG_FLUSH_TILES row tiles, so a uint32 counter never wraps).  Larger tables
// (a manual rule can flag every dictionary entry, a float column can have 10^5+ distinct invalid values) are searched
// in global memory through the read-only cache, and the lanes of a warp that hit the same entry add their rows with one
// atomic.
#include "quad.cuh"

namespace anv {

constexpr int FLAG_SMEM_KEYS = 2048;           // largest table staged in shared memory
constexpr int64_t FLAG_FLUSH_TILES = 1 << 20;  // row tiles of 1024 rows between two flushes of the uint32 counters

template <typename K> struct FlagKey;
template <> struct FlagKey<uint32_t> {
  using Raw = int32_t;
  __device__ static uint32_t of(int32_t v, bool is_float) {
    uint32_t b = (uint32_t)v;
    if (!is_float) return b ^ 0x80000000u;
    if ((b & 0x7fffffffu) > 0x7f800000u) b = 0x7fc00000u;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  }
};
template <> struct FlagKey<unsigned long long> {
  using Raw = int64_t;
  __device__ static unsigned long long of(int64_t v, bool is_float) {
    unsigned long long b = (unsigned long long)v;
    const unsigned long long top = 1ull << 63;
    if (!is_float) return b ^ top;
    if ((b & ~top) > 0x7ff0000000000000ull) b = 0x7ff8000000000000ull;
    return (b & top) ? ~b : (b | top);
  }
};

template <typename K, bool SHARED> __device__ __forceinline__ K key_at(const K* keys, int i) {
  return SHARED ? keys[i] : __ldg(keys + i);
}

// Index of each key in keys[0, n) (n >= 1), or -1: a branchless lower bound whose trip count depends on n only, so the
// four searches of a lane run interleaved.
template <typename K, bool SHARED>
__device__ __forceinline__ void find_keys(const K* keys, int n, const K (&key)[4], int (&idx)[4]) {
  int base[4] = {0, 0, 0, 0};
  for (int len = n; len > 1;) {
    const int half = len >> 1;
#pragma unroll
    for (int k = 0; k < 4; ++k) base[k] = key_at<K, SHARED>(keys, base[k] + half) < key[k] ? base[k] + half : base[k];
    len -= half;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const K v = key_at<K, SHARED>(keys, base[k]);
    const int lb = base[k] + (v < key[k]);
    idx[k] = (lb < n && key_at<K, SHARED>(keys, lb) == key[k]) ? lb : -1;
  }
}

template <typename K, bool SHARED>
__device__ __forceinline__ void flag_column(const anv_column_t& col, const anv_flag_spec_t& sp, int64_t n_rows, K* s_keys,
                                            uint32_t* s_cnt) {
  using Raw = typename FlagKey<K>::Raw;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool is_float = col.dtype == ANV_F32 || col.dtype == ANV_F64;
  const int n_keys = (int)sp.n_keys;
  const K* __restrict__ keys = SHARED ? s_keys : (const K*)sp.keys;
  unsigned long long* __restrict__ counts = sp.counts;
  uint32_t* __restrict__ out_valid = sp.out_valid;
  const Raw* __restrict__ data = (const Raw*)col.data;
  if (SHARED) {
    for (int i = threadIdx.x; i < n_keys; i += blockDim.x) {
      s_keys[i] = __ldg((const K*)sp.keys + i);
      s_cnt[i] = 0;
    }
    __syncthreads();
  }
  const int64_t step = (int64_t)gridDim.x * QUAD_ROWS_PER_CTA;
  int64_t tiles = 0;
  // the trip count is uniform per CTA, so the periodic flush may synchronise the block
  for (int64_t t0 = (int64_t)blockIdx.x * QUAD_ROWS_PER_CTA; t0 < n_rows; t0 += step) {
    const int64_t r0 = t0 + (int64_t)warp * QUAD_ROWS_PER_WARP;
    if (r0 < n_rows) {                                   // warp-uniform
      const uint32_t vb = quad_valid_bits(col.validity, r0, n_rows, lane);
      const int64_t r = r0 + lane * QUAD_ROWS_PER_LANE;
      uint32_t keep = 0;
      int idx[4] = {-1, -1, -1, -1};
      if (r < n_rows) {
        Raw e[4];
        K key[4];
        load_quad<Raw>(data, r, n_rows, e);
#pragma unroll
        for (int k = 0; k < 4; ++k) key[k] = FlagKey<K>::of(e[k], is_float);
        find_keys<K, SHARED>(keys, n_keys, key, idx);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const bool live = r + k < n_rows && ((vb >> k) & 1u);
          if (!live) idx[k] = -1;
          keep |= (uint32_t)(live && idx[k] < 0) << k;
        }
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (SHARED) {
          if (idx[k] >= 0) atomicAdd(s_cnt + idx[k], 1u);
        } else {
          const unsigned peers = __match_any_sync(ANV_FULL, idx[k]);
          if (idx[k] >= 0 && lane == __ffs(peers) - 1) atomicAdd(counts + idx[k], (unsigned long long)__popc(peers));
        }
      }
      if (out_valid) {
        uint32_t word = keep << (4 * (lane & 7));
        word |= __shfl_xor_sync(ANV_FULL, word, 1);
        word |= __shfl_xor_sync(ANV_FULL, word, 2);
        word |= __shfl_xor_sync(ANV_FULL, word, 4);
        const int64_t w = r0 / 32 + (lane >> 3);
        if ((lane & 7) == 0 && w * 32 < n_rows) out_valid[w] = word;
      }
    }
    if (SHARED && ++tiles == FLAG_FLUSH_TILES) {
      tiles = 0;
      __syncthreads();
      for (int i = threadIdx.x; i < n_keys; i += blockDim.x) {
        if (s_cnt[i]) atomicAdd(counts + i, (unsigned long long)s_cnt[i]);
        s_cnt[i] = 0;
      }
      __syncthreads();
    }
  }
  if (SHARED) {
    __syncthreads();
    for (int i = threadIdx.x; i < n_keys; i += blockDim.x)
      if (s_cnt[i]) atomicAdd(counts + i, (unsigned long long)s_cnt[i]);
  }
}

__global__ void __launch_bounds__(ANV_BLOCK) flag_members_kernel(const anv_column_t* __restrict__ cols,
                                                                 const anv_flag_spec_t* __restrict__ specs, int64_t n_rows) {
  __shared__ __align__(16) unsigned long long s_keys[FLAG_SMEM_KEYS];
  __shared__ uint32_t s_cnt[FLAG_SMEM_KEYS];
  const int c = blockIdx.y;
  const anv_column_t col = cols[c];
  const anv_flag_spec_t sp = specs[c];
  // the branches are uniform per CTA
  if (sp.n_keys <= 0 || sp.n_keys > INT32_MAX || !sp.keys || !sp.counts) return;
  if (col.dtype == ANV_I32 || col.dtype == ANV_F32) {
    if (sp.n_keys <= FLAG_SMEM_KEYS)
      flag_column<uint32_t, true>(col, sp, n_rows, reinterpret_cast<uint32_t*>(s_keys), s_cnt);
    else
      flag_column<uint32_t, false>(col, sp, n_rows, nullptr, nullptr);
  } else if (col.dtype == ANV_I64 || col.dtype == ANV_F64) {
    if (sp.n_keys <= FLAG_SMEM_KEYS)
      flag_column<unsigned long long, true>(col, sp, n_rows, s_keys, s_cnt);
    else
      flag_column<unsigned long long, false>(col, sp, n_rows, nullptr, nullptr);
  }
}

int check_common(const void* cols, int n_cols, int64_t n_rows);

}  // namespace anv

using namespace anv;

extern "C" int anv_flag_members_smem_keys() { return FLAG_SMEM_KEYS; }

extern "C" int anv_flag_members(const anv_column_t* cols, const anv_flag_spec_t* specs, int n_cols, int64_t n_rows,
                                void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0 || n_rows == 0) return ANV_OK;
  if (!specs) { set_error("anv_flag_members: specs is NULL"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(quad_grid_x(n_rows, n_cols), (unsigned)n_cols);
  flag_members_kernel<<<grid, ANV_BLOCK, 0, st>>>(cols, specs, n_rows);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}
