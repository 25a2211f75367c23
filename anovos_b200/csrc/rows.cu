// Row-level quality checks: per-row null counts and exact distinct rows.
//
// Replaces the two row-level checks of quality_checker (reference /root/reference/src/main/anovos/data_analyzer/
// quality_checker.py): nullRows_detection (:152-283, a Python UDF counting None per row, then a groupBy of the count) and
// duplicate_detection (:49-149, `idf.groupby(list_of_cols).count()`: a global group-by over whole rows).
//
// Null counts: one thread per 32-row bitmap word adds the inverted validity bits of every column into 17 bit planes
// (a bit-sliced counter per row), then reads each row's count out of the planes.  Histogram in per-CTA shared counters,
// one global add per (CTA, slot): integer, deterministic.  Reads the bitmaps only.
//
// Distinct rows, three stages:
//   keys    one streaming pass over the columns: a 64-bit hash of each row's NORMALISED values (null == null and != every
//           value, the data under a null lane ignored, every NaN equal, -0.0 == 0.0, otherwise bits; string columns by
//           dictionary code), written as key = hash prefix << idx_bits | row, in row order, into the sort's key buffer;
//   sort    the LSD passes of sort.cu over the hash bytes only (keysort.cuh): the keys arrive in row order and the passes
//           are stable, so the row-index bytes never need a pass;
//   verify  runs = sorted keys with the same hash prefix; a run's head (its first key) has the smallest row index.  Run
//           heads come from a max-scan of the run-start positions (tile maxima, one carry scan, in-tile scan).  Every other
//           row is compared with its head over all columns with the same normalised equality: equal -> duplicate.  A
//           mismatch means the prefix collided: such runs are resolved by one CTA each in rounds (the first unresolved
//           row is a new representative, the rest are compared with it), quadratic in the number of distinct values that
//           share one prefix - about 1 at the default width.
// The result never depends on the hash being unique.  The representative of a group is its first row.
#include "common.cuh"
#include "keysort.cuh"

namespace anv {

// ---- row null counts ------------------------------------------------------------------------------------------------

constexpr int NC_PLANES = 17;                 // bit-sliced counters up to 2^17 - 1 columns
constexpr int NC_MAX_COLS = (1 << NC_PLANES) - 1;   // one grid over the rows: the column count is bounded by the planes only
constexpr int NC_SMEM_SLOTS = 6144;           // shared histogram (48 KB of uint64) for up to 6143 columns

__global__ void __launch_bounds__(ANV_BLOCK) row_null_counts_kernel(const uint32_t* const* __restrict__ validity, int n_bm,
                                                                     int n_slots, int64_t n_rows, int max_keep,
                                                                     unsigned long long* __restrict__ counts,
                                                                     uint32_t* __restrict__ keep) {
  extern __shared__ unsigned long long sh[];
  const bool use_smem = n_slots <= NC_SMEM_SLOTS;
  if (use_smem)
    for (int i = threadIdx.x; i < n_slots; i += ANV_BLOCK) sh[i] = 0;
  __syncthreads();
  const int n_planes = n_bm > 0 ? 32 - __clz(n_bm) : 0;
  const int64_t n_words = (n_rows + 31) / 32;
  const int64_t step = (int64_t)gridDim.x * ANV_BLOCK;
  // the loop bound is uniform per warp so that every lane takes part in the match below
  for (int64_t w0 = (int64_t)blockIdx.x * ANV_BLOCK; w0 < n_words; w0 += step) {
    const int64_t w = w0 + threadIdx.x;
    const bool live_word = w < n_words;
    uint32_t pl[NC_PLANES];
#pragma unroll
    for (int j = 0; j < NC_PLANES; ++j) pl[j] = 0;
    if (live_word) {
      for (int b = 0; b < n_bm; ++b) {
        const uint32_t* vb = reinterpret_cast<const uint32_t*>(__ldg(reinterpret_cast<const unsigned long long*>(validity) + b));
        uint32_t carry = ~__ldg(vb + w);   // 1 = null
#pragma unroll
        for (int j = 0; j < NC_PLANES; ++j) {
          const uint32_t t = pl[j] & carry;
          pl[j] ^= carry;
          carry = t;
          if (!carry) break;
        }
      }
    }
    const int live = live_word ? (int)min((int64_t)32, n_rows - w * 32) : 0;
    uint32_t kw = 0;
    for (int r = 0; r < 32; ++r) {
      uint32_t k = 0;
#pragma unroll
      for (int j = 0; j < NC_PLANES; ++j)
        if (j < n_planes) k |= ((pl[j] >> r) & 1u) << j;
      const bool ok = r < live;
      if (ok && (int)k <= max_keep) kw |= 1u << r;
      const uint32_t key = ok ? k : 0xFFFFFFFFu;
      const uint32_t peers = __match_any_sync(ANV_FULL, key);   // lanes with the same count: one add per group
      if (ok && (__ffs(peers) - 1) == (int)(threadIdx.x & 31)) {
        if (use_smem) atomicAdd(&sh[k], (unsigned long long)__popc(peers));
        else atomicAdd(&counts[k], (unsigned long long)__popc(peers));
      }
    }
    if (live_word && keep) keep[w] = kw;
  }
  __syncthreads();
  if (use_smem)
    for (int i = threadIdx.x; i < n_slots; i += ANV_BLOCK)
      if (sh[i]) atomicAdd(&counts[i], sh[i]);
}

// ---- distinct rows: normalised values, hash, row comparison -----------------------------------------------------------

constexpr uint64_t ROW_SEED = 0x243F6A8885A308D3ull;
constexpr uint64_t ROW_MUL = 0x9E3779B97F4A7C15ull;
constexpr uint64_t NULL_TAG = 0x6A09E667F3BCC909ull;   // the value a null lane hashes as (a value with these bits collides: verified)

__device__ __forceinline__ uint64_t fmix64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return k;
}
__device__ __forceinline__ uint64_t norm_f32(float x) {
  return (x != x) ? 0x7fc00000ull : (uint64_t)__float_as_uint(x + 0.0f);   // every NaN one value, -0.0 + 0.0 = +0.0
}
__device__ __forceinline__ uint64_t norm_f64(double x) {
  return (x != x) ? 0x7ff8000000000000ull : (uint64_t)__double_as_longlong(x + 0.0);
}
__device__ __forceinline__ uint64_t combine(uint64_t h, uint64_t v) { return ((h << 23 | h >> 41) ^ v) * ROW_MUL; }

__device__ __forceinline__ bool valid_bit(const uint32_t* v, uint32_t row) { return !v || ((__ldg(v + (row >> 5)) >> (row & 31)) & 1u); }

// Normalised equality of rows a and b over every column; exits at the first column that differs.
__device__ bool rows_equal(const anv_column_t* __restrict__ cols, int n_cols, uint32_t a, uint32_t b) {
  for (int c = 0; c < n_cols; ++c) {
    const void* d = cols[c].data;
    const uint32_t* vb = cols[c].validity;
    const int dt = cols[c].dtype;
    const bool va = valid_bit(vb, a), vv = valid_bit(vb, b);
    if (va != vv) return false;
    if (!va) continue;                          // null == null, whatever lies under the lanes
    switch (dt) {
      case ANV_F32: {
        const float x = __ldg((const float*)d + a), y = __ldg((const float*)d + b);
        if (!(x == y || (x != x && y != y))) return false;
        break;
      }
      case ANV_F64: {
        const double x = __ldg((const double*)d + a), y = __ldg((const double*)d + b);
        if (!(x == y || (x != x && y != y))) return false;
        break;
      }
      case ANV_I32:
        if (__ldg((const int32_t*)d + a) != __ldg((const int32_t*)d + b)) return false;
        break;
      default:
        if (__ldg((const long long*)d + a) != __ldg((const long long*)d + b)) return false;
        break;
    }
  }
  return true;
}

// keys: 4 consecutive rows per thread (one 128-bit load per 4-byte column, two per 8-byte column; the 4 rows share a
// validity word).
__global__ void __launch_bounds__(ANV_BLOCK) row_hash_kernel(const anv_column_t* __restrict__ cols, int n_cols, int64_t n_rows,
                                                             int idx_bits, int hash_bits, uint64_t* __restrict__ keys) {
  const int64_t r0 = ((int64_t)blockIdx.x * ANV_BLOCK + threadIdx.x) * 4;
  if (r0 >= n_rows) return;
  const bool full = r0 + 4 <= n_rows;
  const int nr = full ? 4 : (int)(n_rows - r0);
  uint64_t h[4] = {ROW_SEED, ROW_SEED, ROW_SEED, ROW_SEED};
  for (int c = 0; c < n_cols; ++c) {
    const anv_column_t col = cols[c];
    uint64_t v[4] = {0, 0, 0, 0};
    switch (col.dtype) {
      case ANV_F32: {
        const float* p = (const float*)col.data + r0;
        if (full) { float e[4]; unpack<float>(ldg_stream(p), e); for (int j = 0; j < 4; ++j) v[j] = norm_f32(e[j]); }
        else for (int j = 0; j < 4; ++j) if (j < nr) v[j] = norm_f32(p[j]);
        break;
      }
      case ANV_I32: {
        const int32_t* p = (const int32_t*)col.data + r0;
        if (full) { int32_t e[4]; unpack<int32_t>(ldg_stream(p), e); for (int j = 0; j < 4; ++j) v[j] = (uint64_t)(int64_t)e[j]; }
        else for (int j = 0; j < 4; ++j) if (j < nr) v[j] = (uint64_t)(int64_t)p[j];
        break;
      }
      case ANV_F64: {
        const double* p = (const double*)col.data + r0;
        if (full) {
          double e[2];
          unpack<double>(ldg_stream(p), e); v[0] = norm_f64(e[0]); v[1] = norm_f64(e[1]);
          unpack<double>(ldg_stream(p + 2), e); v[2] = norm_f64(e[0]); v[3] = norm_f64(e[1]);
        } else for (int j = 0; j < 4; ++j) if (j < nr) v[j] = norm_f64(p[j]);
        break;
      }
      default: {
        const int64_t* p = (const int64_t*)col.data + r0;
        if (full) {
          int64_t e[2];
          unpack<int64_t>(ldg_stream(p), e); v[0] = (uint64_t)e[0]; v[1] = (uint64_t)e[1];
          unpack<int64_t>(ldg_stream(p + 2), e); v[2] = (uint64_t)e[0]; v[3] = (uint64_t)e[1];
        } else for (int j = 0; j < 4; ++j) if (j < nr) v[j] = (uint64_t)p[j];
        break;
      }
    }
    if (col.validity) {
      const uint32_t word = __ldg(col.validity + (r0 >> 5)) >> (r0 & 31);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (!((word >> j) & 1u)) v[j] = NULL_TAG;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) h[j] = combine(h[j], v[j]);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (j < nr) keys[r0 + j] = ((fmix64(h[j]) >> (64 - hash_bits)) << idx_bits) | (uint64_t)(r0 + j);
}

// ---- verify -----------------------------------------------------------------------------------------------------------

constexpr int VT_PER = 16;                        // sorted positions per thread
constexpr int VT_TILE = ANV_BLOCK * VT_PER;       // positions per verify tile

struct VerifyParams {
  const anv_column_t* cols;
  int n_cols;
  int64_t n;
  int idx_bits;
  const uint64_t* buf0;
  const uint64_t* buf1;
  const int* cur;                  // the sorted keys are in (cur ? buf1 : buf0)
  uint32_t* tile_start;            // [n_vtiles] largest run start in the tile, then (after the carry scan) the exclusive max
  uint32_t* first;                 // [ceil(n/32)] first-occurrence bitmap by row
  uint32_t* claim;                 // [ceil(n/32)] by sorted position: run heads whose run holds a mismatching row
  uint32_t* unres;                 // [ceil(n/32)] by sorted position: rows not yet resolved (mismatched their head)
  unsigned long long* dups;        // duplicates found
};

__device__ __forceinline__ const uint64_t* sorted_keys(const VerifyParams& P) { return *P.cur ? P.buf1 : P.buf0; }

__global__ void __launch_bounds__(ANV_BLOCK) row_first_init_kernel(uint32_t* first, int64_t n) {
  const int64_t w = (int64_t)blockIdx.x * ANV_BLOCK + threadIdx.x;
  const int64_t nw = (n + 31) / 32;
  if (w >= nw) return;
  const int64_t rem = n - w * 32;
  first[w] = rem >= 32 ? 0xFFFFFFFFu : ((1u << rem) - 1u);
}

__device__ __forceinline__ uint32_t block_max_u32(uint32_t v, uint32_t* sw) {
  v = __reduce_max_sync(ANV_FULL, v);
  if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < ANV_WARPS; ++i) m = max(m, sw[i]);
  __syncthreads();
  return m;
}

// Largest run-start position of each tile (position 0 always starts a run, so "none" can be 0).
__global__ void __launch_bounds__(ANV_BLOCK) row_tile_start_kernel(const VerifyParams P) {
  const uint64_t* keys = sorted_keys(P);
  const int64_t i0 = (int64_t)blockIdx.x * VT_TILE;
  uint32_t best = 0;
  for (int k = 0; k < VT_PER; ++k) {
    const int64_t i = i0 + k * ANV_BLOCK + threadIdx.x;
    if (i < P.n && (i == 0 || (keys[i] >> P.idx_bits) != (keys[i - 1] >> P.idx_bits))) best = max(best, (uint32_t)i);
  }
  __shared__ uint32_t sw[ANV_WARPS];
  best = block_max_u32(best, sw);
  if (threadIdx.x == 0) P.tile_start[blockIdx.x] = best;
}

// tile_start -> exclusive max-scan (the run start in force at the beginning of each tile).  One CTA.
__global__ void __launch_bounds__(1024) row_tile_carry_kernel(uint32_t* tile_start, int n_tiles) {
  __shared__ uint32_t sw[32];
  uint32_t carry = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n_tiles; base += 1024) {
    const int i = base + threadIdx.x;
    const uint32_t v = i < n_tiles ? tile_start[i] : 0u;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o); if (lane >= o) inc = max(inc, t); }
    if (lane == 31) sw[warp] = inc;
    __syncthreads();
    uint32_t woff = carry, tot = carry;
    for (int w = 0; w < 32; ++w) { const uint32_t t = sw[w]; if (w < warp) woff = max(woff, t); tot = max(tot, t); }
    // exclusive: the max over the tiles before i
    const uint32_t prev_in_warp = __shfl_up_sync(ANV_FULL, inc, 1);
    const uint32_t ex = lane == 0 ? woff : max(woff, prev_in_warp);
    __syncthreads();
    if (i < n_tiles) tile_start[i] = ex;
    carry = tot;
  }
}

__device__ __forceinline__ void block_add_dups(unsigned long long* dups, unsigned long long mine) {
  mine = __reduce_add_sync(ANV_FULL, (unsigned)mine);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(dups, mine);
}

// Every sorted position: its run head from the in-tile max-scan (+ the tile's carry), then the comparison with the head row.
__global__ void __launch_bounds__(ANV_BLOCK) row_verify_kernel(const VerifyParams P) {
  const uint64_t* keys = sorted_keys(P);
  const uint64_t mask = (1ull << P.idx_bits) - 1ull;
  const int64_t i0 = (int64_t)blockIdx.x * VT_TILE + (int64_t)threadIdx.x * VT_PER;
  const uint64_t before = (i0 > 0 && i0 - 1 < P.n) ? keys[i0 - 1] : 0ull;
  uint64_t prev = before;
  uint32_t run = 0;                              // the largest start among my positions (0 = none)
  for (int q = 0; q < VT_PER; ++q) {
    const int64_t i = i0 + q;
    const uint64_t kq = i < P.n ? keys[i] : 0ull;
    if (i < P.n && (i == 0 || (kq >> P.idx_bits) != (prev >> P.idx_bits))) run = (uint32_t)i;
    prev = kq;
  }
  // exclusive max-scan of the per-thread `run` over the CTA, seeded with the tile's carry
  __shared__ uint32_t sw[ANV_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o); if (lane >= o) inc = max(inc, t); }
  if (lane == 31) sw[warp] = inc;
  __syncthreads();
  uint32_t ex = P.tile_start[blockIdx.x];
  for (int w = 0; w < warp; ++w) ex = max(ex, sw[w]);
  const uint32_t up = __shfl_up_sync(ANV_FULL, inc, 1);
  if (lane > 0) ex = max(ex, up);
  unsigned long long dup = 0;
  uint32_t head_pos = 0xFFFFFFFFu, head_row = 0, s = ex;
  prev = before;
  for (int q = 0; q < VT_PER; ++q) {           // second walk over my positions (L1 hits): run start of each
    const int64_t i = i0 + q;
    if (i >= P.n) break;
    const uint64_t kq = keys[i];
    const bool starts = i == 0 || (kq >> P.idx_bits) != (prev >> P.idx_bits);
    prev = kq;
    if (starts) { s = (uint32_t)i; continue; }     // a head: first occurrence
    if (s != head_pos) { head_pos = s; head_row = (uint32_t)(keys[s] & mask); }
    const uint32_t r = (uint32_t)(kq & mask);
    if (rows_equal(P.cols, P.n_cols, r, head_row)) {
      atomicAnd(&P.first[r >> 5], ~(1u << (r & 31)));
      ++dup;
    } else {                                       // the prefix collided: resolved by row_collide_kernel
      atomicOr(&P.unres[i >> 5], 1u << (i & 31));
      atomicOr(&P.claim[s >> 5], 1u << (s & 31));
    }
  }
  block_add_dups(P.dups, dup);
}

// One CTA per claimed run (a run holding a row that differs from its head), in rounds: the first unresolved row of the
// run becomes a representative (a first occurrence), every later unresolved row equal to it is a duplicate.
__device__ void resolve_run(const VerifyParams& P, const uint64_t* keys, uint32_t s, unsigned long long& dup) {
  const uint64_t mask = (1ull << P.idx_bits) - 1ull;
  const uint64_t prefix = keys[s] >> P.idx_bits;
  __shared__ unsigned long long s_min;
  // end of the run
  if (threadIdx.x == 0) s_min = ~0ull;
  __syncthreads();
  for (int64_t base = (int64_t)s + 1;; base += ANV_BLOCK) {
    const int64_t p = base + threadIdx.x;
    const bool out = p >= P.n || (keys[p] >> P.idx_bits) != prefix;
    if (out) atomicMin(&s_min, (unsigned long long)p);
    if (__syncthreads_or(out)) break;
  }
  const int64_t e = (int64_t)min(s_min, (unsigned long long)P.n);
  __syncthreads();
  for (;;) {
    if (threadIdx.x == 0) s_min = ~0ull;
    __syncthreads();
    for (int64_t p = (int64_t)s + 1 + threadIdx.x; p < e; p += ANV_BLOCK)
      if ((__ldcg(P.unres + (p >> 5)) >> (p & 31)) & 1u) { atomicMin(&s_min, (unsigned long long)p); break; }
    __syncthreads();
    const unsigned long long a = s_min;
    __syncthreads();
    if (a == ~0ull) break;
    const uint32_t ra = (uint32_t)(keys[a] & mask);
    if (threadIdx.x == 0) atomicAnd(&P.unres[a >> 5], ~(1u << (a & 31)));
    for (int64_t p = (int64_t)a + 1 + threadIdx.x; p < e; p += ANV_BLOCK) {
      if (!((__ldcg(P.unres + (p >> 5)) >> (p & 31)) & 1u)) continue;
      const uint32_t r = (uint32_t)(keys[p] & mask);
      if (rows_equal(P.cols, P.n_cols, r, ra)) {
        atomicAnd(&P.unres[p >> 5], ~(1u << (p & 31)));
        atomicAnd(&P.first[r >> 5], ~(1u << (r & 31)));
        ++dup;
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(ANV_BLOCK) row_collide_kernel(const VerifyParams P) {
  const uint64_t* keys = sorted_keys(P);
  const int64_t n_words = (P.n + 31) / 32;
  __shared__ int s_cnt;
  __shared__ uint32_t s_word[ANV_BLOCK];
  __shared__ int64_t s_w[ANV_BLOCK];
  unsigned long long dup = 0;
  for (int64_t base = (int64_t)blockIdx.x * ANV_BLOCK; base < n_words; base += (int64_t)gridDim.x * ANV_BLOCK) {
    const int64_t w = base + threadIdx.x;
    const uint32_t word = w < n_words ? __ldcg(P.claim + w) : 0u;
    if (!__syncthreads_or(word != 0)) continue;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    if (word) { const int at = atomicAdd(&s_cnt, 1); s_word[at] = word; s_w[at] = w; }
    __syncthreads();
    const int cnt = s_cnt;
    for (int q = 0; q < cnt; ++q) {
      uint32_t bits = s_word[q];
      while (bits) {
        const int b = __ffs(bits) - 1;
        bits &= bits - 1;
        resolve_run(P, keys, (uint32_t)(s_w[q] * 32 + b), dup);
      }
    }
    __syncthreads();
  }
  block_add_dups(P.dups, dup);
}

__global__ void row_distinct_final_kernel(const unsigned long long* dups, int64_t n, int64_t* n_distinct) {
  *n_distinct = n - (int64_t)*dups;
}

struct RowLayout {
  size_t sort, tile_start, claim, unres, dups, total;
  explicit RowLayout(int64_t n) {
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = (o + bytes + 255) & ~(size_t)255; return at; };
    const int64_t nw = (n + 31) / 32 > 0 ? (n + 31) / 32 : 1;
    const int64_t nt = (n + VT_TILE - 1) / VT_TILE > 0 ? (n + VT_TILE - 1) / VT_TILE : 1;
    sort = take(key_sort64_workspace_bytes(n));
    tile_start = take((size_t)nt * 4);
    claim = take((size_t)nw * 4);         // claim, unres and dups are contiguous: one memset
    unres = take((size_t)nw * 4);
    dups = take(8);
    total = o;
  }
};

static int sm_count() {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 132;
}

}  // namespace anv

using namespace anv;

extern "C" int anv_row_null_counts(const uint32_t* const* validity, int n_bitmaps, int n_cols, int64_t n_rows, int max_keep,
                                   uint64_t* counts, uint32_t* keep, void* stream) {
  if (n_bitmaps < 0 || n_cols < 0 || n_bitmaps > n_cols || n_rows < 0) { set_error("anv_row_null_counts: bad arguments"); return ANV_ERR_INVALID; }
  if (n_cols > NC_MAX_COLS) { set_error("anv_row_null_counts: n_cols > %d", NC_MAX_COLS); return ANV_ERR_UNSUPPORTED; }
  if (!counts || (n_bitmaps > 0 && !validity)) { set_error("anv_row_null_counts: NULL argument"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const int n_slots = n_cols + 1;
  ANV_CUDA(cudaMemsetAsync(counts, 0, (size_t)n_slots * sizeof(uint64_t), st));
  if (n_rows == 0) return ANV_OK;
  const int64_t n_words = (n_rows + 31) / 32;
  const int64_t want = (n_words + ANV_BLOCK - 1) / ANV_BLOCK;
  const int grid = (int)min(want, (int64_t)sm_count() * 8);
  const size_t smem = n_slots <= NC_SMEM_SLOTS ? (size_t)n_slots * sizeof(unsigned long long) : 0;
  if (smem > 48 * 1024) ANV_CUDA(cudaFuncSetAttribute(row_null_counts_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  row_null_counts_kernel<<<grid, ANV_BLOCK, smem, st>>>(validity, n_bitmaps, n_slots, n_rows, max_keep,
                                                        reinterpret_cast<unsigned long long*>(counts), keep);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

extern "C" size_t anv_row_distinct_workspace_bytes(int64_t n_rows) {
  if (n_rows < 0) return 256;
  return RowLayout(n_rows).total;
}

extern "C" int anv_row_distinct(const anv_column_t* cols, int n_cols, int64_t n_rows, int hash_bits, int64_t* n_distinct,
                                uint32_t* first, void* workspace, size_t workspace_bytes, void* stream) {
  if (n_cols < 0 || n_rows < 0 || hash_bits < 0 || hash_bits > 64) { set_error("anv_row_distinct: bad arguments"); return ANV_ERR_INVALID; }
  if (n_cols > ANV_MAX_LAUNCH_COLS) { set_error("anv_row_distinct: n_cols > %d is not supported", ANV_MAX_LAUNCH_COLS); return ANV_ERR_UNSUPPORTED; }
  if (n_rows >= ((int64_t)1 << 32)) { set_error("anv_row_distinct: n_rows >= 2^32 is not supported"); return ANV_ERR_UNSUPPORTED; }
  if (!n_distinct || !first || !workspace || (n_cols > 0 && !cols)) { set_error("anv_row_distinct: NULL argument"); return ANV_ERR_INVALID; }
  const RowLayout L(n_rows);
  if (workspace_bytes < L.total) { set_error("anv_row_distinct: workspace too small (%zu < %zu)", workspace_bytes, L.total); return ANV_ERR_WORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  if (n_rows == 0) { ANV_CUDA(cudaMemsetAsync(n_distinct, 0, sizeof(int64_t), st)); return ANV_OK; }
  // row-index width in whole bytes (the LSD passes start above it), hash bits kept above it
  const int need = n_rows > 1 ? 64 - __builtin_clzll((unsigned long long)(n_rows - 1)) : 1;
  const int idx_bits = (need + 7) / 8 * 8;
  const int hb = (hash_bits == 0 || hash_bits > 64 - idx_bits) ? 64 - idx_bits : hash_bits;
  char* w = reinterpret_cast<char*>(workspace);
  KeySort64 ks;
  key_sort64_bind(w + L.sort, n_rows, &ks);
  const int64_t nw = (n_rows + 31) / 32;
  ANV_CUDA(cudaMemsetAsync(w + L.claim, 0, L.total - L.claim, st));
  row_first_init_kernel<<<(int)((nw + ANV_BLOCK - 1) / ANV_BLOCK), ANV_BLOCK, 0, st>>>(first, n_rows);
  ANV_CUDA(cudaGetLastError());
  const int64_t n4 = (n_rows + 3) / 4;
  row_hash_kernel<<<(int)((n4 + ANV_BLOCK - 1) / ANV_BLOCK), ANV_BLOCK, 0, st>>>(cols, n_cols, n_rows, idx_bits, hb, ks.buf[0]);
  ANV_CUDA(cudaGetLastError());
  const int rc = key_sort64(w + L.sort, key_sort64_workspace_bytes(n_rows), n_rows, idx_bits / 8, (idx_bits + hb + 7) / 8, st);
  if (rc != ANV_OK) return rc;
  VerifyParams P;
  P.cols = cols; P.n_cols = n_cols; P.n = n_rows; P.idx_bits = idx_bits;
  P.buf0 = ks.buf[0]; P.buf1 = ks.buf[1]; P.cur = ks.cur;
  P.tile_start = reinterpret_cast<uint32_t*>(w + L.tile_start);
  P.first = first;
  P.claim = reinterpret_cast<uint32_t*>(w + L.claim);
  P.unres = reinterpret_cast<uint32_t*>(w + L.unres);
  P.dups = reinterpret_cast<unsigned long long*>(w + L.dups);
  const int n_tiles = (int)((n_rows + VT_TILE - 1) / VT_TILE);
  row_tile_start_kernel<<<n_tiles, ANV_BLOCK, 0, st>>>(P);
  row_tile_carry_kernel<<<1, 1024, 0, st>>>(P.tile_start, n_tiles);
  row_verify_kernel<<<n_tiles, ANV_BLOCK, 0, st>>>(P);
  ANV_CUDA(cudaGetLastError());
  const int64_t want = (nw + ANV_BLOCK - 1) / ANV_BLOCK;
  row_collide_kernel<<<(int)min(want, (int64_t)sm_count() * 4), ANV_BLOCK, 0, st>>>(P);
  row_distinct_final_kernel<<<1, 1, 0, st>>>(P.dups, n_rows, n_distinct);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}
