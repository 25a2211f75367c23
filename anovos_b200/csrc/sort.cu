// Exact mode / distinct count of numeric columns: batched LSD radix sort of the
// order-preserving keys of the non-null values + a run-length summary of the sorted keys.
//
// Replaces, for numeric columns, the per-column `groupBy(col).count().orderBy(desc).limit(1)`
// Spark jobs of mode_computation and the countDistinct aggregation of
// uniqueCount_computation (reference /root/reference/src/main/anovos/data_analyzer/
// stats_generator.py:386-401 and :611).  String columns never come here (their dictionary
// code histograms already hold the group counts).
//
// Pipeline (all columns of the call advance together, grid.y = column):
//   pack     values -> keys, nulls dropped, exact zeros counted instead of sorted (block compaction: the order
//            before a sort is irrelevant), key count per column kept on the device;
//   8-bit LSD passes: tile histogram -> per-column exclusive scan -> stable scatter (8-ballot peer ranking,
//            shared-memory reorder); a pass in which one digit holds every key is skipped (device-side
//            decision taken from the scanned table, no host sync);
//   runs     per-thread run summaries of 16 consecutive sorted keys (head count, open prefix / suffix run,
//            longest closed run), combined with an associative operator per warp, per tile and per column;
//            the merge kernel splices the zero run back and reads the requested order statistics.
// Counting is integer everywhere => deterministic.  Ties for the mode resolve to the
// smallest value (the reference's choice is arbitrary, stats_generator.py:358).
#include <stdlib.h>

#include "common.cuh"
#include "hll_hash.cuh"
#include "keysort.cuh"

namespace anv {

#ifndef ANV_SCAT_MINB
#define ANV_SCAT_MINB 2          // resident scatter CTAs per SM the register budget is tuned for
#endif
// 3 compiles to 40 registers with 48 bytes of spills in sort_scatter_kernel<uint32> (12 bytes with the ranks held as 16-bit
// halves).  It gained 0.3 % at the bench shape (H100 80GB HBM3, 400 W, sort call of 40 M x 150 float32: 72.2-72.4 ms against
// 72.4-72.7 ms) and 1.5 % at 100 M x 12 (40.1-40.2 against 40.7-40.8 ms), so 2 stays: 64 registers, no spills.
constexpr int SORT_TILE = 4096;  // keys per CTA
constexpr int SCAT_THREADS = 512;  // the scatter kernel runs 16 warps x 8 rounds of 32 keys
constexpr int SCAT_WARPS = SCAT_THREADS / 32;

template <typename K, typename T> __device__ __forceinline__ K make_key(T x);
template <> __device__ __forceinline__ uint32_t make_key<uint32_t, float>(float x) {
  x += 0.0f;
  const uint32_t u = __float_as_uint(x);
  return (x != x) ? 0xFFFFFFFFu : ((u & 0x80000000u) ? ~u : (u | 0x80000000u));
}
template <> __device__ __forceinline__ uint32_t make_key<uint32_t, int32_t>(int32_t x) { return (uint32_t)x ^ 0x80000000u; }
template <> __device__ __forceinline__ uint64_t make_key<uint64_t, double>(double x) {
  x += 0.0;
  const uint64_t u = (uint64_t)__double_as_longlong(x);
  return (x != x) ? ~0ull : ((u >> 63) ? ~u : (u | (1ull << 63)));
}
template <> __device__ __forceinline__ uint64_t make_key<uint64_t, int64_t>(int64_t x) { return (uint64_t)x ^ (1ull << 63); }
template <> __device__ __forceinline__ uint64_t make_key<uint64_t, float>(float x) { return (uint64_t)make_key<uint32_t, float>(x) << 32; }
template <> __device__ __forceinline__ uint64_t make_key<uint64_t, int32_t>(int32_t x) { return (uint64_t)make_key<uint32_t, int32_t>(x) << 32; }
template <> __device__ __forceinline__ uint32_t make_key<uint32_t, double>(double) { return 0; }   // never used
template <> __device__ __forceinline__ uint32_t make_key<uint32_t, int64_t>(int64_t) { return 0; }

__device__ __forceinline__ double sorted_key_to_double(uint64_t k, int dtype) {
  switch (dtype) {
    case ANV_F32: {
      uint32_t u = (uint32_t)(k >> 32);
      u = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u;
      return (double)__uint_as_float(u);
    }
    case ANV_I32: return (double)(int32_t)((uint32_t)(k >> 32) ^ 0x80000000u);
    case ANV_F64: {
      const uint64_t u = (k >> 63) ? (k & ~(1ull << 63)) : ~k;
      return __longlong_as_double((long long)u);
    }
    default: return (double)(int64_t)(k ^ (1ull << 63));
  }
}

// The mode_value slot of a column: the value as a double, except for ANV_I64, whose slot holds the int64 itself, bit for
// bit (a double holds only the int64s up to 2^53 exactly; the caller reads the slot as int64 for those columns).
__device__ __forceinline__ double mode_slot_of_key(uint64_t k, int dtype) {
  return dtype == ANV_I64 ? __longlong_as_double((long long)(k ^ (1ull << 63))) : sorted_key_to_double(k, dtype);
}

// Spark's hash of the VALUE a sorted key stands for (the HLL++ by-product of the run summaries): undo the order-preserving
// transform; every NaN has the key ~0 and hashes as the canonical NaN, like Spark's floatToIntBits / doubleToLongBits.
template <typename K> __device__ __forceinline__ uint64_t spark_hash_of_key(K k, int dtype);
template <> __device__ __forceinline__ uint64_t spark_hash_of_key<uint32_t>(uint32_t k, int dtype) {
  if (dtype == ANV_I32) return xxh64_int(k ^ 0x80000000u);
  const uint32_t u = (k == 0xFFFFFFFFu) ? 0x7fc00000u : ((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
  return xxh64_int(u);
}
template <> __device__ __forceinline__ uint64_t spark_hash_of_key<uint64_t>(uint64_t k, int dtype) {
  switch (dtype) {
    case ANV_F32: return spark_hash_of_key<uint32_t>((uint32_t)(k >> 32), ANV_F32);
    case ANV_I32: return spark_hash_of_key<uint32_t>((uint32_t)(k >> 32), ANV_I32);
    case ANV_I64: return xxh64_long(k ^ (1ull << 63));
    default: {
      const uint64_t u = (k == ~0ull) ? 0x7ff8000000000000ull : ((k >> 63) ? (k & ~(1ull << 63)) : ~k);
      return xxh64_long(u);
    }
  }
}

struct ColState {               // one per column, in the workspace
  unsigned long long n_valid;   // filled by pack_kernel: non-null, NONZERO values = keys that are sorted
  unsigned long long n_zero;    // filled by pack_kernel: non-null values equal to 0 (kept out of the sort, see pack)
  int cur;                      // which ping-pong buffer holds the current order
  int src[8];                   // per pass: source buffer
  int skip[8];                  // per pass: digit constant -> no scatter
  int error;                    // look-back spin limit hit (never expected): the host raises instead of hanging
};

template <typename K> struct TileSummary {
  K first_key, last_key, best_key;
  uint32_t n, prefix_len, suffix_len, best_len, heads_inside;
};

template <typename K> struct SortParams {
  const anv_column_t* cols;
  int n_cols;
  int64_t n_rows;
  int64_t stride;               // keys per column in each buffer
  int n_tiles;                  // ceil(n_rows / SORT_TILE)
  K* buf[2];
  ColState* state;
  uint32_t* tile_hist;          // [n_cols][256][n_tiles]  (digit-major)
  TileSummary<K>* summ;         // [n_cols][n_tiles]
  int pass;
  // one-sweep passes (decoupled look-back): no tile-histogram and no scan kernel
  uint32_t* ghist;              // [n_cols][sizeof(K)][256]  digit counts of the whole column, all passes, taken by pack_kernel
  uint32_t* gbase;              // [n_cols][sizeof(K)][256]  their exclusive scans
  unsigned long long* status;   // [n_cols][n_tiles][256]   (epoch << 56 | kind << 54 | count): tile aggregates / inclusive prefixes
  uint32_t* ticket;             // [n_cols][sizeof(K)]       tile ids are handed out in arrival order
  // optional by-product: HyperLogLog++ registers (Spark's approx_count_distinct) from the DISTINCT sorted keys
  int hll_p;                    // 0 = off; 4..12
  uint32_t* hll_regs;           // [n_cols][1 << hll_p], zeroed by the host wrapper
};
constexpr int PACK_TPC = 8;     // tiles per pack CTA (amortises the flush of the digit histograms)

// byte `pass` of the key: ONE PRMT (selector nibble 0 = the byte, the other result bytes come from the zero operand)
// instead of a shift and a mask - the digit is extracted three times per key and pass in the scatter.
template <typename K> __device__ __forceinline__ uint32_t digit_of(K k, int pass);
template <> __device__ __forceinline__ uint32_t digit_of<uint32_t>(uint32_t k, int pass) {
  return __byte_perm(k, 0u, 0x4440u | (uint32_t)pass);
}
template <> __device__ __forceinline__ uint32_t digit_of<uint64_t>(uint64_t k, int pass) {
  const uint32_t half = (pass & 4) ? (uint32_t)(k >> 32) : (uint32_t)k;
  return __byte_perm(half, 0u, 0x4440u | (uint32_t)(pass & 3));
}

// ---- pack: values -> keys, nulls dropped --------------------------------------------------
// One CTA per 4096-row tile: 128-bit loads, block-level compaction (one atomicAdd per CTA
// reserves the output range; the order before a sort is irrelevant), 64-byte runs per thread.
// Exact zeros are COUNTED here instead of being sorted: sparse / zero-inflated columns (70 % zeros in the
// benchmark's fourth family, > 90 % in the income dataset's capital-gain / capital-loss) then sort only their
// nonzero values; run_merge_kernel splices the zero run back into mode, distinct count and ranks.
template <typename K, typename T>
__device__ __forceinline__ void pack_tile(const SortParams<K>& P, const anv_column_t& col, int c, const int64_t tile, uint32_t* s_warp,
                                          unsigned long long* s_base, K* sk, uint32_t (*s_dh)[256]) {
  constexpr int VEC = Traits<T>::VEC;
  constexpr int PER = SORT_TILE / ANV_BLOCK;  // 16 rows per thread, contiguous
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = tile * SORT_TILE;
  const int n_tile = (int)min((int64_t)SORT_TILE, P.n_rows - r0);
  const T* __restrict__ data = reinterpret_cast<const T*>(col.data) + r0;
  const uint32_t* __restrict__ vbits = col.validity;
  const int row0 = tid * PER;
  K keys[PER];
  uint32_t okmask = 0;
  if (row0 + PER <= n_tile) {
    uint32_t vb = 0xFFFFu;
    if (vbits) {
      const int64_t g = r0 + row0;  // multiple of 16
      vb = (__ldg(vbits + (g >> 5)) >> (g & 31)) & 0xFFFFu;
    }
    okmask = vb;
    const uint4* p = reinterpret_cast<const uint4*>(data + row0);
#pragma unroll
    for (int v = 0; v < PER / VEC; ++v) {
      const uint4 q = ldg_stream(p + v);
      T e[VEC];
      unpack<T>(q, e);
#pragma unroll
      for (int i = 0; i < VEC; ++i) keys[v * VEC + i] = make_key<K, T>(e[i]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int row = row0 + i;
      bool ok = row < n_tile;
      keys[i] = 0;
      if (ok) {
        if (vbits) { const int64_t g = r0 + row; ok = (vbits[g >> 5] >> (g & 31)) & 1u; }
        keys[i] = make_key<K, T>(data[row]);
      }
      okmask |= ok ? (1u << i) : 0u;
    }
  }
  {  // take the zeros out (0.0 and -0.0 share one key; integers: 0)
    constexpr K ZERO_KEY = (K)1 << (sizeof(K) * 8 - 1);
    uint32_t zmask = 0;
#pragma unroll
    for (int i = 0; i < PER; ++i) zmask |= (keys[i] == ZERO_KEY) ? (1u << i) : 0u;
    zmask &= okmask;
    okmask &= ~zmask;
    const uint32_t wz = __reduce_add_sync(ANV_FULL, (uint32_t)__popc(zmask));
    if (lane == 0 && wz) atomicAdd(&P.state[c].n_zero, (unsigned long long)wz);
  }
  // block exclusive scan of the per-thread valid counts
  const uint32_t mine = __popc(okmask);
  uint32_t inc = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (tid == 0) {
    uint32_t acc = 0;
    for (int w = 0; w < ANV_WARPS; ++w) { const uint32_t t = s_warp[w]; s_warp[w] = acc; acc += t; }
    *s_base = acc ? atomicAdd(&P.state[c].n_valid, (unsigned long long)acc) : 0ull;
  }
  __syncthreads();
  // stage the compacted keys in shared memory, then write them out coalesced
  uint32_t o = s_warp[warp] + (inc - mine);
#pragma unroll
  for (int i = 0; i < PER; ++i)
    if ((okmask >> i) & 1u) sk[o++] = keys[i];
  __shared__ uint32_t s_total;
  if (tid == ANV_BLOCK - 1) s_total = s_warp[warp] + inc;
  __syncthreads();
  K* __restrict__ out = P.buf[0] + (size_t)c * P.stride + *s_base;
  const uint32_t total = s_total;
  // copy-out + the digit histograms of EVERY pass from the staged keys (the one-sweep passes need the column-wide digit counts
  // before the first scatter; taking them here replaces one full read of the keys per pass)
  if (P.ghist) {
    for (uint32_t i = tid; i < total; i += ANV_BLOCK) {
      const K k = sk[i];
      out[i] = k;
#pragma unroll
      for (int ps = 0; ps < (int)sizeof(K); ++ps) atomicAdd(&s_dh[ps][digit_of(k, ps)], 1u);
    }
  } else {
    for (uint32_t i = tid; i < total; i += ANV_BLOCK) out[i] = sk[i];
  }
  __syncthreads();   // sk / s_warp are reused by the CTA's next tile
}

// Strided variant (ANV_PACK_STRIDED): thread t takes rows t, t + 256, ... of the tile (coalesced scalar loads, the bitmap
// word of a warp's 32 rows is one broadcast load), a ballot per round ranks the surviving keys of the warp, and the staging
// stores land on CONSECUTIVE shared-memory words per warp.  The contiguous variant above (16 consecutive rows per thread)
// writes its staging stores 16 words apart - two banks per warp, 16-way conflicts (ncu: mio_throttle is its top stall).
template <typename T> __device__ __forceinline__ T ld_stream_scalar(const T* p);
template <> __device__ __forceinline__ float ld_stream_scalar<float>(const float* p) {
  float v; asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p)); return v;
}
template <> __device__ __forceinline__ int32_t ld_stream_scalar<int32_t>(const int32_t* p) {
  int32_t v; asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p)); return v;
}
template <> __device__ __forceinline__ double ld_stream_scalar<double>(const double* p) {
  double v; asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p)); return v;
}
template <> __device__ __forceinline__ int64_t ld_stream_scalar<int64_t>(const int64_t* p) {
  long long v; asm volatile("ld.global.nc.L1::no_allocate.s64 %0, [%1];" : "=l"(v) : "l"(p)); return (int64_t)v;
}

template <typename K, typename T>
__device__ __forceinline__ void pack_tile_strided(const SortParams<K>& P, const anv_column_t& col, int c, const int64_t tile, uint32_t* s_warp,
                                                  unsigned long long* s_base, K* sk, uint32_t (*s_dh)[256]) {
  constexpr int PER = SORT_TILE / ANV_BLOCK;        // 16 rounds of 256 rows
  constexpr int WREG = SORT_TILE / ANV_WARPS;       // a warp stages at most 16 x 32 keys: its own 512 slots of sk
  constexpr K ZERO_KEY = (K)1 << (sizeof(K) * 8 - 1);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = tile * SORT_TILE;              // multiple of 4096: the tile starts on a bitmap word
  const int n_tile = (int)min((int64_t)SORT_TILE, P.n_rows - r0);
  const T* __restrict__ data = reinterpret_cast<const T*>(col.data) + r0 + tid;
  const uint32_t* __restrict__ vw = col.validity ? col.validity + (r0 >> 5) + warp : nullptr;   // round i: word i * 8 + warp, bit = lane
  const uint32_t lbit = 1u << lane, lt = lbit - 1u;
  K* const mine = sk + warp * WREG;
  const bool full = n_tile == SORT_TILE;
  T x[PER];
  // the warp's 16 bitmap words (one per round), lane i holds round i's: one load per lane instead of 16 broadcast loads
  uint32_t wv = ANV_FULL;
  if (vw && lane < PER && (full || lane * ANV_BLOCK + warp * 32 < n_tile)) wv = __ldg(vw + lane * (ANV_BLOCK / 32));
#pragma unroll
  for (int i = 0; i < PER; ++i) {                   // all loads of the tile in flight at once
    const bool in = full || (i * ANV_BLOCK + tid) < n_tile;
    x[i] = in ? ld_stream_scalar<T>(data + i * ANV_BLOCK) : (T)0;
  }
  uint32_t wcount = 0, nzero = 0;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const K k = make_key<K, T>(x[i]);
    bool ok = (__shfl_sync(ANV_FULL, wv, i) & lbit) != 0u;
    if (!full) ok = ok && (i * ANV_BLOCK + tid) < n_tile;
    const bool zero = ok && k == ZERO_KEY;          // 0.0 and -0.0 share one key; integers: 0
    nzero += zero ? 1u : 0u;
    ok = ok && !zero;
    const uint32_t bal = __ballot_sync(ANV_FULL, ok);
    if (ok) mine[wcount + __popc(bal & lt)] = k;    // consecutive lanes, consecutive words
    wcount += __popc(bal);                          // warp-uniform
  }
  const uint32_t wz = __reduce_add_sync(ANV_FULL, nzero);
  if (lane == 0 && wz) atomicAdd(&P.state[c].n_zero, (unsigned long long)wz);
  if (lane == 0) s_warp[warp] = wcount;
  __syncthreads();
  if (tid == 0) {
    uint32_t acc = 0;
    for (int ww = 0; ww < ANV_WARPS; ++ww) { const uint32_t t = s_warp[ww]; s_warp[ww] = acc; acc += t; }
    *s_base = acc ? atomicAdd(&P.state[c].n_valid, (unsigned long long)acc) : 0ull;
  }
  __syncthreads();
  // every warp copies its own staged keys out (the order before a sort is irrelevant): contiguous, coalesced
  K* __restrict__ out = P.buf[0] + (size_t)c * P.stride + *s_base + s_warp[warp];
  if (P.ghist) {
    for (uint32_t j = lane; j < wcount; j += 32) {
      const K k = mine[j];
      out[j] = k;
#pragma unroll
      for (int ps = 0; ps < (int)sizeof(K); ++ps) atomicAdd(&s_dh[ps][digit_of(k, ps)], 1u);
    }
  } else {
    for (uint32_t j = lane; j < wcount; j += 32) out[j] = mine[j];
  }
  __syncthreads();   // sk / s_warp / s_base are reused by the CTA's next tile
}

#ifndef ANV_PACK_STRIDED
#define ANV_PACK_STRIDED 1   // measured (100 M x 12 float32, whole sort call): contiguous 27.29 ms, strided 26.38 ms, identical results
#endif
#if ANV_PACK_STRIDED
#define ANV_PACK_TILE pack_tile_strided
#else
#define ANV_PACK_TILE pack_tile
#endif

#ifndef ANV_PACK_MINB
#define ANV_PACK_MINB 6        // 40 registers, no spills for 32-bit keys (1: 26.64 ms, 5: 26.44, 6: 26.38); 64-bit keys: 5
#endif
template <typename K>
__global__ void __launch_bounds__(ANV_BLOCK, (sizeof(K) == 8 && ANV_PACK_MINB > 5) ? 5 : ANV_PACK_MINB) pack_kernel(const SortParams<K> P) {
  __shared__ uint32_t s_warp[ANV_WARPS];
  __shared__ unsigned long long s_base;
  __shared__ K sk[SORT_TILE];
  __shared__ uint32_t s_dh[sizeof(K)][256];
  const int c = blockIdx.y, tid = threadIdx.x;
  const anv_column_t col = P.cols[c];
#pragma unroll
  for (int ps = 0; ps < (int)sizeof(K); ++ps) s_dh[ps][tid] = 0;
  __syncthreads();
  for (int t = 0; t < PACK_TPC; ++t) {
    const int64_t tile = (int64_t)blockIdx.x * PACK_TPC + t;
    if (tile * SORT_TILE >= P.n_rows) break;
    switch (col.dtype) {
      case ANV_F32: ANV_PACK_TILE<K, float>(P, col, c, tile, s_warp, &s_base, sk, s_dh); break;
      case ANV_I32: ANV_PACK_TILE<K, int32_t>(P, col, c, tile, s_warp, &s_base, sk, s_dh); break;
      case ANV_F64: if (sizeof(K) == 8) ANV_PACK_TILE<K, double>(P, col, c, tile, s_warp, &s_base, sk, s_dh); break;
      case ANV_I64: if (sizeof(K) == 8) ANV_PACK_TILE<K, int64_t>(P, col, c, tile, s_warp, &s_base, sk, s_dh); break;
      default: break;
    }
  }
  if (!P.ghist) return;
  __syncthreads();
  uint32_t* g = P.ghist + (size_t)c * sizeof(K) * 256;
#pragma unroll
  for (int ps = 0; ps < (int)sizeof(K); ++ps) {
    const uint32_t v = s_dh[ps][tid];
    if (v) atomicAdd(&g[ps * 256 + tid], v);
  }
}

// Column-wide exclusive digit offsets of every pass + which passes are no-ops (one digit holds every key) + the ping-pong
// buffer each pass reads: everything the one-sweep passes need is known after the pack kernel.
template <typename K>
__global__ void __launch_bounds__(ANV_BLOCK) sort_bases_kernel(const SortParams<K> P) {
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  ColState& S = P.state[c];
  const unsigned long long n = S.n_valid;
  __shared__ uint32_t wsum[ANV_WARPS];
  __shared__ int s_skip[sizeof(K)];
  if (tid < (int)sizeof(K)) s_skip[tid] = (n == 0) ? 1 : 0;
  __syncthreads();
  for (int ps = 0; ps < (int)sizeof(K); ++ps) {
    const uint32_t v = P.ghist[((size_t)c * sizeof(K) + ps) * 256 + tid];
    if (n > 0 && (unsigned long long)v == n) s_skip[ps] = 1;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    uint32_t woff = 0;
#pragma unroll
    for (int w = 0; w < ANV_WARPS; ++w) woff += (w < warp) ? wsum[w] : 0u;
    P.gbase[((size_t)c * sizeof(K) + ps) * 256 + tid] = woff + inc - v;
    __syncthreads();
  }
  if (tid == 0) {
    int cur = 0;
    for (int ps = 0; ps < (int)sizeof(K); ++ps) {
      S.src[ps] = cur;
      S.skip[ps] = s_skip[ps];
      if (!s_skip[ps]) cur ^= 1;
    }
    S.cur = cur;
  }
}

// Lanes of `act` holding the same 8-bit digit.
// Default: per bit, one small NON-volatile asm block (and, setp, vote.ballot.sync, @!p not) gives the lanes whose bit equals
// mine, and the 8 masks are ANDed in C++.  ptxas turns this into R2P (7 digit bits into predicates at once), VOTE, a
// predicated NOT and a LOP3 AND: about 3 instructions per bit.  The same ballots written with __ballot_sync and a C++
// select compile to 6-7 per bit.  ptxas 12.9 for sm_90a does not finish the scatter kernels when all 8 bits sit in one asm
// block (selp + lop3 0x60), volatile or not, nor when the ANDs are written as asm lop3 next to these blocks.
// ANV_PEERS_MATCH=1: one MATCH.ANY over the whole warp, masked with `act` afterwards (lanes past the end of a partial tile
// hold digit 0: they must take part in the call but match no live lane).  Fewer instructions (sort_scatter_kernel<uint32>
// 1243 SASS against 1650) but slower on an H100 80GB HBM3 at 400 W, whole anv_mode_distinct call with ranks and HLL++,
// two alternating runs each: 100 M x 12 float32 47.8-48.2 ms against 40.7-40.8 ms with the ballots, 40 M x 150
// 83.2-84.5 ms against 72.4-72.7 ms (the C++ ballots before: 43.5-43.7 and 78.1-78.2 ms).
#ifndef ANV_PEERS_MATCH
#define ANV_PEERS_MATCH 0
#endif
__device__ __forceinline__ uint32_t peers8(uint32_t d, uint32_t act) {
#if ANV_PEERS_MATCH
  return __match_any_sync(ANV_FULL, d) & act;
#else
  uint32_t m = act;
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    uint32_t same;
    asm("{\n\t.reg .pred p;\n\t"
        "and.b32 %0, %1, %2;\n\t"
        "setp.ne.u32 p, %0, 0;\n\t"
        "vote.ballot.sync.b32 %0, p, 0xffffffff;\n\t"
        "@!p not.b32 %0, %0;\n\t}"
        : "=r"(same) : "r"(d), "r"(1u << b));
    m &= same;
  }
  return m;
#endif
}


// ---- pass step 1: per-tile digit histogram ------------------------------------------------------
// Plain shared-memory atomics (the hardware resolves same-address lanes itself; a match_any
// pre-aggregation only adds instructions).
#ifndef ANV_HIST_TPC
#define ANV_HIST_TPC 4
#endif
// tiles per tile-histogram CTA: the two dependent loads that start a CTA (column state, then keys) are paid once per 64 KB.
// The same knob on the scatter and the run summaries stays at 1.
constexpr int HIST_TPC = ANV_HIST_TPC;
template <typename K>
__global__ void __launch_bounds__(ANV_BLOCK) sort_hist_kernel(const SortParams<K> P) {
  const int c = blockIdx.y, tid = threadIdx.x;
  const ColState& S = P.state[c];
  const int64_t n = (int64_t)S.n_valid;
  const K* __restrict__ col_keys = (S.cur ? P.buf[1] : P.buf[0]) + (size_t)c * P.stride;
  __shared__ uint32_t h[256];
  const int sh = P.pass * 8;
  for (int tt = 0; tt < HIST_TPC; ++tt) {
    const int tile = blockIdx.x * HIST_TPC + tt;
    if (tile >= P.n_tiles) break;
    const int64_t t0 = (int64_t)tile * SORT_TILE;
    h[tid] = 0;
    __syncthreads();
    if (t0 < n) {
      const K* __restrict__ keys = col_keys + t0;
      const int nt = (int)min((int64_t)SORT_TILE, n - t0);
      constexpr int KV = 16 / sizeof(K);  // keys per 128-bit load
      const int nvec = nt / KV;
      const uint4* __restrict__ kv = reinterpret_cast<const uint4*>(keys);
      for (int j = tid; j < nvec; j += ANV_BLOCK) {
        const uint4 q = kv[j];
        if (sizeof(K) == 4) {
          atomicAdd(&h[(q.x >> sh) & 0xFFu], 1u); atomicAdd(&h[(q.y >> sh) & 0xFFu], 1u);
          atomicAdd(&h[(q.z >> sh) & 0xFFu], 1u); atomicAdd(&h[(q.w >> sh) & 0xFFu], 1u);
        } else {
          const uint64_t k0 = ((uint64_t)q.y << 32) | q.x, k1 = ((uint64_t)q.w << 32) | q.z;
          atomicAdd(&h[(uint32_t)(k0 >> sh) & 0xFFu], 1u); atomicAdd(&h[(uint32_t)(k1 >> sh) & 0xFFu], 1u);
        }
      }
      for (int i = nvec * KV + tid; i < nt; i += ANV_BLOCK) atomicAdd(&h[digit_of(keys[i], P.pass)], 1u);
    }
    __syncthreads();
    P.tile_hist[((size_t)c * 256 + tid) * P.n_tiles + tile] = h[tid];
    __syncthreads();
  }
}

// ---- pass step 2: exclusive scan of [256][n_tiles] per column + skip decision ------------------------------------
// Two launches with one CTA per (digit, column) - 256 x n_cols CTAs instead of n_cols (a batch of 15-50 columns left most of
// the SMs idle while a single CTA per column walked millions of entries):
//   sort_totals_kernel   digit_total[c][d] = sum over tiles of tile_hist[c][d][*]
//   sort_scan_kernel     base(d) = sum of the totals of the smaller digits (256 values, one warp scan per CTA), then the exclusive
//                        scan of the digit's own tile counts on top of it; the CTA of digit 0 also takes the device-side
//                        "one digit holds every key -> skip the pass" decision.
template <typename K>
__global__ void __launch_bounds__(ANV_BLOCK) sort_totals_kernel(const SortParams<K> P, uint32_t* __restrict__ totals) {
  const int d = blockIdx.x, c = blockIdx.y, tid = threadIdx.x;
  const uint32_t* __restrict__ a = P.tile_hist + ((size_t)c * 256 + d) * P.n_tiles;
  uint32_t acc = 0;
  const int n4 = P.n_tiles & ~3;
  if ((((size_t)c * 256 + d) * P.n_tiles & 3) == 0) {
    for (int i = tid * 4; i < n4; i += ANV_BLOCK * 4) { const uint4 q = *reinterpret_cast<const uint4*>(a + i); acc += q.x + q.y + q.z + q.w; }
    for (int i = n4 + tid; i < P.n_tiles; i += ANV_BLOCK) acc += a[i];
  } else {
    for (int i = tid; i < P.n_tiles; i += ANV_BLOCK) acc += a[i];
  }
  acc = __reduce_add_sync(ANV_FULL, acc);
  __shared__ uint32_t w[ANV_WARPS];
  if ((tid & 31) == 0) w[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    uint32_t t = 0;
    for (int i = 0; i < ANV_WARPS; ++i) t += w[i];
    totals[(size_t)c * 256 + d] = t;
  }
}

template <typename K>
__global__ void __launch_bounds__(ANV_BLOCK) sort_scan_kernel(const SortParams<K> P, const uint32_t* __restrict__ totals) {
  const int d = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  ColState& S = P.state[c];
  const unsigned long long n = S.n_valid;
  __shared__ uint32_t s_base, s_skip;
  __shared__ uint32_t wsum[ANV_WARPS + 1];
  if (tid == 0) s_skip = 0;
  __syncthreads();
  {  // base of this digit + skip decision from the 256 totals of the column (each thread owns one digit)
    const uint32_t t = totals[(size_t)c * 256 + tid];
    if (n > 0 && (unsigned long long)t == n) s_skip = 1;          // (benign race: every writer writes 1)
    uint32_t below = (tid < d) ? t : 0u;
    below = __reduce_add_sync(ANV_FULL, below);
    if (lane == 0) wsum[warp] = below;
    __syncthreads();
    if (tid == 0) {
      uint32_t b = 0;
      for (int i = 0; i < ANV_WARPS; ++i) b += wsum[i];
      s_base = b;
    }
    __syncthreads();
  }
  if (d == 0 && tid == 0) {
    const int skip = (n == 0) ? 1 : (int)s_skip;
    S.src[P.pass] = S.cur;
    S.skip[P.pass] = skip;
    if (!skip) S.cur ^= 1;
  }
  if (n == 0) return;
  uint32_t* a = P.tile_hist + ((size_t)c * 256 + d) * P.n_tiles;
  uint32_t carry = s_base;
  constexpr int PER = 8;
  for (int base = 0; base < P.n_tiles; base += ANV_BLOCK * PER) {
    uint32_t v[PER], run = 0;
    const int i0 = base + tid * PER;
#pragma unroll
    for (int k = 0; k < PER; ++k) { v[k] = (i0 + k < P.n_tiles) ? a[i0 + k] : 0u; run += v[k]; }
    uint32_t inc = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o);
      if (lane >= o) inc += t;
    }
    __syncthreads();                       // wsum of the previous chunk has been consumed
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    uint32_t woff = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < ANV_WARPS; ++w) { const uint32_t t = wsum[w]; woff += (w < warp) ? t : 0u; tot += t; }
    uint32_t ex = carry + woff + inc - run;
#pragma unroll
    for (int k = 0; k < PER; ++k) { if (i0 + k < P.n_tiles) a[i0 + k] = ex; ex += v[k]; }
    carry += tot;
  }
}

// ---- pass step 3: stable scatter ---------------------------------------------------------------
// Ranking: warp w owns 512 consecutive keys (16 rounds of 32); the lanes holding the same digit
// are found with 8 ballots (instead of one MATCH.ANY), all 16 rounds' loads and peer
// masks are computed up front (independent), then the warp-private digit counters are advanced
// round by round.  The tile is then REORDERED IN SHARED MEMORY into digit order, so the global
// writes are coalesced runs (full 32-byte sectors) instead of 4-byte scatters.
template <typename K> struct ScatShared {   // declared ONCE in the kernel (statics in the templated body would be replicated)
  uint16_t wcnt[SCAT_WARPS][256];             // <= 4096 keys per tile: 16 bits are enough
  uint32_t gbase[256];
  uint32_t wtot[8];
  K sk[SORT_TILE + 1];                        // + the spare slot of the branch-free placement
};

constexpr unsigned long long LB_AGG = 1ull << 54, LB_PREFIX = 2ull << 54, LB_VALUE = (1ull << 54) - 1ull;
constexpr int LB_SPIN_LIMIT = 1 << 20;

// Decoupled look-back of ONE digit: add up the aggregates of the preceding tiles until one that already knows its inclusive
// prefix, then publish this tile's inclusive prefix.  (Not inlined: keeps the spin loop out of the scatter's control flow.)
__device__ __noinline__ unsigned long long lookback_exclusive(volatile unsigned long long* status, int tile, int d, unsigned long long epoch,
                                                             unsigned long long total, int* error) {
  unsigned long long excl = 0;
  for (int t = tile - 1; t >= 0; --t) {
    unsigned long long v = status[(size_t)t * 256 + d];
    int spins = 0;
    while ((v >> 56) != (epoch >> 56)) {
      // never expected (tiles start in ticket order); once one look-back has given up every other one follows at once
      if (++spins > LB_SPIN_LIMIT || ((spins & 255) == 0 && *reinterpret_cast<volatile int*>(error))) { *error = 1; return excl; }
      v = status[(size_t)t * 256 + d];
    }
    excl += v & LB_VALUE;
    if (v & LB_PREFIX) break;
  }
  status[(size_t)tile * 256 + d] = epoch | LB_PREFIX | (excl + total);
  return excl;
}

// store through the global window (the opaque base pointer below would otherwise compile to a generic ST)
__device__ __forceinline__ void st_global_key(uint32_t* p, uint32_t v) { asm volatile("st.global.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_global_key(uint64_t* p, uint64_t v) { asm volatile("st.global.b64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }

template <typename K, bool FULL, bool LOOKBACK>
__device__ __forceinline__ void scatter_tile(const SortParams<K>& P, const ColState& S, const int c, const int tile, const int64_t t0,
                                             const int nt_in, ScatShared<K>& SH) {
  auto& wcnt = SH.wcnt;
  auto& gbase = SH.gbase;
  auto& wtot = SH.wtot;
  auto& sk = SH.sk;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nt = FULL ? SORT_TILE : nt_in;   // a full tile needs no bounds logic (all but the last tile of a column)
  const int src = S.src[P.pass];
  const K* __restrict__ in = (src ? P.buf[1] : P.buf[0]) + (size_t)c * P.stride + t0;
  K* __restrict__ out = (src ? P.buf[0] : P.buf[1]) + (size_t)c * P.stride;
  static_assert(SCAT_WARPS * 256 / 2 % SCAT_THREADS == 0, "the counters clear in whole rounds");
#pragma unroll
  for (int j = 0; j < SCAT_WARPS * 256 / 2 / SCAT_THREADS; ++j)   // fixed trip count: 4 stores, no loop control
    reinterpret_cast<uint32_t*>(&wcnt[0][0])[tid + j * SCAT_THREADS] = 0;
  if (!LOOKBACK && tid < 256) gbase[tid] = P.tile_hist[((size_t)c * 256 + tid) * P.n_tiles + tile];
  constexpr int WR = SORT_TILE / SCAT_WARPS / 32;  // 8 rounds per warp
  K key[WR];
  uint32_t peers[WR];
  const int w0 = warp * (SORT_TILE / SCAT_WARPS);
#pragma unroll
  for (int r = 0; r < WR; ++r) {
    const int i = w0 + r * 32 + lane;
    key[r] = (FULL || i < nt) ? in[i] : (K)0;
  }
  const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
  for (int r = 0; r < WR; ++r) {
    const bool ok = FULL || (w0 + r * 32 + lane) < nt;
    const uint32_t act = FULL ? ANV_FULL : __ballot_sync(ANV_FULL, ok);
    const uint32_t d = digit_of(key[r], P.pass);
    const uint32_t m = peers8(d, act);
    peers[r] = ok ? m : 0u;
  }
  __syncthreads();
  uint32_t pos[WR];
#pragma unroll
  for (int r = 0; r < WR; ++r) {
    const uint32_t m = peers[r];
    const uint32_t d = digit_of(key[r], P.pass);
    uint32_t before = 0;
    if (m) before = wcnt[warp][d];
    const uint32_t lower = m & lt;               // peers in lower lanes: none <=> this lane leads its group
    pos[r] = before + __popc(lower);
    __syncwarp();
    if (m && lower == 0) wcnt[warp][d] = (uint16_t)(before + __popc(m));
    __syncwarp();
  }
  __syncthreads();
  uint32_t total = 0;
  if (tid < 256) {  // exclusive prefix over warps for digit `tid`, tile total of the digit
    uint32_t acc = 0;
#pragma unroll
    for (int w = 0; w < SCAT_WARPS; ++w) { const uint32_t t = wcnt[w][tid]; wcnt[w][tid] = (uint16_t)acc; acc += t; }
    total = acc;
  }
  const unsigned long long epoch = (unsigned long long)(P.pass + 1) << 56;
  volatile unsigned long long* const status = LOOKBACK ? P.status + ((size_t)c * P.n_tiles) * 256 : nullptr;
  if (LOOKBACK && tid < 256)   // publish this tile's digit counts at once: its successors only need these to move on
    status[(size_t)tile * 256 + tid] = epoch | (tile == 0 ? LB_PREFIX : LB_AGG) | (unsigned long long)total;
  uint32_t ds_keep = 0;
  {  // exclusive scan of the 256 digit totals -> start of each digit inside the reordered tile
    uint32_t inc = total;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31 && warp < 8) wtot[warp] = inc;
    __syncthreads();
    if (tid < 256) {
      uint32_t woff = 0;
#pragma unroll
      for (int w = 0; w < 8; ++w) woff += (w < warp) ? wtot[w] : 0u;
      const uint32_t ds = woff + inc - total;
      // fold the digit's start into the per-warp offsets (one lookup when placing) and keep a single
      // "global base minus tile start" table for the copy-out (one lookup per key there as well)
#pragma unroll
      for (int w = 0; w < SCAT_WARPS; ++w) wcnt[w][tid] = (uint16_t)(wcnt[w][tid] + ds);
      if (LOOKBACK) ds_keep = ds;
      else gbase[tid] -= ds;
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < WR; ++r) {   // branch-free: lanes past the end of a partial tile write to the spare slot
    const uint32_t d = digit_of(key[r], P.pass);
    const uint32_t at = wcnt[warp][d] + pos[r];
    sk[(FULL || peers[r]) ? at : (uint32_t)SORT_TILE] = key[r];
  }
  if (LOOKBACK && tid < 256) {
    const unsigned long long excl = lookback_exclusive(status, tile, tid, epoch, (unsigned long long)total, &P.state[c].error);
    gbase[tid] = P.gbase[((size_t)c * sizeof(K) + P.pass) * 256 + tid] + (uint32_t)excl - ds_keep;
  }
  __syncthreads();
  // the column's output base as ONE 64-bit register pair (opaque to the compiler: it otherwise re-derives
  // c * stride + index in 64 bits for every key - 4 instructions per key of the copy-out)
  K* outc = out;
  asm volatile("" : "+l"(outc));
  if (FULL) {
#pragma unroll
    for (int j = 0; j < SORT_TILE / SCAT_THREADS; ++j) {
      const int p = tid + j * SCAT_THREADS;
      const K k = sk[p];
      st_global_key(outc + (gbase[digit_of(k, P.pass)] + (uint32_t)p), k);
    }
  } else {
    for (int p = tid; p < nt; p += SCAT_THREADS) {
      const K k = sk[p];
      st_global_key(outc + (gbase[digit_of(k, P.pass)] + (uint32_t)p), k);
    }
  }
}

#ifndef ANV_SCAT_TPC
#define ANV_SCAT_TPC 1
#endif
constexpr int SCAT_TPC = ANV_SCAT_TPC;   // tiles per scatter CTA (tuning knob)
template <typename K>
__global__ void __launch_bounds__(SCAT_THREADS, ANV_SCAT_MINB) sort_scatter_kernel(const SortParams<K> P) {
  const int c = blockIdx.y;
  const ColState& S = P.state[c];
  if (S.skip[P.pass]) return;
  const int64_t n = (int64_t)S.n_valid;
  __shared__ ScatShared<K> SH;
  for (int tt = 0; tt < SCAT_TPC; ++tt) {
    const int tile = blockIdx.x * SCAT_TPC + tt;
    const int64_t t0 = (int64_t)tile * SORT_TILE;
    if (t0 >= n) return;
    const int nt = (int)min((int64_t)SORT_TILE, n - t0);
    if (nt == SORT_TILE) scatter_tile<K, true, false>(P, S, c, tile, t0, nt, SH);
    else scatter_tile<K, false, false>(P, S, c, tile, t0, nt, SH);
    __syncthreads();            // the staging area and the digit tables are reused by the next tile
  }
}

// One-sweep pass: the same stable scatter, but the tile's global digit offsets come from the column-wide digit bases
// (sort_bases_kernel) + a decoupled look-back over the preceding tiles' digit counts - one read and one write of the keys per
// pass, no tile-histogram kernel, no scan kernel.  Tile ids are tickets (arrival order), so every tile a CTA waits for has
// already started: the look-back cannot deadlock.
template <typename K>
__global__ void __launch_bounds__(SCAT_THREADS, 2) sort_onesweep_kernel(const SortParams<K> P) {
  const int c = blockIdx.y;
  const ColState& S = P.state[c];
  if (S.skip[P.pass]) return;
  __shared__ int s_tile;
  if (threadIdx.x == 0) s_tile = (int)atomicAdd(&P.ticket[(size_t)c * sizeof(K) + P.pass], 1u);
  __syncthreads();
  const int tile = s_tile;
  const int64_t n = (int64_t)S.n_valid;
  const int64_t t0 = (int64_t)tile * SORT_TILE;
  if (t0 >= n) return;
  const int nt = (int)min((int64_t)SORT_TILE, n - t0);
  __shared__ ScatShared<K> SH;
  if (nt == SORT_TILE) scatter_tile<K, true, true>(P, S, c, tile, t0, nt, SH);
  else scatter_tile<K, false, true>(P, S, c, tile, t0, nt, SH);
}

// Associative combine of two ADJACENT run summaries (left, right) of sorted keys.
template <typename K> __device__ __forceinline__ void best_of(K& bk, uint32_t& bl, K k, uint32_t len) {
  if (len > bl) { bl = len; bk = k; }  // candidates arrive in ascending key order: strict > keeps the smallest key
}
template <typename K>
__device__ __forceinline__ TileSummary<K> combine(const TileSummary<K>& L, const TileSummary<K>& R) {
  if (L.n == 0) return R;
  if (R.n == 0) return L;
  TileSummary<K> o;
  const bool same = L.last_key == R.first_key;
  const bool Ls = L.prefix_len == L.n, Rs = R.prefix_len == R.n;  // the whole side is one run
  o.first_key = L.first_key; o.last_key = R.last_key; o.n = L.n + R.n;
  o.heads_inside = L.heads_inside + R.heads_inside + (same ? 0u : 1u);
  o.prefix_len = (Ls && same) ? L.n + R.prefix_len : L.prefix_len;
  o.suffix_len = (Rs && same) ? R.n + L.suffix_len : R.suffix_len;
  K bk = 0; uint32_t bl = 0;
  if (L.best_len) best_of(bk, bl, L.best_key, L.best_len);
  if (same) {
    if (!Ls && !Rs) best_of(bk, bl, L.last_key, L.suffix_len + R.prefix_len);
  } else {
    if (!Ls) best_of(bk, bl, L.last_key, L.suffix_len);
    if (!Rs) best_of(bk, bl, R.first_key, R.prefix_len);
  }
  if (R.best_len) best_of(bk, bl, R.best_key, R.best_len);
  o.best_key = bk; o.best_len = bl;
  return o;
}
template <typename K> __device__ __forceinline__ K shfl_down_key(K v, int d) {
  if (sizeof(K) == 8) return (K)__shfl_down_sync(ANV_FULL, (unsigned long long)v, d);
  return (K)__shfl_down_sync(ANV_FULL, (uint32_t)v, d);
}
template <typename K> __device__ __forceinline__ TileSummary<K> shfl_down_summary(const TileSummary<K>& s, int d) {
  TileSummary<K> r;
  r.first_key = shfl_down_key(s.first_key, d); r.last_key = shfl_down_key(s.last_key, d);
  r.best_key = shfl_down_key(s.best_key, d);
  r.n = __shfl_down_sync(ANV_FULL, s.n, d); r.prefix_len = __shfl_down_sync(ANV_FULL, s.prefix_len, d);
  r.suffix_len = __shfl_down_sync(ANV_FULL, s.suffix_len, d); r.best_len = __shfl_down_sync(ANV_FULL, s.best_len, d);
  r.heads_inside = __shfl_down_sync(ANV_FULL, s.heads_inside, d);
  return r;
}

// ---- run summary of the sorted keys --------------------------------------------------------------
// Each thread summarises 16 CONSECUTIVE sorted keys in registers (blocked 128-bit loads), the 256
// thread summaries are folded with the associative `combine` (shuffle tree per warp, then 8 warps
// sequentially): no shared-memory tile, no binary search, ~25 instructions per key.
#ifndef ANV_RUN_TPC
#define ANV_RUN_TPC 1
#endif
constexpr int RUN_TPC = ANV_RUN_TPC;     // tiles per run-summary CTA (tuning knob)
template <typename K>
__device__ __forceinline__ void run_tile_one(const SortParams<K>& P, const int c, const int tile) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const ColState& S = P.state[c];
  const int64_t n = (int64_t)S.n_valid;
  const int64_t t0 = (int64_t)tile * SORT_TILE;
  TileSummary<K>& out = P.summ[(size_t)c * P.n_tiles + tile];
  if (t0 >= n) { if (tid == 0) out.n = 0; return; }
  const int nt = (int)min((int64_t)SORT_TILE, n - t0);
  const K* __restrict__ keys = (S.cur ? P.buf[1] : P.buf[0]) + (size_t)c * P.stride + t0;
  constexpr int PER = SORT_TILE / ANV_BLOCK;  // 16
  constexpr int KV = 16 / sizeof(K);
  const int m = max(0, min(PER, nt - tid * PER));
  K k[PER];
  if (m == PER) {
    const uint4* p = reinterpret_cast<const uint4*>(keys + tid * PER);
#pragma unroll
    for (int v = 0; v < PER / KV; ++v) {
      const uint4 q = __ldg(p + v);
      if (sizeof(K) == 4) { k[v * 4] = (K)q.x; k[v * 4 + 1] = (K)q.y; k[v * 4 + 2] = (K)q.z; k[v * 4 + 3] = (K)q.w; }
      else { k[v * KV] = (K)(((uint64_t)q.y << 32) | q.x); k[v * KV + (KV > 1 ? 1 : 0)] = (K)(((uint64_t)q.w << 32) | q.z); }
    }
  } else {
#pragma unroll
    for (int j = 0; j < PER; ++j) k[j] = (j < m) ? keys[tid * PER + j] : (K)0;
  }
  TileSummary<K> s;
  s.n = m; s.first_key = k[0]; s.best_key = 0; s.best_len = 0; s.heads_inside = 0; s.prefix_len = 0;
  uint32_t run = 1;
  K last = k[0];
#pragma unroll
  for (int j = 1; j < PER; ++j) {
    if (j < m) {
      if (k[j] == k[j - 1]) {
        ++run;
      } else {
        if (s.heads_inside == 0) s.prefix_len = run;
        else if (run > s.best_len) { s.best_len = run; s.best_key = k[j - 1]; }
        ++s.heads_inside;
        run = 1;
      }
      last = k[j];
    }
  }
  s.last_key = last;
  s.suffix_len = m ? run : 0;
  if (s.heads_inside == 0) s.prefix_len = m;
  // HLL++ by-product: the registers are a max over the SET of values, so hashing one key per run (plus this thread's first
  // key, whose run may have started in the previous thread - a harmless repeat) replaces the pass over all values
  extern __shared__ __align__(16) uint32_t hll_sh[];
  const int hp = P.hll_p;
  if (hp) {
    // The run heads are first COMPACTED into shared memory (a thread holds between 1 and 16 of them: hashing in place would
    // keep every warp busy for the maximum over its lanes), then hashed by full warps straight against the column's global
    // registers: 2^p words that live in L1 / L2, read before the (rare) atomicMax.  A stale cached register can only be too
    // LOW (registers never decrease), which costs a redundant atomic, never a wrong result - so there is no per-tile copy
    // of the registers to clear and merge.
    K* hk = reinterpret_cast<K*>(hll_sh);                      // [SORT_TILE] head keys
    __shared__ uint32_t s_hw[ANV_WARPS + 1];
    uint32_t hcnt = 0;
#pragma unroll
    for (int j = 0; j < PER; ++j) hcnt += (j < m && (j == 0 || k[j] != k[j - 1])) ? 1u : 0u;
    uint32_t inc = hcnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) s_hw[warp] = inc;
    __syncthreads();
    if (tid == 0) {
      uint32_t acc = 0;
      for (int w2 = 0; w2 < ANV_WARPS; ++w2) { const uint32_t t = s_hw[w2]; s_hw[w2] = acc; acc += t; }
      s_hw[ANV_WARPS] = acc;
    }
    __syncthreads();
    uint32_t at = s_hw[warp] + inc - hcnt;
#pragma unroll
    for (int j = 0; j < PER; ++j)
      if (j < m && (j == 0 || k[j] != k[j - 1])) hk[at++] = k[j];
    __syncthreads();
    const uint32_t n_heads = s_hw[ANV_WARPS];
    const int dt = P.cols[c].dtype;
    uint32_t* G = P.hll_regs + ((size_t)c << hp);
    for (uint32_t i = tid; i < n_heads; i += ANV_BLOCK) {
      uint32_t idx, rho;
      hll_slot(spark_hash_of_key<K>(hk[i], dt), hp, idx, rho);
      if (rho > G[idx]) atomicMax(&G[idx], rho);
    }
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const TileSummary<K> right = shfl_down_summary(s, o);
    if ((lane & (2 * o - 1)) == 0) s = combine(s, right);
  }
  __shared__ TileSummary<K> ws[ANV_WARPS];
  if (lane == 0) ws[warp] = s;
  __syncthreads();
  if (tid == 0) {
    TileSummary<K> acc = ws[0];
#pragma unroll
    for (int w = 1; w < ANV_WARPS; ++w) acc = combine(acc, ws[w]);
    out = acc;
  }
}

template <typename K>
__global__ void __launch_bounds__(ANV_BLOCK) run_tile_kernel(const SortParams<K> P) {
  for (int tt = 0; tt < RUN_TPC; ++tt) {
    const int tile = blockIdx.x * RUN_TPC + tt;
    if (tile >= P.n_tiles) return;
    run_tile_one<K>(P, blockIdx.y, tile);
    __syncthreads();           // the shared staging (head keys, warp summaries) is reused by the next tile
  }
}

// One warp per column: 32 tile summaries per step are combined with an order-preserving
// shuffle tree, the chunk results sequentially by lane 0.  Also reads the requested order
// statistics straight out of the sorted keys.
constexpr int MERGE_WARPS = 8;
template <typename K>
__global__ void __launch_bounds__(32 * MERGE_WARPS) run_merge_kernel(const SortParams<K> P, double* mode_value, int64_t* mode_rows,
                                                       int64_t* n_distinct, const int64_t* ranks, int n_ranks,
                                                       double* rank_values) {
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const ColState& S = P.state[c];
  const int64_t n = (int64_t)S.n_valid;      // sorted (nonzero) keys
  const int64_t nz = (int64_t)S.n_zero;      // the zero run that pack_kernel kept out of the sort
  const int dt = P.cols[c].dtype;
  constexpr K ZERO_KEY = (K)1 << (sizeof(K) * 8 - 1);
  const K* __restrict__ sorted = (S.cur ? P.buf[1] : P.buf[0]) + (size_t)c * P.stride;
  int64_t below = 0;                          // keys smaller than zero: the zero run occupies ranks below+1 .. below+nz
  if (nz > 0 && n_ranks > 0) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (sorted[mid] < ZERO_KEY) lo = mid + 1; else hi = mid;
    }
    below = lo;
  }
  for (int r = tid; r < n_ranks; r += 32 * MERGE_WARPS) {
    const int64_t rk = ranks[(size_t)c * n_ranks + r];
    double v = nan("");
    if (rk > 0 && rk <= n + nz) {
      K k;
      if (rk <= below) k = sorted[rk - 1];
      else if (rk <= below + nz) k = ZERO_KEY;
      else k = sorted[rk - 1 - nz];
      v = sorted_key_to_double(sizeof(K) == 8 ? (uint64_t)k : ((uint64_t)k << 32), dt);
    }
    rank_values[(size_t)c * n_ranks + r] = v;
  }
  if (P.hll_p && nz > 0 && tid == 0) {   // the zero run never reached the sort: its value hashes here
    uint32_t idx, rho;
    hll_slot(spark_hash_of_key<K>(ZERO_KEY, dt), P.hll_p, idx, rho);
    atomicMax(&P.hll_regs[((size_t)c << P.hll_p) + idx], rho);
  }
  if (S.error) {                      // a look-back gave up: make the host raise (results would be garbage)
    if (tid == 0) { mode_value[c] = nan(""); mode_rows[c] = -3; n_distinct[c] = -3; }
    return;
  }
  if (n == 0) {
    if (tid == 0) {
      mode_value[c] = nz ? mode_slot_of_key(sizeof(K) == 8 ? (uint64_t)ZERO_KEY : ((uint64_t)ZERO_KEY << 32), dt) : nan("");
      mode_rows[c] = nz;
      n_distinct[c] = nz ? 1 : 0;
    }
    return;
  }
  const TileSummary<K>* T = P.summ + (size_t)c * P.n_tiles;
  const int tiles = (int)((n + SORT_TILE - 1) / SORT_TILE);
  // every warp folds a contiguous range of tile summaries (order-preserving shuffle tree over 32 at a time), warp 0 then
  // folds the warp results in order: 8 warps instead of one walk the 24 K summaries of a 100 M-row column
  const int wid = tid >> 5;
  const int per_warp = (tiles + MERGE_WARPS - 1) / MERGE_WARPS;
  const int w_lo = wid * per_warp, w_hi = min(tiles, w_lo + per_warp);
  TileSummary<K> acc;
  acc.n = 0;
  for (int t0 = w_lo; t0 < w_hi; t0 += 32) {
    TileSummary<K> mine;
    mine.n = 0;
    if (t0 + lane < w_hi) mine = T[t0 + lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const TileSummary<K> right = shfl_down_summary(mine, o);
      if ((lane & (2 * o - 1)) == 0) mine = combine(mine, right);
    }
    if (lane == 0) acc = combine(acc, mine);
  }
  __shared__ TileSummary<K> s_acc[MERGE_WARPS];
  if (lane == 0) s_acc[wid] = acc;
  __syncthreads();
  if (tid != 0) return;
  acc = s_acc[0];
  for (int w2 = 1; w2 < MERGE_WARPS; ++w2) acc = combine(acc, s_acc[w2]);
  if (lane == 0) {
    K bk = 0; uint32_t bl = 0;
    best_of(bk, bl, acc.first_key, acc.prefix_len);
    if (acc.best_len) best_of(bk, bl, acc.best_key, acc.best_len);
    if (acc.prefix_len != acc.n) best_of(bk, bl, acc.last_key, acc.suffix_len);
    int64_t rows = bl;
    if (nz > rows || (nz == rows && ZERO_KEY < bk)) { bk = ZERO_KEY; rows = nz; }   // ties: the smaller value
    mode_value[c] = mode_slot_of_key(sizeof(K) == 8 ? (uint64_t)bk : ((uint64_t)bk << 32), dt);
    mode_rows[c] = rows;
    n_distinct[c] = (int64_t)acc.heads_inside + 1 + (nz > 0 ? 1 : 0);
  }
}

template <typename K> struct Layout {
  size_t state, buf0, buf1, tile_hist, summ, totals, ghist, gbase, ticket, status, total;
  Layout(int n_cols, int64_t n_rows) {
    const int64_t stride = (n_rows + 63) & ~(int64_t)63;
    const int64_t n_tiles = (n_rows + SORT_TILE - 1) / SORT_TILE;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = (o + bytes + 255) & ~(size_t)255; return at; };
    state = take((size_t)n_cols * sizeof(ColState));
    buf0 = take((size_t)n_cols * stride * sizeof(K));
    buf1 = take((size_t)n_cols * stride * sizeof(K));
    tile_hist = take((size_t)n_cols * 256 * (n_tiles > 0 ? n_tiles : 1) * 4);
    summ = take((size_t)n_cols * (n_tiles > 0 ? n_tiles : 1) * sizeof(TileSummary<K>));
    totals = take((size_t)n_cols * 256 * 4);
    ghist = take((size_t)n_cols * sizeof(K) * 256 * 4);     // ghist, gbase, ticket, status are contiguous: one memset
    gbase = take((size_t)n_cols * sizeof(K) * 256 * 4);
    ticket = take((size_t)n_cols * sizeof(K) * 4);
    status = take((size_t)n_cols * (n_tiles > 0 ? n_tiles : 1) * 256 * 8);
    total = o + 256;
  }
};

template <typename K>
static int run_mode_distinct(const anv_column_t* cols, int n_cols, int64_t n_rows, double* mode_value, int64_t* mode_rows,
                             int64_t* n_distinct, const int64_t* ranks, int n_ranks, double* rank_values, int hll_p,
                             uint32_t* hll_regs, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  Layout<K> L(n_cols, n_rows);
  if (workspace_bytes < L.total) { set_error("anv_mode_distinct: workspace too small (%zu < %zu)", workspace_bytes, L.total); return ANV_ERR_WORKSPACE; }
  char* w = reinterpret_cast<char*>(workspace);
  SortParams<K> P{};
  P.cols = cols; P.n_cols = n_cols; P.n_rows = n_rows;
  P.stride = (n_rows + 63) & ~(int64_t)63;
  P.n_tiles = (int)((n_rows + SORT_TILE - 1) / SORT_TILE);
  if (P.n_tiles < 1) P.n_tiles = 1;
  P.buf[0] = reinterpret_cast<K*>(w + L.buf0);
  P.buf[1] = reinterpret_cast<K*>(w + L.buf1);
  P.state = reinterpret_cast<ColState*>(w + L.state);
  P.tile_hist = reinterpret_cast<uint32_t*>(w + L.tile_hist);
  P.summ = reinterpret_cast<TileSummary<K>*>(w + L.summ);
  uint32_t* totals = reinterpret_cast<uint32_t*>(w + L.totals);
  P.ghist = nullptr;                                   // set below when the one-sweep passes are selected
  P.gbase = reinterpret_cast<uint32_t*>(w + L.gbase);
  P.ticket = reinterpret_cast<uint32_t*>(w + L.ticket);
  P.status = reinterpret_cast<unsigned long long*>(w + L.status);
  P.hll_p = hll_regs ? hll_p : 0;
  P.hll_regs = hll_regs;
  if (hll_regs) ANV_CUDA(cudaMemsetAsync(hll_regs, 0, ((size_t)n_cols << hll_p) * sizeof(uint32_t), st));
  // Default: three kernels per pass (tile histogram, (digit, column)-parallel scan, stable scatter).  ANV_SORT_ONESWEEP=1 selects the
  // one-sweep passes for 32-bit keys (digit histograms in pack + decoupled look-back in the scatter: 10 instead of 14 words of
  // traffic per key).  The look-back walks several predecessor tiles per digit with dependent L2 round trips while the
  // scatter is issue-bound, not HBM-bound, so removing a read of the keys need not pay.  Kept, tested, not the default.
  const char* os_env = getenv("ANV_SORT_ONESWEEP");
  const bool legacy = !(os_env && os_env[0] == '1') || sizeof(K) != 4;
  ANV_CUDA(cudaMemsetAsync(P.state, 0, (size_t)n_cols * sizeof(ColState), st));
  if (!legacy) {
    P.ghist = reinterpret_cast<uint32_t*>(w + L.ghist);
    ANV_CUDA(cudaMemsetAsync(w + L.ghist, 0, L.total - 256 - L.ghist, st));   // digit counts, bases, tickets, look-back status
  }
  if (n_rows > 0) {
    dim3 grid(P.n_tiles, n_cols);
    pack_kernel<K><<<dim3((P.n_tiles + PACK_TPC - 1) / PACK_TPC, n_cols), ANV_BLOCK, 0, st>>>(P);
    ANV_CUDA(cudaGetLastError());
    // 64-bit keys keep the three-kernel passes: ptxas (12.9) does not terminate on the uint64 instantiation of the one-sweep kernel
    if constexpr (sizeof(K) == 4) {
      if (!legacy) {
        sort_bases_kernel<K><<<n_cols, ANV_BLOCK, 0, st>>>(P);
        for (int pass = 0; pass < (int)sizeof(K); ++pass) {
          P.pass = pass;
          sort_onesweep_kernel<K><<<grid, SCAT_THREADS, 0, st>>>(P);
          ANV_CUDA(cudaGetLastError());
        }
      }
    }
    if (legacy || sizeof(K) != 4) {
      for (int pass = 0; pass < (int)sizeof(K); ++pass) {
        P.pass = pass;
        sort_hist_kernel<K><<<dim3((P.n_tiles + HIST_TPC - 1) / HIST_TPC, n_cols), ANV_BLOCK, 0, st>>>(P);
        sort_totals_kernel<K><<<dim3(256, n_cols), ANV_BLOCK, 0, st>>>(P, totals);
        sort_scan_kernel<K><<<dim3(256, n_cols), ANV_BLOCK, 0, st>>>(P, totals);
        sort_scatter_kernel<K><<<dim3((P.n_tiles + SCAT_TPC - 1) / SCAT_TPC, n_cols), SCAT_THREADS, 0, st>>>(P);
        ANV_CUDA(cudaGetLastError());
      }
    }
    const size_t run_smem = P.hll_p ? (size_t)SORT_TILE * sizeof(K) : 0;   // the compacted head keys
    run_tile_kernel<K><<<dim3((P.n_tiles + RUN_TPC - 1) / RUN_TPC, n_cols), ANV_BLOCK, run_smem, st>>>(P);
    ANV_CUDA(cudaGetLastError());
  }
  run_merge_kernel<K><<<n_cols, 32 * MERGE_WARPS, 0, st>>>(P, mode_value, mode_rows, n_distinct, ranks, n_ranks, rank_values);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

// ---- one caller-filled column of 64-bit keys (keysort.cuh) ----------------------------------------------------------
// The same three kernels per pass as anv_mode_distinct's default path, on a single column whose keys the caller wrote
// into buf[0]: no pack kernel (nothing is dropped, zero keys are sorted like any other) and only the passes asked for.
struct KeySortLayout {
  size_t state, buf0, buf1, tile_hist, totals, total;
  explicit KeySortLayout(int64_t n_rows) {
    const int64_t n_tiles = (n_rows + SORT_TILE - 1) / SORT_TILE;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = (o + bytes + 255) & ~(size_t)255; return at; };
    state = take(sizeof(ColState));
    buf0 = take((size_t)(n_rows > 0 ? n_rows : 1) * sizeof(uint64_t));
    buf1 = take((size_t)(n_rows > 0 ? n_rows : 1) * sizeof(uint64_t));
    tile_hist = take((size_t)256 * (n_tiles > 0 ? n_tiles : 1) * 4);
    totals = take((size_t)256 * 4);
    total = o;
  }
};

__global__ void key_sort_init_kernel(ColState* S, int64_t n_rows) {
  ColState z{};
  z.n_valid = (unsigned long long)n_rows;
  *S = z;
}

size_t key_sort64_workspace_bytes(int64_t n_rows) { return KeySortLayout(n_rows).total; }

void key_sort64_bind(void* workspace, int64_t n_rows, KeySort64* out) {
  const KeySortLayout L(n_rows);
  char* w = reinterpret_cast<char*>(workspace);
  out->buf[0] = reinterpret_cast<uint64_t*>(w + L.buf0);
  out->buf[1] = reinterpret_cast<uint64_t*>(w + L.buf1);
  out->cur = &reinterpret_cast<ColState*>(w + L.state)->cur;
}

int key_sort64(void* workspace, size_t workspace_bytes, int64_t n_rows, int first_pass, int end_pass, cudaStream_t st) {
  const KeySortLayout L(n_rows);
  if (workspace_bytes < L.total) { set_error("key_sort64: workspace too small (%zu < %zu)", workspace_bytes, L.total); return ANV_ERR_WORKSPACE; }
  if (first_pass < 0 || end_pass > 8) { set_error("key_sort64: passes %d..%d outside 0..8", first_pass, end_pass); return ANV_ERR_INVALID; }
  char* w = reinterpret_cast<char*>(workspace);
  SortParams<uint64_t> P{};
  P.n_cols = 1;
  P.n_rows = n_rows;
  P.stride = n_rows;
  P.n_tiles = (int)((n_rows + SORT_TILE - 1) / SORT_TILE);
  if (P.n_tiles < 1) P.n_tiles = 1;
  P.buf[0] = reinterpret_cast<uint64_t*>(w + L.buf0);
  P.buf[1] = reinterpret_cast<uint64_t*>(w + L.buf1);
  P.state = reinterpret_cast<ColState*>(w + L.state);
  P.tile_hist = reinterpret_cast<uint32_t*>(w + L.tile_hist);
  uint32_t* totals = reinterpret_cast<uint32_t*>(w + L.totals);
  key_sort_init_kernel<<<1, 1, 0, st>>>(P.state, n_rows);
  ANV_CUDA(cudaGetLastError());
  if (n_rows == 0) return ANV_OK;
  for (int pass = first_pass; pass < end_pass; ++pass) {
    P.pass = pass;
    sort_hist_kernel<uint64_t><<<dim3((P.n_tiles + HIST_TPC - 1) / HIST_TPC, 1), ANV_BLOCK, 0, st>>>(P);
    sort_totals_kernel<uint64_t><<<dim3(256, 1), ANV_BLOCK, 0, st>>>(P, totals);
    sort_scan_kernel<uint64_t><<<dim3(256, 1), ANV_BLOCK, 0, st>>>(P, totals);
    sort_scatter_kernel<uint64_t><<<dim3((P.n_tiles + SCAT_TPC - 1) / SCAT_TPC, 1), SCAT_THREADS, 0, st>>>(P);
    ANV_CUDA(cudaGetLastError());
  }
  return ANV_OK;
}


// =====================================================================================================================
// Two-level bucket count for 32-bit keys (F32 / I32 columns): what mode / distinct / percentiles / HLL++ need is the
// multiset of keys grouped by value and a total order between groups, not a sorted array - so the columns are not sorted:
//   sample     32 * P keys per column (stratified row positions), sorted with the LSD kernels above (tiny);
//   split      P - 1 fine splitters = every 32nd sample key, plus the key of zero as a forced splitter (P = NS); every 32nd
//              fine splitter is also a coarse splitter (G - 1 of them, G = P / 32 coarse groups of 32 fine splitters), with
//              a 4096-cell lookup table over the top 12 key bits that narrows the coarse search to a few steps;
//   coarse     fused into the pack step, ONE read of the raw column: per 4096-row tile, nulls dropped and zeros counted
//              (as in pack_kernel), each key's coarse group found, the keys placed grouped by coarse group inside the tile
//              (one shared-memory atomic per key: unstable, the order inside a group does not matter) and written
//              coalesced to the tile's own range, with the (group, tile) counts in tile_hist's [256][n_tiles] shape;
//   offsets    sort_totals / sort_scan over that table: every (group, tile) segment's offset in group-major order;
//   fine       one CTA per chunk of <= 4096 consecutive group-major keys of one group: the chunk is gathered from its
//              tile segments into shared memory, each key's fine bucket found among the group's 32 splitters (5 steps);
//              keys EQUAL to a splitter are only counted (heavy hitters, discrete columns, NaN runs never move again), the
//              others are written back in fine-bucket order into the chunk's own range of the second buffer, with the
//              chunk's 34 bucket starts;
//   cum        prefix sums over the interleaved (bucket, splitter) counts: total order of the column => every requested
//              rank resolves to a splitter value directly or to (bucket, local rank); splitters that occur add to the
//              distinct count, the mode and the HLL++ registers once each;
//   count      one CTA per (group, column) walks the group's fine buckets: each bucket's chunk segments are copied into a
//              shared-memory stage while the bucket before is counted, in a shared-memory hash table sized from the
//              bucket's exact count (a bucket larger than the stage is streamed in pieces and swept by hash class), its
//              distinct keys hashed once into shared-memory HLL++ registers, and the ranks that land in it selected.
// Sizes are exact at every level: nothing is estimated, nothing overflows.  Global atomics happen once per (chunk,
// bucket) or per (CTA, register), never per key.  HBM traffic: one read of the column + 4 words per key that is not a
// splitter (written and read back twice) against ~14 for the LSD path; no ranking, no stable scatter.  Counting is
// integer everywhere => deterministic results (the placement inside a group is not, and does not matter).
constexpr uint32_t PC_ZERO_KEY = 0x80000000u;    // key of +-0.0 / integer 0: always a splitter, doubles as EMPTY in the hash table
constexpr int PC_OVERSAMPLE = 32;
constexpr int PC_LUT_BITS = 12;
constexpr int PC_LUT_CELLS = 1 << PC_LUT_BITS;
constexpr int PC_FPG = 32;                       // fine splitters per coarse group
constexpr int PC_MAX_P = 8192;                   // => at most 256 coarse groups: the rows of the (group, tile) table
constexpr int PC_CHUNK = 4096;                   // keys per fine-pass CTA
constexpr int PC_CST = PC_FPG + 2;               // chunk table row: start of each of the 33 fine buckets + the end
constexpr int PC_WIN = 512;                      // fine pass: tile segments located per round
constexpr int PC_TPC = 16;                       // coarse pass: tiles per CTA (amortises the coarse splitters and table)
constexpr int PC_SLOTS_LOG = 13;
constexpr int PC_SLOTS = 1 << PC_SLOTS_LOG;      // hash table slots per CTA (64 KB: keys + counts)
constexpr int PC_SWEEP_KEYS = 5120;              // keys one sweep of the table is sized for (<= 62.5 % load), and of a stage
constexpr int PC_GROUP_SMEM = PC_SLOTS * 8 + 2 * PC_SWEEP_KEYS * 4;   // count pass: table + 2 stage buffers, before HLL++
// Key values a direct bucket may span: 16-bit counters, two per word (32 KB).  2^15 covers a few % more keys but halves the
// CTAs per SM; at c3 on H100 (700 W) the count stage took 34.8 ms at 2^14 and 42.3 ms at 2^15.
constexpr int PC_DIRECT_RANGE = 1 << 14;
constexpr int PC_DIRECT_SMEM = PC_DIRECT_RANGE * 2 + PC_SWEEP_KEYS * 4;   // direct count: counters + 1 stage, before HLL++
constexpr int PC_MAX_RANKS = 16;

struct PcCol {                     // per column, in the workspace (zeroed per call)
  unsigned long long distinct;     // sum of the buckets' distinct counts + splitters that occur
  unsigned long long best;         // max over (multiplicity << 32 | ~key): the mode, ties -> smallest key
  int n_queries;                   // ranks that fall inside a bucket
  int q_bucket[PC_MAX_RANKS];
  uint32_t q_local[PC_MAX_RANKS];  // 1-based rank inside the bucket
  int q_slot[PC_MAX_RANKS];        // index into rank_values
};

struct PcParams {
  const anv_column_t* cols;
  int n_cols;
  int64_t n_rows;
  int64_t stride;                  // keys per column in each key buffer
  int n_tiles;
  int P, NS, NB, G;                // NS = P splitters (P - 1 from the sample + zero), NB = NS + 1 buckets, G = P / 32 groups
  int max_chunks;                  // fine chunks per column, upper bound: stride / PC_CHUNK + G
  int64_t m;                       // sample slots per column
  uint32_t* split;                 // [n_cols][NS]
  uint16_t* clut;                  // [n_cols][PC_LUT_CELLS + 1]  first coarse splitter >= each top-12-bit cell
  uint32_t* keys[2];               // [n_cols][stride]  coarse output (per tile, grouped) / fine output (group-major)
  ColState* state;                 // n_valid (nonzero keys) and n_zero per column, the scan's bookkeeping
  uint32_t* tile_hist;             // [n_cols][256][n_tiles]  keys per (group, tile); after the scan: group-major offset
  uint16_t* tile_start;            // [n_cols][256][n_tiles]  start of the group's keys inside the tile's range
  uint32_t* totals;                // [n_cols][256]           keys per group
  uint32_t* gstart;                // [n_cols][G + 1]         group-major offset of each group (+ the total)
  uint32_t* chunk_base;            // [n_cols][G + 1]         first fine chunk of each group (+ the total)
  uint16_t* cst;                   // [n_cols][PC_CST][max_chunks]  bucket starts inside each chunk's range, bucket-major
  uint32_t* cnt_lt;                // [n_cols][NB]  keys strictly between two splitters, per bucket
  uint32_t* cnt_eq;                // [n_cols][NS]  keys equal to each splitter (the zero run is added by pc_cum_kernel)
  uint32_t* cum;                   // [n_cols][2 * NB]  inclusive prefix over lt_0, eq_0, lt_1, eq_1, ...
  PcCol* st;
  int hll_p;                       // 0 = off
  uint32_t* hll_regs;              // [n_cols][1 << hll_p]
};

template <typename T> __device__ __forceinline__ T load_elem(const void* base, int64_t row) {
  return reinterpret_cast<const T*>(base)[row];
}

// ---- sample: m stratified row positions per column -> keys (nulls and zeros dropped), compacted into the LSD buffers ----
__global__ void __launch_bounds__(ANV_BLOCK) pc_sample_kernel(const SortParams<uint32_t> S, const int64_t n_rows, const int64_t m) {
  const int c = blockIdx.y;
  const anv_column_t col = S.cols[c];
  const int64_t i = (int64_t)blockIdx.x * ANV_BLOCK + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  bool ok = false;
  uint32_t key = 0;
  if (i < m) {
    const int64_t stride = n_rows / m > 0 ? n_rows / m : 1;
    uint32_t h = (uint32_t)i * 0x9E3779B1u + (uint32_t)c * 0x85EBCA6Bu;
    h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
    const int64_t row = i * stride + (int64_t)(h % (uint32_t)stride);
    if (row < n_rows) {
      ok = col.validity ? ((col.validity[row >> 5] >> (row & 31)) & 1u) : true;
      if (ok) {
        key = (col.dtype == ANV_F32) ? make_key<uint32_t, float>(load_elem<float>(col.data, row))
                                     : make_key<uint32_t, int32_t>(load_elem<int32_t>(col.data, row));
        ok = key != PC_ZERO_KEY;
      }
    }
  }
  __shared__ uint32_t s_w[ANV_WARPS];
  __shared__ unsigned long long s_base;
  const uint32_t bal = __ballot_sync(ANV_FULL, ok);
  if (lane == 0) s_w[warp] = __popc(bal);
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t acc = 0;
    for (int w = 0; w < ANV_WARPS; ++w) { const uint32_t t = s_w[w]; s_w[w] = acc; acc += t; }
    s_base = acc ? atomicAdd(&S.state[c].n_valid, (unsigned long long)acc) : 0ull;
  }
  __syncthreads();
  if (ok) S.buf[0][(size_t)c * S.stride + s_base + s_w[warp] + __popc(bal & ((1u << lane) - 1u))] = key;
}

// ---- split: fine splitters + the lookup table over the coarse ones, per column ---------------------------------------
__global__ void __launch_bounds__(256) pc_split_kernel(const SortParams<uint32_t> S, const PcParams P) {
  const int c = blockIdx.x, tid = threadIdx.x;
  const ColState& st = S.state[c];
  const uint32_t* __restrict__ sorted = (st.cur ? S.buf[1] : S.buf[0]) + (size_t)c * S.stride;
  const int64_t ms = (int64_t)st.n_valid;          // sample keys that survived (non-null, nonzero)
  const int ns = P.P - 1;                          // splitters taken from the sample
  auto sample_split = [&](int j) -> uint32_t {     // non-decreasing in j
    if (ms == 0) return PC_ZERO_KEY;
    int64_t idx = ((int64_t)(j + 1) * ms) / P.P;
    if (idx >= ms) idx = ms - 1;
    return sorted[idx];
  };
  int lo = 0, hi = ns;                             // z = number of sample splitters below the key of zero
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (sample_split(mid) < PC_ZERO_KEY) lo = mid + 1; else hi = mid; }
  const int z = lo;
  uint32_t* out = P.split + (size_t)c * P.NS;
  for (int j = tid; j < ns; j += 256) { const uint32_t v = sample_split(j); out[j < z ? j : j + 1] = v; }
  if (tid == 0) out[z] = PC_ZERO_KEY;
  __syncthreads();
  // coarse splitter j = fine splitter 32 j + 31 (j < G - 1): a key's coarse group is the number of coarse splitters below it
  uint16_t* lut = P.clut + (size_t)c * (PC_LUT_CELLS + 1);
  const int nc = P.G - 1;
  for (int q = tid; q <= PC_LUT_CELLS; q += 256) {
    int a = 0, b = nc;
    if (q == PC_LUT_CELLS) { a = nc; }
    else {
      const uint32_t v = (uint32_t)q << (32 - PC_LUT_BITS);
      while (a < b) { const int mid = (a + b) >> 1; if (out[mid * PC_FPG + PC_FPG - 1] < v) a = mid + 1; else b = mid; }
    }
    lut[q] = (uint16_t)a;
  }
}

// ---- coarse: raw column -> keys grouped by coarse group inside each tile ------------------------------------------------
template <typename T>
__device__ __forceinline__ void pc_coarse_tile(const PcParams& P, const anv_column_t& col, const int c, const int64_t tile,
                                               const uint32_t* sC, const uint16_t* sL, uint32_t* hc, uint32_t* s_warp, uint32_t* sk,
                                               uint32_t& n_zero, uint32_t& n_keys) {
  constexpr int PER = SORT_TILE / ANV_BLOCK;        // 16 rounds of 256 rows (the strided pack: coalesced scalar loads)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = tile * SORT_TILE;              // multiple of 4096: the tile starts on a bitmap word
  const int n_tile = (int)min((int64_t)SORT_TILE, P.n_rows - r0);
  const T* __restrict__ data = reinterpret_cast<const T*>(col.data) + r0 + tid;
  const uint32_t* __restrict__ vw = col.validity ? col.validity + (r0 >> 5) + warp : nullptr;
  const bool full = n_tile == SORT_TILE;
  uint32_t wv = ANV_FULL;                           // lane i holds the warp's bitmap word of round i
  if (vw && lane < PER && (full || lane * ANV_BLOCK + warp * 32 < n_tile)) wv = __ldg(vw + lane * (ANV_BLOCK / 32));
  T x[PER];
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const bool in = full || (i * ANV_BLOCK + tid) < n_tile;
    x[i] = in ? ld_stream_scalar<T>(data + i * ANV_BLOCK) : (T)0;
  }
  uint32_t key[PER], slot[PER];                     // slot: group << 16 | rank inside the group, ~0 = no key
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const uint32_t k = make_key<uint32_t, T>(x[i]);
    bool ok = (__shfl_sync(ANV_FULL, wv, i) >> lane) & 1u;
    if (!full) ok = ok && (i * ANV_BLOCK + tid) < n_tile;
    const bool zero = ok && k == PC_ZERO_KEY;      // 0.0 and -0.0 share one key; integers: 0
    n_zero += zero ? 1u : 0u;
    ok = ok && !zero;
    key[i] = k;
    slot[i] = ~0u;
    if (ok) {
      const uint32_t q = k >> (32 - PC_LUT_BITS);
      int lo = sL[q], hi = sL[q + 1];
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (sC[mid] < k) lo = mid + 1; else hi = mid; }
      slot[i] = ((uint32_t)lo << 16) | atomicAdd(&hc[lo], 1u);
    }
  }
  __syncthreads();
  // exclusive scan of the 256 group counts (thread = group; groups >= G hold 0) -> the (group, tile) table
  const uint32_t cnt = hc[tid];
  uint32_t inc = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  uint32_t woff = 0, total = 0;
#pragma unroll
  for (int w = 0; w < ANV_WARPS; ++w) { const uint32_t t = s_warp[w]; woff += (w < warp) ? t : 0u; total += t; }
  const uint32_t start = woff + inc - cnt;
  const size_t row = ((size_t)c * 256 + tid) * P.n_tiles + tile;
  P.tile_hist[row] = cnt;
  P.tile_start[row] = (uint16_t)start;
  hc[tid] = start;                                  // every thread read its own count above and nothing else
  __syncthreads();
#pragma unroll
  for (int i = 0; i < PER; ++i)
    if (slot[i] != ~0u) sk[hc[slot[i] >> 16] + (slot[i] & 0xFFFFu)] = key[i];
  __syncthreads();
  uint32_t* __restrict__ out = P.keys[0] + (size_t)c * P.stride + r0;
  for (uint32_t i = tid; i < total; i += ANV_BLOCK) out[i] = sk[i];
  if (tid == 0) n_keys += total;
  hc[tid] = 0;
  __syncthreads();                                  // sk / hc / s_warp are reused by the CTA's next tile
}

__global__ void __launch_bounds__(ANV_BLOCK, 4) pc_coarse_kernel(const PcParams P) {
  __shared__ uint32_t sC[PC_MAX_P / PC_FPG];
  __shared__ uint16_t sL[PC_LUT_CELLS + 1];
  __shared__ uint32_t hc[256], s_warp[ANV_WARPS];
  __shared__ uint32_t sk[SORT_TILE];
  const int c = blockIdx.y, tid = threadIdx.x;
  const anv_column_t col = P.cols[c];
  const uint32_t* S = P.split + (size_t)c * P.NS;
  if (tid < P.G - 1) sC[tid] = S[tid * PC_FPG + PC_FPG - 1];
  const uint16_t* L = P.clut + (size_t)c * (PC_LUT_CELLS + 1);
  for (int i = tid; i <= PC_LUT_CELLS; i += ANV_BLOCK) sL[i] = L[i];
  hc[tid] = 0;
  __syncthreads();
  uint32_t n_zero = 0, n_keys = 0;
  for (int t = 0; t < PC_TPC; ++t) {
    const int64_t tile = (int64_t)blockIdx.x * PC_TPC + t;
    if (tile >= P.n_tiles) break;
    if (col.dtype == ANV_F32) pc_coarse_tile<float>(P, col, c, tile, sC, sL, hc, s_warp, sk, n_zero, n_keys);
    else pc_coarse_tile<int32_t>(P, col, c, tile, sC, sL, hc, s_warp, sk, n_zero, n_keys);
  }
  n_zero = __reduce_add_sync(ANV_FULL, n_zero);
  if ((tid & 31) == 0 && n_zero) atomicAdd(&P.state[c].n_zero, (unsigned long long)n_zero);
  if (tid == 0 && n_keys) atomicAdd(&P.state[c].n_valid, (unsigned long long)n_keys);
}

// ---- group starts and fine chunks per column (after the (group, tile) scan) -----------------------------------------------
__global__ void __launch_bounds__(256) pc_chunks_kernel(const PcParams P) {
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t t = tid < P.G ? P.totals[(size_t)c * 256 + tid] : 0u;
  const uint32_t k = t / PC_CHUNK + (t % PC_CHUNK != 0u);   // (t + PC_CHUNK - 1) would wrap for t > 2^32 - PC_CHUNK
  uint32_t it = t, ik = k;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t a = __shfl_up_sync(ANV_FULL, it, o), b = __shfl_up_sync(ANV_FULL, ik, o);
    if (lane >= o) { it += a; ik += b; }
  }
  __shared__ uint32_t wt[8], wk[8];
  if (lane == 31) { wt[warp] = it; wk[warp] = ik; }
  __syncthreads();
  uint32_t ot = 0, ok = 0, tt = 0, tk = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) { ot += (w < warp) ? wt[w] : 0u; ok += (w < warp) ? wk[w] : 0u; tt += wt[w]; tk += wk[w]; }
  uint32_t* gs = P.gstart + (size_t)c * (P.G + 1);
  uint32_t* cb = P.chunk_base + (size_t)c * (P.G + 1);
  if (tid < P.G) { gs[tid] = ot + it - t; cb[tid] = ok + ik - k; }
  if (tid == 0) { gs[P.G] = tt; cb[P.G] = tk; }
}

// 4-byte cp.async copies into shared memory: a thread issues all of its copies before it waits for any
__device__ __forceinline__ void pc_cp_async4(uint32_t* dst, const uint32_t* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void pc_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void pc_cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// lower bound of k among the 32 sorted fine splitters of a group: 0..32 (32 only in the last group)
__device__ __forceinline__ uint32_t pc_fine_bucket(const uint32_t* sF, uint32_t k) {
  uint32_t f = (sF[15] < k) ? 16u : 0u;
  f += (sF[f + 7] < k) ? 8u : 0u;
  f += (sF[f + 3] < k) ? 4u : 0u;
  f += (sF[f + 1] < k) ? 2u : 0u;
  f += (sF[f] < k) ? 1u : 0u;
  return f + ((f == 31u && sF[31] < k) ? 1u : 0u);
}

// ---- fine: one CTA per chunk of <= 4096 group-major keys -------------------------------------------------------------
__global__ void __launch_bounds__(ANV_BLOCK) pc_fine_kernel(const PcParams P) {
  const int c = blockIdx.y, b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t* cb = P.chunk_base + (size_t)c * (P.G + 1);
  if ((uint32_t)b >= cb[P.G]) return;               // (uniform) the grid is sized for the largest possible chunk count
  __shared__ uint32_t sk[PC_CHUNK], sk2[PC_CHUNK];
  __shared__ uint32_t sO[PC_WIN + 1];
  __shared__ uint16_t sTS[PC_WIN];
  __shared__ uint32_t sF[PC_FPG], lc[PC_FPG + 1], ec[PC_FPG], ls[PC_CST];
  __shared__ int s_g, s_t0;
  const uint32_t* gs = P.gstart + (size_t)c * (P.G + 1);
  if (warp == 0) {
    int g = 0;
    if (lane == 0) {                                // the group owning chunk b: last g with cb[g] <= b
      int lo = 0, hi = P.G;
      while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (cb[mid] <= (uint32_t)b) lo = mid; else hi = mid - 1; }
      g = lo;
    }
    g = __shfl_sync(ANV_FULL, g, 0);
    const uint32_t p0 = gs[g] + ((uint32_t)b - cb[g]) * PC_CHUNK;
    // the tile whose segment holds p0: last t with O[t] <= p0, 32-ary search (O is non-decreasing over the tiles)
    const uint32_t* O = P.tile_hist + ((size_t)c * 256 + g) * P.n_tiles;
    int lo = 0, hi = P.n_tiles;
    while (hi - lo > 1) {
      const int step = (hi - lo + 31) / 32;
      const int idx = lo + lane * step;
      const uint32_t bal = __ballot_sync(ANV_FULL, idx < hi && O[idx] <= p0);   // lane 0 always: O[lo] <= p0
      lo += (31 - __clz(bal)) * step;
      hi = min(hi, lo + step);
    }
    if (lane == 0) { s_g = g; s_t0 = lo; }
  }
  if (tid < PC_FPG) ec[tid] = 0;
  if (tid <= PC_FPG) lc[tid] = 0;
  __syncthreads();
  const int g = s_g;
  const uint32_t gend = gs[g + 1];
  const uint32_t p0 = gs[g] + ((uint32_t)b - cb[g]) * PC_CHUNK;
  const uint32_t p1 = p0 + min((uint32_t)PC_CHUNK, gend - p0);   // p0 + PC_CHUNK may pass 2^32 in a column of < 2^32 keys
  const uint32_t* O = P.tile_hist + ((size_t)c * 256 + g) * P.n_tiles;
  const uint16_t* TS = P.tile_start + ((size_t)c * 256 + g) * P.n_tiles;
  const uint32_t* __restrict__ src = P.keys[0] + (size_t)c * P.stride;
  if (tid < PC_FPG) sF[tid] = P.split[(size_t)c * P.NS + g * PC_FPG + tid];
  // gather: the chunk's keys are the segments of consecutive tiles, in tile order; a round locates PC_WIN of them
  for (int t0 = s_t0;; t0 += PC_WIN) {
    for (int i = tid; i <= PC_WIN; i += ANV_BLOCK) {
      const int t = t0 + i;
      sO[i] = t < P.n_tiles ? O[t] : gend;
      if (i < PC_WIN && t < P.n_tiles) sTS[i] = TS[t];
    }
    __syncthreads();
    const uint32_t wlo = max(p0, sO[0]), whi = min(p1, sO[PC_WIN]);
    // positions relative to p0 (< PC_CHUNK): q += ANV_BLOCK could wrap past 2^32 near the end of a long column
    const uint32_t i1 = whi > p0 ? whi - p0 : 0u;
    for (uint32_t i = wlo - p0 + tid; i < i1; i += ANV_BLOCK) {
      const uint32_t q = p0 + i;
      int lo = 0, hi = PC_WIN - 1;                  // last i with sO[i] <= q
      while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (sO[mid] <= q) lo = mid; else hi = mid - 1; }
      pc_cp_async4(&sk[i], src + (size_t)(t0 + lo) * SORT_TILE + sTS[lo] + (q - sO[lo]));   // nothing waits for it
    }
    const bool done = whi >= p1;
    __syncthreads();                                // sO / sTS are refilled by the next round
    if (done) break;
  }
  pc_cp_commit();
  pc_cp_wait<0>();
  __syncthreads();
  // fine buckets: keys equal to a splitter are counted, the others ranked inside their bucket (unstable)
  constexpr int PER = PC_CHUNK / ANV_BLOCK;
  const uint32_t nk = p1 - p0;
  uint32_t slot[PER];
#pragma unroll
  for (int r = 0; r < PER; ++r) {
    const uint32_t i = tid + r * ANV_BLOCK;
    slot[r] = ~0u;
    if (i < nk) {
      const uint32_t k = sk[i];
      const uint32_t f = pc_fine_bucket(sF, k);
      if (f < PC_FPG && sF[f] == k) atomicAdd(&ec[f], 1u);
      else slot[r] = (f << 16) | atomicAdd(&lc[f], 1u);
    }
  }
  __syncthreads();
  if (warp == 0) {                                  // bucket starts inside the chunk: exclusive scan of lc[0..32]
    const uint32_t v = lc[lane];
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o); if (lane >= o) inc += t; }
    ls[lane] = inc - v;
    if (lane == 31) { ls[32] = inc; ls[33] = inc + lc[32]; }
  }
  __syncthreads();
  const int bucket0 = g * PC_FPG;
  if (tid < PC_CST) P.cst[((size_t)c * PC_CST + tid) * P.max_chunks + b] = (uint16_t)ls[tid];
  if (tid <= PC_FPG && lc[tid]) atomicAdd(&P.cnt_lt[(size_t)c * P.NB + bucket0 + tid], lc[tid]);
  if (tid >= 64 && tid < 64 + PC_FPG && ec[tid - 64]) atomicAdd(&P.cnt_eq[(size_t)c * P.NS + bucket0 + tid - 64], ec[tid - 64]);
#pragma unroll
  for (int r = 0; r < PER; ++r)
    if (slot[r] != ~0u) sk2[ls[slot[r] >> 16] + (slot[r] & 0xFFFFu)] = sk[tid + r * ANV_BLOCK];
  __syncthreads();
  uint32_t* __restrict__ out = P.keys[1] + (size_t)c * P.stride + p0;
  const uint32_t n_out = ls[PC_CST - 1];
  for (uint32_t i = tid; i < n_out; i += ANV_BLOCK) out[i] = sk2[i];
}

// ---- cum: total order of the column from the interleaved counts; rank queries; splitter contributions ---------------------
__global__ void __launch_bounds__(1024) pc_cum_kernel(const PcParams P, const int64_t* ranks, const int n_ranks, double* rank_values) {
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  PcCol& st = P.st[c];
  const uint32_t* cnt_lt = P.cnt_lt + (size_t)c * P.NB;
  const uint32_t* cnt_eq = P.cnt_eq + (size_t)c * P.NS;
  const uint32_t* S = P.split + (size_t)c * P.NS;
  const uint32_t nz = (uint32_t)P.state[c].n_zero;       // the zero run never left the coarse pass: it is splitter PC_ZERO_KEY's
  const int dt = P.cols[c].dtype;
  uint32_t* cum = P.cum + (size_t)c * 2 * P.NB;
  const int n_ent = 2 * P.NB - 1;                                     // lt_0, eq_0, lt_1, ..., eq_{NS-1}, lt_NS
  const int per = (n_ent + 1023) / 1024;
  const int e0 = tid * per, e1 = min(e0 + per, n_ent);
  auto entry = [&](int e) -> uint32_t {
    if (!(e & 1)) return cnt_lt[e >> 1];
    const int i = e >> 1;                                              // the zero run goes to the first splitter of zero
    return cnt_eq[i] + ((S[i] == PC_ZERO_KEY && (i == 0 || S[i - 1] != PC_ZERO_KEY)) ? nz : 0u);
  };
  unsigned long long run = 0, eq_distinct = 0, best = 0;
  for (int e = e0; e < e1; ++e) {
    const uint32_t n = entry(e);
    run += n;
    if ((e & 1) && n) {
      const uint32_t k = S[e >> 1];
      ++eq_distinct;
      const unsigned long long cand = ((unsigned long long)n << 32) | (uint32_t)~k;
      if (cand > best) best = cand;
      if (P.hll_p) {
        uint32_t idx, rho;
        hll_slot(spark_hash_of_key<uint32_t>(k, dt), P.hll_p, idx, rho);
        uint32_t* G = P.hll_regs + ((size_t)c << P.hll_p);
        if (rho > G[idx]) atomicMax(&G[idx], rho);
      }
    }
  }
  __shared__ unsigned long long wsum[32];
  __shared__ unsigned long long wbest[32], wdist[32];
  unsigned long long inc = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(ANV_FULL, inc, o); if (lane >= o) inc += t; }
  unsigned long long rb = best, rd = eq_distinct;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long ob = __shfl_down_sync(ANV_FULL, rb, o); if (ob > rb) rb = ob;
    rd += __shfl_down_sync(ANV_FULL, rd, o);
  }
  if (lane == 31) wsum[warp] = inc;
  if (lane == 0) { wbest[warp] = rb; wdist[warp] = rd; }
  __syncthreads();
  if (warp == 0) {
    const unsigned long long w = wsum[lane];
    unsigned long long wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(ANV_FULL, wi, o); if (lane >= o) wi += t; }
    wsum[lane] = wi - w;
    unsigned long long b2 = wbest[lane], d2 = wdist[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ob = __shfl_down_sync(ANV_FULL, b2, o); if (ob > b2) b2 = ob;
      d2 += __shfl_down_sync(ANV_FULL, d2, o);
    }
    if (lane == 0) { if (b2) atomicMax(&st.best, b2); if (d2) atomicAdd(&st.distinct, d2); }
  }
  __syncthreads();
  unsigned long long acc = wsum[warp] + inc - run;
  for (int e = e0; e < e1; ++e) { acc += entry(e); cum[e] = (uint32_t)acc; }
  __syncthreads();
  // rank queries: first entry whose inclusive prefix reaches the rank
  if (tid < n_ranks) {
    const int64_t rk = ranks[(size_t)c * n_ranks + tid];
    const unsigned long long total = n_ent > 0 ? cum[n_ent - 1] : 0;
    double v = nan("");
    if (rk > 0 && (unsigned long long)rk <= total) {
      int lo = 0, hi = n_ent - 1;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if ((unsigned long long)cum[mid] < (unsigned long long)rk) lo = mid + 1; else hi = mid; }
      if (lo & 1) {
        v = sorted_key_to_double((uint64_t)S[lo >> 1] << 32, dt);
      } else {
        const int q = atomicAdd(&st.n_queries, 1);
        st.q_bucket[q] = lo >> 1;
        st.q_local[q] = (uint32_t)(rk - (lo ? cum[lo - 1] : 0));
        st.q_slot[q] = tid;
      }
    }
    rank_values[(size_t)c * n_ranks + tid] = v;
  }
}

// ---- count: one CTA per (group, column) walks the group's fine buckets ------------------------------------------------------
// A bucket's keys are copied into a shared-memory stage with cp.async before they are counted, and the next bucket's copies
// are issued before this one is counted: every thread keeps all of its copies in flight at once, and the count's shared
// atomics never wait for HBM.
struct PcCursor { uint32_t j, q; };  // next key of a bucket to stage: q keys into chunk j's segment (j = cb1: none left)

struct PcStageScratch {              // one window of a bucket's segment list
  uint32_t off[ANV_BLOCK], len[ANV_BLOCK], src[ANV_BLOCK];
  uint32_t wsum[ANV_WARPS];
  uint32_t cut_j, cut_q;
};

// Issues the copies of the next (at most PC_SWEEP_KEYS) keys of fine bucket f into dst and returns how many; `cur` moves
// past them.  The segment list is walked ANV_BLOCK chunks at a time (a group can span thousands of chunks): thread t reads
// chunk j + t's start and end (coalesced: cst is bucket-major), a block scan places the segments in the stage, and warp w
// issues the copies of segments w, w + 8, ...  Nothing waits for the copies.  Every thread of the CTA calls it (barriers).
__device__ uint32_t pc_stage_fill(const PcParams& P, const int c, const int f, const uint32_t* keys, const uint32_t cb0,
                                  const uint32_t cb1, PcCursor& cur, uint32_t* dst, PcStageScratch& S) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint16_t* starts = P.cst + ((size_t)c * PC_CST + f) * P.max_chunks;   // + max_chunks: the segment ends
  uint32_t n = 0;
  while (cur.j < cb1 && n < PC_SWEEP_KEYS) {
    const uint32_t j = cur.j + tid;
    uint32_t s = 0, len = 0;
    if (j < cb1) {
      s = starts[j];
      len = starts[j + P.max_chunks] - s;
      if (tid == 0) { s += cur.q; len -= cur.q; }
    }
    uint32_t inc = len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) S.wsum[warp] = inc;
    __syncthreads();
    uint32_t woff = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < ANV_WARPS; ++w) { const uint32_t t = S.wsum[w]; woff += (w < warp) ? t : 0u; tot += t; }
    const uint32_t off = n + woff + inc - len;       // the segment's place in the stage
    S.off[tid] = off;
    S.len[tid] = len;
    S.src[tid] = (j - cb0) * PC_CHUNK + s;
    if (len && off <= (uint32_t)PC_SWEEP_KEYS && (uint32_t)PC_SWEEP_KEYS < off + len) {   // the stage ends inside it
      S.cut_j = j;
      S.cut_q = (tid == 0 ? cur.q : 0u) + (PC_SWEEP_KEYS - off);
    }
    __syncthreads();
    const uint32_t nwin = min(cb1 - cur.j, (uint32_t)ANV_BLOCK);
    for (uint32_t t = warp; t < nwin; t += ANV_WARPS) {
      const uint32_t o = S.off[t];
      if (o >= (uint32_t)PC_SWEEP_KEYS) break;       // (uniform per warp) the offsets do not decrease
      const uint32_t m = min(S.len[t], (uint32_t)PC_SWEEP_KEYS - o);
      const uint32_t* from = keys + S.src[t];
      for (uint32_t q = lane; q < m; q += 32) pc_cp_async4(dst + o + q, from + q);
    }
    if (n + tot <= (uint32_t)PC_SWEEP_KEYS) { n += tot; cur.j += nwin; cur.q = 0; }
    else { n = PC_SWEEP_KEYS; cur.j = S.cut_j; cur.q = S.cut_q; }
    __syncthreads();                                  // S is rewritten by the next window
  }
  return n;
}

// The one rule that splits the nonempty fine buckets between the two count kernels.  A bucket holds only keys strictly
// between its neighbouring splitters lo and hi (lo = -1 below the first one, hi = 2^32 above the last), so it spans at
// most R = hi - lo - 1 key values, known before anything is counted.  It is direct - counted by pc_direct_kernel in
// 16-bit counters indexed by k - lo - 1 - when R <= PC_DIRECT_RANGE and its n keys fit a 16-bit counter; all other
// buckets go to pc_group_kernel's hash table.  In float data a bucket of a few thousand keys spans few representable values.
__device__ __forceinline__ bool pc_is_direct(const uint32_t* split, const int NS, const int bucket, const uint32_t n) {
  const int64_t lo = bucket > 0 ? (int64_t)split[bucket - 1] : -1;
  const int64_t hi = bucket < NS ? (int64_t)split[bucket] : (int64_t)1 << 32;
  return n < (1u << 16) && hi - lo - 1 <= PC_DIRECT_RANGE;
}

__global__ void __launch_bounds__(ANV_BLOCK, 2) pc_group_kernel(const PcParams P, const int n_ranks, double* rank_values) {
  const int g = blockIdx.x, c = blockIdx.y, tid = threadIdx.x;
  const uint32_t cb0 = P.chunk_base[(size_t)c * (P.G + 1) + g], cb1 = P.chunk_base[(size_t)c * (P.G + 1) + g + 1];
  if (cb0 == cb1) return;                               // (uniform) no key between this group's splitters
  const int nf = (g == P.G - 1) ? PC_FPG + 1 : PC_FPG;  // the last group also holds the keys above the top splitter
  __shared__ uint32_t s_cnt[PC_FPG + 1];
  uint32_t n_hash = 0;                                  // direct buckets count as empty here
  if (tid < nf) {
    const int bucket = g * PC_FPG + tid;
    n_hash = P.cnt_lt[(size_t)c * P.NB + bucket];
    if (pc_is_direct(P.split + (size_t)c * P.NS, P.NS, bucket, n_hash)) n_hash = 0;
  }
  if (tid <= PC_FPG) s_cnt[tid] = n_hash;
  if (!__syncthreads_or(n_hash != 0)) return;           // (uniform) every bucket of the group is direct or empty
  extern __shared__ __align__(16) uint32_t pc_tab[];
  uint32_t* tkey = pc_tab;
  uint32_t* tcnt = pc_tab + PC_SLOTS;
  uint32_t* stage = pc_tab + 2 * PC_SLOTS;              // [2][PC_SWEEP_KEYS] two stage buffers
  uint32_t* sreg = stage + 2 * PC_SWEEP_KEYS;           // [1 << hll_p] this CTA's HLL++ registers
  __shared__ PcStageScratch S;
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_sel[2];
  __shared__ int s_full;
  PcCol& st = P.st[c];
  const int dt = P.cols[c].dtype;
  const int hp = P.hll_p;
  const uint32_t* __restrict__ keys = P.keys[1] + (size_t)c * P.stride + P.gstart[(size_t)c * (P.G + 1) + g];
  // the table is cleared once: every bucket and every sweep leaves the slots it used empty again
  for (int i = tid; i < PC_SLOTS; i += ANV_BLOCK) { tkey[i] = PC_ZERO_KEY; tcnt[i] = 0; }
  if (hp) for (int i = tid; i < (1 << hp); i += ANV_BLOCK) sreg[i] = 0;
  if (tid == 0) s_full = 0;
  __syncthreads();
  unsigned long long best = 0;
  uint32_t distinct = 0;
  auto fold = [&](uint32_t k, uint32_t cnt) {           // one distinct key of the bucket, with its multiplicity
    ++distinct;
    const unsigned long long cand = ((unsigned long long)cnt << 32) | (uint32_t)~k;
    if (cand > best) best = cand;
    if (hp) {
      uint32_t idx, rho;
      hll_slot(spark_hash_of_key<uint32_t>(k, dt), hp, idx, rho);
      atomicMax(&sreg[idx], rho);
    }
  };
  // counts k in the table's first 1 << tlog slots: its slot (claimed: k took an empty one), or ~0u when they are all taken
  auto insert = [&](uint32_t k, int tlog, bool& claimed) -> uint32_t {
    const uint32_t mask = (1u << tlog) - 1u;
    uint32_t slot = (k * 0x9E3779B1u) >> (32 - tlog);
    for (uint32_t probes = 0; probes <= mask; ++probes) {
      const uint32_t prev = atomicCAS(&tkey[slot], PC_ZERO_KEY, k);
      if (prev == PC_ZERO_KEY || prev == k) { atomicAdd(&tcnt[slot], 1u); claimed = prev == PC_ZERO_KEY; return slot; }
      slot = (slot + 1) & mask;
    }
    claimed = false;
    return ~0u;
  };
  // requested ranks inside a bucket: 4-pass radix select, each pass over the bucket's keys as each_key visits them
  auto select = [&](const int bucket, auto&& each_key) {
    const int nq = st.n_queries;
    for (int q = 0; q < nq; ++q) {
      if (st.q_bucket[q] != bucket) continue;           // uniform across the CTA
      uint32_t prefix = 0, r = st.q_local[q];
      for (int pass = 3; pass >= 0; --pass) {
        s_hist[tid] = 0;
        __syncthreads();
        const int sh = pass * 8;
        each_key([&](uint32_t k) {
          if (pass == 3 || ((k ^ prefix) >> (sh + 8)) == 0) atomicAdd(&s_hist[(k >> sh) & 0xFFu], 1u);
        });
        __syncthreads();
        if (tid == 0) {
          uint32_t acc = 0, d = 0;
          for (; d < 255; ++d) { if (acc + s_hist[d] >= r) break; acc += s_hist[d]; }
          s_sel[0] = d; s_sel[1] = r - acc;
        }
        __syncthreads();
        prefix |= s_sel[0] << sh;
        r = s_sel[1];
        __syncthreads();
      }
      if (tid == 0) rank_values[(size_t)c * n_ranks + st.q_slot[q]] = sorted_key_to_double((uint64_t)prefix << 32, dt);
    }
  };
  auto next_bucket = [&](int f) { do ++f; while (f < nf && s_cnt[f] == 0); return f; };
  int buf = 0;                                          // stage buffer of the current bucket
  bool staged = false;                                  // its copies were issued with the bucket before
  for (int f = next_bucket(-1), fn; f < nf; f = fn) {
    const int bucket = g * PC_FPG + f;
    const uint32_t n = s_cnt[f];
    fn = next_bucket(f);
    if (n <= (uint32_t)PC_SWEEP_KEYS) {
      // ---- the bucket fits the stage: counted from shared memory while the next one is copied into the other buffer
      uint32_t* sk = stage + buf * PC_SWEEP_KEYS;
      if (!staged) { PcCursor cu{cb0, 0}; pc_stage_fill(P, c, f, keys, cb0, cb1, cu, sk, S); pc_cp_commit(); }
      staged = fn < nf && s_cnt[fn] <= (uint32_t)PC_SWEEP_KEYS;
      if (staged) {
        PcCursor cu{cb0, 0};
        pc_stage_fill(P, c, fn, keys, cb0, cb1, cu, stage + (buf ^ 1) * PC_SWEEP_KEYS, S);
        pc_cp_commit();
        pc_cp_wait<1>();
      } else {
        pc_cp_wait<0>();
      }
      __syncthreads();
      // one sweep: the table holds n keys at <= 62.5 % load, so it never fills up
      int tlog = 9;
      while (tlog < PC_SLOTS_LOG && (5u << tlog) < 8u * n) ++tlog;
      uint32_t owned = 0;                               // bit r: this thread's key tid + r * ANV_BLOCK claimed a slot
      for (uint32_t i = tid, r = 0; i < n; i += ANV_BLOCK, ++r) {
        bool claimed;
        const uint32_t slot = insert(sk[i], tlog, claimed);
        if (claimed) { sk[i] = slot; owned |= 1u << r; }
      }
      __syncthreads();
      while (owned) {                                   // each distinct key is folded by the thread that claimed its slot
        const uint32_t i = tid + (__ffs(owned) - 1) * ANV_BLOCK;
        owned &= owned - 1;
        const uint32_t slot = sk[i], k = tkey[slot];
        fold(k, tcnt[slot]);
        tkey[slot] = PC_ZERO_KEY;
        tcnt[slot] = 0;
        sk[i] = k;                                      // the stage holds the bucket's keys again, for the select
      }
      __syncthreads();
      select(bucket, [&](auto&& fn_key) { for (uint32_t i = tid; i < n; i += ANV_BLOCK) fn_key(sk[i]); });
      buf ^= 1;
    } else {
      // ---- a larger bucket is streamed through both buffers in pieces, each piece copied while the one before is counted.
      // Its keys are swept by hash classes, the top `lv` bits of k * odd (a bijection).  A class whose distinct keys do not
      // fit the table is split in two; a class of 2^13 hash values holds at most 2^13 distinct keys, so the splitting
      // stops by lv = 19.  Every sweep streams all the pieces again.
      int lv0 = 0;
      while ((n >> lv0) > (uint32_t)PC_SWEEP_KEYS) ++lv0;
      int lv = lv0;
      uint64_t lo = 0;                                  // first hash value of the current class
      int b = 0;
      PcCursor cu{cb0, 0};
      uint32_t m_next = pc_stage_fill(P, c, f, keys, cb0, cb1, cu, stage, S);
      pc_cp_commit();
      while (true) {
        const uint32_t cls = (uint32_t)(lo >> (32 - lv));
        bool last;
        do {
          const uint32_t m = m_next;
          last = cu.j >= cb1;
          if (last) cu = PcCursor{cb0, 0};              // the piece after the last is the first again, for the next sweep
          m_next = pc_stage_fill(P, c, f, keys, cb0, cb1, cu, stage + (b ^ 1) * PC_SWEEP_KEYS, S);
          pc_cp_commit();
          pc_cp_wait<1>();
          __syncthreads();
          const uint32_t* sk = stage + b * PC_SWEEP_KEYS;
          for (uint32_t i = tid; i < m; i += ANV_BLOCK) {
            const uint32_t k = sk[i];
            if (((k * 0x85EBCA6Bu) >> (32 - lv)) != cls) continue;
            bool claimed;
            if (insert(k, PC_SLOTS_LOG, claimed) == ~0u) s_full = 1;
          }
          __syncthreads();                              // the buffer is refilled by the next piece
          b ^= 1;
        } while (!last);
        const int full = s_full;
        for (int i = tid; i < PC_SLOTS; i += ANV_BLOCK) {   // fold the class (unless it is split) and empty the table
          const uint32_t cnt = tcnt[i];
          if (cnt) {
            if (!full) fold(tkey[i], cnt);
            tkey[i] = PC_ZERO_KEY;
            tcnt[i] = 0;
          }
        }
        __syncthreads();                                // everyone has read s_full and the table is empty
        if (tid == 0) s_full = 0;
        if (full) { ++lv; continue; }                   // (uniform) split this class and start over with its first half
        lo += 1ull << (32 - lv);
        while (lv > lv0 && (lo & ((1ull << (33 - lv)) - 1)) == 0) --lv;   // both halves done: back to the parent's level
        if (lo >= (1ull << 32)) break;
      }
      pc_cp_wait<0>();                                  // the first piece again, copied for a sweep that did not come
      __syncthreads();
      select(bucket, [&](auto&& fn_key) {
        PcCursor sc{cb0, 0};
        do {
          const uint32_t m = pc_stage_fill(P, c, f, keys, cb0, cb1, sc, stage, S);
          pc_cp_commit();
          pc_cp_wait<0>();
          __syncthreads();
          for (uint32_t i = tid; i < m; i += ANV_BLOCK) fn_key(stage[i]);
          __syncthreads();
        } while (sc.j < cb1);
      });
      staged = false;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long ob = __shfl_down_sync(ANV_FULL, best, o); if (ob > best) best = ob;
    distinct += __shfl_down_sync(ANV_FULL, distinct, o);
  }
  if ((tid & 31) == 0) {
    if (best) atomicMax(&st.best, best);
    if (distinct) atomicAdd(&st.distinct, (unsigned long long)distinct);
  }
  if (hp) {                                             // one global atomic per (CTA, register) that this CTA raised
    __syncthreads();
    uint32_t* G = P.hll_regs + ((size_t)c << hp);
    for (int i = tid; i < (1 << hp); i += ANV_BLOCK) {
      const uint32_t v = sreg[i];
      if (v > G[i]) atomicMax(&G[i], v);
    }
  }
}

// ---- direct count: one CTA per (group, column) walks the group's direct buckets (pc_is_direct) ------------------------------
// Each key of a bucket bumps its own 16-bit counter, k - lo - 1, with a shared-memory add whose result nothing waits for:
// no probing, no sweeps, one pass whatever the bucket's size.  A scan over the bucket's counters in key order then folds
// each distinct key (multiplicity, mode, HLL++) and empties the counters again, so they are cleared once per CTA.  A count
// never exceeds n < 2^16, so no carry reaches the neighbouring counter.
__global__ void __launch_bounds__(ANV_BLOCK, 3) pc_direct_kernel(const PcParams P, const int n_ranks, double* rank_values) {
  const int g = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t cb0 = P.chunk_base[(size_t)c * (P.G + 1) + g], cb1 = P.chunk_base[(size_t)c * (P.G + 1) + g + 1];
  if (cb0 == cb1) return;                               // (uniform) no key between this group's splitters
  const int nf = (g == P.G - 1) ? PC_FPG + 1 : PC_FPG;
  const uint32_t* split = P.split + (size_t)c * P.NS;
  __shared__ uint32_t s_cnt[PC_FPG + 1];                // keys of each direct bucket, 0 for the others
  __shared__ uint32_t s_base[PC_FPG + 1];               // lo + 1: the key of the bucket's counter 0
  __shared__ uint32_t s_range[PC_FPG + 1];              // R: the bucket's counters
  uint32_t n_direct = 0;
  if (tid < nf) {
    const int bucket = g * PC_FPG + tid;
    const uint32_t n = P.cnt_lt[(size_t)c * P.NB + bucket];
    if (n && pc_is_direct(split, P.NS, bucket, n)) n_direct = n;
    const uint32_t lo1 = bucket > 0 ? split[bucket - 1] + 1u : 0u;
    s_base[tid] = lo1;
    s_range[tid] = n_direct ? (bucket < P.NS ? split[bucket] : 0u) - lo1 : 0u;   // hi - lo - 1 (mod 2^32: hi = 2^32 -> 0)
  }
  if (tid <= PC_FPG) s_cnt[tid] = n_direct;
  if (!__syncthreads_or(n_direct != 0)) return;         // (uniform) no direct bucket in this group
  extern __shared__ __align__(16) uint32_t pc_dir[];
  uint32_t* cw = pc_dir;                                // [PC_DIRECT_RANGE / 2] counter i in bits 16 (i & 1) of word i >> 1
  uint32_t* stage = cw + PC_DIRECT_RANGE / 2;           // [PC_SWEEP_KEYS]
  uint32_t* sreg = stage + PC_SWEEP_KEYS;               // [1 << hll_p] this CTA's HLL++ registers
  __shared__ PcStageScratch S;
  __shared__ uint32_t s_w[ANV_WARPS];
  PcCol& st = P.st[c];
  const int dt = P.cols[c].dtype;
  const int hp = P.hll_p;
  const uint32_t* __restrict__ keys = P.keys[1] + (size_t)c * P.stride + P.gstart[(size_t)c * (P.G + 1) + g];
  uint4* cw4 = reinterpret_cast<uint4*>(cw);
  for (int i = tid; i < PC_DIRECT_RANGE / 8; i += ANV_BLOCK) cw4[i] = make_uint4(0u, 0u, 0u, 0u);
  if (hp) for (int i = tid; i < (1 << hp); i += ANV_BLOCK) sreg[i] = 0;
  unsigned long long best = 0;
  uint32_t distinct = 0;
  const int nq = st.n_queries;
  for (int f = 0; f < nf; ++f) {
    if (s_cnt[f] == 0) continue;                        // (uniform)
    const int bucket = g * PC_FPG + f;
    const uint32_t base = s_base[f];
    // ---- count: the bucket's segments are staged PC_SWEEP_KEYS keys at a time, all of a thread's copies in flight at once
    PcCursor cu{cb0, 0};
    do {                                                // pc_stage_fill's barriers order the last count / scan before its copies
      const uint32_t m = pc_stage_fill(P, c, f, keys, cb0, cb1, cu, stage, S);
      pc_cp_commit();
      pc_cp_wait<0>();
      __syncthreads();
      for (uint32_t i = tid; i < m; i += ANV_BLOCK) {
        const uint32_t d = stage[i] - base;
        atomicAdd(&cw[d >> 1], 1u << ((d & 1u) << 4));
      }
    } while (cu.j < cb1);
    __syncthreads();
    // ---- ranks: first counter whose inclusive prefix reaches the local rank (threads own contiguous counter words)
    for (int q = 0; q < nq; ++q) {
      if (st.q_bucket[q] != bucket) continue;           // uniform across the CTA
      constexpr int WPT = PC_DIRECT_RANGE / 2 / ANV_BLOCK;
      static_assert((WPT & (WPT - 1)) == 0 && WPT >= 32, "the rotated reads need a power of two >= 32");
      const uint32_t r = st.q_local[q];
      uint32_t sum = 0;
      for (int i = 0; i < WPT; ++i) {                   // each lane starts at its own word: no bank conflicts
        const uint32_t w = cw[tid * WPT + ((i + lane) & (WPT - 1))];
        sum += (w & 0xFFFFu) + (w >> 16);
      }
      uint32_t inc = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(ANV_FULL, inc, o); if (lane >= o) inc += t; }
      if (lane == 31) s_w[warp] = inc;
      __syncthreads();
      uint32_t acc = inc - sum;
      for (int w = 0; w < warp; ++w) acc += s_w[w];
      if (acc < r && r <= acc + sum) {                  // exactly one thread holds the rank
        uint32_t i = tid * WPT * 2;
        for (;; ++i) {
          acc += (cw[i >> 1] >> ((i & 1u) << 4)) & 0xFFFFu;
          if (acc >= r) break;
        }
        rank_values[(size_t)c * n_ranks + st.q_slot[q]] = sorted_key_to_double((uint64_t)(base + i) << 32, dt);
      }
      __syncthreads();                                  // s_w is rewritten by the next query
    }
    // ---- scan: every nonzero counter is one distinct key, visited in key order; the words read are emptied again
    const uint32_t nv = (s_range[f] + 7u) / 8u;
    for (uint32_t v = tid; v < nv; v += ANV_BLOCK) {
      const uint4 w4 = cw4[v];
      if ((w4.x | w4.y | w4.z | w4.w) == 0u) continue;
      cw4[v] = make_uint4(0u, 0u, 0u, 0u);
      const uint32_t ws[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t cnt = (ws[e >> 1] >> ((e & 1) << 4)) & 0xFFFFu;
        if (!cnt) continue;
        const uint32_t k = base + 8u * v + (uint32_t)e;
        ++distinct;
        const unsigned long long cand = ((unsigned long long)cnt << 32) | (uint32_t)~k;
        if (cand > best) best = cand;
        if (hp) {
          uint32_t idx, rho;
          hll_slot(spark_hash_of_key<uint32_t>(k, dt), hp, idx, rho);
          atomicMax(&sreg[idx], rho);
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long ob = __shfl_down_sync(ANV_FULL, best, o); if (ob > best) best = ob;
    distinct += __shfl_down_sync(ANV_FULL, distinct, o);
  }
  if ((tid & 31) == 0) {
    if (best) atomicMax(&st.best, best);
    if (distinct) atomicAdd(&st.distinct, (unsigned long long)distinct);
  }
  if (hp) {                                             // one global atomic per (CTA, register) that this CTA raised
    __syncthreads();
    uint32_t* G = P.hll_regs + ((size_t)c << hp);
    for (int i = tid; i < (1 << hp); i += ANV_BLOCK) {
      const uint32_t v = sreg[i];
      if (v > G[i]) atomicMax(&G[i], v);
    }
  }
}

__global__ void pc_final_kernel(const PcParams P, double* mode_value, int64_t* mode_rows, int64_t* n_distinct) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= P.n_cols) return;
  const PcCol& st = P.st[c];
  if (st.best == 0) { mode_value[c] = nan(""); mode_rows[c] = 0; n_distinct[c] = 0; return; }   // no non-null value
  const uint32_t key = ~(uint32_t)(st.best & 0xFFFFFFFFull);
  mode_value[c] = sorted_key_to_double((uint64_t)key << 32, P.cols[c].dtype);
  mode_rows[c] = (int64_t)(st.best >> 32);
  n_distinct[c] = (int64_t)st.distinct;
}

struct PcLayout {
  int P, NS, NB, G, n_tiles, max_chunks;
  int64_t m, stride;
  size_t state, split, clut, cnt_lt, cnt_eq, cum, st, totals, gstart, chunk_base, lsd, keys0, keys1, tile_hist, tile_start, cst, total;
  PcLayout(int n_cols, int64_t n_rows) {
    int p = 256;                                   // fine buckets of ~4096 rows
    while (p < PC_MAX_P && (int64_t)p * SORT_TILE < n_rows) p <<= 1;
    P = p; NS = p; NB = p + 1; G = p / PC_FPG;
    m = (int64_t)PC_OVERSAMPLE * p;
    if (m > n_rows) m = n_rows > 0 ? n_rows : 1;
    stride = (n_rows + 63) & ~(int64_t)63;
    const int64_t nt = (n_rows + SORT_TILE - 1) / SORT_TILE;
    n_tiles = nt > 0 ? (int)nt : 1;
    max_chunks = (int)((stride + PC_CHUNK - 1) / PC_CHUNK) + G;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = (o + bytes + 255) & ~(size_t)255; return at; };
    state = take((size_t)n_cols * sizeof(ColState));
    split = take((size_t)n_cols * NS * 4);
    clut = take((size_t)n_cols * (PC_LUT_CELLS + 1) * 2);
    cnt_lt = take((size_t)n_cols * NB * 4);        // cnt_lt, cnt_eq, cum, st are contiguous: one memset
    cnt_eq = take((size_t)n_cols * NS * 4);
    cum = take((size_t)n_cols * 2 * NB * 4);
    st = take((size_t)n_cols * sizeof(PcCol));
    totals = take((size_t)n_cols * 256 * 4);
    gstart = take((size_t)n_cols * (G + 1) * 4);
    chunk_base = take((size_t)n_cols * (G + 1) * 4);
    // the sample sort's workspace is dead once the splitters are taken: it shares its space with the key buffers
    lsd = o;
    keys0 = take((size_t)n_cols * stride * 4);
    keys1 = take((size_t)n_cols * stride * 4);
    tile_hist = take((size_t)n_cols * 256 * n_tiles * 4);
    tile_start = take((size_t)n_cols * 256 * n_tiles * 2);
    cst = take((size_t)n_cols * max_chunks * PC_CST * 2);
    const size_t sample_end = lsd + Layout<uint32_t>(n_cols, m).total;
    total = (o > sample_end ? o : sample_end) + 256;
  }
};

static int run_partition_count(const anv_column_t* cols, int n_cols, int64_t n_rows, double* mode_value, int64_t* mode_rows,
                               int64_t* n_distinct, const int64_t* ranks, int n_ranks, double* rank_values, int hll_p,
                               uint32_t* hll_regs, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  PcLayout L(n_cols, n_rows);
  if (workspace_bytes < L.total) { set_error("anv_mode_distinct_partition: workspace too small (%zu < %zu)", workspace_bytes, L.total); return ANV_ERR_WORKSPACE; }
  char* w = reinterpret_cast<char*>(workspace);
  // --- the sample sort reuses the LSD machinery on m keys per column ---
  Layout<uint32_t> LS(n_cols, L.m);
  char* ws = w + L.lsd;
  SortParams<uint32_t> S{};
  S.cols = cols; S.n_cols = n_cols; S.n_rows = L.m;
  S.stride = (L.m + 63) & ~(int64_t)63;
  S.n_tiles = (int)((L.m + SORT_TILE - 1) / SORT_TILE);
  if (S.n_tiles < 1) S.n_tiles = 1;
  S.buf[0] = reinterpret_cast<uint32_t*>(ws + LS.buf0);
  S.buf[1] = reinterpret_cast<uint32_t*>(ws + LS.buf1);
  S.state = reinterpret_cast<ColState*>(ws + LS.state);
  S.tile_hist = reinterpret_cast<uint32_t*>(ws + LS.tile_hist);
  S.summ = reinterpret_cast<TileSummary<uint32_t>*>(ws + LS.summ);
  uint32_t* sample_totals = reinterpret_cast<uint32_t*>(ws + LS.totals);
  PcParams P{};
  P.cols = cols; P.n_cols = n_cols; P.n_rows = n_rows; P.stride = L.stride; P.n_tiles = L.n_tiles;
  P.P = L.P; P.NS = L.NS; P.NB = L.NB; P.G = L.G; P.max_chunks = L.max_chunks; P.m = L.m;
  P.split = reinterpret_cast<uint32_t*>(w + L.split);
  P.clut = reinterpret_cast<uint16_t*>(w + L.clut);
  P.keys[0] = reinterpret_cast<uint32_t*>(w + L.keys0);
  P.keys[1] = reinterpret_cast<uint32_t*>(w + L.keys1);
  P.state = reinterpret_cast<ColState*>(w + L.state);
  P.tile_hist = reinterpret_cast<uint32_t*>(w + L.tile_hist);
  P.tile_start = reinterpret_cast<uint16_t*>(w + L.tile_start);
  P.totals = reinterpret_cast<uint32_t*>(w + L.totals);
  P.gstart = reinterpret_cast<uint32_t*>(w + L.gstart);
  P.chunk_base = reinterpret_cast<uint32_t*>(w + L.chunk_base);
  P.cst = reinterpret_cast<uint16_t*>(w + L.cst);
  P.cnt_lt = reinterpret_cast<uint32_t*>(w + L.cnt_lt);
  P.cnt_eq = reinterpret_cast<uint32_t*>(w + L.cnt_eq);
  P.cum = reinterpret_cast<uint32_t*>(w + L.cum);
  P.st = reinterpret_cast<PcCol*>(w + L.st);
  P.hll_p = hll_regs ? hll_p : 0;
  P.hll_regs = hll_regs;
  // the (group, tile) table goes through the LSD path's totals / scan kernels
  SortParams<uint32_t> T{};
  T.cols = cols; T.n_cols = n_cols; T.n_rows = n_rows; T.stride = L.stride; T.n_tiles = L.n_tiles;
  T.state = P.state; T.tile_hist = P.tile_hist; T.pass = 0;
  if (hll_regs) ANV_CUDA(cudaMemsetAsync(hll_regs, 0, ((size_t)n_cols << hll_p) * sizeof(uint32_t), st));
  ANV_CUDA(cudaMemsetAsync(S.state, 0, (size_t)n_cols * sizeof(ColState), st));
  ANV_CUDA(cudaMemsetAsync(P.state, 0, (size_t)n_cols * sizeof(ColState), st));
  ANV_CUDA(cudaMemsetAsync(w + L.cnt_lt, 0, L.st + (size_t)n_cols * sizeof(PcCol) - L.cnt_lt, st));   // cnt_lt, cnt_eq, cum, st
  {
    dim3 grid((unsigned)((L.m + ANV_BLOCK - 1) / ANV_BLOCK), n_cols);
    pc_sample_kernel<<<grid, ANV_BLOCK, 0, st>>>(S, n_rows, L.m);
    ANV_CUDA(cudaGetLastError());
    for (int pass = 0; pass < 4; ++pass) {
      S.pass = pass;
      sort_hist_kernel<uint32_t><<<dim3((S.n_tiles + HIST_TPC - 1) / HIST_TPC, n_cols), ANV_BLOCK, 0, st>>>(S);
      sort_totals_kernel<uint32_t><<<dim3(256, n_cols), ANV_BLOCK, 0, st>>>(S, sample_totals);
      sort_scan_kernel<uint32_t><<<dim3(256, n_cols), ANV_BLOCK, 0, st>>>(S, sample_totals);
      sort_scatter_kernel<uint32_t><<<dim3((S.n_tiles + SCAT_TPC - 1) / SCAT_TPC, n_cols), SCAT_THREADS, 0, st>>>(S);
      ANV_CUDA(cudaGetLastError());
    }
    pc_split_kernel<<<n_cols, 256, 0, st>>>(S, P);
    ANV_CUDA(cudaGetLastError());
  }
  if (n_rows > 0) {
    pc_coarse_kernel<<<dim3((L.n_tiles + PC_TPC - 1) / PC_TPC, n_cols), ANV_BLOCK, 0, st>>>(P);
    sort_totals_kernel<uint32_t><<<dim3(256, n_cols), ANV_BLOCK, 0, st>>>(T, P.totals);
    sort_scan_kernel<uint32_t><<<dim3(256, n_cols), ANV_BLOCK, 0, st>>>(T, P.totals);
    pc_chunks_kernel<<<n_cols, 256, 0, st>>>(P);
    pc_fine_kernel<<<dim3(L.max_chunks, n_cols), ANV_BLOCK, 0, st>>>(P);
    ANV_CUDA(cudaGetLastError());
  }
  pc_cum_kernel<<<n_cols, 1024, 0, st>>>(P, ranks, n_ranks, rank_values);
  ANV_CUDA(cudaGetLastError());
  if (n_rows > 0) {
    const size_t smem = (size_t)PC_GROUP_SMEM + (P.hll_p ? ((size_t)4 << P.hll_p) : 0);
    static bool attr_done = false;
    if (!attr_done) {                               // sized for hll_p = 12; the carveout lets 2 CTAs share an SM at hll_p = 9
      ANV_CUDA(cudaFuncSetAttribute(pc_group_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PC_GROUP_SMEM + (4 << 12)));
      ANV_CUDA(cudaFuncSetAttribute(pc_group_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
      attr_done = true;
    }
    pc_group_kernel<<<dim3(L.G, n_cols), ANV_BLOCK, smem, st>>>(P, n_ranks, rank_values);
    ANV_CUDA(cudaGetLastError());
    const size_t dsmem = (size_t)PC_DIRECT_SMEM + (P.hll_p ? ((size_t)4 << P.hll_p) : 0);
    static bool dattr_done = false;
    if (!dattr_done) {                              // sized for hll_p = 12; 3 CTAs share an SM at hll_p = 9
      ANV_CUDA(cudaFuncSetAttribute(pc_direct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PC_DIRECT_SMEM + (4 << 12)));
      ANV_CUDA(cudaFuncSetAttribute(pc_direct_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
      dattr_done = true;
    }
    pc_direct_kernel<<<dim3(L.G, n_cols), ANV_BLOCK, dsmem, st>>>(P, n_ranks, rank_values);
    ANV_CUDA(cudaGetLastError());
  }
  pc_final_kernel<<<(n_cols + 127) / 128, 128, 0, st>>>(P, mode_value, mode_rows, n_distinct);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

}  // namespace anv

using namespace anv;

extern "C" size_t anv_mode_distinct_workspace_bytes(int n_cols, int64_t n_rows, int key_bits) {
  if (n_cols <= 0 || n_rows < 0) return 256;
  return key_bits == 32 ? Layout<uint32_t>(n_cols, n_rows).total : Layout<uint64_t>(n_cols, n_rows).total;
}

extern "C" int anv_mode_distinct_hll(const anv_column_t* cols, int n_cols, int64_t n_rows, int key_bits, double* mode_value,
                                     int64_t* mode_rows, int64_t* n_distinct, const int64_t* ranks, int n_ranks,
                                     double* rank_values, int hll_p, uint32_t* hll_regs, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  if (n_ranks < 0 || (n_ranks > 0 && (!ranks || !rank_values))) { set_error("anv_mode_distinct: bad ranks arguments"); return ANV_ERR_INVALID; }
  if (n_cols < 0 || n_rows < 0 || (key_bits != 32 && key_bits != 64)) { set_error("anv_mode_distinct: bad arguments"); return ANV_ERR_INVALID; }
  if (hll_regs && (hll_p < 4 || hll_p > 12)) { set_error("anv_mode_distinct_hll: 4 <= hll_p <= 12"); return ANV_ERR_INVALID; }
  if (n_cols == 0) return ANV_OK;
  if (n_cols > ANV_MAX_LAUNCH_COLS) { set_error("n_cols > %d: split the frame into column blocks", ANV_MAX_LAUNCH_COLS); return ANV_ERR_UNSUPPORTED; }
  if (n_rows >= ((int64_t)1 << 32)) { set_error("anv_mode_distinct: n_rows >= 2^32 per call is not supported"); return ANV_ERR_UNSUPPORTED; }
  if (!cols || !mode_value || !mode_rows || !n_distinct || !workspace) { set_error("anv_mode_distinct: NULL argument"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  if (key_bits == 32) return run_mode_distinct<uint32_t>(cols, n_cols, n_rows, mode_value, mode_rows, n_distinct, ranks, n_ranks, rank_values, hll_p, hll_regs, workspace, workspace_bytes, st);
  return run_mode_distinct<uint64_t>(cols, n_cols, n_rows, mode_value, mode_rows, n_distinct, ranks, n_ranks, rank_values, hll_p, hll_regs, workspace, workspace_bytes, st);
}

extern "C" int anv_mode_distinct(const anv_column_t* cols, int n_cols, int64_t n_rows, int key_bits, double* mode_value,
                                 int64_t* mode_rows, int64_t* n_distinct, const int64_t* ranks, int n_ranks,
                                 double* rank_values, void* workspace, size_t workspace_bytes, void* stream) {
  return anv_mode_distinct_hll(cols, n_cols, n_rows, key_bits, mode_value, mode_rows, n_distinct, ranks, n_ranks, rank_values, 0,
                               nullptr, workspace, workspace_bytes, stream);
}

extern "C" size_t anv_mode_distinct_partition_workspace_bytes(int n_cols, int64_t n_rows) {
  if (n_cols <= 0 || n_rows < 0) return 256;
  return PcLayout(n_cols, n_rows).total;
}

extern "C" int anv_mode_distinct_partition_hll(const anv_column_t* cols, int n_cols, int64_t n_rows, double* mode_value,
                                               int64_t* mode_rows, int64_t* n_distinct, const int64_t* ranks, int n_ranks,
                                               double* rank_values, int hll_p, uint32_t* hll_regs, void* workspace,
                                               size_t workspace_bytes, void* stream) {
  if (n_ranks < 0 || n_ranks > PC_MAX_RANKS || (n_ranks > 0 && (!ranks || !rank_values))) { set_error("anv_mode_distinct_partition: bad ranks arguments (n_ranks <= 16)"); return ANV_ERR_INVALID; }
  if (n_cols < 0 || n_rows < 0) { set_error("anv_mode_distinct_partition: bad arguments"); return ANV_ERR_INVALID; }
  if (hll_regs && (hll_p < 4 || hll_p > 12)) { set_error("anv_mode_distinct_partition_hll: 4 <= hll_p <= 12"); return ANV_ERR_INVALID; }
  if (n_cols == 0) return ANV_OK;
  if (n_cols > ANV_MAX_LAUNCH_COLS) { set_error("n_cols > %d: split the frame into column blocks", ANV_MAX_LAUNCH_COLS); return ANV_ERR_UNSUPPORTED; }
  if (n_rows >= ((int64_t)1 << 32)) { set_error("anv_mode_distinct_partition: n_rows >= 2^32 per call is not supported"); return ANV_ERR_UNSUPPORTED; }
  if (!cols || !mode_value || !mode_rows || !n_distinct || !workspace) { set_error("anv_mode_distinct_partition: NULL argument"); return ANV_ERR_INVALID; }
  return run_partition_count(cols, n_cols, n_rows, mode_value, mode_rows, n_distinct, ranks, n_ranks, rank_values, hll_p, hll_regs,
                             workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int anv_mode_distinct_partition(const anv_column_t* cols, int n_cols, int64_t n_rows, double* mode_value,
                                           int64_t* mode_rows, int64_t* n_distinct, const int64_t* ranks, int n_ranks,
                                           double* rank_values, void* workspace, size_t workspace_bytes, void* stream) {
  return anv_mode_distinct_partition_hll(cols, n_cols, n_rows, mode_value, mode_rows, n_distinct, ranks, n_ranks, rank_values, 0,
                                         nullptr, workspace, workspace_bytes, stream);
}
