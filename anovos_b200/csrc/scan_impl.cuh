// K1 / K2: the fused streaming column scan (implementation header; instantiated by
// scan_mom.cu / scan_hist.cu / scan_fused.cu / scan_assign.cu so nvcc compiles them in parallel).
//
// One CTA handles one (column, row-tile): it streams the tile with 128-bit no-allocate
// loads (coalesced: consecutive threads read consecutive 16 B, 8 loads in flight per
// thread, immediate offsets, 32-bit in-tile indexing; an opt-in second instantiation of the fused
// kernel stages null-free columns through a thread-private cp.async ring instead) and keeps
//   K1  count / nonzero / min / max in native-type lanes and the pivot-shifted power sums
//       sum d, d^2, d^3, d^4 (d = double(x) - pivot) in FP64 registers;
//   K2  the bin id from ONE fused multiply-add guess fixed up by ONE exact native-type
//       threshold compare (or a branch-free binary search / the dictionary code), counted
//       in per-thread PRIVATE shared-memory counters (bank = lane: conflict-free, no atomics);
// then reduces with warp shuffles + one shared-memory stage and emits a mergeable partial per
// tile.  A second tiny kernel Pebay-merges the tile partials of each column in a fixed
// order, so results are run-to-run bit-stable.
//
// Replaces (reference, /root/reference/src/main/anovos): the Spark summary()/agg scans of
// data_analyzer/stats_generator.py:163,240-241,310,488,813,908,993, the min/max agg of
// data_transformer/transformers.py:217-219, the Python UDF bucket_label
// transformers.py:248-280 and the groupBy counts of drift_stability/drift_detector.py:252-264.
#pragma once
#include "common.cuh"

namespace anv {

struct Partial {  // one per (column, tile); 64 B
  int64_t n, nz;
  double mn, mx;
  double mean, m2, m3, m4;
};

struct ScanParams {
  const anv_column_t* cols;
  int n_cols;
  int64_t n_rows;
  int tile_rows;  // multiple of 1024, <= 262144
  // K1
  Partial* partials;
  int tiles_per_col;
  // K2
  const anv_binspec_t* specs;
  const uint64_t* cuts;
  const int32_t* card;  // codes mode: cardinality per column
  unsigned long long* counts;
  int count_stride;
  int thr_slots;  // threshold slots reserved in shared memory
  // bin-id materialisation
  int32_t* out_bins;
  int64_t out_stride;
  // cp.async staging ring of the STAGED kernels: byte offset inside the dynamic shared memory (behind the counters)
  uint32_t stage_off;
};

// Per-kernel tuning (scripts/tune.sh sweeps ANV_UNROLL / ANV_MINBLOCKS): 8 x 128-bit loads in flight per thread and
// 4 CTAs of 256 threads per SM (<= 64 registers).
template <bool MOM, int HPATH, bool ASSIGN> struct Tune {
#ifdef ANV_UNROLL
  static constexpr int U = ANV_UNROLL;
#else
  static constexpr int U = 8;
#endif
#ifdef ANV_MINBLOCKS
  static constexpr int MINB = ANV_MINBLOCKS;
#else
  static constexpr int MINB = 4;
#endif
  // software pipelining (loads of half-batch k+1 in flight while half-batch k is consumed) pays for
  // the histogram-only kernel (+13 %); with the FP64 moments it only adds register pressure
  static constexpr bool PF = !MOM && HPATH == 0 && !ASSIGN;
};

// STAGED kernels: every thread keeps ST_D groups of ST_CH 128-bit vectors in flight as cp.async (LDGSTS) copies into its
// OWN shared-memory slots (no cross-thread hazard, no barrier: cp.async.wait_group is per thread) and consumes the oldest
// group with LDS.128 while the younger ones are still on their way.  The loads no longer sit in 32 staging registers and
// the latency of a batch is hidden by the thread's own next batches instead of by other warps only.
#ifndef ANV_ST_D
#define ANV_ST_D 4
#endif
#ifndef ANV_ST_CH
#define ANV_ST_CH 2
#endif
#ifndef ANV_FUSED_STAGED_DEFAULT
#define ANV_FUSED_STAGED_DEFAULT 0
#endif
constexpr int ST_D = ANV_ST_D, ST_CH = ANV_ST_CH;
constexpr size_t STAGE_BYTES = (size_t)ST_D * ST_CH * ANV_BLOCK * 16;

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* g) {
  asm volatile("cp.async.cg.shared.global.L2::128B [%0], [%1], 16;" ::"r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ uint4 lds_v4(uint32_t saddr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(saddr) : "memory");
  return r;
}

__device__ __forceinline__ float lds_f32(uint32_t saddr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr));
  return v;
}
__device__ __forceinline__ void red_shared_inc(uint32_t saddr) {
  asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(saddr) : "memory");
}

enum BinMode { BIN_SEARCH = 0, BIN_GUESS = 1, BIN_CODE = 2, BIN_GUESS_FOLD = 3 };  // FOLD: device-side refinement of GUESS

// ---- bin lookup -----------------------------------------------------------------------
// S[0] = lowest, S[1..B-1] = thresholds theta_0..theta_{B-2}, S[B..P] = highest.
// slot(x) = 1 + #(theta_i < x) for non-null x (bucket_label, transformers.py:248-271).
template <typename T, int MODE> struct Binner {
  const T* S;
  int B, P;
  T lo, invw;
  __device__ __forceinline__ int slot(T x) const;
};

template <typename T> __device__ __forceinline__ int search_slot(const T* S, int P, int B, T x) {
  int k = 0;
  const T* G = S + 1;
#pragma unroll 1
  for (int s = P >> 1; s > 0; s >>= 1) k += (G[k + s - 1] < x) ? s : 0;
  if (Traits<T>::is_nan(x)) k = B - 1;  // `NaN <= c` is False for every cutoff -> last bin
  return k + 1;
}
template <> __device__ __forceinline__ int Binner<float, BIN_SEARCH>::slot(float x) const { return search_slot(S, P, B, x); }
template <> __device__ __forceinline__ int Binner<double, BIN_SEARCH>::slot(double x) const { return search_slot(S, P, B, x); }
template <> __device__ __forceinline__ int Binner<int32_t, BIN_SEARCH>::slot(int32_t x) const { return search_slot(S, P, B, x); }
template <> __device__ __forceinline__ int Binner<int64_t, BIN_SEARCH>::slot(int64_t x) const { return search_slot(S, P, B, x); }
template <> __device__ __forceinline__ int Binner<int32_t, BIN_CODE>::slot(int32_t x) const {
  return min(max(x + 1, 1), B);  // an out-of-range code is clamped, never scribbles
}
template <> __device__ __forceinline__ int Binner<float, BIN_GUESS>::slot(float x) const {
  // r = round((x - lo) * invw) clamped to [0, B-1] via the 1.5*2^23 magic (ALU only); the true
  // 0-based bin is r-1 or r, decided by ONE exact compare against theta_{r-1} = S[r].
  float t = fmaf(x - lo, invw, 12582912.0f);
  t = fmaxf(fminf(t, 12582912.0f + (float)(B - 1)), 12582912.0f);  // NaN -> B-1
  const int r = __float_as_int(t) - 0x4B400000;
  return r + (!(x <= S[r]) ? 1 : 0);  // S[0] = NaN => >= 1; NaN x => B
}
template <> __device__ __forceinline__ int Binner<double, BIN_GUESS>::slot(double x) const {
  double t = fma(x - lo, invw, 6755399441055744.0);
  t = fmax(fmin(t, 6755399441055744.0 + (double)(B - 1)), 6755399441055744.0);  // NaN -> B-1
  const int r = __double2loint(t);
  return r + (!(x <= S[r]) ? 1 : 0);
}

// Fast float32 equal_range path of the private-counter histogram.  Everything is expressed
// on the raw bits of a float that carries the (reversed) bin guess, and the exact threshold of
// every slot is REPLICATED PER THREAD right behind the private counters (same [slot][tid]
// layout, bank = lane: conflict-free), so one multiply-add yields the address of both:
//   v    = sat(1 - (x - lo) * c)            c = inv_w / (B-1);   NaN, +inf -> 0;  -inf -> 1
//   r'   = round(v * (B-1)) = bits(v * (B-1) + 1.5*2^23) - 0x4B400000      (= B-1-r)
//   a0   = cnt_t + (B-1-r') * 1024          counter of slot r = B-1-r'      (ONE IMAD)
//   th   = [a0 + toff]                      = S[r]: theta_{r-1}; S[0] = NaN (ONE LDS, immediate offset)
//   a    = a0 + (x > th or unordered ? 1024 : 0)   => slot = r + !(x <= th)  (setp + predicated add)
//   red.shared.add [a], 1                   NaN x: r' = 0, compare unordered => slot = B
// FFMA.SAT saturates for free (no min/max clamp) and maps NaN to 0.
// FOLD: when the range does not sit far from zero (fold_ok below), `x - lo` is folded into the multiply-add,
//   v = sat(x * (-c) + k),  k = 1 + lo * c  (one instruction less per element).
// The guess then carries the rounding errors of k and of c times |x| instead of |x - lo|: at most
// (B-1) * 2^-23 * (2 + |lo| * c) bins, which fold_ok keeps below 1/32 - and ANY error below half a bin leaves the true
// bin in {r-1, r}, which is all the exact threshold compare needs.
struct FastF32 {
  uint32_t c_adj, toff;
  float lo, negc, bm1, k;
  template <bool FOLD> __device__ __forceinline__ uint32_t counter_addr(float x) const {
    float v;
    if (FOLD) asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(v) : "f"(x), "f"(negc), "f"(k));
    else asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(v) : "f"(x - lo), "f"(negc), "f"(1.0f));
    const uint32_t bits = __float_as_uint(fmaf(v, bm1, 12582912.0f));
    uint32_t a = c_adj - (bits << 10);
    const float th = lds_f32(a + toff);
    asm("{\n\t.reg .pred p;\n\tsetp.gtu.f32 p, %1, %2;\n\t@p add.u32 %0, %0, 1024;\n\t}" : "+r"(a) : "f"(x), "f"(th));
    return a;
  }
};

// (B-1) * (2 + |lo| * c) <= 2^18  =>  guess error <= 2^-5 bins (c = inv_w / (B-1), so (B-1) * |lo| * c = |lo| * inv_w)
__device__ __forceinline__ bool fold_ok(const anv_binspec_t& sp) {
  const double e = 2.0 * (double)(sp.n_bins - 1) + fabs(sp.lo) * sp.inv_w;
  return sp.n_bins >= 2 && e <= 262144.0;   // NaN / inf fail the compare
}

// n += (x != 0) as compare + predicated add (2 instructions; the C++ form costs a third, a select)
template <typename T> __device__ __forceinline__ void count_nonzero(uint32_t& n, T x) { n += (x != (T)0) ? 1u : 0u; }
template <> __device__ __forceinline__ void count_nonzero<float>(uint32_t& n, float x) {
  asm("{\n\t.reg .pred p;\n\tsetp.neu.f32 p, %1, 0f00000000;\n\t@p add.u32 %0, %0, 1;\n\t}" : "+r"(n) : "f"(x));
}
template <> __device__ __forceinline__ void count_nonzero<int32_t>(uint32_t& n, int32_t x) {
  asm("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %1, 0;\n\t@p add.u32 %0, %0, 1;\n\t}" : "+r"(n) : "r"(x));
}

// 3-input min / max.  sm_90a has no 3-input FMNMX (the PTX form needs sm_100): two FMNMX for floats, one VIMNMX3
// for int32.  fminf / fmaxf drop a NaN operand exactly as PTX min / max do.
__device__ __forceinline__ float min3(float a, float b, float c) { return fminf(a, fminf(b, c)); }
__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(a, fmaxf(b, c)); }
__device__ __forceinline__ int32_t min3(int32_t a, int32_t b, int32_t c) { return __vimin3_s32(a, b, c); }
__device__ __forceinline__ int32_t max3(int32_t a, int32_t b, int32_t c) { return __vimax3_s32(a, b, c); }
__device__ __forceinline__ double min3(double a, double b, double c) { return fmin(a, fmin(b, c)); }
__device__ __forceinline__ double max3(double a, double b, double c) { return fmax(a, fmax(b, c)); }
__device__ __forceinline__ int64_t min3(int64_t a, int64_t b, int64_t c) { return min(a, min(b, c)); }
__device__ __forceinline__ int64_t max3(int64_t a, int64_t b, int64_t c) { return max(a, max(b, c)); }

template <typename T> __device__ __forceinline__ T cut_as(uint64_t raw);
template <> __device__ __forceinline__ float cut_as<float>(uint64_t raw) { return __uint_as_float((uint32_t)raw); }
template <> __device__ __forceinline__ int32_t cut_as<int32_t>(uint64_t raw) { return (int32_t)(uint32_t)raw; }
template <> __device__ __forceinline__ double cut_as<double>(uint64_t raw) { return __longlong_as_double((long long)raw); }
template <> __device__ __forceinline__ int64_t cut_as<int64_t>(uint64_t raw) { return (int64_t)raw; }

struct ScanShared {  // declared once in the kernel (not per template instantiation)
  double red[ANV_WARPS][6];
  uint32_t redn[ANV_WARPS][2];
  int fix;
};

// Tile power sums t_k = sum (x - pivot)^k over n valid rows -> central form (mean, M2, M3, M4).  The cancellation is
// bounded by the tile's spread around the pivot, so the pivot must be an element of the tile.
__device__ __forceinline__ void central_from_power_sums(Partial& out, double pivot, double t1, double t2, double t3,
                                                        double t4) {
  const double dl = t1 / (double)out.n;  // mean - pivot
  out.mean = pivot + dl;
  out.m2 = t2 - t1 * dl;
  out.m3 = t3 - 3.0 * dl * t2 + 2.0 * dl * dl * t1;
  out.m4 = t4 - 4.0 * dl * t3 + 6.0 * dl * dl * t2 - 3.0 * dl * dl * dl * t1;
}

// ---- the tile body --------------------------------------------------------------------
// HPATH: -1 no histogram, 0 private per-thread counters, 1 per-CTA shared atomics, 2 global atomics
template <typename T, bool MOM, int HPATH, bool ASSIGN, bool NULLS, int MODE, bool STAGED = false>
__device__ __forceinline__ void scan_tile(const ScanParams& P, const anv_column_t& col, int c, unsigned char* smem,
                                          ScanShared& SS) {
  constexpr bool HIST = HPATH >= 0;
  constexpr int VEC = Traits<T>::VEC;
  constexpr int WSTEP = ANV_BLOCK * VEC / 32;  // bitmap words between two unrolled loads of a thread
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * P.tile_rows;
  const int n_tile = (int)min((int64_t)P.tile_rows, P.n_rows - r0);
  const T* __restrict__ data = reinterpret_cast<const T*>(col.data) + r0;
  const uint32_t* __restrict__ vwords = NULLS ? col.validity + (r0 >> 5) : nullptr;

  // ---- K2 setup: thresholds + counters in shared memory ------------------------------
  Binner<T, (MODE == BIN_GUESS_FOLD ? (int)BIN_GUESS : MODE)> bn;
  uint32_t* cnt = nullptr;
  int n_slots = 0;
  if (HIST || ASSIGN) {
    T* S = reinterpret_cast<T*>(smem);
    cnt = reinterpret_cast<uint32_t*>(smem + (size_t)P.thr_slots * 8);
    bn.S = S;
    if (MODE == BIN_CODE) {
      bn.B = P.card[c]; bn.P = 2; bn.lo = 0; bn.invw = 0;
    } else {
      const anv_binspec_t sp = P.specs[c];
      bn.B = sp.n_bins;
      int p2 = 2;
      while (p2 < bn.B) p2 <<= 1;
      bn.P = p2;
      bn.lo = (T)sp.lo; bn.invw = (T)sp.inv_w;
      for (int i = tid; i <= p2; i += ANV_BLOCK) {
        T v;
        if (i == 0) v = Traits<T>::first_slot();  // NaN for floats: `x <= S[0]` is never true
        else if (i <= bn.B - 1) v = cut_as<T>(P.cuts[sp.cut_offset + i - 1]);
        else v = Traits<T>::highest();
        S[i] = v;
      }
    }
    n_slots = bn.B + 1;
    if (HPATH == 0) {
      for (int i = tid; i < n_slots * ANV_BLOCK; i += ANV_BLOCK) cnt[i] = 0;
    } else if (HPATH == 1) {
      for (int i = tid; i < n_slots; i += ANV_BLOCK) cnt[i] = 0;
    }
    __syncthreads();
  }
  uint32_t* const cnt_t = cnt + tid;
  unsigned long long* const gcnt = P.counts + (size_t)c * P.count_stride;
  constexpr bool GUESS = MODE == BIN_GUESS || MODE == BIN_GUESS_FOLD;
  constexpr bool FAST = HPATH == 0 && !ASSIGN && GUESS && sizeof(T) == 4;
  constexpr bool FOLD = MODE == BIN_GUESS_FOLD;
  FastF32 ff{};
  uint32_t cnt_t_saddr = 0;
  if (HPATH == 0) cnt_t_saddr = (uint32_t)__cvta_generic_to_shared(cnt_t);
  if (FAST) {
    // per-thread replica of the thresholds, [slot][tid] right behind the counters (this thread's own words)
    ff.toff = (uint32_t)P.count_stride * ANV_BLOCK * 4;
    float* rep = reinterpret_cast<float*>(cnt_t) + (size_t)P.count_stride * ANV_BLOCK;
    for (int r = 0; r < bn.B; ++r) rep[r * ANV_BLOCK] = reinterpret_cast<const float*>(smem)[r];
    ff.c_adj = cnt_t_saddr + ((uint32_t)(bn.B - 1) << 10) + (0x4B400000u << 10);
    ff.lo = (float)bn.lo; ff.bm1 = (float)(bn.B - 1); ff.negc = -((float)bn.invw / ff.bm1);
    ff.k = (float)(1.0 - (double)ff.lo * (double)ff.negc);
  }

  // ---- pivot = first finite non-null value among the tile's first rows ----------------------
  // It is an actual element, exactly representable in T.  K1 shifts the power sums by it
  // (d = double(x) - pivot keeps them well conditioned) and, in tiles with a validity
  // bitmap, NULL LANES IMPERSONATE THE PIVOT: one select per element up front, then the
  // null-free code runs unchanged (d == 0 exactly; min/max see a real element; the nonzero
  // count and the pivot's histogram slot are corrected per thread in the epilogue).
  constexpr bool PIVOT = MOM || NULLS;
  T pivot_t = (T)0;
  double pivot = 0.0;
  bool have_pivot = false;
  if (PIVOT) {
    for (int g = 0; g < n_tile && g < 1024 && !have_pivot; g += 32) {  // warp-uniform loop
      const int idx = g + lane;
      bool ok = idx < n_tile;
      T pv = (T)0;
      if (ok) {
        pv = data[idx];
        if (NULLS) ok = (vwords[idx >> 5] >> (idx & 31)) & 1u;
        ok = ok && isfinite(Traits<T>::to_double(pv));
      }
      const uint32_t m = __ballot_sync(ANV_FULL, ok);
      if (m) {
        const int src = __ffs(m) - 1;
        if (sizeof(T) == 8) {
          const unsigned long long raw = __shfl_sync(ANV_FULL, *reinterpret_cast<unsigned long long*>(&pv), src);
          pivot_t = *reinterpret_cast<const T*>(&raw);
        } else {
          const uint32_t raw = __shfl_sync(ANV_FULL, *reinterpret_cast<uint32_t*>(&pv), src);
          pivot_t = *reinterpret_cast<const T*>(&raw);
        }
        have_pivot = true;
      }
    }
    pivot = Traits<T>::to_double(pivot_t);
  }

  double s1 = 0.0, s2 = 0.0, s3 = 0.0, s4 = 0.0;
  T mn = Traits<T>::highest(), mx = Traits<T>::lowest();
  uint32_t n_ok = 0, n_nz = 0;
  constexpr bool SLOT0 = ASSIGN || HPATH > 0;  // these paths need the literal slot 0 for null rows

  // x is already pivot-substituted on null lanes; `valid` is only consulted where slot 0 is needed
  auto elem = [&](T x, bool valid) -> int {
    int slot = 0;
    if (MOM) {
      const double d = Traits<T>::to_double(x) - pivot;
      const double d2 = d * d;
      s1 += d;
      s2 += d2;
      s3 = fma(d2, d, s3);
      s4 = fma(d2, d2, s4);
      count_nonzero<T>(n_nz, x);
    }
    if (FAST) {
      red_shared_inc(ff.template counter_addr<FOLD>(*reinterpret_cast<const float*>(&x)));
    } else if (HIST || ASSIGN) {
      slot = bn.slot(x);
      if (NULLS && SLOT0) slot = valid ? slot : 0;
      if (HIST) {
        if (HPATH == 0) red_shared_inc(cnt_t_saddr + ((uint32_t)slot << 10));
        else if (HPATH == 1) atomicAdd(&cnt[slot], 1u);
        else atomicAdd(&gcnt[slot], 1ull);
      }
    }
    return slot;
  };
  // vb: the validity bits of the vector's elements at bit positions 1 .. VEC (the bitmap word ROTATED so that the vector's
  // first bit lands on bit 1: one SHF, no mask, and bits 1 .. VEC move into predicates with a single R2P; with the bits at
  // 0 .. VEC-1 the compiler tested bit 0 separately - a LOP3 and an ISETP more per vector)
  auto vec = [&](T (&e)[VEC], uint32_t vb, int (&sl)[VEC]) {
    if (NULLS) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) e[i] = ((vb >> (i + 1)) & 1u) ? e[i] : pivot_t;
    }
    if (MOM) {  // two elements per min3 / max3
#pragma unroll
      for (int i = 0; i < VEC; i += 2) {
        mn = min3(mn, e[i], e[i + 1]);
        mx = max3(mx, e[i], e[i + 1]);
      }
    }
#pragma unroll
    for (int i = 0; i < VEC; ++i) sl[i] = elem(e[i], (vb >> (i + 1)) & 1u);
  };
  int32_t* __restrict__ obins = ASSIGN ? P.out_bins + (size_t)c * P.out_stride + r0 : nullptr;
  auto store_bins = [&](int row, const int (&sl)[VEC]) {
    if (VEC == 4) *reinterpret_cast<int4*>(obins + row) = make_int4(sl[0], sl[1], sl[2], sl[3]);
    else *reinterpret_cast<int2*>(obins + row) = make_int2(sl[0], sl[VEC - 1]);
  };

  // ---- stream the tile (32-bit in-tile indexing; the unrolled loads use immediate offsets) ---
  constexpr int UNROLL = Tune<MOM, HPATH, ASSIGN>::U;
  const int nvec = n_tile / VEC;  // full 16-byte vectors in this tile
  const uint4* __restrict__ vdata = reinterpret_cast<const uint4*>(data);
  const int vsh = (((tid * VEC) & 31) + 31) & 31;  // rotate amount: bit offset of this thread's vector inside its bitmap word, minus 1 (loop-invariant)
  int base = 0;
  if constexpr (STAGED) {
  // thread-private cp.async ring: slot (s, u) of this thread at ring + ((s * ST_CH + u) * ANV_BLOCK) * 16 (+ tid * 16):
  // consecutive lanes, consecutive 16 bytes - conflict-free for the copy-in and for LDS.128.  Same vector -> thread
  // mapping as the register-staged loop (vector base + u * ANV_BLOCK + tid), so the per-thread sums are bit-identical.
  constexpr int STEPV = ANV_BLOCK * ST_CH;  // vectors per group, CTA-wide
  constexpr int WGRP = STEPV * VEC / 32;    // bitmap words per group
  const int n_groups = nvec / STEPV;
  const uint32_t ring = (uint32_t)__cvta_generic_to_shared(smem + P.stage_off) + (uint32_t)tid * 16u;
  uint32_t vw[ST_D][ST_CH];  // raw validity words of the groups in flight (shifted / masked when consumed)
  const uint4* pn = vdata + tid;                                             // next group to issue (running pointers:
  const uint32_t* wn = NULLS ? vwords + ((tid * VEC) >> 5) : nullptr;        //  one 64-bit add per group)
  auto issue = [&](int s) {
#pragma unroll
    for (int u = 0; u < ST_CH; ++u) {
      cp_async16(ring + (uint32_t)((s * ST_CH + u) * ANV_BLOCK * 16), pn + u * ANV_BLOCK);
      if (NULLS) vw[s][u] = __ldg(wn + u * WSTEP);
    }
    pn += STEPV;
    if (NULLS) wn += WGRP;
  };
  auto consume = [&](int g, int s) {
#pragma unroll
    for (int u = 0; u < ST_CH; ++u) {
      const uint4 q = lds_v4(ring + (uint32_t)((s * ST_CH + u) * ANV_BLOCK * 16));
      T e[VEC];
      unpack<T>(q, e);
      int sl[VEC];
      vec(e, NULLS ? __funnelshift_r(vw[s][u], vw[s][u], vsh) : ANV_FULL, sl);
      if (ASSIGN) store_bins((g * STEPV + u * ANV_BLOCK + tid) * VEC, sl);
    }
  };
#pragma unroll
  for (int s = 0; s < ST_D; ++s) {  // prologue: one commit per slot, empty when the tile is short (keeps the group count fixed)
    if (s < n_groups) issue(s);
    cp_async_commit();
  }
  int g0 = 0;
  for (; g0 + 2 * ST_D <= n_groups; g0 += ST_D) {  // steady state: every slot is drained and refilled (conditions CTA-uniform)
#pragma unroll
    for (int s = 0; s < ST_D; ++s) {
      cp_async_wait<ST_D - 1>();     // ST_D + g groups committed so far: group g = g0 + s has landed
      consume(g0 + s, s);
      issue(s);                      // refill the slot just drained (same thread, LSU order: the LDS is ahead of the copy)
      cp_async_commit();
    }
  }
  for (; g0 < n_groups; g0 += ST_D) {              // drain: at most 2 * ST_D - 1 groups left
#pragma unroll
    for (int s = 0; s < ST_D; ++s) {
      const int g = g0 + s;
      if (g < n_groups) {
        cp_async_wait<ST_D - 1>();
        consume(g, s);
        if (g + ST_D < n_groups) issue(s);
        cp_async_commit();
      }
    }
  }
  cp_async_wait<0>();
  base = n_groups * STEPV;
  } else if constexpr (Tune<MOM, HPATH, ASSIGN>::PF) {
  // software pipeline: the loads of batch k+1 are in flight while batch k is consumed
  constexpr int HB = UNROLL / 2;  // vectors per half batch
  constexpr int STEP = ANV_BLOCK * HB;
  auto load_half = [&](int b, uint4 (&q)[HB], uint32_t (&vb)[HB]) {
    const uint4* p = vdata + b + tid;
    const uint32_t* wp = NULLS ? vwords + (((b + tid) * VEC) >> 5) : nullptr;
#pragma unroll
    for (int u = 0; u < HB; ++u) {
      q[u] = ldg_stream(p + u * ANV_BLOCK);
      if (NULLS) vb[u] = __ldg(wp + u * WSTEP);
    }
  };
  auto use_half = [&](int b, const uint4 (&q)[HB], const uint32_t (&vb)[HB]) {
#pragma unroll
    for (int u = 0; u < HB; ++u) {
      T e[VEC];
      unpack<T>(q[u], e);
      int sl[VEC];
      vec(e, NULLS ? __funnelshift_r(vb[u], vb[u], vsh) : ANV_FULL, sl);
      if (ASSIGN) store_bins((b + u * ANV_BLOCK + tid) * VEC, sl);
    }
  };
  if (STEP <= nvec) {
    uint4 qa[HB], qb[HB];
    uint32_t va[HB], vbb[HB];
    load_half(0, qa, va);
    // invariant at the top: qa holds the unconsumed half batch at `base` (all conditions are CTA-uniform)
    while (true) {
      const bool more_b = base + 2 * STEP <= nvec;
      if (more_b) load_half(base + STEP, qb, vbb);
      use_half(base, qa, va);
      base += STEP;
      if (!more_b) break;
      const bool more_a = base + 2 * STEP <= nvec;
      if (more_a) load_half(base + STEP, qa, va);
      use_half(base, qb, vbb);
      base += STEP;
      if (!more_a) break;
    }
  }
  } else {
  for (; base + ANV_BLOCK * UNROLL <= nvec; base += ANV_BLOCK * UNROLL) {
    uint4 q[UNROLL];
    uint32_t vb[UNROLL];
    const uint4* p = vdata + base + tid;
    const uint32_t* wp = NULLS ? vwords + (((base + tid) * VEC) >> 5) : nullptr;
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      q[u] = ldg_stream(p + u * ANV_BLOCK);
      if (NULLS) vb[u] = __ldg(wp + u * WSTEP);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      T e[VEC];
      unpack<T>(q[u], e);
      int sl[VEC];
      vec(e, NULLS ? __funnelshift_r(vb[u], vb[u], vsh) : ANV_FULL, sl);
      if (ASSIGN) store_bins((base + u * ANV_BLOCK + tid) * VEC, sl);
    }
  }
  }
  for (int j = base + tid; j < nvec; j += ANV_BLOCK) {  // remainder vectors
    const uint4 q = ldg_stream(vdata + j);
    const int row = j * VEC;
    uint32_t vb = ANV_FULL;
    if (NULLS) { const uint32_t w = __ldg(vwords + (row >> 5)); vb = __funnelshift_r(w, w, ((row & 31) + 31) & 31); }
    T e[VEC];
    unpack<T>(q, e);
    int sl[VEC];
    vec(e, vb, sl);
    if (ASSIGN) store_bins(row, sl);
  }
  if (tid == 0) {  // scalar tail (< VEC rows, last tile only)
    for (int row = nvec * VEC; row < n_tile; ++row) {
      bool valid = true;
      if (NULLS) valid = (vwords[row >> 5] >> (row & 31)) & 1u;
      const T x = valid ? data[row] : pivot_t;
      if (MOM) { mn = min(mn, x); mx = max(mx, x); }
      const int sl = elem(x, valid);
      if (ASSIGN) obins[row] = sl;
    }
  }

  // ---- undo the impersonation: this thread's null lanes were counted as pivot values --------
  // The streaming loop does not count valid lanes (that cost a mask, a POPC and two adds per vector): the tile's bitmap
  // words are popcounted here instead, 32 rows per load, each thread its own share of the words.  The corrections only
  // have to be right IN TOTAL over the CTA (the private counters and n_nz are summed over the threads afterwards), so every
  // thread corrects by the nulls of the words IT popcounted, whichever lanes impersonated them; a thread's counter may
  // wrap below zero on the way, the sums are taken modulo 2^32.
  uint32_t n_null = 0u;
  if (NULLS) {
    const int nw = (n_tile + 31) >> 5;
    uint32_t rows_cov = 0u;
    for (int w = tid; w < nw; w += ANV_BLOCK) {
      uint32_t v = __ldg(vwords + w);
      const int left = n_tile - (w << 5);
      if (left < 32) v &= (1u << left) - 1u;    // rows past the end of the frame
      n_ok += __popc(v);
      rows_cov += (uint32_t)min(left, 32);
    }
    n_null = rows_cov - n_ok;
  }
  if (NULLS && MOM && pivot_t != (T)0) n_nz -= n_null;
  if (NULLS && HPATH == 0 && n_null) {
    const int sp = bn.slot(pivot_t);
    cnt_t[sp * ANV_BLOCK] -= n_null;  // own private counters: plain read-modify-write
    cnt_t[0] += n_null;
  }

  // ---- K2 tile epilogue: fold the private counters, one integer atomic per slot -----------
  if (HIST && HPATH != 2) {
    __syncthreads();
    if (HPATH == 0) {
      for (int s = warp; s < n_slots; s += ANV_WARPS) {
        uint32_t v = 0;
#pragma unroll
        for (int i = 0; i < ANV_BLOCK / 32; ++i) v += cnt[s * ANV_BLOCK + i * 32 + lane];
        v = __reduce_add_sync(ANV_FULL, v);
        if (lane == 0 && v) atomicAdd(gcnt + s, (unsigned long long)v);
      }
    } else {
      for (int s = tid; s < n_slots; s += ANV_BLOCK) {
        const uint32_t v = cnt[s];
        if (v) atomicAdd(gcnt + s, (unsigned long long)v);
      }
    }
  }

  // ---- K1 tile epilogue: block reduce, convert to central form, write the partial ----------
  if (MOM) {
    if (!NULLS) {  // every row in range is valid: count analytically
      const int mine_full = (nvec > tid) ? (nvec - tid + ANV_BLOCK - 1) / ANV_BLOCK : 0;
      n_ok = (uint32_t)(mine_full * VEC) + (tid == 0 ? (uint32_t)(n_tile - nvec * VEC) : 0u);
    }
    double dmn = Traits<T>::to_double(mn), dmx = Traits<T>::to_double(mx);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += shfl_down_d(s1, o);
      s2 += shfl_down_d(s2, o);
      s3 += shfl_down_d(s3, o);
      s4 += shfl_down_d(s4, o);
      dmn = fmin(dmn, shfl_down_d(dmn, o));
      dmx = fmax(dmx, shfl_down_d(dmx, o));
      n_ok += __shfl_down_sync(ANV_FULL, n_ok, o);
      n_nz += __shfl_down_sync(ANV_FULL, n_nz, o);
    }
    if (lane == 0) {
      SS.red[warp][0] = s1; SS.red[warp][1] = s2; SS.red[warp][2] = s3; SS.red[warp][3] = s4;
      SS.red[warp][4] = dmn; SS.red[warp][5] = dmx;
      SS.redn[warp][0] = n_ok; SS.redn[warp][1] = n_nz;
    }
    __syncthreads();
    if (tid == 0) {
      double t1 = 0, t2 = 0, t3 = 0, t4 = 0, a = INFINITY, b = -INFINITY;
      uint32_t n32 = 0, nz32 = 0;   // modulo 2^32: a warp's nonzero partial may have wrapped (null corrections, above)
#pragma unroll
      for (int w = 0; w < ANV_WARPS; ++w) {  // fixed order: deterministic
        t1 += SS.red[w][0]; t2 += SS.red[w][1]; t3 += SS.red[w][2]; t4 += SS.red[w][3];
        a = fmin(a, SS.red[w][4]); b = fmax(b, SS.red[w][5]);
        n32 += SS.redn[w][0]; nz32 += SS.redn[w][1];
      }
      const int64_t n = (int64_t)n32, nz = (int64_t)nz32;   // a tile holds <= 262144 rows
      Partial out;
      out.n = n; out.nz = nz; out.mn = a; out.mx = b;
      if (n > 0) {
        // the power sums ran over n_tile lanes (null lanes contributed d == 0): shift to the mean of the n valid ones
        central_from_power_sums(out, pivot, t1, t2, t3, t4);
      } else {
        out.mean = 0.0; out.m2 = out.m3 = out.m4 = 0.0;
      }
      P.partials[(size_t)c * P.tiles_per_col + blockIdx.x] = out;
      if (NULLS) SS.fix = (!have_pivot && n > 0) ? 1 : 0;
    }
    if (NULLS) {
      // Rare repair: no finite non-null value among the first 1024 rows, so null lanes impersonated 0.  0 is not an
      // element: it may have polluted min / max, and power sums taken around 0 lose the spread to cancellation when the
      // values sit far from 0 (a column that starts partway through a table).  Redo the tile around its first finite
      // valid element.  A tile without one keeps pivot 0: its sums are NaN / inf whatever the pivot.
      __syncthreads();
      if (SS.fix) {
        int first = n_tile;
        for (int row = tid; row < n_tile; row += ANV_BLOCK) {
          if (((vwords[row >> 5] >> (row & 31)) & 1u) && isfinite(Traits<T>::to_double(data[row]))) {
            first = row;
            break;
          }
        }
        first = __reduce_min_sync(ANV_FULL, first);
        if (lane == 0) SS.redn[warp][0] = (uint32_t)first;
        __syncthreads();
        for (int w = 0; w < ANV_WARPS; ++w) first = min(first, (int)SS.redn[w][0]);
        const double pv = first < n_tile ? Traits<T>::to_double(data[first]) : 0.0;
        double a = INFINITY, b = -INFINITY, u1 = 0.0, u2 = 0.0, u3 = 0.0, u4 = 0.0;
        for (int row = tid; row < n_tile; row += ANV_BLOCK) {
          if ((vwords[row >> 5] >> (row & 31)) & 1u) {
            const double v = Traits<T>::to_double(data[row]);
            a = fmin(a, v);
            b = fmax(b, v);
            const double d = v - pv, d2 = d * d;
            u1 += d;
            u2 += d2;
            u3 = fma(d2, d, u3);
            u4 = fma(d2, d2, u4);
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          a = fmin(a, shfl_down_d(a, o));
          b = fmax(b, shfl_down_d(b, o));
          u1 += shfl_down_d(u1, o);
          u2 += shfl_down_d(u2, o);
          u3 += shfl_down_d(u3, o);
          u4 += shfl_down_d(u4, o);
        }
        if (lane == 0) {
          SS.red[warp][0] = u1; SS.red[warp][1] = u2; SS.red[warp][2] = u3; SS.red[warp][3] = u4;
          SS.red[warp][4] = a; SS.red[warp][5] = b;
        }
        __syncthreads();
        if (tid == 0) {
          for (int w = 1; w < ANV_WARPS; ++w) {  // fixed order: deterministic
            u1 += SS.red[w][0]; u2 += SS.red[w][1]; u3 += SS.red[w][2]; u4 += SS.red[w][3];
            a = fmin(a, SS.red[w][4]); b = fmax(b, SS.red[w][5]);
          }
          Partial& out = P.partials[(size_t)c * P.tiles_per_col + blockIdx.x];
          out.mn = a;
          out.mx = b;
          central_from_power_sums(out, pv, u1, u2, u3, u4);
        }
      }
    }
  }
}

template <bool MOM, int HPATH, bool ASSIGN, bool STAGED = false>
__global__ void __launch_bounds__(ANV_BLOCK, Tune<MOM, HPATH, ASSIGN>::MINB) scan_kernel(const ScanParams P) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ ScanShared SS;
  const int c = blockIdx.y;
  const anv_column_t col = P.cols[c];
  constexpr bool BINS = HPATH >= 0 || ASSIGN;
  int mode = BIN_SEARCH;
  if (BINS) mode = P.card ? BIN_CODE : P.specs[c].mode;
#define ANV_TILE(T, MODE)                                                                   \
  do {                                                                                      \
    /* columns with a bitmap keep the register-staged loop (measured: the cp.async ring pays */ \
    /* for null-free columns, +9 %, and costs 3 % where the bitmap words ride along)         */ \
    if (col.validity) scan_tile<T, MOM, HPATH, ASSIGN, true, MODE, false>(P, col, c, smem, SS);   \
    else scan_tile<T, MOM, HPATH, ASSIGN, false, MODE, STAGED>(P, col, c, smem, SS);        \
  } while (0)
  switch (col.dtype) {
    case ANV_F32:
      if (BINS && mode == BIN_GUESS) {
        // private-counter kernels: fold `x - lo` into the multiply-add when the guess stays within 1/32 bin (fold_ok)
        if ((HPATH == 0 && !ASSIGN) && fold_ok(P.specs[c])) ANV_TILE(float, (HPATH == 0 && !ASSIGN) ? BIN_GUESS_FOLD : BIN_GUESS);
        else ANV_TILE(float, BIN_GUESS);
      } else ANV_TILE(float, BIN_SEARCH);
      break;
    case ANV_F64:
      if (BINS && mode == BIN_GUESS) ANV_TILE(double, BIN_GUESS); else ANV_TILE(double, BIN_SEARCH);
      break;
    case ANV_I32:
      if (BINS && mode == BIN_CODE) ANV_TILE(int32_t, BIN_CODE); else ANV_TILE(int32_t, BIN_SEARCH);
      break;
    case ANV_I64: ANV_TILE(int64_t, BIN_SEARCH); break;
    default: break;
  }
#undef ANV_TILE
}

// ---- host-side helpers shared by the translation units -----------------------------------
int pick_tile_rows(int64_t n_rows, int n_cols);
size_t hist_smem(int count_stride, int* path, int* thr_slots, bool codes = false);
int check_common(const void* cols, int n_cols, int64_t n_rows);

template <bool MOM, int HPATH, bool ASSIGN, bool STAGED = false>
static int launch_scan(ScanParams& P, size_t smem, cudaStream_t st) {
  if (P.n_cols <= 0 || P.n_rows <= 0) return ANV_OK;
  dim3 grid((unsigned)((P.n_rows + P.tile_rows - 1) / P.tile_rows), (unsigned)P.n_cols);
  if (STAGED) {  // the ring sits behind the counters, 16-byte aligned
    P.stage_off = (uint32_t)((smem + 15) & ~(size_t)15);
    smem = P.stage_off + STAGE_BYTES;
    // four CTAs of (counters + ring) per SM need most of the 228 KB of an H100 SM: ask for the largest shared-memory carve-out
    ANV_CUDA(cudaFuncSetAttribute(scan_kernel<MOM, HPATH, ASSIGN, STAGED>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                  (int)cudaSharedmemCarveoutMaxShared));
  }
  if (smem > 40 * 1024)
    ANV_CUDA(cudaFuncSetAttribute(scan_kernel<MOM, HPATH, ASSIGN, STAGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  scan_kernel<MOM, HPATH, ASSIGN, STAGED><<<grid, ANV_BLOCK, smem, st>>>(P);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

// explicit-instantiation entry points (one per translation unit)
int launch_mom(ScanParams& P, cudaStream_t st);
int launch_hist(ScanParams& P, int path, size_t smem, cudaStream_t st);
int launch_fused(ScanParams& P, size_t smem, cudaStream_t st);
int launch_assign(ScanParams& P, size_t smem, cudaStream_t st);

}  // namespace anv
