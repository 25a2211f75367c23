// K4: exact multi-rank selection per column (radix select on order-preserving keys).
//
// Replaces the Greenwald-Khanna sketches behind Spark's summary() percentiles and
// approxQuantile (reference /root/reference/src/main/anovos/data_analyzer/
// stats_generator.py:488,813,908 and data_transformer/transformers.py:215).  Spark
// returns an element within eps*n ranks of rank ceil(p*n); this kernel returns the
// element of exactly that rank (rank error 0, inside the reference's own band).
//
// Pass 0 histograms the top 12 key bits of every non-null value (4096 bins in shared
// memory); a tiny scan kernel locates, for each requested rank, the bin it falls in and
// the residual rank inside it; passes 1.. refine 10 more bits, touching shared memory
// only for values whose prefix matches one of the <= 16 (deduplicated) target prefixes,
// found through a 4096-cell hash table of the target prefixes (one byte load + one compare).
// 3 passes for 32-bit keys, 7 for 64-bit keys; all counting is integer => deterministic.
#include "common.cuh"

namespace anv {

constexpr int SEL_MAX_RANKS = 16;
constexpr int SEL_BITS0 = 12, SEL_BITS = 10;

struct SelState {  // one per column, lives in the caller's workspace
  uint64_t prefix[SEL_MAX_RANKS];       // key bits decided so far (right-aligned), per rank
  int64_t rank[SEL_MAX_RANKS];          // residual 1-based rank inside the prefix bucket (0 = skip)
  int32_t slot[SEL_MAX_RANKS];          // histogram slot of each rank (ranks sharing a prefix share a slot)
  uint64_t slot_prefix[SEL_MAX_RANKS];  // prefix of each slot
  int32_t n_slots;
  int32_t pad;
};

template <typename T> __device__ __forceinline__ uint64_t sort_key(T x);
template <> __device__ __forceinline__ uint64_t sort_key<float>(float x) {
  x += 0.0f;  // -0.0 -> +0.0
  uint32_t u = __float_as_uint(x);
  u = (x != x) ? 0xFFFFFFFFu : ((u & 0x80000000u) ? ~u : (u | 0x80000000u));  // NaN sorts last (Spark)
  return (uint64_t)u << 32;
}
template <> __device__ __forceinline__ uint64_t sort_key<int32_t>(int32_t x) {
  return (uint64_t)((uint32_t)x ^ 0x80000000u) << 32;
}
template <> __device__ __forceinline__ uint64_t sort_key<double>(double x) {
  x += 0.0;
  uint64_t u = (uint64_t)__double_as_longlong(x);
  return (x != x) ? ~0ull : ((u >> 63) ? ~u : (u | (1ull << 63)));
}
template <> __device__ __forceinline__ uint64_t sort_key<int64_t>(int64_t x) {
  return (uint64_t)x ^ (1ull << 63);
}

__device__ __forceinline__ double key_to_double(uint64_t k, int dtype) {
  switch (dtype) {
    case ANV_F32: {
      uint32_t u = (uint32_t)(k >> 32);
      u = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u;
      return (double)__uint_as_float(u);
    }
    case ANV_I32: return (double)(int32_t)((uint32_t)(k >> 32) ^ 0x80000000u);
    case ANV_F64: {
      uint64_t u = (k >> 63) ? (k & ~(1ull << 63)) : ~k;
      return __longlong_as_double((long long)u);
    }
    default: return (double)(int64_t)(k ^ (1ull << 63));
  }
}

struct SelParams {
  const anv_column_t* cols;
  int n_cols;
  int64_t n_rows;
  int tile_rows;
  int n_ranks;
  SelState* state;
  unsigned long long* hist;  // [n_cols][n_ranks][1 << SEL_BITS] (pass 0: [n_cols][1 << SEL_BITS0])
  int pass, shift, bits;     // digit = (key >> shift) & ((1 << bits) - 1); prefix = key >> (shift + bits)
};

struct SelShared {  // declared ONCE in the kernel (statics inside the templated tile body would be replicated per instantiation)
  uint64_t prefix[SEL_MAX_RANKS];
  uint32_t tbl[(1 << SEL_BITS0) / 4];  // byte table: hash(prefix) -> slot (0xFF = no target prefix hashes here)
  int nslots;
};

// 12-bit multiplicative hash of a decided-bits prefix (the top-12-bit bucket alone is a poor filter for
// floats: it holds sign + exponent + 3 mantissa bits, so a handful of buckets cover most of a column)
__device__ __forceinline__ uint32_t prefix_hash(uint64_t pf) {
  const uint32_t x = (uint32_t)pf * 0x9E3779B1u + (uint32_t)(pf >> 32) * 0x85EBCA77u;
  return x >> (32 - SEL_BITS0);
}

template <typename T, bool NULLS, bool FIRST>
__device__ __forceinline__ void select_tile(const SelParams& P, const anv_column_t& col, int c, uint32_t* sh, SelShared& SS) {
  constexpr int VEC = Traits<T>::VEC;
  constexpr uint32_t VMASK = (1u << VEC) - 1u;
  const int tid = threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.x * P.tile_rows;
  const int64_t r1 = min(r0 + (int64_t)P.tile_rows, P.n_rows);
  const T* __restrict__ data = reinterpret_cast<const T*>(col.data);
  const uint32_t* __restrict__ vbits = col.validity;
  const int nbins = 1 << P.bits;
  const uint32_t dmask = (uint32_t)nbins - 1u;

  uint64_t* s_prefix = SS.prefix;
  uint8_t* s_tbl = reinterpret_cast<uint8_t*>(SS.tbl);
  int& s_nslots = SS.nslots;
  int n_slots = 1;
  if (!FIRST) {
    const SelState& S = P.state[c];
    if (tid == 0) s_nslots = S.n_slots;
    for (int i = tid; i < (1 << SEL_BITS0) / 4; i += ANV_BLOCK) SS.tbl[i] = 0xFFFFFFFFu;
    __syncthreads();
    n_slots = s_nslots;
    if (n_slots == 0) return;  // nothing requested for this column (uniform per CTA)
    if (tid < n_slots) s_prefix[tid] = S.slot_prefix[tid];
    __syncthreads();
    if (tid == 0) {  // first slot wins a hash cell (deterministic); colliding prefixes fall back to the linear search
      for (int q = 0; q < n_slots; ++q) {
        const uint32_t h = prefix_hash(s_prefix[q]);
        if (s_tbl[h] == 0xFFu) s_tbl[h] = (uint8_t)q;
      }
    }
  }
  for (int i = tid; i < n_slots * nbins; i += ANV_BLOCK) sh[i] = 0;
  __syncthreads();

  // Per-thread run aggregation: a heavy value (e.g. the 70% exact zeros of a zero-inflated column) lands
  // in ONE counter; consecutive hits of the same counter are added once instead of serialising the
  // whole CTA on one shared-memory address.
  uint32_t run_idx = 0xffffffffu, run_cnt = 0;
  auto count = [&](uint32_t idx) {
    if (idx == run_idx) { ++run_cnt; return; }
    if (run_cnt) atomicAdd(&sh[run_idx], run_cnt);
    run_idx = idx; run_cnt = 1;
  };
  auto elem = [&](T x, bool valid) {
    if (NULLS && !valid) return;
    const uint64_t k = sort_key<T>(x);
    const uint32_t d = (uint32_t)(k >> P.shift) & dmask;
    if (FIRST) {
      atomicAdd(&sh[d], 1u);   // 4096 bins: contention is not the limiter here (measured), keep the loop lean
    } else {
      const uint64_t pf = k >> (P.shift + P.bits);
      const uint32_t cand = s_tbl[prefix_hash(pf)];
      if (cand != 0xFFu) {
        if (s_prefix[cand] == pf) {
          count(cand * (uint32_t)nbins + d);
        } else {  // hash collision between two target prefixes, or a foreign prefix in a used cell: rare
          for (int s = 0; s < n_slots; ++s)
            if (s_prefix[s] == pf) { count((uint32_t)(s * nbins) + d); break; }
        }
      }
    }
  };

  const int64_t nvec = (r1 - r0) / VEC;
  const uint4* __restrict__ vdata = reinterpret_cast<const uint4*>(data + r0);
  constexpr int U = 4;
  int64_t base = 0;
  for (; base + (int64_t)ANV_BLOCK * U <= nvec; base += (int64_t)ANV_BLOCK * U) {
    uint4 q[U];
    uint32_t vb[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t j = base + u * ANV_BLOCK + tid;
      q[u] = ldg_stream(vdata + j);
      if (NULLS) {
        const int64_t row = r0 + j * VEC;
        vb[u] = (__ldg(vbits + (row >> 5)) >> (row & 31)) & VMASK;
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      T e[VEC];
      unpack<T>(q[u], e);
#pragma unroll
      for (int i = 0; i < VEC; ++i) elem(e[i], NULLS ? ((vb[u] >> i) & 1u) : true);
    }
  }
  for (int64_t j = base + tid; j < nvec; j += ANV_BLOCK) {
    const uint4 q = ldg_stream(vdata + j);
    const int64_t row = r0 + j * VEC;
    uint32_t vb = VMASK;
    if (NULLS) vb = (__ldg(vbits + (row >> 5)) >> (row & 31)) & VMASK;
    T e[VEC];
    unpack<T>(q, e);
#pragma unroll
    for (int i = 0; i < VEC; ++i) elem(e[i], (vb >> i) & 1u);
  }
  if (tid == 0) {
    for (int64_t row = r0 + nvec * VEC; row < r1; ++row) {
      bool valid = true;
      if (NULLS) valid = (vbits[row >> 5] >> (row & 31)) & 1u;
      elem(data[row], valid);
    }
  }
  if (run_cnt) atomicAdd(&sh[run_idx], run_cnt);
  __syncthreads();
  unsigned long long* out = P.hist + (size_t)c * P.n_ranks * (1 << SEL_BITS);
  if (FIRST) out = P.hist + (size_t)c * (1 << SEL_BITS0);
  for (int i = tid; i < n_slots * nbins; i += ANV_BLOCK) {
    const uint32_t v = sh[i];
    if (v) atomicAdd(out + i, (unsigned long long)v);
  }
}

template <bool FIRST>
__global__ void __launch_bounds__(ANV_BLOCK) select_pass_kernel(const SelParams P) {
  extern __shared__ __align__(16) uint32_t sel_sh[];
  __shared__ SelShared SS;
  const int c = blockIdx.y;
  const anv_column_t col = P.cols[c];
#define ANV_DISPATCH(T)                                                \
  if (col.validity) select_tile<T, true, FIRST>(P, col, c, sel_sh, SS); \
  else select_tile<T, false, FIRST>(P, col, c, sel_sh, SS);
  switch (col.dtype) {
    case ANV_F32: ANV_DISPATCH(float) break;
    case ANV_F64: ANV_DISPATCH(double) break;
    case ANV_I32: ANV_DISPATCH(int32_t) break;
    case ANV_I64: ANV_DISPATCH(int64_t) break;
    default: break;
  }
#undef ANV_DISPATCH
}

// One CTA per column: locate every rank's digit in its slot histogram, update the
// prefixes / residual ranks, re-deduplicate the slots and clear the histogram.
__global__ void __launch_bounds__(256) select_scan_kernel(SelState* state, unsigned long long* hist, const int64_t* ranks,
                                                          int n_ranks, int pass, int bits, int last, int total_bits,
                                                          const anv_column_t* cols, double* out) {
  const int c = blockIdx.x, tid = threadIdx.x;
  SelState& S = state[c];
  const int nbins = 1 << bits;
  __shared__ unsigned long long cum[1 << SEL_BITS0];
  __shared__ unsigned long long wsum[8];
  __shared__ int s_digit[SEL_MAX_RANKS];
  __shared__ long long s_below[SEL_MAX_RANKS];
  if (pass == 0 && tid == 0) {  // initial state: every requested rank shares slot 0, empty prefix
    int any = 0;
    for (int r = 0; r < n_ranks; ++r) {
      S.rank[r] = ranks[(size_t)c * n_ranks + r];
      S.prefix[r] = 0;
      S.slot[r] = 0;
      any |= S.rank[r] > 0;
    }
    S.slot_prefix[0] = 0;
    S.n_slots = any ? 1 : 0;
  }
  __syncthreads();
  const int n_slots = S.n_slots;
  unsigned long long* H = hist + (size_t)c * (pass == 0 ? (1 << SEL_BITS0) : n_ranks * (1 << SEL_BITS));
  for (int s = 0; s < n_slots; ++s) {
    // inclusive scan of this slot's histogram (nbins <= 4096 = 256 threads x 16)
    const int per = (nbins + 255) / 256;
    unsigned long long loc[16];
    unsigned long long run = 0;
    for (int i = 0; i < per; ++i) {
      const int b = tid * per + i;
      if (b < nbins) run += H[s * nbins + b];
      loc[i] = run;
    }
    unsigned long long v = run;
    for (int o = 1; o < 32; o <<= 1) {
      unsigned long long n = __shfl_up_sync(ANV_FULL, v, o);
      if ((tid & 31) >= o) v += n;
    }
    if ((tid & 31) == 31) wsum[tid >> 5] = v;
    __syncthreads();
    unsigned long long woff = 0;
    for (int w = 0; w < (tid >> 5); ++w) woff += wsum[w];
    const unsigned long long excl = woff + v - run;
    for (int i = 0; i < per; ++i)
      if (tid * per + i < nbins) cum[tid * per + i] = excl + loc[i];
    __syncthreads();
    // each rank of this slot: first bin with cum >= rank (binary search by one thread per rank)
    if (tid < n_ranks && S.rank[tid] > 0 && S.slot[tid] == s) {
      const unsigned long long r = (unsigned long long)S.rank[tid];
      int lo = 0, hi = nbins - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cum[mid] >= r) hi = mid; else lo = mid + 1;
      }
      s_digit[tid] = lo;
      s_below[tid] = lo ? (long long)cum[lo - 1] : 0;
    }
    __syncthreads();
  }
  if (tid == 0) {
    int ns = 0;
    for (int r = 0; r < n_ranks; ++r) {
      if (S.rank[r] <= 0) continue;
      S.prefix[r] = (S.prefix[r] << bits) | (uint64_t)s_digit[r];
      S.rank[r] -= s_below[r];
      int found = -1;
      for (int q = 0; q < ns; ++q) if (S.slot_prefix[q] == S.prefix[r]) { found = q; break; }
      if (found < 0) { found = ns; S.slot_prefix[ns++] = S.prefix[r]; }
      S.slot[r] = found;
    }
    S.n_slots = ns;
    if (last) {
      const int dt = cols[c].dtype;
      for (int r = 0; r < n_ranks; ++r)
        out[(size_t)c * n_ranks + r] = (ranks[(size_t)c * n_ranks + r] > 0)
            ? key_to_double(total_bits < 64 ? (S.prefix[r] << (64 - total_bits)) : S.prefix[r], dt) : nan("");
    }
  }
  __syncthreads();
  // clear what the next pass will accumulate into
  const size_t nclear = (size_t)n_ranks * (1 << SEL_BITS);
  unsigned long long* Hn = hist + (size_t)c * nclear;
  if (pass == 0) {
    for (int i = tid; i < (1 << SEL_BITS0); i += 256) H[i] = 0;
  } else {
    for (size_t i = tid; i < nclear; i += 256) Hn[i] = 0;
  }
}

static int sel_tile_rows(int64_t n_rows, int n_cols) {
  int sms = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int64_t want = (int64_t)sms * 4;
  int64_t per_col = (want + n_cols - 1) / (n_cols > 0 ? n_cols : 1);
  int64_t tr = per_col > 0 ? n_rows / per_col : n_rows;
  int64_t t = 32768;
  while (t < tr && t < 1048576) t <<= 1;
  return (int)t;
}

}  // namespace anv

using namespace anv;

// hist0 [n_cols][4096] u64 and histN [n_cols][n_ranks][1024] u64 are SEPARATE regions of the workspace.
extern "C" size_t anv_select_workspace_bytes(int n_cols, int n_ranks) {
  if (n_cols <= 0 || n_ranks <= 0) return 64;
  return (size_t)n_cols * sizeof(SelState) + (size_t)n_cols * (1 << SEL_BITS0) * 8 +
         (size_t)n_cols * n_ranks * (1 << SEL_BITS) * 8 + 256;
}

namespace {
struct SelLayout {
  SelState* state;
  unsigned long long* hist0;
  unsigned long long* histN;
  size_t h0, hN;
};
SelLayout sel_layout(void* workspace, int n_cols, int n_ranks) {
  char* w = reinterpret_cast<char*>(workspace);
  SelLayout L;
  L.state = reinterpret_cast<SelState*>(w);
  const size_t off = ((size_t)n_cols * sizeof(SelState) + 127) & ~(size_t)127;
  L.hist0 = reinterpret_cast<unsigned long long*>(w + off);
  L.h0 = (size_t)n_cols * (1 << SEL_BITS0) * 8;
  L.histN = reinterpret_cast<unsigned long long*>(w + off + L.h0);
  L.hN = (size_t)n_cols * n_ranks * (1 << SEL_BITS) * 8;
  return L;
}
// digit width / position of pass `pass` (12 bits first, then 10 at a time); returns 0 past the last pass
int sel_pass_geometry(int key_bits, int pass, int* bits, int* shift) {
  int decided = 0;
  for (int p = 0; decided < key_bits; ++p) {
    const int b = p == 0 ? SEL_BITS0 : ((key_bits - decided) < SEL_BITS ? (key_bits - decided) : SEL_BITS);
    if (p == pass) { *bits = b; *shift = 64 - decided - b; return (decided + b >= key_bits) ? 2 : 1; }
    decided += b;
  }
  return 0;
}
int sel_check(const char* who, int n_cols, int n_ranks, int key_bits, const void* ws, size_t ws_bytes) {
  if (n_cols < 0 || n_ranks < 1 || n_ranks > SEL_MAX_RANKS || (key_bits != 32 && key_bits != 64)) {
    set_error("%s: bad arguments (1 <= n_ranks <= %d, key_bits 32|64)", who, SEL_MAX_RANKS);
    return ANV_ERR_INVALID;
  }
  if (n_cols > ANV_MAX_LAUNCH_COLS) { set_error("n_cols > %d: split the frame into column blocks", ANV_MAX_LAUNCH_COLS); return ANV_ERR_UNSUPPORTED; }
  if (n_cols && !ws) { set_error("%s: NULL workspace", who); return ANV_ERR_INVALID; }
  if (n_cols && ws_bytes < anv_select_workspace_bytes(n_cols, n_ranks)) {
    set_error("%s: workspace too small", who);
    return ANV_ERR_WORKSPACE;
  }
  return ANV_OK;
}
}  // namespace

extern "C" int anv_select_passes(int key_bits) { return key_bits == 32 ? 3 : (key_bits == 64 ? 7 : -1); }

extern "C" int anv_select_begin(int n_cols, int n_ranks, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = sel_check("anv_select_begin", n_cols, n_ranks, 32, workspace, workspace_bytes)) return rc;
  if (n_cols == 0) return ANV_OK;
  const SelLayout L = sel_layout(workspace, n_cols, n_ranks);
  ANV_CUDA(cudaMemsetAsync(L.hist0, 0, L.h0 + L.hN, (cudaStream_t)stream));
  return ANV_OK;
}

extern "C" int anv_select_hist_region(int n_cols, int n_ranks, int pass, size_t* offset, size_t* bytes) {
  if (n_cols < 0 || n_ranks < 1 || n_ranks > SEL_MAX_RANKS || pass < 0 || !offset || !bytes) {
    set_error("anv_select_hist_region: bad arguments");
    return ANV_ERR_INVALID;
  }
  const size_t off = ((size_t)n_cols * sizeof(SelState) + 127) & ~(size_t)127;
  const size_t h0 = (size_t)n_cols * (1 << SEL_BITS0) * 8;
  *offset = pass == 0 ? off : off + h0;
  *bytes = pass == 0 ? h0 : (size_t)n_cols * n_ranks * (1 << SEL_BITS) * 8;
  return ANV_OK;
}

extern "C" int anv_select_accumulate(const anv_column_t* cols, int n_cols, int64_t n_rows, int n_ranks, int key_bits,
                                     int pass, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = sel_check("anv_select_accumulate", n_cols, n_ranks, key_bits, workspace, workspace_bytes)) return rc;
  int bits = 0, shift = 0;
  if (n_rows < 0 || !sel_pass_geometry(key_bits, pass, &bits, &shift)) {
    set_error("anv_select_accumulate: bad pass %d / n_rows", pass);
    return ANV_ERR_INVALID;
  }
  if (n_cols == 0 || n_rows == 0) return ANV_OK;
  if (!cols) { set_error("anv_select_accumulate: NULL argument"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const SelLayout L = sel_layout(workspace, n_cols, n_ranks);
  SelParams P{};
  P.cols = cols; P.n_cols = n_cols; P.n_rows = n_rows; P.n_ranks = n_ranks; P.state = L.state;
  P.tile_rows = sel_tile_rows(n_rows, n_cols);
  P.pass = pass; P.bits = bits; P.shift = shift;
  P.hist = pass == 0 ? L.hist0 : L.histN;
  dim3 grid((unsigned)((n_rows + P.tile_rows - 1) / P.tile_rows), (unsigned)n_cols);
  if (pass == 0) {
    select_pass_kernel<true><<<grid, ANV_BLOCK, (size_t)(1 << SEL_BITS0) * 4, st>>>(P);
  } else {
    const size_t smemN = (size_t)n_ranks * (1 << SEL_BITS) * 4;
    if (smemN > 40 * 1024)
      ANV_CUDA(cudaFuncSetAttribute(select_pass_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemN));
    select_pass_kernel<false><<<grid, ANV_BLOCK, smemN, st>>>(P);
  }
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

extern "C" int anv_select_advance(const anv_column_t* cols, int n_cols, const int64_t* ranks, int n_ranks, int key_bits,
                                  int pass, double* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = sel_check("anv_select_advance", n_cols, n_ranks, key_bits, workspace, workspace_bytes)) return rc;
  int bits = 0, shift = 0;
  const int g = sel_pass_geometry(key_bits, pass, &bits, &shift);
  if (!g) { set_error("anv_select_advance: bad pass %d", pass); return ANV_ERR_INVALID; }
  if (n_cols == 0) return ANV_OK;
  if (!cols || !ranks || !out) { set_error("anv_select_advance: NULL argument"); return ANV_ERR_INVALID; }
  const SelLayout L = sel_layout(workspace, n_cols, n_ranks);
  select_scan_kernel<<<n_cols, 256, 0, (cudaStream_t)stream>>>(L.state, pass == 0 ? L.hist0 : L.histN, ranks, n_ranks, pass,
                                                                bits, g == 2, key_bits, cols, out);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

extern "C" int anv_select_ranks(const anv_column_t* cols, int n_cols, int64_t n_rows, const int64_t* ranks, int n_ranks,
                                int key_bits, double* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = sel_check("anv_select_ranks", n_cols, n_ranks, key_bits, workspace, workspace_bytes)) return rc;
  if (n_rows < 0) { set_error("anv_select_ranks: n_rows < 0"); return ANV_ERR_INVALID; }
  if (n_cols == 0) return ANV_OK;
  if (!cols || !ranks || !out) { set_error("anv_select_ranks: NULL argument"); return ANV_ERR_INVALID; }
  if (int rc = anv_select_begin(n_cols, n_ranks, workspace, workspace_bytes, stream)) return rc;
  const int n_pass = anv_select_passes(key_bits);
  for (int pass = 0; pass < n_pass; ++pass) {
    if (int rc = anv_select_accumulate(cols, n_cols, n_rows, n_ranks, key_bits, pass, workspace, workspace_bytes, stream)) return rc;
    if (int rc = anv_select_advance(cols, n_cols, ranks, n_ranks, key_bits, pass, out, workspace, workspace_bytes, stream)) return rc;
  }
  return ANV_OK;
}
