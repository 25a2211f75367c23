// K6: HyperLogLog++ registers of Spark's approx_count_distinct(col, rsd)
// (reference /root/reference/src/main/anovos/data_analyzer/stats_generator.py:605-608).
// Spark hashes every non-null value with XXH64 (seed 42) using a per-type encoding
// (hashInt for int/float bits, hashLong for long/double bits), takes idx = top p bits and
// rho = clz(rest) + 1 and keeps the max per register.  max is order-independent, so the
// registers - and therefore the estimate - are bit-identical to Spark's whatever the
// partitioning.  Registers live in shared memory per CTA (plain read first: after warm-up
// almost no value raises a register, so atomics are rare), merged with global atomicMax.
#include "common.cuh"
#include "hll_hash.cuh"

namespace anv {

struct HllParams {
  const anv_column_t* cols;
  int n_cols;
  int64_t n_rows;
  int tile_rows;
  int p;
  uint32_t* regs;  // [n_cols][1 << p]
  int use_smem;
};

// SMEM: registers of the tile live in shared memory (p <= 14) - a compile-time fact, so the register update is an LDS +
// (rarely) an ATOMS.MAX instead of generic-address loads and atomics.
template <typename T, bool NULLS, bool SMEM>
__device__ __forceinline__ void hll_tile(const HllParams& P, const anv_column_t& col, int c, uint32_t* sh) {
  constexpr int VEC = Traits<T>::VEC;
  constexpr uint32_t VMASK = (1u << VEC) - 1u;
  const int tid = threadIdx.x;
  const int m = 1 << P.p;
  const int64_t r0 = (int64_t)blockIdx.x * P.tile_rows;
  const int64_t r1 = min(r0 + (int64_t)P.tile_rows, P.n_rows);
  const T* __restrict__ data = reinterpret_cast<const T*>(col.data);
  const uint32_t* __restrict__ vbits = col.validity;
  uint32_t* const G = P.regs + (size_t)c * m;
  if (SMEM) {
    for (int i = tid; i < m; i += ANV_BLOCK) sh[i] = 0;
    __syncthreads();
  }
  const int p = P.p;
  const int ps = 64 - p;
  const uint64_t guard = 1ull << (p - 1);
  auto elem = [&](T x, bool valid) {
    if (NULLS && !valid) return;
    const uint64_t h = spark_hash<T>(x);
    const uint32_t idx = (uint32_t)(h >> ps);
    const uint64_t w = (h << p) | guard;
    const uint32_t rho = (uint32_t)__clzll((long long)w) + 1u;
    if (SMEM) {
      if (rho > sh[idx]) atomicMax(&sh[idx], rho);     // after warm-up almost no value raises a register
    } else {
      if (rho > G[idx]) atomicMax(&G[idx], rho);
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
  if (SMEM) {
    __syncthreads();
    for (int i = tid; i < m; i += ANV_BLOCK) {
      const uint32_t v = sh[i];
      if (v) atomicMax(&G[i], v);
    }
  }
}

template <bool SMEM>
__global__ void __launch_bounds__(ANV_BLOCK) hll_kernel(const HllParams P) {
  extern __shared__ __align__(16) uint32_t hll_sh[];
  const int c = blockIdx.y;
  const anv_column_t col = P.cols[c];
#define ANV_DISPATCH(T)                                          \
  if (col.validity) hll_tile<T, true, SMEM>(P, col, c, hll_sh);  \
  else hll_tile<T, false, SMEM>(P, col, c, hll_sh);
  switch (col.dtype) {
    case ANV_F32: ANV_DISPATCH(float) break;
    case ANV_F64: ANV_DISPATCH(double) break;
    case ANV_I32: ANV_DISPATCH(int32_t) break;
    case ANV_I64: ANV_DISPATCH(int64_t) break;
    default: break;
  }
#undef ANV_DISPATCH
}

}  // namespace anv

using namespace anv;

extern "C" int anv_hll_registers(const anv_column_t* cols, int n_cols, int64_t n_rows, int p, uint32_t* regs,
                                 void* stream) {
  if (n_cols < 0 || n_rows < 0 || p < 4 || p > 18) { set_error("anv_hll_registers: bad arguments (4 <= p <= 18)"); return ANV_ERR_INVALID; }
  if (n_cols == 0) return ANV_OK;
  if (n_cols > ANV_MAX_LAUNCH_COLS) { set_error("n_cols > %d: split the frame into column blocks", ANV_MAX_LAUNCH_COLS); return ANV_ERR_UNSUPPORTED; }
  if (!cols || !regs) { set_error("anv_hll_registers: NULL argument"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  ANV_CUDA(cudaMemsetAsync(regs, 0, ((size_t)n_cols << p) * sizeof(uint32_t), st));
  if (n_rows == 0) return ANV_OK;
  HllParams P{};
  P.cols = cols; P.n_cols = n_cols; P.n_rows = n_rows; P.p = p; P.regs = regs;
  P.use_smem = p <= 14;
  int sms = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int64_t per_col = ((int64_t)sms * 4 + n_cols - 1) / n_cols;
  int64_t tr = n_rows / (per_col > 0 ? per_col : 1), t = 65536;
  while (t < tr && t < 1048576) t <<= 1;
  P.tile_rows = (int)t;
  const size_t smem = P.use_smem ? ((size_t)4 << p) : 0;
  if (smem > 48 * 1024)
    ANV_CUDA(cudaFuncSetAttribute(hll_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((unsigned)((n_rows + P.tile_rows - 1) / P.tile_rows), (unsigned)n_cols);
  if (P.use_smem) hll_kernel<true><<<grid, ANV_BLOCK, smem, st>>>(P);
  else hll_kernel<false><<<grid, ANV_BLOCK, 0, st>>>(P);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

// Host helper: Spark's XXH64 (seed 42) of UTF-8 strings given Arrow-style offsets.  Used for
// the (small) dictionaries of string columns; the per-row work stays on the device.
extern "C" int anv_xxh64_utf8(const uint8_t* bytes, const int64_t* offsets, int64_t n, uint64_t* out) {
  if (n < 0 || (n > 0 && (!offsets || !out))) { set_error("anv_xxh64_utf8: bad arguments"); return ANV_ERR_INVALID; }
  auto rd64 = [](const uint8_t* p) { uint64_t v = 0; for (int i = 7; i >= 0; --i) v = (v << 8) | p[i]; return v; };
  auto rd32 = [](const uint8_t* p) { uint32_t v = 0; for (int i = 3; i >= 0; --i) v = (v << 8) | p[i]; return v; };
  for (int64_t s = 0; s < n; ++s) {
    const uint8_t* b = bytes + offsets[s];
    const int64_t len = offsets[s + 1] - offsets[s];
    int64_t off = 0;
    uint64_t h;
    if (len >= 32) {
      uint64_t v1 = HLL_SEED + XP1 + XP2, v2 = HLL_SEED + XP2, v3 = HLL_SEED, v4 = HLL_SEED - XP1;
      for (; off + 32 <= len; off += 32) {
        v1 = rotl64(v1 + rd64(b + off) * XP2, 31) * XP1;
        v2 = rotl64(v2 + rd64(b + off + 8) * XP2, 31) * XP1;
        v3 = rotl64(v3 + rd64(b + off + 16) * XP2, 31) * XP1;
        v4 = rotl64(v4 + rd64(b + off + 24) * XP2, 31) * XP1;
      }
      h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
      const uint64_t vs[4] = {v1, v2, v3, v4};
      for (int i = 0; i < 4; ++i) h = (h ^ (rotl64(vs[i] * XP2, 31) * XP1)) * XP1 + XP4;
    } else {
      h = HLL_SEED + XP5;
    }
    h += (uint64_t)len;
    for (; off + 8 <= len; off += 8) { h ^= rotl64(rd64(b + off) * XP2, 31) * XP1; h = rotl64(h, 27) * XP1 + XP4; }
    if (off + 4 <= len) { h ^= (uint64_t)rd32(b + off) * XP1; h = rotl64(h, 23) * XP2 + XP3; off += 4; }
    for (; off < len; ++off) { h ^= (uint64_t)b[off] * XP5; h = rotl64(h, 11) * XP1; }
    out[s] = fmix64(h);
  }
  return ANV_OK;
}
