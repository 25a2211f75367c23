// feature_transformation and boxcox_transformation (reference data_transformer/transformers.py:3171-3486): one streaming
// pass per column writes op(x), with the semantics of the Spark expression the reference builds (header: ANV_TF_*).
//
// Grid (row tiles, columns), four rows per lane with 128-bit loads and stores (quad.cuh).  Each lane converts its quad to
// double (and to int64 for integer columns), evaluates the column's op on the four values and stores them in the output
// type, so the op code is compiled once per kernel whatever the input and output types.  The ops Java takes from
// java.lang.Math (cbrt and the trigonometric functions) run in a kernel of their own: CUDA's large-argument reduction of
// sin / cos / tan keeps an array in local memory, and the main kernel stays free of local memory.  Both kernels are
// launched over all columns; a CTA whose column belongs to the other kernel returns at once.
//
// This file is compiled with -fmad=false: every double operation is rounded on its own, as Java evaluates it.  The only
// fused multiply-adds are the explicit __fma_rn of the exact products and remainders in round_decimal.
//
// Null rows are written as 0.  Ops that make nulls (logs of x <= 0, 1 / 0, factorial outside 0..20) write the output
// bitmap: each lane tests its quad, the 8 lanes of a word OR their nibbles together and the word's first lane writes it.
// Null counts of the output: one atomic per warp.
#include "fdlibm.cuh"
#include "keysort.cuh"
#include "quad.cuh"

#include <algorithm>
#include <type_traits>

namespace anv {

__host__ __device__ __forceinline__ bool tf_is_math(int op) { return op >= ANV_TF_CBRT && op <= ANV_TF_ATAN; }
__host__ __device__ __forceinline__ bool tf_makes_nulls(int op) {
  return op == ANV_TF_LN || op == ANV_TF_LOG10 || op == ANV_TF_LOG2 || op == ANV_TF_MUL_INV || op == ANV_TF_FACTORIAL;
}

// The output types an op may write from a column of type `in` (header table).
__host__ __device__ __forceinline__ bool tf_valid(int op, int in, int out, long long n) {
  if (op < ANV_TF_LN || op > ANV_TF_ROUND) return false;
  if (op == ANV_TF_FLOOR || op == ANV_TF_CEIL || op == ANV_TF_FACTORIAL) return out == ANV_I64;
  if (op == ANV_TF_REMAINDER) {
    if (out == ANV_F64) return true;
    if (out == ANV_F32) return in == ANV_F32;
    if (out == ANV_I32) return in == ANV_I32 && n != 0;
    if (out == ANV_I64) return (in == ANV_I32 || in == ANV_I64) && n != 0;
    return false;
  }
  if (op == ANV_TF_ROUND) return out == in && (!(in == ANV_F32 || in == ANV_F64) || (n >= -22 && n <= 22));
  return out == ANV_F64;
}

// Double.toLong / Double.toInt: truncation toward zero, saturating, NaN -> 0.
__device__ __forceinline__ long long java_d2l(double v) {
  if (v != v) return 0;
  if (v >= 9223372036854775807.0) return 9223372036854775807ll;
  if (v <= -9223372036854775808.0) return (-9223372036854775807ll - 1);
  return (long long)v;
}
__device__ __forceinline__ int java_d2i(double v) {
  if (v != v) return 0;
  if (v >= 2147483647.0) return 2147483647;
  if (v <= -2147483648.0) return (-2147483647 - 1);
  return (int)v;
}

__device__ __forceinline__ double pow10_exact(int e) {       // 10^e for 0 <= e <= 22: every partial product is exact
  double p = 1.0;
  for (int i = 0; i < e; ++i) p *= 10.0;
  return p;
}

// The decimal M * 10^-n (M an integer below 2^53) read back as a double, correctly rounded (BigDecimal.doubleValue).
__device__ __forceinline__ double decimal_value(double M, int n) {
  return n >= 0 ? M / pow10_exact(n) : M * pow10_exact(-n);
}

// The same decimal correctly rounded to float (BigDecimal.floatValue): q is the decimal rounded to double and r the sign
// of the exact remainder; only a q that lies exactly halfway between two floats needs r.
__device__ __forceinline__ float decimal_value_f(double M, int n) {
  double q, r;
  if (n >= 0) {
    const double p = pow10_exact(n);
    q = M / p;
    r = __fma_rn(-q, p, M);
  } else {
    const double p = pow10_exact(-n);
    q = M * p;
    r = __fma_rn(M, p, -q);
  }
  float f = __double2float_rn(q);
  const double fd = (double)f;
  if (r != 0.0 && fd != q && isfinite(f)) {
    const float g = nextafterf(f, fd < q ? INFINITY : -INFINITY);
    if (((fd + (double)g) * 0.5) == q) f = (r > 0.0) == ((double)g > fd) ? g : f;
  }
  return f;
}

// Spark's round(x, n) of a float or double: BigDecimal(Double.toString(x)).setScale(n, HALF_UP), read back in x's type.
// Double.toString gives the shortest decimal d that reads back as x, so the answer is HALF_UP of d, not of x's binary
// value.  With y = |x| * 10^n (kept as hi + lo; lo's sign and zero are exact) and m = floor(y):
//   - if a decimal with n fraction digits reads back as x, d has at most n of them and the answer is x;
//   - otherwise d lies strictly between m and m + 1 (in units of 10^-n) and only its side of the tie t = m + 1/2 counts.
//     When t itself reads back as x, d is t unless the interval of decimals that read back as x holds an (n+1)-digit
//     decimal nearer to x; when it does not, d is on x's side of t.
__device__ __forceinline__ double round_decimal(double x, int n, bool to_float) {
  if (!isfinite(x)) return x;
  if (x == 0.0) return 0.0;                                    // BigDecimal has no -0
  const double ax = fabs(x);
  const double p = pow10_exact(n >= 0 ? n : -n);
  const double ulp = __longlong_as_double(__double_as_longlong(ax) + 1) - ax;
  // the interval of decimals that read back as x is ulp(x) wide: when that is at least 10^-n it holds a decimal with
  // n fraction digits, d has at most n of them and the answer is x
  if (n >= 0 ? ulp * p >= 1.0 : ulp >= p) return x;
  const double w = 0.5 * (n >= 0 ? ulp * p : ulp / p);        // the interval's half-width, in units of 10^-n
  double hi, lo;                                               // y = |x| 10^n = hi + lo, hi < 2^53
  if (n >= 0) {
    hi = ax * p;
    lo = __fma_rn(ax, p, -hi);
  } else {
    hi = ax / p;
    lo = __fma_rn(-hi, p, ax) / p;
  }
  double fl = floor(hi);
  if (fl == hi && lo < 0.0) fl -= 1.0;
  const double f = hi - fl;                                    // exact, in [0, 1]
  const double e = (f - 0.5) + lo;                             // frac(y) - 1/2 = x - t, to within rounding
  const int cmp = f != 0.5 ? (f > 0.5 ? 1 : -1) : (lo > 0.0) - (lo < 0.0);
  if (decimal_value(fl, n) == ax || decimal_value(fl + 1.0, n) == ax) return x;
  bool t_in;                                                   // does t read back as x?
  if (hi < 4503599627370496.0) {
    t_in = decimal_value(fl + 0.5, n) == ax;                   // fl + 1/2 is exact below 2^52
  } else {
    // ulp(hi) = 1, so f is 0 or 1 and |x - t| = |(f - 1/2) + lo|, which is 1/2 - |lo| when lo and f - 1/2 differ in
    // sign; here w is in [1/4, 1/2), so 1/2 - w is exact
    t_in = lo != 0.0 && (lo < 0.0) == (f > 0.5) && fabs(lo) >= 0.5 - w;
  }
  bool up;
  if (t_in) {
    double j = rint(10.0 * e);                                 // the (n+1)-digit decimal nearest x, relative to t
    if (j != 0.0 && fabs(10.0 * e - j) > 10.0 * w) j -= (j > 0.0 ? 1.0 : -1.0);
    up = j >= 0.0;
  } else {
    up = cmp > 0;
  }
  const double M = fl + (up ? 1.0 : 0.0);
  const double res = to_float ? (double)decimal_value_f(M, n) : decimal_value(M, n);
  if (res == 0.0) return 0.0;
  return x < 0.0 ? -res : res;
}

// HALF_UP of an integer at n < 0 decimal places, wrapping to 64 bits (BigDecimal.longValue; intValue keeps the low 32).
__device__ __forceinline__ long long round_integer(long long x, long long n) {
  if (n >= 0) return x;
  if (n <= -20) return 0;                                      // 10^20 > 2 |x|
  unsigned long long p = 1;
  for (long long i = 0; i < -n; ++i) p *= 10ull;
  const unsigned long long ax = x < 0 ? 0ull - (unsigned long long)x : (unsigned long long)x;
  const unsigned long long q = ax / p, r = ax % p;
  const unsigned long long m = (q + (r >= p - r ? 1ull : 0ull)) * p;
  return (long long)(x < 0 ? 0ull - m : m);
}

struct TfValue {
  double d;       // floating outputs
  long long i;    // integer outputs
  bool ok;        // false: the row is null
};

// op(x) of one row: v is x as a double, iv is x for integer columns.
template <bool MATH>
__device__ __forceinline__ TfValue tf_value(const anv_transform_spec_t& sp, int in, double v, long long iv) {
  TfValue o{0.0, 0, true};
  const bool is_int = in == ANV_I32 || in == ANV_I64;
  if constexpr (MATH) {
    switch (sp.op) {
      case ANV_TF_CBRT: o.d = cbrt(v); break;
      case ANV_TF_SIN: o.d = sin(v); break;
      case ANV_TF_COS: o.d = cos(v); break;
      case ANV_TF_TAN: o.d = tan(v); break;
      case ANV_TF_ASIN: o.d = asin(v); break;
      case ANV_TF_ACOS: o.d = acos(v); break;
      default: o.d = atan(v); break;
    }
    return o;
  } else {
    switch (sp.op) {
      case ANV_TF_LN: o.ok = !(v <= 0.0); o.d = fdlibm::log(v); break;
      case ANV_TF_LOG10: o.ok = !(v <= 0.0); o.d = fdlibm::log10(v); break;
      case ANV_TF_LOG2: o.ok = !(v <= 0.0); o.d = fdlibm::log(v) / fdlibm::log(2.0); break;
      case ANV_TF_EXP: o.d = fdlibm::exp(v); break;
      case ANV_TF_POW_BASE: o.d = fdlibm::pow(sp.a, v); break;
      case ANV_TF_POW: o.d = fdlibm::pow(v, sp.a); break;
      case ANV_TF_SQRT: o.d = __dsqrt_rn(v); break;
      case ANV_TF_RADIANS: o.d = v * 0.017453292519943295; break;
      case ANV_TF_MUL_INV: o.ok = v != 0.0; o.d = 1.0 / v; break;
      case ANV_TF_FLOOR: o.i = is_int ? iv : java_d2l(floor(v)); break;
      case ANV_TF_CEIL: o.i = is_int ? iv : java_d2l(ceil(v)); break;
      case ANV_TF_FACTORIAL: {
        const int k = in == ANV_I32 ? (int)iv : in == ANV_I64 ? (int)(unsigned)(unsigned long long)iv : java_d2i(v);
        o.ok = k >= 0 && k <= 20;
        long long f = 1;
        for (int j = 2; j <= (o.ok ? k : 0); ++j) f *= j;
        o.i = f;
        break;
      }
      case ANV_TF_REMAINDER:
        if (sp.out_dtype == ANV_F32 || sp.out_dtype == ANV_F64) o.d = fmod(v, sp.a);
        else o.i = sp.n == -1 ? 0 : iv % sp.n;
        break;
      default:                                                 // ANV_TF_ROUND
        if (is_int) o.i = round_integer(iv, sp.n);
        else o.d = round_decimal(v, (int)sp.n, in == ANV_F32);
        break;
    }
    return o;
  }
}

template <typename T> __device__ __forceinline__ void load_as(const void* src, int64_t r, int64_t n_rows, double (&v)[4],
                                                              long long (&iv)[4]) {
  T e[4];
  load_quad<T>((const T*)src, r, n_rows, e);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    v[k] = (double)e[k];
    if constexpr (std::is_floating_point<T>::value) iv[k] = 0;
    else iv[k] = (long long)e[k];
  }
}

template <typename U> __device__ __forceinline__ void store_as(void* dst, int64_t r, const TfValue (&o)[4]) {
  U e[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if constexpr (std::is_floating_point<U>::value) e[k] = o[k].ok ? (U)o[k].d : U(0);
    else e[k] = o[k].ok ? (U)o[k].i : U(0);
  }
  store_quad<U>((U*)dst, r, e);
}

template <bool MATH>
__global__ void __launch_bounds__(ANV_BLOCK) transform_kernel(const anv_column_t* __restrict__ cols,
                                                              const anv_transform_spec_t* __restrict__ specs,
                                                              void* const* __restrict__ out_ptrs,
                                                              uint32_t* const* __restrict__ out_valid_ptrs,
                                                              unsigned long long* __restrict__ null_counts, int64_t n_rows) {
  const int c = blockIdx.y;
  const anv_column_t col = cols[c];
  const anv_transform_spec_t sp = specs[c];
  if (tf_is_math(sp.op) != MATH || !tf_valid(sp.op, col.dtype, sp.out_dtype, sp.n)) return;   // uniform per CTA
  const bool nulls_out = tf_makes_nulls(sp.op);
  uint32_t* out_valid = nulls_out && out_valid_ptrs ? out_valid_ptrs[c] : nullptr;
  if (nulls_out && !out_valid) return;
  void* dst = out_ptrs[c];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t step = (int64_t)gridDim.x * QUAD_ROWS_PER_CTA;
  unsigned long long nulls = 0;
  for (int64_t r0 = (int64_t)blockIdx.x * QUAD_ROWS_PER_CTA + (int64_t)warp * QUAD_ROWS_PER_WARP; r0 < n_rows; r0 += step) {
    const uint32_t vb = quad_valid_bits(col.validity, r0, n_rows, lane);
    const int64_t r = r0 + lane * QUAD_ROWS_PER_LANE;
    uint32_t keep = 0;
    if (r < n_rows) {
      double v[4];
      long long iv[4];
      switch (col.dtype) {
        case ANV_F32: load_as<float>(col.data, r, n_rows, v, iv); break;
        case ANV_F64: load_as<double>(col.data, r, n_rows, v, iv); break;
        case ANV_I32: load_as<int32_t>(col.data, r, n_rows, v, iv); break;
        default: load_as<int64_t>(col.data, r, n_rows, v, iv); break;
      }
      TfValue o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        o[k] = tf_value<MATH>(sp, col.dtype, v[k], iv[k]);
        const bool live = r + k < n_rows;
        o[k].ok = o[k].ok && live && ((vb >> k) & 1u);
        keep |= (uint32_t)o[k].ok << k;
        nulls += (unsigned long long)(live && !o[k].ok);
      }
      switch (sp.out_dtype) {
        case ANV_F32: store_as<float>(dst, r, o); break;
        case ANV_F64: store_as<double>(dst, r, o); break;
        case ANV_I32: store_as<int32_t>(dst, r, o); break;
        default: store_as<int64_t>(dst, r, o); break;
      }
    }
    if (nulls_out) {
      uint32_t word = keep << (4 * (lane & 7));
      word |= __shfl_xor_sync(ANV_FULL, word, 1);
      word |= __shfl_xor_sync(ANV_FULL, word, 2);
      word |= __shfl_xor_sync(ANV_FULL, word, 4);
      const int64_t w = r0 / 32 + (lane >> 3);
      if ((lane & 7) == 0 && w * 32 < n_rows) out_valid[w] = word;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nulls += __shfl_down_sync(ANV_FULL, nulls, o);
  if (lane == 0 && nulls) atomicAdd(null_counts + c, nulls);
}

// ---- Box-Cox lambda search: the Kolmogorov-Smirnov statistics of every candidate from one sort ------------------------
//
// The reference tests y = pow(x, lambda) for 14 lambdas and y = log(x) against N(0, 1) (Statistics.kolmogorovSmirnovTest)
// and keeps the best p-value.  Null rows enter every test as the value 0.  On positive data each transform is monotone in
// x, so the column is sorted once (as 64-bit keys: the bits of a positive double order like its value; null rows get key
// 0 and sort first) and the rank of every valid value in each transformed sample follows from its rank among the valid
// values: pow with lambda > 0 keeps the order after the n_null zeros, lambda < 0 reverses it, and log puts the values
// below 1 before the zeros and the others after them.  ks_candidates_kernel reduces, per candidate, the largest
//   max(Phi(y) - (r - 1) / n, r / n - Phi(y))
// over the valid values (r is y's 1-based rank among all n rows).  Over a run of ties that maximum is reached at the
// run's ends, so ties need no care.  The run of zeros is one term per candidate, which the host adds (it needs the count
// of values below 1, which the kernel also returns).

constexpr int KS_MAX_LAMBDAS = 16;
struct KsParams {
  double lam[KS_MAX_LAMBDAS];   // pow candidates, then one log candidate
  int n_pow;
  int64_t n_rows, n_null;
  const uint64_t* buf[2];       // the sort's ping-pong buffers; *cur picks the sorted one
  const int* cur;
};

// NormalDistribution(0, 1).cumulativeProbability: 0.5 * erfc(-x / sqrt(2)), 0 / 1 beyond 40 standard deviations.
__device__ __forceinline__ double std_normal_cdf(double x) {
  if (fabs(x) > 40.0) return x < 0.0 ? 0.0 : 1.0;
  return 0.5 * erfc(-x / 1.4142135623730951);
}

__global__ void ks_keys_kernel(const anv_column_t* __restrict__ cols, int c, int64_t n_rows, uint64_t* __restrict__ keys) {
  const anv_column_t col = cols[c];
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    const bool valid = !col.validity || ((__ldg(col.validity + r / 32) >> (r % 32)) & 1u);
    double v = 0.0;
    if (valid) {
      switch (col.dtype) {
        case ANV_F32: v = (double)((const float*)col.data)[r]; break;
        case ANV_F64: v = ((const double*)col.data)[r]; break;
        case ANV_I32: v = (double)((const int32_t*)col.data)[r]; break;
        default: v = (double)((const int64_t*)col.data)[r]; break;
      }
    }
    keys[r] = valid ? (unsigned long long)__double_as_longlong(v) : 0ull;
  }
}

// d_out [n_pow + 1] holds the statistics as the bits of non-negative doubles (atomicMax on their integer image).
__global__ void __launch_bounds__(ANV_BLOCK) ks_candidates_kernel(const KsParams P, unsigned long long* __restrict__ d_out,
                                                                  unsigned long long* __restrict__ n_below_one) {
  __shared__ double red[KS_MAX_LAMBDAS][ANV_WARPS];
  const uint64_t* sorted = P.buf[*P.cur];
  const int64_t n_valid = P.n_rows - P.n_null;
  const double n = (double)P.n_rows;
  const int n_cand = P.n_pow + 1;
  double best[KS_MAX_LAMBDAS];
#pragma unroll
  for (int k = 0; k < KS_MAX_LAMBDAS; ++k) best[k] = 0.0;
  unsigned long long below = 0;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_valid; j += (int64_t)gridDim.x * blockDim.x) {
    const double x = __longlong_as_double((long long)sorted[P.n_null + j]);
#pragma unroll
    for (int k = 0; k < KS_MAX_LAMBDAS; ++k) {
      if (k > P.n_pow) break;
      double y, r;
      if (k < P.n_pow) {
        y = fdlibm::pow(x, P.lam[k]);
        r = (double)(P.n_null + (P.lam[k] > 0.0 ? j : n_valid - 1 - j) + 1);
      } else {
        y = fdlibm::log(x);
        r = (double)(j + (x < 1.0 ? 0 : P.n_null) + 1);
      }
      const double f = std_normal_cdf(y);
      best[k] = fmax(best[k], fmax(f - (r - 1.0) / n, r / n - f));
    }
    below += x < 1.0;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < KS_MAX_LAMBDAS; ++k) {
    double v = best[k];
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_down_sync(ANV_FULL, v, o));
    if (lane == 0) red[k][warp] = v;
  }
  for (int o = 16; o > 0; o >>= 1) below += __shfl_down_sync(ANV_FULL, below, o);
  if (lane == 0 && below) atomicAdd(n_below_one, below);
  __syncthreads();
  if (threadIdx.x < n_cand) {
    double v = 0.0;
    for (int w = 0; w < ANV_WARPS; ++w) v = fmax(v, red[threadIdx.x][w]);
    atomicMax(d_out + threadIdx.x, (unsigned long long)__double_as_longlong(v));
  }
}

int check_common(const void* cols, int n_cols, int64_t n_rows);

}  // namespace anv

using namespace anv;

extern "C" int anv_transform_columns(const anv_column_t* cols, const anv_transform_spec_t* specs, void* const* out_ptrs,
                                     uint32_t* const* out_valid_ptrs, int64_t* null_counts, int n_cols, int64_t n_rows, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0) return ANV_OK;
  if (!specs || !out_ptrs || !null_counts) {
    set_error("anv_transform_columns: specs / out_ptrs / null_counts is NULL");
    return ANV_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  ANV_CUDA(cudaMemsetAsync(null_counts, 0, (size_t)n_cols * sizeof(int64_t), st));
  if (n_rows == 0) return ANV_OK;
  dim3 grid(quad_grid_x(n_rows, n_cols), (unsigned)n_cols);
  auto* nc = reinterpret_cast<unsigned long long*>(null_counts);
  transform_kernel<false><<<grid, ANV_BLOCK, 0, st>>>(cols, specs, out_ptrs, out_valid_ptrs, nc, n_rows);
  ANV_CUDA(cudaGetLastError());
  transform_kernel<true><<<grid, ANV_BLOCK, 0, st>>>(cols, specs, out_ptrs, out_valid_ptrs, nc, n_rows);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

extern "C" size_t anv_ks_candidates_workspace_bytes(int64_t n_rows) {
  return key_sort64_workspace_bytes(n_rows);
}

extern "C" int anv_ks_candidates(const anv_column_t* cols, int c, int64_t n_rows, int64_t n_null, const double* lambdas,
                                 int n_pow, double* d_out, int64_t* n_below_one, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  if (!cols || c < 0 || n_rows < 0 || n_null < 0 || n_null > n_rows || !lambdas || n_pow < 0 || n_pow >= KS_MAX_LAMBDAS ||
      !d_out || !n_below_one || !workspace) {
    set_error("anv_ks_candidates: bad arguments");
    return ANV_ERR_INVALID;
  }
  if (n_rows >= ((int64_t)1 << 32)) { set_error("anv_ks_candidates: n_rows >= 2^32 is not supported"); return ANV_ERR_UNSUPPORTED; }
  if (workspace_bytes < anv_ks_candidates_workspace_bytes(n_rows)) {
    set_error("anv_ks_candidates: workspace too small (%zu < %zu)", workspace_bytes, anv_ks_candidates_workspace_bytes(n_rows));
    return ANV_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  ANV_CUDA(cudaMemsetAsync(d_out, 0, (size_t)(n_pow + 1) * sizeof(double), st));
  ANV_CUDA(cudaMemsetAsync(n_below_one, 0, sizeof(int64_t), st));
  if (n_rows == 0) return ANV_OK;
  char* w = reinterpret_cast<char*>(workspace);
  const size_t sort_bytes = key_sort64_workspace_bytes(n_rows);
  KeySort64 ks;
  key_sort64_bind(w, n_rows, &ks);
  const int grid = (int)std::min<int64_t>((n_rows + ANV_BLOCK - 1) / ANV_BLOCK, 132 * 16);
  ks_keys_kernel<<<grid, ANV_BLOCK, 0, st>>>(cols, c, n_rows, ks.buf[0]);
  ANV_CUDA(cudaGetLastError());
  if (int rc = key_sort64(w, sort_bytes, n_rows, 0, 8, st)) return rc;
  KsParams P{};
  for (int k = 0; k < n_pow; ++k) P.lam[k] = lambdas[k];
  P.n_pow = n_pow;
  P.n_rows = n_rows;
  P.n_null = n_null;
  P.buf[0] = ks.buf[0];
  P.buf[1] = ks.buf[1];
  P.cur = ks.cur;
  ks_candidates_kernel<<<grid, ANV_BLOCK, 0, st>>>(P, reinterpret_cast<unsigned long long*>(d_out),
                                                    reinterpret_cast<unsigned long long*>(n_below_one));
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}
