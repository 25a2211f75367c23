// Synthetic column generator for bench.py / tests (SURVEY.md 8d): counter-based
// Philox4x32-10, key = (seed, column), counter = (row/4, stream).  Any chunk of any
// column is reproducible independently of the launch geometry.
#include "common.cuh"

namespace anv {

__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0; key.y += W1;
  }
  return ctr;
}
// ---- deterministic float32 math ------------------------------------------------------------------
// Every operation below is a correctly rounded IEEE-754 binary32 add / mul / div / sqrt or an integer
// operation, written with the _rn intrinsics so that nvcc never contracts a mul + add into an FMA.  The
// NumPy twin (anovos_b200/synth.py: host_column / host_codes) performs the same operations in the same
// order, so a column generated on the host is BIT-IDENTICAL to the device column (SURVEY.md 8d: "(seed,
// column, row) so CPU baseline and GPU see identical values").  Accuracy of the elementary functions is
// ~1e-6 relative, which is all a synthetic distribution needs; MUFU-based __logf / __sincosf / __expf
// are not reproducible off the GPU and are not used.
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float mad(float a, float b, float c) { return __fadd_rn(__fmul_rn(a, b), c); }  // two roundings

__device__ __forceinline__ float u01(uint32_t b) {  // (0, 1]
  return mul(add(__uint2float_rn(b >> 8), 0.5f), 5.9604644775390625e-08f);
}

// natural logarithm of a positive normal float: x = m * 2^e, m in [sqrt(1/2), sqrt(2)),
// ln m = 2 s (1 + z/3 + z^2/5 + z^3/7 + z^4/9), s = (m-1)/(m+1), z = s^2
__device__ __forceinline__ float det_log(float x) {
  const uint32_t bits = __float_as_uint(x);
  int e = (int)(bits >> 23) - 127;
  float m = __uint_as_float((bits & 0x007FFFFFu) | 0x3F800000u);
  if (m > 1.41421354f) { m = mul(m, 0.5f); e += 1; }
  const float s = __fdiv_rn(sub(m, 1.0f), add(m, 1.0f));
  const float z = mul(s, s);
  float p = 0.111111112f;
  p = mad(p, z, 0.142857149f);
  p = mad(p, z, 0.2f);
  p = mad(p, z, 0.333333343f);
  p = mad(p, z, 1.0f);
  const float lnm = mul(mul(2.0f, s), p);
  return mad(__int2float_rn(e), 0.693147182f, lnm);
}

// e^y for |y| < 80: y = k ln2 + r, e^r by its Taylor polynomial of degree 6 (|r| <= 0.35), scaled by 2^k
__device__ __forceinline__ float det_exp(float y) {
  const float k = floorf(mad(y, 1.44269502f, 0.5f));
  float r = sub(y, mul(k, 0.693359375f));
  r = sub(r, mul(k, -2.12194440e-4f));
  float p = 1.38888892e-3f;
  p = mad(p, r, 8.33333377e-3f);
  p = mad(p, r, 4.16666679e-2f);
  p = mad(p, r, 0.166666672f);
  p = mad(p, r, 0.5f);
  p = mad(p, r, 1.0f);
  p = mad(p, r, 1.0f);
  int ki = (int)k;
  ki = ki < -126 ? -126 : (ki > 127 ? 127 : ki);
  return mul(p, __uint_as_float((uint32_t)(ki + 127) << 23));
}

// (cos, sin) of 2 pi u, u in (0, 1]: quadrant q = floor(4u), angle pi/4 + th inside it with
// th = (4u - q - 1/2) pi/2 in [-pi/4, pi/4): Taylor polynomials of sin / cos in th, then a rotation.
__device__ __forceinline__ void det_sincos2pi(float u, float& s_out, float& c_out) {
  const float t = mul(u, 4.0f);
  const int q = (int)t;
  const float f = sub(t, __int2float_rn(q));
  const float th = mul(sub(f, 0.5f), 1.57079637f);
  const float z = mul(th, th);
  float sp = 2.75573188e-6f;
  sp = mad(sp, z, -1.98412701e-4f);
  sp = mad(sp, z, 8.33333377e-3f);
  sp = mad(sp, z, -0.166666672f);
  sp = mad(sp, z, 1.0f);
  const float sn = mul(th, sp);
  float cp = -2.75573200e-7f;
  cp = mad(cp, z, 2.48015876e-5f);
  cp = mad(cp, z, -1.38888892e-3f);
  cp = mad(cp, z, 4.16666679e-2f);
  cp = mad(cp, z, -0.5f);
  const float cs = mad(cp, z, 1.0f);
  const float a = mul(sub(cs, sn), 0.707106769f);  // cos(pi/4 + th)
  const float b = mul(add(cs, sn), 0.707106769f);  // sin(pi/4 + th)
  switch (q & 3) {
    case 0: c_out = a; s_out = b; break;
    case 1: c_out = -b; s_out = a; break;
    case 2: c_out = -a; s_out = -b; break;
    default: c_out = b; s_out = -a; break;
  }
}

__device__ __forceinline__ void normals4(const uint4& r, float (&z)[4]) {  // Box-Muller
  const float r0 = __fsqrt_rn(mul(-2.0f, det_log(u01(r.x)))), r1 = __fsqrt_rn(mul(-2.0f, det_log(u01(r.z))));
  float s0, c0, s1, c1;
  det_sincos2pi(u01(r.y), s0, c0);
  det_sincos2pi(u01(r.w), s1, c1);
  z[0] = mul(r0, c0); z[1] = mul(r0, s0); z[2] = mul(r1, c1); z[3] = mul(r1, s1);
}

template <typename OutT, typename F>
__device__ __forceinline__ void synth_loop(OutT* data, uint32_t* validity, int64_t n_rows, int64_t row0, uint2 key, float null_rate, F gen) {
  const int64_t n4 = (n_rows + 3) / 4;
  const int64_t n4_pad = (n4 + 31) & ~(int64_t)31;  // whole warps so the bitmap words are assembled uniformly
  const uint32_t null_thr = (uint32_t)fminf(__fmul_rn(null_rate, 4294967296.0f), 4294967040.0f);
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n4_pad; j += (int64_t)gridDim.x * blockDim.x) {
    OutT v[4];
    const int64_t g = j + (row0 >> 2);  // counter of the GLOBAL row group: chunk [row0, row0+n) of a frame == the frame's rows
    const uint4 r = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), 0u, 0u), key);
    gen(r, v);
    const int64_t row = j * 4;
    if (row + 3 < n_rows) {
      if (sizeof(OutT) == 4) *reinterpret_cast<uint4*>(data + row) = *reinterpret_cast<uint4*>(v);
    } else {
      for (int i = 0; i < 4; ++i) if (row + i < n_rows) data[row + i] = v[i];
    }
    if (validity) {
      const uint4 nr = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), 1u, 0u), key);
      uint32_t nib = 0;
      nib |= (nr.x >= null_thr && row + 0 < n_rows) ? 1u : 0u;
      nib |= (nr.y >= null_thr && row + 1 < n_rows) ? 2u : 0u;
      nib |= (nr.z >= null_thr && row + 2 < n_rows) ? 4u : 0u;
      nib |= (nr.w >= null_thr && row + 3 < n_rows) ? 8u : 0u;
      uint32_t w = nib << ((threadIdx.x & 7) * 4);
      w |= __shfl_xor_sync(ANV_FULL, w, 1);
      w |= __shfl_xor_sync(ANV_FULL, w, 2);
      w |= __shfl_xor_sync(ANV_FULL, w, 4);
      if ((threadIdx.x & 7) == 0 && row < n_rows) validity[row >> 5] = w;
    }
  }
}

__global__ void __launch_bounds__(256) synth_f32_kernel(float* data, uint32_t* validity, int64_t n_rows, int64_t row0, uint2 key, int family,
                                                        float a, float b, float null_rate) {
  synth_loop<float>(data, validity, n_rows, row0, key, null_rate, [=](const uint4& r, float (&v)[4]) {
    if (family == 0) {
      normals4(r, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = mad(v[i], b, a);
    } else if (family == 1) {
      normals4(r, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = det_exp(mad(v[i], b, a));
    } else if (family == 2) {
      const float w = sub(b, a);
      v[0] = mad(u01(r.x), w, a); v[1] = mad(u01(r.y), w, a);
      v[2] = mad(u01(r.z), w, a); v[3] = mad(u01(r.w), w, a);
    } else {
      const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        // low 8 bits choose zero-inflation (70% exact zeros), high 24 bits the exponential
        const bool zero = (rr[i] & 0xffu) < 179u;
        v[i] = zero ? 0.0f : mul(-b, det_log(u01(rr[i])));
      }
    }
  });
}

__global__ void __launch_bounds__(256) synth_codes_kernel(int32_t* data, uint32_t* validity, int64_t n_rows, int64_t row0, uint2 key,
                                                          int card, float span, float inv, float null_rate) {
  synth_loop<int32_t>(data, validity, n_rows, row0, key, null_rate, [=](const uint4& r, int32_t (&v)[4]) {
    const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      // inverse CDF of the continuous power law on [1, card+1): Zipf-like ranks.  x = base^inv = exp(inv * ln base)
      const float x = det_exp(mul(inv, det_log(mad(u01(rr[i]), span, 1.0f))));
      v[i] = min(max((int)x - 1, 0), card - 1);
    }
  });
}

static uint2 make_key(uint64_t seed, uint32_t column) {
  const uint64_t k = seed ^ (0x9E3779B97F4A7C15ull * (uint64_t)(column + 1));
  return make_uint2((uint32_t)k, (uint32_t)(k >> 32));
}

}  // namespace anv

extern "C" int anv_synth_f32_rows(float* data, uint32_t* validity, int64_t n_rows, int64_t row0, uint64_t seed, uint32_t column,
                                  int family, float a, float b, float null_rate, void* stream) {
  if (!data || n_rows < 0 || row0 < 0 || (row0 & 31) || family < 0 || family > 3 || ((uintptr_t)data & 15)) {
    anv::set_error("anv_synth_f32: bad arguments (row0 must be a multiple of 32)");
    return ANV_ERR_INVALID;
  }
  if (n_rows == 0) return ANV_OK;
  const int64_t n4 = (n_rows + 3) / 4;
  const int blocks = (int)((n4 + 255) / 256 < 132 * 16 ? (n4 + 255) / 256 : 132 * 16);
  anv::synth_f32_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(data, validity, n_rows, row0, anv::make_key(seed, column), family,
                                                                  a, b, null_rate);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

extern "C" int anv_synth_f32(float* data, uint32_t* validity, int64_t n_rows, uint64_t seed, uint32_t column, int family,
                             float a, float b, float null_rate, void* stream) {
  return anv_synth_f32_rows(data, validity, n_rows, 0, seed, column, family, a, b, null_rate, stream);
}

extern "C" int anv_synth_codes_rows(int32_t* data, uint32_t* validity, int64_t n_rows, int64_t row0, uint64_t seed,
                                    uint32_t column, int cardinality, float zipf_s, float null_rate, void* stream) {
  if (!data || n_rows < 0 || row0 < 0 || (row0 & 31) || cardinality < 1 || zipf_s <= 1.0f || ((uintptr_t)data & 15)) {
    anv::set_error("anv_synth_codes: bad arguments (zipf_s must be > 1)");
    return ANV_ERR_INVALID;
  }
  if (n_rows == 0) return ANV_OK;
  const int64_t n4 = (n_rows + 3) / 4;
  const int blocks = (int)((n4 + 255) / 256 < 132 * 16 ? (n4 + 255) / 256 : 132 * 16);
  // span = (card+1)^(1-s) - 1 and inv = 1/(1-s) in double on the host (the NumPy twin does the same), rounded to float once
  const double oms = 1.0 - (double)zipf_s;
  const float span = (float)(pow((double)cardinality + 1.0, oms) - 1.0);
  const float inv = (float)(1.0 / oms);
  anv::synth_codes_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(data, validity, n_rows, row0, anv::make_key(seed, column),
                                                                    cardinality, span, inv, null_rate);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

extern "C" int anv_synth_codes(int32_t* data, uint32_t* validity, int64_t n_rows, uint64_t seed, uint32_t column,
                               int cardinality, float zipf_s, float null_rate, void* stream) {
  return anv_synth_codes_rows(data, validity, n_rows, 0, seed, column, cardinality, zipf_s, null_rate, stream);
}
