// fdlibm 5.3's __ieee754_log, __ieee754_log10, __ieee754_exp and __ieee754_pow, restated as device functions.
//
// java.lang.StrictMath specifies these algorithms, so each result has one right bit pattern.  The code follows the
// published fdlibm sources step for step, with the word access __HI / __LO done on __double_as_longlong.  fdlibm
// specifies no fused multiply-add: the file that includes this header is compiled with -fmad=false, so every `a * b + c`
// here is a rounded multiply followed by a rounded add, as in the C reference.  tests/transform_oracle.py restates the
// same routines in Python, and the GPU tests compare the two bit for bit.
#pragma once
#include <cstdint>

namespace anv {
namespace fdlibm {

__device__ __forceinline__ int hi_word(double x) { return (int)(__double_as_longlong(x) >> 32); }
__device__ __forceinline__ unsigned lo_word(double x) { return (unsigned)(__double_as_longlong(x) & 0xffffffffull); }
__device__ __forceinline__ double from_words(int hi, unsigned lo) {
  return __longlong_as_double((long long)(((unsigned long long)(unsigned)hi << 32) | lo));
}
__device__ __forceinline__ double with_hi(double x, int hi) { return from_words(hi, lo_word(x)); }
__device__ __forceinline__ double with_lo(double x, unsigned lo) { return from_words(hi_word(x), lo); }

constexpr double two54 = 1.80143985094819840000e+16;
constexpr double twom54 = 5.55111512312578270212e-17;
constexpr double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10;
constexpr double huge = 1.0e300, tiny = 1.0e-300;

__device__ __forceinline__ double log(double x) {
  constexpr double Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01, Lg3 = 2.857142874366239149e-01,
                   Lg4 = 2.222219843214978396e-01, Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01,
                   Lg7 = 1.479819860511658591e-01;
  double hfsq, f, s, z, R, w, t1, t2, dk;
  int k, hx, i, j;
  unsigned lx;
  hx = hi_word(x);
  lx = lo_word(x);
  k = 0;
  if (hx < 0x00100000) {                                      // x < 2**-1022
    if (((hx & 0x7fffffff) | lx) == 0) return -__longlong_as_double(0x7ff0000000000000ll);   // log(+-0) = -inf
    if (hx < 0) return __longlong_as_double(0x7ff8000000000000ll);                             // log(-#) = NaN
    k -= 54;
    x *= two54;                                               // subnormal: scale up
    hx = hi_word(x);
  }
  if (hx >= 0x7ff00000) return x + x;
  k += (hx >> 20) - 1023;
  hx &= 0x000fffff;
  i = (hx + 0x95f64) & 0x100000;
  x = with_hi(x, hx | (i ^ 0x3ff00000));                      // normalize x or x/2
  k += (i >> 20);
  f = x - 1.0;
  if ((0x000fffff & (2 + hx)) < 3) {                          // |f| < 2**-20
    if (f == 0.0) {
      if (k == 0) return 0.0;
      dk = (double)k;
      return dk * ln2_hi + dk * ln2_lo;
    }
    R = f * f * (0.5 - 0.33333333333333333 * f);
    if (k == 0) return f - R;
    dk = (double)k;
    return dk * ln2_hi - ((R - dk * ln2_lo) - f);
  }
  s = f / (2.0 + f);
  dk = (double)k;
  z = s * s;
  i = hx - 0x6147a;
  w = z * z;
  j = 0x6b851 - hx;
  t1 = w * (Lg2 + w * (Lg4 + w * Lg6));
  t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)));
  i |= j;
  R = t2 + t1;
  if (i > 0) {
    hfsq = 0.5 * f * f;
    if (k == 0) return f - (hfsq - s * (hfsq + R));
    return dk * ln2_hi - ((hfsq - (s * (hfsq + R) + dk * ln2_lo)) - f);
  }
  if (k == 0) return f - s * (f - R);
  return dk * ln2_hi - ((s * (f - R) - dk * ln2_lo) - f);
}

__device__ __forceinline__ double log10(double x) {
  constexpr double ivln10 = 4.34294481903251816668e-01, log10_2hi = 3.01029995663611771306e-01,
                   log10_2lo = 3.69423907715893078616e-13;
  double y, z;
  int i, k, hx;
  unsigned lx;
  hx = hi_word(x);
  lx = lo_word(x);
  k = 0;
  if (hx < 0x00100000) {
    if (((hx & 0x7fffffff) | lx) == 0) return -__longlong_as_double(0x7ff0000000000000ll);
    if (hx < 0) return __longlong_as_double(0x7ff8000000000000ll);
    k -= 54;
    x *= two54;
    hx = hi_word(x);
  }
  if (hx >= 0x7ff00000) return x + x;
  k += (hx >> 20) - 1023;
  i = (int)(((unsigned)k & 0x80000000u) >> 31);
  hx = (hx & 0x000fffff) | ((0x3ff - i) << 20);
  y = (double)(k + i);
  x = with_hi(x, hx);
  z = y * log10_2lo + ivln10 * log(x);
  return z + y * log10_2hi;
}

constexpr double P1 = 1.66666666666666019037e-01, P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
                 P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;

__device__ __forceinline__ double exp(double x) {
  constexpr double o_threshold = 7.09782712893383973096e+02, u_threshold = -7.45133219101941108420e+02,
                   twom1000 = 9.33263618503218878990e-302, invln2 = 1.44269504088896338700e+00;
  double y, hi = 0.0, lo = 0.0, c, t;
  int k = 0, xsb;
  unsigned hx;
  hx = (unsigned)hi_word(x);
  xsb = (hx >> 31) & 1;
  hx &= 0x7fffffff;
  if (hx >= 0x40862E42) {                                     // |x| >= 709.78...
    if (hx >= 0x7ff00000) {
      if (((hx & 0xfffff) | lo_word(x)) != 0) return x + x;  // NaN
      return (xsb == 0) ? x : 0.0;                            // exp(+-inf) = {inf, 0}
    }
    if (x > o_threshold) return huge * huge;
    if (x < u_threshold) return twom1000 * twom1000;
  }
  if (hx > 0x3fd62e42) {                                      // |x| > 0.5 ln2
    if (hx < 0x3FF0A2B2) {                                    // and |x| < 1.5 ln2
      hi = x - (xsb ? -ln2_hi : ln2_hi);
      lo = xsb ? -ln2_lo : ln2_lo;
      k = 1 - xsb - xsb;
    } else {
      k = (int)(invln2 * x + (xsb ? -0.5 : 0.5));
      t = k;
      hi = x - t * ln2_hi;                                    // t * ln2_hi is exact here
      lo = t * ln2_lo;
    }
    x = hi - lo;
  } else if (hx < 0x3e300000) {                               // |x| < 2**-28
    if (huge + x > 1.0) return 1.0 + x;
  } else {
    k = 0;
  }
  t = x * x;
  c = x - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
  if (k == 0) return 1.0 - ((x * c) / (c - 2.0) - x);
  y = 1.0 - ((lo - (x * c) / (2.0 - c)) - hi);
  if (k >= -1021) return with_hi(y, hi_word(y) + (k << 20));
  return with_hi(y, hi_word(y) + ((k + 1000) << 20)) * twom1000;
}

__device__ __forceinline__ double pow(double x, double y) {
  constexpr double two53 = 9007199254740992.0;
  constexpr double L1 = 5.99999999999994648725e-01, L2 = 4.28571428578550184252e-01, L3 = 3.33333329818377432918e-01,
                   L4 = 2.72728123808534006489e-01, L5 = 2.30660745775561754067e-01, L6 = 2.06975017800338417784e-01;
  constexpr double lg2 = 6.93147180559945286227e-01, lg2_h = 6.93147182464599609375e-01,
                   lg2_l = -1.90465429995776804525e-09, ovt = 8.0085662595372944372e-17;
  constexpr double cp = 9.61796693925975554329e-01, cp_h = 9.61796700954437255859e-01, cp_l = -7.02846165095275826516e-09;
  constexpr double ivln2 = 1.44269504088896338700e+00, ivln2_h = 1.44269502162933349609e+00,
                   ivln2_l = 1.92596299112661746887e-08;
  double z, ax, z_h, z_l, p_h, p_l;
  double y1, t1, t2, r, s, t, u, v, w;
  int i, j, k, yisint, n;
  int hx, hy, ix, iy;
  unsigned lx, ly;

  hx = hi_word(x); lx = lo_word(x);
  hy = hi_word(y); ly = lo_word(y);
  ix = hx & 0x7fffffff; iy = hy & 0x7fffffff;

  if ((iy | ly) == 0) return 1.0;                             // x**0 = 1
  if (ix > 0x7ff00000 || ((ix == 0x7ff00000) && (lx != 0)) || iy > 0x7ff00000 || ((iy == 0x7ff00000) && (ly != 0)))
    return x + y;                                             // NaN

  // yisint = 0: y is not an integer, 1: an odd integer, 2: an even integer (decided when x < 0)
  yisint = 0;
  if (hx < 0) {
    if (iy >= 0x43400000) {
      yisint = 2;
    } else if (iy >= 0x3ff00000) {
      k = (iy >> 20) - 0x3ff;
      if (k > 20) {
        j = (int)(ly >> (52 - k));
        if (((unsigned)j << (52 - k)) == ly) yisint = 2 - (j & 1);
      } else if (ly == 0) {
        j = iy >> (20 - k);
        if ((j << (20 - k)) == iy) yisint = 2 - (j & 1);
      }
    }
  }

  if (ly == 0) {
    if (iy == 0x7ff00000) {                                   // y is +-inf
      if (((ix - 0x3ff00000) | lx) == 0) return y - y;        // (+-1)**+-inf is NaN
      if (ix >= 0x3ff00000) return (hy >= 0) ? y : 0.0;       // (|x|>1)**+-inf = inf, 0
      return (hy < 0) ? -y : 0.0;                             // (|x|<1)**-,+inf = inf, 0
    }
    if (iy == 0x3ff00000) return (hy < 0) ? 1.0 / x : x;      // y is +-1
    if (hy == 0x40000000) return x * x;                       // y is 2
    if (hy == 0x3fe00000 && hx >= 0) return __dsqrt_rn(x);    // y is 0.5, x >= +0
  }

  ax = fabs(x);
  if (lx == 0) {
    if (ix == 0x7ff00000 || ix == 0 || ix == 0x3ff00000) {    // x is +-0, +-inf, +-1
      z = ax;
      if (hy < 0) z = 1.0 / z;
      if (hx < 0) {
        if (((ix - 0x3ff00000) | yisint) == 0) z = (z - z) / (z - z);   // (-1)**non-int is NaN
        else if (yisint == 1) z = -z;
      }
      return z;
    }
  }

  n = (hx < 0) ? 0 : 1;                                       // fdlibm's (hx >> 31) + 1
  if ((n | yisint) == 0) return (x - x) / (x - x);            // (x<0)**(non-int) is NaN

  s = 1.0;
  if ((n | (yisint - 1)) == 0) s = -1.0;                      // (-ve)**(odd int)

  if (iy > 0x41e00000) {                                      // |y| > 2**31
    if (iy > 0x43f00000) {                                    // |y| > 2**64: must over/underflow
      if (ix <= 0x3fefffff) return (hy < 0) ? huge * huge : tiny * tiny;
      if (ix >= 0x3ff00000) return (hy > 0) ? huge * huge : tiny * tiny;
    }
    if (ix < 0x3fefffff) return (hy < 0) ? s * huge * huge : s * tiny * tiny;
    if (ix > 0x3ff00000) return (hy > 0) ? s * huge * huge : s * tiny * tiny;
    t = ax - 1.0;                                             // |1-x| <= 2**-20: log(x) by its series
    w = (t * t) * (0.5 - t * (0.3333333333333333333333 - t * 0.25));
    u = ivln2_h * t;
    v = t * ivln2_l - w * ivln2;
    t1 = with_lo(u + v, 0);
    t2 = v - (t1 - u);
  } else {
    double ss, s2, s_h, s_l, t_h, t_l;
    n = 0;
    if (ix < 0x00100000) {                                    // subnormal x
      ax *= two53;
      n -= 53;
      ix = hi_word(ax);
    }
    n += ((ix) >> 20) - 0x3ff;
    j = ix & 0x000fffff;
    ix = j | 0x3ff00000;
    if (j <= 0x3988E) k = 0;                                  // |x| < sqrt(3/2)
    else if (j < 0xBB67A) k = 1;                              // |x| < sqrt(3)
    else { k = 0; n += 1; ix -= 0x00100000; }
    ax = with_hi(ax, ix);
    const double bp = k ? 1.5 : 1.0, dp_h = k ? 5.84962487220764160156e-01 : 0.0,
                 dp_l = k ? 1.35003920212974897128e-08 : 0.0;

    u = ax - bp;                                              // ss = s_h + s_l = (x-1)/(x+1) or (x-1.5)/(x+1.5)
    v = 1.0 / (ax + bp);
    ss = u * v;
    s_h = with_lo(ss, 0);
    t_h = from_words(((ix >> 1) | 0x20000000) + 0x00080000 + (k << 18), 0);
    t_l = ax - (t_h - bp);
    s_l = v * ((u - s_h * t_h) - s_h * t_l);
    s2 = ss * ss;                                             // log(ax)
    r = s2 * s2 * (L1 + s2 * (L2 + s2 * (L3 + s2 * (L4 + s2 * (L5 + s2 * L6)))));
    r += s_l * (s_h + ss);
    s2 = s_h * s_h;
    t_h = with_lo(3.0 + s2 + r, 0);
    t_l = r - ((t_h - 3.0) - s2);
    u = s_h * t_h;
    v = s_l * t_h + t_l * ss;
    p_h = with_lo(u + v, 0);
    p_l = v - (p_h - u);
    z_h = cp_h * p_h;
    z_l = cp_l * p_h + p_l * cp + dp_l;
    t = (double)n;                                            // log2(ax) = n + dp_h + z_h + z_l
    t1 = with_lo(((z_h + z_l) + dp_h) + t, 0);
    t2 = z_l - (((t1 - t) - dp_h) - z_h);
  }

  y1 = with_lo(y, 0);                                         // (y1 + y2) * (t1 + t2)
  p_l = (y - y1) * t1 + y * t2;
  p_h = y1 * t1;
  z = p_l + p_h;
  j = hi_word(z);
  i = (int)lo_word(z);
  if (j >= 0x40900000) {                                      // z >= 1024
    if (((j - 0x40900000) | i) != 0) return s * huge * huge;
    if (p_l + ovt > z - p_h) return s * huge * huge;
  } else if ((j & 0x7fffffff) >= 0x4090cc00) {                // z <= -1075
    if (((j - (int)0xc090cc00) | i) != 0) return s * tiny * tiny;
    if (p_l <= z - p_h) return s * tiny * tiny;
  }
  i = j & 0x7fffffff;                                         // 2**(p_h + p_l)
  k = (i >> 20) - 0x3ff;
  n = 0;
  if (i > 0x3fe00000) {                                       // |z| > 0.5: n = [z + 0.5]
    n = j + (0x00100000 >> (k + 1));
    k = ((n & 0x7fffffff) >> 20) - 0x3ff;
    t = from_words(n & ~(0x000fffff >> k), 0);
    n = ((n & 0x000fffff) | 0x00100000) >> (20 - k);
    if (j < 0) n = -n;
    p_h -= t;
  }
  t = with_lo(p_l + p_h, 0);
  u = t * lg2_h;
  v = (p_l - (t - p_h)) * lg2 + t * lg2_l;
  z = u + v;
  w = v - (z - u);
  t = z * z;
  t1 = z - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
  r = (z * t1) / (t1 - 2.0) - (w + z * w);
  z = 1.0 - (r - z);
  j = hi_word(z);
  j += (n << 20);
  if ((j >> 20) <= 0) {                                       // subnormal output: fdlibm's scalbn(z, n)
    int e = ((hi_word(z) & 0x7ff00000) >> 20) + n;
    if (e <= -54) z = tiny * copysign(tiny, z);
    else z = from_words((hi_word(z) & 0x800fffff) | ((e + 54) << 20), lo_word(z)) * twom54;
  } else {
    z = with_hi(z, j);
  }
  return s * z;
}

}  // namespace fdlibm
}  // namespace anv
