"""Reference semantics of feature_transformation and boxcox_transformation (reference transformers.py:3171-3486) in plain
Python, for the tests.

- fdlibm 5.3's __ieee754_log, __ieee754_log10, __ieee754_exp and __ieee754_pow, which java.lang.StrictMath specifies,
  restated on Python floats (IEEE doubles; every operation rounded on its own, no fused multiply-add).  Word access goes
  through struct.
- Spark's typing and null rules of the expressions the reference builds (log of x <= 0 and 1 / 0 are null, floor / ceil
  / factorial are bigint, x % N takes the wider type, round keeps it).
- round(x, N) as BigDecimal(Double.toString(x)).setScale(N, HALF_UP): repr() is the shortest round-trip decimal, and
  decimal does the HALF_UP.
- `transform_reference` is the exact image of one column of anv_transform_columns, except for the java.lang.Math group
  (cbrt, sin ... atan), where it uses Python's math module and the kernel uses CUDA's functions.
"""
from __future__ import annotations

import decimal
import math
import struct
from fractions import Fraction

import numpy as np

F32, F64, I32, I64 = 0, 1, 2, 3
(LN, LOG10, LOG2, EXP, POW_BASE, POW, SQRT, CBRT, SIN, COS, TAN, ASIN, ACOS, ATAN, RADIANS, MUL_INV, FLOOR, CEIL, FACTORIAL,
 REMAINDER, ROUND) = range(21)
MATH_OPS = (CBRT, SIN, COS, TAN, ASIN, ACOS, ATAN)
MAKES_NULLS = (LN, LOG10, LOG2, MUL_INV, FACTORIAL)
NP_OF = {F32: np.float32, F64: np.float64, I32: np.int32, I64: np.int64}
METHODS = ["ln", "log10", "log2", "exp", "powOf2", "powOf10", "powOfN", "sqrt", "cbrt", "sq", "cb", "toPowerN", "sin", "cos",
           "tan", "asin", "acos", "atan", "radians", "remainderDivByN", "factorial", "mul_inv", "floor", "ceil", "roundN"]
INF, NAN = float("inf"), float("nan")


# ---- word access ---------------------------------------------------------------------------------------------------

def _bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def _hi(x):
    return _bits(x) >> 32                       # signed, like fdlibm's __HI


def _lo(x):
    return _bits(x) & 0xffffffff


def _make(hi, lo):
    u = ((hi & 0xffffffff) << 32) | (lo & 0xffffffff)
    return struct.unpack("<d", struct.pack("<Q", u))[0]


def _i32(v):
    v &= 0xffffffff
    return v - (1 << 32) if v >= 1 << 31 else v


def _mul(a, b):
    """a * b with IEEE overflow to inf (Python raises instead)."""
    return float(np.float64(a) * np.float64(b))


# ---- fdlibm 5.3 -----------------------------------------------------------------------------------------------------

two54 = 1.80143985094819840000e+16
twom54 = 5.55111512312578270212e-17
ln2_hi, ln2_lo = 6.93147180369123816490e-01, 1.90821492927058770002e-10
Lg1, Lg2, Lg3 = 6.666666666666735130e-01, 3.999999999940941908e-01, 2.857142874366239149e-01
Lg4, Lg5, Lg6, Lg7 = 2.222219843214978396e-01, 1.818357216161805012e-01, 1.531383769920937332e-01, 1.479819860511658591e-01
P1, P2, P3 = 1.66666666666666019037e-01, -2.77777777770155933842e-03, 6.61375632143793436117e-05
P4, P5 = -1.65339022054652515390e-06, 4.13813679705723846039e-08


def fd_log(x):
    hx, lx = _hi(x), _lo(x)
    k = 0
    if hx < 0x00100000:
        if ((hx & 0x7fffffff) | lx) == 0:
            return -INF
        if hx < 0:
            return NAN
        k -= 54
        x *= two54
        hx = _hi(x)
    if hx >= 0x7ff00000:
        return x + x
    k += (hx >> 20) - 1023
    hx &= 0x000fffff
    i = (hx + 0x95f64) & 0x100000
    x = _make(hx | (i ^ 0x3ff00000), _lo(x))
    k += i >> 20
    f = x - 1.0
    if (0x000fffff & (2 + hx)) < 3:
        if f == 0.0:
            if k == 0:
                return 0.0
            dk = float(k)
            return dk * ln2_hi + dk * ln2_lo
        R = f * f * (0.5 - 0.33333333333333333 * f)
        if k == 0:
            return f - R
        dk = float(k)
        return dk * ln2_hi - ((R - dk * ln2_lo) - f)
    s = f / (2.0 + f)
    dk = float(k)
    z = s * s
    i = hx - 0x6147a
    w = z * z
    j = 0x6b851 - hx
    t1 = w * (Lg2 + w * (Lg4 + w * Lg6))
    t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)))
    i |= j
    R = t2 + t1
    if i > 0:
        hfsq = 0.5 * f * f
        if k == 0:
            return f - (hfsq - s * (hfsq + R))
        return dk * ln2_hi - ((hfsq - (s * (hfsq + R) + dk * ln2_lo)) - f)
    if k == 0:
        return f - s * (f - R)
    return dk * ln2_hi - ((s * (f - R) - dk * ln2_lo) - f)


def fd_log10(x):
    ivln10, log10_2hi, log10_2lo = 4.34294481903251816668e-01, 3.01029995663611771306e-01, 3.69423907715893078616e-13
    hx, lx = _hi(x), _lo(x)
    k = 0
    if hx < 0x00100000:
        if ((hx & 0x7fffffff) | lx) == 0:
            return -INF
        if hx < 0:
            return NAN
        k -= 54
        x *= two54
        hx = _hi(x)
    if hx >= 0x7ff00000:
        return x + x
    k += (hx >> 20) - 1023
    i = 1 if k < 0 else 0
    hx = (hx & 0x000fffff) | ((0x3ff - i) << 20)
    y = float(k + i)
    x = _make(hx, _lo(x))
    z = y * log10_2lo + ivln10 * fd_log(x)
    return z + y * log10_2hi


def fd_exp(x):
    o_threshold, u_threshold = 7.09782712893383973096e+02, -7.45133219101941108420e+02
    invln2 = 1.44269504088896338700e+00
    hx = _hi(x) & 0xffffffff
    xsb = (hx >> 31) & 1
    hx &= 0x7fffffff
    hi = lo = 0.0
    k = 0
    if hx >= 0x40862E42:
        if hx >= 0x7ff00000:
            if ((hx & 0xfffff) | _lo(x)) != 0:
                return x + x
            return x if xsb == 0 else 0.0
        if x > o_threshold:
            return INF
        if x < u_threshold:
            return 0.0
    if hx > 0x3fd62e42:
        if hx < 0x3FF0A2B2:
            hi = x - (-ln2_hi if xsb else ln2_hi)
            lo = -ln2_lo if xsb else ln2_lo
            k = 1 - xsb - xsb
        else:
            k = int(invln2 * x + (-0.5 if xsb else 0.5))          # C's (int) truncates toward zero
            t = float(k)
            hi = x - t * ln2_hi
            lo = t * ln2_lo
        x = hi - lo
    elif hx < 0x3e300000:
        return 1.0 + x
    t = x * x
    c = x - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))))
    if k == 0:
        return 1.0 - ((x * c) / (c - 2.0) - x)
    y = 1.0 - ((lo - (x * c) / (2.0 - c)) - hi)
    if k >= -1021:
        return _make(_hi(y) + (k << 20), _lo(y))
    return _make(_hi(y) + ((k + 1000) << 20), _lo(y)) * 9.33263618503218878990e-302


def fd_pow(x, y):
    two53 = 9007199254740992.0
    L1, L2, L3 = 5.99999999999994648725e-01, 4.28571428578550184252e-01, 3.33333329818377432918e-01
    L4, L5, L6 = 2.72728123808534006489e-01, 2.30660745775561754067e-01, 2.06975017800338417784e-01
    lg2, lg2_h, lg2_l = 6.93147180559945286227e-01, 6.93147182464599609375e-01, -1.90465429995776804525e-09
    ovt = 8.0085662595372944372e-17
    cp, cp_h, cp_l = 9.61796693925975554329e-01, 9.61796700954437255859e-01, -7.02846165095275826516e-09
    ivln2, ivln2_h, ivln2_l = 1.44269504088896338700e+00, 1.44269502162933349609e+00, 1.92596299112661746887e-08
    hx, lx, hy, ly = _hi(x), _lo(x), _hi(y), _lo(y)
    ix, iy = hx & 0x7fffffff, hy & 0x7fffffff
    if (iy | ly) == 0:
        return 1.0
    if ix > 0x7ff00000 or (ix == 0x7ff00000 and lx != 0) or iy > 0x7ff00000 or (iy == 0x7ff00000 and ly != 0):
        return x + y
    yisint = 0
    if hx < 0:
        if iy >= 0x43400000:
            yisint = 2
        elif iy >= 0x3ff00000:
            k = (iy >> 20) - 0x3ff
            if k > 20:
                j = ly >> (52 - k)
                if ((j << (52 - k)) & 0xffffffff) == ly:
                    yisint = 2 - (j & 1)
            elif ly == 0:
                j = iy >> (20 - k)
                if (j << (20 - k)) == iy:
                    yisint = 2 - (j & 1)
    if ly == 0:
        if iy == 0x7ff00000:
            if ((ix - 0x3ff00000) | lx) == 0:
                return NAN
            if ix >= 0x3ff00000:
                return y if hy >= 0 else 0.0
            return -y if hy < 0 else 0.0
        if iy == 0x3ff00000:
            return (1.0 / x if x != 0 else math.copysign(INF, x)) if hy < 0 else x
        if hy == 0x40000000:
            return _mul(x, x)
        if hy == 0x3fe00000 and hx >= 0:
            return math.sqrt(x)
    ax = abs(x)
    if lx == 0 and ix in (0x7ff00000, 0, 0x3ff00000):
        z = ax
        if hy < 0:
            z = 1.0 / z if z != 0 else INF
        if hx < 0:
            if ((ix - 0x3ff00000) | yisint) == 0:
                z = NAN
            elif yisint == 1:
                z = -z
        return z
    n = 0 if hx < 0 else 1
    if (n | yisint) == 0:
        return NAN
    s = 1.0
    if (n | (yisint - 1)) == 0:
        s = -1.0
    if iy > 0x41e00000:
        if iy > 0x43f00000:
            if ix <= 0x3fefffff:
                return INF if hy < 0 else 0.0
            if ix >= 0x3ff00000:
                return INF if hy > 0 else 0.0
        if ix < 0x3fefffff:
            return s * INF if hy < 0 else s * 0.0
        if ix > 0x3ff00000:
            return s * INF if hy > 0 else s * 0.0
        t = ax - 1.0
        w = (t * t) * (0.5 - t * (0.3333333333333333333333 - t * 0.25))
        u = ivln2_h * t
        v = t * ivln2_l - w * ivln2
        t1 = _make(_hi(u + v), 0)
        t2 = v - (t1 - u)
    else:
        n = 0
        if ix < 0x00100000:
            ax *= two53
            n -= 53
            ix = _hi(ax)
        n += (ix >> 20) - 0x3ff
        j = ix & 0x000fffff
        ix = j | 0x3ff00000
        if j <= 0x3988E:
            k = 0
        elif j < 0xBB67A:
            k = 1
        else:
            k = 0
            n += 1
            ix -= 0x00100000
        ax = _make(ix, _lo(ax))
        bp, dp_h, dp_l = (1.5, 5.84962487220764160156e-01, 1.35003920212974897128e-08) if k else (1.0, 0.0, 0.0)
        u = ax - bp
        v = 1.0 / (ax + bp)
        ss = u * v
        s_h = _make(_hi(ss), 0)
        t_h = _make(((ix >> 1) | 0x20000000) + 0x00080000 + (k << 18), 0)
        t_l = ax - (t_h - bp)
        s_l = v * ((u - s_h * t_h) - s_h * t_l)
        s2 = ss * ss
        r = s2 * s2 * (L1 + s2 * (L2 + s2 * (L3 + s2 * (L4 + s2 * (L5 + s2 * L6)))))
        r += s_l * (s_h + ss)
        s2 = s_h * s_h
        t_h = _make(_hi(3.0 + s2 + r), 0)
        t_l = r - ((t_h - 3.0) - s2)
        u = s_h * t_h
        v = s_l * t_h + t_l * ss
        p_h = _make(_hi(u + v), 0)
        p_l = v - (p_h - u)
        z_h = cp_h * p_h
        z_l = cp_l * p_h + p_l * cp + dp_l
        t = float(n)
        t1 = _make(_hi(((z_h + z_l) + dp_h) + t), 0)
        t2 = z_l - (((t1 - t) - dp_h) - z_h)
    y1 = _make(_hi(y), 0)
    p_l = (y - y1) * t1 + y * t2
    p_h = y1 * t1
    z = p_l + p_h
    j, i = _hi(z), _i32(_lo(z))
    if j >= 0x40900000:
        if ((j - 0x40900000) | i) != 0:
            return s * INF
        if p_l + ovt > z - p_h:
            return s * INF
    elif (j & 0x7fffffff) >= 0x4090cc00:
        if (_i32(j - 0xc090cc00) | i) != 0:
            return s * 0.0
        if p_l <= z - p_h:
            return s * 0.0
    i = j & 0x7fffffff
    k = (i >> 20) - 0x3ff
    n = 0
    if i > 0x3fe00000:
        n = _i32(j + (0x00100000 >> (k + 1)))
        k = ((n & 0x7fffffff) >> 20) - 0x3ff
        t = _make(n & ~(0x000fffff >> k), 0)
        n = ((n & 0x000fffff) | 0x00100000) >> (20 - k)
        if j < 0:
            n = -n
        p_h -= t
    t = _make(_hi(p_l + p_h), 0)
    u = t * lg2_h
    v = (p_l - (t - p_h)) * lg2 + t * lg2_l
    z = u + v
    w = v - (z - u)
    t = z * z
    t1 = z - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))))
    r = (z * t1) / (t1 - 2.0) - (w + z * w)
    z = 1.0 - (r - z)
    j = _hi(z) + (n << 20)
    if (j >> 20) <= 0:                          # subnormal output: fdlibm's scalbn(z, n), one rounding
        e = ((_hi(z) & 0x7ff00000) >> 20) + n
        if e <= -54:
            z = math.copysign(0.0, z)
        else:
            z = _make((_hi(z) & 0x800fffff) | ((e + 54) << 20), _lo(z)) * twom54
    else:
        z = _make(j, _lo(z))
    return s * z


LOG_2 = fd_log(2.0)


# ---- Spark's expressions ---------------------------------------------------------------------------------------------

def java_d2l(v, bits=64):
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    if v != v:
        return 0
    if v >= hi:
        return hi
    if v <= lo:
        return lo
    return int(v)


def _wrap(v, bits):
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >= 1 << (bits - 1) else v


def _nearest_float32(q: Fraction) -> float:
    """The float32 nearest to the rational q (ties to even), as a Python float."""
    if q == 0:
        return 0.0
    f = np.float32(float(q))                    # within one float ulp of the answer
    cands = [f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))]
    cands = [c for c in cands if np.isfinite(c)]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c).view(np.uint32)) & 1))
    return float(best)


def round_half_up(x, n, is_float32=False):
    """BigDecimal(Double.toString(x)).setScale(n, HALF_UP).doubleValue() (floatValue() for a float column)."""
    if not math.isfinite(x):
        return x
    d = decimal.Decimal(repr(float(x)))
    with decimal.localcontext() as ctx:
        ctx.prec = 1000
        q = d.quantize(decimal.Decimal(1).scaleb(-n), rounding=decimal.ROUND_HALF_UP)
    if q == 0:
        return 0.0
    if is_float32:
        return _nearest_float32(Fraction(q))
    return float(q)


def round_integer(x, n, bits):
    if n >= 0:
        return x
    p = 10 ** (-n)
    q, r = divmod(abs(x), p)
    m = (q + (1 if 2 * r >= p else 0)) * p
    return _wrap(-m if x < 0 else m, bits)


def _factorial_arg(x, in_dtype):
    if in_dtype == I32:
        return int(x)
    if in_dtype == I64:
        return _wrap(int(x), 32)
    return java_d2l(float(x), 32)


def value(op, x, in_dtype, out_dtype, n=0, a=0.0):
    """op(x) of one non-null row -> (value in the output type as a Python number, is it non-null)."""
    is_int = in_dtype in (I32, I64)
    v = float(x)
    if op in (LN, LOG10, LOG2):
        if v <= 0:
            return 0.0, False
        return (fd_log(v) if op == LN else fd_log10(v) if op == LOG10 else fd_log(v) / LOG_2), True
    if op == EXP:
        return fd_exp(v), True
    if op == POW_BASE:
        return fd_pow(a, v), True
    if op == POW:
        return fd_pow(v, a), True
    if op == SQRT:
        return (NAN if v < 0 else math.sqrt(v)), True
    if op in MATH_OPS:
        f = {CBRT: np.cbrt, SIN: np.sin, COS: np.cos, TAN: np.tan, ASIN: np.arcsin, ACOS: np.arccos, ATAN: np.arctan}[op]
        with np.errstate(all="ignore"):
            return float(f(np.float64(v))), True
    if op == RADIANS:
        return v * 0.017453292519943295, True
    if op == MUL_INV:
        if v == 0:
            return 0.0, False
        return 1.0 / v, True
    if op in (FLOOR, CEIL):
        if is_int:
            return int(x), True
        if not math.isfinite(v):
            return java_d2l(v), True
        return java_d2l(float(math.floor(v) if op == FLOOR else math.ceil(v))), True
    if op == FACTORIAL:
        k = _factorial_arg(x, in_dtype)
        return (math.factorial(k), True) if 0 <= k <= 20 else (0, False)
    if op == REMAINDER:
        if out_dtype in (F32, F64):
            with np.errstate(all="ignore"):
                return float(np.fmod(np.float64(v), np.float64(a))), True
        q = int(x)
        return (abs(q) % abs(n)) * (1 if q >= 0 else -1), True        # Java's %: the sign of the dividend
    # ROUND
    if is_int:
        return round_integer(int(x), n, 32 if in_dtype == I32 else 64), True
    return round_half_up(v, n, in_dtype == F32), True


def transform_reference(vals, valid, in_dtype, spec):
    """One column of anv_transform_columns: spec = (op, out dtype, n, a) -> (output ndarray with null rows 0, bool keep)."""
    op, od, n, a = spec
    out = np.zeros(len(vals), NP_OF[od])
    keep = np.zeros(len(vals), bool)
    for r, (x, ok) in enumerate(zip(vals.tolist(), np.asarray(valid, bool).tolist())):
        if not ok:
            continue
        y, k = value(op, x, in_dtype, od, n, a)
        keep[r] = k
        if k:
            with np.errstate(over="ignore"):
                out[r] = NP_OF[od](y) if od in (F32, F64) else y
    return out, keep


# ---- Box-Cox lambda search ---------------------------------------------------------------------------------------------

BOXCOX_LAMBDAS = (1, -1, 0.5, -0.5, 2, -2, 0.25, -0.25, 3, -3, 4, -4, 5, -5)


def std_normal_cdf(x):
    """NormalDistribution(0, 1).cumulativeProbability."""
    if abs(x) > 40:
        return 0.0 if x < 0 else 1.0
    return 0.5 * math.erfc(-x / 1.4142135623730951)


def ks_statistic(sample):
    """max over the sorted sample of max(Phi(y_i) - (i-1)/n, i/n - Phi(y_i)), by a plain sort."""
    y = sorted(sample)
    n = len(y)
    return max(max(std_normal_cdf(v) - i / n, (i + 1) / n - std_normal_cdf(v)) for i, v in enumerate(y))


def boxcox_statistics(values, valid):
    """The statistic of each candidate (BOXCOX_LAMBDAS, then log), with null rows entering as 0."""
    xs = [float(v) for v in values]
    out = []
    for lam in list(BOXCOX_LAMBDAS) + [None]:
        sample = [(fd_log(x) if lam is None else fd_pow(x, float(lam))) if ok else 0.0 for x, ok in zip(xs, valid)]
        out.append(ks_statistic(sample))
    return out


def boxcox_lambdas(columns, p_value):
    """The reference's selection loop over columns [(values, valid)], with p_value(D, n); carry-over included."""
    out, best = [], None
    for values, valid in columns:
        best_p = 0
        for lam, d in zip(list(BOXCOX_LAMBDAS) + [0], boxcox_statistics(values, valid)):
            p = p_value(d, len(values))
            if p > best_p:
                best_p, best = p, lam
        if best is None:
            raise UnboundLocalError("best_lambdaVal")
        out.append(best)
    return out
