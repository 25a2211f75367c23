"""The one-sample Kolmogorov-Smirnov p-value Spark reports (mllib Statistics.kolmogorovSmirnovTest): 1 - cdf(D, n) with
commons-math 3's KolmogorovSmirnovTest.cdf(d, n, exact=False), restated in Python doubles:
  d <= 1/2n -> 0;  d <= 1/n -> n! (2d - 1/n)^n;  d >= 1 - 1/n -> 1 - 2 (1 - d)^n;  d >= 1 -> 1;
  otherwise Durbin's matrix H^n (roundedK) for n <= 140 and the Pelz-Good series above.
commons-math evaluates exp / sqrt / pow with FastMath; here they are Python's, so a p-value at rounding-noise level (a D
near 1) can differ in its last bits."""
from __future__ import annotations

import math

import numpy as np

PG_SUM_RELATIVE_ERROR = 1.0e-10
MAXIMUM_PARTIAL_SUM_COUNT = 100000
PI_SQUARED = math.pi * math.pi


def _rounded_h(d, n):
    k = int(math.ceil(n * d))
    m = 2 * k - 1
    h = k - n * d
    if h >= 1:
        raise ArithmeticError("could not convert %r to a fraction" % h)
    H = np.zeros((m, m))
    for i in range(m):
        for j in range(m):
            H[i, j] = 1.0 if i - j + 1 >= 0 else 0.0
    hp = [h ** (i + 1) for i in range(m)]
    for i in range(m):
        H[i, 0] -= hp[i]
        H[m - 1, i] -= hp[m - i - 1]
    if 2 * h - 1 > 0:
        H[m - 1, 0] += (2 * h - 1) ** m
    for i in range(m):
        for j in range(i + 1):
            if i - j + 1 > 0:
                for g in range(2, i - j + 2):
                    H[i, j] /= g
    return H, k


def _rounded_k(d, n):
    H, k = _rounded_h(d, n)
    p = np.linalg.matrix_power(H, n)[k - 1, k - 1]
    for i in range(1, n + 1):
        p *= i / n
    return float(p)


def _sum(term, k0):
    s, k = 0.0, k0
    while k < MAXIMUM_PARTIAL_SUM_COUNT:
        inc = term(k)
        s += inc
        if abs(inc) < PG_SUM_RELATIVE_ERROR * abs(s):
            return s
        k += 1
    raise RuntimeError("Pelz-Good series did not converge")


def _pelz_good(d, n):
    sqrt_n = math.sqrt(n)
    z = d * sqrt_n
    z2 = d * d * n
    z4, z6, z8 = z2 * z2, z2 * z2 * z2, z2 * z2 * z2 * z2
    z2term = PI_SQUARED / (8 * z2)
    s, k = 0.0, 1
    while k < MAXIMUM_PARTIAL_SUM_COUNT:                 # K_0(z)
        kt = 2 * k - 1
        inc = math.exp(-z2term * kt * kt)
        s += inc
        if inc <= PG_SUM_RELATIVE_ERROR * s:
            break
        k += 1
    ret = s * math.sqrt(2 * math.pi) / z
    two_z2 = 2 * z2
    s = _sum(lambda k: (PI_SQUARED * (k + 0.5) ** 2 - z2) * math.exp(-PI_SQUARED * (k + 0.5) ** 2 / two_z2), 0)
    sqrt_half_pi = math.sqrt(math.pi / 2)
    ret += s * sqrt_half_pi / (3 * z4 * sqrt_n)         # K_1(z)
    z4t, z6t, z2t = 2 * z4, 6 * z6, 5 * z2
    pi4 = PI_SQUARED * PI_SQUARED

    def k2(k):
        kt2 = (k + 0.5) ** 2
        return (z6t + z4t + PI_SQUARED * (z4t - z2t) * kt2 + pi4 * (1 - two_z2) * kt2 * kt2) * \
            math.exp(-PI_SQUARED * kt2 / two_z2)
    s = _sum(k2, 0)
    s2 = _sum(lambda k: PI_SQUARED * k * k * math.exp(-PI_SQUARED * k * k / two_z2), 1)
    ret += (sqrt_half_pi / n) * (s / (36 * z2 * z2 * z2 * z) - s2 / (18 * z2 * z))   # K_2(z)
    pi6 = pi4 * PI_SQUARED

    def k3(k):
        kt2 = (k + 0.5) ** 2
        kt4, kt6 = kt2 * kt2, kt2 * kt2 * kt2
        return (pi6 * kt6 * (5 - 30 * z2) + pi4 * kt4 * (-60 * z2 + 212 * z4) + PI_SQUARED * kt2 * (135 * z4 - 96 * z6)
                - 30 * z6 - 90 * z8) * math.exp(-PI_SQUARED * kt2 / two_z2)
    s = _sum(k3, 0)
    s2 = _sum(lambda k: (-pi4 * k ** 4 + 3 * PI_SQUARED * k * k * z2) * math.exp(-PI_SQUARED * k * k / two_z2), 1)
    return ret + (sqrt_half_pi / (sqrt_n * n)) * (s / (3240 * z6 * z4) + s2 / (108 * z6))   # K_3(z)


def cdf(d, n):
    """P(D_n < d), commons-math's KolmogorovSmirnovTest.cdf(d, n, false)."""
    ninv = 1 / float(n)
    ninvhalf = 0.5 * ninv
    if d <= ninvhalf:
        return 0.0
    if d <= ninv:
        res, f = 1.0, 2 * d - ninv
        for i in range(1, n + 1):
            res *= i * f
        return res
    if 1 - ninv <= d < 1:
        return 1 - 2 * (1 - d) ** n
    if d >= 1:
        return 1.0
    if n <= 140:
        return _rounded_k(d, n)
    return _pelz_good(d, n)


def p_value(d, n):
    """Spark's pValue of the one-sample test with statistic d over n values."""
    return 1 - cdf(d, n)
