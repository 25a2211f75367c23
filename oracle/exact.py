"""Exact references for the kernel tests: moments and bin ids computed without rounding, rounded once at the end.

Every float32 / float64 / integer value is m * 2^e exactly, so a column scaled by 2^-E (E = the smallest exponent in it)
is a list of Python ints.  Its power sums S1..S4 are then exact integers, and n, the mean and M2..M4 follow as
`fractions.Fraction`s that are rounded to float64 once.  This is the yardstick for the 1e-6 contract of the moments
kernels on inputs where a float64 two-pass reference (`spark_semantics.central_moments`) would itself lose digits."""
import bisect
import math
from fractions import Fraction

import numpy as np


def _scaled_ints(x: np.ndarray):
    """Finite values -> (list of Python ints N_i, E) with x_i == N_i * 2^E exactly."""
    x = np.asarray(x)
    if x.dtype.kind in "iu":
        return [int(v) for v in x.tolist()], 0
    x = x.astype(np.float64)                  # exact for float32
    mant, ex = np.frexp(x)                    # x = mant * 2^ex, 0.5 <= |mant| < 1
    m = (mant * 2.0 ** 53).astype(np.int64)   # exact: |mant| * 2^53 < 2^53 and carries the 53 significant bits
    e = ex.astype(np.int64) - 53
    nz = m != 0
    if not nz.any():
        return [0] * x.size, 0
    E = int(e[nz].min())
    return [int(mi) << (int(ei) - E) if mi else 0 for mi, ei in zip(m.tolist(), e.tolist())], E


def exact_central(x: np.ndarray):
    """Finite non-null values -> (n, mean, M2, M3, M4) as Fractions, M_k = sum (x - mean)^k; (0, None, 0, 0, 0) if empty."""
    N, E = _scaled_ints(x)
    n = len(N)
    if n == 0:
        return 0, None, Fraction(0), Fraction(0), Fraction(0)
    s1 = s2 = s3 = s4 = 0
    for v in N:
        v2 = v * v
        s1 += v
        s2 += v2
        s3 += v2 * v
        s4 += v2 * v2
    a = Fraction(s1, n)                       # mean, in units of 2^E
    m2 = s2 - a * s1
    m3 = s3 - 3 * a * s2 + 2 * a * a * s1
    m4 = s4 - 4 * a * s3 + 6 * a * a * s2 - 3 * a * a * a * s1
    sc = Fraction(2) ** E
    return n, a * sc, m2 * sc ** 2, m3 * sc ** 3, m4 * sc ** 4


def exact_moments(x: np.ndarray):
    """exact_central rounded once to float64: (n, mean, M2, M3, M4); mean None when empty."""
    n, mean, m2, m3, m4 = exact_central(x)
    return n, (None if mean is None else float(mean)), float(m2), float(m3), float(m4)


def exact_bins(values: np.ndarray, valid: np.ndarray, cutoffs) -> np.ndarray:
    """bucket_label's bin id with Python's exact int / float comparisons: 1 + #(c < v), NaN -> len(cutoffs) + 1,
    null -> 0.  Evaluated once per distinct value; the cutoffs must not hold NaN."""
    values = np.asarray(values)
    cut = sorted(float(c) for c in cutoffs)
    as_py = int if values.dtype.kind in "iu" else float
    u, inv = np.unique(values, return_inverse=True)
    ids_u = np.empty(u.size, np.int32)
    for j, v in enumerate(u.tolist()):
        v = as_py(v)
        # bisect_left counts the cutoffs c < v with Python's own (exact) int / float comparison
        ids_u[j] = len(cut) + 1 if (isinstance(v, float) and math.isnan(v)) else 1 + bisect.bisect_left(cut, v)
    out = ids_u[inv.reshape(-1)]
    out[~np.asarray(valid, bool)] = 0
    return out
