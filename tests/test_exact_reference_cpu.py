"""The exact references of the kernel-edge tests (oracle/exact.py) against independent computations, on CPU."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import exact as X
from oracle import spark_semantics as S


def _direct(values):
    """Central moments straight from the definition, every value a Fraction."""
    xs = [Fraction(v) for v in values]
    n = len(xs)
    mean = sum(xs) / n
    return (n, mean, sum((v - mean) ** 2 for v in xs), sum((v - mean) ** 3 for v in xs),
            sum((v - mean) ** 4 for v in xs))


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64])
def test_exact_moments_equal_the_definition(dtype):
    rng = np.random.default_rng(3)
    if np.dtype(dtype).kind == "f":
        x = np.concatenate([rng.normal(1e5, 1.0, 20), [0.0, -0.0, 2.0 ** -140, -3e-300, 1e30, 0.1, -7.25]]).astype(dtype)
        if dtype == np.float32:
            x = x[np.isfinite(x)]
    else:
        info = np.iinfo(dtype)
        x = np.concatenate([rng.integers(-50, 50, 25), [info.min, info.max, 0, 1, -1]]).astype(dtype)
    assert X.exact_central(x) == _direct(x.tolist())
    n, mean, m2, m3, m4 = _direct(x.tolist())
    assert X.exact_moments(x) == (n, float(mean), float(m2), float(m3), float(m4))


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int64])
def test_exact_moments_agree_with_the_two_pass_reference_on_benign_data(dtype):
    rng = np.random.default_rng(11)
    x = rng.normal(3.0, 2.0, 5000)
    x = x.astype(dtype) if np.dtype(dtype).kind == "f" else np.round(x * 1000).astype(dtype)
    n, mean, m2, m3, m4 = X.exact_moments(x)
    en, emean, em2, em3, em4 = S.central_moments(x.astype(np.float64))
    assert n == en
    assert abs(mean - emean) <= 1e-14 * abs(emean)
    sd = math.sqrt(m2 / n)
    for k, (g, e) in enumerate(((m2, em2), (m3, em3), (m4, em4))):
        assert abs(g - e) <= 1e-12 * abs(e) + 1e-12 * n * sd ** (k + 2), (k + 2, g, e)


def test_exact_moments_of_a_constant_and_an_empty_column():
    assert X.exact_central(np.full(7, 1e12)) == (7, Fraction(10 ** 12), 0, 0, 0)
    assert X.exact_moments(np.zeros(0, np.float32))[:2] == (0, None)
    assert X.exact_moments(np.array([-0.0, 0.0])) == (2, 0.0, 0.0, 0.0, 0.0)


def test_exact_bins_compare_ints_exactly():
    cut = [float(2 ** 53), 2.0 ** 62]
    v = np.array([2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 62 - 1, 2 ** 62, 2 ** 62 + 1, -2 ** 63], np.int64)
    valid = np.ones(v.size, bool)
    assert X.exact_bins(v, valid, cut).tolist() == [1, 1, 2, 2, 2, 3, 1]
    # the oracle's assign_bins compares integer columns exactly too (float64(2^53 + 1) rounds to the cutoff)
    assert S.assign_bins(v, valid, cut, 3).tolist() == [1, 1, 2, 2, 2, 3, 1]
    assert S.assign_bins(v, valid, [-math.inf, 1e300, math.inf], 4).tolist() == [2] * v.size
    assert S.assign_bins(v, valid, [-1e300, 0.5], 3).tolist() == [3, 3, 3, 3, 3, 3, 2]
    f = np.array([np.nan, -np.inf, 1.0, np.nextafter(1.0, 2.0), np.inf, -0.0], np.float64)
    valid = np.array([1, 1, 1, 1, 1, 0], bool)
    assert X.exact_bins(f, valid, [0.0, 1.0]).tolist() == [3, 1, 2, 3, 3, 0]
    assert S.assign_bins(f, valid, [0.0, 1.0], 3).tolist() == [3, 1, 2, 3, 3, 0]
