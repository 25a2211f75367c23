"""bigint outlier thresholds and mode strings, without a GPU.

The reference flags an outlier of a bigint column after rounding the value to double (`v.astype(float)`, then
`v - lower < 0` / `v - upper > 0`); the product compares the int64 itself against exact integer thresholds.  Both must
flag the same rows for every value and every double bound, including where doubles are 1 024 apart and at the ends of the
int64 range."""
import decimal
import math

import numpy as np
import pyarrow as pa
import pytest

from anovos_b200 import engine
from anovos_b200.data_analyzer import quality_checker as qc
from anovos_b200.data_analyzer.stats_generator import _mode_str
from anovos_b200.frame import ColumnFrame
from oracle import spark_semantics as S

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
CENTERS = [1 << 53, 1 << 54, 1 << 62, 1_600_000_000_000_000_000, I64_MAX]


def _values():
    out = set()
    for c in CENTERS:
        for s in (1, -1):
            out.update(v for v in range(s * c - 600, s * c + 601) if I64_MIN <= v <= I64_MAX)
    return np.array(sorted(out), dtype=np.int64)


def _bounds():
    out = {math.inf, -math.inf, 1e19, -1e19, 2.0 ** 63, -2.0 ** 63, 2.0 ** 64, -2.0 ** 64, 0.5, -0.5}
    for c in CENTERS:
        for s in (1, -1):
            x, top = float(s * c - 600), float(s * c + 600)
            while x <= top:
                out.add(x)
                x = math.nextafter(x, math.inf)
    out.update([math.nextafter(2.0 ** 63, -math.inf), math.nextafter(-2.0 ** 63, -math.inf)])
    return sorted(out)


VALUES, BOUNDS = _values(), _bounds()


def _ref(lo, hi):
    """-1 / 0 / +1 per value: the reference's compare through double (NaN bounds flag nothing)."""
    f = VALUES.astype(np.float64)
    with np.errstate(invalid="ignore"):
        low = (f - lo) < 0 if lo is not None else np.zeros(f.size, bool)
        up = (f - hi) > 0 if hi is not None else np.zeros(f.size, bool)
    return up.astype(np.int64) - low.astype(np.int64)


def _product(lo, hi, side):
    """The flags the binning kernels give for the product's exact thresholds: bin 1 + #(thresholds < v), then the flag
    of that bin."""
    cuts, flags, ths = qc._outlier_thresholds_i64([lo, hi], side)
    assert len(cuts) == len(ths) == len(flags) - 1 and ths == sorted(ths)
    assert all(I64_MIN <= t <= I64_MAX for t in ths)
    bins = np.searchsorted(np.array(ths, dtype=np.int64), VALUES, side="left")
    return np.array(flags, dtype=np.int64)[bins]


def test_windows_cover_the_interesting_spacings():
    assert len(BOUNDS) > 2000 and VALUES.size > 10_000
    assert I64_MIN in VALUES and I64_MAX in VALUES
    # doubles are 1 024 apart near 2^63: many values share a double, so an exact compare would differ
    assert np.unique(VALUES.astype(np.float64)).size < VALUES.size // 2


def test_i64_at_most_is_the_largest_int_whose_double_is_not_above():
    f = VALUES.astype(np.float64)
    for c in BOUNDS + [math.nan]:
        t = engine.i64_at_most(c)
        assert np.array_equal(VALUES <= t, f <= c), c
        if I64_MIN <= t < I64_MAX:
            assert float(t) <= c and not float(t + 1) <= c, c      # float(int) rounds like astype(float64)
    assert engine.i64_at_most(math.nan) == engine.i64_at_most(-math.inf) == I64_MIN - 1
    assert engine.i64_at_most(math.inf) == engine.i64_at_most(2.0 ** 63) == I64_MAX
    assert engine.i64_at_most(2.0 ** 53) == 2 ** 53 + 1                  # 2^53 + 1 is a tie and rounds to even: 2^53


@pytest.mark.parametrize("side", ["upper", "lower"])
def test_one_sided_flags_match_the_reference_compare(side):
    for c in BOUNDS + [math.nan]:
        lo, hi = (c, None) if side == "lower" else (None, c)
        assert np.array_equal(_product(lo, hi, side), _ref(lo, hi)), (side, c)


def test_two_sided_flags_match_the_reference_compare():
    """Both bounds, crossed ones included: a value between crossed bounds is flagged by both sides (-1 + 1 = 0)."""
    rng = np.random.default_rng(1)
    b = np.array(BOUNDS)
    pairs = [(b[i], b[j]) for i, j in rng.integers(0, b.size, (1500, 2))]
    pairs += [(-math.inf, -math.inf), (math.inf, -math.inf), (-2.0 ** 64, -2.0 ** 64), (2.0 ** 64, -2.0 ** 64),
              (math.nan, 2.0 ** 53), (2.0 ** 53 + 2, math.nan), (2.0 ** 53 + 2, 2.0 ** 53)]
    for lo, hi in pairs:
        assert np.array_equal(_product(lo, hi, "both"), _ref(lo, hi)), (lo, hi)


def test_counterexamples_next_to_2_to_the_53():
    """upper = 2^53, v = 2^53 + 1: double(v) = 2^53 is not above it.  lower = 2^53 + 2, v = 2^53 + 1: double(v) = 2^53
    is below it."""
    v = 2 ** 53 + 1
    _, flags, ths = qc._outlier_thresholds_i64([None, 2.0 ** 53], "upper")
    assert flags[int(np.searchsorted(ths, v))] == 0
    _, flags, ths = qc._outlier_thresholds_i64([2.0 ** 53 + 2, None], "lower")
    assert flags[int(np.searchsorted(ths, v))] == -1


def test_bin_model_takes_exact_int64_thresholds():
    t = pa.table({"x": pa.array([1, 2], pa.int64()), "f": pa.array([1.0, 2.0])})
    fr = ColumnFrame.from_arrow(t)
    m = engine.BinModel(fr, ["x"], [[float(2 ** 53 + 1)]], exact=[[2 ** 53 + 1]])
    assert m.cuts_host.view(np.int64).tolist() == [2 ** 53 + 1]
    assert engine.BinModel(fr, ["x"], [[float(I64_MAX)]], exact=[[I64_MAX]]).cuts_host.view(np.int64).tolist() == [I64_MAX]
    with pytest.raises(OverflowError):
        engine.BinModel(fr, ["x"], [[0.0]], exact=[[I64_MAX + 1]])
    with pytest.raises(ValueError):
        engine.BinModel(fr, ["f"], [[0.0]], exact=[[0]])


@pytest.mark.parametrize("v", [I64_MIN, I64_MIN + 1, -(2 ** 53) - 1, -1, 0, 2 ** 53 + 1, 1_600_000_000_000_000_001,
                               I64_MAX - 1, I64_MAX])
def test_bigint_mode_strings_are_exact(v):
    col = ColumnFrame.from_arrow(pa.table({"x": pa.array([v], pa.int64())})).column("x")
    assert _mode_str(col, v) == str(v) == S.mode_to_string(np.int64(v), "bigint")
    assert _mode_str(col, np.int64(v)) == str(v)
    if float(v) != v:                             # the digits a float has already lost cannot come back
        assert _mode_str(col, float(v)) != str(v)


def test_mode_computation_host_path_keeps_bigint_modes_exact():
    """mode_computation / measures_of_centralTendency through the NumPy stand-in of the kernels: the mode of a bigint
    column is an exact int from the engine to the result table."""
    import warnings
    import cpu_engine
    import anovos.data_analyzer.stats_generator as sg
    from oracle import api as O
    rng = np.random.default_rng(4)
    n = 5000
    cols = {"ext": rng.choice(np.array([I64_MIN, I64_MAX, I64_MAX - 1], np.int64), n, p=[0.3, 0.4, 0.3]),
            "ts": 1_600_000_000_000_000_000 + np.where(rng.random(n) < 0.2, 1, rng.integers(0, 1 << 20, n))}
    t = pa.table({k: pa.array(v, mask=rng.random(n) < 0.05) for k, v in cols.items()})
    with cpu_engine.installed(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = sg.mode_computation(None, t).toPandas()
        ct = sg.measures_of_centralTendency(None, t).toPandas()
    exp = O.mode_computation(t)
    assert got.values.tolist() == exp.values.tolist()
    assert got["mode"].tolist() == [str(I64_MAX), "1600000000000000001"]
    assert ct["mode"].tolist() == exp["mode"].tolist()


@pytest.mark.parametrize("x", [6.376e37, -1.7976931348623157e308, 2.0 ** 126 + 2.0 ** 73, 1e24 + 0.5e9, 123456789.00005])
def test_spark_round_of_values_with_more_digits_than_a_default_decimal_context(x):
    """round(x, 4) of the variance of a bigint column (~1e37): Spark's BigDecimal keeps every digit, so the value comes
    back unchanged; a 28-digit decimal context cannot even quantize it."""
    from anovos_b200.shared.utils import spark_round, spark_round_array
    exp = float(decimal.Decimal(repr(x)).quantize(decimal.Decimal("0.0001"), rounding=decimal.ROUND_HALF_UP,
                                                  context=decimal.Context(prec=400)))
    assert spark_round(x) == exp == S.round_half_up(x)
    assert spark_round_array(np.array([x]))[0] == exp
    if abs(x) >= 1e20:
        assert exp == x
