"""GPU tests of the scan, select and sort kernels where they take shortcuts, against exact references.

* moments: tiles without a finite non-null value in their first 1024 rows (no early pivot), far from zero, constant, NaN /
  inf prefixes, an outlier as the pivot, all-NaN / only-inf / subnormal columns, a ragged scalar tail with nulls -
  against `oracle.exact` (power sums in Python ints, rounded once);
* binning: values on every threshold, one ulp either side, at the 8-ulp width limit of the guess path and on both sides
  of its fold limit, int64 beyond 2^53 - against 1 + #(c < v) with Python's exact int / float comparison;
* order statistics, mode, distinct and HLL++ registers on special values: NaNs with the sign bit set and other payloads,
  -0.0, subnormals, +-FLT_MAX / DBL_MAX, INT_MIN / LLONG_MIN / LLONG_MAX - against NumPy.
Every input is built from a seed."""
import math

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu

from oracle import exact as X

BLOCK = 16384   # tiles are multiples of this many rows
PREFIX = 1024   # the pivot is looked for in a tile's first 1024 rows


def _frame(cols):
    from anovos_b200.frame import ColumnFrame
    t = pa.table({k: pa.array(v, mask=m) for k, (v, m) in cols.items()})
    return t, ColumnFrame.from_arrow(t)


def _nan32(bits):
    return np.array(bits, np.uint32).view(np.float32)


def _nan64(bits):
    return np.array(bits, np.uint64).view(np.float64)


NAN32 = _nan32([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF, 0x7FC00123])   # canonical, 0 * inf on x86, payloads
NAN64 = _nan64([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF])


def _prefix_rows(n):
    """Rows [k * 16384, k * 16384 + 1024) of every 16384-row block: whatever tile size is picked, no tile has an early pivot."""
    return (np.arange(n) % BLOCK) < PREFIX


# ---- moments -------------------------------------------------------------------------------------

def _expected_minmax(x):
    """min / max skip NaN; a column of nothing but NaN has NaN extrema (as its order statistics)."""
    f = x[~np.isnan(x)] if x.dtype.kind == "f" else x
    if f.size == 0:
        return math.nan, math.nan
    return float(f.min()), float(f.max())


def _check_moments(rec, vals, valid, name):
    x = vals[valid]
    n = int(x.size)
    assert rec["n_valid"] == n, name                                           # counts bit-exact
    assert rec["n_nonzero"] == int(np.count_nonzero(x != 0)), name                  # NaN counts as nonzero
    if n == 0:
        assert math.isnan(rec["min"]) and math.isnan(rec["max"]), name
        return
    mn, mx = _expected_minmax(x)
    assert rec["min"] == mn or (math.isnan(mn) and math.isnan(rec["min"])), (name, rec["min"], mn)   # extrema exact
    assert rec["max"] == mx or (math.isnan(mx) and math.isnan(rec["max"])), (name, rec["max"], mx)
    if x.dtype.kind == "f" and not np.isfinite(x).all():
        for f in ("mean", "m2", "m3", "m4"):                                   # a NaN / inf value makes every moment non-finite
            assert not math.isfinite(rec[f]), (name, f, rec[f])
        return
    en, mean, m2, m3, m4 = X.exact_moments(x)
    sd = math.sqrt(m2 / n)
    # + n * 2^-1074: a merge step scales (mean_b - mean_a) / n, rounded to the subnormal spacing, by up to n rows
    assert abs(rec["mean"] - mean) <= 1e-9 * max(abs(mean), sd) + n * 2.0 ** -1074, (name, rec["mean"], mean)
    if m2 == 0.0 and np.all(x == x[0]):                                        # constant column: exactly zero
        assert rec["m2"] == 0.0 and rec["m3"] == 0.0 and rec["m4"] == 0.0, (name, rec["m2"], rec["m3"], rec["m4"])
        return
    for k, (g, e) in enumerate(((rec["m2"], m2), (rec["m3"], m3), (rec["m4"], m4))):
        tol = 1e-6 * abs(e) + 1e-9 * n * sd ** (k + 2)                         # the 1e-6 contract
        assert abs(g - e) <= tol, (name, "M%d" % (k + 2), g, e)


def _all_moment_paths(t, fr, names, monkeypatch):
    """(label, moment records) of every K1 entry point: anv_moments, anv_moments_hist with either staging, and a
    row-partitioned frame whose chunks start on 16384-row boundaries."""
    from anovos_b200 import engine
    from anovos_b200.partitioned import PartitionedFrame
    out = [("moments", engine.moments(fr, names))]
    cuts, lohi = [], []
    for i in range(len(names)):
        mn, mx = float(out[0][1]["min"][i]), float(out[0][1]["max"][i])
        ok = math.isfinite(mn) and math.isfinite(mx) and mx > mn
        cuts.append([0.0] if not ok else [mn + (mx - mn) * j / 10 for j in range(1, 10)])
        lohi.append((mn, mx) if ok else None)
    model = engine.BinModel(fr, names, cuts, lohi)
    for flag in ("0", "1"):
        monkeypatch.setenv("ANV_FUSED_STAGED", flag)
        m, h = engine.moments_histogram(fr, model)
        for i, c in enumerate(names):                                          # the histogram next to the repaired moments
            exp = np.bincount(X.exact_bins(*_col_values(t, c), cuts[i]), minlength=len(cuts[i]) + 2)
            assert np.array_equal(h[i, :len(cuts[i]) + 2], exp.astype(np.uint64)), (c, flag)
        out.append(("moments_hist staged=" + flag, m))
    monkeypatch.delenv("ANV_FUSED_STAGED")
    out.append(("partitioned", engine.moments(PartitionedFrame.from_frame(fr, 2 * BLOCK), names)))
    return out


def _col_values(t, c):
    from oracle import spark_semantics as S
    return S.column_values(t, c)


def _far_columns(n, rng, prefix, null_rate):
    """Columns far from zero relative to their spread (and controls) behind a prefix of nulls / NaN / +-inf."""
    pre = _prefix_rows(n)
    base = {
        "f32_far": rng.normal(1e5, 1.0, n).astype(np.float32),
        "f64_far": rng.normal(1e6, 1e-2, n),
        "i64_far": (2 ** 30 + rng.integers(-10, 11, n)).astype(np.int64),
        "i32_far": (10 ** 9 + rng.integers(-10, 11, n)).astype(np.int32),
        "f32_const": np.full(n, 1e6, np.float32),
        "f64_const": np.full(n, 1e12),
        "f32_zero_mean": rng.normal(0.0, 1.0, n).astype(np.float32),
    }
    cols = {}
    for k, v in base.items():
        m = rng.random(n) < null_rate if null_rate else np.zeros(n, bool)
        m[pre] = False
        if prefix == "null":
            m = m | pre
        elif v.dtype.kind == "f":
            v = v.copy()
            v[pre] = {"nan": np.nan, "inf": np.inf, "-inf": -np.inf}[prefix]
        else:
            m = m | pre                                                        # integers have no NaN: a null prefix
        cols[k] = (v, m if m.any() else None)
    return cols


@pytest.mark.parametrize("prefix,null_rate", [("null", 0.05), ("null", 0.0), ("nan", 0.0), ("nan", 0.05),
                                              ("inf", 0.05), ("-inf", 0.0)])
def test_moments_of_tiles_without_an_early_pivot(prefix, null_rate, monkeypatch):
    rng = np.random.default_rng(17 + int(null_rate * 100))
    n = 5 * BLOCK + 4099
    t, fr = _frame(_far_columns(n, rng, prefix, null_rate))
    names = t.column_names
    for label, m in _all_moment_paths(t, fr, names, monkeypatch):
        for i, c in enumerate(names):
            vals, valid = _col_values(t, c)
            _check_moments(m[i], vals, valid, (label, c))


@pytest.mark.xfail(strict=True, reason="tile and partition moments are merged through float64 means: with |mean| / sigma "
                   "above ~1e8 the rounding of the means alone moves M3 beyond 1e-9 n sigma^3")
def test_odd_moment_of_columns_1e11_sigma_from_zero():
    rng = np.random.default_rng(41)
    n = 5 * BLOCK + 4099
    t, fr = _frame({"f64": (rng.normal(1e9, 1e-3, n), None), "i64": ((2 ** 40 + rng.integers(-10, 11, n)).astype(np.int64), None)})
    from anovos_b200 import engine
    m = engine.moments(fr, t.column_names)
    for i, c in enumerate(t.column_names):
        _check_moments(m[i], *_col_values(t, c), c)


def _isnull(v):
    return v is None or (isinstance(v, float) and math.isnan(v))


def test_constant_column_behind_nulls_has_zero_spread_in_the_stats_tables():
    """stddev 0, skewness and kurtosis null - the same as for the column without the null prefix."""
    import anovos.data_analyzer.stats_generator as sg
    n = 3 * BLOCK + 100
    v = np.full(n, 1e12)
    t = pa.table({"prefixed": pa.array(v, mask=_prefix_rows(n)), "plain": pa.array(v)})
    from anovos_b200.frame import ColumnFrame
    fr = ColumnFrame.from_arrow(t)
    d = sg.measures_of_dispersion(None, fr).toPandas().set_index("attribute")
    s = sg.measures_of_shape(None, fr).toPandas().set_index("attribute")
    for c in ("prefixed", "plain"):
        assert d.loc[c, "stddev"] == 0.0 and d.loc[c, "variance"] == 0.0, c
        assert _isnull(s.loc[c, "skewness"]) and _isnull(s.loc[c, "kurtosis"]), c


def test_moments_with_an_outlier_pivot(monkeypatch):
    """Every tile starts with an outlier 10^6 sigma away: the pivot is that element, and the conditioning of the power
    sums stays bounded by the tile length."""
    rng = np.random.default_rng(23)
    n = 4 * BLOCK + 333
    first = (np.arange(n) % BLOCK) == 0
    f32 = rng.normal(0.0, 1.0, n).astype(np.float32)
    f32[first] = 1e6
    f64 = rng.normal(100.0, 1.0, n)
    f64[first] = 100.0 - 1e6
    i64 = rng.integers(-3, 4, n).astype(np.int64)
    i64[first] = 3 * 10 ** 6
    m = rng.random(n) < 0.05
    m[first] = False
    t, fr = _frame({"f32": (f32, None), "f64": (f64, None), "i64": (i64, None), "f32_nulls": (f32, m), "f64_nulls": (f64, m)})
    names = t.column_names
    for label, mom in _all_moment_paths(t, fr, names, monkeypatch):
        for i, c in enumerate(names):
            vals, valid = _col_values(t, c)
            _check_moments(mom[i], vals, valid, (label, c))


def test_moments_of_special_columns(monkeypatch):
    """All-NaN with and without nulls, only +-inf, only +inf, subnormals only, NaN among numbers, and a row count that
    is no multiple of the vector width with nulls in the scalar tail."""
    rng = np.random.default_rng(29)
    n = 3 * BLOCK + 4003                      # 4003 = 4 * 1000 + 3: three f32 rows (one f64 row) in the scalar tail
    tail = np.zeros(n, bool)
    tail[-3:] = [True, False, True]
    some = rng.random(n) < 0.1
    mixed = rng.normal(5.0, 2.0, n).astype(np.float32)
    mixed[rng.random(n) < 0.01] = NAN32[1]
    cols = {
        "f32_all_nan": (rng.choice(NAN32, n), None),
        "f32_all_nan_nulls": (rng.choice(NAN32, n), some | tail),
        "f64_all_nan": (rng.choice(NAN64, n), None),
        "f64_all_nan_nulls": (rng.choice(NAN64, n), some),
        "f32_pm_inf": (np.where(rng.random(n) < 0.5, np.inf, -np.inf).astype(np.float32), some),
        "f64_pos_inf": (np.full(n, np.inf), None),
        "f32_subnormal": (((rng.integers(1, 2 ** 23, n) * np.where(rng.random(n) < 0.3, -1, 1)).astype(np.float64)
                           * 2.0 ** -149).astype(np.float32), tail),
        "f64_subnormal": (rng.integers(1, 2 ** 40, n).astype(np.float64) * 2.0 ** -1074, some),
        "f32_nan_among_numbers": (mixed, some),
        # the first chunk of the row-partitioned frame (2 * BLOCK rows) is all NaN: it must not change min / max
        "f64_nan_first_chunk": (np.where(np.arange(n) < 2 * BLOCK, np.nan, rng.normal(2.0, 1.0, n)), some),
        "f32_tail_nulls": (rng.normal(-3.0, 0.5, n).astype(np.float32), tail),
        "f64_tail_nulls": (rng.normal(7.0, 0.5, n), tail),
        "i32_extremes": (rng.choice(np.array([-2 ** 31, 2 ** 31 - 1, 0, -1], np.int32), n), tail),
        "i64_extremes": (rng.choice(np.array([-2 ** 63, 2 ** 63 - 1, 0, 2 ** 53 + 1], np.int64), n), some),
    }
    assert np.all(np.abs(cols["f32_subnormal"][0]) < np.finfo(np.float32).tiny)
    t, fr = _frame(cols)
    names = t.column_names
    for label, m in _all_moment_paths(t, fr, names, monkeypatch):
        for i, c in enumerate(names):
            vals, valid = _col_values(t, c)
            _check_moments(m[i], vals, valid, (label, c))
        # pinned: NaN among numbers is skipped by min / max (Spark would rank NaN largest; DESIGN.md section 1)
        j = names.index("f32_nan_among_numbers")
        x = mixed[~some].astype(np.float64)
        assert m["max"][j] == np.nanmax(x) and m["min"][j] == np.nanmin(x) and math.isnan(m["mean"][j]), label


# ---- binning ------------------------------------------------------------------------------------

_NP = {"f32": np.float32, "f64": np.float64, "i32": np.int32, "i64": np.int64}


def _catalogue(dt, cuts, lo, hi):
    """Every threshold theta_j as the kernel holds it, one step either side, the float64 cutoffs themselves, lo / hi
    and one step outside, and the special values of the type."""
    T = _NP[dt]
    from anovos_b200 import _lib, engine
    anv = {"f32": _lib.ANV_F32, "f64": _lib.ANV_F64, "i32": _lib.ANV_I32, "i64": _lib.ANV_I64}[dt]
    raw = engine.native_thresholds(cuts, anv)
    if dt == "f32":
        th = raw.astype(np.uint32).view(np.float32)
        pts = [th, np.nextafter(th, np.float32(np.inf)), np.nextafter(th, np.float32(-np.inf)),
               np.array(cuts, np.float64).astype(np.float32)]
        lh = np.array([lo, hi], np.float32)
        pts += [lh, np.nextafter(lh, np.float32(np.inf)), np.nextafter(lh, np.float32(-np.inf))]
        f = np.finfo(np.float32)
        pts += [np.array([1e30, -1e30, f.max, -f.max, np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-40, f.tiny], np.float32),
                NAN32]
        return np.concatenate(pts).astype(np.float32)
    if dt == "f64":
        th = raw.view(np.float64)
        lh = np.array([lo, hi], np.float64)
        f = np.finfo(np.float64)
        pts = [th, np.nextafter(th, np.inf), np.nextafter(th, -np.inf), lh, np.nextafter(lh, np.inf), np.nextafter(lh, -np.inf),
               np.array([1e30, -1e30, f.max, -f.max, np.inf, -np.inf, 0.0, -0.0, 5e-324, -5e-324, 1e-310, f.tiny]), NAN64]
        return np.concatenate(pts)
    info = np.iinfo(T)
    th = raw.view(np.int64).astype(np.int64) if dt == "i64" else raw.astype(np.uint32).view(np.int32).astype(np.int64)
    vals = set()
    for v in th.tolist() + [math.floor(lo) if math.isfinite(lo) else 0, math.ceil(hi) if math.isfinite(hi) else 0]:
        vals.update((v - 1, v, v + 1))
    vals.update((info.min, info.min + 1, info.max - 1, info.max, 0, -1, 1))
    return np.array(sorted(v for v in vals if info.min <= v <= info.max), dtype=T)


def _tile(cat, n, rng, lo, hi, dt):
    """The catalogue spread over n rows (some rows uniform over three times the model's range: a target frame that
    exceeds its source model's range, as drift sees), with 5 % nulls."""
    v = cat[rng.integers(0, cat.size, n)]
    span = hi - lo
    u = rng.uniform(lo - span, hi + span, n)
    with np.errstate(all="ignore"):                  # beyond the type's range: +-inf, or the clipped integer extremes
        if np.dtype(_NP[dt]).kind == "i":
            info = np.iinfo(_NP[dt])
            u = np.clip(np.floor(u), float(info.min), float(np.nextafter(float(info.max), 0.0)))
        u = u.astype(_NP[dt])
    v = np.where(rng.random(n) < 0.2, u, v).astype(_NP[dt])
    return v, rng.random(n) < 0.05


# the last one is a negative range.  A float32 column binned over [-3e38, 3e38] cannot run the guess (hi - lo overflows
# float32), an integer column gets the widest range its type holds (cutoffs below its minimum: see the xfail test below)
RANGES = [(0.0, 1.0), (-1.0, 1.0), (-3e38, 3e38), (-1000.0, -3.0)]
INT_WIDE = {"i32": (-2.0 ** 31, 2.0 ** 31 - 1), "i64": (-2.0 ** 63, 2.0 ** 63 - 4096)}


def _binning_models(B, rng, n):
    from oracle import spark_semantics as S
    cols, cuts, lohi, expect_mode = {}, [], [], []
    def add(name, dt, lo, hi, mode=None):
        cut = S.equal_range_cutoffs(lo, hi, B)
        cat = _catalogue(dt, cut, lo, hi)
        cols[name] = _tile(cat, n, rng, lo, hi, dt)
        cuts.append(cut)
        lohi.append((lo, hi))
        expect_mode.append(mode)
    for dt in ("f32", "f64", "i32", "i64"):
        for r, (lo, hi) in enumerate(RANGES):
            if dt in INT_WIDE and r == 2:
                lo, hi = INT_WIDE[dt]
            add("%s_r%d" % (dt, r), dt, lo, hi, 0 if dt in INT_WIDE or (dt == "f32" and r == 2) else 1)
    # width at the host's 8-ulp limit of the guess path (ulp of max(|lo|, |hi|) = ulp of 1.0)
    add("f32_w8ulp", "f32", 1.0, 1.0 + B * 8 * 2.0 ** -23, 1)
    add("f32_w8ulp_minus", "f32", 1.0, 1.0 + B * 8 * 2.0 ** -23 - 2.0 ** -23, 0)
    add("f64_w8ulp", "f64", 1.0, 1.0 + B * 8 * 2.0 ** -52, 1)
    add("f64_w8ulp_minus", "f64", 1.0, 1.0 + B * 8 * 2.0 ** -52 - 2.0 ** -52, 0)
    # lo on either side of fold_ok's limit 2 (B - 1) + |lo| / w <= 2^18 (w = 1)
    lim = 2 ** 18 - 2 * (B - 1)
    add("f32_fold_in", "f32", float(lim), float(lim + B), 1)
    add("f32_fold_out", "f32", float(lim + 1), float(lim + 1 + B), 1)
    add("f32_fold_in_neg", "f32", -float(lim), -float(lim) + B, 1)
    return cols, cuts, lohi, expect_mode


@pytest.mark.parametrize("B", [2, 3, 10, 39, 40, 300])
def test_binning_on_and_around_every_threshold(B, monkeypatch):
    from anovos_b200 import engine
    rng = np.random.default_rng(1000 + B)
    n = 300_003
    cols, cuts, lohi, expect_mode = _binning_models(B, rng, n)
    t, fr = _frame(cols)
    names = t.column_names
    model = engine.BinModel(fr, names, cuts, lohi)
    for i, c in enumerate(names):
        assert model.specs_host["mode"][i] == expect_mode[i], (c, B)
    sp = model.specs_host
    fold = {c: 2.0 * (sp["n_bins"][i] - 1) + abs(sp["lo"][i]) * sp["inv_w"][i] <= 2 ** 18 for i, c in enumerate(names)}
    assert fold["f32_fold_in"] and fold["f32_fold_in_neg"] and not fold["f32_fold_out"]
    exp = [X.exact_bins(*_col_values(t, c), cuts[i]) for i, c in enumerate(names)]
    counts = [np.bincount(e, minlength=B + 1).astype(np.uint64) for e in exp]
    ids = engine.bin_assign(fr, model).cpu().numpy()
    h = engine.histogram(fr, model)
    got = {"hist": h}
    for flag in ("0", "1"):
        monkeypatch.setenv("ANV_FUSED_STAGED", flag)
        got["moments_hist staged=" + flag] = engine.moments_histogram(fr, model)[1]
    for i, c in enumerate(names):
        bad = np.flatnonzero(ids[i] != exp[i])
        assert bad.size == 0, (c, B, [(cols[c][0][j], int(ids[i][j]), int(exp[i][j])) for j in bad[:5]])
        for label, hh in got.items():
            assert np.array_equal(hh[i, :B + 1], counts[i]), (c, B, label)


def test_bin_assign_with_4096_bins():
    from anovos_b200 import engine
    rng = np.random.default_rng(4096)
    n = 300_001
    cols, cuts, lohi = {}, [], []
    from oracle import spark_semantics as S
    for dt, (lo, hi) in (("f32", (0.0, 1.0)), ("f64", (-1.0, 1.0)), ("f32", (-3e38, 3e38)), ("f64", (-3e38, 3e38)),
                         ("i64", (-5000.0, 5000.0)), ("i32", INT_WIDE["i32"])):
        cut = S.equal_range_cutoffs(lo, hi, 4096)
        cols["%s_%d" % (dt, len(cols))] = _tile(_catalogue(dt, cut, lo, hi), n, rng, lo, hi, dt)
        cuts.append(cut)
        lohi.append((lo, hi))
    t, fr = _frame(cols)
    model = engine.BinModel(fr, t.column_names, cuts, lohi)
    ids = engine.bin_assign(fr, model).cpu().numpy()
    for i, c in enumerate(t.column_names):
        assert np.array_equal(ids[i], X.exact_bins(*_col_values(t, c), cuts[i])), c


@pytest.mark.xfail(strict=True, reason="the kernels compare in the column's type: a cutoff below INT_MIN / LLONG_MIN becomes a "
                   "threshold at the minimum, so a value equal to the minimum lands one bin low")
def test_integer_cutoffs_below_the_type_minimum():
    from anovos_b200 import engine
    v = np.array([-2 ** 31, -2 ** 31 + 1, 0, 2 ** 31 - 1] * 8, np.int32)
    t, fr = _frame({"i32": (v, None), "i64": (v.astype(np.int64) * 2 ** 32, None)})
    cuts = [[-1e38, 0.5], [-1e38, 0.5]]
    ids = engine.bin_assign(fr, engine.BinModel(fr, t.column_names, cuts, None)).cpu().numpy()
    for i, c in enumerate(t.column_names):
        assert np.array_equal(ids[i], X.exact_bins(*_col_values(t, c), cuts[i])), c


def test_int64_binning_beyond_2_to_the_53(monkeypatch):
    """float64(v) rounds above 2^53; v <= c must be decided on the integer."""
    from anovos_b200 import engine
    rng = np.random.default_rng(53)
    n = 300_007
    p53, p62 = 2 ** 53, 2 ** 62
    cuts = [-2.0 ** 63, -float(p62) - 2048, -float(p62), -float(p62) + 1024, float(p53), float(p53 + 2), float(p53 + 4),
            float(p62) - 1024, float(p62), 2.0 ** 63]
    around = [-2 ** 63, -2 ** 63 + 1, 2 ** 63 - 1, 0]
    for c in (-p62 - 2048, -p62, -p62 + 1024, p53, p53 + 2, p53 + 4, p62 - 1024, p62):
        around += [c + d for d in (-1025, -1024, -513, -2, -1, 0, 1, 2, 513, 1023, 1024)]
    cat = np.array(sorted(set(v for v in around if -2 ** 63 <= v < 2 ** 63)), dtype=np.int64)
    v = cat[rng.integers(0, cat.size, n)]
    t, fr = _frame({"i64": (v, rng.random(n) < 0.05), "i64_dense": (v, None)})
    names = t.column_names
    model = engine.BinModel(fr, names, [cuts, cuts], None)
    exp = [X.exact_bins(*_col_values(t, c), cuts) for c in names]
    # python's int / float comparison and the float64 one differ on these rows: the test would catch a float64 compare
    vals, valid = _col_values(t, "i64")
    f64 = 1 + np.searchsorted(np.array(cuts), vals.astype(np.float64), side="left")
    assert np.any(f64[valid] != exp[0][valid])
    ids = engine.bin_assign(fr, model).cpu().numpy()
    h = engine.histogram(fr, model)
    monkeypatch.setenv("ANV_FUSED_STAGED", "1")
    _, h2 = engine.moments_histogram(fr, model)
    for i, c in enumerate(names):
        assert np.array_equal(ids[i], exp[i]), c
        cnt = np.bincount(exp[i], minlength=len(cuts) + 2).astype(np.uint64)
        assert np.array_equal(h[i, :len(cuts) + 2], cnt) and np.array_equal(h2[i, :len(cuts) + 2], cnt), c


# ---- order statistics, mode, distinct, HLL++ ------------------------------------------------------

def _special_columns(n, rng):
    f = np.finfo(np.float32)
    d = np.finfo(np.float64)
    f32 = np.concatenate([NAN32, np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, f.tiny, f.max, -f.max, np.inf, -np.inf, 1.0, -1.0,
                                           3.5, -2.25], np.float32)])
    f64 = np.concatenate([NAN64, np.array([0.0, -0.0, 5e-324, -5e-324, 1e-310, d.tiny, d.max, -d.max, np.inf, -np.inf,
                                           1.0, -1.0, 1e300, -7.5])])
    i32 = np.array([-2 ** 31, -2 ** 31 + 1, 2 ** 31 - 1, 2 ** 31 - 2, 0, -1, 1], np.int32)
    i64 = np.array([-2 ** 63, -2 ** 63 + 1, 2 ** 63 - 1, 2 ** 63 - 2, 0, -1, 1, 2 ** 53 + 1, 2 ** 53], np.int64)

    def draw(cat, null_rate, spread=None):
        v = cat[rng.integers(0, cat.size, n)]
        if spread is not None:                      # many distinct ordinary values around the specials
            pick = rng.random(n) < 0.5
            v = np.where(pick, spread, v).astype(cat.dtype)
        return v, (rng.random(n) < null_rate) if null_rate else None
    return {
        "f32_special": draw(f32, 0.1),
        "f32_special_spread": draw(f32, 0.0, rng.normal(0, 1e3, n).astype(np.float32)),
        "f32_nan_heavy": draw(np.concatenate([NAN32] * 20 + [f32]), 0.02),
        "i32_extremes": draw(i32, 0.1),
        "i32_extremes_spread": draw(i32, 0.0, rng.integers(-2 ** 31, 2 ** 31 - 1, n).astype(np.int32)),
        "f64_special": draw(f64, 0.1),
        "f64_special_spread": draw(f64, 0.0, rng.normal(0, 1e6, n)),
        "i64_extremes": draw(i64, 0.05),
        "i64_extremes_spread": draw(i64, 0.0, rng.integers(-2 ** 63, 2 ** 63 - 1, n)),
    }


def _sorted_reference(vals, valid):
    x = vals[valid]
    return np.sort(x.astype(np.float64) if x.dtype.kind == "f" else x)   # NaN last; ints sorted exactly


def _ranks(n_valid):
    """16 ranks (the n_ranks limit of one selection): 1, n and ranks in between."""
    if n_valid == 0:
        return [0] * 16
    r = [1, n_valid, 2, n_valid - 1] + [max(1, int(n_valid * q)) for q in (0.01, 0.05, 0.1, 0.25, 0.4, 0.5, 0.6, 0.75, 0.9, 0.95, 0.99, 0.999)]
    return [min(max(1, v), n_valid) for v in r]


def _same_float(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.array_equal(a, b, equal_nan=True)        # -0.0 == 0.0, NaN == NaN


@pytest.mark.parametrize("frame_kind", ["32bit", "mixed"])
def test_select_ranks_on_special_values(frame_kind):
    from anovos_b200 import engine
    rng = np.random.default_rng(61)
    n = 250_007
    cols = _special_columns(n, rng)
    if frame_kind == "32bit":
        cols = {k: v for k, v in cols.items() if k.startswith(("f32", "i32"))}
    t, fr = _frame(cols)
    names = t.column_names
    rk, exp = [], []
    for c in names:
        vals, valid = _col_values(t, c)
        srt = _sorted_reference(vals, valid)
        r = _ranks(srt.size)
        rk.append(r)
        exp.append([float(srt[k - 1]) if k else np.nan for k in r])
    got = engine.select_ranks(fr, names, np.array(rk))
    for i, c in enumerate(names):
        assert _same_float(got[i], exp[i]), (c, got[i], exp[i])


@pytest.fixture(params=["lsd", "lsd-onesweep", "partition"])
def sort_algo(request, monkeypatch):
    from anovos_b200 import engine
    if request.param == "lsd-onesweep":
        monkeypatch.setenv("ANV_SORT_ONESWEEP", "1")
    else:
        monkeypatch.delenv("ANV_SORT_ONESWEEP", raising=False)
    old, engine.sort_algorithm = engine.sort_algorithm, request.param.split("-")[0]
    yield request.param
    engine.sort_algorithm = old


def test_exact_mode_distinct_on_special_values(sort_algo):
    """Order statistics, mode and distinct count with all NaNs one value and -0.0 == 0.0.  The mode of an int64 column is
    an exact int: 2^63 - 1 and 2^53 + 1 must not come back as the doubles they round to."""
    from anovos_b200 import engine
    rng = np.random.default_rng(67)
    n = 200_003
    t, fr = _frame(_special_columns(n, rng))
    names = t.column_names
    rk = [_ranks(int((~np.asarray(t.column(c).is_null())).sum())) for c in names]
    got, qv = engine.sort_mode_distinct(fr, names, np.array(rk))
    for i, c in enumerate(names):
        vals, valid = _col_values(t, c)
        srt = _sorted_reference(vals, valid)
        assert _same_float(qv[i], [float(srt[k - 1]) for k in rk[i]]), (c, qv[i])
        x = vals[valid]
        if x.dtype.kind == "f":
            x = x.astype(np.float64) + 0.0                    # -0.0 -> 0.0
            x[np.isnan(x)] = np.nan                           # every payload -> one NaN
        u, k = np.unique(x, return_counts=True)
        assert got[i][2] == u.size, (c, got[i], u.size)
        assert got[i][1] == int(k.max()), (c, got[i])
        best = u[k == k.max()]
        mode = best[0].item()                                 # smallest value among ties, NaN ranked last; int64: exact
        assert type(got[i][0]) is (int if x.dtype == np.int64 else float), (c, got[i])
        assert got[i][0] == mode or (math.isnan(got[i][0]) and math.isnan(mode)), (c, got[i], mode)


def test_hll_registers_on_special_values():
    """The registers hashed from the sorted runs, the stand-alone HLL++ kernel and the oracle's XXH64 agree on NaN
    payloads, -0.0, subnormals and integer extremes."""
    from anovos_b200 import engine
    from oracle import spark_semantics as S
    rng = np.random.default_rng(71)
    n = 150_001
    t, fr = _frame(_special_columns(n, rng))
    names = t.column_names
    for p in (9, 12):
        _, _, regs = engine.sort_mode_distinct(fr, names, None, hll_p=p)
        direct = engine.hll_registers(fr, names, p)
        for i, c in enumerate(names):
            vals, valid = _col_values(t, c)
            ref = S.hll_registers(S.hll_hashes(vals[valid], S.spark_dtype(t.schema.field(c).type)), p)
            assert np.array_equal(direct[i], ref), (c, p)
            assert np.array_equal(regs[i], ref), (c, p)
