"""CUDA implementation of `anovos.data_analyzer.stats_generator` (reference
/root/reference/src/main/anovos/data_analyzer/stats_generator.py:33-1011): same function
names, arguments, output columns, rounding and error behaviour; `spark` is accepted and
ignored (it may be None), `idf` is anything `anovos_b200.frame.as_frame` accepts.  All
per-row work runs in the CUDA kernels of libanovos_b200.so; this module only normalises
arguments and post-processes one small row per attribute on the host.
"""
from __future__ import annotations

import math
import warnings

import numpy as np
import pandas as pd

from .. import profile
from ..frame import as_frame
from ..result import ResultFrame
from ..shared.utils import attributeType_segregation, jvm_double_str, names, spark_round, spark_round_array, unique

_R = spark_round


def _empty(cols):
    return ResultFrame(pd.DataFrame({c: pd.Series([], dtype=object) for c in cols}))


def _opt(a):
    """float64 column of a result frame, NaN = null: what pandas infers from a row-wise list holding None (the dtype the
    frames have always had; `pd.isna` is the null test either way)."""
    return np.asarray(a, dtype=np.float64)


def _show(odf, n, print_impact):
    if print_impact:
        odf.show(max(n, 1))
    return odf


def _disp(col, v):
    """summary() prints FloatType min/max/percentiles with Float.toString and Anovos casts the
    string back to double (stats_generator.py:818-822,910-912); other dtypes are unchanged."""
    if v is None:
        return None
    if col.sdtype == "float":
        return float(str(np.float32(v)))
    return float(v)


def _disp_array(col, values):
    """_disp over a list of floats / None -> float64 array (None -> NaN)."""
    a = np.array([np.nan if v is None else v for v in values], dtype=np.float64)
    if col.sdtype == "float":
        ok = np.isfinite(a)
        if ok.any():
            a[ok] = a[ok].astype(np.float32).astype("U32").astype(np.float64)   # Float.toString round trip
    return a


_F32_EPS = 2.0 ** -23


def _f32_trip(a):
    """Float.toString round trip of float32-representable doubles (vectorised; slow: ~1 us per value)."""
    return a.astype(np.float32).astype("U32").astype(np.float64)


def _near_tie(x, unc):
    """Could changing x by at most `unc` change round(x, 4)?"""
    with np.errstate(invalid="ignore", over="ignore"):
        t = x * 10000.0
        return ~(np.abs((t - np.floor(t)) - 0.5) > unc * 10000.0 + 1e-6) & np.isfinite(x)


def _disp_matrix(fr, cols, vals):
    """_disp over a [n_cols, k] float64 matrix (NaN = null) whose entries are about to be ROUNDED to 4 decimals: the rows
    of FloatType columns take the Float.toString round trip, which moves a value by less than half a float32 ulp - so
    only the entries that sit within that distance of a rounding tie are actually converted."""
    rows = [i for i, c in enumerate(cols) if fr.column(c).sdtype == "float"]
    if rows:
        sub = vals[rows]
        need = _near_tie(sub, np.abs(sub) * _F32_EPS)
        if need.any():
            sub[need] = _f32_trip(sub[need])
            vals[rows] = sub
    return vals


def _disp_diff(fr, cols, hi, lo):
    """round-ready `_disp(hi) - _disp(lo)` per column (IQR, range) with the same shortcut."""
    d = hi - lo
    rows = np.array([fr.column(c).sdtype == "float" for c in cols], dtype=bool)
    need = rows & _near_tie(d, (np.abs(hi) + np.abs(lo)) * _F32_EPS)
    if need.any():
        d[need] = _f32_trip(hi[need]) - _f32_trip(lo[need])
    return d


def global_summary(spark, idf, list_of_cols="all", drop_cols=[], print_impact=False):
    """reference :33-113 - every value is a string."""
    fr = as_frame(idf)
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = fr.columns
    cols = unique(names(list_of_cols), names(drop_cols))
    if any(c not in fr.columns for c in cols) or not cols:
        raise TypeError("Invalid input for Column(s)")
    num, cat, other = attributeType_segregation(fr.select(cols))
    if print_impact:
        print("No. of Rows: %s" % "{0:,}".format(fr.count()))
        print("No. of Columns: %s" % "{0:,}".format(len(cols)))
        print("Numerical Columns: %s" % "{0:,}".format(len(num)))
        if num:
            print(num)
        print("Categorical Columns: %s" % "{0:,}".format(len(cat)))
        if cat:
            print(cat)
        if other:
            print("Other Columns: %s" % "{0:,}".format(len(other)))
            print(other)
    rows = [["rows_count", str(fr.count())], ["columns_count", str(len(cols))],
            ["numcols_count", str(len(num))], ["numcols_name", ", ".join(num)],
            ["catcols_count", str(len(cat))], ["catcols_name", ", ".join(cat)],
            ["othercols_count", str(len(other))], ["othercols_name", ", ".join(other)]]
    return ResultFrame(pd.DataFrame(rows, columns=["metric", "value"]))


def _discrete_cols(fr, list_of_cols, drop_cols, allow_empty=False):
    """The "all -> num + cat" normalisation idiom (reference :150-161 and its copies)."""
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        num, cat, _ = attributeType_segregation(fr)
        list_of_cols = num + cat
    cols = unique(names(list_of_cols), names(drop_cols))
    if any(c not in fr for c in cols) or (not cols and not allow_empty):
        raise TypeError("Invalid input for Column(s)")
    bad = [c for c in cols if fr.column(c).kind == "other"]
    if bad:
        raise TypeError("Invalid input for Column(s): dtype of %s is not numerical/categorical" % bad)
    return cols


def _numeric_cols(fr, list_of_cols, drop_cols):
    """The "all -> num" idiom of the numeric-only functions (reference :217-224, :784-795 ...)."""
    num = attributeType_segregation(fr)[0]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num
    cols = unique(names(list_of_cols), names(drop_cols))
    numset = set(num)
    if any(c not in numset for c in cols):
        raise TypeError("Invalid input for Column(s)")
    return cols


def missingCount_computation(spark, idf, list_of_cols="all", drop_cols=[], print_impact=False):
    """reference :116-176: missing_count = N - count(col); missing_pct = round(missing/N, 4)."""
    fr = as_frame(idf)
    cols = _discrete_cols(fr, list_of_cols, drop_cols)
    N = fr.count()
    nv = profile.n_valid(fr, cols)
    rows = [[c, N - nv[c], _R((N - nv[c]) / N) if N else None] for c in cols]
    return _show(ResultFrame(pd.DataFrame(rows, columns=["attribute", "missing_count", "missing_pct"])),
                 len(cols), print_impact)


def nonzeroCount_computation(spark, idf, list_of_cols="all", drop_cols=[], print_impact=False):
    """reference :179-248 (MLlib colStats.numNonzeros after fillna(0)); pct over ALL rows."""
    fr = as_frame(idf)
    cols = _numeric_cols(fr, list_of_cols, drop_cols)
    if not cols:
        warnings.warn("No Non-Zero Count Computation - No numerical column(s) to analyze")
        return _empty(["attribute", "nonzero_count", "nonzero_pct"])
    N = fr.count()
    m = profile.moments(fr, cols)
    rows = [[c, int(m[c]["n_nonzero"]), _R(int(m[c]["n_nonzero"]) / N) if N else None] for c in cols]   # x / 0: null
    return _show(ResultFrame(pd.DataFrame(rows, columns=["attribute", "nonzero_count", "nonzero_pct"])),
                 len(cols), print_impact)


def measures_of_counts(spark, idf, list_of_cols="all", drop_cols=[], print_impact=False):
    """reference :251-325.  missing_pct = round(1 - round(fill/N, 4), 4) (quirk kept, :313-319)."""
    fr = as_frame(idf)
    cols = _discrete_cols(fr, list_of_cols, drop_cols)
    N = fr.count()
    is_num = np.array([fr.column(c).kind == "num" for c in cols], dtype=bool)
    m = profile.moments(fr, [c for c, k in zip(cols, is_num) if k])
    nv = profile.n_valid(fr, cols)       # string columns: from the code histogram when a pass already left one
    fill = np.array([nv[c] for c in cols], dtype=np.int64)
    nz = np.array([int(m[c]["n_nonzero"]) if k else 0 for c, k in zip(cols, is_num)], dtype=np.int64)
    if N:
        fill_pct = spark_round_array(fill / N)
        miss_pct = spark_round_array(1 - fill_pct)
        nz_pct = spark_round_array(np.where(is_num, nz / N, np.nan))
    else:
        fill_pct = miss_pct = nz_pct = np.full(len(cols), np.nan)
    nz_col = nz if is_num.all() else np.where(is_num, nz.astype(np.float64), np.nan)   # string columns: null
    odf = ResultFrame.from_columns({"attribute": cols, "fill_count": fill, "fill_pct": _opt(fill_pct), "missing_count": N - fill,
                                    "missing_pct": _opt(miss_pct), "nonzero_count": nz_col, "nonzero_pct": _opt(nz_pct)})
    return _show(odf, len(cols), print_impact)


def _mode_str(col, value):
    if value is None:
        return None
    if col.kind == "cat":
        return str(value)
    if col.sdtype in ("int", "bigint", "long"):
        # Long.toString: the engine hands the mode of a bigint column over as an exact int, which int() keeps digit for
        # digit (an int32 mode arrives as a float, which holds it exactly)
        return str(int(value))
    return jvm_double_str(float(value))


def mode_computation(spark, idf, list_of_cols="all", drop_cols=[], print_impact=False):
    """reference :328-421: most frequent non-null value (as string) and its row count."""
    fr = as_frame(idf)
    cols = _discrete_cols(fr, list_of_cols, drop_cols, allow_empty=True)
    if not cols:
        warnings.warn("No Mode Computation - No discrete column(s) to analyze")
        return _empty(["attribute", "mode", "mode_rows"])
    md = profile.mode_distinct(fr, cols)
    rows = [[c, _mode_str(fr.column(c), md[c][0]), md[c][1]] for c in cols if md[c][1] is not None]
    return _show(ResultFrame(pd.DataFrame(rows, columns=["attribute", "mode", "mode_rows"])), len(cols), print_impact)


def measures_of_centralTendency(spark, idf, list_of_cols="all", drop_cols=[], print_impact=False):
    """reference :424-526: mean, median (numeric only), mode, mode_rows, mode_pct."""
    fr = as_frame(idf)
    cols = _discrete_cols(fr, list_of_cols, drop_cols)
    kinds = [fr.column(c) for c in cols]
    num = [c for c, col in zip(cols, kinds) if col.kind == "num"]
    m = profile.moments(fr, num)
    nvd = profile.n_valid(fr, cols)             # string columns: from their code histogram (no second pass over them)
    md = profile.mode_distinct(fr, cols)       # the sort also yields the exact percentiles (cached)
    med = profile.quantiles(fr, num, [0.5])
    k = len(cols)
    nv = np.array([nvd[c] for c in cols], dtype=np.float64)
    mean, median = np.full(k, np.nan), np.full(k, np.nan)
    mode, mode_rows = [None] * k, np.full(k, np.nan)
    for i, (c, col) in enumerate(zip(cols, kinds)):
        if col.kind == "num" and nv[i]:
            mean[i] = m[c]["mean"]
            v = med[c][0]
            median[i] = np.nan if v is None else v
        mo, rows_ = md[c][0], md[c][1]
        mode[i] = _mode_str(col, mo)
        if rows_ is not None:
            mode_rows[i] = rows_
    fl = np.array([col.sdtype == "float" for col in kinds], dtype=bool) & np.isfinite(median)
    if fl.any():
        median[fl] = _f32_trip(median[fl])                      # FloatType: Float.toString round trip (_disp)
    with np.errstate(all="ignore"):
        pct = spark_round_array(np.where(nv > 0, mode_rows / nv, np.nan))
    has_null_rows = np.isnan(mode_rows).any()
    odf = ResultFrame.from_columns({"attribute": cols, "mean": spark_round_array(mean), "median": spark_round_array(median), "mode": mode,
                                    "mode_rows": mode_rows if has_null_rows else mode_rows.astype(np.int64), "mode_pct": pct})
    return _show(odf, len(cols), print_impact)


def _unique_values(fr, cols, approx, rsd):
    """-> dict name -> (unique_values, hll_bias_band_flag)."""
    out = {}
    if approx:
        est = profile.hll(fr, cols, rsd)
        band = [c for c in cols if est[c][1]]
        exact = profile.mode_distinct(fr, band) if band else {}
        for c in cols:
            # HLL++ bias-correction tables are unavailable offline: in that band fall back to the
            # exact distinct count and flag the row (SURVEY 8a item 7, "parity unpinned")
            out[c] = (exact[c][2], True) if c in exact else (est[c][0], False)
    else:
        md = profile.mode_distinct(fr, cols)
        for c in cols:
            out[c] = (md[c][2], False)
    return out


def uniqueCount_computation(spark, idf, list_of_cols="all", drop_cols=[], compute_approx_unique_count=False,
                            rsd=None, print_impact=False):
    """reference :529-620: countDistinct or approx_count_distinct(col, rsd) (HLL++)."""
    fr = as_frame(idf)
    cols = _discrete_cols(fr, list_of_cols, drop_cols, allow_empty=True)
    if rsd is not None and rsd < 0:
        raise ValueError("rsd value can not be less than 0 (default value is 0.05)")
    if not cols:
        warnings.warn("No Unique Count Computation - No discrete column(s) to analyze")
        return _empty(["attribute", "unique_values"])
    u = _unique_values(fr, cols, compute_approx_unique_count, rsd)
    odf = pd.DataFrame([[c, int(u[c][0])] for c in cols], columns=["attribute", "unique_values"])
    return _show(ResultFrame(odf), len(cols), print_impact)


def measures_of_cardinality(spark, idf, list_of_cols="all", drop_cols=[], use_approx_unique_count=True, rsd=None,
                            print_impact=False):
    """reference :623-733: unique_values + IDness = round(unique / (N - missing), 4)."""
    fr = as_frame(idf)
    cols = _discrete_cols(fr, list_of_cols, drop_cols, allow_empty=True)
    if rsd is not None and rsd < 0:
        raise ValueError("rsd value can not be less than 0 (default value is 0.05)")
    if not cols:
        warnings.warn("No Cardinality Computation - No discrete column(s) to analyze")
        return _empty(["attribute", "unique_values", "IDness"])
    u = _unique_values(fr, cols, use_approx_unique_count, rsd)
    nv = profile.n_valid(fr, cols)
    uv = np.array([int(u[c][0]) for c in cols], dtype=np.int64)
    nva = np.array([nv[c] for c in cols], dtype=np.float64)
    with np.errstate(all="ignore"):
        idness = spark_round_array(np.where(nva > 0, uv / nva, np.nan))
    odf = ResultFrame.from_columns({"attribute": cols, "unique_values": uv, "IDness": idness},
                                   attrs={"hll_bias_band": [c for c in cols if u[c][1]]})
    return _show(odf, len(cols), print_impact)


def _stddev(rec):
    n = int(rec["n_valid"])
    if n <= 1:
        return None  # stddev_samp of <= 1 value: null (Spark >= 3.1 default; parity unpinned)
    return math.sqrt(float(rec["m2"]) / (n - 1))


def measures_of_dispersion(spark, idf, list_of_cols="all", drop_cols=[], print_impact=False):
    """reference :736-829.  variance = round(round(stddev,4)^2, 4); cov = round(round(stddev,4)/mean, 4)."""
    fr = as_frame(idf)
    cols = _numeric_cols(fr, list_of_cols, drop_cols)
    if not cols:
        warnings.warn("No Dispersion Computation - No numerical column(s) to analyze")
        return _empty(["attribute", "stddev", "variance", "cov", "IQR", "range"])
    m = profile.moments_table(fr, cols)
    q = profile.quantiles(fr, cols, [0.25, 0.75])
    k = len(cols)
    nv, m2, mean = m["n_valid"], m["m2"], m["mean"]
    raw = np.full((k, 4), np.nan)                     # q25, q75, min, max (display values)
    raw[:, 2], raw[:, 3] = m["min"], m["max"]
    for i, c in enumerate(cols):
        if nv[i]:
            raw[i, 0], raw[i, 1] = q[c]
        else:
            raw[i] = np.nan
    with np.errstate(all="ignore"):
        sd = spark_round_array(np.where(nv > 1, np.sqrt(m2 / np.maximum(nv - 1, 1)), np.nan))   # n <= 1: null (Spark >= 3.1)
        var = spark_round_array(sd * sd)
        cov = spark_round_array(np.where(mean == 0, np.nan, sd / mean))                           # x / 0 is null in Spark SQL
        iqr = spark_round_array(_disp_diff(fr, cols, raw[:, 1].copy(), raw[:, 0].copy()))
        rng = spark_round_array(_disp_diff(fr, cols, raw[:, 3].copy(), raw[:, 2].copy()))
    odf = ResultFrame.from_columns({"attribute": cols, "stddev": sd, "variance": var, "cov": cov, "IQR": iqr, "range": rng})
    return _show(odf, len(cols), print_impact)


_PCT = [("1%", 0.01), ("5%", 0.05), ("10%", 0.1), ("25%", 0.25), ("50%", 0.5), ("75%", 0.75), ("90%", 0.9),
        ("95%", 0.95), ("99%", 0.99)]


def measures_of_percentiles(spark, idf, list_of_cols="all", drop_cols=[], print_impact=False):
    """reference :832-916: min, 1..99 %, max, each round(..., 4); percentile p = element of rank
    ceil(p * n) (exact; Spark's GK sketch is within 1e-4 * n ranks of it)."""
    fr = as_frame(idf)
    cols = _numeric_cols(fr, list_of_cols, drop_cols)
    names = ["attribute", "min"] + [p for p, _ in _PCT] + ["max"]
    if not cols:
        warnings.warn("No Percentiles Computation - No numerical column(s) to analyze")
        return _empty(names)
    m = profile.moments_table(fr, cols)
    q = profile.quantiles(fr, cols, [p for _, p in _PCT])
    vals = np.full((len(cols), 11), np.nan)
    vals[:, 0], vals[:, 10] = m["min"], m["max"]
    nonempty = m["n_valid"] > 0
    for i, c in enumerate(cols):
        if nonempty[i]:
            vals[i, 1:10] = [np.nan if v is None else v for v in q[c]]
        else:
            vals[i] = np.nan
    vals = spark_round_array(_disp_matrix(fr, cols, vals))
    data = {"attribute": cols}
    for j, nme in enumerate(names[1:]):
        data[nme] = vals[:, j]
    return _show(ResultFrame.from_columns(data), len(cols), print_impact)


def measures_of_shape(spark, idf, list_of_cols="all", drop_cols=[], print_impact=False):
    """reference :919-1011: population skewness sqrt(n) M3 / M2^1.5, excess kurtosis n M4 / M2^2 - 3."""
    fr = as_frame(idf)
    cols = _numeric_cols(fr, list_of_cols, drop_cols)
    if not cols:
        warnings.warn("No Skewness/Kurtosis Computation - No numerical column(s) to analyze")
        return _empty(["attribute", "skewness", "kurtosis"])
    m = profile.moments_table(fr, cols)
    n, m2, m3, m4 = m["n_valid"].astype(np.float64), m["m2"], m["m3"], m["m4"]
    with np.errstate(all="ignore"):
        ok = (n > 0) & (m2 != 0)                 # Spark >= 3.1: null when M2 == 0 (parity unpinned)
        skew = spark_round_array(np.where(ok, np.sqrt(n) * m3 / np.sqrt(m2 * m2 * m2), np.nan))
        kurt = spark_round_array(np.where(ok, n * m4 / (m2 * m2) - 3.0, np.nan))
    return _show(ResultFrame.from_columns({"attribute": cols, "skewness": _opt(skew), "kurtosis": _opt(kurt)}), len(cols), print_impact)
