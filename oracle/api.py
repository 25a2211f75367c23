"""Oracle restatement of the reference's Python API for the hot path, on pyarrow
Tables, returning pandas DataFrames with the reference's column names.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Follows (relative to /root/reference/src/main/anovos):
  data_analyzer/stats_generator.py:33-1011
  data_transformer/transformers.py:87-291   (attribute_binning)
  drift_stability/drift_detector.py:16-371  (statistics)
  drift_stability/validations.py:8-94
  shared/utils.py:28-73
"""
from __future__ import annotations

import json
import math
import os
import warnings

import numpy as np
import pandas as pd
import pyarrow as pa

from . import spark_semantics as S

R = S.round_half_up


def with_spark_partitions(table: pa.Table, rows_per_partition) -> pa.Table:
    """Tag a table with the way Spark partitioned it (rows per partition, in order): percentiles then follow the
    per-partition Greenwald-Khanna sketches merged in partition order, like Dataset.summary() / approxQuantile."""
    md = dict(table.schema.metadata or {})
    md[b"spark_partition_rows"] = json.dumps([int(k) for k in rows_per_partition]).encode()
    return table.replace_schema_metadata(md)


def table_from_rows(rows, names) -> pa.Table:
    """spark.createDataFrame(rows, names) analogue used by the ported reference tests:
    python int -> bigint, float -> double, str -> string, None -> null."""
    cols = list(zip(*rows)) if rows else [[] for _ in names]
    arrays = []
    for c in cols:
        non_null = [v for v in c if v is not None]
        if non_null and all(isinstance(v, str) for v in non_null):
            arrays.append(pa.array(list(c), type=pa.string()))
        elif non_null and all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in non_null):
            arrays.append(pa.array(list(c), type=pa.int64()))
        else:
            arrays.append(pa.array(list(c), type=pa.float64()))
    return pa.table(arrays, names=list(names))


# ---------------------------------------------------------------------------
# argument normalisation (stats_generator.py:295-307 idiom)
# ---------------------------------------------------------------------------


def _split(x):
    if isinstance(x, str):
        return [s.strip() for s in x.split("|")]
    return list(x)


def _dedupe(cols, drop):
    drop = set(drop)
    return [c for c in dict.fromkeys(cols) if c not in drop]  # reference: list(set(...)) - order arbitrary, we keep input order


def _resolve(table, list_of_cols, drop_cols, default, universe=None, allow_empty=False):
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = default
    cols = _dedupe(_split(list_of_cols), _split(drop_cols))
    universe = set(table.column_names if universe is None else universe)
    if any(c not in universe for c in cols) or (len(cols) == 0 and not allow_empty):
        raise TypeError("Invalid input for Column(s)")
    return cols


_GK_CACHE = {}


class ColumnProfile:
    """Everything the stats functions need from one column (float64 semantics)."""

    def __init__(self, table, name):
        self.name = name
        self.sdtype = S.spark_dtype(table.schema.field(name).type)
        vals, valid = S.column_values(table, name)
        self.N = len(vals)
        self.valid = valid
        self.values = vals
        self.nn = vals[valid]
        self.n = int(self.nn.size)
        self.is_num = self.sdtype in ("double", "int", "bigint", "float", "long") or self.sdtype.startswith("decimal")
        self._x64 = None
        self._sorted = None
        self._sketch = {}
        md = table.schema.metadata or {}
        self.partition_rows = json.loads(md[b"spark_partition_rows"]) if b"spark_partition_rows" in md else None
        if self.partition_rows is not None and sum(self.partition_rows) != self.N:
            raise ValueError("spark_partition_rows does not add up to the table's rows")

    @property
    def x64(self):
        if self._x64 is None:
            self._x64 = self.nn.astype(np.float64)
        return self._x64

    @property
    def sorted64(self):
        if self._sorted is None:
            self._sorted = np.sort(self.x64, kind="stable")
        return self._sorted

    def _disp(self, v):
        """summary() string round trip for float32 min/max/percentiles."""
        if v is None:
            return None
        if self.sdtype == "float":
            return S.float32_via_string(v)
        return float(v)

    def minmax(self):
        if self.n == 0:
            return None, None
        x = self.x64
        if np.isnan(x).any():  # Spark: NaN is the largest value (unpinned)
            nn = x[~np.isnan(x)]
            return (float(nn.min()) if nn.size else float("nan")), float("nan")
        return float(x.min()), float(x.max())

    def _partition_values(self):
        """Non-null float64 values of each Spark partition (schema metadata `spark_partition_rows`), arrival order."""
        out, r0 = [], 0
        for k in self.partition_rows:
            sel = slice(r0, r0 + k)
            out.append(self.values[sel][self.valid[sel]].astype(np.float64))
            r0 += k
        return out

    def quantile(self, p, eps=S.SUMMARY_EPS):
        """summary() percentile (eps 1e-4) or approxQuantile(..., eps): Spark's sketch position for one partition
        of < 50 000 values, the exact rank otherwise (S.approx_quantile_rank)."""
        if self.n == 0:
            return None
        if self.partition_rows is not None and eps is not None:    # the full sketch: per partition, merged in order
            key = ("parts", eps)
            if key not in self._sketch:
                samples, n = [], 0
                for part in self._partition_values():
                    s_, c_ = S.gk_sketch(part, eps)
                    samples, n = S.gk_merge(samples, n, s_, c_, eps)
                self._sketch[key] = (samples, n)
            samples, n = self._sketch[key]
            return float(S.gk_query_value(samples, n, eps, p))
        key = (self.n, eps)
        if key not in _GK_CACHE:
            _GK_CACHE[key] = S.gk_single_batch_summary(self.n, eps) if (eps is not None and self.n < S.GK_HEAD_SIZE) else None
        sm = _GK_CACHE[key]
        if sm is None:
            return float(S.quantile_sorted(self.sorted64, p))
        return float(self.sorted64[S.gk_query_position(sm, self.n, eps, p)])

    def equal_frequency_cutoffs(self, bin_size):
        """transformers.py:210-215: approxQuantile(cols, [j * (1 / bin_size)], 0.01) - through the same sketch logic as
        every other percentile (one partition / Spark partitions of the table / exact beyond the head buffer)."""
        w = 1 / bin_size
        return [self.quantile(j * w, S.APPROX_QUANTILE_EPS) for j in range(1, bin_size)]

    def nonzero(self):
        if self.n == 0:
            return 0
        return int(np.count_nonzero(self.x64 != 0))

    def mode(self):
        """-> (mode value, rows) over non-null values; ties arbitrary (first in sort
        order here).  stats_generator.py:386-401."""
        if self.n == 0:
            return None, None
        if self.sdtype == "string":
            u, c = np.unique(self.nn.astype(str), return_counts=True)
        else:
            # Spark 3 groups -0.0 with 0.0 under the key 0.0 (NormalizeFloatingNumbers)
            u, c = np.unique(self.nn + 0.0 if self.nn.dtype.kind == "f" else self.nn, return_counts=True)
        i = int(np.argmax(c))
        return u[i], int(c[i])

    def distinct(self):
        if self.n == 0:
            return 0
        if self.sdtype == "string":
            return int(len(set(self.nn.tolist())))
        x = self.nn
        if x.dtype.kind == "f":
            x = x.copy()
            x[x == 0] = 0.0
        return int(np.unique(x).size)


_PROFILE_LRU = []   # [(table, {name: ColumnProfile})], most recent last: pyarrow Tables are immutable, so a profile
_PROFILE_LRU_SIZE = 3  # (values, float64 image, sorted copy) can be shared by the functions called on the same table


def _profiles(table, cols):
    """ColumnProfiles of `cols`, memoised per table OBJECT (the scale tests call ten functions on one 10M-row table:
    one sort per column instead of one per function).  Strong references keep id() stable."""
    for i, (t, d) in enumerate(_PROFILE_LRU):
        if t is table:
            _PROFILE_LRU.append(_PROFILE_LRU.pop(i))
            break
    else:
        d = {}
        _PROFILE_LRU.append((table, d))
        del _PROFILE_LRU[:-_PROFILE_LRU_SIZE]
    for c in cols:
        if c not in d:
            d[c] = ColumnProfile(table, c)
    return {c: d[c] for c in cols}


# ---------------------------------------------------------------------------
# stats_generator
# ---------------------------------------------------------------------------


def global_summary(table, list_of_cols="all", drop_cols=[]):
    """stats_generator.py:33-113."""
    cols = _resolve(table, list_of_cols, drop_cols, table.column_names)
    num, cat, other = S.segregate(table.select(cols))
    rows = [["rows_count", str(table.num_rows)], ["columns_count", str(len(cols))],
            ["numcols_count", str(len(num))], ["numcols_name", ", ".join(num)],
            ["catcols_count", str(len(cat))], ["catcols_name", ", ".join(cat)],
            ["othercols_count", str(len(other))], ["othercols_name", ", ".join(other)]]
    return pd.DataFrame(rows, columns=["metric", "value"])


def missingCount_computation(table, list_of_cols="all", drop_cols=[]):
    """stats_generator.py:116-176."""
    num, cat, _ = S.segregate(table)
    cols = _resolve(table, list_of_cols, drop_cols, num + cat)
    N = table.num_rows
    rows = []
    for c, p in _profiles(table, cols).items():
        miss = N - p.n
        rows.append([c, miss, R(miss / N) if N else None])
    return pd.DataFrame(rows, columns=["attribute", "missing_count", "missing_pct"])


def nonzeroCount_computation(table, list_of_cols="all", drop_cols=[]):
    """stats_generator.py:179-248 (MLlib colStats.numNonzeros after fillna(0))."""
    num = S.segregate(table)[0]
    cols = _resolve(table, list_of_cols, drop_cols, num, universe=num, allow_empty=True)
    if not cols:
        warnings.warn("No Non-Zero Count Computation - No numerical column(s) to analyze")
        return pd.DataFrame(columns=["attribute", "nonzero_count", "nonzero_pct"])
    N = table.num_rows
    rows = []
    for c, p in _profiles(table, cols).items():
        nz = p.nonzero()
        rows.append([c, nz, R(nz / N) if N else None])          # x / 0 is null in Spark SQL
    return pd.DataFrame(rows, columns=["attribute", "nonzero_count", "nonzero_pct"])


def measures_of_counts(table, list_of_cols="all", drop_cols=[]):
    """stats_generator.py:251-325."""
    num, cat, _ = S.segregate(table)
    cols = _resolve(table, list_of_cols, drop_cols, num + cat)
    num_sel = S.segregate(table.select(cols))[0]
    N = table.num_rows
    rows = []
    for c, p in _profiles(table, cols).items():
        fill_pct = R(p.n / N) if N else None
        row = [c, p.n, fill_pct, N - p.n, None if fill_pct is None else R(1 - fill_pct)]       # :313-319
        if c in num_sel:
            nz = p.nonzero()
            row += [nz, R(nz / N) if N else None]
        else:
            row += [None, None]
        rows.append(row)
    return pd.DataFrame(rows, columns=["attribute", "fill_count", "fill_pct", "missing_count",
                                       "missing_pct", "nonzero_count", "nonzero_pct"])


def mode_computation(table, list_of_cols="all", drop_cols=[]):
    """stats_generator.py:328-421."""
    num, cat, _ = S.segregate(table)
    cols = _resolve(table, list_of_cols, drop_cols, num + cat, allow_empty=True)
    if not cols:
        warnings.warn("No Mode Computation - No discrete column(s) to analyze")
        return pd.DataFrame(columns=["attribute", "mode", "mode_rows"])
    rows = []
    for c, p in _profiles(table, cols).items():
        m, r = p.mode()
        if m is None:
            continue  # all-null column: groupBy on empty frame yields no row (:386-401)
        rows.append([c, S.mode_to_string(m, p.sdtype), r])
    return pd.DataFrame(rows, columns=["attribute", "mode", "mode_rows"])


def measures_of_centralTendency(table, list_of_cols="all", drop_cols=[], raw=False):
    """stats_generator.py:424-526.  raw=True skips the round(...,4)."""
    num, cat, _ = S.segregate(table)
    cols = _resolve(table, list_of_cols, drop_cols, num + cat)
    rnd = (lambda v: v) if raw else R
    rows = []
    for c, p in _profiles(table, cols).items():
        mean = median = None
        if c in num and p.n:
            mean = rnd(S.central_moments(p.x64)[1])
            median = rnd(p._disp(p.quantile(0.5)))
        m, r = p.mode()
        rows.append([c, mean, median, None if m is None else S.mode_to_string(m, p.sdtype), r,
                     None if r is None else rnd(r / p.n)])
    return pd.DataFrame(rows, columns=["attribute", "mean", "median", "mode", "mode_rows", "mode_pct"])


def uniqueCount_computation(table, list_of_cols="all", drop_cols=[], compute_approx_unique_count=False,
                            rsd=None, with_flags=False):
    """stats_generator.py:529-620."""
    num, cat, _ = S.segregate(table)
    cols = _resolve(table, list_of_cols, drop_cols, num + cat, allow_empty=True)
    if rsd is not None and rsd < 0:
        raise ValueError("rsd value can not be less than 0 (default value is 0.05)")
    if not cols:
        warnings.warn("No Unique Count Computation - No discrete column(s) to analyze")
        return pd.DataFrame(columns=["attribute", "unique_values"])
    rows = []
    for c, p in _profiles(table, cols).items():
        if compute_approx_unique_count:
            est, band = S.approx_count_distinct(p.nn, p.sdtype, rsd)
            if band:  # HLL++ bias-correction band: tables unavailable offline -> exact distinct,
                est = p.distinct()  # row flagged "HLL bias band, parity unpinned" (SURVEY 8a item 7)
            rows.append([c, est, band])
        else:
            rows.append([c, p.distinct(), False])
    df = pd.DataFrame(rows, columns=["attribute", "unique_values", "hll_bias_band"])
    return df if with_flags else df[["attribute", "unique_values"]]


def measures_of_cardinality(table, list_of_cols="all", drop_cols=[], use_approx_unique_count=True, rsd=None,
                            with_flags=False):
    """stats_generator.py:623-733."""
    num, cat, _ = S.segregate(table)
    cols = _resolve(table, list_of_cols, drop_cols, num + cat, allow_empty=True)
    if rsd is not None and rsd < 0:
        raise ValueError("rsd value can not be less than 0 (default value is 0.05)")
    if not cols:
        warnings.warn("No Cardinality Computation - No discrete column(s) to analyze")
        return pd.DataFrame(columns=["attribute", "unique_values", "IDness"])
    u = uniqueCount_computation(table, cols, compute_approx_unique_count=use_approx_unique_count, rsd=rsd,
                                with_flags=True)
    N = table.num_rows
    profs = _profiles(table, cols)
    idn = []
    for c, uv in zip(u["attribute"], u["unique_values"]):
        denom = N - (N - profs[c].n)
        idn.append(R(uv / denom) if denom else None)     # x/0 -> null in Spark SQL
    u["IDness"] = idn
    return u if with_flags else u[["attribute", "unique_values", "IDness"]]


def measures_of_dispersion(table, list_of_cols="all", drop_cols=[], raw=False):
    """stats_generator.py:736-829.  raw=True: unrounded stddev/variance/cov/IQR/range
    (variance = stddev^2 without the intermediate rounding)."""
    num = S.segregate(table)[0]
    cols = _resolve(table, list_of_cols, drop_cols, num, universe=num, allow_empty=True)
    if not cols:
        warnings.warn("No Dispersion Computation - No numerical column(s) to analyze")
        return pd.DataFrame(columns=["attribute", "stddev", "variance", "cov", "IQR", "range"])
    rows = []
    for c, p in _profiles(table, cols).items():
        if p.n == 0:
            rows.append([c, None, None, None, None, None])
            continue
        n, mean, m2, _, _ = S.central_moments(p.x64)
        sd = S.stddev_samp(n, m2)
        mn, mx = p.minmax()
        q25, q75 = p._disp(p.quantile(0.25)), p._disp(p.quantile(0.75))
        mn, mx = p._disp(mn), p._disp(mx)
        if raw:
            rows.append([c, sd, None if sd is None else sd * sd, None if sd is None else sd / mean,
                         q75 - q25, mx - mn])
            continue
        sd_r = R(sd)                                                           # :818
        var = None if sd_r is None else R(sd_r * sd_r)                         # :819
        rng = R(mx - mn)                                                       # :820
        if sd_r is None:
            cov = None
        elif mean == 0:
            cov = None  # Spark SQL: division by zero -> null
        else:
            cov = R(sd_r / mean)                                               # :821
        rows.append([c, sd_r, var, cov, R(q75 - q25), rng])                    # :822
    return pd.DataFrame(rows, columns=["attribute", "stddev", "variance", "cov", "IQR", "range"])


PCT_STATS = ["min", "1%", "5%", "10%", "25%", "50%", "75%", "90%", "95%", "99%", "max"]


def measures_of_percentiles(table, list_of_cols="all", drop_cols=[], raw=False):
    """stats_generator.py:832-916."""
    num = S.segregate(table)[0]
    cols = _resolve(table, list_of_cols, drop_cols, num, universe=num, allow_empty=True)
    if not cols:
        warnings.warn("No Percentiles Computation - No numerical column(s) to analyze")
        return pd.DataFrame(columns=["attribute"] + PCT_STATS)
    rnd = (lambda v: v) if raw else R
    rows = []
    for c, p in _profiles(table, cols).items():
        if p.n == 0:
            rows.append([c] + [None] * 11)
            continue
        mn, mx = p.minmax()
        row = [c, rnd(p._disp(mn))]
        for s in PCT_STATS[1:-1]:
            row.append(rnd(p._disp(p.quantile(S.SUMMARY_PCTS[s]))))
        row.append(rnd(p._disp(mx)))
        rows.append(row)
    return pd.DataFrame(rows, columns=["attribute"] + PCT_STATS)


def measures_of_shape(table, list_of_cols="all", drop_cols=[], raw=False):
    """stats_generator.py:919-1011."""
    num = S.segregate(table)[0]
    cols = _resolve(table, list_of_cols, drop_cols, num, universe=num, allow_empty=True)
    if not cols:
        warnings.warn("No Skewness/Kurtosis Computation - No numerical column(s) to analyze")
        return pd.DataFrame(columns=["attribute", "skewness", "kurtosis"])
    rnd = (lambda v: v) if raw else R
    rows = []
    for c, p in _profiles(table, cols).items():
        n, mean, m2, m3, m4 = S.central_moments(p.x64)
        rows.append([c, rnd(S.skewness(n, m2, m3)), rnd(S.kurtosis(n, m2, m4))])
    return pd.DataFrame(rows, columns=["attribute", "skewness", "kurtosis"])


# ---------------------------------------------------------------------------
# attribute_binning (transformers.py:87-291)
# ---------------------------------------------------------------------------


def binning_cutoffs(table, cols, method_type="equal_range", bin_size=10):
    """-> (kept cols, cutoffs list-of-lists) following transformers.py:210-240."""
    kept, cuts, dropped = [], [], []
    for c in cols:
        p = _profiles(table, [c])[c]
        if method_type == "equal_frequency":
            if p.n == 0:
                kept.append(c)
                cuts.append([float("nan")] * (bin_size - 1))  # approxQuantile on empty: unpinned
                continue
            kept.append(c)
            cuts.append(p.equal_frequency_cutoffs(bin_size))
        else:
            if p.n == 0:
                dropped.append(c)                       # :226-228
                continue
            mn, mx = p.minmax()
            kept.append(c)
            cuts.append(S.equal_range_cutoffs(mn, mx, bin_size))
    if dropped:
        warnings.warn("Columns contains too much null values. Dropping " + ", ".join(dropped))
    return kept, cuts


def _write_model(model_path, cols, cuts):
    import pyarrow.parquet as pq
    d = os.path.join(model_path, "attribute_binning")
    os.makedirs(d, exist_ok=True)
    t = pa.table({"attribute": pa.array(cols, pa.string()),
                  "parameters": pa.array(cuts, pa.list_(pa.float64()))})
    pq.write_table(t, os.path.join(d, "part-00000.parquet"))


def _read_model(model_path):
    import pyarrow.parquet as pq
    t = pq.read_table(os.path.join(model_path, "attribute_binning"))
    return dict(zip(t.column("attribute").to_pylist(), t.column("parameters").to_pylist()))


def attribute_binning(table, list_of_cols="all", drop_cols=[], method_type="equal_range", bin_size=10,
                      bin_dtype="numerical", pre_existing_model=False, model_path="NA", output_mode="replace"):
    """transformers.py:87-291 -> pyarrow Table with int32 bin ids (null stays null)."""
    num = S.segregate(table)[0]
    cols = _resolve(table, list_of_cols, drop_cols, num, universe=num, allow_empty=True)
    if not cols:
        warnings.warn("No Binning Performed - No numerical column(s) to transform")
        return table
    if method_type not in ("equal_frequency", "equal_range"):
        raise TypeError("Invalid input for method_type")
    if bin_size < 2:
        raise TypeError("Invalid input for bin_size")
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")
    if pre_existing_model:
        model = _read_model(model_path)
        cuts = []
        for c in cols:
            if c not in model:
                raise IndexError("list index out of range")      # test_transformers.py:63-73
            cuts.append(model[c])
    else:
        cols, cuts = binning_cutoffs(table, cols, method_type, bin_size)
        if model_path != "NA":
            _write_model(model_path, cols, cuts)
    out = table
    n_over = (len(cuts[0]) + 1) if cuts else bin_size            # :269 quirk (Appendix C #3)
    for c, cut in zip(cols, cuts):
        p = _profiles(table, [c])[c]
        ids = S.assign_bins(p.values, p.valid, cut, bin_size)   # the column's own values: a bigint compares exactly
        ids[(ids == len(cut) + 1)] = n_over
        if bin_dtype == "numerical":
            arr = pa.array(ids, type=pa.int32(), mask=~p.valid)
        else:
            labels = []
            for k, ok in zip(ids.tolist(), p.valid.tolist()):
                if not ok:
                    labels.append(None)
                elif k == 1:
                    labels.append("<= " + str(round(cut[0], 4)))
                elif k <= len(cut):
                    labels.append(str(round(cut[k - 2], 4)) + "-" + str(round(cut[k - 1], 4)))
                else:
                    labels.append("> " + str(round(cut[len(cuts[0]) - 1], 4)))
            arr = pa.array(labels, type=pa.string())
        if output_mode == "replace":
            out = out.set_column(out.column_names.index(c), c, arr)
        else:
            out = out.append_column(c + "_binned", arr)
    return out


# ---------------------------------------------------------------------------
# drift_detector.statistics (drift_detector.py:16-371)
# ---------------------------------------------------------------------------


def _check_columns(table, list_of_cols, drop_cols):
    """validations.py:19-66."""
    if isinstance(list_of_cols, str):
        if list_of_cols == "all":
            num, cat, _ = S.segregate(table)
            cols = num + cat
        else:
            cols = [x.strip() for x in list_of_cols.split("|")]
    elif isinstance(list_of_cols, list):
        cols = list_of_cols
    else:
        raise TypeError("'list_of_cols' must be either a string or a list of strings. Received %s." % type(list_of_cols))
    if drop_cols is None:
        drop_cols = []
    if isinstance(drop_cols, str):
        drops = [x.strip() for x in drop_cols.split("|")]
    elif isinstance(drop_cols, list):
        drops = drop_cols
    else:
        raise TypeError("'drop_cols' must be either a string or a list of strings. Received %s." % type(drop_cols))
    final = _dedupe(cols, drops)
    if not final:
        raise ValueError("Empty set of columns is given. Columns to select: %s, columns to drop: %s." % (cols, drops))
    if any(c not in table.column_names for c in final):
        raise ValueError("Not all columns are in the input dataframe. Missing columns: %s"
                         % (set(final) - set(table.column_names)))
    return final


def _check_methods(method_type):
    """validations.py:71-94."""
    m = method_type
    if isinstance(m, str):
        m = ["PSI", "JSD", "HD", "KS"] if m == "all" else [x.strip() for x in m.split("|")]
    if any(x not in ("PSI", "JSD", "HD", "KS") for x in m):
        raise TypeError("Invalid input for method_type")
    return m


def _group_counts(table, col, is_binned_numeric):
    """groupBy(col).agg(count(col)): dict key -> non-null count; null group -> key -1
    (numeric, after fillna(-1)) or dropped from matching (string: SQL null never joins)."""
    vals, valid = S.column_values(table, col)
    groups = {}
    if valid.any():
        nn = vals[valid]
        if nn.dtype == object:
            u, c = np.unique(nn.astype(str), return_counts=True)
            u = u.tolist()
        else:
            u, c = np.unique(nn, return_counts=True)
            u = u.tolist()
        for k, v in zip(u, c.tolist()):
            groups[k] = int(v)
    has_null = bool((~valid).any())
    if has_null and is_binned_numeric:
        groups[-1] = 0
    return groups, (has_null and not is_binned_numeric)


def _partition_slices(table):
    md = table.schema.metadata or {}
    rows = json.loads(md[b"spark_partition_rows"]) if b"spark_partition_rows" in md else [table.num_rows]
    out, r0 = [], 0
    for k in rows:
        out.append((r0, k))
        r0 += k
    return out


def _cast_string(v, sdtype):
    if sdtype == "string":
        return str(v)
    if sdtype in ("int", "bigint", "long"):
        return str(int(v))
    if sdtype == "float":
        return S.java_double_to_string(float(str(np.float32(v))))
    return S.java_double_to_string(float(v))


def data_sample(table, strata_cols="all", drop_cols=[], fraction=0.1, method_type="random", stratified_type="population",
                seed_value=12, unique_threshold=0.5):
    """data_sampling.py:8-149 on a pyarrow Table (Spark partitions from the `spark_partition_rows` metadata, else one
    partition): Bernoulli sampling with Spark's XORShiftRandom(seed + partition index), one draw per row
    (`sample`) or per row surviving na.drop (`sampleBy`)."""
    if type(fraction) != float and type(fraction) != int:
        raise TypeError("Invalid input for fraction")
    if fraction <= 0 or fraction > 1:
        raise TypeError("Invalid input for fraction: fraction value is between 0 and 1")
    if type(seed_value) != int:
        raise TypeError("Invalid input for seed_value")
    if method_type not in ["stratified", "random"]:
        raise TypeError("Invalid input for data_sample method_type")
    parts = _partition_slices(table)
    if method_type == "random":
        keep = np.concatenate([S.bernoulli_keep(k, seed_value + i, fraction) for i, (r0, k) in enumerate(parts)]) \
            if table.num_rows else np.zeros(0, bool)
        return table.filter(pa.array(keep))
    if type(unique_threshold) != float and type(unique_threshold) != int:
        raise TypeError("Invalid input for unique_threshold")
    if unique_threshold > 1 and type(unique_threshold) != int:
        raise TypeError("Invalid input for unique_threshold: unique_threshold can only be integer if larger than 1")
    if unique_threshold <= 0:
        raise TypeError("Invalid input for unique_threshold: unique_threshold value is either between 0 and 1, or an integer > 1")
    if stratified_type not in ["population", "balanced"]:
        raise TypeError("Invalid input for stratified_type")
    if isinstance(strata_cols, str) and strata_cols == "all":
        strata_cols = table.column_names
    strata_cols = _split(strata_cols)
    drop_cols = _split(drop_cols)
    strata_cols = list(dict.fromkeys(e for e in strata_cols if e not in drop_cols))
    if not strata_cols:
        raise TypeError("Missing strata_cols value")
    N = table.num_rows
    skip = []
    for c in strata_cols:
        if c not in table.column_names:
            raise TypeError("Invalid input for strata_cols: " + c + " does not exist")
        p = _profiles(table, [c])[c]
        distinct = p.distinct() + (1 if p.n < N else 0)          # distinct() keeps the null group
        if float(distinct) > (unique_threshold * float(N) if unique_threshold <= 1 else unique_threshold):
            skip.append(c)
    if skip:
        warnings.warn("Columns dropped from strata due to high cardinality: " + ",".join(skip))
    strata_cols = [c for c in strata_cols if c not in skip]
    if not strata_cols:
        warnings.warn("No Stratified Sampling Computation - No strata column(s) to sample")
        return table
    profs = _profiles(table, strata_cols)
    ok = np.ones(N, bool)
    for c in strata_cols:
        ok &= profs[c].valid
    merge = np.array(["".join(_cast_string(profs[c].values[i], profs[c].sdtype) for c in strata_cols) if ok[i] else ""
                      for i in range(N)], dtype=object)
    keys, counts = np.unique(merge[ok].astype(str), return_counts=True) if ok.any() else (np.array([]), np.array([]))
    frac = {k: float(fraction) for k in keys}
    if stratified_type == "balanced" and len(keys):
        smallest = int(counts.min())
        frac = {k: float(fraction * smallest / int(c)) for k, c in zip(keys.tolist(), counts.tolist())}
    keep = np.zeros(N, bool)
    for i, (r0, k) in enumerate(parts):
        idx = np.flatnonzero(ok[r0:r0 + k]) + r0                 # the rows that reach the rand() filter, in order
        if idx.size:
            f = np.array([frac[str(m)] for m in merge[idx]])
            keep[idx] = S.bernoulli_keep(idx.size, seed_value + i, f)
    return table.filter(pa.array(keep))


def statistics(idf_target, idf_source, *, list_of_cols="all", drop_cols=None, method_type="PSI",
               bin_method="equal_range", bin_size=10, threshold=0.1, use_sampling=True, sample_size=100000,
               pre_existing_source=False, source_save=True, source_path="NA",
               model_directory="drift_statistics", return_groups=False, sample_method="random", strata_cols="all",
               stratified_type="population", sample_seed=42):
    """drift_detector.py:16-371, including the default sampling step (:187-211 -> data_sample)."""
    cols = _check_columns(idf_target, list_of_cols, drop_cols)
    methods = _check_methods(method_type)
    num_cols = S.segregate(idf_target.select(cols))[0]
    if use_sampling:
        if idf_target.num_rows > sample_size:
            idf_target = data_sample(idf_target, strata_cols=strata_cols, fraction=sample_size / idf_target.num_rows,
                                     method_type=sample_method, stratified_type=stratified_type, seed_value=sample_seed)
        if idf_source is not None and idf_source.num_rows > sample_size:
            idf_source = data_sample(idf_source, strata_cols=strata_cols, fraction=sample_size / idf_source.num_rows,
                                     method_type=sample_method, stratified_type=stratified_type, seed_value=sample_seed)
    n_t, n_s = idf_target.num_rows, (idf_source.num_rows if idf_source is not None else None)
    if source_path == "NA":
        source_path = "intermediate_data"
    model_path = source_path + "/" + model_directory
    if not pre_existing_source:
        source_bin = attribute_binning(idf_source, list_of_cols=num_cols, method_type=bin_method,
                                       bin_size=bin_size, pre_existing_model=False, model_path=model_path) \
            if num_cols else idf_source
    # equal_range drops all-null source columns from the model: the target then keeps raw values
    model = _read_model(model_path) if num_cols else {}
    tgt_num = [c for c in num_cols if c in model]
    target_bin = attribute_binning(idf_target, list_of_cols=tgt_num, method_type=bin_method, bin_size=bin_size,
                                   pre_existing_model=True, model_path=model_path) if tgt_num else idf_target
    rows, dbg = [], {}
    for c in cols:
        binned = c in num_cols
        if pre_existing_source:
            f = pd.read_csv(os.path.join(model_path, "frequency_counts", c, "part-00000.csv"))
            src = {k: v for k, v in zip(f[c].tolist(), f["p"].tolist()) if not (isinstance(k, float) and math.isnan(k))}
            src_null = len(src) != len(f)
            src_p_direct = True
        else:
            src, src_null = _group_counts(source_bin, c, binned)
            src_p_direct = False
            if source_save:
                d = os.path.join(model_path, "frequency_counts", c)
                os.makedirs(d, exist_ok=True)
                keys = sorted(src)
                kcol, pcol = ([None] if src_null else []) + keys, ([0.0] if src_null else []) + [src[k] / n_s for k in keys]
                pd.DataFrame({c: kcol, "p": pcol}).to_csv(
                    os.path.join(d, "part-00000.csv"), index=False)
        tgt, tgt_null = _group_counts(target_bin, c, binned)
        keys = sorted(set(src) | set(tgt))
        nulls = int(src_null) + int(tgt_null)
        if src_p_direct:
            # p comes from the saved CSV (drift_detector.py:245-250): already proportions
            tgt_p = {k: v / n_t for k, v in tgt.items()}
            psi, hd, jsd, ks = S.drift_from_groups(src, tgt_p, 1, 1, keys, nulls)
        else:
            psi, hd, jsd, ks = S.drift_from_groups(src, tgt, n_s, n_t, keys, nulls)
        if psi is None:
            psi = hd = jsd = ks = None
        row = {"attribute": c}
        for name, v in (("PSI", psi), ("HD", hd), ("JSD", jsd), ("KS", ks)):   # code order :273-335
            if name in methods:
                row[name] = v
        vals = [row[m] for m in row if m != "attribute"]
        row["flagged"] = int(any(v is not None and v > threshold for v in vals))  # :353-356
        rows.append(row)
        dbg[c] = (src, tgt)
    out = pd.DataFrame(rows)
    return (out, dbg) if return_groups else out


# ---------------------------------------------------------------------------
# N1: stability_index_computation (drift_stability/stability.py:15-332, validations.py:97-172)
# ---------------------------------------------------------------------------


def compute_score(value, method_type, cv_thresholds=(0.03, 0.1, 0.2, 0.5)):
    """validations.py:97-126."""
    if value is None:
        return None
    if method_type == "cv":
        cv = abs(value)
        for i, th in enumerate(cv_thresholds):
            if cv < th:
                return float([4, 3, 2, 1, 0][i])
        return 0.0
    if method_type == "sd":
        sd = value
        if sd <= 0.005:
            return 4.0
        if sd <= 0.01:
            return round(-100 * sd + 4.5, 1)
        if sd <= 0.05:
            return round(-50 * sd + 4, 1)
        if sd <= 0.1:
            return round(-30 * sd + 3, 1)
        return 0.0
    raise TypeError("method_type must be either 'cv' or 'sd'.")


def _samp_std(vals):
    vals = [v for v in vals if v is not None]
    if len(vals) < 2:
        return None
    m = sum(vals) / len(vals)
    return math.sqrt(sum((v - m) ** 2 for v in vals) / (len(vals) - 1))


def _mean(vals):
    vals = [v for v in vals if v is not None]
    return sum(vals) / len(vals) if vals else None


def _div(a, b):
    if a is None or b is None or b == 0:
        return None
    return a / b


def stability_index_computation(tables, list_of_cols="all", drop_cols=[], metric_weightages=None, binary_cols=[],
                                existing_metric_path="", appended_metric_path="", threshold=1):
    """stability.py:150-332 on a list of pyarrow Tables."""
    metric_weightages = metric_weightages or {"mean": 0.5, "stddev": 0.3, "kurtosis": 0.2}
    num = S.segregate(tables[0])[0]
    cols = _resolve(tables[0], list_of_cols, drop_cols, num, universe=num)
    binary_cols = _split(binary_cols)
    if any(c not in cols for c in binary_cols):
        raise TypeError("Invalid input for Binary Column(s)")
    if round(sum(metric_weightages.get(k, 0) for k in ("mean", "stddev", "kurtosis")), 3) != 1:
        raise ValueError("Invalid input for metric weightages. Either metric name is incorrect or sum of metric "
                         "weightages is not 1.0.")
    if threshold < 0 or threshold > 4:
        raise ValueError("Invalid input for metric threshold. It must be a number between 0 and 4.")
    existing = None
    start = 1
    if existing_metric_path:
        files = sorted(f for f in os.listdir(existing_metric_path) if f.endswith(".csv"))
        existing = pd.concat([pd.read_csv(os.path.join(existing_metric_path, f)) for f in files], ignore_index=True)
        start = int(existing["idx"].max()) + 1
    rows, appended = [], []
    for c in cols:
        ctype = "Binary" if c in binary_cols else "Numerical"
        means, sds, kurts = [], [], []
        for k, t in enumerate(tables):
            p = ColumnProfile(t, c)
            n, mean, m2, m3, m4 = S.central_moments(p.x64)
            sd = S.stddev_samp(n, m2)
            ku = S.kurtosis(n, m2, m4)
            ku = None if ku is None else ku + 3
            means.append(mean); sds.append(sd); kurts.append(ku)
            appended.append([start + k, c, ctype, mean, sd, ku])
        if existing is not None:
            e = existing[existing["attribute"] == c]
            means += [None if pd.isna(v) else float(v) for v in e["mean"]]
            sds += [None if pd.isna(v) else float(v) for v in e["stddev"]]
            kurts += [None if pd.isna(v) else float(v) for v in e["kurtosis"]]
        mean_sd = _samp_std(means)
        mean_cv = _div(mean_sd, _mean(means))
        sd_cv = _div(_samp_std(sds), _mean(sds))
        ku_cv = _div(_samp_std(kurts), _mean(kurts))
        if ctype == "Binary":
            mean_si = compute_score(mean_sd, "sd")
            sd_si = ku_si = None
            si = mean_si
        else:
            mean_si, sd_si, ku_si = compute_score(mean_cv, "cv"), compute_score(sd_cv, "cv"), compute_score(ku_cv, "cv")
            si = None if None in (mean_si, sd_si, ku_si) else round(
                mean_si * metric_weightages.get("mean", 0) + sd_si * metric_weightages.get("stddev", 0)
                + ku_si * metric_weightages.get("kurtosis", 0), 4)
        f32 = lambda v: None if v is None else float(np.float32(v))      # ArrayType(FloatType()) (:293)
        rows.append([c, ctype, R(mean_sd), R(mean_cv), R(sd_cv), R(ku_cv), f32(mean_si), f32(sd_si), f32(ku_si), f32(si),
                     int(si is None or si < threshold)])
    if appended_metric_path:
        os.makedirs(appended_metric_path, exist_ok=True)
        df = pd.DataFrame(appended, columns=["idx", "attribute", "type", "mean", "stddev", "kurtosis"])
        if existing is not None:
            df = pd.concat([df, existing], ignore_index=True)
        df.sort_values("idx", kind="stable").to_csv(os.path.join(appended_metric_path, "part-00000.csv"), index=False)
    return pd.DataFrame(rows, columns=["attribute", "type", "mean_stddev", "mean_cv", "stddev_cv", "kurtosis_cv", "mean_si",
                                       "stddev_si", "kurtosis_si", "stability_index", "flagged"])


# ---------------------------------------------------------------------------
# N3: IV_calculation / IG_calculation (data_analyzer/association_evaluator.py:253-586)
# ---------------------------------------------------------------------------


def _label_classes(table, label_col, event_label):
    vals, valid = S.column_values(table, label_col)
    if vals.dtype == object:
        ev = valid & (vals.astype(str) == str(event_label))
    else:
        ev = valid & (vals.astype(np.float64) == float(event_label))
    return ev, valid & ~ev          # event rows, non-event rows (label null -> neither)


def _encoded_groups(table, col, encoding_configs):
    """-> (group key per row [object array, None = null group])."""
    p = ColumnProfile(table, col)
    if p.is_num and encoding_configs:
        if encoding_configs.get("monotonicity_check", 0) == 1:
            raise NotImplementedError("monotonic_binning is not restated")
        bs, bm = encoding_configs["bin_size"], encoding_configs["bin_method"]
        if p.n == 0:
            return np.array([None] * p.N, dtype=object)
        cut = p.equal_frequency_cutoffs(bs) if bm == "equal_frequency" else S.equal_range_cutoffs(*p.minmax(), bs)
        ids = S.assign_bins(p.values, p.valid, cut, bs)
        return np.array([int(k) if ok else None for k, ok in zip(ids, p.valid)], dtype=object)
    return np.array([(v if ok else None) for v, ok in zip(p.values.tolist(), p.valid)], dtype=object)


def _group_counts_by_class(keys, nev, ev):
    """groupBy(attribute): per group (null = its own group) -> (non-event rows, event rows, all rows) as floats."""
    is_null = np.array([k is None for k in keys.tolist()])
    labels = np.array(["\0null" if k is None else ("s" + k if isinstance(k, str) else "n%r" % (k,)) for k in keys.tolist()], dtype=object)
    _, inv = np.unique(labels.astype(str), return_inverse=True)
    g = int(inv.max()) + 1 if inv.size else 0
    l0 = np.bincount(inv, weights=nev.astype(np.float64), minlength=g)
    l1 = np.bincount(inv, weights=ev.astype(np.float64), minlength=g)
    tc = np.bincount(inv, minlength=g).astype(np.float64)
    return list(zip(l0.tolist(), l1.tolist(), tc.tolist()))


def _iv_ig_cols(table, list_of_cols, drop_cols, label_col, event_label):
    if label_col not in table.column_names:
        raise TypeError("Invalid input for Label Column")
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        num, cat, _ = S.segregate(table)
        list_of_cols = num + cat
    cols = _dedupe(_split(list_of_cols), _split(drop_cols) + [label_col])
    if any(c not in table.column_names for c in cols) or not cols:
        raise TypeError("Invalid input for Column(s)")
    ev, nev = _label_classes(table, label_col, event_label)
    if ev.sum() == 0:
        raise TypeError("Invalid input for Event Label Value")
    return cols, ev, nev


_DEFAULT_ENC = {"bin_method": "equal_frequency", "bin_size": 10, "monotonicity_check": 0}


def IV_calculation(table, list_of_cols="all", drop_cols=[], label_col="label", event_label=1, encoding_configs=_DEFAULT_ENC):
    """association_evaluator.py:253-424."""
    cols, ev, nev = _iv_ig_cols(table, list_of_cols, drop_cols, label_col, event_label)
    rows = []
    for c in cols:
        keys = _encoded_groups(table, c, encoding_configs)
        t0, t1 = float(nev.sum()), float(ev.sum())
        iv = 0.0
        for l0, l1, _ in _group_counts_by_class(keys, nev, ev):
            ne, e = l0 / t0, l1 / t1
            woe = math.log(ne / e) if (ne != 0 and e != 0) else math.log(((l0 + 0.5) / t0) / ((l1 + 0.5) / t1))
            iv += woe * (ne - e)
        rows.append([c, iv])
    return pd.DataFrame(rows, columns=["attribute", "iv"])


def IG_calculation(table, list_of_cols="all", drop_cols=[], label_col="label", event_label=1, encoding_configs=_DEFAULT_ENC):
    """association_evaluator.py:427-586.  log2(0) is NULL in Spark SQL, so a segment whose event_pct is 0 or 1
    contributes nothing to entropy_sum."""
    cols, ev, nev = _iv_ig_cols(table, list_of_cols, drop_cols, label_col, event_label)
    n = table.num_rows
    te = ev.sum() / n
    total_entropy = -(te * math.log2(te) + (1 - te) * math.log2(1 - te))
    rows = []
    for c in cols:
        keys = _encoded_groups(table, c, encoding_configs)
        s = 0.0
        any_term = False
        for _, ec, tc in _group_counts_by_class(keys, nev, ev):    # count(label) after the when/otherwise recode: every row
            p = ec / tc
            if 0 < p < 1:
                s += -(tc / n) * (p * math.log2(p) + (1 - p) * math.log2(1 - p))
                any_term = True
        # F.sum over segments whose entropy is NULL everywhere is NULL (an id-like column: every segment pure), pinned
        # by the reference notebook (ifa: NaN)
        rows.append([c, total_entropy - s if any_term else None])
    return pd.DataFrame(rows, columns=["attribute", "ig"])


# ---------------------------------------------------------------------------
# quality_checker.outlier_detection (data_analyzer/quality_checker.py:550-1045)
# ---------------------------------------------------------------------------

_DEFAULT_OUTLIER_CFG = {"pctile_lower": 0.05, "pctile_upper": 0.95, "stdev_lower": 3.0, "stdev_upper": 3.0,
                        "IQR_lower": 1.5, "IQR_upper": 1.5, "min_validation": 2}


def outlier_methodologies(detection_side, detection_configs):
    """:788-830 -> (methodologies, min_validation); raises the reference's TypeErrors."""
    sides = {"lower": ["lower"], "upper": ["upper"], "both": ["lower", "upper"]}[detection_side]
    check = {m: {"lower": 0, "upper": 0} for m in ("pctile", "stdev", "IQR")}
    for m in check:
        for s in sides:
            if m + "_" + s in detection_configs:
                check[m][s] = 1
    methods = []
    for m, val in check.items():
        vals = list(val.values())
        if detection_side == "both":
            if vals in ([1, 0], [0, 1]):
                raise TypeError("Invalid input for detection_configs. If detection_side is 'both', the methodologies "
                                "used on both sides should be the same")
            if vals[0]:
                methods.append(m)
        elif val[detection_side]:
            methods.append(m)
    if "min_validation" in detection_configs:
        if detection_configs["min_validation"] > len(methods):
            raise TypeError("Invalid input for min_validation of detection_configs. It cannot be larger than the total "
                            "number of methodologies on any side that detection will be applied over.")
        n = detection_configs["min_validation"]
    else:
        n = len(methods)
    return methods, n


def outlier_bounds(table, cols, detection_side="upper", detection_configs=_DEFAULT_OUTLIER_CFG):
    """-> (kept cols, [[lower|None, upper|None]], skewed cols).  Percentiles follow approxQuantile(cols, p, 0.01)
    (:845,883) through S.approx_quantile_rank: the GK sketch position for one partition of < 50 000 values (this
    reproduces all 13 pinned counts / clamp values of test_quality_checker.py:526-637), the exact rank beyond."""
    methods, n = outlier_methodologies(detection_side, detection_configs)
    prof = _profiles(table, cols)
    pl, pu = detection_configs.get("pctile_lower", 0.05), detection_configs.get("pctile_upper", 0.95)
    E = S.APPROX_QUANTILE_EPS
    pct = {c: [prof[c].quantile(pl, E), prof[c].quantile(pu, E)] for c in cols}
    skewed = [c for c in cols if pct[c][0] == pct[c][1]]
    kept = [c for c in cols if c not in skewed]
    params = []
    for c in kept:
        p = prof[c]
        x = pct[c] if "pctile" in methods else [None, None]
        y = [None, None]
        if "stdev" in methods:
            cnt, mean, m2, _, _ = S.central_moments(p.x64)
            sd = S.stddev_samp(cnt, m2)
            sd = float("nan") if sd is None else sd
            y = [mean - detection_configs.get("stdev_lower", 0.0) * sd, mean + detection_configs.get("stdev_upper", 0.0) * sd]
        z = [None, None]
        if "IQR" in methods:
            q1, q3 = p.quantile(0.25, E), p.quantile(0.75, E)
            z = [q1 - detection_configs.get("IQR_lower", 0.0) * (q3 - q1), q3 + detection_configs.get("IQR_upper", 0.0) * (q3 - q1)]
        lower = sorted([i for i in (x[0], y[0], z[0]) if i is not None], reverse=True)[n - 1]
        upper = sorted([i for i in (x[1], y[1], z[1]) if i is not None])[n - 1]
        params.append([lower, None] if detection_side == "lower" else ([None, upper] if detection_side == "upper" else [lower, upper]))
    return kept, params, skewed


def outlier_detection(table, list_of_cols="all", drop_cols=[], detection_side="upper", detection_configs=None,
                      treatment=True, treatment_method="value_replacement", output_mode="replace", params=None):
    """-> (treated pyarrow table, odf_print pandas [attribute, lower_outliers, upper_outliers,
    excluded_due_to_skewness]).  `params` = (cols, bounds, skewed) of a saved model instead of computing them."""
    cfg = dict(_DEFAULT_OUTLIER_CFG if detection_configs is None else detection_configs)
    num = [f.name for f in table.schema if ColumnProfile(table.slice(0, 0), f.name).is_num]
    cols = _dedupe(num if (isinstance(list_of_cols, str) and list_of_cols == "all") else _split(list_of_cols), _split(drop_cols))
    if any(c not in num for c in cols):
        raise TypeError("Invalid input for Column(s)")
    if detection_side not in ("upper", "lower", "both"):
        raise TypeError("Invalid input for detection_side")
    if treatment_method not in ("null_replacement", "row_removal", "value_replacement"):
        raise TypeError("Invalid input for treatment_method")
    kept, bounds, skewed = params if params is not None else outlier_bounds(table, cols, detection_side, cfg)
    rows, flags, new_cols = [], {}, {}
    for c, (lo, hi) in zip(kept, bounds):
        vals, valid = S.column_values(table, c)
        v = vals.astype(np.float64)
        with np.errstate(invalid="ignore"):
            low = valid & ((v - lo) < 0) if lo is not None and detection_side in ("lower", "both") else np.zeros(len(v), bool)
            up = valid & ((v - hi) > 0) if hi is not None and detection_side in ("upper", "both") else np.zeros(len(v), bool)
        flags[c] = low | up
        rows.append((c, int(low.sum()), int(up.sum()), 0))
        if treatment and treatment_method == "value_replacement":
            out = v.copy()
            out[low], out[up] = (lo if lo is not None else 0.0), (hi if hi is not None else 0.0)
            new_cols[c] = pa.array(out, mask=~valid)
        elif treatment and treatment_method == "null_replacement":
            new_cols[c] = pa.array(vals, mask=~valid | low | up)
    rows += [(c, 0, 0, 1) for c in skewed]
    odf = table
    if treatment and treatment_method == "row_removal":
        keep = np.ones(table.num_rows, bool)
        for c in kept:
            keep &= ~flags[c]
        odf = table.filter(pa.array(keep))
    elif treatment:
        for c, arr in new_cols.items():
            if output_mode == "replace":
                odf = odf.set_column(odf.schema.get_field_index(c), c, arr)
            else:
                odf = odf.append_column(c + "_outliered", arr)
    return odf, pd.DataFrame(rows, columns=["attribute", "lower_outliers", "upper_outliers", "excluded_due_to_skewness"])
