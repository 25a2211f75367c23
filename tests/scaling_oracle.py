"""TEST INFRASTRUCTURE: the oracle of the scalers z_standardization, IQR_standardization and normalization (reference
data_transformer/transformers.py:965-1366) on pyarrow Tables, written from the reference and Spark's semantics with
NumPy, independently of the product's code.

    z_standardization(table, ...) / IQR_standardization(table, ...) / normalization(table, ...)
        -> (pyarrow Table, parameters per listed column, excluded columns)
    scale_reference(vals, valid, spec) -> (values, bool valid): the exact NumPy image of one anv_scale_columns column

Spark semantics restated:
  - z: mean = avg, stddev = stddev_samp (null for fewer than two values); `float(x) if x else None` turns a zero mean or
    stddev into null; a fresh fit excludes a column whose stddev is null or rounds to 0.0 at 5 places; the transform
    `(col - mean) / stddev` is double, null where a parameter is null or the divisor is 0 (Divide), NaN stays NaN;
  - IQR: approxQuantile(cols, [0.25, 0.5, 0.75], 0.01), which skips null and NaN ([] for a column without a value; the
    GK sketch merged over the table's Spark partitions when it is tagged with them); excluded on both paths when [] or
    round(p25, 5) == round(p75, 5); `(col - p50) / (p75 - p25)`;
  - normalization: VectorAssembler(handleInvalid="keep") turns null into NaN; MinMaxScaler's Summarizer skips NaN in
    min / max (an all-NaN feature keeps min = Double.MaxValue, max = Double.MinValue: recalled from Spark's
    SummarizerBuffer, not checked against a Spark run); MinMaxScalerModel (Spark 3): scale = (hi - lo) / (max - min),
    (x - min) * scale + lo where scale != 0, else 0.5 * (hi - lo) + lo, NaN kept; the UDF's FloatType rounds to float;
    NaN becomes null.  The column list is positional over the model's vectors.
Column order is first-seen (the reference's list(set()) order is arbitrary).
"""
from __future__ import annotations

import json
import math
import os
import warnings

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from oracle import api as O
from oracle import spark_semantics as S

DIV, AFFINE, CONST = 0, 1, 2           # ANV_SCALE_* of the header
F32, F64 = 0, 1
NAN_TO_NULL = 1
DOUBLE_MAX = 1.7976931348623157e308


def scale_reference(vals, valid, spec):
    """spec = (mode, out dtype, flags, a, b, c).  Each operation is a separately rounded float64 NumPy ufunc; F32 outputs
    are rounded to nearest; null rows are 0."""
    mode, od, flags, a, b, c = spec
    x = np.asarray(vals).astype(np.float64)
    valid = np.asarray(valid, bool)
    with np.errstate(all="ignore"):
        if mode == DIV:
            v = np.divide(np.subtract(x, np.float64(a)), np.float64(b))
        elif mode == AFFINE:
            v = np.add(np.multiply(np.subtract(x, np.float64(a)), np.float64(b)), np.float64(c))
        else:
            v = np.full(x.shape, np.float64(c))
        ok = valid.copy()
        if flags & NAN_TO_NULL:
            ok &= ~np.isnan(x) & ~np.isnan(v)
        out = v.astype(np.float32 if od == F32 else np.float64)
    out[~ok] = 0
    return out, ok


def _values(table, c):
    arr = table.column(c).combine_chunks()
    valid = np.asarray(arr.is_valid())
    return (arr.fill_null(0) if arr.null_count else arr).to_numpy(zero_copy_only=False), valid


def _nan_free(table, c):
    vals, valid = _values(table, c)
    keep = valid & ~np.isnan(vals.astype(np.float64)) if vals.dtype.kind == "f" else valid
    return table.set_column(table.column_names.index(c), c, pa.array(vals, mask=~keep))


def _cols(table, list_of_cols, drop_cols, output_mode, what):
    num = S.segregate(table)[0]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num
    if isinstance(list_of_cols, str):
        list_of_cols = [x.strip() for x in list_of_cols.split("|")]
    if isinstance(drop_cols, str):
        drop_cols = [x.strip() for x in drop_cols.split("|")]
    cols = [c for c in dict.fromkeys(list_of_cols) if c not in drop_cols]
    if any(x not in num for x in cols):
        raise TypeError("Invalid input for Column(s)")
    if not cols:
        warnings.warn("No %s Performed - No numerical column(s) to transform" % what)
        return None
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")
    return cols


def _out(table, cols, outs, output_mode):
    """outs: name -> pa.Array of the scaled column (only the columns that were transformed)."""
    names, arrays = list(table.column_names), [table.column(n) for n in table.column_names]
    for c in cols:
        if c not in outs:
            continue
        if output_mode == "replace":
            arrays[names.index(c)] = outs[c]
        else:
            names.append(c + "_scaled")
            arrays.append(outs[c])
    return pa.table(arrays, names=names)


def _divide(table, c, a, b):
    """Spark's `(col - a) / b`, double."""
    x, valid = _values(table, c)
    n = len(x)
    if a is None or b is None or b == 0:
        return pa.array(np.zeros(n), mask=np.ones(n, bool))
    out, ok = scale_reference(x, valid, (DIV, F64, 0, a, b, 0.0))
    return pa.array(out, mask=~ok)


# ---- models --------------------------------------------------------------------------------------------------------

def _parquet_files(d):
    return sorted(os.path.join(d, f) for f in os.listdir(d) if f.startswith("part-") and f.endswith(".parquet"))


def write_param_model(model_path, name, cols, params):
    d = os.path.join(model_path, name)
    os.makedirs(d, exist_ok=True)
    for f in _parquet_files(d):
        os.remove(f)
    pq.write_table(pa.table({"feature": pa.array(cols, pa.string()), "parameters": pa.array(params, pa.list_(pa.float64()))}),
                   os.path.join(d, "part-00000.parquet"))


def read_param_model(model_path, name, cols):
    t = pa.concat_tables([pq.read_table(f) for f in _parquet_files(os.path.join(model_path, name))])
    rows = list(zip(t.column("feature").to_pylist(), t.column("parameters").to_pylist()))
    out = []
    for c in cols:
        hit = [p for f, p in rows if f == c]
        out.append(hit[0])          # IndexError("list index out of range") when the model lacks the column
    return out


def _vec(v):
    if v["type"] == 1:
        return list(v["values"])
    out = [0.0] * v["size"]
    for i, x in zip(v["indices"], v["values"]):
        out[i] = x
    return out


def read_minmax_model(model_path):
    d = os.path.join(model_path, "normalization")
    md = sorted(f for f in os.listdir(os.path.join(d, "metadata")) if f.startswith("part-") and not f.endswith(".crc"))[0]
    meta = json.loads(open(os.path.join(d, "metadata", md)).readline())
    p = dict(meta.get("defaultParamMap", {}), **meta.get("paramMap", {}))
    row = pa.concat_tables([pq.read_table(f) for f in _parquet_files(os.path.join(d, "data"))]).to_pylist()[0]
    return float(p.get("min", 0.0)), float(p.get("max", 1.0)), _vec(row["originalMin"]), _vec(row["originalMax"])


def write_minmax_model(model_path, mins, maxs):
    d = os.path.join(model_path, "normalization")
    for sub in ("metadata", "data"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    with open(os.path.join(d, "metadata", "part-00000"), "w") as f:
        f.write(json.dumps({"class": "org.apache.spark.ml.feature.MinMaxScalerModel", "paramMap": {},
                            "defaultParamMap": {"min": 0.0, "max": 1.0}}) + "\n")
    vec = pa.struct([("type", pa.int8()), ("size", pa.int32()), ("indices", pa.list_(pa.int32())),
                     ("values", pa.list_(pa.float64()))])
    pq.write_table(pa.table({k: pa.array([{"type": 1, "size": None, "indices": None, "values": list(v)}], vec)
                             for k, v in (("originalMin", mins), ("originalMax", maxs))}),
                   os.path.join(d, "data", "part-00000.parquet"))


# ---- the three functions -------------------------------------------------------------------------------------------

def z_standardization(table, list_of_cols="all", drop_cols=[], pre_existing_model=False, model_path="NA",
                      output_mode="replace"):
    cols = _cols(table, list_of_cols, drop_cols, output_mode, "Standardization")
    if cols is None:
        return table, [], []
    excluded = []
    if pre_existing_model:
        params = read_param_model(model_path, "z_standardization", cols)
    else:
        params = []
        for c in cols:
            x, valid = _values(table, c)
            x = x[valid].astype(np.float64)
            n, mean, m2, _, _ = S.central_moments(x)
            sd = math.sqrt(m2 / (n - 1)) if n > 1 else None
            params.append([float(mean) if mean else None, float(sd) if sd else None])
            if not sd or round(sd, 5) == 0.0:
                excluded.append(c)
        if model_path != "NA":
            write_param_model(model_path, "z_standardization", cols, params)
    if excluded:
        warnings.warn("The following column(s) are excluded from standardization because the standard deviation is zero:"
                      + str(excluded))
    outs = {c: _divide(table, c, p[0], p[1]) for c, p in zip(cols, params) if c not in excluded}
    return _out(table, cols, outs, output_mode), params, excluded


def quartiles(table, c):
    t = _nan_free(table, c)
    prof = O.ColumnProfile(t, c)
    if prof.n == 0:
        return []
    return [float(prof.quantile(p, 0.01)) for p in (0.25, 0.5, 0.75)]


def IQR_standardization(table, list_of_cols="all", drop_cols=[], pre_existing_model=False, model_path="NA",
                        output_mode="replace"):
    cols = _cols(table, list_of_cols, drop_cols, output_mode, "Standardization")
    if cols is None:
        return table, [], []
    if pre_existing_model:
        params = read_param_model(model_path, "IQR_standardization", cols)
    else:
        params = [quartiles(table, c) for c in cols]
        if model_path != "NA":
            write_param_model(model_path, "IQR_standardization", cols, params)
    excluded = [c for c, p in zip(cols, params) if len(p) == 0 or round(p[0], 5) == round(p[2], 5)]
    if excluded:
        warnings.warn("The following column(s) are excluded from standardization because the 75th and 25th percentiles "
                      "are the same:" + str(excluded))
    outs = {c: _divide(table, c, p[1], p[2] - p[0]) for c, p in zip(cols, params) if c not in excluded}
    return _out(table, cols, outs, output_mode), params, excluded


def minmax(table, c):
    """MinMaxScaler's Summarizer min / max of one feature: NaN (and null, assembled as NaN) skipped."""
    x, valid = _values(table, c)
    x = x[valid].astype(np.float64)
    x = x[~np.isnan(x)]
    if x.size == 0:
        return DOUBLE_MAX, -DOUBLE_MAX
    return float(x.min()), float(x.max())


def minmax_transform(x, valid, mn, mx, lo=0.0, hi=1.0):
    """MinMaxScalerModel.transform of one feature, the FloatType cast, then NaN -> null: (float32 values, bool valid)."""
    v = np.where(valid, np.asarray(x).astype(np.float64), np.nan)       # handleInvalid="keep": null -> NaN
    rng = mx - mn
    scale = (hi - lo) / rng if rng != 0 else 0.0
    with np.errstate(all="ignore"):
        if scale != 0:
            out = (v - mn) * scale + lo
        else:
            out = np.where(np.isnan(v), np.nan, 0.5 * (hi - lo) + lo)
        f = out.astype(np.float32)
    ok = ~np.isnan(f)
    f[~ok] = 0
    return f, ok


def normalization(table, list_of_cols="all", drop_cols=[], pre_existing_model=False, model_path="NA",
                  output_mode="replace"):
    cols = _cols(table, list_of_cols, drop_cols, output_mode, "Normalization")
    if cols is None:
        return table, [], []
    if pre_existing_model:
        lo, hi, mins, maxs = read_minmax_model(model_path)
        if len(mins) != len(cols):
            raise ValueError("model size")
    else:
        lo, hi = 0.0, 1.0
        mins, maxs = zip(*[minmax(table, c) for c in cols])
        if model_path != "NA":
            write_minmax_model(model_path, mins, maxs)
    outs = {}
    for c, mn, mx in zip(cols, mins, maxs):
        x, valid = _values(table, c)
        f, ok = minmax_transform(x, valid, mn, mx, lo, hi)
        outs[c] = pa.array(f, mask=~ok)
    return _out(table, cols, outs, output_mode), [list(p) for p in zip(mins, maxs)], []
