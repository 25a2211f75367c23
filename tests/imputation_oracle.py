"""TEST INFRASTRUCTURE: the oracle of imputation_MMM (reference data_transformer/transformers.py:1369-1676) on pyarrow
Tables, written from the reference and Spark ML's Imputer with NumPy, independently of the product's code.

    imputation_MMM(table, ...) -> (pyarrow Table, before / after impact table as pandas | None)

Spark semantics restated:
  - numeric columns that are not float / double are recast to double before anything else (:1496-1502);
  - "mean" / "median" (Imputer, Spark 3.x): NaN counts as missing; mean = avg, median = approxQuantile(0.5, 0.001)
    (the GK sketch, merged over the table's Spark partitions when it is tagged with them); no value left: an error;
    transform `when(ic.isNull, s).when(ic == NaN, s).otherwise(ic).cast(inputType)`, then `_imputed` cast back from
    double with Java's d2i / d2l;
  - "mode" and categorical columns: the most frequent non-null value (ties: the smallest), filled where null only;
    str(None) = "None" for an all-null categorical column.  Numeric mode outputs stay numbers in the recast type
    (the product's documented deviation from the reference's string columns);
  - only columns with nulls keep their `_imputed`; "replace" drops the original and renames, at the end of the frame.
"""
from __future__ import annotations

import csv
import json
import math
import os
import warnings

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.parquet as pq

from oracle import api as O
from oracle import spark_semantics as S

REL_ERR = 0.001


def d2i(x):
    if x != x:
        return 0
    if x >= 2147483647.0:
        return 2147483647
    if x <= -2147483648.0:
        return -2147483648
    return int(x)


def d2l(x):
    if x != x:
        return 0
    if x >= 9.223372036854775807e18:
        return (1 << 63) - 1
    if x <= -9.223372036854775808e18:
        return -(1 << 63)
    return int(x)


def cast_double(x, sdtype):
    """Spark's cast of a double to the column type."""
    if sdtype == "double":
        return float(x)
    if sdtype == "float":
        with np.errstate(over="ignore"):
            return float(np.float32(x))
    if sdtype == "int":
        return d2i(float(x))
    return d2l(float(x))


_PA = {"double": pa.float64(), "float": pa.float32(), "int": pa.int32(), "bigint": pa.int64(), "long": pa.int64()}


def _values(table, c):
    arr = table.column(c).combine_chunks()
    if pa.types.is_dictionary(arr.type):
        arr = arr.cast(arr.type.value_type)
    valid = np.asarray(arr.is_valid())
    if pa.types.is_string(arr.type):
        return np.array(arr.to_pylist(), dtype=object), valid
    vals = (arr.fill_null(0) if arr.null_count else arr).to_numpy(zero_copy_only=False)
    return vals, valid


def _nan_free(table, c):
    """The table with NaN of column c turned into null (Imputer's `when(isnan(x), null)`), Spark partition tags kept."""
    vals, valid = _values(table, c)
    keep = valid & ~np.isnan(vals.astype(np.float64)) if vals.dtype.kind == "f" else valid
    return table.set_column(table.column_names.index(c), c, pa.array(vals, mask=~keep))


def surrogate(table, c, method_type):
    t = _nan_free(table, c)
    vals, valid = _values(t, c)
    x = vals[valid].astype(np.float64)
    if x.size == 0:
        raise ValueError("surrogate cannot be computed. All the values in %s are Null, Nan or missingValue(NaN)" % c)
    if method_type == "mean":
        return float(np.sum(x) / x.size)
    return float(O.ColumnProfile(t, c).quantile(0.5, REL_ERR))


def mode_value(table, c):
    """groupBy(c).count() over dropna (null and NaN dropped) -> most frequent value, ties -> smallest; None if empty."""
    vals, valid = _values(table, c)
    x = vals[valid]
    if x.dtype.kind == "f":
        x = x[~np.isnan(x)] + 0.0
    if x.size == 0:
        return None
    if x.dtype == object:
        u, k = np.unique(x.astype(str), return_counts=True)
        best = min(u[k == k.max()].tolist(), key=lambda s: s.encode("utf-8"))
        return best
    u, k = np.unique(x, return_counts=True)
    return u[int(np.argmax(k))].item()


def missing_counts(table):
    num, cat, _ = S.segregate(table)
    return pd.DataFrame([[c, table.num_rows - int(np.asarray(table.column(c).is_valid()).sum())] for c in num + cat],
                        columns=["attribute", "missing_count"])


def fill_reference(vals, valid, out_dtype, nan_missing, round_double, fill):
    """Exact NumPy image of one anv_impute_fill column: keep = valid and not (nan_missing and NaN); kept rows converted
    (bigint under round_double: (long)(double)x with d2l saturation), the others `fill` (already in out_dtype)."""
    vals = np.asarray(vals)
    keep = np.asarray(valid, bool).copy()
    if nan_missing:
        keep &= ~np.isnan(vals)
    out_dtype = np.dtype(out_dtype)
    if round_double and vals.dtype == np.int64:
        f = vals.astype(np.float64)
        big = f >= 2.0 ** 63
        conv = np.where(big, 0.0, f).astype(np.int64)
        conv[big] = np.iinfo(np.int64).max
    else:
        conv = vals.astype(out_dtype)
    out = conv.copy()
    out[~keep] = np.array([fill], dtype=out_dtype)[0]
    return out


# ---- models (Spark's layouts) -------------------------------------------------------------------------------------

def _parts(d):
    return sorted(os.path.join(d, f) for f in os.listdir(d) if f.startswith("part-") and not f.endswith(".crc"))


def read_num_model(model_path):
    d = os.path.join(model_path, "imputation_MMM", "num_imputer-model")
    meta = json.loads(open(_parts(os.path.join(d, "metadata"))[0]).readline())
    ins, outs = meta["paramMap"]["inputCols"], meta["paramMap"]["outputCols"]
    t = pa.concat_tables([pq.read_table(f) for f in _parts(os.path.join(d, "data")) if f.endswith(".parquet")])
    return ins, outs, {c: float(t.column(c)[0].as_py()) for c in ins}


def write_num_model(model_path, ins, outs, strategy, sur):
    d = os.path.join(model_path, "imputation_MMM", "num_imputer-model")
    for sub in ("metadata", "data"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    with open(os.path.join(d, "metadata", "part-00000"), "w") as f:
        f.write(json.dumps({"class": "org.apache.spark.ml.feature.ImputerModel",
                            "paramMap": {"strategy": strategy, "inputCols": ins, "outputCols": outs}}) + "\n")
    pq.write_table(pa.table({c: [float(sur[c])] for c in ins}), os.path.join(d, "data", "part-00000.parquet"))


def read_cat_model(model_path):
    d = os.path.join(model_path, "imputation_MMM", "cat_imputer")
    rows = []
    for f in _parts(d):
        rows += [(a, p or None) for a, p in list(csv.reader(open(f, newline=""), doublequote=False, escapechar="\\"))[1:]]
    return rows


def write_cat_model(model_path, cols, params):
    d = os.path.join(model_path, "imputation_MMM", "cat_imputer")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "part-00000.csv"), "w", newline="") as f:
        w = csv.writer(f, doublequote=False, escapechar="\\", lineterminator="\n")
        w.writerow(["attribute", "parameters"])
        for c, p in zip(cols, params):
            w.writerow([c, "" if p is None else p])


# ---- imputation_MMM ---------------------------------------------------------------------------------------------

def imputation_MMM(table, list_of_cols="missing", drop_cols=[], method_type="median", pre_existing_model=False,
                   model_path="NA", output_mode="replace", stats_missing=None, stats_mode=None):
    """stats_missing: pandas [attribute, missing_count] or None; stats_mode: pandas [attribute, mode] or None."""
    missing_df = missing_counts(table) if stats_missing is None else stats_missing
    missing_cols = missing_df.loc[missing_df["missing_count"] > 0, "attribute"].tolist()
    if str(pre_existing_model).lower() not in ("true", "false"):
        raise TypeError("Non-Boolean input for pre_existing_model")
    pre = str(pre_existing_model).lower() == "true"
    if not missing_cols and not pre and model_path == "NA":
        return table, None
    num_all, cat_all, _ = S.segregate(table)
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num_all + cat_all
    if isinstance(list_of_cols, str) and list_of_cols == "missing":
        list_of_cols = [x for x in missing_cols if x in num_all + cat_all]
    if isinstance(list_of_cols, str):
        list_of_cols = [x.strip() for x in list_of_cols.split("|")]
    if isinstance(drop_cols, str):
        drop_cols = [x.strip() for x in drop_cols.split("|")]
    list_of_cols = [c for c in dict.fromkeys(list_of_cols) if c not in drop_cols]
    if not list_of_cols:
        warnings.warn("No Imputation performed- No column(s) to impute")
        return table, None
    if any(x not in num_all + cat_all for x in list_of_cols):
        raise TypeError("Invalid input for Column(s)")
    if method_type not in ("mode", "mean", "median"):
        raise TypeError("Invalid input for method_type")
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")
    types = dict(zip(table.column_names, [S.spark_dtype(f.type) for f in table.schema]))
    num_cols = [c for c in list_of_cols if c in num_all]
    cat_cols = [c for c in list_of_cols if c in cat_all]
    saved_mode = None
    if stats_mode is not None:
        saved_mode = {}
        for a, m in zip(stats_mode["attribute"], stats_mode["mode"]):
            saved_mode.setdefault(a, []).append(None if m is None or str(m) in ("None", "nan") else str(m))

    cols = {n: table.column(n) for n in table.column_names}       # odf, insertion-ordered
    recast = [c for c in num_cols if types[c] not in ("float", "double")]
    for c in recast:
        cols[c] = table.column(c).cast(pa.float64(), safe=False)
    created = {}

    def add(name, vals, valid, pa_type):
        created[name] = pa.array(vals, type=pa_type, mask=~valid)

    if num_cols:
        if method_type == "mode":
            for c in num_cols:
                if saved_mode is not None and c in saved_mode:
                    p = None if saved_mode[c][0] is None else float(saved_mode[c][0])
                else:
                    m = mode_value(table, c)
                    p = None if m is None else float(m)
                out_t = "float" if types[c] == "float" else "double"
                x, valid = _values(table, c)
                x = x.astype(np.float32 if out_t == "float" else np.float64)
                if p is None:
                    add(c + "_imputed", x, valid, _PA[out_t])
                else:
                    add(c + "_imputed", np.where(valid, x, cast_double(p, out_t)).astype(x.dtype), np.ones(len(x), bool),
                        _PA[out_t])
        else:
            if pre:
                ins, outs, sur = read_num_model(model_path)
            else:
                ins, outs = num_cols, [c + "_imputed" for c in num_cols]
                sur = {c: surrogate(table, c, method_type) for c in num_cols}
                if model_path != "NA":
                    write_num_model(model_path, ins, outs, method_type, sur)
            for c, o in zip(ins, outs):
                t = types[c]
                x, valid = _values(table, c)
                ic = x.astype(np.float64)                                   # ic = double(x)
                miss = ~valid | np.isnan(ic)
                if t in ("float", "double"):
                    out = np.where(miss, sur[c], ic).astype(np.float32 if t == "float" else np.float64)
                else:                                                       # cast back: d2i / d2l
                    fill = cast_double(sur[c], t)
                    back = np.array([cast_double(v, t) for v in ic.tolist()], dtype=object) if t != "int" else x
                    out = np.where(miss, fill, back)
                add(o, out.tolist() if out.dtype == object else out, np.ones(len(x), bool), _PA[t])
            for c in recast:
                if c + "_imputed" not in created:
                    raise ValueError("cannot resolve '%s_imputed'" % c)

    if cat_cols:
        if pre:
            model = read_cat_model(model_path)
            params = []
            for c in cat_cols:
                hit = [p for a, p in model if a == c]
                if not hit:
                    raise IndexError("list index out of range")
                params.append(hit[0])
        elif saved_mode is None:
            params = [str(mode_value(table, c)) for c in cat_cols]
        else:
            params = []
            for c in cat_cols:
                if c not in saved_mode:
                    raise IndexError("list index out of range")
                params.append(saved_mode[c][0])
        for c, p in zip(cat_cols, params):
            x, valid = _values(table, c)
            vals = [v if ok else p for v, ok in zip(x.tolist(), valid.tolist())]
            created[c + "_imputed"] = pa.array(vals, type=pa.string())
        if not pre and model_path != "NA":
            write_cat_model(model_path, cat_cols, params)

    for i in num_cols + cat_cols:
        if i not in missing_cols:
            created.pop(i + "_imputed", None)
        elif output_mode == "replace":
            cols.pop(i)
            if i + "_imputed" in created:
                created[i] = created.pop(i + "_imputed")
    names = list(cols) + list(created)
    odf = pa.table([cols[n] if n in cols else created[n] for n in names], names=names)

    before = dict(zip(missing_df["attribute"], missing_df["missing_count"]))
    if output_mode == "replace":
        rows = [[a, int(before[a]), odf.num_rows - int(np.asarray(odf.column(a).is_valid()).sum())]
                for a in list_of_cols if a in before]
        impact = ["attribute", "missingCount_before", "missingCount_after"]
    else:
        outs_ = [i + "_imputed" for i in num_cols + cat_cols if i in missing_cols]
        rows = [[a[:-8], int(before[a[:-8]]), a, odf.num_rows - int(np.asarray(odf.column(a).is_valid()).sum())]
                for a in outs_ if a[:-8] in before]
        impact = ["attribute", "missingCount_before", "attribute_after", "missing_count"]
    rows.sort(key=lambda r: r[0])
    return odf, pd.DataFrame(rows, columns=impact)


def nullColumns_detection_MMM(table, list_of_cols="missing", drop_cols=[], treatment_configs={}, stats_unique=None,
                              stats_mode=None):
    """quality_checker.py:491-519 (treatment=True, treatment_method="MMM") -> (table, impact)."""
    num_all, cat_all, _ = S.segregate(table)
    md = missing_counts(table)
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num_all + cat_all
    if isinstance(list_of_cols, str) and list_of_cols == "missing":
        list_of_cols = md.loc[md["missing_count"] > 0, "attribute"].tolist()
    cols = [c for c in dict.fromkeys(O._split(list_of_cols)) if c not in O._split(drop_cols)]
    cfg = dict(treatment_configs)
    thr = cfg.pop("treatment_threshold", None)
    N = table.num_rows
    if stats_unique is None:
        uq = {c: len(set(x for x, ok in zip(*_values(table, c)) if ok)) for c in cols}
    else:
        uq = dict(zip(stats_unique["attribute"], stats_unique["unique_values"]))
    remove = [c for c in uq if uq[c] < 2]
    sub = [c for c in cols if c not in remove]
    if thr:
        pct = {a: S.round_half_up(m / N) for a, m in zip(md["attribute"], md["missing_count"])}
        sub = [c for c in cols if pct[c] > float(thr) and c not in remove]
    return imputation_MMM(table, sub, **cfg, stats_mode=stats_mode)
