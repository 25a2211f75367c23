"""Oracle restatement of the reference's row-level quality checks on pyarrow Tables, returning what the reference
returns (the treated table and a pandas stats frame with the reference's column names).
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Follows (relative to /root/reference/src/main/anovos):
  data_analyzer/quality_checker.py:49-149   (duplicate_detection)
  data_analyzer/quality_checker.py:152-283  (nullRows_detection)
"""
from __future__ import annotations

import warnings

import numpy as np
import pandas as pd
import pyarrow as pa

from . import spark_semantics as S
from .api import _resolve

R = S.round_half_up


def _row_default(table):
    num, cat, _ = S.segregate(table)
    return num + cat


def row_group_keys(table, cols):
    """pandas frame of the normalised values of `cols`, one column per input column, for `duplicated()`: null -> None
    (equal to null, different from every value, whatever the data under the lane), every NaN -> one NaN value, -0.0 ->
    0.0 (Spark >= 3 grouping), numbers by their bits, strings by value."""
    out = {}
    for c in cols:
        arr = table.column(c).combine_chunks()
        if pa.types.is_dictionary(arr.type):
            arr = arr.cast(arr.type.value_type)
        valid = np.asarray(arr.is_valid())
        if pa.types.is_string(arr.type) or pa.types.is_large_string(arr.type):
            vals = np.array(arr.to_pylist(), dtype=object)
        else:
            if pa.types.is_decimal(arr.type):
                arr = arr.cast(pa.float64())
            x = np.asarray(arr.fill_null(0).to_numpy(zero_copy_only=False))
            if x.dtype.kind == "f":
                with np.errstate(invalid="ignore"):
                    x64 = x.astype(np.float64) + 0.0
                x64[np.isnan(x64)] = np.nan
                vals = np.where(np.isnan(x64), "nan", x64.view(np.int64).astype(str)).astype(object)
            else:
                vals = x.astype(np.int64).astype(object)
        vals = vals.astype(object)
        vals[~valid] = None
        out[c] = vals
    return pd.DataFrame(out, columns=list(cols))


def first_occurrence(table, cols):
    """bool [n_rows]: the first row of every group of equal rows (pandas ~duplicated(keep="first"))."""
    if table.num_rows == 0:
        return np.zeros(0, bool)
    return ~row_group_keys(table, cols).duplicated(keep="first").to_numpy()


def duplicate_detection(table, list_of_cols="all", drop_cols=[], treatment=True, print_impact=False):
    """-> table | (table, stats) like the reference; the treated table keeps the first occurrences in row order."""
    if not treatment and not print_impact:
        warnings.warn("The original idf will be the only output. Set print_impact=True to perform detection without treatment")
        return table
    cols = _resolve(table, list_of_cols, drop_cols, _row_default(table))
    if str(treatment).lower() not in ("true", "false"):
        raise TypeError("Non-Boolean input for treatment")
    treatment = str(treatment).lower() == "true"
    keep = first_occurrence(table, cols)
    n, u = table.num_rows, int(keep.sum())
    odf = table.select(cols).filter(pa.array(keep)) if treatment else table
    if not print_impact:
        return odf
    stats = pd.DataFrame([["rows_count", float(n)], ["unique_rows_count", float(u)], ["duplicate_rows", float(n - u)],
                          ["duplicate_pct", round((n - u) / n, 4)]], columns=["metric", "value"])
    return odf, stats


def row_null_counts(table, cols):
    """int64 [n_rows]: null columns of each row among `cols` (NaN is a value)."""
    cnt = np.zeros(table.num_rows, np.int64)
    for c in cols:
        cnt += ~np.asarray(table.column(c).combine_chunks().is_valid())
    return cnt


def nullRows_detection(table, list_of_cols="all", drop_cols=[], treatment=False, treatment_threshold=0.8, print_impact=False):
    """-> (table, stats [null_cols_count, row_count, row_pct, flagged | treated])."""
    cols = _resolve(table, list_of_cols, drop_cols, _row_default(table))
    if str(treatment).lower() not in ("true", "false"):
        raise TypeError("Non-Boolean input for treatment")
    treatment = str(treatment).lower() == "true"
    treatment_threshold = float(treatment_threshold)
    if treatment_threshold < 0 or treatment_threshold > 1:
        raise TypeError("Invalid input for Treatment Threshold Value")
    cnt = row_null_counts(table, cols)
    flagged = cnt > len(cols) * treatment_threshold
    if treatment_threshold == 1:
        flagged = cnt == len(cols)
    ks, rows = np.unique(cnt, return_counts=True)
    flag_of = {int(k): int(f) for k, f in zip(cnt.tolist(), flagged.tolist())}
    name = "treated" if treatment else "flagged"
    stats = pd.DataFrame({"null_cols_count": [int(k) for k in ks], "row_count": [int(r) for r in rows],
                          "row_pct": [R(int(r) / float(table.num_rows)) for r in rows],
                          name: [flag_of[int(k)] for k in ks]}, columns=["null_cols_count", "row_count", "row_pct", name])
    odf = table.filter(pa.array(~flagged)) if treatment else table
    return odf, stats
