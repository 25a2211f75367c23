"""TEST INFRASTRUCTURE: the oracle of monotonic_binning (reference data_transformer/transformers.py:294-425) and of the
monotonicity check of IV / IG (data_analyzer/association_evaluator.py:350-357) on pyarrow Tables, written from the
reference row by row with pandas and scipy on top of oracle.api's attribute_binning, independently of the product's code.

    monotonic_binning(table, ...) -> pyarrow Table;  chosen_bins(table, ...) -> {col: accepted n or None}
    IV_calculation / IG_calculation(table, ..., encoding_configs={..., "monotonicity_check": 1}) -> pandas, through
    oracle.api's IV_calculation / IG_calculation on the binned table

Restated per column, n = 20 .. 3: bin the INPUT table with attribute_binning(bin_size=n, output_mode="append"), recode
the label as 1 if label == event_label else 0 (a null label is 0), groupBy(binned).agg(avg(x), avg(label01)).dropna()
with the real avg(x) (null group, NaN averages dropped), and accept n iff scipy.stats.spearmanr gives exactly 1.0.  An
equal_range column without a non-null value has no `_binned` column: ValueError, as the product raises.
"""
from __future__ import annotations

import warnings

import numpy as np
import pandas as pd
from scipy import stats

from oracle import api as O
from oracle import spark_semantics as S

LADDER = tuple(range(20, 2, -1))


def _label01(table, label_col, event_label):
    vals, valid = S.column_values(table, label_col)
    if vals.dtype == object:
        ev = valid & (vals.astype(str) == str(event_label))
    else:
        ev = valid & (vals.astype(np.float64) == float(event_label))
    return ev.astype(np.int64)


def accepted(table, col, label_col, event_label, bin_method, n):
    """The reference's test of one n: r == 1.0 of spearmanr over the groupBy table."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        binned = O.attribute_binning(table, [col], method_type=bin_method, bin_size=n, output_mode="append")
    if col + "_binned" not in binned.column_names:
        raise ValueError("monotonic_binning: column %r holds no non-null value" % col)
    ids, ok = S.column_values(binned, col + "_binned")
    vals, valid = S.column_values(table, col)
    df = pd.DataFrame({"b": np.where(ok, ids, -1), "x": np.where(valid, vals.astype(np.float64), np.nan),
                       "y": _label01(table, label_col, event_label).astype(np.float64)})
    df = df[ok]                                              # the null group averages to null and is dropped
    with np.errstate(all="ignore"):
        tmp = df.groupby("b").agg(mean_val=("x", "mean"), mean_label=("y", "mean")).dropna()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        r, _ = stats.spearmanr(tmp[["mean_val"]], tmp[["mean_label"]])
    return r == 1.0


def chosen_bins(table, cols, label_col, event_label, bin_method):
    out = {}
    for c in cols:
        out[c] = next((n for n in LADDER if accepted(table, c, label_col, event_label, bin_method, n)), None)
    return out


def _cols(table, list_of_cols, drop_cols, label_col):
    num = S.segregate(table)[0]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num
    cols = O._dedupe(O._split(list_of_cols), O._split(drop_cols) + [label_col])
    if any(c not in num for c in cols):
        raise TypeError("Invalid input for Column(s)")
    return cols


def monotonic_binning(table, list_of_cols="all", drop_cols=[], label_col="label", event_label=1, bin_method="equal_range",
                      bin_size=10, bin_dtype="numerical", output_mode="replace"):
    cols = _cols(table, list_of_cols, drop_cols, label_col)
    chosen = chosen_bins(table, cols, label_col, event_label, bin_method)
    out = table
    for c in cols:
        n = chosen[c] if chosen[c] is not None else bin_size
        # the reference bins the partly transformed table: column c itself is still the input's
        out = O.attribute_binning(out, [c], method_type=bin_method, bin_size=n, bin_dtype=bin_dtype, output_mode=output_mode)
    return out


def _encoded(table, cols, label_col, event_label, encoding_configs):
    """idf_encoded of association_evaluator.py:350-357: the numeric attributes of `cols` binned by monotonic_binning."""
    num = [c for c in cols if c in S.segregate(table)[0]]
    if not num:
        return table
    return monotonic_binning(table, num, [], label_col, event_label, encoding_configs["bin_method"],
                             encoding_configs["bin_size"])


def IV_calculation(table, list_of_cols="all", drop_cols=[], label_col="label", event_label=1, encoding_configs=None):
    """oracle.api.IV_calculation over the binned table: without encoding_configs it groups every attribute by its value,
    as the reference groups idf_encoded."""
    cols = O._iv_ig_cols(table, list_of_cols, drop_cols, label_col, event_label)[0]
    enc = _encoded(table, cols, label_col, event_label, encoding_configs)
    return O.IV_calculation(enc, cols, [], label_col, event_label, encoding_configs={})


def IG_calculation(table, list_of_cols="all", drop_cols=[], label_col="label", event_label=1, encoding_configs=None):
    cols = O._iv_ig_cols(table, list_of_cols, drop_cols, label_col, event_label)[0]
    enc = _encoded(table, cols, label_col, event_label, encoding_configs)
    return O.IG_calculation(enc, cols, [], label_col, event_label, encoding_configs={})
