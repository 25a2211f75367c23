"""TEST INFRASTRUCTURE: the oracle of invalidEntries_detection (reference data_analyzer/quality_checker.py:1342-1711) on
pyarrow Tables, written from the reference row by row with pandas, independently of the product's code.

    invalidEntries_detection(table, ...) -> (pyarrow Table, odf_print as pandas, list of columns handed to imputation_MMM)

Restated:
  - `detect` runs per row over the values Spark hands a Python UDF (str / int / float, None for null); the rows of a
    column are judged on their own (the product's rule; the reference's UDF can append two flags for one value in
    manual / both mode and shift later columns, DESIGN.md section 1);
  - invalid_entries = the distinct raw values of the flagged rows as str(x), joined by "|", in first-seen row order
    (compare them as sets); invalid_count = flagged rows; invalid_pct = Python's round(count / rows, 4);
  - treatments: null_replacement / MMM null the flagged rows (replace: the column moves to the end; append: <c>_invalid,
    dropped again when its rounded pct is 0.0), with a threshold only the columns whose pct exceeds it; MMM then drops
    the columns with fewer than 2 distinct values and runs imputation_MMM; column_removal drops the columns over the
    threshold.  `treatment_threshold` is popped from treatment_configs and tested by truthiness.
"""
from __future__ import annotations

import re
import warnings

import pandas as pd
import pyarrow as pa

NULL_VOCAB = ["", " ", "nan", "null", "na", "inf", "n/a", "not defined", "none", "undefined", "blank", "unknown"]
SPECIAL_CHARS_VOCAB = ["&", "$", ";", ":", ".", ",", "*", "#", "@", "_", "?", "%", "!", "^", "(", ")", "-", "/", "'"]
PRINT_COLS = ["attribute", "invalid_entries", "invalid_count", "invalid_pct"]


def detect(v, detection_type="auto", invalid_entries=(), valid_entries=(), partial_match=False):
    """reference :1540-1607 for one value -> None (null), 1 (invalid) or 0.  The reference appends a second 1 for a value
    that matches an invalid pattern and misses every valid pattern; for one column that is still the verdict 1."""
    e = v
    if e is None:
        return None
    if detection_type in ("auto", "both"):
        e = str(e).lower().strip()
        if e in (NULL_VOCAB + SPECIAL_CHARS_VOCAB):
            return 1
        if re.search(re.compile("\\b([a-zA-Z0-9])\\1\\1+\\b"), e):
            return 1
        n = len(e)
        if n >= 3:
            check = 0
            for i in range(1, n):
                if ord(e[i]) - ord(e[i - 1]) != 1:
                    check = 1
                    break
            if check == 0:
                return 1
    check = 0
    if detection_type in ("manual", "both"):
        e = str(e).lower().strip()
        for regex in invalid_entries:
            p = re.compile(regex)
            if (re.search(p, e) if partial_match else p.fullmatch(e)):
                check = 1
                break
        match_valid = []
        for regex in valid_entries:
            p = re.compile(regex)
            match_valid.append(1 if (re.search(p, e) if partial_match else p.fullmatch(e)) else 0)
        if len(match_valid) > 0 and sum(match_valid) == 0:
            check = 1
    return 1 if check else 0


def _sdtype(t):
    if pa.types.is_string(t) or pa.types.is_large_string(t) or pa.types.is_dictionary(t):
        return "string"
    if pa.types.is_int32(t):
        return "int"
    if pa.types.is_int64(t):
        return "bigint"
    if pa.types.is_float32(t):
        return "float"
    if pa.types.is_float64(t):
        return "double"
    return str(t)


def _split(x):
    return [s.strip() for s in x.split("|")] if isinstance(x, str) else list(x)


def invalidEntries_detection(table, list_of_cols="all", drop_cols=[], detection_type="auto", invalid_entries=[],
                             valid_entries=[], partial_match=False, treatment=False, treatment_method="null_replacement",
                             treatment_configs={}, output_mode="replace", impute=None):
    """-> (odf Table, odf_print pandas, columns handed to imputation_MMM or None).  impute(table, cols, **configs) runs
    the MMM imputation (tests pass the imputation oracle); None returns the null-replaced frame and the column list."""
    if list_of_cols == "all":
        list_of_cols = [f.name for f in table.schema if _sdtype(f.type) in ("string", "int", "bigint", "long")]
    cols = list(dict.fromkeys(c for c in _split(list_of_cols) if c not in _split(drop_cols)))
    if any(c not in table.column_names for c in cols):
        raise TypeError("Invalid input for Column(s)")
    if not cols:
        warnings.warn("No Invalid Entries Check - No discrete column(s) to analyze")
        return table, pd.DataFrame(columns=PRINT_COLS), None
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")
    if str(treatment).lower() == "true":
        treatment = True
    elif str(treatment).lower() == "false":
        treatment = False
    else:
        raise TypeError("Non-Boolean input for treatment")
    if treatment_method not in ("MMM", "null_replacement", "column_removal"):
        raise TypeError("Invalid input for method_type")
    threshold = treatment_configs.pop("treatment_threshold", None)
    if threshold:
        threshold = float(threshold)
    elif treatment_method == "column_removal":
        raise TypeError("Invalid input for column removal threshold")

    n = table.num_rows
    flags, rows = {}, []
    for c in cols:
        vals = table.column(c).to_pylist()
        f = [detect(v, detection_type, invalid_entries, valid_entries, partial_match) for v in vals]
        flags[c] = f
        hit = list(dict.fromkeys(str(v) for v, x in zip(vals, f) if x == 1))
        cnt = sum(1 for x in f if x == 1)
        rows.append([c, "|".join(hit), cnt, round(cnt / n, 4)])
    odf_print = pd.DataFrame(rows, columns=PRINT_COLS)
    if not treatment:
        return table, odf_print, None
    pct = dict(zip(odf_print["attribute"], odf_print["invalid_pct"]))
    threshold_cols = [c for c in cols if pct[c] > threshold] if threshold else []
    if treatment_method == "column_removal":
        return table.drop(threshold_cols), odf_print, None
    names, arrays = list(table.column_names), [table.column(c) for c in table.column_names]
    for c in cols:
        if threshold and c not in threshold_cols:
            continue
        vals = table.column(c).to_pylist()
        new = pa.array([None if x == 1 else v for v, x in zip(vals, flags[c])], table.column(c).type)
        if output_mode == "replace":
            k = names.index(c)
            del names[k], arrays[k]
            names.append(c)
            arrays.append(new)
        elif pct[c] != 0.0:
            names.append(c + "_invalid")
            arrays.append(new)
    odf = pa.table(arrays, names=names)
    if treatment_method == "null_replacement":
        return odf, odf_print, None
    uniq = {c: len({v for v in odf.column(c).to_pylist() if v is not None}) for c in cols}
    remove = {c for c in cols if uniq[c] < 2}
    sub = [c for c in cols if c not in remove]
    if threshold:
        sub = [c for c in threshold_cols if c not in remove]
    if output_mode == "append" and sub:
        sub = [c + "_invalid" for c in sub]
    if impute is not None:
        odf = impute(odf, sub, **treatment_configs)
    return odf, odf_print, sub
