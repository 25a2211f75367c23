"""Consumers of the stats hot path from `anovos.data_analyzer.quality_checker` (SURVEY.md 8f, row
N2), same signatures and outputs as the reference
(/root/reference/src/main/anovos/data_analyzer/quality_checker.py):
  duplicate_detection   :49-149   (rows: hash, sort and exact comparison on the device - csrc/rows.cu)
  nullRows_detection    :152-283  (rows: per-row null counts from the validity bitmaps - csrc/rows.cu)
  nullColumns_detection :286-547  (treatment: none / row_removal / column_removal)
  outlier_detection     :550-1045
  IDness_detection      :1048-1182
  biasedness_detection  :1185-1339
  invalidEntries_detection :1342-1711 (per-value rules on the host once per distinct value, one table-membership pass
                        on the device that counts and nulls the flagged rows - csrc/invalid.cu)
Each returns (odf, odf_print) where the reference does.  The per-row work (row null counts, distinct rows, null counts,
distinct counts, modes, percentile / moment thresholds, the outlier compare pass) runs in the CUDA kernels.  The imputation
treatments KNN / regression / MF / auto are not part of this build."""
from __future__ import annotations

import math
import os
import warnings
from collections import OrderedDict

import numpy as np
import pandas as pd

from .. import _lib, engine, profile
from ..frame import Column, ColumnFrame, as_frame, pack_bits_device
from ..result import ResultFrame
from ..shared.utils import attributeType_segregation, jvm_double_str, names, spark_round, unique
from .stats_generator import _mode_str, measures_of_cardinality, missingCount_computation


def _as_bool(v, what):
    if str(v).lower() == "true":
        return True
    if str(v).lower() == "false":
        return False
    raise TypeError("Non-Boolean input for " + what)


def _read_stats(spec, columns):
    """read_dataset(spark, **stats_x): file_path + file_type (csv / parquet) of a saved stats frame."""
    path, ftype = spec["file_path"], spec.get("file_type", "csv")
    import os
    if os.path.isdir(path):
        files = sorted(os.path.join(path, f) for f in os.listdir(path) if f.endswith("." + ftype))
    else:
        files = [path]
    df = pd.concat([pd.read_csv(f) if ftype == "csv" else pd.read_parquet(f) for f in files], ignore_index=True)
    return df[columns]


# ---- row-level checks ----------------------------------------------------------------------------------

def _row_cols(fr, list_of_cols, drop_cols):
    """reference :103-114 / :224-235: "all" = numeric + categorical; an unknown name or an empty list is an error."""
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        num, cat, _ = attributeType_segregation(fr)
        list_of_cols = num + cat
    cols = unique(names(list_of_cols), names(drop_cols))
    known = set(fr.columns)
    if any(c not in known for c in cols) or len(cols) == 0:
        raise TypeError("Invalid input for Column(s)")
    other = [c for c in cols if fr.column(c).kind == "other"]
    if other:
        raise TypeError("Column(s) %s have dtypes the GPU path does not hold (%s); row-level checks take numeric and "
                        "string columns" % (",".join(other), ",".join(fr.column(c).sdtype for c in other)))
    return cols


def _canonical_codes(fr, cols):
    """A frame whose string columns compare by code: a dictionary that repeats a string (a dictionary-typed Arrow input
    can) has its codes mapped to the string's first code.  Other columns pass through untouched."""
    out, changed = OrderedDict(), False
    for c in cols:
        col = fr.column(c)
        dic = col.dictionary
        if dic is not None and len(set(dic)) != len(dic):
            torch = _lib.require_cuda()
            first = {}
            canon = np.array([first.setdefault(s, i) for i, s in enumerate(dic)], dtype=np.int32)
            d, v = col.device()
            lut = torch.from_numpy(canon).to(d.device)
            codes = lut[d.long().clamp(0, len(dic) - 1)].to(torch.int32).contiguous()   # codes under null lanes are ignored
            col = Column(c, col.sdtype, fr.n_rows, dev=codes, dev_valid=v, anv_dtype=_lib.ANV_I32, dictionary=dic)
            changed = True
        out[c] = col
    return ColumnFrame(out, fr.n_rows) if changed else fr


def duplicate_detection(spark, idf, list_of_cols="all", drop_cols=[], treatment=True, print_impact=False):
    """reference :49-149.  Rows are grouped exactly on the device: a hash of each row's normalised values, an LSD sort of
    (hash prefix, row) and a comparison of every row with its group's first row (csrc/rows.cu).  Nulls group together,
    every NaN is one value and -0.0 == 0.0 (Spark 3 grouping).  The treated frame holds the `list_of_cols` columns of
    the first occurrence of every distinct row, in row order (Spark's row and column order there is arbitrary)."""
    fr = as_frame(idf)
    if not treatment and not print_impact:
        warnings.warn("The original idf will be the only output. Set print_impact=True to perform detection without treatment")
        return fr
    cols = _row_cols(fr, list_of_cols, drop_cols)
    treatment = _as_bool(treatment, "treatment")
    if getattr(fr, "is_partitioned", False):
        raise NotImplementedError("duplicate_detection needs every row resident on one device to compare rows; "
                                  "materialize() the row-partitioned frame first")
    n = fr.count()
    n_unique, first = engine.row_distinct(_canonical_codes(fr, cols), cols)
    odf = fr.select(cols).filter_rows(engine.bitmap_to_bool(first, n)) if treatment else fr
    if print_impact:
        pct = round((n - n_unique) / n, 4)
        odf_print = ResultFrame(pd.DataFrame([["rows_count", float(n)], ["unique_rows_count", float(n_unique)],
                                              ["duplicate_rows", float(n - n_unique)], ["duplicate_pct", pct]],
                                             columns=["metric", "value"]))
        print("No. of Rows: " + str(n))
        print("No. of UNIQUE Rows: " + str(n_unique))
        print("No. of Duplicate Rows: " + str(n - n_unique))
        print("Percentage of Duplicate Rows: " + str(pct))
        return odf, odf_print
    return odf


def _null_rows_max_keep(n_cols, threshold):
    """Largest null count that is NOT flagged: flagged when count > n_cols * threshold (product in Python float, as the
    reference hands it to Spark), and at threshold 1 when count == n_cols (:255-264)."""
    if threshold == 1:
        return n_cols - 1
    return min(int(math.floor(n_cols * threshold)), n_cols)


def nullRows_detection(spark, idf, list_of_cols="all", drop_cols=[], treatment=False, treatment_threshold=0.8,
                       print_impact=False):
    """reference :152-283.  Per-row null counts come from the validity bitmaps on the device (csrc/rows.cu); NaN is a
    value, not a null (the reference's UDF counts Python None).  A row-partitioned frame adds up the histograms of its
    chunks (and of every rank of its process group); its treatment filters each chunk lazily."""
    fr = as_frame(idf)
    cols = _row_cols(fr, list_of_cols, drop_cols)
    treatment = _as_bool(treatment, "treatment")
    treatment_threshold = float(treatment_threshold)
    if treatment_threshold < 0 or treatment_threshold > 1:
        raise TypeError("Invalid input for Treatment Threshold Value")
    max_keep = _null_rows_max_keep(len(cols), treatment_threshold)
    n = fr.count()
    odf = fr
    if getattr(fr, "is_partitioned", False):
        hist = np.zeros(len(cols) + 1, np.uint64)
        kept = []
        for ch in fr.chunks(cols):
            h, _ = engine.row_null_counts(ch, cols)
            hist += h
            kept.append(int(h[:max_keep + 1].sum()) if max_keep >= 0 else 0)
        if fr.group is not None:
            hist = fr.group.all_reduce(hist)
        if treatment:
            def drop_flagged(ch):
                _, keep = engine.row_null_counts(ch, cols, max_keep)
                return ch.filter_rows(engine.bitmap_to_bool(keep, ch.n_rows))
            odf = fr.map_chunks(fr._schema, drop_flagged)
            odf.chunk_rows = kept
            odf.n_rows_local = sum(kept)
            odf.n_rows = odf.n_rows_local
            if fr.group is not None:
                odf.n_rows = int(fr.group.all_reduce(np.array([odf.n_rows_local], np.int64))[0])
    else:
        hist, keep = engine.row_null_counts(fr, cols, max_keep if treatment else None)
        if treatment:
            odf = fr.filter_rows(engine.bitmap_to_bool(keep, n))
    ks = [k for k in range(len(cols) + 1) if int(hist[k]) > 0]
    counts = [int(hist[k]) for k in ks]
    flag = "treated" if treatment else "flagged"
    odf_print = ResultFrame(pd.DataFrame({"null_cols_count": ks, "row_count": counts,
                                          "row_pct": [spark_round(c / float(n)) for c in counts],
                                          flag: [1 if k > max_keep else 0 for k in ks]},
                                         columns=["null_cols_count", "row_count", "row_pct", flag]))
    if print_impact:
        odf_print.show(odf.count())
    return odf, odf_print


def nullColumns_detection(spark, idf, list_of_cols="missing", drop_cols=[], treatment=False, treatment_method="row_removal",
                          treatment_configs={}, stats_missing={}, stats_unique={}, stats_mode={}, print_impact=False):
    fr = as_frame(idf)
    if stats_missing == {}:
        stats = missingCount_computation(spark, fr).toPandas()
    else:
        stats = _read_stats(stats_missing, ["attribute", "missing_count", "missing_pct"])
    missing_cols = stats.loc[stats["missing_count"] > 0, "attribute"].tolist()
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        num, cat, _ = attributeType_segregation(fr)
        list_of_cols = num + cat
    if isinstance(list_of_cols, str) and list_of_cols == "missing":
        list_of_cols = missing_cols
    cols = unique(names(list_of_cols), names(drop_cols))
    if not cols:
        warnings.warn("No Null Detection - No column(s) to analyze")
        return fr, ResultFrame(pd.DataFrame(columns=["attribute", "missing_count", "missing_pct"]))
    if any(c not in fr.columns for c in cols):
        raise TypeError("Invalid input for Column(s)")
    treatment = _as_bool(treatment, "treatment")
    if treatment_method not in ("MMM", "row_removal", "column_removal", "KNN", "regression", "MF", "auto"):
        raise TypeError("Invalid input for method_type")
    treatment_configs = dict(treatment_configs)
    threshold = treatment_configs.pop("treatment_threshold", None)
    if threshold:
        threshold = float(threshold)
    elif treatment_method == "column_removal":
        raise TypeError("Invalid input for column removal threshold")
    stats = stats[stats["attribute"].isin(cols)].reset_index(drop=True)
    odf = fr
    if treatment:
        threshold_cols = stats.loc[stats["missing_pct"] > threshold, "attribute"].tolist() if threshold else []
        if treatment_method == "column_removal":
            odf = fr.drop(threshold_cols)
            if print_impact:
                print("Removed Columns: ", threshold_cols)
        elif treatment_method == "row_removal":
            remove = stats.loc[stats["missing_pct"] == 1.0, "attribute"].tolist()
            sub = [c for c in cols if c not in remove]
            if threshold:
                sub = [c for c in threshold_cols if c not in remove]
            odf = fr.dropna(subset=sub)
            if print_impact:
                print("Before Count: " + str(fr.count()))
                print("After Count: " + str(odf.count()))
        elif treatment_method == "MMM":
            # reference :491-519: drop columns with fewer than 2 distinct values, apply the threshold, impute
            from ..data_transformer.transformers import imputation_MMM
            from .stats_generator import uniqueCount_computation
            if stats_unique == {}:
                uq = uniqueCount_computation(spark, fr, cols).toPandas()
            else:
                uq = _read_stats(stats_unique, ["attribute", "unique_values"])
            remove = set(uq.loc[uq["unique_values"] < 2, "attribute"].tolist())
            sub = [c for c in cols if c not in remove]
            if threshold:
                sub = [c for c in threshold_cols if c not in remove]
            odf = imputation_MMM(spark, fr, sub, **treatment_configs, stats_missing=stats_missing, stats_mode=stats_mode,
                                 print_impact=print_impact)
            return odf, ResultFrame(stats)        # the reference prints imputation_MMM's table only
        else:
            raise NotImplementedError("treatment_method=%r (imputation) is outside the GPU hot-path build" % treatment_method)
    out = ResultFrame(stats)
    if print_impact:
        out.show(len(cols))
    return odf, out


def _discrete(fr, list_of_cols, drop_cols):
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        num, cat, _ = attributeType_segregation(fr)
        list_of_cols = num + cat
    cols = unique(names(list_of_cols), names(drop_cols))
    if any(c not in fr.columns for c in cols):
        raise TypeError("Invalid input for Column(s)")
    types = dict(fr.dtypes)
    return [c for c in cols if types[c] in ("string", "int", "bigint", "long")]   # reference :1122-1124


def IDness_detection(spark, idf, list_of_cols="all", drop_cols=[], treatment=False, treatment_threshold=0.8, stats_unique={},
                     print_impact=False):
    fr = as_frame(idf)
    cols = _discrete(fr, list_of_cols, drop_cols)
    if not cols:
        warnings.warn("No IDness Check - No discrete column(s) to analyze")
        return fr, ResultFrame(pd.DataFrame(columns=["attribute", "unique_values", "IDness", "flagged"]))
    treatment_threshold = float(treatment_threshold)
    if treatment_threshold < 0 or treatment_threshold > 1:
        raise TypeError("Invalid input for Treatment Threshold Value")
    treatment = _as_bool(treatment, "treatment")
    if stats_unique == {}:
        stats = measures_of_cardinality(spark, fr, cols).toPandas()
    else:
        stats = _read_stats(stats_unique, ["attribute", "unique_values", "IDness"])
        stats = stats[stats["attribute"].isin(cols)].reset_index(drop=True)
    stats["flagged"] = (stats["IDness"] >= treatment_threshold).astype(int)
    odf = fr
    if treatment:
        remove = stats.loc[stats["flagged"] == 1, "attribute"].tolist()
        odf = fr.drop(remove)
        stats = stats.rename(columns={"flagged": "treated"})
        if print_impact:
            print("Removed Columns: ", remove)
    out = ResultFrame(stats)
    if print_impact:
        out.show(len(cols))
    return odf, out


def biasedness_detection(spark, idf, list_of_cols="all", drop_cols=[], treatment=False, treatment_threshold=0.8, stats_mode={},
                         print_impact=False):
    fr = as_frame(idf)
    cols = _discrete(fr, list_of_cols, drop_cols)
    if not cols:
        warnings.warn("No biasedness Check - No discrete column(s) to analyze")
        return fr, ResultFrame(pd.DataFrame(columns=["attribute", "mode", "mode_rows", "mode_pct", "flagged"]))
    if treatment_threshold < 0 or treatment_threshold > 1:
        raise TypeError("Invalid input for Treatment Threshold Value")
    treatment = _as_bool(treatment, "treatment")
    if stats_mode == {}:
        nv = profile.n_valid(fr, cols)
        md = profile.mode_distinct(fr, cols)
        rows = []
        for c in cols:
            mode, mrows = md[c][0], md[c][1]
            rows.append([c, _mode_str(fr.column(c), mode), mrows, None if mrows is None else spark_round(mrows / nv[c])])
        stats = pd.DataFrame(rows, columns=["attribute", "mode", "mode_rows", "mode_pct"])
    else:
        stats = _read_stats(stats_mode, ["attribute", "mode", "mode_rows", "mode_pct"])
        stats = stats[stats["attribute"].isin(cols)].reset_index(drop=True)
    flag = [(1 if (p is None or pd.isna(p) or p >= treatment_threshold) else 0) for p in stats["mode_pct"].tolist()]
    stats["flagged"] = flag
    odf = fr
    if treatment:
        remove = stats.loc[stats["flagged"] == 1, "attribute"].tolist()
        odf = fr.drop(remove)
        stats = stats.rename(columns={"flagged": "treated"})
        if print_impact:
            print("Removed Columns: ", remove)
    out = ResultFrame(stats)
    if print_impact:
        out.show(len(cols))
    return odf, out


# ---- outlier_detection ---------------------------------------------------------------------------------

_OUTLIER_DEFAULTS = {"pctile_lower": 0.05, "pctile_upper": 0.95, "stdev_lower": 3.0, "stdev_upper": 3.0,
                     "IQR_lower": 1.5, "IQR_upper": 1.5, "min_validation": 2}
_PRINT_COLS = ["attribute", "lower_outliers", "upper_outliers", "excluded_due_to_skewness"]


def _outlier_methodologies(detection_side, cfg):
    """reference :788-830 -> (methodologies, min_validation)."""
    sides = {"lower": ["lower"], "upper": ["upper"], "both": ["lower", "upper"]}[detection_side]
    check = OrderedDict((m, OrderedDict((("lower", 0), ("upper", 0)))) for m in ("pctile", "stdev", "IQR"))
    for m in check:
        for side in sides:
            if m + "_" + side in cfg:
                check[m][side] = 1
    methods = []
    for m, val in check.items():
        vals = list(val.values())
        if detection_side == "both":
            if vals in ([1, 0], [0, 1]):
                raise TypeError("Invalid input for detection_configs. If detection_side is 'both', the methodologies used on "
                                "both sides should be the same")
            if vals[0]:
                methods.append(m)
        elif val[detection_side]:
            methods.append(m)
    if "min_validation" in cfg:
        if cfg["min_validation"] > len(methods):
            raise TypeError("Invalid input for min_validation of detection_configs. It cannot be larger than the total number "
                            "of methodologies on any side that detection will be applied over.")
        return methods, cfg["min_validation"]
    return methods, len(methods)     # if min_validation is not present, the number of specified methodologies is used


def _outlier_model_dir(model_path):
    return os.path.join(model_path, "outlier_numcols")


def _save_outlier_model(model_path, cols, params):
    """parquet [attribute: string, parameters: array<string>] (:912-934).  The reference hands Python floats to a
    StringType field, which the JVM stringifies: Java Double.toString."""
    import pyarrow as pa
    import pyarrow.parquet as pq
    d = _outlier_model_dir(model_path)
    os.makedirs(d, exist_ok=True)
    for f in os.listdir(d):
        if f.endswith(".parquet"):
            os.remove(os.path.join(d, f))
    enc = [[p if (p is None or isinstance(p, str)) else jvm_double_str(float(p)) for p in pr] for pr in params]
    t = pa.table({"attribute": pa.array(list(cols), pa.string()), "parameters": pa.array(enc, pa.list_(pa.string()))})
    pq.write_table(t, os.path.join(d, "part-00000.parquet"))


def _load_outlier_model(model_path):
    import pyarrow.parquet as pq
    t = pq.read_table(_outlier_model_dir(model_path))
    return dict(zip(t.column("attribute").to_pylist(), t.column("parameters").to_pylist()))


def _outlier_bounds(fr, cols, detection_side, cfg, methods, n_val):
    """-> (kept cols, [[lower|None, upper|None]], skewed cols): thresholds of :836-906 from the moments kernel and
    the selection kernel (approxQuantile(..., 0.01) ranks per shared/gk.py)."""
    E = profile.APPROX_QUANTILE_EPS
    pct = profile.quantiles(fr, cols, [cfg.get("pctile_lower", 0.05), cfg.get("pctile_upper", 0.95)], E)
    skewed = [c for c in cols if pct[c][0] == pct[c][1]]            # incl. all-null columns (None == None)
    kept = [c for c in cols if c not in skewed]
    if skewed:
        warnings.warn("Columns excluded from outlier detection due to highly skewed distribution: " + ",".join(skewed))
    mom = profile.moments(fr, kept) if "stdev" in methods else {}
    iqr = profile.quantiles(fr, kept, [0.25, 0.75], E) if "IQR" in methods else {}
    params = []
    for c in kept:
        x = list(pct[c]) if "pctile" in methods else [None, None]
        y, z = [None, None], [None, None]
        if "stdev" in methods:
            m = mom[c]
            n = int(m["n_valid"])
            mean = float(m["mean"])
            sd = math.sqrt(float(m["m2"]) / (n - 1)) if n > 1 else float("nan")
            y = [mean - cfg.get("stdev_lower", 0.0) * sd, mean + cfg.get("stdev_upper", 0.0) * sd]
        if "IQR" in methods:
            q1, q3 = iqr[c]
            z = [q1 - cfg.get("IQR_lower", 0.0) * (q3 - q1), q3 + cfg.get("IQR_upper", 0.0) * (q3 - q1)]
        lower = sorted([i for i in (x[0], y[0], z[0]) if i is not None], reverse=True)[n_val - 1]
        upper = sorted([i for i in (x[1], y[1], z[1]) if i is not None])[n_val - 1]
        params.append([lower, None] if detection_side == "lower" else ([None, upper] if detection_side == "upper"
                                                                        else [lower, upper]))
    return kept, params, skewed


def _outlier_cutoffs(param, detection_side):
    """Thresholds -> (cutoffs for the binning kernels, flag of each bin 1..len+1).  `v < lower` is the bin
    `v <= prev_double(lower)`; `v > upper` is the bin above `upper`."""
    lo = np.nextafter(param[0], -np.inf) if param[0] is not None else None
    hi = param[1]
    if detection_side == "lower":
        return [lo], [-1, 0]
    if detection_side == "upper":
        return [hi], [0, 1]
    if lo <= hi:
        return [lo, hi], [-1, 0, 1]
    return [hi, lo], [-1, 0, 1]      # crossed bounds: a value between them is flagged by both sides: -1 + 1 = 0 (:952)


def _outlier_thresholds_i64(param, detection_side):
    """_outlier_cutoffs for a bigint column -> (cutoffs, flags of bins 1..len+1, exact int64 thresholds).  The reference
    compares double(v) with the bounds (`v.astype(float)`, :937-950), so a bigint beyond 2^53 is rounded first: the flags
    are `v <= T_lo` (<=> double(v) < lower) and `v > T_hi` (<=> double(v) > upper), with the exact integers
    T_lo = the largest int64 whose double is < lower and T_hi = the largest whose double is <= upper (engine.i64_at_most).
    NaN bounds flag nothing, like the reference's compare."""
    lo = engine.i64_at_most(np.nextafter(param[0], -np.inf)) if param[0] is not None else None
    hi = None if param[1] is None else (engine.I64_MAX if param[1] != param[1] else engine.i64_at_most(param[1]))
    if detection_side == "lower":
        ths, flags = [lo], [-1, 0]
    elif detection_side == "upper":
        ths, flags = [hi], [0, 1]
    else:
        ths, flags = sorted([lo, hi]), [-1, 0, 1]    # crossed bounds: as _outlier_cutoffs
    # a threshold below -2^63 (no int64 qualifies) has an empty bin below it: clamp it to -2^63, and the values equal to
    # -2^63, which then land in bin 1, take the flag of the first bin above every such threshold
    k = sum(t < engine.I64_MIN for t in ths)
    if k:
        ths = [max(t, engine.I64_MIN) for t in ths]
        flags = [flags[k]] + flags[1:]
    return [float(t) for t in ths], flags, ths


def outlier_detection(spark, idf, list_of_cols="all", drop_cols=[], detection_side="upper", detection_configs=_OUTLIER_DEFAULTS,
                      treatment=True, treatment_method="value_replacement", pre_existing_model=False, model_path="NA",
                      sample_size=1000000, output_mode="replace", print_impact=False):
    """Same arguments, errors, model format and outputs as the reference (:550-1045).  Thresholds come from the
    moments / selection kernels, the per-value compare (the reference's pandas UDF, :937-966) from the binning
    kernels; the treated columns are assembled with tensor ops on the device."""
    torch = _lib.require_cuda()
    fr = as_frame(idf)
    column_order = fr.columns
    num_cols = attributeType_segregation(fr)[0]
    if not treatment and not print_impact:
        if (not pre_existing_model and model_path == "NA") or pre_existing_model:
            warnings.warn("The original idf will be the only output. Set print_impact=True to perform detection without treatment")
            return fr
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num_cols
    cols = unique(names(list_of_cols), names(drop_cols))
    empty_print = ResultFrame(pd.DataFrame(columns=_PRINT_COLS[:3]))
    if not cols:
        warnings.warn("No Outlier Check - No numerical column to analyze")
        return (fr, empty_print) if print_impact else fr
    if any(c not in num_cols for c in cols):
        raise TypeError("Invalid input for Column(s)")
    if detection_side not in ("upper", "lower", "both"):
        raise TypeError("Invalid input for detection_side")
    if treatment_method not in ("null_replacement", "row_removal", "value_replacement"):
        raise TypeError("Invalid input for treatment_method")
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")
    treatment = _as_bool(treatment, "treatment")
    pre_existing_model = _as_bool(pre_existing_model, "pre_existing_model")
    cfg = dict(detection_configs)
    for arg in ("pctile_lower", "pctile_upper"):
        if arg in cfg and (cfg[arg] < 0 or cfg[arg] > 1):
            raise TypeError("Invalid input for " + arg)

    if pre_existing_model:
        model = _load_outlier_model(model_path)
        params, present, skewed = [], [], []
        for c in cols:
            p = model.get(c)
            if p:
                if "skewed_attribute" in p:
                    skewed.append(c)
                else:
                    params.append([float(v) if v else v for v in p])
                    present.append(c)
        missing = [c for c in cols if c not in present and c not in skewed]
        if missing:
            warnings.warn("Columns not found in model_path: " + ",".join(missing))
        if skewed:
            warnings.warn("Columns excluded from outlier detection due to highly skewed distribution: " + ",".join(skewed))
        cols = present
        if not cols:
            warnings.warn("No Outlier Check - No numerical column to analyze")
            return (fr, empty_print) if print_impact else fr
    else:
        methods, n_val = _outlier_methodologies(detection_side, cfg)
        cfg["min_validation"] = n_val
        sample = fr
        if fr.count() > sample_size:
            # thresholds from a Bernoulli sample (:832-838): `idf.sample(sample_size / idf_count, False, 11)`.  With a float in
            # first position pyspark shifts the arguments (withReplacement omitted): fraction = the float, seed = int(False)
            # = 0, and the 11 is dropped - so Spark's XORShiftRandom stream is seeded with 0 (+ partition index).
            from ..data_ingest.data_sampling import data_sample
            sample = data_sample(fr.select(cols), fraction=sample_size / fr.count(), method_type="random", seed_value=0)
        cols, params, skewed = _outlier_bounds(sample, cols, detection_side, cfg, methods, n_val)
        if model_path != "NA":
            sk = {"lower": ["skewed_attribute", None], "upper": [None, "skewed_attribute"]}.get(
                detection_side, ["skewed_attribute", "skewed_attribute"])
            _save_outlier_model(model_path, cols + skewed, params + [sk] * len(skewed))
            if not treatment and not print_impact:
                return fr

    # ---- the compare pass: bin ids against [prev(lower), upper] ------------------------------------------
    rows = []
    odf = fr
    if cols:
        specs = [_outlier_thresholds_i64(p, detection_side) if fr.column(c).anv_dtype == _lib.ANV_I64
                 else _outlier_cutoffs(p, detection_side) + (None,) for c, p in zip(cols, params)]
        model = engine.BinModel(fr, cols, [s_[0] for s_ in specs], exact=[s_[2] for s_ in specs])
        need_rows = treatment and not getattr(fr, "is_partitioned", False)
        if need_rows:
            ids = engine.bin_assign(fr, model)                        # [n_cols, n_rows] int32, 0 = null
        else:
            if treatment:
                raise NotImplementedError("outlier treatment of a row-partitioned frame is not implemented "
                                          "(detection with print_impact=True is)")
            hist = engine.histogram(fr, model)
        made = OrderedDict()
        keep = torch.ones(fr.n_rows, dtype=torch.bool, device=ids.device) if need_rows else None
        for i, c in enumerate(cols):
            flags_of_bin = specs[i][1]
            if need_rows:
                flag = torch.zeros(fr.n_rows, dtype=torch.int8, device=ids.device)
                for b, f in enumerate(flags_of_bin, start=1):
                    if f:
                        flag[ids[i] == b] = f
                dcol = fr.column(c).device()[0]
                if dcol.is_floating_point():       # the binning kernels put NaN in the last bin; `(v - upper) > 0` is
                    flag[dcol != dcol] = 0         # False for NaN in the reference's compare (:937-966): never an outlier
                lower_n, upper_n = int((flag == -1).sum()), int((flag == 1).sum())
            else:
                lower_n = sum(int(hist[i, b]) for b, f in enumerate(flags_of_bin, start=1) if f == -1)
                upper_n = sum(int(hist[i, b]) for b, f in enumerate(flags_of_bin, start=1) if f == 1)
                if flags_of_bin[-1] == 1 and fr.column(c).anv_dtype in (_lib.ANV_F32, _lib.ANV_F64):
                    nan_rows = 0                   # NaN values sit in the last bin: not outliers (see above)
                    for ch in (fr.chunks([c]) if getattr(fr, "is_partitioned", False) else [fr]):
                        dch, vch = ch.column(c).device()
                        isn = dch != dch
                        if vch is not None:
                            isn &= ch.valid_mask(c)
                        nan_rows += int(isn.sum())
                    upper_n -= nan_rows
            rows.append((c, lower_n, upper_n, 0))
            if not need_rows:
                continue
            src = fr.column(c)
            d, v = src.device()
            name = c if output_mode == "replace" else c + "_outliered"
            if treatment_method == "value_replacement":
                lo, hi = params[i]
                out = d.to(torch.float64)
                if lo is not None:
                    out = torch.where(flag == -1, torch.tensor(float(lo), dtype=torch.float64, device=out.device), out)
                if hi is not None:
                    out = torch.where(flag == 1, torch.tensor(float(hi), dtype=torch.float64, device=out.device), out)
                made[name] = Column(name, "double", fr.n_rows, dev=out, dev_valid=v, anv_dtype=_lib.ANV_F64,
                                    null_count=src.null_count)
            elif treatment_method == "null_replacement":
                valid = (ids[i] != 0) & (flag == 0)
                nv = None if bool(valid.all()) else pack_bits_device(valid)
                made[name] = Column(name, src.sdtype, fr.n_rows, dev=d, dev_valid=nv, anv_dtype=src.anv_dtype,
                                    dictionary=src.dictionary)
            else:
                keep &= flag == 0
        if need_rows:
            if treatment_method == "row_removal":
                odf = fr.filter_rows(keep)
            else:
                odf = fr.with_columns(made)
    rows += [(c, 0, 0, 1) for c in (skewed if print_impact else [])]
    if treatment and output_mode == "replace":
        odf = odf.select(column_order)
    if not treatment:
        odf = fr
    if print_impact:
        out = ResultFrame(pd.DataFrame(rows, columns=_PRINT_COLS))
        out.show(len(rows))
        return odf, out
    return odf


# ---- invalidEntries_detection --------------------------------------------------------------------------

_INVALID_PRINT_COLS = ["attribute", "invalid_entries", "invalid_count", "invalid_pct"]


def _distinct_numeric(fr, c):
    """Distinct values of numeric column c over its valid rows (host array of its dtype, NaN payloads canonical): a sort
    on the device of the raw bits, so -0.0 and 0.0 stay apart.  A row-partitioned frame unions its chunks'."""
    from ..shared.invalid_rules import canonical_nan_bits
    if getattr(fr, "is_partitioned", False):
        if fr.group is not None:
            raise NotImplementedError("invalidEntries_detection of float columns, or of integer columns in manual / both "
                                      "mode, needs each column's distinct values on one rank; use "
                                      "partitioned.repartition_to_columns first (auto mode on integer and string columns "
                                      "works on row slabs)")
        parts = [_distinct_numeric(ch, c) for ch in fr.chunks([c])]
        return np.concatenate(parts) if parts else np.zeros(0, engine._NP_OF_ANV[fr.column(c).anv_dtype])
    torch = _lib.require_cuda()
    col = fr.column(c)
    d, v = col.device()
    d = d[:fr.n_rows]
    if v is not None:
        d = d[fr.valid_mask(c)]
    if d.is_floating_point():
        d = torch.where(torch.isnan(d), torch.full_like(d, float("nan")), d)
        d = d.view(torch.int32 if d.element_size() == 4 else torch.int64)
    host = torch.unique(d).cpu().numpy()
    if col.anv_dtype in (_lib.ANV_F32, _lib.ANV_F64):
        host = canonical_nan_bits(host.view(np.float32 if col.anv_dtype == _lib.ANV_F32 else np.float64))
    return host


def _invalid_table(fr, c, rule):
    """-> (sorted table of the column's invalid values for engine.flag_members, their strings as str(x) shows them)."""
    from ..shared import invalid_rules as R
    col = fr.column(c)
    if col.dictionary is not None:
        codes = R.dictionary_table(col.dictionary, rule)
        return codes, [str(col.dictionary[i]) for i in codes]
    if rule.flags_nothing:
        table = np.zeros(0, engine._NP_OF_ANV[col.anv_dtype])
    elif rule.auto_only and col.anv_dtype in (_lib.ANV_I32, _lib.ANV_I64):
        table = R.int_auto_table(engine._NP_OF_ANV[col.anv_dtype])
    else:
        table = R.numeric_table(_distinct_numeric(fr, c), rule)
    is_float = col.anv_dtype in (_lib.ANV_F32, _lib.ANV_F64)
    return table, [R.value_str(x, is_float) for x in table.tolist()]


def _with_flags_nulled(fr, cols, bitmaps, counts, output_mode, append_cols, schema=False):
    """The null-replacement frame: each column of `cols` (processing order) with its flagged rows nulled, the same device
    data under a new bitmap.  replace: the column moves to the end of the frame (the reference drops it and re-adds it);
    append: <c>_invalid is appended for the columns in `append_cols`.  schema=True: names, dtypes and dictionaries only
    (the schema of a row-partitioned result)."""
    made = OrderedDict()
    for c, bm, cnt in zip(cols, bitmaps, counts):
        if output_mode == "append" and c not in append_cols:
            continue
        src = fr.column(c)
        base = src.null_count if src.null_count is not None else (None if src.has_validity else 0)
        if schema:
            d = v = nulls = None
        elif bm is None:                   # an empty table: the column's own validity
            d, v = src.device()
            nulls = base
        else:
            d, v = src.device()
            nulls = None if base is None else base + int(np.sum(cnt))
        name = c if output_mode == "replace" else c + "_invalid"
        made[name] = Column(name, src.sdtype, fr.n_rows, dev=d, dev_valid=bm if bm is not None else v,
                            anv_dtype=src.anv_dtype, null_count=nulls, dictionary=src.dictionary)
    return fr.with_columns(made, drop=list(made) if output_mode == "replace" else ())


def invalidEntries_detection(spark, idf, list_of_cols="all", drop_cols=[], detection_type="auto", invalid_entries=[],
                             valid_entries=[], partial_match=False, treatment=False, treatment_method="null_replacement",
                             treatment_configs={}, stats_missing={}, stats_unique={}, stats_mode={}, output_mode="replace",
                             print_impact=False):
    """reference :1342-1711, same arguments, errors and outputs.  Every verdict depends on one value only, so the host
    decides once which distinct values are invalid (shared/invalid_rules.py: per dictionary entry for string columns,
    a closed-form table for int / bigint columns in auto mode, the column's distinct values otherwise) and one pass on
    the device (csrc/invalid.cu) counts the rows holding each of them and writes the nulled bitmaps of the treatment.

    Orders are deterministic where the reference's are not: the rows of odf_print follow the first-seen order of
    list_of_cols (the reference goes through a set()), and invalid_entries lists the values in table order - dictionary
    code order for strings, ascending numeric order for numbers (Spark's distinct() order is arbitrary).  In manual /
    both mode each value gets one verdict per column (the reference's UDF can flag one value twice and shift the flags of
    every later column; DESIGN.md section 1).  `treatment_threshold` is popped from treatment_configs, as the reference
    does, so the caller's dict loses it.  "all" takes the string / int / bigint / long columns; float and double columns
    are checked when listed."""
    from ..shared.invalid_rules import Rule
    fr = as_frame(idf)
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = [n for n, t in fr.dtypes if t in ("string", "int", "bigint", "long")]
    cols = unique(names(list_of_cols), names(drop_cols))
    if any(c not in fr.columns for c in cols):
        raise TypeError("Invalid input for Column(s)")
    if not cols:
        warnings.warn("No Invalid Entries Check - No discrete column(s) to analyze")
        return fr, ResultFrame(pd.DataFrame(columns=_INVALID_PRINT_COLS))
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")
    treatment = _as_bool(treatment, "treatment")
    if treatment_method not in ("MMM", "null_replacement", "column_removal"):
        raise TypeError("Invalid input for method_type")
    threshold = treatment_configs.pop("treatment_threshold", None)
    if threshold:
        threshold = float(threshold)
    elif treatment_method == "column_removal":
        raise TypeError("Invalid input for column removal threshold")
    bad = [c for c in cols if fr.column(c).kind == "other" or fr.column(c).sdtype.startswith("decimal")]
    if bad:
        raise TypeError("Column(s) %s have dtypes invalidEntries_detection does not check on the GPU path (%s); it takes "
                        "string, integer and floating columns" % (",".join(bad), ",".join(fr.column(c).sdtype for c in bad)))

    rule = Rule(detection_type, invalid_entries, valid_entries, partial_match)
    tables, strings = zip(*[_invalid_table(fr, c, rule) for c in cols])
    partitioned = getattr(fr, "is_partitioned", False)
    nulling = treatment and treatment_method in ("null_replacement", "MMM")
    counts, bitmaps = engine.flag_members(fr, cols, tables, nulling and not partitioned)
    n = fr.count()
    rows = []
    for c, cnt, s in zip(cols, counts, strings):
        hit = [s[i] for i in np.flatnonzero(cnt)]
        total = int(cnt.sum())
        rows.append([c, "|".join(dict.fromkeys(hit)), total, round(total / n, 4)])
    odf_print = ResultFrame(pd.DataFrame(rows, columns=_INVALID_PRINT_COLS))

    odf = fr
    if treatment:
        pct = {r[0]: r[3] for r in rows}
        threshold_cols = [c for c in cols if pct[c] > threshold] if threshold else []
        if nulling:
            sel = [i for i, c in enumerate(cols) if not threshold or c in threshold_cols]
            tcols = [cols[i] for i in sel]
            append_cols = {c for c in tcols if pct[c] != 0.0}
            if partitioned:
                ttables = [tables[i] for i in sel]

                def treat(ch):
                    cnt, bms = engine.flag_members(ch, tcols, ttables, bool(ch.n_rows))
                    return _with_flags_nulled(ch, tcols, bms, cnt, output_mode, append_cols)
                odf = fr.map_chunks(_with_flags_nulled(fr._schema, tcols, [None] * len(tcols), [0] * len(tcols),
                                                       output_mode, append_cols, schema=True), treat)
            else:
                odf = _with_flags_nulled(fr, tcols, [bitmaps[i] for i in sel], [counts[i] for i in sel], output_mode,
                                         append_cols)
        if treatment_method == "column_removal":
            odf = fr.drop(threshold_cols)
            if print_impact:
                print("Removed Columns: ", threshold_cols)
        if treatment_method == "MMM":
            from ..data_transformer.transformers import imputation_MMM
            from .stats_generator import uniqueCount_computation
            if stats_unique == {} or output_mode == "append":
                uq = uniqueCount_computation(spark, odf, cols).toPandas()
            else:
                uq = _read_stats(stats_unique, ["attribute", "unique_values"])
            remove = set(uq.loc[uq["unique_values"] < 2, "attribute"].tolist())
            cols = [c for c in cols if c not in remove]
            if threshold:
                cols = [c for c in threshold_cols if c not in remove]
            if output_mode == "append" and cols:
                cols = [c + "_invalid" for c in cols]
            odf = imputation_MMM(spark, odf, cols, **treatment_configs, stats_missing=stats_missing, stats_mode=stats_mode,
                                 print_impact=print_impact)
    if print_impact:
        odf_print.show(len(cols))
    return odf, odf_print
