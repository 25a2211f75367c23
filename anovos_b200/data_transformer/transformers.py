"""CUDA implementation of `anovos.data_transformer.transformers.attribute_binning`
(reference /root/reference/src/main/anovos/data_transformer/transformers.py:87-291), `imputation_MMM` (:1369-1676) and
the scalers `z_standardization`, `IQR_standardization` and `normalization` (:965-1366, at the end of this module).

The reference computes the cutoffs with one Spark agg (equal_range, :216-232) or
approxQuantile (equal_frequency, :210-215) and then calls a Python UDF once per value
(:248-280).  Here the min/max come from the fused moments kernel, the quantile cutoffs
from the exact radix-select kernel and the bin ids from the bin-assign kernel; the cutoff
ARITHMETIC (`min + j * ((max - min) / bin_size)` in Python float64) stays on the host so
the model is bit-identical to the reference's.  The saved model keeps the reference's
format: parquet [attribute: string, parameters: array<double>] at
`<model_path>/attribute_binning`.
"""
from __future__ import annotations

import math
import os
import warnings
from collections import OrderedDict

import numpy as np

from .. import _lib, engine, profile
from ..frame import Column, ColumnFrame, as_frame
from ..shared.utils import attributeType_segregation


def _names(x):
    if isinstance(x, str):
        return [s.strip() for s in x.split("|")]
    return list(x)


def _model_dir(model_path):
    return os.path.join(model_path, "attribute_binning")


def save_binning_model(model_path, cols, cutoffs):
    import pyarrow as pa
    import pyarrow.parquet as pq
    d = _model_dir(model_path)
    os.makedirs(d, exist_ok=True)
    for f in os.listdir(d):  # mode="overwrite"
        if f.endswith(".parquet"):
            os.remove(os.path.join(d, f))
    t = pa.table({"attribute": pa.array(list(cols), pa.string()),
                  "parameters": pa.array([list(map(float, c)) for c in cutoffs], pa.list_(pa.float64()))})
    pq.write_table(t, os.path.join(d, "part-00000.parquet"))


def load_binning_model(model_path):
    import pyarrow.parquet as pq
    t = pq.read_table(_model_dir(model_path))
    return OrderedDict(zip(t.column("attribute").to_pylist(), t.column("parameters").to_pylist()))


def compute_cutoffs(fr: ColumnFrame, cols, method_type, bin_size):
    """-> (kept cols, cutoffs, (min,max) per kept col | None).  transformers.py:210-240."""
    mom = profile.moments(fr, cols)
    if method_type == "equal_frequency":
        width = 1 / bin_size
        probs = [j * width for j in range(1, bin_size)]               # :211-214 (float artefacts kept)
        q = profile.quantiles(fr, cols, probs, profile.APPROX_QUANTILE_EPS)   # approxQuantile(cols, probs, 0.01), :215
        cuts = [[float("nan") if v is None else float(v) for v in q[c]] for c in cols]
        return list(cols), cuts, [None] * len(cols)
    kept, cuts, lohi, dropped = [], [], [], []
    for c in cols:
        if int(mom[c]["n_valid"]) == 0:                                 # max is null (:226-228)
            dropped.append(c)
            continue
        mx, mn = float(mom[c]["max"]), float(mom[c]["min"])
        w = (mx - mn) / bin_size                                        # :229
        cuts.append([mn + j * w for j in range(1, bin_size)])           # :230-231
        kept.append(c)
        lohi.append((mn, mx))
    if dropped:
        warnings.warn("Columns contains too much null values. Dropping " + ", ".join(dropped))
    return kept, cuts, lohi


def _labels(cut, n_over_cut):
    """bin_dtype="categorical" range strings of bucket_label (:257-264,271), bins 1..len(cut)+1."""
    out = ["<= " + str(round(cut[0], 4))]
    for i in range(1, len(cut)):
        out.append(str(round(cut[i - 1], 4)) + "-" + str(round(cut[i], 4)))
    out.append("> " + str(round(cut[n_over_cut - 1], 4)))
    return out


def _apply_binning(fr: ColumnFrame, cols, cuts, lohi, bin_dtype, output_mode) -> ColumnFrame:
    """bucket_label (:248-280) for every value of `cols` with the given cutoffs -> new frame."""
    bm = engine.BinModel(fr, cols, cuts, lohi)
    ids = engine.bin_assign(fr, bm)                         # [n_cols, n_rows] int32, 0 = null
    n_over = len(cuts[0]) + 1                               # `len(bin_cutoffs[0]) + 1` quirk (:269)
    new_cols = OrderedDict((n, fr.column(n)) for n in fr.columns)
    for i, c in enumerate(cols):
        src = fr.column(c)
        _, v = src.device()
        data = ids[i]
        if len(cuts[i]) + 1 != n_over:                      # only reachable with a hand-made model
            data = data.clone()
            data[data == len(cuts[i]) + 1] = n_over
        if bin_dtype == "numerical":
            col = Column(c, "int", fr.n_rows, dev=data, dev_valid=v, anv_dtype=_lib.ANV_I32,
                         null_count=src.null_count)
        else:
            col = Column(c, "string", fr.n_rows, dev=(data - 1).clamp_(min=0), dev_valid=v, anv_dtype=_lib.ANV_I32,
                         null_count=src.null_count, dictionary=_labels(cuts[i], len(cuts[0])))
        if output_mode == "replace":
            new_cols[c] = col
        else:
            col.name = c + "_binned"
            new_cols[c + "_binned"] = col
    return ColumnFrame(new_cols, fr.n_rows)


def attribute_binning(spark, idf, list_of_cols="all", drop_cols=[], method_type="equal_range", bin_size=10,
                      bin_dtype="numerical", pre_existing_model=False, model_path="NA", output_mode="replace",
                      print_impact=False):
    """Same arguments / errors as the reference; returns a ColumnFrame whose binned columns hold
    int32 bin ids 1..bin_size on the device (null rows stay null)."""
    fr = as_frame(idf)
    num_cols = attributeType_segregation(fr)[0]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num_cols
    drop = _names(drop_cols)
    cols = []
    for c in _names(list_of_cols):
        if c not in drop and c not in cols:
            cols.append(c)
    if any(c not in num_cols for c in cols):
        raise TypeError("Invalid input for Column(s)")
    if not cols:
        warnings.warn("No Binning Performed - No numerical column(s) to transform")
        return fr
    if method_type not in ("equal_frequency", "equal_range"):
        raise TypeError("Invalid input for method_type")
    if bin_size < 2:
        raise TypeError("Invalid input for bin_size")
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")

    lohi = None
    if pre_existing_model:
        model = load_binning_model(model_path)
        cuts = []
        for c in cols:
            if c not in model:
                raise IndexError("list index out of range")   # reference: .collect()[0] on an empty list
            cuts.append(model[c])
    else:
        cols, cuts, lohi = compute_cutoffs(fr, cols, method_type, bin_size)
        if model_path != "NA":
            save_binning_model(model_path, cols, cuts)
    if not cols:
        return fr

    if getattr(fr, "is_partitioned", False):
        # lazy per-chunk transform with the (global) model: the binned frame is partitioned like its input
        schema = _apply_binning(fr._schema, cols, cuts, lohi, bin_dtype, output_mode)
        odf = fr.map_chunks(schema, lambda ch: _apply_binning(ch, cols, cuts, lohi, bin_dtype, output_mode))
    else:
        odf = _apply_binning(fr, cols, cuts, lohi, bin_dtype, output_mode)
    if print_impact:
        from ..data_analyzer.stats_generator import uniqueCount_computation
        out_cols = cols if output_mode == "replace" else [c + "_binned" for c in cols]
        uniqueCount_computation(spark, odf, out_cols).show(len(out_cols))
    return odf


# ---- imputation_MMM (reference transformers.py:1369-1676) -------------------------------------------------------------
#
# Numeric columns under "mean" / "median" go through Spark ML's Imputer: statistics over the non-null, non-NaN values of
# double(x) (the moments pass / the GK median at relativeError 0.001), then
# `when(ic.isNull, s).when(ic == NaN, s).otherwise(ic).cast(inputType)`; columns that are not float / double were recast
# to double first and their `_imputed` outputs are cast back (:1496-1502, :1571-1572).  Categorical columns, and numeric
# ones under "mode", get their mode where they are null (:1505-1552, :1580-1636).  The fill itself is one streaming pass
# (anv_impute_fill).  Deviations from the reference: DESIGN.md section 1.

IMPUTER_RELATIVE_ERROR = 0.001       # Imputer's default relativeError (its median is approxQuantile(0.5, 0.001))
_IMPUTE_DIR, _NUM_MODEL, _CAT_MODEL = "imputation_MMM", "num_imputer-model", "cat_imputer"
_ANV_OF_SDTYPE = {"float": _lib.ANV_F32, "double": _lib.ANV_F64, "int": _lib.ANV_I32, "bigint": _lib.ANV_I64,
                  "long": _lib.ANV_I64}
_SDTYPE_OF_ANV = {_lib.ANV_F32: "float", _lib.ANV_F64: "double", _lib.ANV_I32: "int", _lib.ANV_I64: "bigint"}


def _spark_parts(d):
    """The data files of a directory Spark (or this module) wrote: `part-*`, without checksum files and markers."""
    return sorted(os.path.join(d, f) for f in os.listdir(d) if f.startswith("part-") and not f.endswith(".crc"))


def _clear_dir(d):
    import shutil
    if os.path.isdir(d):                                   # mode="overwrite"
        shutil.rmtree(d)
    os.makedirs(d)


def save_imputer_model(model_path, input_cols, output_cols, strategy, surrogates):
    """Spark ML's ImputerModel directory: metadata/part-00000 (one JSON line) and data/*.parquet (one row, one double
    column per input column), each with a _SUCCESS marker."""
    import json
    import time
    import uuid
    import pyarrow as pa
    import pyarrow.parquet as pq
    d = os.path.join(model_path, _IMPUTE_DIR, _NUM_MODEL)
    _clear_dir(d)
    uid = "Imputer_" + uuid.uuid4().hex[:12]
    meta = {"class": "org.apache.spark.ml.feature.ImputerModel", "timestamp": int(time.time() * 1000),
            "sparkVersion": "3.2.1", "uid": uid,
            "paramMap": {"strategy": strategy, "inputCols": list(input_cols), "outputCols": list(output_cols)},
            "defaultParamMap": {"strategy": "mean", "missingValue": "NaN", "relativeError": IMPUTER_RELATIVE_ERROR,
                                "outputCols": [uid + "__output"]}}
    for sub in ("metadata", "data"):
        os.makedirs(os.path.join(d, sub))
        open(os.path.join(d, sub, "_SUCCESS"), "w").close()
    with open(os.path.join(d, "metadata", "part-00000"), "w") as f:
        f.write(json.dumps(meta) + "\n")
    t = pa.table({c: pa.array([float(s)], pa.float64()) for c, s in zip(input_cols, surrogates)})
    pq.write_table(t, os.path.join(d, "data", "part-00000.snappy.parquet"), compression="snappy")


def load_imputer_model(model_path):
    """-> (input cols, output cols, {input col: surrogate}) of an ImputerModel directory (Spark's own or ours)."""
    import json
    import pyarrow.parquet as pq
    d = os.path.join(model_path, _IMPUTE_DIR, _NUM_MODEL)
    meta = json.loads(open(_spark_parts(os.path.join(d, "metadata"))[0]).readline())
    pm = meta.get("paramMap", {})
    ins = pm.get("inputCols") or [pm["inputCol"]]
    outs = pm.get("outputCols") or [pm["outputCol"]]
    files = [f for f in _spark_parts(os.path.join(d, "data")) if f.endswith(".parquet")]
    t = pq.read_table(files[0]) if len(files) == 1 else __import__("pyarrow").concat_tables([pq.read_table(f) for f in files])
    return list(ins), list(outs), {c: float(t.column(c)[0].as_py()) for c in ins}


def save_cat_imputer(model_path, cols, params):
    """The categorical model: a CSV directory with the header `attribute,parameters` (null -> empty field)."""
    import csv
    d = os.path.join(model_path, _IMPUTE_DIR, _CAT_MODEL)
    _clear_dir(d)
    with open(os.path.join(d, "part-00000.csv"), "w", newline="") as f:
        w = csv.writer(f, doublequote=False, escapechar="\\", lineterminator="\n")
        w.writerow(["attribute", "parameters"])
        for c, p in zip(cols, params):
            w.writerow([c, "" if p is None else p])
    open(os.path.join(d, "_SUCCESS"), "w").close()


def load_cat_imputer(model_path):
    """-> [(attribute, parameter | None)] in file order."""
    import csv
    d = os.path.join(model_path, _IMPUTE_DIR, _CAT_MODEL)
    rows = []
    for fn in [f for f in _spark_parts(d) if f.endswith(".csv")]:
        with open(fn, newline="") as f:
            r = list(csv.reader(f, doublequote=False, escapechar="\\"))
        rows += [(a, p if p != "" else None) for a, p in r[1:]]
    return rows


def _read_mode_stats(stats_mode):
    """read_dataset(**stats_mode).replace("None", None): attribute -> [mode | None, ...] (every row of the attribute)."""
    from ..data_analyzer.quality_checker import _read_stats
    df = _read_stats(stats_mode, ["attribute", "mode"])
    out = {}
    for a, m in zip(df["attribute"].tolist(), df["mode"].tolist()):
        m = None if (m is None or (isinstance(m, float) and m != m) or str(m) == "None") else str(m)
        out.setdefault(a, []).append(m)
    return out


def _nan_view(fr, cols):
    """`fr` with the validity of `cols` replaced by "non-null and not NaN" (anv_valid_not_nan): the Imputer's statistics
    are the moments / selection of this view."""
    if not cols:
        return fr
    if getattr(fr, "is_partitioned", False):
        return fr.map_chunks(fr._schema, lambda ch: _nan_view(ch, cols))
    words, _ = engine.valid_not_nan(fr, cols)
    new = OrderedDict((n, fr.column(n)) for n in fr.columns)
    for i, c in enumerate(cols):
        src = fr.column(c)
        d, _v = src.device()
        new[c] = Column(c, src.sdtype, fr.n_rows, dev=d, dev_valid=words[i], anv_dtype=src.anv_dtype)
    return ColumnFrame(new, fr.n_rows)


def _surrogates(fr, cols, method_type):
    """Imputer.fit (Spark 3.x): avg / approxQuantile(0.5, 0.001) over the non-null, non-NaN double(x) of each column.
    Float columns whose cached mean is NaN hold NaN (or both infinities): their statistics run on the NaN-free view."""
    if not cols:
        return []
    mom = profile.moments(fr, cols)
    nan_cols = [c for c in cols if fr.column(c).anv_dtype in (_lib.ANV_F32, _lib.ANV_F64) and math.isnan(float(mom[c]["mean"]))
                and int(mom[c]["n_valid"]) > 0]
    view = _nan_view(fr, nan_cols)
    out = {}
    if nan_cols:
        vm = engine.moments(view, nan_cols)
        for c, r in zip(nan_cols, vm):
            out[c] = r
    for c in cols:
        rec = out.get(c, mom[c])
        if int(rec["n_valid"]) == 0:
            raise ValueError("surrogate cannot be computed. All the values in %s are Null, Nan or missingValue(NaN)" % c)
    if method_type == "mean":
        return [float(out.get(c, mom[c])["mean"]) for c in cols]
    q = dict(profile.quantiles(fr, [c for c in cols if c not in nan_cols], [0.5], IMPUTER_RELATIVE_ERROR))
    if nan_cols:
        q.update(profile.quantiles(view, nan_cols, [0.5], IMPUTER_RELATIVE_ERROR))
    return [float(q[c][0]) for c in cols]


def _numeric_modes(fr, cols):
    """`idf.select(i).dropna().groupby(i).count().orderBy("count").first()` (:1507-1519): dropna drops NaN too, so float
    columns holding NaN take their mode from the NaN-free view.  Ties: the smallest value."""
    if not cols:
        return {}
    mom = profile.moments(fr, cols)
    nan_cols = [c for c in cols if fr.column(c).anv_dtype in (_lib.ANV_F32, _lib.ANV_F64) and math.isnan(float(mom[c]["mean"]))]
    md = dict(profile.mode_distinct(fr, [c for c in cols if c not in nan_cols]))
    if nan_cols:
        md.update(profile.mode_distinct(_nan_view(fr, nan_cols), nan_cols))
    return {c: md[c][0] for c in cols}


class _Plan:
    """What imputation_MMM writes: recasts (int / bigint -> double, nulls kept) and fills, by output name."""

    def __init__(self):
        self.recast = []          # source columns replaced in place by their double
        self.fills = []           # (output name, source, out anv dtype, flags, fill value | None, dictionary | None)


def _fill_dictionary(col, value):
    """(dictionary, code) of a categorical fill string; a string not in the dictionary is appended to it."""
    dic = col.dictionary
    try:
        return dic, dic.index(value)
    except ValueError:
        return list(dic) + [value], len(dic)


def _apply_plan(fr, plan: _Plan, order):
    """Run the recasts and fills of `plan` on a (resident) frame in ONE anv_impute_fill launch; `order` = the output
    column names, in order."""
    srcs, outs_dt, flags, bits = [], [], [], []
    for c in plan.recast:
        srcs.append(c)
        outs_dt.append(_lib.ANV_F64)
        flags.append(0)
        bits.append(0)
    for name, src, od, fl, val, dic in plan.fills:
        srcs.append(src)
        outs_dt.append(od)
        flags.append(fl)
        bits.append(0 if val is None else engine.fill_bits(val, od))
    data = engine.impute_fill(fr, srcs, outs_dt, flags, bits)
    made = {}
    for c, d in zip(plan.recast, data[:len(plan.recast)]):
        s = fr.column(c)
        _, v = s.device()
        made[c] = Column(c, "double", fr.n_rows, dev=d, dev_valid=v, anv_dtype=_lib.ANV_F64, null_count=s.null_count)
    for (name, src, od, fl, val, dic), d in zip(plan.fills, data[len(plan.recast):]):
        s = fr.column(src)
        v, nc = None, 0
        if val is None:                                    # a null fill leaves the nulls where they are
            v, nc = s.device()[1], s.null_count
        sd = "string" if dic is not None else _SDTYPE_OF_ANV[od]
        made[name] = Column(name, sd, fr.n_rows, dev=d, dev_valid=v, anv_dtype=od, null_count=nc, dictionary=dic)
    return ColumnFrame(OrderedDict((n, made[n] if n in made else fr.column(n)) for n in order), fr.n_rows)


def _impact(spark, odf, missing_df, list_of_cols, num_cols, cat_cols, missing_cols, output_mode):
    """The before / after table of print_impact (:1644-1673); rows in attribute order, as Spark's join returns them."""
    import pandas as pd
    from ..data_analyzer.stats_generator import missingCount_computation
    from ..result import ResultFrame
    before = dict(zip(missing_df["attribute"].tolist(), missing_df["missing_count"].tolist()))
    if output_mode == "replace":
        after = missingCount_computation(spark, odf, list_of_cols).toPandas()
        rows = [[a, int(before[a]), int(m)] for a, m in zip(after["attribute"], after["missing_count"]) if a in before]
        cols = ["attribute", "missingCount_before", "missingCount_after"]
    else:
        out_cols = [i + "_imputed" for i in num_cols + cat_cols if i in missing_cols]
        after = missingCount_computation(spark, odf, out_cols).toPandas() if out_cols else pd.DataFrame(
            {"attribute": [], "missing_count": []})
        rows = [[a[:-8], int(before[a[:-8]]), a, int(m)] for a, m in zip(after["attribute"], after["missing_count"])
                if a[:-8] in before]
        cols = ["attribute", "missingCount_before", "attribute_after", "missing_count"]
    rows.sort(key=lambda r: r[0])
    return ResultFrame(pd.DataFrame(rows, columns=cols))


def imputation_MMM(spark, idf, list_of_cols="missing", drop_cols=[], method_type="median", pre_existing_model=False,
                   model_path="NA", output_mode="replace", stats_missing={}, stats_mode={}, print_impact=False):
    """Same arguments, errors and returned frame as the reference (transformers.py:1369-1676).  Imputed columns are dense
    device columns; numeric columns are processed before categorical ones, each in list order."""
    from ..data_analyzer.quality_checker import _as_bool, _read_stats
    from ..data_analyzer.stats_generator import missingCount_computation
    fr = as_frame(idf)
    if stats_missing == {}:
        missing_df = missingCount_computation(spark, fr).toPandas()
    else:
        missing_df = _read_stats(stats_missing, ["attribute", "missing_count", "missing_pct"])
    missing_cols = missing_df.loc[missing_df["missing_count"] > 0, "attribute"].tolist()
    pre_existing_model = _as_bool(pre_existing_model, "pre_existing_model")
    if not missing_cols and not pre_existing_model and model_path == "NA":
        return fr

    num_all, cat_all, _ = attributeType_segregation(fr)
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num_all + cat_all
    if isinstance(list_of_cols, str) and list_of_cols == "missing":
        list_of_cols = [x for x in missing_cols if x in num_all + cat_all]
    drop = _names(drop_cols)
    list_of_cols = [c for c in dict.fromkeys(_names(list_of_cols)) if c not in drop]
    if not list_of_cols:
        warnings.warn("No Imputation performed- No column(s) to impute")
        return fr
    if any(x not in num_all + cat_all for x in list_of_cols):
        raise TypeError("Invalid input for Column(s)")
    if method_type not in ("mode", "mean", "median"):
        raise TypeError("Invalid input for method_type")
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")
    num_cols = [c for c in list_of_cols if fr.column(c).kind == "num"]
    cat_cols = [c for c in list_of_cols if fr.column(c).kind == "cat"]
    sdt = dict(fr.dtypes)
    for c in num_cols:
        if sdt[c] not in _ANV_OF_SDTYPE:
            raise TypeError("imputation of %s column %r is not supported on the device" % (sdt[c], c))

    plan = _Plan()
    created = []                                            # `_imputed` outputs in the order Spark adds them
    recast = [c for c in num_cols if sdt[c] not in ("float", "double")]
    if num_cols:
        if method_type == "mode":
            if stats_mode == {}:
                md = _numeric_modes(fr, num_cols)
                params = [None if md[c] is None else float(md[c]) for c in num_cols]
            else:
                saved = _read_mode_stats(stats_mode)
                todo = [c for c in num_cols if c not in saved]
                md = _numeric_modes(fr, todo)
                params = [(None if md[c] is None else float(md[c])) if c not in saved else
                          (None if saved[c][0] is None else float(saved[c][0])) for c in num_cols]
            for c, p in zip(num_cols, params):
                od = fr.column(c).anv_dtype if c not in recast else _lib.ANV_F64    # deviation 2: the recast type
                val = None if p is None else engine.java_cast(p, od)
                plan.fills.append((c + "_imputed", c, od, 0, val, None))
                created.append(c + "_imputed")
        else:
            if pre_existing_model:
                ins, outs, sur = load_imputer_model(model_path)
                for c in ins:
                    if c not in fr.columns:
                        raise ValueError("cannot resolve '%s' given input columns" % c)
                missing_out = [c + "_imputed" for c in recast if c + "_imputed" not in outs]
                if missing_out:
                    raise ValueError("cannot resolve '%s' given input columns" % missing_out[0])
                pairs = [(c, o, sur[c]) for c, o in zip(ins, outs)]
            else:
                sv = _surrogates(fr, num_cols, method_type)
                pairs = [(c, c + "_imputed", s) for c, s in zip(num_cols, sv)]
                if model_path != "NA":
                    save_imputer_model(model_path, num_cols, [o for _, o, _ in pairs], method_type, sv)
            for c, o, s in pairs:
                od = fr.column(c).anv_dtype                 # Imputer output cast to the input type (then back from double)
                fl = _lib.IMPUTE_NAN_MISSING if od in (_lib.ANV_F32, _lib.ANV_F64) else 0
                if od in (_lib.ANV_I32, _lib.ANV_I64):
                    fl |= _lib.IMPUTE_ROUND_DOUBLE
                plan.fills.append((o, c, od, fl, engine.java_cast(s, od), None))
                created.append(o)

    if cat_cols:
        if pre_existing_model:
            model = load_cat_imputer(model_path)
            params = []
            for c in cat_cols:
                hit = [p for a, p in model if a == c]
                if not hit:
                    raise IndexError("list index out of range")     # `.collect()[0]` on no row (:1589-1594)
                params.append(hit[0])
        elif stats_mode == {}:
            md = profile.mode_distinct(fr, cat_cols)
            params = [str(md[c][0]) for c in cat_cols]               # str(None) = "None" for an all-null column
        else:
            saved = _read_mode_stats(stats_mode)
            params = []
            for c in cat_cols:
                if c not in saved:
                    raise IndexError("list index out of range")
                params.append(saved[c][0])
        for c, p in zip(cat_cols, params):
            col = fr.column(c)
            dic, code = (col.dictionary, 0) if p is None else _fill_dictionary(col, p)
            plan.fills.append((c + "_imputed", c, _lib.ANV_I32, 0, None if p is None else code, dic))
            created.append(c + "_imputed")
        if not pre_existing_model and model_path != "NA":
            save_cat_imputer(model_path, cat_cols, params)

    # :1638-1642 - only columns with nulls keep their `_imputed`; "replace" moves it into the original's name, at the end
    order = [c for c in fr.columns]
    kept = list(created)
    for i in num_cols + cat_cols:
        if i not in missing_cols:
            kept = [k for k in kept if k != i + "_imputed"]
        elif output_mode == "replace":
            order = [c for c in order if c != i]
    renamed = {}
    for k in kept:
        base = k[:-8] if k.endswith("_imputed") else None
        if output_mode == "replace" and base in missing_cols and base in num_cols + cat_cols:
            renamed[k] = base
    order = order + [renamed.get(k, k) for k in kept]
    plan.recast = [c for c in recast if c in order]
    plan.fills = [(renamed.get(f[0], f[0]),) + f[1:] for f in plan.fills if f[0] in kept]

    if getattr(fr, "is_partitioned", False):
        odf = fr.map_chunks(_apply_plan(fr._schema, plan, order), lambda ch: _apply_plan(ch, plan, order))
    else:
        odf = _apply_plan(fr, plan, order)
    if print_impact:
        _impact(spark, odf, missing_df, list_of_cols, num_cols, cat_cols, missing_cols, output_mode).show(len(list_of_cols), False)
    return odf


# ---- scaling: z_standardization, IQR_standardization, normalization (reference transformers.py:965-1366) --------------
#
# The parameters come from the existing passes (moments for mean / stddev / min / max, the GK sketch of approxQuantile
# for the quartiles) and the transform is one streaming pass (anv_scale_columns).  All parameter arithmetic is IEEE
# double on the host, as in the reference's Python and Spark's JVM.  Semantics and deviations: DESIGN.md section 1.

_SCALE_DIR = {"z": "z_standardization", "iqr": "IQR_standardization", "norm": "normalization"}
_MINMAX_CLASS = "org.apache.spark.ml.feature.MinMaxScalerModel"
_DOUBLE_MAX = 1.7976931348623157e308      # Scala's Double.MaxValue: an all-NaN feature's min in MinMaxScalerModel


def _scale_cols(fr, list_of_cols, drop_cols, output_mode, what):
    """The reference's argument checks, in its order; -> the columns (first-seen order), or None (warned: nothing to do)."""
    num_cols = attributeType_segregation(fr)[0]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num_cols
    drop = _names(drop_cols)
    cols = [c for c in dict.fromkeys(_names(list_of_cols)) if c not in drop]
    if any(c not in num_cols for c in cols):
        raise TypeError("Invalid input for Column(s)")
    if not cols:
        warnings.warn("No %s Performed - No numerical column(s) to transform" % what)
        return None
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")
    sdt = dict(fr.dtypes)
    for c in cols:
        if sdt[c] not in _ANV_OF_SDTYPE:
            raise TypeError("scaling of %s column %r is not supported on the device" % (sdt[c], c))
    return cols


def _save_param_model(model_path, kind, cols, params):
    """parquet [feature: string, parameters: array<double>] at <model_path>/<kind> (elements may be null)."""
    import pyarrow as pa
    import pyarrow.parquet as pq
    d = os.path.join(model_path, _SCALE_DIR[kind])
    _clear_dir(d)
    t = pa.table({"feature": pa.array(list(cols), pa.string()),
                  "parameters": pa.array([[None if v is None else float(v) for v in p] for p in params],
                                         pa.list_(pa.float64()))})
    pq.write_table(t, os.path.join(d, "part-00000.snappy.parquet"), compression="snappy")
    open(os.path.join(d, "_SUCCESS"), "w").close()


def _load_param_model(model_path, kind, cols):
    """`df_model.where(feature == c).select("parameters")...collect()[0]` per column; a missing column raises the
    reference's IndexError."""
    import pyarrow.parquet as pq
    d = os.path.join(model_path, _SCALE_DIR[kind])
    model = {}
    for f in _spark_parts(d):
        if f.endswith(".parquet"):
            t = pq.read_table(f)
            for a, p in zip(t.column("feature").to_pylist(), t.column("parameters").to_pylist()):
                model.setdefault(a, p)
    out = []
    for c in cols:
        if c not in model:
            raise IndexError("list index out of range")
        out.append(model[c])
    return out


def save_minmax_model(model_path, lo, hi, mins, maxs):
    """Spark ML's MinMaxScalerModel directory at <model_path>/normalization: metadata/part-00000 (one JSON line) and
    data/*.parquet (one row: originalMin, originalMax as dense vectors), each with a _SUCCESS marker."""
    import json
    import time
    import uuid
    import pyarrow as pa
    import pyarrow.parquet as pq
    d = os.path.join(model_path, _SCALE_DIR["norm"])
    _clear_dir(d)
    uid = "MinMaxScaler_" + uuid.uuid4().hex[:12]
    meta = {"class": _MINMAX_CLASS, "timestamp": int(time.time() * 1000), "sparkVersion": "3.2.1", "uid": uid,
            "paramMap": {"inputCol": "list_of_cols_vector", "outputCol": "list_of_cols_scaled"},
            "defaultParamMap": {"min": float(lo), "max": float(hi), "outputCol": uid + "__output"}}
    for sub in ("metadata", "data"):
        os.makedirs(os.path.join(d, sub))
        open(os.path.join(d, sub, "_SUCCESS"), "w").close()
    with open(os.path.join(d, "metadata", "part-00000"), "w") as f:
        f.write(json.dumps(meta) + "\n")
    vec = pa.struct([pa.field("type", pa.int8(), False), pa.field("size", pa.int32()),
                     pa.field("indices", pa.list_(pa.field("element", pa.int32(), False))),
                     pa.field("values", pa.list_(pa.field("element", pa.float64(), False)))])

    def dense(v):
        return pa.array([{"type": 1, "size": None, "indices": None, "values": [float(x) for x in v]}], vec)
    t = pa.table({"originalMin": dense(mins), "originalMax": dense(maxs)})
    pq.write_table(t, os.path.join(d, "data", "part-00000.snappy.parquet"), compression="snappy")


def _vector_values(v):
    """A Spark ML vector struct {type, size, indices, values} -> list of doubles (dense: type 1; sparse: type 0)."""
    if v["type"] == 1:
        return [float(x) for x in v["values"]]
    out = [0.0] * int(v["size"])
    for i, x in zip(v["indices"], v["values"]):
        out[i] = float(x)
    return out


def load_minmax_model(model_path):
    """-> (lo, hi, originalMin, originalMax) of a MinMaxScalerModel directory (Spark's own or ours)."""
    import json
    import pyarrow.parquet as pq
    d = os.path.join(model_path, _SCALE_DIR["norm"])
    meta = json.loads(open(_spark_parts(os.path.join(d, "metadata"))[0]).readline())
    pm, dm = meta.get("paramMap", {}), meta.get("defaultParamMap", {})
    lo, hi = float(pm.get("min", dm.get("min", 0.0))), float(pm.get("max", dm.get("max", 1.0)))
    rows = []
    for f in _spark_parts(os.path.join(d, "data")):
        if f.endswith(".parquet"):
            rows += pq.read_table(f).to_pylist()
    return lo, hi, _vector_values(rows[0]["originalMin"]), _vector_values(rows[0]["originalMax"])


def _stddev(rec):
    n = int(rec["n_valid"])
    return math.sqrt(float(rec["m2"]) / (n - 1)) if n > 1 else None


def _nan_free_moments(fr, cols):
    """Moments over the non-null, non-NaN values: float columns whose mean is NaN (they hold NaN, or both infinities) take
    theirs from the NaN-free view, like `_surrogates`.  -> (moments by name, the view, the columns read through it)."""
    mom = profile.moments(fr, cols)
    nan_cols = [c for c in cols if fr.column(c).anv_dtype in (_lib.ANV_F32, _lib.ANV_F64)
                and math.isnan(float(mom[c]["mean"])) and int(mom[c]["n_valid"]) > 0]
    view = _nan_view(fr, nan_cols)
    out = dict(mom)
    if nan_cols:
        out.update(zip(nan_cols, engine.moments(view, nan_cols)))
    return out, view, nan_cols


def _quartiles(fr, cols):
    """approxQuantile(cols, [0.25, 0.5, 0.75], 0.01), which skips NaN as well as null: [] for a column without a value."""
    _, view, nan_cols = _nan_free_moments(fr, cols)
    probs = [0.25, 0.5, 0.75]
    q = dict(profile.quantiles(fr, [c for c in cols if c not in nan_cols], probs, profile.APPROX_QUANTILE_EPS))
    if nan_cols:
        q.update(profile.quantiles(view, nan_cols, probs, profile.APPROX_QUANTILE_EPS))
    return [[] if any(v is None for v in q[c]) else [float(v) for v in q[c]] for c in cols]


def _div_spec(a, b):
    """`(col - a) / b` in Spark: a null parameter or a zero divisor (Divide returns null) -> None (an all-null column)."""
    if a is None or b is None or b == 0:
        return None
    return (_lib.SCALE_DIV, _lib.ANV_F64, 0, float(a), float(b), 0.0)


def minmax_spec(mn, mx, lo=0.0, hi=1.0):
    """MinMaxScalerModel.transform of one feature: scale = (hi - lo) / (max - min); a zero scale (a constant column, or
    an infinite range) maps every value to 0.5 * (hi - lo) + lo.  NaN results become null, the output is float."""
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        rng = np.float64(mx) - np.float64(mn)
        scale = float(np.float64(hi - lo) / rng) if rng != 0 else 0.0
    if scale != 0:
        return (_lib.SCALE_AFFINE, _lib.ANV_F32, _lib.SCALE_NAN_TO_NULL, float(mn), scale, float(lo))
    return (_lib.SCALE_CONST, _lib.ANV_F32, _lib.SCALE_NAN_TO_NULL, 0.0, 0.0, 0.5 * (hi - lo) + lo)


def _apply_scaling(fr, cols, specs, output_mode):
    """Write the scaled columns (spec None: an all-null double column) -> new frame.  "replace": each takes its source's
    name and position; "append": `<c>_scaled` after all existing columns, in list order."""
    run = [i for i, s in enumerate(specs) if s is not None]
    data, valid, nulls = engine.scale_columns(fr, [cols[i] for i in run], [specs[i] for i in run])
    made = {}
    for k, i in enumerate(run):
        src = fr.column(cols[i])
        od = specs[i][1]
        if specs[i][2] & _lib.SCALE_NAN_TO_NULL:
            v, nc = valid[k], int(nulls[k])
        else:
            v, nc = src.device()[1], src.null_count
        made[cols[i]] = Column(cols[i], _SDTYPE_OF_ANV[od], fr.n_rows, dev=data[k], dev_valid=v, anv_dtype=od, null_count=nc)
    for i, s in enumerate(specs):
        if s is None:
            d, _ = fr.column(cols[i]).device()
            torch = _lib.require_cuda()
            made[cols[i]] = Column(cols[i], "double", fr.n_rows, dev=torch.zeros(max(fr.n_rows, 1), dtype=torch.float64,
                                                                                  device=d.device)[:fr.n_rows],
                                   dev_valid=torch.zeros(max((fr.n_rows + 31) // 32, 1), dtype=torch.int32, device=d.device),
                                   anv_dtype=_lib.ANV_F64, null_count=fr.n_rows)
    new = OrderedDict()
    for n in fr.columns:
        new[n] = made[n] if output_mode == "replace" and n in made else fr.column(n)
    if output_mode == "append":
        for c in cols:
            if c in made:
                col = made[c]
                col.name = c + "_scaled"
                new[col.name] = col
    return ColumnFrame(new, fr.n_rows)


def _scaled_frame(fr, cols, specs, output_mode):
    if getattr(fr, "is_partitioned", False):
        schema = _apply_scaling(fr._schema, cols, specs, output_mode)
        return fr.map_chunks(schema, lambda ch: _apply_scaling(ch, cols, specs, output_mode))
    return _apply_scaling(fr, cols, specs, output_mode)


def _describe_value(v, sdtype):
    from ..shared.utils import jvm_double_str
    if v is None or (v != v and sdtype in ("int", "bigint", "long")):
        return "null"
    if sdtype in ("int", "bigint", "long"):
        return str(int(v))
    if sdtype == "float":                  # Float.toString: the shortest float32 digits
        return jvm_double_str(float(str(np.float32(v))))
    return jvm_double_str(v)


def describe(fr, cols):
    """`idf.select(cols).describe()` (count, mean, stddev, min, max as strings) from the moments pass."""
    import pandas as pd
    from ..result import ResultFrame
    mom = profile.moments(fr, cols)
    sdt = dict(fr.dtypes)
    rows = {"count": [], "mean": [], "stddev": [], "min": [], "max": []}
    for c in cols:
        r = mom[c]
        n = int(r["n_valid"])
        rows["count"].append(str(n))
        rows["mean"].append(_describe_value(float(r["mean"]) if n else None, "double"))
        rows["stddev"].append(_describe_value(_stddev(r), "double"))
        rows["min"].append(_describe_value(float(r["min"]) if n else None, sdt[c]))
        rows["max"].append(_describe_value(float(r["max"]) if n else None, sdt[c]))
    return ResultFrame(pd.DataFrame([[k] + v for k, v in rows.items()], columns=["summary"] + list(cols)))


def _print_impact(fr, odf, cols, out_cols):
    print("Before: ")
    describe(fr, cols).show(5, False)
    print("After: ")
    describe(odf, out_cols).show(5, False)


def z_standardization(spark, idf, list_of_cols="all", drop_cols=[], pre_existing_model=False, model_path="NA",
                      output_mode="replace", print_impact=False):
    """Same arguments, errors and returned frame as the reference (transformers.py:965-1099): (x - mean) / stddev as a
    double column that keeps the source's nulls."""
    fr = as_frame(idf)
    cols = _scale_cols(fr, list_of_cols, drop_cols, output_mode, "Standardization")
    if cols is None:
        return fr
    excluded = []
    if pre_existing_model:
        params = _load_param_model(model_path, "z", cols)
    else:
        mom = profile.moments(fr, cols)
        params = []
        for c in cols:
            n = int(mom[c]["n_valid"])
            mean, sd = (float(mom[c]["mean"]) if n else None), _stddev(mom[c])
            params.append([mean if mean else None, sd if sd else None])   # `float(mean) if mean else None`
            if not sd or round(sd, 5) == 0.0:
                excluded.append(c)
    if excluded:
        warnings.warn("The following column(s) are excluded from standardization because the standard deviation is zero:"
                      + str(excluded))
    kept = [c for c in cols if c not in excluded]
    specs = [_div_spec(p[0], p[1]) for c, p in zip(cols, params) if c not in excluded]
    odf = _scaled_frame(fr, kept, specs, output_mode)
    if not pre_existing_model and model_path != "NA":
        _save_param_model(model_path, "z", cols, params)
    if print_impact:
        _print_impact(fr, odf, cols, cols if output_mode == "replace" else [c + "_scaled" for c in kept])
    return odf


def IQR_standardization(spark, idf, list_of_cols="all", drop_cols=[], pre_existing_model=False, model_path="NA",
                        output_mode="replace", print_impact=False):
    """Same arguments, errors and returned frame as the reference (transformers.py:1102-1230): (x - p50) / (p75 - p25)
    with the quartiles of approxQuantile(..., 0.01), as a double column that keeps the source's nulls."""
    fr = as_frame(idf)
    cols = _scale_cols(fr, list_of_cols, drop_cols, output_mode, "Standardization")
    if cols is None:
        return fr
    params = _load_param_model(model_path, "iqr", cols) if pre_existing_model else _quartiles(fr, cols)
    excluded = [c for c, p in zip(cols, params) if len(p) == 0 or round(p[0], 5) == round(p[2], 5)]
    if excluded:
        warnings.warn("The following column(s) are excluded from standardization because the 75th and 25th percentiles "
                      "are the same:" + str(excluded))
    kept = [c for c in cols if c not in excluded]
    specs = [_div_spec(p[1], None if p[2] is None or p[0] is None else p[2] - p[0])
             for c, p in zip(cols, params) if c not in excluded]
    odf = _scaled_frame(fr, kept, specs, output_mode)
    if not pre_existing_model and model_path != "NA":
        _save_param_model(model_path, "iqr", cols, params)
    if print_impact:
        _print_impact(fr, odf, cols, cols if output_mode == "replace" else [c + "_scaled" for c in kept])
    return odf


def normalization(idf, list_of_cols="all", drop_cols=[], pre_existing_model=False, model_path="NA", output_mode="replace",
                  print_impact=False):
    """Same arguments, errors and returned frame as the reference (transformers.py:1233-1366): Spark ML's MinMaxScaler to
    [0, 1] over the non-null, non-NaN values, as a float column; NaN (input or result) becomes null."""
    fr = as_frame(idf)
    cols = _scale_cols(fr, list_of_cols, drop_cols, output_mode, "Normalization")
    if cols is None:
        return fr
    if pre_existing_model:
        lo, hi, mins, maxs = load_minmax_model(model_path)
        if len(mins) != len(cols) or len(maxs) != len(cols):
            raise ValueError("normalization model has %d features, the column list %d" % (len(mins), len(cols)))
    else:
        lo, hi = 0.0, 1.0
        mom, _, _ = _nan_free_moments(fr, cols)
        mins = [float(mom[c]["min"]) if int(mom[c]["n_valid"]) else _DOUBLE_MAX for c in cols]
        maxs = [float(mom[c]["max"]) if int(mom[c]["n_valid"]) else -_DOUBLE_MAX for c in cols]
        if model_path != "NA":
            save_minmax_model(model_path, lo, hi, mins, maxs)
    odf = _scaled_frame(fr, cols, [minmax_spec(a, b, lo, hi) for a, b in zip(mins, maxs)], output_mode)
    if print_impact:
        _print_impact(fr, odf, cols, cols if output_mode == "replace" else [c + "_scaled" for c in cols])
    return odf


# ---- feature_transformation, boxcox_transformation (reference transformers.py:3171-3486) ------------------------------
#
# Every method is one streaming pass (anv_transform_columns) with the semantics of the Spark expression the reference
# builds: StrictMath's fdlibm for log / exp / pow, Spark's result types and nulls, round as HALF_UP of the shortest
# decimal.  Every op is row-local, so a partitioned frame transforms chunk by chunk.  Semantics and deviations: DESIGN.md
# section 1.

_TF_METHODS = ("ln", "log10", "log2", "exp", "powOf2", "powOf10", "powOfN", "sqrt", "cbrt", "sq", "cb", "toPowerN", "sin",
               "cos", "tan", "asin", "acos", "atan", "radians", "remainderDivByN", "factorial", "mul_inv", "floor", "ceil",
               "roundN")
_TF_WITH_N = ("powOfN", "toPowerN", "remainderDivByN", "roundN")
_TF_DOUBLE = {"ln": _lib.TF_LN, "log10": _lib.TF_LOG10, "log2": _lib.TF_LOG2, "exp": _lib.TF_EXP, "sqrt": _lib.TF_SQRT,
              "cbrt": _lib.TF_CBRT, "sin": _lib.TF_SIN, "cos": _lib.TF_COS, "tan": _lib.TF_TAN, "asin": _lib.TF_ASIN,
              "acos": _lib.TF_ACOS, "atan": _lib.TF_ATAN, "radians": _lib.TF_RADIANS, "mul_inv": _lib.TF_MUL_INV}
_TF_POW = {"powOf2": (_lib.TF_POW_BASE, 2.0), "powOf10": (_lib.TF_POW_BASE, 10.0), "sq": (_lib.TF_POW, 2.0),
           "cb": (_lib.TF_POW, 3.0)}
_INT_RANK = {_lib.ANV_I32: 0, _lib.ANV_I64: 1, _lib.ANV_F32: 2, _lib.ANV_F64: 3}


def _number(N, method_type):
    if isinstance(N, bool) or not isinstance(N, (int, float)):
        raise TypeError("N must be a number for method_type %s" % method_type)
    return N


def _literal_dtype(N):
    """The type of F.lit(N): int in 32 bits -> int, other ints -> bigint, float -> double."""
    if isinstance(N, float):
        return _lib.ANV_F64
    return _lib.ANV_I32 if -(1 << 31) <= N < (1 << 31) else _lib.ANV_I64


def transform_spec(method_type, N, in_dtype):
    """The anv_transform_columns spec (op, out dtype, n, a) of one column, or (None, out dtype) for a column that is all
    null (x % 0, Spark's Remainder by zero)."""
    if method_type in _TF_DOUBLE:
        return (_TF_DOUBLE[method_type], _lib.ANV_F64, 0, 0.0)
    if method_type in _TF_POW:
        op, a = _TF_POW[method_type]
        return (op, _lib.ANV_F64, 0, a)
    if method_type in ("powOfN", "toPowerN"):
        if N is None:                                   # F.pow(None, x) / x ** None: a null literal, an all-null column
            return (None, _lib.ANV_F64)
        return (_lib.TF_POW_BASE if method_type == "powOfN" else _lib.TF_POW, _lib.ANV_F64, 0, float(_number(N, method_type)))
    if method_type in ("floor", "ceil", "factorial"):
        op = {"floor": _lib.TF_FLOOR, "ceil": _lib.TF_CEIL, "factorial": _lib.TF_FACTORIAL}[method_type]
        return (op, _lib.ANV_I64, 0, 0.0)
    if method_type == "remainderDivByN":
        if N is None:                                   # x % F.lit(None): null in the column's type
            return (None, in_dtype)
        N = _number(N, method_type)
        lit = _literal_dtype(N)
        od = in_dtype if _INT_RANK[in_dtype] >= _INT_RANK[lit] else lit
        if N == 0:
            return (None, od)
        if od in (_lib.ANV_F32, _lib.ANV_F64):
            a = float(np.float32(N)) if od == _lib.ANV_F32 else float(N)
            return (_lib.TF_REMAINDER, od, 0, a)
        return (_lib.TF_REMAINDER, od, int(N), 0.0)
    # roundN: F.round(x, N) takes an int scale
    if isinstance(N, bool) or not isinstance(N, int):
        raise TypeError("N must be an integer for method_type roundN")
    if in_dtype in (_lib.ANV_F32, _lib.ANV_F64) and not -22 <= N <= 22:
        raise ValueError("roundN of a float or double column takes -22 <= N <= 22 on the device, got %d" % N)
    return (_lib.TF_ROUND, in_dtype, int(N), 0.0)


def _transform_cols(fr, list_of_cols, drop_cols):
    """The reference's column checks: -> the numeric columns, first-seen order."""
    num_cols = attributeType_segregation(fr)[0]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num_cols
    drop = _names(drop_cols)
    cols = [c for c in dict.fromkeys(_names(list_of_cols)) if c not in drop]
    if len(cols) == 0 or any(c not in num_cols for c in cols):
        raise TypeError("Invalid input for Column(s)")
    sdt = dict(fr.dtypes)
    for c in cols:
        if sdt[c] not in _ANV_OF_SDTYPE:
            raise TypeError("transformation of %s column %r is not supported on the device" % (sdt[c], c))
    return cols


def _apply_transform(fr, cols, specs, out_names):
    """Write op(col) for each (col, spec) under its output name -> new frame: a name that exists keeps its position (the
    reference's withColumn), a new one goes after all existing columns, in list order."""
    torch = None
    run = [i for i, s in enumerate(specs) if s[0] is not None]
    data, valid, nulls = engine.transform_columns(fr, [cols[i] for i in run], [specs[i] for i in run])
    made = {}
    for k, i in enumerate(run):
        src = fr.column(cols[i])
        od = specs[i][1]
        if valid[k] is not None:
            v, nc = valid[k], int(nulls[k])
        else:
            v, nc = src.device()[1], src.null_count
        made[out_names[i]] = Column(out_names[i], _SDTYPE_OF_ANV[od], fr.n_rows, dev=data[k], dev_valid=v, anv_dtype=od,
                                    null_count=nc)
    for i, s in enumerate(specs):
        if s[0] is None:
            torch = torch or _lib.require_cuda()
            d, _ = fr.column(cols[i]).device()
            od = s[1]
            made[out_names[i]] = Column(out_names[i], _SDTYPE_OF_ANV[od], fr.n_rows,
                                        dev=torch.zeros(max(fr.n_rows, 1), dtype=getattr(torch, engine._TORCH_OF_ANV[od]),
                                                        device=d.device)[:fr.n_rows],
                                        dev_valid=torch.zeros(max((fr.n_rows + 31) // 32, 1), dtype=torch.int32,
                                                              device=d.device),
                                        anv_dtype=od, null_count=fr.n_rows)
    new = OrderedDict()
    for n in fr.columns:
        new[n] = made.pop(n) if n in made else fr.column(n)
    for n in out_names:
        if n in made:
            new[n] = made.pop(n)
    return ColumnFrame(new, fr.n_rows)


def _transformed_frame(fr, cols, specs, out_names):
    if getattr(fr, "is_partitioned", False):
        schema = _apply_transform(fr._schema, cols, specs, out_names)
        return fr.map_chunks(schema, lambda ch: _apply_transform(ch, cols, specs, out_names))
    return _apply_transform(fr, cols, specs, out_names)


def feature_transformation(idf, list_of_cols="all", drop_cols=[], method_type="sqrt", N=None, output_mode="replace",
                           print_impact=False):
    """Same arguments, errors and returned frame as the reference (transformers.py:3171-3324): one of 25 row-wise maths
    transforms, with Spark's result types and nulls."""
    fr = as_frame(idf)
    cols = _transform_cols(fr, list_of_cols, drop_cols)
    if method_type not in _TF_METHODS:
        raise TypeError("Invalid input method_type")
    sdt = dict(fr.dtypes)
    specs = [transform_spec(method_type, N, _ANV_OF_SDTYPE[sdt[c]]) for c in cols]
    if output_mode == "replace":
        out_names = list(cols)
    elif method_type in _TF_WITH_N:
        out_names = [c + "_" + method_type[:-1] + str(N) for c in cols]
    else:
        out_names = [c + "_" + method_type for c in cols]
    odf = _transformed_frame(fr, cols, specs, out_names)
    if print_impact:
        print("Before:")
        describe(fr, cols).show(5, False)
        print("After:")
        describe(odf, out_names).show(5, False)
    return odf


BOXCOX_LAMBDAS = (1, -1, 0.5, -0.5, 2, -2, 0.25, -0.25, 3, -3, 4, -4, 5, -5)


def ks_statistics(fr, c):
    """The Kolmogorov-Smirnov statistic against N(0, 1) of pow(c, lambda) for each BOXCOX_LAMBDAS and of log(c), over all
    rows with null rows as the value 0 (recalled from PySpark: `rdd.flatMap` hands None to the JVM, which unboxes it as
    0.0).  One sort and one candidate pass on the device (anv_ks_candidates); the run of zeros adds one term here."""
    n = fr.n_rows
    n_null = n - int(profile.moments(fr, [c])[c]["n_valid"])
    d, below = engine.ks_candidates(fr, c, BOXCOX_LAMBDAS, n_null)
    if n_null:
        for k in range(len(d)):
            a = below if k == len(BOXCOX_LAMBDAS) else 0       # zeros sit after the log values below 0
            d[k] = max(d[k], 0.5 - a / n, (a + n_null) / n - 0.5)
    return d


def boxcox_search(fr, cols):
    """The reference's lambda search (transformers.py:3424-3443), its selection loop kept literally: per column the first
    candidate with a strictly larger p-value wins, starting from 0; a column where none beats 0 keeps the previous
    column's lambda, and the first column raises UnboundLocalError."""
    from ..shared.ks import p_value
    if getattr(fr, "is_partitioned", False):                 # the test needs each column whole
        import pyarrow as pa
        fr = as_frame(pa.concat_tables([ch.to_arrow().select(cols) for ch in fr.chunks(cols)]))
    out, best = [], None
    for c in cols:
        d = ks_statistics(fr, c)
        best_p = 0
        for lam, dk in zip(list(BOXCOX_LAMBDAS) + [0], d):
            p = p_value(float(dk), fr.n_rows)
            if p > best_p:
                best_p, best = p, lam
        if best is None:
            raise UnboundLocalError("cannot access local variable 'best_lambdaVal' where it is not associated with a value")
        out.append(best)
    return out


def skewness_row(fr, cols):
    """`F.skewness` of each column from the moments pass: sqrt(n) * m3 / sqrt(m2^3), null for n = 0 or m2 = 0."""
    from ..shared.utils import jvm_double_str
    mom = profile.moments(fr, cols)
    out = []
    for c in cols:
        n, m2, m3 = int(mom[c]["n_valid"]), float(mom[c]["m2"]), float(mom[c]["m3"])
        out.append("null" if n == 0 or m2 == 0 else jvm_double_str(math.sqrt(n) * m3 / math.sqrt(m2 * m2 * m2)))
    return out


def _describe_skew(fr, cols):
    import pandas as pd
    from ..result import ResultFrame
    d = describe(fr, cols).toPandas()
    d = pd.concat([d, pd.DataFrame([["skewness"] + skewness_row(fr, cols)], columns=d.columns)], ignore_index=True)
    return ResultFrame(d)


def boxcox_transformation(idf, list_of_cols="all", drop_cols=[], boxcox_lambda=None, output_mode="replace",
                          print_impact=False):
    """Same arguments, errors and returned frame as the reference (transformers.py:3327-3486): pow(x, lambda), or log(x)
    for lambda 0; lambda 1 leaves the column as it is.  boxcox_lambda=None picks each column's lambda by the reference's
    Kolmogorov-Smirnov search (boxcox_search)."""
    fr = as_frame(idf)
    cols = _transform_cols(fr, list_of_cols, drop_cols)
    mom = profile.moments(fr, cols)
    mins = [float(mom[c]["min"]) if int(mom[c]["n_valid"]) else None for c in cols]
    if any(m is None for m in mins):
        raise TypeError("'<=' not supported between instances of 'NoneType' and 'int'")
    if any(m <= 0 for m in mins):
        print(" ".join("min(%s)=%r" % (c, m) for c, m in zip(cols, mins)))
        raise ValueError("Data must be positive")
    if boxcox_lambda is None:
        lambdas = boxcox_search(fr, cols)
    elif isinstance(boxcox_lambda, (list, tuple)):
        if len(boxcox_lambda) != len(cols) or not all(isinstance(v, (float, int)) for v in boxcox_lambda):
            raise TypeError("Invalid input for boxcox_lambda")
        lambdas = list(boxcox_lambda)
    elif isinstance(boxcox_lambda, (float, int)):
        lambdas = [boxcox_lambda] * len(cols)
    else:
        raise TypeError("Invalid input for boxcox_lambda")
    run = [(c, lam) for c, lam in zip(cols, lambdas) if lam != 1]
    if not run:
        warnings.warn("lambdaVal for all columns are 1 so no transformation is performed and idf is returned")
        return idf
    specs = [(_lib.TF_LN, _lib.ANV_F64, 0, 0.0) if lam == 0 else (_lib.TF_POW, _lib.ANV_F64, 0, float(lam)) for _, lam in run]
    out_names = [c + "_bxcx_" + str(lam) if output_mode == "append" else c for c, lam in run]
    odf = _transformed_frame(fr, [c for c, _ in run], specs, out_names)
    if print_impact:
        print("Transformed Columns: ", cols)
        print("Best BoxCox Parameter(s): ", lambdas)
        print("Before:")
        _describe_skew(fr, cols).show(6, False)
        print("After:")
        _describe_skew(odf, cols if output_mode == "replace" else out_names).show(6, False)
    return odf


# ---- categorical encoding: cat_to_num_unsupervised, cat_to_num_supervised, outlier_categories ------------------------
# (reference transformers.py:428-962, 3489-3671)
#
# Every fit reads the per-category counts of the code histogram pass (profile.code_counts, merged over row chunks); the
# supervised encoder adds one masked pass for the event rows.  Every transform is one streaming pass: anv_code_map looks
# each row's code up in a per-column table (label index, rate or new code), anv_one_hot expands it into n + 1 dense int
# columns.  Dictionaries are not sorted in general (imputation_MMM appends its fill strings), so every order below comes
# from an explicit sort of the categories with a nonzero count, in UTF-8 byte order as Spark compares strings.  Semantics
# and deviations: DESIGN.md section 1.

_OUTLIER = "outlier_categories"
_INDEX_ORDERS = ("frequencyDesc", "frequencyAsc", "alphabetDesc", "alphabetAsc")
_PRINT_TYPE = {"string": "string", "int": "integer", "bigint": "long", "long": "long", "float": "float",
               "double": "double"}


def _utf8(s):
    return s.encode("utf-8")


def _split(x):
    return [s.strip() for s in x.split("|")] if isinstance(x, str) else list(x)


def _present(fr, cols):
    """-> {col: [(category, count)]} over the categories with a nonzero count, and {col: null rows}."""
    cc = profile.code_counts(fr, cols)
    out, nulls = {}, {}
    for c in cols:
        h, dic = cc[c], fr.column(c).dictionary
        out[c] = [(dic[k], int(h[k + 1])) for k in range(len(dic)) if int(h[k + 1]) > 0]
        nulls[c] = int(h[0])
    return out, nulls


def string_indexer_labels(counts, index_order):
    """StringIndexer (Spark 3) labels of [(category, count)]: frequency orders break ties by label ascending."""
    if index_order == "frequencyDesc":
        key = lambda t: (-t[1], _utf8(t[0]))          # noqa: E731
    elif index_order == "frequencyAsc":
        key = lambda t: (t[1], _utf8(t[0]))           # noqa: E731
    else:
        key = lambda t: _utf8(t[0])                   # noqa: E731
    labels = [t[0] for t in sorted(counts, key=key)]
    return labels[::-1] if index_order == "alphabetDesc" else labels


def _label_index(dictionary, labels):
    """int32 table of len(dictionary) + 1 entries: a category's position in `labels`, n for one it lacks and the null slot
    (StringIndexer's handleInvalid="keep")."""
    pos = {s: i for i, s in enumerate(labels)}
    return np.array([pos.get(s, len(labels)) for s in dictionary] + [len(labels)], np.int32)


def _write_json_part(d, obj):
    import json
    os.makedirs(d)
    with open(os.path.join(d, "part-00000"), "w") as f:
        f.write(json.dumps(obj) + "\n")
    open(os.path.join(d, "_SUCCESS"), "w").close()


def _read_json_part(d):
    import json
    return json.loads(open(_spark_parts(d)[0]).readline())


def save_indexer_model(model_path, cols, labels, index_order):
    """Spark 3 StringIndexerModel directory at <model_path>/cat_to_num_unsupervised/indexer: metadata/part-00000 (one
    JSON line) and data/*.parquet (one row, labelsArray: array<array<string>>)."""
    import time
    import uuid
    import pyarrow as pa
    import pyarrow.parquet as pq
    d = os.path.join(model_path, "cat_to_num_unsupervised", "indexer")
    _clear_dir(d)
    uid = "StringIndexer_" + uuid.uuid4().hex[:12]
    _write_json_part(os.path.join(d, "metadata"), {
        "class": "org.apache.spark.ml.feature.StringIndexerModel", "timestamp": int(time.time() * 1000),
        "sparkVersion": "3.2.1", "uid": uid,
        "paramMap": {"inputCols": list(cols), "outputCols": [c + "_index" for c in cols], "stringOrderType": index_order,
                     "handleInvalid": "keep"},
        "defaultParamMap": {"outputCol": uid + "__output", "stringOrderType": "frequencyDesc", "handleInvalid": "error"}})
    os.makedirs(os.path.join(d, "data"))
    t = pa.table({"labelsArray": pa.array([[list(x) for x in labels]], pa.list_(pa.list_(pa.string())))})
    pq.write_table(t, os.path.join(d, "data", "part-00000.snappy.parquet"), compression="snappy")
    open(os.path.join(d, "data", "_SUCCESS"), "w").close()


def load_indexer_model(model_path):
    """-> {input col: labels} of a StringIndexerModel directory (Spark 3's own or ours)."""
    import pyarrow.parquet as pq
    d = os.path.join(model_path, "cat_to_num_unsupervised", "indexer")
    pm = _read_json_part(os.path.join(d, "metadata")).get("paramMap", {})
    ins = pm.get("inputCols") or [pm["inputCol"]]
    rows = []
    for f in _spark_parts(os.path.join(d, "data")):
        if f.endswith(".parquet"):
            rows += pq.read_table(f).to_pylist()
    labels = rows[0]["labelsArray"] if "labelsArray" in rows[0] else [rows[0]["labels"]]
    return dict(zip(ins, labels))


def save_onehot_model(model_path, cols):
    """The OneHotEncoder estimator at <model_path>/cat_to_num_unsupervised/encoder: metadata/part-00000 only."""
    import time
    import uuid
    d = os.path.join(model_path, "cat_to_num_unsupervised", "encoder")
    _clear_dir(d)
    uid = "OneHotEncoder_" + uuid.uuid4().hex[:12]
    _write_json_part(os.path.join(d, "metadata"), {
        "class": "org.apache.spark.ml.feature.OneHotEncoder", "timestamp": int(time.time() * 1000),
        "sparkVersion": "3.2.1", "uid": uid,
        "paramMap": {"inputCols": [c + "_index" for c in cols], "outputCols": [c + "_vec" for c in cols],
                     "handleInvalid": "keep"},
        "defaultParamMap": {"outputCol": uid + "__output", "dropLast": True, "handleInvalid": "error"}})


def _free_device_bytes():
    """Free device memory, counting what torch's allocator holds unused."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    return int(free) + int(torch.cuda.memory_reserved()) - int(torch.cuda.memory_allocated())


def _apply_label(fr, cols, labels, output_mode):
    tables = [_label_index(fr.column(c).dictionary, labels[c]) for c in cols]
    data, _, _ = engine.code_map(fr, cols, tables, [None] * len(cols))
    made = OrderedDict()
    for c, d in zip(cols, data):
        src = fr.column(c)
        name = c if output_mode == "replace" else c + "_index"
        made[name] = Column(name, "int", fr.n_rows, dev=d, dev_valid=src.device()[1], anv_dtype=_lib.ANV_I32,
                            null_count=src.null_count)
    new = OrderedDict((n, made[n] if n in made else fr.column(n)) for n in fr.columns)
    for n, col in made.items():
        new.setdefault(n, col)
    return ColumnFrame(new, fr.n_rows)


def _apply_onehot(fr, cols, labels, output_mode):
    stride = engine.one_hot_stride(fr.n_rows)
    free, need = _free_device_bytes() if fr.n_rows else 0, 0
    for c in cols:                                   # one engine.one_hot call allocates the outputs of every column
        need += (len(labels[c]) + 1) * stride * 4
        if fr.n_rows and need > free:
            raise _lib.AnvError("one-hot encoding of column %r needs %d output columns; with the columns before it that "
                                "is %.1f GB of device memory, more than the %.1f GB free: drop columns, lower "
                                "cardinality_threshold or cap the categories with outlier_categories"
                                % (c, len(labels[c]) + 1, need / 1e9, free / 1e9))
    idx = [_label_index(fr.column(c).dictionary, labels[c]) for c in cols]
    outs = engine.one_hot(fr, cols, idx, [len(labels[c]) + 1 for c in cols])
    new = OrderedDict((n, fr.column(n)) for n in fr.columns if not (output_mode == "replace" and n in cols))
    for c, o in zip(cols, outs):
        for j in range(len(labels[c]) + 1):
            name = "%s_%d" % (c, j)
            new[name] = Column(name, "int", fr.n_rows, dev=o[j], anv_dtype=_lib.ANV_I32, null_count=0)
    return ColumnFrame(new, fr.n_rows)


def _per_chunk(fr, fn):
    if getattr(fr, "is_partitioned", False):
        return fr.map_chunks(fn(fr._schema), fn)
    return fn(fr)


def _summary_value(v, sdtype):
    return "null" if v is None else _describe_value(v, sdtype)


def summary_count_min_max(fr, cols):
    """`idf.select(cols).summary("count", "min", "max")`: strings compare in UTF-8 order, numbers through the moments."""
    import pandas as pd
    from ..result import ResultFrame
    cat = [c for c in cols if fr.column(c).kind == "cat"]
    num = [c for c in cols if c not in cat]
    present, _ = _present(fr, cat) if cat else ({}, {})
    mom = profile.moments(fr, num) if num else {}
    sdt = dict(fr.dtypes)
    rows = {"count": [], "min": [], "max": []}
    for c in cols:
        if c in present:
            keys = sorted((k for k, _ in present[c]), key=_utf8)
            rows["count"].append(str(sum(n for _, n in present[c])))
            rows["min"].append(keys[0] if keys else "null")
            rows["max"].append(keys[-1] if keys else "null")
        else:
            n = int(mom[c]["n_valid"])
            rows["count"].append(str(n))
            rows["min"].append(_summary_value(float(mom[c]["min"]) if n else None, sdt[c]))
            rows["max"].append(_summary_value(float(mom[c]["max"]) if n else None, sdt[c]))
    return ResultFrame(pd.DataFrame([[k] + v for k, v in rows.items()], columns=["summary"] + list(cols)))


def print_schema(fr, cols):
    """`idf.select(cols).printSchema()` text."""
    sdt = dict(fr.dtypes)
    return "root\n" + "".join(" |-- %s: %s (nullable = true)\n" % (c, _PRINT_TYPE.get(sdt[c], sdt[c])) for c in cols)


def _unique_over(fr, cols, cardinality_threshold, stats_unique):
    """Columns whose unique count exceeds the threshold, from the code counts or a saved uniqueCount table."""
    if stats_unique == {}:
        present, _ = _present(fr, cols)
        return [c for c in cols if len(present[c]) > cardinality_threshold]
    from ..data_analyzer.quality_checker import _read_stats
    df = _read_stats(stats_unique, ["attribute", "unique_values"])
    return [a for a, u in zip(df["attribute"].tolist(), df["unique_values"].tolist()) if float(u) > cardinality_threshold]


def cat_to_num_unsupervised(spark, idf, list_of_cols="all", drop_cols=[], method_type="label_encoding",
                            index_order="frequencyDesc", cardinality_threshold=50, pre_existing_model=False,
                            model_path="NA", stats_unique={}, output_mode="replace", print_impact=False):
    """Same arguments, errors and returned frame as the reference (transformers.py:506-773, Spark 3): StringIndexer labels
    (handleInvalid="keep") as an int column that keeps the source's nulls, or OneHotEncoder (keep, dropLast) as n + 1
    dense int columns `<c>_0 .. <c>_n` appended after all columns, where nulls and unseen categories set `<c>_n`."""
    fr = as_frame(idf)
    cat_cols = attributeType_segregation(fr)[1]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = cat_cols
    list_of_cols, drop_cols = _split(list_of_cols), _split(drop_cols)
    if any(x not in cat_cols for x in list_of_cols):
        raise TypeError("Invalid input for Column(s)")
    if method_type not in ("onehot_encoding", "label_encoding"):
        raise TypeError("Invalid input for method_type")
    if index_order not in _INDEX_ORDERS:
        raise TypeError("Invalid input for Encoding Index Order")
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")
    wanted = [c for c in dict.fromkeys(list_of_cols)]
    over = set(_unique_over(fr, wanted, cardinality_threshold, stats_unique))
    skip = [c for c in wanted if c in over and c not in drop_cols]
    if skip:
        warnings.warn("Columns dropped from encoding due to high cardinality: " + ",".join(skip))
    cols = [c for c in wanted if c not in drop_cols + skip]
    if not cols:
        warnings.warn("No Encoding Computation - No categorical column(s) to transform")
        return fr

    if pre_existing_model:
        model = load_indexer_model(model_path)
        for c in cols:
            if c not in model:
                raise ValueError("cannot resolve '%s_index' given input columns" % c)
        labels = {c: list(model[c]) for c in cols}
        if method_type == "onehot_encoding":
            _read_json_part(os.path.join(model_path, "cat_to_num_unsupervised", "encoder", "metadata"))
    else:
        present, _ = _present(fr, cols)
        labels = {c: string_indexer_labels(present[c], index_order) for c in cols}
        if model_path != "NA":
            save_indexer_model(model_path, cols, [labels[c] for c in cols], index_order)
            if method_type == "onehot_encoding":
                save_onehot_model(model_path, cols)

    if method_type == "onehot_encoding":
        odf = _per_chunk(fr, lambda f: _apply_onehot(f, cols, labels, output_mode))
    else:
        odf = _per_chunk(fr, lambda f: _apply_label(f, cols, labels, output_mode))
    if print_impact:
        if method_type == "label_encoding":
            new_cols = cols if output_mode == "replace" else [c + "_index" for c in cols]
            print("Before")
            summary_count_min_max(fr, cols).show(3, False)
            print("After")
            summary_count_min_max(odf, new_cols).show(3, False)
        else:
            new_cols = ["%s_%d" % (c, j) for c in cols for j in range(len(labels[c]) + 1)]
            print("Before")
            print(print_schema(fr, cols))
            print("After")
            print(print_schema(odf, (cols if output_mode == "append" else []) + new_cols))
        if skip:
            print("Columns dropped from encoding due to high cardinality: " + ",".join(skip))
    return odf


def _csv_field(v):
    """A field as Spark's CSV writer puts it: null -> empty, "" -> \"\", quotes where needed, `\\` escapes quotes."""
    if v is None:
        return ""
    if v == "" or any(ch in v for ch in ',"\n\r\\'):
        return '"' + v.replace("\\", "\\\\").replace('"', '\\"') + '"'
    return v


def _csv_rows(path):
    """Rows of a CSV file written by Spark or by _csv_field: an unquoted empty field is None, a quoted one ""."""
    rows = []
    for line in open(path, encoding="utf-8").read().splitlines():
        out, i = [], 0
        while True:
            if i < len(line) and line[i] == '"':
                j, buf = i + 1, []
                while j < len(line) and line[j] != '"':
                    if line[j] == "\\" and j + 1 < len(line):
                        j += 1
                    buf.append(line[j])
                    j += 1
                out.append("".join(buf))
                i = j + 1
            else:
                j = line.find(",", i)
                j = len(line) if j < 0 else j
                out.append(line[i:j] if j > i else None)
                i = j
            if i >= len(line):
                break
            i += 1                                   # the comma
            if i == len(line):
                out.append(None)
                break
        rows.append(out)
    return rows


def _write_csv_dir(d, header, rows):
    _clear_dir(d)
    with open(os.path.join(d, "part-00000-c000.csv"), "w", encoding="utf-8") as f:
        f.write(",".join(header) + "\n")
        for r in rows:
            f.write(",".join(_csv_field(v) for v in r) + "\n")
    open(os.path.join(d, "_SUCCESS"), "w").close()


def _read_csv_dir(d):
    rows = []
    for fn in _spark_parts(d):
        if fn.endswith(".csv"):
            rows += _csv_rows(fn)[1:]
    return rows


def save_supervised_model(model_path, col, table):
    """<model_path>/cat_to_num_supervised/<col>/part-*.csv, header `<col>,<col>_encoded`: keys verbatim (null -> empty
    field), values as java.lang.Double.toString."""
    from ..shared.utils import jvm_double_str
    _write_csv_dir(os.path.join(model_path, "cat_to_num_supervised", col), [col, col + "_encoded"],
                   [[k, jvm_double_str(v)] for k, v in table])


def load_supervised_model(model_path, col):
    """-> [(key | None, value | None)] of a saved supervised model, keys read as strings."""
    return [(r[0], None if len(r) < 2 or r[1] is None else float(r[1]))
            for r in _read_csv_dir(os.path.join(model_path, "cat_to_num_supervised", col))]


def _class_counts(fr, cols, label_col, event_label):
    """-> ({col: all counts [size + 1]}, {col: event counts [size + 1]}, event rows, rows); slot 0 = the null group.  The
    event class is label == event_label; every other row, a null label included, is class "0"."""
    from ..shared.label_classes import label_bitmaps, masked
    allc = profile.code_counts(fr, cols)
    if getattr(fr, "is_partitioned", False):
        n_event = sum(label_bitmaps(ch, label_col, event_label)[2] for ch in fr.chunks([label_col]))
        if fr.group is not None:                     # row slabs on several ranks: the counts below are all-reduced
            n_event = int(fr.group.all_reduce(np.array([n_event], np.int64))[0])
        view = fr.map_chunks(fr._schema.select(cols), lambda ch: masked(ch, cols, label_bitmaps(ch, label_col, event_label)[0]))
    else:
        ev_w, _, n_event = label_bitmaps(fr, label_col, event_label)
        view = masked(fr, cols, ev_w)
    ev = {}
    for c, h in zip(cols, engine.code_counts(view, cols)):
        h = np.asarray(h, np.int64).copy()
        h[0] = n_event - int(h[1:].sum())            # slot 0 of the masked pass mixes null and non-event rows
        ev[c] = h
    return {c: np.asarray(allc[c], np.int64) for c in cols}, ev, n_event, fr.n_rows


def _supervised_table(fr, c, allc, ev):
    """The reference's pivot: [(category | None, round(c1 / (c1 + c0), 4))] over the groups with rows."""
    from ..shared.utils import spark_round
    dic = fr.column(c).dictionary
    out = [(None, spark_round(ev[0] / allc[0], 4))] if allc[0] else []
    order = sorted((k for k in range(len(dic)) if allc[k + 1]), key=lambda k: _utf8(dic[k]))
    return out + [(dic[k], spark_round(ev[k + 1] / allc[k + 1], 4)) for k in order]


def _rate_table(dictionary, model):
    """code_map table (float64) and entry validity of a supervised model: more than one row joins on the key (null rows
    and keys the model lacks become null); exactly one row is a cross join (every row gets it, nulls included)."""
    n = len(dictionary)
    if len(model) == 1:
        v = model[0][1]
        return np.full(n + 1, 0.0 if v is None else v, np.float64), np.full(n + 1, v is not None)
    m = {k: v for k, v in model if k is not None}
    vals = [m.get(s) for s in dictionary] + [None]
    return np.array([0.0 if v is None else v for v in vals], np.float64), np.array([v is not None for v in vals])


def _apply_rates(fr, cols, models, output_mode):
    tabs = [_rate_table(fr.column(c).dictionary, models[c]) for c in cols]
    data, valid, nulls = engine.code_map(fr, cols, [t for t, _ in tabs], [v for _, v in tabs])
    made = OrderedDict()
    for c, d, v, nc in zip(cols, data, valid, nulls):
        name = c if output_mode == "replace" else c + "_encoded"
        made[name] = Column(name, "double", fr.n_rows, dev=d, dev_valid=v, anv_dtype=_lib.ANV_F64, null_count=int(nc))
    new = OrderedDict((n, made[n] if n in made else fr.column(n)) for n in fr.columns)
    for n, col in made.items():
        new.setdefault(n, col)
    return ColumnFrame(new, fr.n_rows)


def cat_to_num_supervised(spark, idf, list_of_cols="all", drop_cols=[], label_col="label", event_label=1,
                          pre_existing_model=False, model_path="NA", output_mode="replace", persist=False,
                          persist_option=None, print_impact=False):
    """Same arguments, errors and returned frame as the reference (transformers.py:776-962): each category becomes its
    event rate round(c1 / (c1 + c0), 4) as a double column.  `persist` / `persist_option` are accepted and have nothing
    to do on a resident frame.  model_path="NA" keeps the table in memory instead of round-tripping it through
    `intermediate_data/`."""
    fr = as_frame(idf)
    cat_cols = attributeType_segregation(fr)[1]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = cat_cols
    list_of_cols, drop_cols = _split(list_of_cols), _split(drop_cols)
    cols = [e for e in dict.fromkeys(list_of_cols) if e not in drop_cols and e != label_col]
    if any(x not in cat_cols for x in cols):
        raise TypeError("Invalid input for Column(s)")
    if not cols:
        warnings.warn("No Categorical Encoding - No categorical column(s) to transform")
        return fr
    if label_col not in fr.columns:
        raise TypeError("Invalid input for Label Column")

    if pre_existing_model:
        path = model_path if model_path != "NA" else "intermediate_data"
        models = {c: load_supervised_model(path, c) for c in cols}
    else:
        allc, ev, n_event, n_rows = _class_counts(fr, cols, label_col, event_label)
        if n_event == 0 or n_event == n_rows:
            raise ValueError("cannot resolve '%s' given input columns: the label has no %s rows"
                             % ("1" if n_event == 0 else "0", "event" if n_event == 0 else "non-event"))
        models = {c: _supervised_table(fr, c, allc[c], ev[c]) for c in cols}
        if model_path != "NA":
            for c in cols:
                save_supervised_model(model_path, c, models[c])
    odf = _per_chunk(fr, lambda f: _apply_rates(f, cols, models, output_mode))
    if print_impact:
        out_cols = cols if output_mode == "replace" else [c + "_encoded" for c in cols]
        print("Before: ")
        summary_count_min_max(fr, cols).show(3, False)
        print("After: ")
        summary_count_min_max(odf, out_cols).show(3, False)
    return odf


def outlier_kept(counts, coverage, max_category):
    """The categories outlier_categories keeps of [(category, count)] (non-null): in count-descending order (ties in UTF-8
    order), with count_pct = count / total, rank = Spark's rank(), cumu = the running sum of count_pct and lag_cumu the
    previous cumu (0 for the first), keep where not (cumu >= coverage and lag_cumu >= coverage) and rank <= max - 1."""
    items = sorted(counts, key=lambda t: (-t[1], _utf8(t[0])))
    total = float(sum(n for _, n in items))
    kept, cumu, rank, prev = [], 0.0, 0, None
    for i, (k, n) in enumerate(items):
        if n != prev:
            rank, prev = i + 1, n
        lag = cumu
        cumu += n / total
        if not (cumu >= coverage and lag >= coverage) and rank <= max_category - 1:
            kept.append(k)
    return kept


def save_outlier_model(model_path, params):
    """<model_path>/outlier_categories/part-*.csv with `attribute,parameters` rows.  Spark's CSV writer trims leading and
    trailing whitespace by default, so the saved categories are trimmed."""
    _write_csv_dir(os.path.join(model_path, "outlier_categories"), ["attribute", "parameters"],
                   [[c, k.strip()] for c, ks in params for k in ks])


def load_outlier_model(model_path):
    out = {}
    for r in _read_csv_dir(os.path.join(model_path, "outlier_categories")):
        if r and r[0] is not None:
            out.setdefault(r[0], []).append(r[1] if len(r) > 1 else None)
    return out


def _outlier_map(dictionary, kept):
    """-> (new dictionary: the kept categories and "outlier_categories" once, in UTF-8 order; int32 code table)."""
    keep = set(kept)
    new = sorted(set(s for s in dictionary if s in keep) | {_OUTLIER}, key=_utf8)
    pos = {s: i for i, s in enumerate(new)}
    return new, np.array([pos[s] if s in keep else pos[_OUTLIER] for s in dictionary] + [0], np.int32)


def _apply_outliers(fr, cols, params, output_mode):
    maps = [_outlier_map(fr.column(c).dictionary, params.get(c) or []) for c in cols]
    data, _, _ = engine.code_map(fr, cols, [t for _, t in maps], [None] * len(cols))
    made = OrderedDict()
    for c, d, (dic, _) in zip(cols, data, maps):
        src = fr.column(c)
        name = c if output_mode == "replace" else c + "_outliered"
        made[name] = Column(name, "string", fr.n_rows, dev=d, dev_valid=src.device()[1], anv_dtype=_lib.ANV_I32,
                            null_count=src.null_count, dictionary=dic)
    new = OrderedDict((n, made[n] if n in made else fr.column(n)) for n in fr.columns)
    for n, col in made.items():
        new.setdefault(n, col)
    return ColumnFrame(new, fr.n_rows)


def outlier_categories(spark, idf, list_of_cols="all", drop_cols=[], coverage=1.0, max_category=50,
                       pre_existing_model=False, model_path="NA", output_mode="replace", print_impact=False):
    """Same arguments, errors and returned frame as the reference (transformers.py:3489-3671): the less frequent
    categories of each column become "outlier_categories"; nulls stay null."""
    fr = as_frame(idf)
    cat_cols = attributeType_segregation(fr)[1]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = cat_cols
    list_of_cols, drop_cols = _split(list_of_cols), _split(drop_cols)
    cols = [e for e in dict.fromkeys(list_of_cols) if e not in drop_cols]
    if any(x not in cat_cols for x in cols):
        raise TypeError("Invalid input for Column(s)")
    if not cols:
        warnings.warn("No Outlier Categories Computation - No categorical column(s) to transform")
        return fr
    if (coverage <= 0) | (coverage > 1):
        raise TypeError("Invalid input for Coverage Value")
    if max_category < 2:
        raise TypeError("Invalid input for Maximum No. of Categories Allowed")
    if output_mode not in ("replace", "append"):
        raise TypeError("Invalid input for output_mode")

    if pre_existing_model:
        params = load_outlier_model(model_path)
    else:
        present, _ = _present(fr, cols)
        params = OrderedDict((c, outlier_kept(present[c], coverage, max_category)) for c in cols)
    odf = _per_chunk(fr, lambda f: _apply_outliers(f, cols, params, output_mode))
    if not pre_existing_model and model_path != "NA":
        save_outlier_model(model_path, params.items())
    if print_impact:
        from ..data_analyzer.stats_generator import uniqueCount_computation
        out_cols = cols if output_mode == "replace" else [c + "_outliered" for c in cols]
        before = uniqueCount_computation(spark, fr, cols).toPandas().rename(columns={"unique_values": "uniqueValues_before"})
        after = uniqueCount_computation(spark, odf, out_cols).toPandas().rename(columns={"unique_values": "uniqueValues_after"})
        from ..result import ResultFrame
        ResultFrame(before).show(len(cols), False)
        ResultFrame(after).show(len(cols), False)
    return odf


def cat_to_num_transformer(spark, idf, list_of_cols, drop_cols, method_type, encoding, label_col, event_label):
    """The reference's dispatcher (transformers.py:428-503), kept as written: it validates `list_of_cols` and then calls
    the encoders with their defaults.  Supervised mode turns the label into an int 0 / 1 column; "unsupervised" with a
    label column returns None."""
    fr = as_frame(idf)
    cat_cols = attributeType_segregation(fr)[1]
    if len(cat_cols) > 0:
        if isinstance(list_of_cols, str) and list_of_cols == "all":
            list_of_cols = cat_cols
        list_of_cols = _split(list_of_cols)
        if any(x not in cat_cols for x in list_of_cols):
            raise TypeError("Invalid input for Column(s)")
        if method_type == "supervised" and label_col is not None:
            odf = cat_to_num_supervised(spark, fr, label_col=label_col, event_label=event_label)
            return _label_to_int(odf, label_col, event_label)
        elif method_type == "unsupervised" and label_col is None:
            return cat_to_num_unsupervised(spark, fr, method_type=encoding, index_order="frequencyDesc")
        return None
    return fr


def _label_to_int(fr, label_col, event_label):
    """`withColumn(label, when(label == event_label, 1).otherwise(0))` as an int column with no nulls."""
    from ..shared.label_classes import label_bitmaps

    def one(f):
        import torch
        ev_w, _, _ = label_bitmaps(f, label_col, event_label)
        rows = torch.arange(f.n_rows, device=ev_w.device)
        bit = ((ev_w[rows >> 5] >> (rows & 31).to(torch.int32)) & 1).to(torch.int32)
        new = OrderedDict((n, f.column(n)) for n in f.columns)
        new[label_col] = Column(label_col, "int", f.n_rows, dev=bit, anv_dtype=_lib.ANV_I32, null_count=0)
        return ColumnFrame(new, f.n_rows)
    return _per_chunk(fr, one)
