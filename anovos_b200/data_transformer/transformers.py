"""CUDA implementation of `anovos.data_transformer.transformers.attribute_binning`
(reference /root/reference/src/main/anovos/data_transformer/transformers.py:87-291) and `imputation_MMM` (:1369-1676,
at the end of this module).

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
