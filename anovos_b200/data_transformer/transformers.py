"""CUDA implementation of `anovos.data_transformer.transformers.attribute_binning`
(reference /root/reference/src/main/anovos/data_transformer/transformers.py:87-291).

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
