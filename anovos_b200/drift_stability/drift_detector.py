"""CUDA implementation of `anovos.drift_stability.drift_detector.statistics` (reference
/root/reference/src/main/anovos/drift_stability/drift_detector.py:16-371).

Data path: source frame -> K1 (min/max) -> cutoffs on the host (bit-identical model) ->
K2 histogram; target frame -> K1+K2 fused in ONE read; string columns -> dictionary-code
histograms; the per-column (p, q) tables are reduced to PSI / HD / JSD / KS by the drift
kernel.  The reference instead runs a Python UDF per value plus 2 groupBys, a join and
4 aggregations per column.  Saved artefacts keep the reference's formats
(`<source_path>/<model_directory>/attribute_binning` parquet and
`.../frequency_counts/<col>` CSVs with header [<col>, p]).
"""
from __future__ import annotations

import math
import os
import re

import numpy as np
import pandas as pd

from .. import engine, profile
from ..data_transformer.transformers import check_bin_size, compute_cutoffs, load_binning_model, save_binning_model
from ..frame import as_frame
from ..result import ResultFrame
from .validations import check_distance_method, check_list_of_columns

try:  # the reference logs through loguru; it is optional here
    from loguru import logger
except Exception:  # pragma: no cover
    import logging
    logger = logging.getLogger("anovos_b200")

_ORDER = ("PSI", "HD", "JSD", "KS")   # code order of the reference (:273-335), not method_type order


def _freq_dir(model_path, col):
    return os.path.join(model_path, "frequency_counts", col)


_NEEDS_QUOTES = re.compile(r'[,"\n\r]')


def _csv_field(v):
    if v is None:
        return ""
    s = v if type(v) is str else str(v)
    if _NEEDS_QUOTES.search(s):
        s = '"' + s.replace('"', '""') + '"'
    return s


def _save_frequency(model_path, col, keys, p):
    """`x.coalesce(1).write.csv(.../frequency_counts/<col>, header=True, mode="overwrite")` (:257-262)."""
    d = _freq_dir(model_path, col)
    os.makedirs(d, exist_ok=True)
    for f in os.listdir(d):
        if f.endswith(".csv"):
            os.remove(os.path.join(d, f))
    ks = list(map(_csv_field, keys))
    vs = list(map(repr, np.asarray(p, dtype=np.float64).tolist()))
    with open(os.path.join(d, "part-00000.csv"), "w", newline="") as fh:
        fh.write(_csv_field(col) + ",p\n")
        if ks:
            fh.write("\n".join(map(",".join, zip(ks, vs))) + "\n")


def _utf8_sorted(fr, col):
    """Is the dictionary of string column `col` in UTF-8 byte order (Spark's orderBy on strings)?  True for
    frames built from Arrow / pandas; a hand-made dictionary is checked once."""
    key = ("dict_utf8_sorted", col)
    if key not in fr._cache:
        b = [s.encode("utf-8") for s in fr.column(col).dictionary]
        fr._cache[key] = all(x < y for x, y in zip(b, b[1:]))
    return fr._cache[key]


def _load_frequency(model_path, col, string_keys=False):
    """The saved [<col>, p] table of a source column (:245-250).  Keys of string columns are read back as the strings
    that were written: Spark's CSV reader treats only the EMPTY field as null, so categories spelled "NA", "null",
    "None", "nan" ... stay categories and "00501" / "1.0" keep their spelling (pandas' defaults would turn the former
    into NaN and re-type the latter, silently changing the join with the target's keys).  Bin ids stay integers."""
    d = _freq_dir(model_path, col)
    files = sorted(f for f in os.listdir(d) if f.endswith(".csv"))
    kw = dict(dtype={col: str}, keep_default_na=False, na_values={col: [""]}) if string_keys else {}
    return pd.concat([pd.read_csv(os.path.join(d, f), **kw) for f in files], ignore_index=True)


@check_distance_method
@check_list_of_columns
def statistics(spark, idf_target, idf_source, list_of_cols="all", drop_cols=None, method_type="PSI",
               bin_method="equal_range", bin_size=10, threshold=0.1, use_sampling=True, sample_method="random",
               strata_cols="all", stratified_type="population", sample_size=100000, sample_seed=42, persist=True,
               persist_option=None, pre_existing_source=False, source_save=True, source_path="NA",
               model_directory="drift_statistics", print_impact=False):
    """Same signature as the reference (:18-41).  Returns [attribute, <metrics in PSI,HD,JSD,KS
    order>, flagged]; metrics are not rounded; flagged = 1 if any metric > threshold."""
    check_bin_size(bin_size)
    tgt = as_frame(idf_target)
    src = as_frame(idf_source) if idf_source is not None else None
    if src is None and not pre_existing_source:
        raise ValueError("idf_source is required unless pre_existing_source=True")
    cols = list(list_of_cols)
    methods = [m for m in _ORDER if m in method_type]
    num_cols = [c for c in cols if tgt.column(c).kind == "num"]
    cat_cols = [c for c in cols if tgt.column(c).kind == "cat"]
    other = [c for c in cols if tgt.column(c).kind == "other"]
    if other:
        raise TypeError("columns %s have a dtype the drift path does not handle" % other)

    if use_sampling:      # :187-211 - Spark's Bernoulli / sampleBy row set, reproduced on the device (data_sampling.py)
        from ..data_ingest.data_sampling import data_sample
        kw = dict(strata_cols=strata_cols, method_type=sample_method, stratified_type=stratified_type, seed_value=sample_seed)
        if tgt.count() > sample_size:
            tgt = data_sample(tgt, fraction=sample_size / tgt.count(), **kw)
        if src is not None and src.count() > sample_size:
            src = data_sample(src, fraction=sample_size / src.count(), **kw)
    count_target = tgt.count()
    count_source = src.count() if src is not None else None

    if source_path == "NA":
        source_path = "intermediate_data"
    model_path = source_path + "/" + model_directory

    # ---- numeric columns: binning model from the source, histograms of both frames --------------
    src_num_counts, binned = {}, []
    if pre_existing_source:
        model = load_binning_model(model_path) if num_cols else {}
        # a column the source pass dropped (all-null under equal_range) is absent from the model; the
        # reference would crash here with IndexError - we keep it unbinned (metrics 0), see SURVEY C#12
        binned = [c for c in num_cols if c in model]
        missing = [c for c in num_cols if c not in model]
        if missing:
            import warnings
            warnings.warn("Columns absent from the saved binning model are not binned: " + ", ".join(missing))
        cuts, lohi = [model[c] for c in binned], None
    else:
        if num_cols:
            binned, cuts, lohi = compute_cutoffs(src, num_cols, bin_method, bin_size)
            save_binning_model(model_path, binned, cuts)          # the reference always writes the model (:217-225)
            sm = engine.BinModel(src, binned, cuts, lohi)
            hs = engine.histogram(src, sm)
            for i, c in enumerate(binned):
                src_num_counts[c] = hs[i, :len(cuts[i]) + 2]
        else:
            cuts, lohi = [], None
    tgt_num_counts = {}
    if binned:
        tm = engine.BinModel(tgt, binned, cuts, None if lohi is None else lohi)
        mt, ht = engine.moments_histogram(tgt, tm)                 # ONE read of the target frame
        tc = profile._cache(tgt, "moments")                        # ... whose moments the stats functions reuse
        for i, c in enumerate(binned):
            tc.setdefault(c, mt[i])
        for i, c in enumerate(binned):
            tgt_num_counts[c] = ht[i, :len(cuts[i]) + 2]
    unbinned = [c for c in num_cols if c not in binned]            # all-null source columns (SURVEY C#12)

    # ---- categorical columns: code histograms aligned on the union of keys -----------------------
    tgt_cat = profile.code_counts(tgt, cat_cols) if cat_cols else {}
    src_cat = profile.code_counts(src, cat_cols) if (cat_cols and not pre_existing_source) else {}

    S, T, P, kinds, order = [], [], [], [], []
    use_p = pre_existing_source
    for c in cols:
        if c in unbinned:
            continue
        if c in tgt_num_counts:
            t = tgt_num_counts[c]
            if use_p:
                f = _load_frequency(model_path, c)
                p = np.full(len(t), np.nan)
                for k, v in zip(f[c].tolist(), f["p"].tolist()):
                    k = int(k)
                    p[0 if k == -1 else k] = v
                P.append(p)
            else:
                s = src_num_counts[c]
                S.append(s)
                if source_save:
                    keys = ([-1] if s[0] > 0 else []) + [k for k in range(1, len(s)) if s[k] > 0]
                    _save_frequency(model_path, c, keys, [0.0 if k == -1 else int(s[k]) / count_source for k in keys])
            T.append(t)
            kinds.append(0)
        else:
            tdic, th = tgt.column(c).dictionary, tgt_cat[c]
            if use_p:
                f = _load_frequency(model_path, c, string_keys=True)
                sk = {}
                s_null = False
                for k, v in zip(f[c].tolist(), f["p"].tolist()):
                    if isinstance(k, float) and math.isnan(k):
                        s_null = True
                    else:
                        sk[str(k)] = float(v)
                keys = sorted(set(sk) | {tdic[i] for i in np.flatnonzero(th[1:])}, key=lambda s: s.encode("utf-8"))
                tpos = {k: i for i, k in enumerate(tdic)}
                t = np.zeros(len(keys) + 1, np.uint64)
                t[0] = th[0]
                p = np.full(len(keys) + 1, np.nan)
                p[0] = 0.0 if s_null else np.nan
                for j, k in enumerate(keys):
                    if k in tpos:
                        t[j + 1] = th[tpos[k] + 1]
                    if k in sk:
                        p[j + 1] = sk[k]
                P.append(p)
                T.append(t)
            else:
                sdic, sh = src.column(c).dictionary, src_cat[c]
                if (sdic is tdic or sdic == tdic) and _utf8_sorted(src, c):
                    # same (UTF-8 ordered) dictionary on both sides - the usual case: the key union is a mask
                    keep = np.flatnonzero((sh[1:] > 0) | (th[1:] > 0))
                    s = np.concatenate([sh[:1], sh[1:][keep]]).astype(np.uint64)
                    t = np.concatenate([th[:1], th[1:][keep]]).astype(np.uint64)
                    S.append(s)
                    T.append(t)
                    if source_save:
                        nz = np.flatnonzero(s[1:] > 0)
                        kk = ([None] if s[0] > 0 else []) + [sdic[i] for i in keep[nz].tolist()]
                        pp = np.concatenate([np.zeros(1 if s[0] > 0 else 0), s[1:][nz].astype(np.float64) / count_source])
                        _save_frequency(model_path, c, kk, pp)
                    kinds.append(1)
                    order.append(c)
                    continue
                keys = sorted({sdic[i] for i in np.flatnonzero(sh[1:])} | {tdic[i] for i in np.flatnonzero(th[1:])},
                              key=lambda s: s.encode("utf-8"))        # orderBy(i): UTF-8 byte order
                spos, tpos = {k: i for i, k in enumerate(sdic)}, {k: i for i, k in enumerate(tdic)}
                s = np.zeros(len(keys) + 1, np.uint64)
                t = np.zeros(len(keys) + 1, np.uint64)
                s[0], t[0] = sh[0], th[0]
                for j, k in enumerate(keys):
                    if k in spos:
                        s[j + 1] = sh[spos[k] + 1]
                    if k in tpos:
                        t[j + 1] = th[tpos[k] + 1]
                S.append(s)
                T.append(t)
                if source_save:
                    kk = ([None] if s[0] > 0 else []) + [k for j, k in enumerate(keys) if s[j + 1] > 0]
                    pp = ([0.0] if s[0] > 0 else []) + [int(s[j + 1]) / count_source for j in range(len(keys)) if s[j + 1] > 0]
                    _save_frequency(model_path, c, kk, pp)
            kinds.append(1)
        order.append(c)

    d = engine.drift_reduce(None if use_p else S, T, kinds, count_source if count_source else 1, count_target,
                            src_p=P if use_p else None)
    by_col = {c: d[i] for i, c in enumerate(order)}
    rows = []
    for c in cols:
        row = {"attribute": c}
        if c in by_col and by_col[c]["n_rows"] > 0:
            r = by_col[c]
            vals = {"PSI": float(r["psi"]), "HD": float(r["hd"]), "JSD": float(r["jsd"]), "KS": float(r["ks"])}
        else:  # all-null numeric source column: raw (all null) groups on both sides -> (1e-4, 1e-4) rows only
            vals = {"PSI": 0.0, "HD": 0.0, "JSD": 0.0, "KS": 0.0}
        for mname in methods:
            row[mname] = vals[mname]
        row["flagged"] = int(any(vals[mname] > threshold for mname in methods))     # strict > (:353-356)
        rows.append(row)
    odf = ResultFrame(pd.DataFrame(rows, columns=["attribute"] + methods + ["flagged"]))
    if print_impact:
        logger.info("All Attributes:")
        odf.show(len(cols))
        logger.info("Attributes meeting Data Drift threshold:")
        odf.where("flagged == 1").show(len(cols))
    return odf
