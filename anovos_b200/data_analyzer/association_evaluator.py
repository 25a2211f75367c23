"""`IV_calculation` / `IG_calculation` of `anovos.data_analyzer.association_evaluator` (SURVEY.md 8f, row
N3; reference /root/reference/src/main/anovos/data_analyzer/association_evaluator.py:253-586).

Both are a (group x label) contingency table per attribute.  The reference bins the numeric
attributes with the Python UDF of attribute_binning and then runs one groupBy per attribute;
here the table comes from THREE runs of the histogram kernel (K2 / the code histogram) over
the same columns with the validity bitmap AND-ed with the label-class bitmaps (all rows /
event rows / non-event rows): bit-exact counts, then a few logs per group on the host.  With
`monotonicity_check=1` the numeric attributes are binned as monotonic_binning bins them (:350-357), and their table comes
from the same label-class histogram (anv_class_hist) that chose each attribute's bin count; only an attribute that falls
back to a bin_size outside 3 .. 20 takes the three K2 passes."""
from __future__ import annotations

import math

import numpy as np
import pandas as pd

from .. import engine
from ..data_transformer.transformers import check_bin_size, compute_cutoffs
from ..frame import as_frame
from ..result import ResultFrame
from ..shared.label_classes import label_bitmaps as _label_bitmaps, masked as _masked
from ..shared.utils import attributeType_segregation, names, unique

_DEFAULT_ENC = {"bin_method": "equal_frequency", "bin_size": 10, "monotonicity_check": 0}


def _prepare(idf, list_of_cols, drop_cols, label_col, event_label, encoding_configs):
    if encoding_configs and "bin_size" in encoding_configs:
        check_bin_size(encoding_configs["bin_size"])
    fr = as_frame(idf)
    if getattr(fr, "is_partitioned", False):
        # chunked / Spark-partitioned table: the cutoffs come from the partitioned frame (so approxQuantile follows Spark's
        # per-partition sketches), the label-class histograms from the concatenated columns
        if fr.group is not None:
            raise NotImplementedError("IV / IG on row slabs of several ranks: repartition_to_columns first")
        part = fr
        fr = part.materialize()
        fr._cut_source = part
    if label_col not in fr.columns:
        raise TypeError("Invalid input for Label Column")
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        num, cat, _ = attributeType_segregation(fr)
        list_of_cols = num + cat
    cols = unique(names(list_of_cols), names(drop_cols) + [label_col])
    if any(c not in fr.columns for c in cols) or not cols:
        raise TypeError("Invalid input for Column(s)")
    ev_w, nev_w, n_event = _label_bitmaps(fr, label_col, event_label)
    if n_event == 0:
        raise TypeError("Invalid input for Event Label Value")
    num = [c for c in cols if fr.column(c).kind == "num"]
    cat = [c for c in cols if fr.column(c).kind == "cat"]
    if any(fr.column(c).kind == "other" for c in cols):
        raise TypeError("Invalid input for Column(s)")
    binned = bool(num) and bool(encoding_configs)
    return fr, cols, num, cat, ev_w, nev_w, binned


def _contingency(fr, cols, num, cat, ev_w, nev_w, binned, encoding_configs, label):
    """dict col -> (all[g], event[g], nonevent[g]) count arrays; index 0 = the null group."""
    out = {}
    if num and not binned:
        raise NotImplementedError("raw (unbinned) numeric attributes: pass encoding_configs")

    def views(names):                        # the class views of the columns a pass reads
        return {"all": fr, "ev": _masked(fr, names, ev_w), "nev": _masked(fr, names, nev_w)}

    hists = {"all": {}, "ev": {}, "nev": {}}
    k2 = []                                  # (col, cutoffs, lohi) counted by K2 over the three views
    if num and encoding_configs.get("monotonicity_check", 0) == 1:
        k2 = _monotonic_groups(fr, num, encoding_configs, *label, hists)
    elif num:
        kept, cuts, lohi = compute_cutoffs(getattr(fr, "_cut_source", fr), num, encoding_configs["bin_method"],
                                           encoding_configs["bin_size"])
        k2 = list(zip(kept, cuts, lohi))
        for c in num:
            if c not in kept:                  # all-null attribute: only the null group exists
                hists["all"][c] = hists["ev"][c] = hists["nev"][c] = None
    if k2:
        names = [c for c, _, _ in k2]
        for k, f in views(names).items():
            model = engine.BinModel(f, names, [cut for _, cut, _ in k2], [lh for _, _, lh in k2])
            h = engine.histogram(f, model)
            hists[k].update({c: h[i, :len(cut) + 2].astype(np.int64) for i, (c, cut, _) in enumerate(k2)})
    if cat:
        for k, f in views(cat).items():
            cc = engine.code_counts(f, cat)
            hists[k].update({c: h.astype(np.int64) for c, h in zip(cat, cc)})
    n_rows = fr.n_rows
    tot_ev = int(_unpack_count(ev_w))
    tot_nev = int(_unpack_count(nev_w))
    for c in cols:
        a = hists["all"][c]
        if a is None:
            out[c] = (np.array([n_rows]), np.array([tot_ev]), np.array([tot_nev]))
            continue
        e, ne = hists["ev"][c].copy(), hists["nev"][c].copy()
        # slot 0 of a masked pass mixes "attribute null" with "row outside the class": rebuild the null group
        e[0] = tot_ev - e[1:].sum()
        ne[0] = tot_nev - ne[1:].sum()
        out[c] = (a, e, ne)
    return out, tot_ev, tot_nev


def _monotonic_groups(fr, num, encoding_configs, label_col, event_label, hists):
    """Fills hists["all" / "ev" / "nev"][col] for the numeric attributes binned as monotonic_binning bins them.  The groups
    of an accepted n (or of a fallback bin_size inside 3 .. 20) are sums of the ladder's class histogram.  -> the
    (col, cutoffs, lohi) of the columns that fall back to a bin_size outside that range, for the K2 passes."""
    from ..data_transformer.transformers import monotonic_models
    from ..shared import monotonic
    models, lad = monotonic_models(getattr(fr, "_cut_source", fr), fr, num, label_col, event_label,
                                   encoding_configs["bin_method"], encoding_configs["bin_size"])
    rest = []
    for c in num:
        n, cut, lohi = models[c]
        if n in lad[c].um.bins:
            hists["all"][c], hists["ev"][c], hists["nev"][c] = monotonic.model_table(lad[c].um, lad[c].counts, n)
        else:
            rest.append((c, cut, lohi))
    return rest


def _unpack_count(words):
    import torch
    w = words.to(torch.int64) & 0xFFFFFFFF
    # popcount of 32-bit words
    w = w - ((w >> 1) & 0x55555555)
    w = (w & 0x33333333) + ((w >> 2) & 0x33333333)
    w = (w + (w >> 4)) & 0x0F0F0F0F
    return int(((w * 0x01010101) >> 24 & 0xFF).sum().item())


def IV_calculation(spark, idf, list_of_cols="all", drop_cols=[], label_col="label", event_label=1,
                   encoding_configs=_DEFAULT_ENC, print_impact=False):
    """[attribute, iv]; iv = sum_g (nonevent_pcr - event_pcr) * woe_g with the reference's +0.5 smoothing
    when one side of a group is empty (:369-392)."""
    fr, cols, num, cat, ev_w, nev_w, binned = _prepare(idf, list_of_cols, drop_cols, label_col, event_label, encoding_configs)
    tab, t1, t0 = _contingency(fr, cols, num, cat, ev_w, nev_w, binned, encoding_configs,
                               (label_col, event_label))
    rows = []
    for c in cols:
        a, e, ne = tab[c]
        iv = 0.0
        for g in range(len(a)):
            if a[g] == 0:
                continue                       # the group does not exist
            l0, l1 = float(ne[g]), float(e[g])
            p0, p1 = l0 / t0, l1 / t1
            woe = math.log(p0 / p1) if (p0 != 0 and p1 != 0) else math.log(((l0 + 0.5) / t0) / ((l1 + 0.5) / t1))
            iv += woe * (p0 - p1)
        rows.append([c, iv])
    odf = ResultFrame(pd.DataFrame(rows, columns=["attribute", "iv"]))
    if print_impact:
        odf.show(len(cols))
    return odf


def IG_calculation(spark, idf, list_of_cols="all", drop_cols=[], label_col="label", event_label=1,
                   encoding_configs=_DEFAULT_ENC, print_impact=False):
    """[attribute, ig]; ig = H(label) - sum_g segment_pct * H(label | g); log2(0) is NULL in Spark SQL, so a
    segment whose event_pct is 0 or 1 adds nothing (:540-566)."""
    fr, cols, num, cat, ev_w, nev_w, binned = _prepare(idf, list_of_cols, drop_cols, label_col, event_label, encoding_configs)
    tab, t1, t0 = _contingency(fr, cols, num, cat, ev_w, nev_w, binned, encoding_configs,
                               (label_col, event_label))
    n = fr.n_rows
    te = t1 / n
    total_entropy = -(te * math.log2(te) + (1 - te) * math.log2(1 - te))
    rows = []
    for c in cols:
        a, e, ne = tab[c]
        s, any_term = 0.0, False
        for g in range(len(a)):
            if a[g] == 0:
                continue
            p = float(e[g]) / float(a[g])
            if 0 < p < 1:
                s += -(float(a[g]) / n) * (p * math.log2(p) + (1 - p) * math.log2(1 - p))
                any_term = True
        # Spark's sum over all-NULL segment entropies is NULL (id-like column: every segment pure) -> null ig
        rows.append([c, total_entropy - s if any_term else None])
    odf = ResultFrame(pd.DataFrame(rows, columns=["attribute", "ig"]))
    if print_impact:
        odf.show(len(cols))
    return odf
