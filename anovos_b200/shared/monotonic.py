"""The bin-count ladder of monotonic_binning (reference data_transformer/transformers.py:294-425), shared by
data_transformer.transformers.monotonic_binning and the monotonicity check of IV / IG (data_analyzer.association_evaluator).

For each column the reference bins with n = 20, 19, ..., 3 bins, groups the rows by bin, and accepts the first n whose
(avg(x), avg(label == event_label)) table has a Spearman correlation of exactly 1.0.  Here:
  - the 18 candidate cutoff lists come from ONE moments call (equal_range) or ONE quantiles call over the union of the
    probabilities j * (1 / n) (equal_frequency), value for value what compute_cutoffs(fr, [c], method, n) returns;
  - their native thresholds are merged into one sorted union; slot(x) = 1 + #(theta < x) is monotone in the threshold set,
    so every candidate bin is a run of consecutive union slots and a host table maps slot -> bin for each n;
  - one anv_class_hist pass counts the rows per (union slot, label class) and the host sums slots into each model's bins.
The bins of a model are disjoint ordered intervals, so their averages are in bin order and the bin index stands in for
avg(x) (Spearman sees ranks only).  The one exception, a finite bin sum that overflows a double, is a recorded deviation
(DESIGN.md section 1)."""
from __future__ import annotations

import warnings

import numpy as np

from .. import _lib, engine, profile

LADDER = tuple(range(20, 2, -1))      # bin counts tried, in order


def ladder_cutoffs(fr, cols, method):
    """-> (cuts, lohi): cuts[c] = {n: cutoffs} for n in LADDER, each equal to compute_cutoffs(fr, [c], method, n); lohi[c]
    = (min, max) for equal_range, None for equal_frequency.  An equal_range column without a non-null value has no entry."""
    cuts, lohi = {}, {}
    if method == "equal_frequency":
        probs = list(dict.fromkeys(j * (1 / n) for n in LADDER for j in range(1, n)))   # compute_cutoffs' float artefacts
        at = {p: i for i, p in enumerate(probs)}
        q = profile.quantiles(fr, cols, probs, profile.APPROX_QUANTILE_EPS)
        for c in cols:
            vals = [float("nan") if v is None else float(v) for v in q[c]]
            cuts[c] = {n: [vals[at[j * (1 / n)]] for j in range(1, n)] for n in LADDER}
            lohi[c] = None
        return cuts, lohi
    mom = profile.moments(fr, cols)
    for c in cols:
        if int(mom[c]["n_valid"]) == 0:
            continue
        mx, mn = float(mom[c]["max"]), float(mom[c]["min"])
        cuts[c] = {}
        for n in LADDER:
            w = (mx - mn) / n
            cuts[c][n] = [mn + j * w for j in range(1, n)]
        lohi[c] = (mn, mx)
    return cuts, lohi


def typed_thresholds(cutoffs, anv_dtype) -> np.ndarray:
    """engine.native_thresholds as values of the column's own dtype (the order the kernels compare in)."""
    raw = engine.native_thresholds(cutoffs, anv_dtype)
    if anv_dtype == _lib.ANV_F32:
        return raw.astype(np.uint32).view(np.float32)
    if anv_dtype == _lib.ANV_I32:
        return raw.astype(np.uint32).view(np.int32)
    return raw.view(np.float64 if anv_dtype == _lib.ANV_F64 else np.int64)


class UnionModel:
    """The sorted, de-duplicated union of a column's candidate thresholds and, per n, the bin of every union slot.
    Slots: 0 = null value, 1 .. len(union) + 1 = 1 + #(union < x), len(union) + 2 = NaN."""

    def __init__(self, cuts_by_n, anv_dtype):
        typed = {n: np.sort(typed_thresholds(cut, anv_dtype)) for n, cut in cuts_by_n.items()}
        self.thresholds = np.unique(np.concatenate(list(typed.values())))   # -0.0 and 0.0 compare equal: one entry
        u = len(self.thresholds)
        self.n_slots = u + 3
        self.bins = {}
        for n, th in typed.items():
            m = np.empty(self.n_slots, np.int64)
            m[0], m[1], m[u + 2] = 0, 1, n       # a NaN value is above no cutoff: `NaN <= c` is False, so bin n
            m[2:u + 2] = 1 + np.searchsorted(th, self.thresholds, side="right")
            self.bins[n] = m
        # slots of the infinities: nothing is below -inf; +inf is above every threshold but +inf itself
        self.inf_slots = (1, 1 + int(np.searchsorted(self.thresholds, np.inf, side="left"))) \
            if self.thresholds.dtype.kind == "f" else None


def model_table(um: UnionModel, counts, n):
    """-> (all, event, non-event) int64 arrays [n + 1] of model n: index 0 = the null group, b = bin b."""
    c = np.asarray(counts[:3 * um.n_slots], np.uint64).astype(np.int64).reshape(3, um.n_slots)
    m = um.bins[n]
    out = []
    for row in (c.sum(axis=0), c[0], c[1]):
        t = np.zeros(n + 1, np.int64)
        np.add.at(t, m, row)
        out.append(t)
    return tuple(out)


def nan_mean_bins(um: UnionModel, counts, n):
    """Bins of model n whose avg(x) is NaN: the bin holding a NaN value, and a bin holding both -inf and +inf."""
    bad = set()
    if int(np.asarray(counts[:3 * um.n_slots]).reshape(3, um.n_slots)[:, um.n_slots - 1].sum()):
        bad.add(n)
    ninf, pinf = int(counts[3 * um.n_slots]), int(counts[3 * um.n_slots + 1])
    if ninf and pinf and um.inf_slots is not None:
        lo, hi = (int(um.bins[n][s]) for s in um.inf_slots)
        if lo == hi:
            bad.add(lo)
    return bad


def spearman_r(mean_val, mean_label):
    """scipy.stats.spearmanr over the two single-column tables, as the reference calls it (NaN below 2 groups)."""
    import pandas as pd
    from scipy import stats
    tmp = pd.DataFrame({"mean_val": np.asarray(mean_val, np.float64), "mean_label": np.asarray(mean_label, np.float64)})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        r, _ = stats.spearmanr(tmp[["mean_val"]], tmp[["mean_label"]])
    return float(r)


def accepts(count, events, drop=()):
    """The groupBy(bin).agg(avg(x), avg(label01)).dropna() table of one model from its per-bin rows and events (index b =
    bin b, index 0 unused), without empty bins and the bins in `drop`; accepted iff spearmanr gives exactly 1.0."""
    keep = [b for b in range(1, len(count)) if count[b] > 0 and b not in drop]
    r = spearman_r([float(b) for b in keep], [float(events[b]) / float(count[b]) for b in keep])
    return r == 1.0


def choose(um: UnionModel, counts):
    """The first n of LADDER the reference accepts, or None."""
    for n in LADDER:
        a, e, _ = model_table(um, counts, n)
        if accepts(a, e, nan_mean_bins(um, counts, n)):
            return n
    return None


class Ladder:
    """One column's candidate models, class histogram and accepted n (None: no n accepted)."""

    def __init__(self, cuts, lohi, um, counts, n):
        self.cuts, self.lohi, self.um, self.counts, self.n = cuts, lohi, um, counts, n


def ladders(cut_fr, hist_fr, cols, label_col, event_label, method):
    """-> {col: Ladder} for numeric `cols`: cutoffs from cut_fr (a chunked frame keeps its per-partition quantile
    sketches), the class histogram from hist_fr (the same rows).  One class-histogram pass serves every column."""
    cuts, lohi = ladder_cutoffs(cut_fr, cols, method)
    missing = [c for c in cols if c not in cuts]
    if missing:
        raise ValueError("monotonic_binning: column(s) %s hold no non-null value, so equal_range binning has no range to "
                         "cut" % ", ".join(repr(c) for c in missing))
    ums = {c: UnionModel(cuts[c], hist_fr.column(c).anv_dtype) for c in cols}
    counts = engine.class_hist(hist_fr, cols, [ums[c].thresholds for c in cols], label_col, event_label)
    return {c: Ladder(cuts[c], lohi[c], ums[c], h, choose(ums[c], h)) for c, h in zip(cols, counts)}
