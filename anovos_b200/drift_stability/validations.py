"""Keyword-argument normalisers of `drift_detector.statistics` and the scoring rules of
`stability_index_computation`, written from the behavioural contract of the reference module
(/root/reference/src/main/anovos/drift_stability/validations.py):

* :8-71  `check_list_of_columns` - reads KEYWORD arguments only (a positional list_of_cols is ignored and treated as
  "all", SURVEY.md Appendix C #6); "all" = numerical + categorical columns of the target frame; "a|b" strings or lists;
  drops removed, duplicates collapsed in first-seen order; wrong type -> TypeError, empty selection or a name the target
  lacks -> ValueError; the wrapped function receives list_of_cols=<resolved list> and drop_cols=[].
* :74-94 `check_distance_method` - "all" = PSI, JSD, HD, KS; "A|B" strings or lists; anything else -> TypeError.
* :97-172 CV / SD -> 0..4 scores, the weighted stability index, and the two argument checks.
"""
from __future__ import annotations

import bisect
import functools

from ..frame import as_frame
from ..shared.utils import attributeType_segregation, unique

DISTANCE_METHODS = ("PSI", "JSD", "HD", "KS")


def _name_list(value, what):
    """"a| b" -> ["a", "b"]; lists pass through; None -> []."""
    if value is None:
        return []
    if isinstance(value, str):
        return [part.strip() for part in value.split("|")]
    if isinstance(value, list):
        return value
    raise TypeError("'%s' must be either a string or a list of strings. Received %s." % (what, type(value)))


def _keyword_rewriter(rewrite):
    """Decorator factory: `rewrite(args, kwargs)` edits the keyword arguments in place before the call.  Usable bare
    (`@deco`) or configured (`@deco(name=...)`), like the reference decorators."""
    def deco(func=None, **config):
        if func is None:
            return functools.partial(deco, **config)

        @functools.wraps(func)
        def wrapper(*args, **kwargs):
            rewrite(args, kwargs, **config)
            return func(*args, **kwargs)
        return wrapper
    return deco


def _resolve_columns(args, kwargs, columns="list_of_cols", target_idx=1, target="idf_target", drop="drop_cols"):
    frame = kwargs.get(target)
    frame = as_frame(args[target_idx] if frame is None else frame)
    wanted = kwargs.get(columns, "all")
    if wanted is None:      # only drop_cols may be None
        raise TypeError("'%s' must be either a string or a list of strings. Received %s." % (columns, type(None)))
    if isinstance(wanted, str) and wanted == "all":
        num, cat, _ = attributeType_segregation(frame)
        wanted = num + cat
    wanted = _name_list(wanted, columns)
    dropped = set(_name_list(kwargs.get(drop, []), drop))
    kept = unique(wanted, dropped)
    if not kept:
        raise ValueError("Empty set of columns is given. Columns to select: %s, columns to drop: %s." % (wanted, sorted(dropped)))
    unknown = set(kept) - set(frame.columns)
    if unknown:
        raise ValueError("Not all columns are in the input dataframe. Missing columns: %s" % unknown)
    kwargs[columns], kwargs[drop] = kept, []


def _resolve_methods(args, kwargs, param="method_type"):
    methods = kwargs.get(param, "PSI")
    if isinstance(methods, str):
        methods = list(("PSI", "JSD", "HD", "KS")) if methods == "all" else [m.strip() for m in methods.split("|")]
    if any(m not in DISTANCE_METHODS for m in methods):
        raise TypeError("Invalid input for %s" % param)
    kwargs[param] = methods


check_list_of_columns = _keyword_rewriter(_resolve_columns)
check_distance_method = _keyword_rewriter(_resolve_methods)


# ---- stability scoring (:97-172) ------------------------------------------------------------------

# sd score: 4 up to 0.005, then three straight segments (slope, intercept) up to their right edge, 0 beyond 0.1
_SD_EDGES = (0.005, 0.01, 0.05, 0.1)
_SD_LINES = ((0.0, 4.0), (-100.0, 4.5), (-50.0, 4.0), (-30.0, 3.0))


def compute_score(value, method_type, cv_thresholds=[0.03, 0.1, 0.2, 0.5]):
    """CV or SD of a metric over time -> score in [0, 4] (higher = more stable).
    "cv": 4 minus the number of thresholds |value| has reached; "sd": piecewise linear in value, one decimal."""
    if value is None:
        return None
    if method_type == "cv":
        return float(len(cv_thresholds) - bisect.bisect_right(list(cv_thresholds), abs(value)))
    if method_type == "sd":
        seg = bisect.bisect_left(_SD_EDGES, value)
        if seg >= len(_SD_LINES):
            return 0.0
        slope, intercept = _SD_LINES[seg]
        return 4.0 if seg == 0 else round(slope * value + intercept, 1)
    raise TypeError("method_type must be either 'cv' or 'sd'.")


def compute_si(metric_weightages):
    """-> f(attr_type, mean_stddev, mean_cv, stddev_cv, kurtosis_cv) = [mean_si, stddev_si, kurtosis_si, stability_index].
    Binary attributes are scored on the SD of their mean alone; numerical ones on the weighted CV scores (None as soon
    as one of them is undefined), rounded to 4 decimals."""
    weights = [metric_weightages.get(k, 0) for k in ("mean", "stddev", "kurtosis")]

    def score(attr_type, mean_stddev, mean_cv, stddev_cv, kurtosis_cv):
        if attr_type == "Binary":
            s = compute_score(mean_stddev, "sd")
            return [s, None, None, s]
        parts = [compute_score(v, "cv") for v in (mean_cv, stddev_cv, kurtosis_cv)]
        total = None if any(p is None for p in parts) else round(sum(p * w for p, w in zip(parts, weights)), 4)
        return parts + [total]
    return score


def check_metric_weightages(metric_weightages):
    if round(sum(metric_weightages.get(k, 0) for k in ("mean", "stddev", "kurtosis")), 3) != 1:
        raise ValueError("Invalid input for metric weightages. Either metric name is incorrect or sum of metric "
                         "weightages is not 1.0.")


def check_threshold(threshold):
    if not 0 <= threshold <= 4:
        raise ValueError("Invalid input for metric threshold. It must be a number between 0 and 4.")
