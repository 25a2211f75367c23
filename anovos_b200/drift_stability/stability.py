"""CUDA implementation of `anovos.drift_stability.stability.stability_index_computation`
(reference /root/reference/src/main/anovos/drift_stability/stability.py:15-332): the inner
loop of the reference - one `select(mean, stddev, kurtosis)` Spark job per column per dataset
(:239-245) - is exactly the fused moments kernel (K1), one launch per dataset; the rest is a
few arithmetic operations per attribute on the host.  `feature_stability_estimation`
(symbolic, sympy) is out of scope."""
from __future__ import annotations

import math
import os

import numpy as np
import pandas as pd

from .. import profile
from ..frame import as_frame
from ..result import ResultFrame
from ..shared.utils import attributeType_segregation, names, spark_round, unique
from .validations import check_metric_weightages, check_threshold, compute_si

try:
    from loguru import logger
except Exception:  # pragma: no cover
    import logging
    logger = logging.getLogger("anovos_b200")


def _sample_std(vals):
    vals = [v for v in vals if v is not None]
    if len(vals) < 2:
        return None               # stddev_samp of < 2 values: null
    m = sum(vals) / len(vals)
    return math.sqrt(sum((v - m) * (v - m) for v in vals) / (len(vals) - 1))


def _avg(vals):
    vals = [v for v in vals if v is not None]
    return sum(vals) / len(vals) if vals else None


def _ratio(a, b):
    return None if (a is None or b is None or b == 0) else a / b   # Spark SQL: x / 0 and null / x are null


def _read_metrics(path):
    files = sorted(f for f in os.listdir(path) if f.endswith(".csv"))
    return pd.concat([pd.read_csv(os.path.join(path, f)) for f in files], ignore_index=True)


def stability_index_computation(spark, idfs, list_of_cols="all", drop_cols=[],
                                metric_weightages={"mean": 0.5, "stddev": 0.3, "kurtosis": 0.2}, binary_cols=[],
                                existing_metric_path="", appended_metric_path="", persist: bool = True,
                                persist_option=None, threshold=1, print_impact=False):
    """Same arguments, output columns and saved CSV layout ([idx, attribute, type, mean, stddev,
    kurtosis]) as the reference."""
    frames = [as_frame(f) for f in idfs]
    num_cols = attributeType_segregation(frames[0])[0]
    if isinstance(list_of_cols, str) and list_of_cols == "all":
        list_of_cols = num_cols
    binary = names(binary_cols)
    cols = unique(names(list_of_cols), names(drop_cols))
    if any(c not in num_cols for c in cols) or not cols:
        raise TypeError("Invalid input for Column(s)")
    if any(c not in cols for c in binary):
        raise TypeError("Invalid input for Binary Column(s)")
    check_metric_weightages(metric_weightages)
    check_threshold(threshold)

    existing, start = None, 1
    if existing_metric_path:
        existing = _read_metrics(existing_metric_path)
        start = int(existing["idx"].max()) + 1

    per_ds = [profile.moments(fr, cols) for fr in frames]      # one fused K1 pass per dataset
    score = compute_si(metric_weightages)
    rows, appended = [], []
    for c in cols:
        ctype = "Binary" if c in binary else "Numerical"
        means, sds, kurts = [], [], []
        for k, mom in enumerate(per_ds):
            r = mom[c]
            n, m2, m4 = int(r["n_valid"]), float(r["m2"]), float(r["m4"])
            mean = float(r["mean"]) if n else None
            sd = math.sqrt(m2 / (n - 1)) if n > 1 else None
            ku = (n * m4 / (m2 * m2)) if (n and m2 != 0) else None       # F.kurtosis + 3 (:243)
            means.append(mean); sds.append(sd); kurts.append(ku)
            appended.append([start + k, c, ctype, mean, sd, ku])
        if existing is not None:
            e = existing[existing["attribute"] == c]
            means += [None if pd.isna(v) else float(v) for v in e["mean"]]
            sds += [None if pd.isna(v) else float(v) for v in e["stddev"]]
            kurts += [None if pd.isna(v) else float(v) for v in e["kurtosis"]]
        mean_stddev = _sample_std(means)
        mean_cv = _ratio(mean_stddev, _avg(means))
        stddev_cv = _ratio(_sample_std(sds), _avg(sds))
        kurtosis_cv = _ratio(_sample_std(kurts), _avg(kurts))
        si = score(ctype, mean_stddev, mean_cv, stddev_cv, kurtosis_cv)
        si = [None if v is None else float(np.float32(v)) for v in si]   # the UDF returns ArrayType(FloatType())
        flagged = int(si[3] is None or si[3] < threshold)
        rows.append([c, ctype, spark_round(mean_stddev), spark_round(mean_cv), spark_round(stddev_cv),
                     spark_round(kurtosis_cv), si[0], si[1], si[2], si[3], flagged])
    if appended_metric_path:
        os.makedirs(appended_metric_path, exist_ok=True)
        df = pd.DataFrame(appended, columns=["idx", "attribute", "type", "mean", "stddev", "kurtosis"])
        if existing is not None:
            df = pd.concat([df, existing], ignore_index=True)
        for f in os.listdir(appended_metric_path):
            if f.endswith(".csv"):
                os.remove(os.path.join(appended_metric_path, f))
        df.sort_values("idx", kind="stable").to_csv(os.path.join(appended_metric_path, "part-00000.csv"), index=False)
    odf = ResultFrame(pd.DataFrame(rows, columns=["attribute", "type", "mean_stddev", "mean_cv", "stddev_cv", "kurtosis_cv",
                                                  "mean_si", "stddev_si", "kurtosis_si", "stability_index", "flagged"]))
    if print_impact:
        logger.info("All Attributes:")
        odf.show(len(cols))
        logger.info("Potential Unstable Attributes:")
        odf.where("flagged == 1").show(len(cols))
    return odf
