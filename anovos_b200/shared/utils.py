"""Host helpers mirroring reference shared/utils.py (attributeType_segregation :48-73,
get_dtype :76-90, ends_with :93-110) plus the Spark formatting rules the result frames
need (round HALF_UP, Double.toString)."""
from __future__ import annotations

import math
from decimal import ROUND_HALF_UP, Context, Decimal

from ..frame import as_frame, kind_of

_QUANT = {4: Decimal("0.0001")}
_WIDE = Context(prec=340)


def attributeType_segregation(idf):
    """-> (num_cols, cat_cols, other_cols) by Spark dtype string (shared/utils.py:64-72)."""
    fr = as_frame(idf)
    seg = getattr(fr, "_segregation", None)        # frames are immutable: the split is computed once per frame
    if seg is None:
        out = {"num": [], "cat": [], "other": []}
        for name, sd in fr.dtypes:
            out[kind_of(sd)].append(name)
        seg = (tuple(out["num"]), tuple(out["cat"]), tuple(out["other"]))
        try:
            fr._segregation = seg
        except AttributeError:
            pass
    return list(seg[0]), list(seg[1]), list(seg[2])


def get_dtype(idf, col):
    return [d for n, d in as_frame(idf).dtypes if n == col][0]


def ends_with(string, end_str="/"):
    string = str(string)
    return string if string.endswith(end_str) else string + end_str


def _small_frame(idf):
    """Result-sized frames only (the reference reshapes `summary()` outputs with these helpers)."""
    import pandas as pd
    if hasattr(idf, "toPandas"):
        return idf.toPandas()
    if isinstance(idf, pd.DataFrame):
        return idf
    raise TypeError("flatten_dataframe / transpose_dataframe reshape small result frames (ResultFrame or pandas)")


def flatten_dataframe(idf, fixed_cols):
    """reference shared/utils.py:6-26: every column not in fixed_cols is melted into (key, value) rows - Spark's
    `explode(create_map(...))`: for each input row, one output row per melted column, in column order."""
    from ..result import ResultFrame
    df = _small_frame(idf)
    fixed_cols = list(fixed_cols)
    valid = [c for c in df.columns if c not in fixed_cols]
    out = df.melt(id_vars=fixed_cols, value_vars=valid, var_name="key", value_name="value")
    order = {c: i for i, c in enumerate(valid)}
    out = out.assign(_r=list(range(len(df))) * len(valid), _k=out["key"].map(order)).sort_values(["_r", "_k"])
    return ResultFrame(out.drop(columns=["_r", "_k"]).reset_index(drop=True))


def transpose_dataframe(idf, fixed_col):
    """reference shared/utils.py:29-45: `groupBy("key").pivot(fixed_col).agg(first("value"))` - one row per melted
    column, one output column per distinct value of fixed_col (sorted, like Spark's pivot)."""
    from ..result import ResultFrame
    flat = flatten_dataframe(idf, [fixed_col]).toPandas()
    keys = list(dict.fromkeys(flat["key"].tolist()))
    cols = sorted(flat[fixed_col].dropna().unique().tolist())
    first = flat.groupby(["key", fixed_col], sort=False)["value"].first()
    rows = [[k] + [first.get((k, c)) for c in cols] for k in keys]
    import pandas as pd
    return ResultFrame(pd.DataFrame(rows, columns=["key"] + [str(c) for c in cols]))


def spark_round(x, scale=4):
    """F.round(double, scale): HALF_UP on the shortest decimal repr of the double."""
    if x is None:
        return None
    x = float(x)
    if x != x or x in (math.inf, -math.inf):
        return x
    if scale == 4:
        # fast path: away from a decimal tie every correct rounding agrees with HALF_UP on the repr
        t = x * 10000.0
        if abs(t) < 1e11 and abs((t - math.floor(t)) - 0.5) > 1e-6 + abs(t) * 2e-15:
            return round(x, 4)
    q = _QUANT.get(scale)
    if q is None:
        q = _QUANT[scale] = Decimal(1).scaleb(-scale)
    # Spark's BigDecimal has no digit limit: a variance of a bigint column (~1e37) has more digits than the default
    # 28-digit context can quantize to `scale` places, so the context holds every digit a double can have
    return float(Decimal(repr(x)).quantize(q, rounding=ROUND_HALF_UP, context=_WIDE))


def spark_round_array(x, scale=4):
    """Vectorised spark_round over a float64 array (NaN = null stays NaN): the fast path is exact away from decimal
    ties (rint(x * 10^scale) / 10^scale is then the correctly rounded double of the decimal value); elements near a tie
    go through the decimal slow path one by one."""
    import numpy as np
    x = np.asarray(x, dtype=np.float64)
    if scale != 4:
        return np.array([np.nan if v != v else spark_round(v, scale) for v in x.ravel().tolist()]).reshape(x.shape)
    with np.errstate(invalid="ignore", over="ignore"):
        t = x * 10000.0
        safe = (np.abs(t) < 1e11) & (np.abs((t - np.floor(t)) - 0.5) > 1e-6 + np.abs(t) * 2e-15)
        out = np.where(safe, np.rint(t) / 10000.0, x)
    for i in np.flatnonzero(~safe.ravel() & np.isfinite(x.ravel())):
        out.ravel()[i] = spark_round(float(x.ravel()[i]), 4)
    return out


def jvm_double_str(x: float) -> str:
    """java.lang.Double.toString of x: decimal notation for 1e-3 <= |x| < 1e7, otherwise
    d.dddE[-]n (what `mode` looks like after the reference casts it to string,
    stats_generator.py:405-411)."""
    x = float(x)
    if x != x:
        return "NaN"
    if x in (math.inf, -math.inf):
        return "Infinity" if x > 0 else "-Infinity"
    if x == 0:
        return "-0.0" if math.copysign(1.0, x) < 0 else "0.0"
    if 1e-3 <= abs(x) < 1e7:
        return repr(x)      # Python prints the same shortest digits in plain decimal notation over this range
    sign, digits, exp = Decimal(repr(x)).as_tuple()
    ds = "".join(map(str, digits)).rstrip("0") or "0"
    exp += len(digits) - len(ds) if ds != "0" else 0
    # value = 0.ds * 10**point
    point = len(ds) + exp
    neg = "-" if sign else ""
    if 1e-3 <= abs(x) < 1e7:
        if point <= 0:
            body = "0." + "0" * (-point) + ds
        elif point >= len(ds):
            body = ds + "0" * (point - len(ds)) + ".0"
        else:
            body = ds[:point] + "." + ds[point:]
        return neg + body
    return "%s%s.%sE%d" % (neg, ds[0], ds[1:] or "0", point - 1)
