"""Helpers to compare result frames with the notebook tables in tests/golden/."""
import math


def cell_value(s):
    if s in ("NaN", "None", ""):
        return None
    try:
        return float(s)
    except ValueError:
        return s


def shown_close(got, shown: str, decimals_hint=4):
    """`shown` is a pandas-rendered number (6 significant digits or fixed 4/6 decimals)."""
    exp = cell_value(shown)
    if exp is None:
        return got is None or (isinstance(got, float) and math.isnan(got))
    if isinstance(exp, str):
        return str(got) == exp
    if got is None:
        return False
    got = float(got)
    if "e" in shown.lower():
        return abs(got - exp) <= 1e-6 * abs(exp) + 1e-12
    nd = len(shown.split(".")[1]) if "." in shown else 0
    return abs(got - exp) <= 0.5000001 * 10 ** (-nd) + 1e-12


def frame_by_attr(df):
    return {r["attribute"]: r for r in df.to_dict("records")}


def table_by_attr(t):
    cols = t["columns"]
    return {r[0]: dict(zip(cols, r)) for r in t["rows"]}


def assert_frames_match(got, exp, flip=1.0001e-4, rel=1e-9):
    """Product result frame (pandas) vs the oracle's, cell for cell.  Strings, counts and nulls must be equal.
    Floats are outputs of round(x, 4) of float64 values that agree to ~1e-12: they may differ by ONE rounding step
    (`flip`) when the unrounded value sits on a rounding boundary; `variance` = round(stddev, 4) ** 2 and
    `cov` = round(stddev, 4) / mean propagate a flipped stddev (Appendix C #1), hence their wider bands."""
    assert list(got.columns) == list(exp.columns), (list(got.columns), list(exp.columns))
    assert got["attribute"].tolist() == exp["attribute"].tolist()
    bad = []
    for c in exp.columns:
        if c == "attribute":
            continue
        for a, g, e in zip(exp["attribute"], got[c].tolist(), exp[c].tolist()):
            g_none = g is None or (isinstance(g, float) and math.isnan(g))
            e_none = e is None or (isinstance(e, float) and math.isnan(e))
            if g_none or e_none:
                ok = g_none and e_none
            elif isinstance(e, str) or isinstance(g, str):
                ok = str(g) == str(e)
            elif c.endswith(("count", "rows", "values")):
                ok = float(g) == float(e)
            else:
                band = flip
                if c == "variance":
                    band = flip * (1.0 + 2.0 * abs(float(e)) ** 0.5)
                elif c == "cov":
                    band = flip * (1.0 + abs(float(e)))
                ok = float(g) == float(e) or abs(float(g) - float(e)) <= band + rel * abs(float(e))   # equal infinities too
            if not ok:
                bad.append((a, c, g, e))
    assert not bad, bad[:20]
