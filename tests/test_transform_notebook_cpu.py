"""feature_transformation and boxcox_transformation against the transformers notebook's stored Spark outputs
(tests/golden/notebook_transform.json, cells 108-112 and 115-116), through the product's host layer on the NumPy
stand-ins of test_transform_cpu: counts, mins and maxes exactly (they pin StrictMath's bits, e.g. log(99999) =
11.512915464920228), means, stddevs and skewness to 1e-12 relative (Spark sums in another order).  Plus the Box-Cox lambda
search's selection loop: the reference's carry-over and UnboundLocalError, and an exact pick."""
import json
import math
import os

import numpy as np
import pyarrow as pa
import pytest

import transform_oracle as TO
from test_transform_cpu import product, stand_ins

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _tables(cell):
    return [t for t in json.load(open(os.path.join(GOLDEN, "notebook_transform.json"))) if t["cell"] == cell]


def _shows(cell):
    return [t for t in _tables(cell) if t["kind"] == "show"]


def _stats(t, c):
    col = t.column(c)
    v = np.asarray(col.drop_null().to_numpy(zero_copy_only=False)).astype(np.float64)
    n = len(v)
    mean = float(np.mean(v))
    m2 = float(np.sum((v - mean) ** 2))
    m3 = float(np.sum((v - mean) ** 3))
    return {"count": n, "mean": mean, "stddev": math.sqrt(m2 / (n - 1)), "min": float(v.min()), "max": float(v.max()),
            "skewness": math.sqrt(n) * m3 / math.sqrt(m2 ** 3)}


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


def check_table(t, table):
    for j, c in enumerate(table["columns"][1:], start=1):
        st = _stats(t, c)
        for row in table["rows"]:
            key, want = row[0], row[j]
            if key == "count":
                assert st["count"] == int(want), c
            elif key in ("min", "max"):
                assert st[key] == float(want), (c, key, st[key], want)
            else:
                assert _rel(st[key], float(want)) <= 1e-12, (c, key, st[key], want)


def _run(fn, table, src_kw):
    return product(fn, table, **src_kw)


def test_feature_transformation_cells(income_spark):
    cols = ["education-num", "capital-gain", "capital-loss", "age"]
    for cell, kw in ((108, dict(list_of_cols=cols, method_type="sqrt")),
                     (109, dict(list_of_cols=cols, method_type="ln", output_mode="append")),
                     (111, dict(list_of_cols="age", method_type="sq")),
                     (112, dict(list_of_cols=cols, method_type="remainderDivByN", N=10))):
        before, after = _shows(cell)
        check_table(income_spark, before)
        check_table(product("feature_transformation", income_spark, **kw), after)
    ln = product("feature_transformation", income_spark, list_of_cols=cols, method_type="ln", output_mode="append")
    before, after = _shows(110)
    check_table(ln, before)
    check_table(product("feature_transformation", ln, list_of_cols=[c + "_ln" for c in cols], method_type="roundN", N=1), after)


def test_boxcox_cell_116_and_skewness_rows(income_spark, capsys):
    before, after = _shows(116)
    odf = product("boxcox_transformation", income_spark, list_of_cols="age", boxcox_lambda=0, output_mode="append",
                  print_impact=True)
    check_table(income_spark, before)
    check_table(odf, after)
    out = capsys.readouterr().out
    skew = [float(line.split()[-1]) for line in out.splitlines() if line.strip().startswith("skewness")]
    assert len(skew) == 2
    assert _rel(skew[0], 0.5127993362812433) <= 1e-12 and _rel(skew[1], -0.14607838263666723) <= 1e-12
    check_table(income_spark, _shows(115)[0])               # cell 115's Before table, skewness row included
    assert [t["lambdas"] for t in _tables(115) if t["kind"] == "lambdas"] == [[0, 3, 1, 3, 1]]


# ---- the lambda search's selection loop ------------------------------------------------------------------------------

def test_lognormal_picks_log():
    rng = np.random.default_rng(3)
    x = rng.lognormal(0, 1, 300)
    t = pa.table({"a": x})
    with stand_ins(), ks_stand_in():
        from anovos_b200.data_transformer import transformers as TB
        from anovos_b200.frame import as_frame
        assert TB.boxcox_search(as_frame(t), ["a"]) == [0]
        odf = TB.boxcox_transformation(t, output_mode="append").to_arrow()
        assert odf.column_names == ["a", "a_bxcx_0"]
    from anovos_b200.shared.ks import p_value
    assert TO.boxcox_lambdas([(x, np.ones(300, bool))], p_value) == [0]


def test_carry_over_and_unbound_local_error(monkeypatch):
    """A column where no p-value beats 0 keeps the previous column's lambda; on the first column that is an error."""
    from anovos_b200 import engine
    from anovos_b200.data_transformer import transformers as T
    n = 2000
    t = pa.table({"a": np.full(n, 2.0), "b": np.full(n, 3.0)})
    good = np.full(15, 1.0)
    good[4] = 0.01                                          # lambda 2 wins on the first column
    hopeless = np.full(15, 1.0)                             # 1 - cdf(1, n) is 0: no candidate beats 0
    seq = {"a": good, "b": hopeless}
    with stand_ins():
        monkeypatch.setattr(engine, "ks_candidates", lambda fr, c, lams, n_null: (seq[c].copy(), 0))
        from anovos_b200.frame import as_frame
        assert T.boxcox_search(as_frame(t), ["a", "b"]) == [2, 2]
        with pytest.raises(UnboundLocalError):
            T.boxcox_search(as_frame(t), ["b", "a"])


import contextlib  # noqa: E402


@contextlib.contextmanager
def ks_stand_in():
    """engine.ks_candidates from the oracle: the statistic over all rows (the zeros' term is then already in it)."""
    from anovos_b200 import engine
    import cpu_engine
    saved = engine.ks_candidates

    def ks(fr, c, lambdas, n_null):
        vals, ok = cpu_engine._values(fr, c)
        return np.array(TO.boxcox_statistics(vals, ok)), int(np.sum(ok & (np.asarray(vals, float) < 1)))
    engine.ks_candidates = ks
    try:
        yield
    finally:
        engine.ks_candidates = saved
