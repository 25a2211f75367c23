"""The product's HOST layer on CPU: the per-frame cache that the kernels normally fill (moments, order statistics,
mode / distinct, HLL++ estimates, code histograms) is filled from the oracle's numbers instead, and every stats function
of the product must then return exactly what the oracle's function returns - argument normalisation, Spark rounding,
Float.toString display values, Java number strings, null handling and output schemas are all host logic.
No kernel runs (and none could: there is no GPU under `-m "not gpu"`)."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from anovos_b200 import _lib, engine, profile
from anovos_b200.frame import ColumnFrame
from oracle import api as O
from oracle import spark_semantics as S

FUNCS = ["global_summary", "missingCount_computation", "nonzeroCount_computation", "measures_of_counts", "mode_computation",
         "measures_of_centralTendency", "measures_of_cardinality", "measures_of_dispersion", "measures_of_percentiles",
         "measures_of_shape"]


def _fill_cache(fr: ColumnFrame, table: pa.Table):
    """What the kernels would leave in the frame cache, computed by the oracle."""
    mom, q, mode, hll, codes = {}, {}, {}, {}, {}
    for name in fr.columns:
        col = fr.column(name)
        if col.kind == "other":
            continue
        p = O.ColumnProfile(table, name)
        rec = np.zeros(1, dtype=engine._MOM_DT)[0]
        rec["n_valid"] = p.n
        if col.kind == "num":
            rec["n_nonzero"] = p.nonzero()
            if p.n:
                cnt, mean, m2, m3, m4 = S.central_moments(p.x64)
                mn, mx = p.minmax()
                rec["min"], rec["max"], rec["mean"], rec["m2"], rec["m3"], rec["m4"] = mn, mx, mean, m2, m3, m4
            else:
                rec["min"] = rec["max"] = rec["mean"] = np.nan
            for r in range(1, p.n + 1) if p.n <= 64 else set(engine.quantile_ranks(p.n, profile.SUMMARY_PROBS, profile.SUMMARY_EPS)):
                q.setdefault(name, {})[int(r)] = float(p.sorted64[r - 1])
            mv, mr = p.mode()
            exact = col.anv_dtype == _lib.ANV_I64            # the kernels' mode of a bigint column is an exact int
            mode[name] = ((int(mv) if exact else float(mv)), int(mr), p.distinct()) if p.n else (None, None, 0)
        else:
            mv, mr = p.mode()
            mode[name] = (str(mv), int(mr), p.distinct()) if p.n else (None, None, 0)
            h = np.zeros(len(col.dictionary) + 1, np.uint64)
            h[0] = p.N - p.n
            u, k = np.unique(p.nn.astype(str), return_counts=True) if p.n else ([], [])
            pos = {s: i for i, s in enumerate(col.dictionary)}
            for s, c in zip(u, k):
                h[pos[s] + 1] = c
            codes[name] = h
        mom[name] = rec
        hll[name] = S.hll_estimate(S.hll_registers(S.hll_hashes(p.nn, p.sdtype), 9), 9)
    fr._cache.update({"moments": mom, "quantiles": q, "mode": mode, ("hll", 9): hll, "codes": codes})


def _same(got: pd.DataFrame, exp: pd.DataFrame, what):
    assert list(got.columns) == list(exp.columns) and len(got) == len(exp), what
    for c in got.columns:
        for x, y in zip(got[c].tolist(), exp[c].tolist()):
            assert (pd.isna(x) and (y is None or pd.isna(y))) or x == y or str(x) == str(y), (what, c, x, y)


def _tables(income):
    rng = np.random.default_rng(3)
    n = 20_011
    synth = pa.table({
        "f32": pa.array(rng.normal(30, 7, n).astype(np.float32), mask=rng.random(n) < 0.02),
        "f64": pa.array(np.round(rng.lognormal(0, 0.75, n), 3)),
        "i32": pa.array(rng.integers(-5, 90, n).astype(np.int32), mask=rng.random(n) < 0.3),
        "zi": pa.array(np.where(rng.random(n) < 0.7, 0.0, rng.exponential(2.0, n))),
        "all_null": pa.array([None] * n, pa.float64()),
        # epoch-ns timestamps: doubles are 256 apart here; the mode 1.6e18 + 1 is not a double
        "i64_ns": pa.array(np.where(rng.random(n) < 0.05, 1_600_000_000_000_000_001,
                                    1_600_000_000_000_000_000 + rng.integers(0, 1 << 20, n)), mask=rng.random(n) < 0.05),
        "cat": pa.array(rng.choice(["a", "bb", "ccc", "d,e"], n), mask=rng.random(n) < 0.1),
    })
    tiny = O.table_from_rows([("27520a", 51, 9000, "HS-grad"), ("10a", 42, 7000, "Postgrad"), ("11a", 35, None, None),
                              ("1100b", 23, 6000, "HS-grad")], ["ifa", "age", "income", "education"])
    return {"income": income, "synthetic": synth, "tiny": tiny}


@pytest.mark.parametrize("which", ["income", "synthetic", "tiny"])
def test_stats_functions_host_layer_equals_oracle(which, income):
    import anovos.data_analyzer.stats_generator as sg
    table = _tables(income)[which]
    fr = ColumnFrame.from_arrow(table)
    _fill_cache(fr, table)
    for fn in FUNCS:
        _same(getattr(sg, fn)(None, fr).toPandas(), getattr(O, fn)(table), (which, fn))
    # argument forms: pipe-separated strings, drop_cols, explicit lists
    num = [c for c in fr.columns if fr.column(c).kind == "num"]
    if len(num) >= 2:
        _same(sg.measures_of_percentiles(None, fr, list_of_cols="|".join(num[:2])).toPandas(),
              O.measures_of_percentiles(table, list_of_cols=num[:2]), (which, "pipe"))
        _same(sg.measures_of_dispersion(None, fr, drop_cols=[num[0]]).toPandas(),
              O.measures_of_dispersion(table, drop_cols=[num[0]]), (which, "drop"))
    with pytest.raises(TypeError):
        sg.measures_of_counts(None, fr, list_of_cols=["no_such_column"])
