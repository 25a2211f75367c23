"""imputation_MMM and the MMM treatment of nullColumns_detection without a GPU:
  - the oracle (tests/imputation_oracle.py) against the reference's own unit tests and the stored Spark outputs of its
    notebooks (tests/golden/notebook_imputation.json);
  - the product's host layer (argument handling, column order, models, impact tables) against the oracle, with the
    kernels replaced by exact NumPy stand-ins of anv_impute_fill / anv_valid_not_nan (below) and tests/cpu_engine.py;
  - the host conversion of the surrogate (Java's (float) / d2i / d2l)."""
import contextlib
import json
import math
import os

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

import cpu_engine
import imputation_oracle as IO
from anovos_b200 import _lib, engine
from oracle import api as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_NP = {_lib.ANV_F32: np.float32, _lib.ANV_F64: np.float64, _lib.ANV_I32: np.int32, _lib.ANV_I64: np.int64}


# ---- NumPy stand-ins of the two entry points -----------------------------------------------------------------------

def impute_fill(fr, names, out_dtypes, flags, fills):
    import torch
    out = []
    for n, od, fl, fb in zip(names, out_dtypes, flags, fills):
        vals, valid = cpu_engine._values(fr, n)
        raw = np.array([fb], np.uint64)
        fill = (raw.astype(np.uint32).view(_NP[od]) if np.dtype(_NP[od]).itemsize == 4 else raw.view(_NP[od]))[0]
        out.append(torch.from_numpy(IO.fill_reference(vals, valid, _NP[od], bool(fl & _lib.IMPUTE_NAN_MISSING),
                                                      bool(fl & _lib.IMPUTE_ROUND_DOUBLE), fill)))
    return out


def valid_not_nan(fr, names):
    import torch
    n_words = (fr.n_rows + 31) // 32
    words = np.zeros((max(len(names), 1), max(n_words, 1)), np.int32)
    nan = np.zeros(len(names), np.int64)
    for i, n in enumerate(names):
        vals, valid = cpu_engine._values(fr, n)
        isn = np.isnan(vals) if vals.dtype.kind == "f" else np.zeros(len(vals), bool)
        nan[i] = int((valid & isn).sum())
        bits = np.packbits(valid & ~isn, bitorder="little")
        bits = np.concatenate([bits, np.zeros(n_words * 4 - len(bits), np.uint8)])
        words[i, :n_words] = bits.view(np.int32)
    return torch.from_numpy(words[:len(names), :n_words]), nan


@contextlib.contextmanager
def stand_ins():
    saved = engine.impute_fill, engine.valid_not_nan
    try:
        engine.impute_fill, engine.valid_not_nan = impute_fill, valid_not_nan
        with cpu_engine.installed():
            yield
    finally:
        engine.impute_fill, engine.valid_not_nan = saved


# ---- helpers -------------------------------------------------------------------------------------------------------

def _nulls(t, c):
    return t.num_rows - int(np.asarray(t.column(c).is_valid()).sum())


def _nb():
    return json.load(open(os.path.join(GOLDEN, "notebook_imputation.json")))


def _table(nb, notebook, cell, kind="show"):
    for t in nb:
        if t["notebook"] == notebook and t["code_cell"] == cell and t["kind"] == kind:
            return t
    raise KeyError((notebook, cell, kind))


def _as_rows(df):
    return [[str(v) for v in r] for r in df.itertuples(index=False)]


def _same_tables(got: pa.Table, exp: pa.Table, rel=0.0):
    assert got.column_names == exp.column_names
    for c in exp.column_names:
        g, e = got.column(c).combine_chunks(), exp.column(c).combine_chunks()
        if pa.types.is_dictionary(g.type):
            g = g.cast(g.type.value_type)
        assert g.type == e.type, (c, g.type, e.type)
        gv, ev = g.to_pylist(), e.to_pylist()
        for x, y in zip(gv, ev):
            # a mean surrogate matches Spark's avg to rel: small int casts are then exact, a bigint mean near 1e16 is off by ulps
            close = rel and x is not None and y is not None and (isinstance(y, (int, float)) and not isinstance(y, bool))
            if close and not (isinstance(y, float) and math.isnan(x) and math.isnan(y)):
                assert abs(x - y) <= rel * max(abs(y), 1e-300), (c, x, y)
            else:
                assert (x == y) or (x is not None and y is not None and isinstance(y, float) and math.isnan(x) and math.isnan(y)), (c, x, y)


# ---- the oracle against the reference -----------------------------------------------------------------------------

def test_oracle_reproduces_reference_transformer_test(income_part1, tmp_path):
    """test_transformers.py:424-470 on part-00001 of the test dataset."""
    cols = ["age", "fnlwgt", "hours-per-week", "relationship", "race"]
    odf, _ = IO.imputation_MMM(income_part1, list_of_cols=cols, method_type="mode", model_path=str(tmp_path))
    assert odf.num_columns == 17
    for c in cols:
        assert _nulls(odf, c) == 0
    assert _nulls(odf, "logfnl") == 10214 and _nulls(odf, "education") == 258
    # a numeric column under "mode" needs no saved model: the reference's try / except never reaches its assert
    odf, _ = IO.imputation_MMM(income_part1, list_of_cols=["education-num"], method_type="mode", pre_existing_model=True,
                               model_path=str(tmp_path))
    assert _nulls(odf, "education-num") == 0
    odf, _ = IO.imputation_MMM(income_part1, list_of_cols=[], method_type="mode")
    assert [_nulls(odf, c) for c in ["age", "fnlwgt", "hours-per-week", "race", "relationship"]] == [30, 8, 59, 162, 4]
    odf, _ = IO.imputation_MMM(income_part1, list_of_cols=cols, method_type="mean", output_mode="append")
    assert odf.num_columns == 22


def _tiny():
    return O.table_from_rows([("27520a", 51, 8000, "HS-grad"), ("10a", 42, 7000, "HS-grad"), ("10b", 34, 6000, "grad"),
                              ("10c", 29, 9000, "HS-grad"), ("11a", 35, None, None), ("1100b", 23, 9000, "Postgrad")],
                             ["ifa", "age", "income", "education"])


def test_oracle_reproduces_reference_quality_checker_test():
    """test_quality_checker.py:423-460."""
    odf, _ = IO.imputation_MMM(_tiny())
    assert odf.num_rows == 6
    row = odf.column("ifa").to_pylist().index("11a")
    assert odf.column("income")[row].as_py() == 8000 and odf.column("education")[row].as_py() == "HS-grad"


def test_oracle_reproduces_notebook_tables(income_spark):
    nb = _nb()
    # transformers notebook cell 44: imputation_MMM(spark, df, print_impact=True)
    odf, imp = IO.imputation_MMM(income_spark)
    assert _as_rows(imp) == _table(nb, "transformers", 44)["rows"]
    assert set(odf.column("empty").to_pylist()) == {"None"}
    age_null = ~np.asarray(income_spark.column("age").is_valid())
    assert set(np.asarray(odf.column("age").to_pylist())[age_null].tolist()) == {37}        # median, cast back to int
    # cell 45: mean + append
    odf, _ = IO.imputation_MMM(income_spark, list_of_cols="all", method_type="mean", output_mode="append")
    assert odf.num_columns == 36
    for c, v in [("education-num", 10), ("hours-per-week", 40)]:
        nul = ~np.asarray(income_spark.column(c).is_valid())
        assert set(np.asarray(odf.column(c + "_imputed").to_pylist())[nul].tolist()) == {v}
        assert odf.schema.field(c).type == pa.float64() and odf.schema.field(c + "_imputed").type == pa.int32()
    # cell 49: selected columns (pre-saved stats are what the frame gives)
    _, imp = IO.imputation_MMM(income_spark, list_of_cols=["marital-status", "sex", "occupation", "age"])
    assert _as_rows(imp) == _table(nb, "transformers", 49)["rows"]
    # quality checker cells 22 (median) and 23 (mean): the 20-row table without `empty`
    for cell, mt in [(22, "median"), (23, "mean")]:
        _, imp = IO.nullColumns_detection_MMM(income_spark, "all", treatment_configs={"method_type": mt})
        assert _as_rows(imp) == _table(nb, "quality_checker", cell)["rows"]
    _, imp = IO.nullColumns_detection_MMM(income_spark, "all", treatment_configs={"method_type": "mean",
                                                                                  "output_mode": "append"})
    assert _as_rows(imp) == _table(nb, "quality_checker", 25)["rows"]


# ---- Java casts of the surrogate ----------------------------------------------------------------------------------

@pytest.mark.parametrize("x,dt,want", [
    (0.5, _lib.ANV_I32, 0), (-0.5, _lib.ANV_I32, 0), (2.0 ** 31, _lib.ANV_I32, 2 ** 31 - 1), (-2.0 ** 31 - 5, _lib.ANV_I32, -2 ** 31),
    (float("nan"), _lib.ANV_I32, 0), (float("inf"), _lib.ANV_I32, 2 ** 31 - 1), (float("-inf"), _lib.ANV_I32, -2 ** 31),
    (0.5, _lib.ANV_I64, 0), (-0.5, _lib.ANV_I64, 0), (2.0 ** 63, _lib.ANV_I64, 2 ** 63 - 1), (-2.0 ** 63, _lib.ANV_I64, -2 ** 63),
    (float("nan"), _lib.ANV_I64, 0), (float("inf"), _lib.ANV_I64, 2 ** 63 - 1), (float("-inf"), _lib.ANV_I64, -2 ** 63),
    (10.08, _lib.ANV_I32, 10), (-10.9, _lib.ANV_I64, -10), (2.0 ** 31, _lib.ANV_I64, 2 ** 31),
    (0.1, _lib.ANV_F32, float(np.float32(0.1))), (1e300, _lib.ANV_F32, float("inf")), (-0.5, _lib.ANV_F64, -0.5),
])
def test_java_cast_of_surrogate(x, dt, want):
    got = engine.java_cast(x, dt)
    assert got == want and type(got) is type(want)
    oracle_t = {_lib.ANV_I32: "int", _lib.ANV_I64: "bigint", _lib.ANV_F32: "float", _lib.ANV_F64: "double"}[dt]
    assert IO.cast_double(x, oracle_t) == want


def test_java_cast_nan_to_float_stays_nan():
    assert math.isnan(engine.java_cast(float("nan"), _lib.ANV_F32)) and math.isnan(engine.java_cast(float("nan"), _lib.ANV_F64))


# ---- the product's host layer against the oracle -------------------------------------------------------------------

def _synthetic(seed=5, n=3001):
    rng = np.random.default_rng(seed)
    f32 = rng.normal(3, 2, n).astype(np.float32)
    f32[rng.random(n) < 0.05] = np.nan
    f64 = rng.lognormal(0, 1, n)
    f64[rng.random(n) < 0.03] = np.nan
    big = rng.integers(-(1 << 62), 1 << 62, n)
    big[:3] = [(1 << 53) + 1, (1 << 63) - 1, -(1 << 63)]
    return pa.table({
        "f32": pa.array(f32, mask=rng.random(n) < 0.1),
        "f64": pa.array(f64, mask=rng.random(n) < 0.2),
        "i32": pa.array(rng.integers(-50, 50, n).astype(np.int32), mask=rng.random(n) < 0.3),
        "i64": pa.array(big, mask=rng.random(n) < 0.01),
        "full": pa.array(rng.integers(0, 9, n).astype(np.int32)),
        "cat": pa.array(rng.choice(["a", "bb", "ccc"], n), mask=rng.random(n) < 0.15),
        "cat_null": pa.array([None] * n, pa.string()),
    })


def _product(table, **kw):
    import anovos.data_transformer.transformers as T
    from anovos_b200.frame import ColumnFrame
    with stand_ins():
        return T.imputation_MMM(None, ColumnFrame.from_arrow(table), **kw).to_arrow()


@pytest.mark.parametrize("method_type", ["mean", "median", "mode"])
@pytest.mark.parametrize("output_mode", ["replace", "append"])
@pytest.mark.parametrize("cols", ["missing", "all", "i64|cat|f32"])
def test_host_layer_equals_oracle(method_type, output_mode, cols):
    t = _synthetic()
    kw = dict(list_of_cols=cols, method_type=method_type, output_mode=output_mode)
    got = _product(t, **kw)
    exp, _ = IO.imputation_MMM(t, **kw)
    _same_tables(got, exp, rel=1e-12 if method_type == "mean" else 0.0)


def test_print_impact_tables_equal_oracle(capsys):
    from anovos_b200.result import ResultFrame
    t = _synthetic()
    for mode in ("replace", "append"):
        _product(t, list_of_cols="all", method_type="median", output_mode=mode, print_impact=True)
        got = capsys.readouterr().out
        _, imp = IO.imputation_MMM(t, list_of_cols="all", method_type="median", output_mode=mode)
        ResultFrame(imp).show(len(t.column_names))
        assert got == capsys.readouterr().out


def test_model_save_reload_apply(tmp_path):
    t = _synthetic()
    mp = str(tmp_path)
    _product(t, list_of_cols="all", method_type="median", model_path=mp)
    assert sorted(os.listdir(os.path.join(mp, "imputation_MMM"))) == ["cat_imputer", "num_imputer-model"]
    ins, outs, sur = IO.read_num_model(mp)
    assert ins == ["f32", "f64", "i32", "i64", "full"] and outs == [c + "_imputed" for c in ins]
    for c in ins:
        assert sur[c] == IO.surrogate(t, c, "median")
    got = _product(t.slice(0, 1000), list_of_cols="all", method_type="median", pre_existing_model=True, model_path=mp)
    # the oracle reads the product's model: same numbers applied to a different frame
    exp, _ = IO.imputation_MMM(t.slice(0, 1000), list_of_cols="all", method_type="median", pre_existing_model=True,
                               model_path=mp)
    _same_tables(got, exp)


def test_reads_model_directory_in_sparks_layout(tmp_path):
    """A hand-made ImputerModel / CSV directory as Spark writes them: uuid'd part files, .crc files, _SUCCESS markers."""
    import pyarrow.parquet as pq
    d = tmp_path / "imputation_MMM" / "num_imputer-model"
    (d / "metadata").mkdir(parents=True)
    (d / "data").mkdir()
    meta = {"class": "org.apache.spark.ml.feature.ImputerModel", "timestamp": 1, "sparkVersion": "3.2.1",
            "uid": "Imputer_0123456789ab", "paramMap": {"outputCols": ["i32_imputed", "f64_imputed"],
                                                        "inputCols": ["i32", "f64"], "strategy": "mean"},
            "defaultParamMap": {"missingValue": "NaN", "relativeError": 0.001, "strategy": "mean"}}
    (d / "metadata" / "part-00000").write_text(json.dumps(meta) + "\n")
    (d / "metadata" / ".part-00000.crc").write_bytes(b"\0\1")
    (d / "metadata" / "_SUCCESS").write_text("")
    pq.write_table(pa.table({"i32": [-7.9], "f64": [2.5]}),
                   str(d / "data" / "part-00000-5f1c2b9e-0000-4000-8000-000000000000-c000.snappy.parquet"))
    (d / "data" / "_SUCCESS").write_text("")
    c = tmp_path / "imputation_MMM" / "cat_imputer"
    c.mkdir()
    (c / "part-00000-aaaa-c000.csv").write_text("attribute,parameters\ncat,zz\n")
    (c / "_SUCCESS").write_text("")
    t = _synthetic()
    got = _product(t, list_of_cols=["i32", "f64", "cat"], method_type="mean", pre_existing_model=True, model_path=str(tmp_path))
    exp, _ = IO.imputation_MMM(t, list_of_cols=["i32", "f64", "cat"], method_type="mean", pre_existing_model=True,
                               model_path=str(tmp_path))
    _same_tables(got, exp)
    i32_null = ~np.asarray(t.column("i32").is_valid())
    assert set(np.asarray(got.column("i32").to_pylist())[i32_null].tolist()) == {-7}
    assert "zz" in got.column("cat").to_pylist()


def test_errors():
    t = _synthetic()
    with pytest.raises(TypeError, match="Invalid input for Column"):
        _product(t, list_of_cols=["nope"])
    with pytest.raises(TypeError, match="method_type"):
        _product(t, method_type="max")
    with pytest.raises(TypeError, match="output_mode"):
        _product(t, output_mode="both")
    with pytest.raises(TypeError, match="pre_existing_model"):
        _product(t, pre_existing_model="maybe")
    nan_only = pa.table({"x": pa.array([np.nan, None, np.nan], pa.float64())})
    with pytest.raises(ValueError, match="surrogate cannot be computed"):
        _product(nan_only, method_type="mean")
    with pytest.raises(ValueError, match="surrogate cannot be computed"):
        IO.imputation_MMM(nan_only, method_type="mean")


def test_missing_categorical_in_saved_model_raises_index_error(tmp_path):
    t = _synthetic()
    _product(t, list_of_cols=["cat"], method_type="mode", model_path=str(tmp_path))
    with pytest.raises(IndexError, match="list index out of range"):
        _product(t, list_of_cols=["cat", "cat_null"], method_type="mode", pre_existing_model=True, model_path=str(tmp_path))


def test_reference_unit_tests_on_host_layer(income_part1):
    cols = ["age", "fnlwgt", "hours-per-week", "relationship", "race"]
    for kw in [dict(list_of_cols=cols, method_type="mode"), dict(list_of_cols=[], method_type="mode"),
               dict(list_of_cols=cols, method_type="mean", output_mode="append")]:
        _same_tables(_product(income_part1, **kw), IO.imputation_MMM(income_part1, **kw)[0], rel=1e-12)
    _same_tables(_product(_tiny()), IO.imputation_MMM(_tiny())[0])


@pytest.mark.parametrize("mt,mode", [("median", "replace"), ("mean", "replace"), ("mean", "append")])
def test_null_columns_detection_mmm_equals_oracle(mt, mode, capsys):
    import anovos.data_analyzer.quality_checker as qc
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.result import ResultFrame
    t = _synthetic()
    with stand_ins():
        odf, stats = qc.nullColumns_detection(None, ColumnFrame.from_arrow(t), list_of_cols="all", treatment=True,
                                              treatment_method="MMM", treatment_configs={"method_type": mt, "output_mode": mode},
                                              print_impact=True)
        got = odf.to_arrow()
    printed = capsys.readouterr().out
    exp, imp = IO.nullColumns_detection_MMM(t, "all", treatment_configs={"method_type": mt, "output_mode": mode})
    _same_tables(got, exp, rel=1e-12)
    ResultFrame(imp).show(100)
    assert printed == capsys.readouterr().out
    assert "cat_null" not in [r[0] for r in imp.itertuples(index=False)]      # fewer than 2 distinct values: left alone


def test_other_imputation_treatments_stay_unimplemented():
    import anovos.data_analyzer.quality_checker as qc
    from anovos_b200.frame import ColumnFrame
    with stand_ins():
        for m in ("KNN", "regression", "MF", "auto"):
            with pytest.raises(NotImplementedError):
                qc.nullColumns_detection(None, ColumnFrame.from_arrow(_synthetic()), treatment=True, treatment_method=m)
