"""z_standardization, IQR_standardization and normalization without a GPU:
  - the oracle (tests/scaling_oracle.py) against the reference's unit tests and the stored Spark outputs of its
    transformers notebook (tests/golden/notebook_scaling.json);
  - the product's host layer (argument handling, exclusions, models, column order, partitioned frames, impact tables)
    against the oracle, with anv_scale_columns replaced by the oracle's exact image of one kernel column
    (scale_reference) and the other kernels by tests/cpu_engine.py."""
import contextlib
import json
import math
import os
import warnings

import numpy as np
import pyarrow as pa
import pytest

import cpu_engine
import scaling_oracle as SO
from anovos_b200 import engine
from test_imputation_cpu import valid_not_nan

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---- NumPy stand-in of anv_scale_columns ---------------------------------------------------------------------------

def scale_columns(fr, names, specs):
    import torch
    outs, valid, nulls = [], [], []
    for n, sp in zip(names, specs):
        vals, ok = cpu_engine._values(fr, n)
        out, keep = SO.scale_reference(vals, ok, sp)
        outs.append(torch.from_numpy(out))
        nulls.append(int((~keep).sum()))
        if sp[2] & SO.NAN_TO_NULL:
            bits = np.packbits(keep, bitorder="little")
            n_words = (fr.n_rows + 31) // 32
            valid.append(torch.from_numpy(np.concatenate([bits, np.zeros(n_words * 4 - len(bits), np.uint8)]).view(np.int32)))
        else:
            valid.append(None)
    return outs, valid, np.array(nulls, np.int64)


@contextlib.contextmanager
def stand_ins():
    saved = engine.scale_columns, engine.valid_not_nan
    try:
        engine.scale_columns, engine.valid_not_nan = scale_columns, valid_not_nan
        with cpu_engine.installed():
            yield
    finally:
        engine.scale_columns, engine.valid_not_nan = saved


def _fn(name):
    import anovos.data_transformer.transformers as T
    return getattr(T, name)


def product(name, table_or_frame, **kw):
    """The product's function on a host frame (pyarrow tables become frames, Spark-partition tags included)."""
    with stand_ins():
        args = () if name == "normalization" else (None,)
        odf = _fn(name)(*args, table_or_frame, **kw)
        if getattr(odf, "is_partitioned", False):
            return _chunks_to_arrow(odf)
        return odf.to_arrow()


def _chunks_to_arrow(pf):
    return pa.concat_tables([ch.to_arrow() for ch in pf.chunks()])


def oracle(name, table, **kw):
    return getattr(SO, name)(table, **kw)[0]


def same_tables(got, exp):
    assert got.column_names == exp.column_names
    for c in exp.column_names:
        g, e = got.column(c).combine_chunks(), exp.column(c).combine_chunks()
        if pa.types.is_dictionary(g.type):
            g = g.cast(g.type.value_type)
        if pa.types.is_dictionary(e.type):
            e = e.cast(e.type.value_type)
        assert g.type == e.type, (c, g.type, e.type)
        assert np.array_equal(np.asarray(g.is_valid()), np.asarray(e.is_valid())), c
        if pa.types.is_floating(e.type):
            gv = g.fill_null(0).to_numpy(zero_copy_only=False)
            ev = e.fill_null(0).to_numpy(zero_copy_only=False)
            assert np.array_equal(gv.view(np.uint8), ev.view(np.uint8)) or np.array_equal(gv, ev, equal_nan=True), c
        else:
            assert g.to_pylist() == e.to_pylist(), c


def _nb():
    return json.load(open(os.path.join(GOLDEN, "notebook_scaling.json")))


def _after(cell):
    """The "After" describe() table of a notebook cell -> {column: {summary: string}}."""
    t = [x for x in _nb() if x["code_cell"] == cell][1]
    return {c: {r[0]: r[j + 1] for r in t["rows"]} for j, c in enumerate(t["columns"][1:])}


def _stats(table, c):
    x = table.column(c).drop_null().to_numpy(zero_copy_only=False).astype(np.float64)
    return {"count": x.size, "mean": float(np.mean(x)), "stddev": float(np.std(x, ddof=1)), "min": float(x.min()),
            "max": float(x.max())}


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


# ---- the oracle against the reference ------------------------------------------------------------------------------

COLS3 = ["age", "fnlwgt", "hours-per-week"]


def test_oracle_reproduces_reference_unit_tests(income_part1, tmp_path):
    """test_transformers.py:176-310 on part-00001 of the test dataset."""
    mp = str(tmp_path)
    odf = oracle("z_standardization", income_part1, list_of_cols=COLS3, model_path=mp)
    assert odf.num_columns == 17
    assert all(round(_stats(odf, c)["stddev"]) == 1.0 for c in COLS3)
    with pytest.raises(IndexError, match="list index out of range"):
        oracle("z_standardization", income_part1, list_of_cols=["education-num"], pre_existing_model=True, model_path=mp)
    with pytest.warns(UserWarning, match="No Standardization Performed"):
        odf = oracle("z_standardization", income_part1, list_of_cols=[])
    assert all(round(_stats(odf, c)["stddev"]) != 1.0 for c in COLS3)
    assert oracle("z_standardization", income_part1, list_of_cols=COLS3, output_mode="append").num_columns == 20

    odf = oracle("IQR_standardization", income_part1, list_of_cols=COLS3, model_path=mp)
    assert odf.num_columns == 17
    for c in COLS3:
        assert round(float(np.median(odf.column(c).drop_null().to_numpy()))) == 0.0
    with pytest.raises(IndexError, match="list index out of range"):
        oracle("IQR_standardization", income_part1, list_of_cols=["education-num"], pre_existing_model=True, model_path=mp)
    assert oracle("IQR_standardization", income_part1, list_of_cols=COLS3, output_mode="append").num_columns == 20

    odf = oracle("normalization", income_part1, list_of_cols=COLS3, model_path=mp)
    assert odf.num_columns == 17
    assert all(round(_stats(odf, c)["min"]) == 0.0 and round(_stats(odf, c)["max"]) == 1.0 for c in COLS3)
    odf = oracle("normalization", income_part1, list_of_cols=COLS3, pre_existing_model=True, model_path=mp)
    assert all(_stats(odf, c)["min"] == 0.0 and _stats(odf, c)["max"] == 1.0 for c in COLS3)
    with pytest.warns(UserWarning, match="No Normalization Performed"):
        odf = oracle("normalization", income_part1, list_of_cols=[])
    assert all(round(_stats(odf, c)["max"]) != 1.0 for c in COLS3)
    assert oracle("normalization", income_part1, list_of_cols=COLS3, output_mode="append").num_columns == 20


def check_notebook(run, income_spark):
    """run(name, table, **kw) -> output table, against the notebook's "After" tables."""
    # z: cell 30 (Spark's mean / stddev come from another summation order: min / max to 1e-14)
    odf = run("z_standardization", income_spark, list_of_cols=["fnlwgt", "age", "hours-per-week"])
    for c, row in _after(30).items():
        st = _stats(odf, c)
        assert st["count"] == int(row["count"])
        assert _rel(st["min"], float(row["min"])) <= 1e-14 and _rel(st["max"], float(row["max"])) <= 1e-14, c
    # IQR: cell 35, min / max exact (the quartiles are Spark's sketch over its partitions)
    odf = run("IQR_standardization", income_spark, list_of_cols=["fnlwgt", "age", "hours-per-week"])
    for c, row in _after(35).items():
        st = _stats(odf, c)
        assert st["min"] == float(row["min"]) and st["max"] == float(row["max"]), c
        assert _rel(st["mean"], float(row["mean"])) <= 1e-12, c
    # normalization: cells 40 (all columns) and 41, means of the float outputs to 1e-15
    for cell, cols in [(40, "all"), (41, ["fnlwgt", "age", "hours-per-week"])]:
        odf = run("normalization", income_spark, list_of_cols=cols)
        for c, row in _after(cell).items():
            st = _stats(odf, c)
            assert odf.schema.field(c).type == pa.float32()
            assert st["count"] == int(row["count"]) and st["min"] == 0.0 and st["max"] == 1.0
            assert _rel(st["mean"], float(row["mean"])) <= 1e-15, (cell, c, st["mean"], row["mean"])


def test_oracle_reproduces_notebook_tables(income_spark):
    check_notebook(oracle, income_spark)


def test_iqr_notebook_pins(income_spark):
    odf = oracle("IQR_standardization", income_spark, list_of_cols=["hours-per-week", "age"])
    assert _stats(odf, "hours-per-week")["min"] == -7.8 and _stats(odf, "hours-per-week")["max"] == 10.8
    assert _stats(odf, "age")["min"] == -1.0526315789473684


def test_normalization_float32_cast_matches_notebook_and_double_does_not(income_spark):
    row = _after(41)["age"]
    x = income_spark.column("age").drop_null().to_numpy().astype(np.float64)
    d = (x - x.min()) * (1 / (x.max() - x.min()))
    assert float(np.mean(d.astype(np.float32).astype(np.float64))) == pytest.approx(float(row["mean"]), rel=1e-15)
    assert _rel(float(np.mean(d)), float(row["mean"])) > 1e-12


# ---- the product's host layer against the oracle ---------------------------------------------------------------------

def synthetic(seed=3, n=2003):
    rng = np.random.default_rng(seed)
    f32 = rng.normal(3, 2, n).astype(np.float32)
    f32[rng.random(n) < 0.05] = np.nan
    f64 = rng.lognormal(0, 1, n)
    big = rng.integers(-(1 << 62), 1 << 62, n)
    big[:4] = [(1 << 53) + 1, (1 << 63) - 1, -(1 << 63), -(1 << 53) - 1]
    one = np.zeros(n)
    return pa.table({
        "f32": pa.array(f32, mask=rng.random(n) < 0.1),
        "f64": pa.array(f64, mask=rng.random(n) < 0.2),
        "i32": pa.array(rng.integers(-50, 50, n).astype(np.int32), mask=rng.random(n) < 0.3),
        "i64": pa.array(big, mask=rng.random(n) < 0.01),
        "const": pa.array(np.full(n, 7, np.int32)),
        "nulls": pa.array(np.zeros(n), mask=np.ones(n, bool)),
        "one": pa.array(one, mask=np.arange(n) != 5),
        "nan_only": pa.array(np.full(n, np.nan, np.float32), mask=rng.random(n) < 0.5),
        "cat": pa.array(rng.choice(["a", "bb"], n)),
    })


@pytest.mark.parametrize("name", ["z_standardization", "IQR_standardization", "normalization"])
@pytest.mark.parametrize("output_mode", ["replace", "append"])
@pytest.mark.parametrize("cols", ["all", "i64|f32|const", ["nulls", "f64", "one", "f64"]])
def test_host_layer_equals_oracle(name, output_mode, cols):
    t = synthetic()
    kw = dict(list_of_cols=cols, output_mode=output_mode, drop_cols="i32" if cols == "all" else [])
    with warnings.catch_warnings(record=True) as wg:
        warnings.simplefilter("always")
        got = product(name, t, **kw)
    with warnings.catch_warnings(record=True) as we:
        warnings.simplefilter("always")
        exp = oracle(name, t, **kw)
    same_tables(got, exp)
    assert [str(w.message) for w in wg] == [str(w.message) for w in we]


def test_exclusions_and_warnings():
    t = synthetic()
    with pytest.warns(UserWarning, match=r"standard deviation is zero:\['const', 'nulls', 'one'\]"):
        got = product("z_standardization", t, list_of_cols="const|nulls|one|f64", output_mode="append")
    assert got.column_names[-1] == "f64_scaled" and "const_scaled" not in got.column_names
    _, params, excl = SO.z_standardization(t, list_of_cols="f32|nan_only|nulls")
    assert math.isnan(params[0][1]) and "f32" not in excl             # a NaN stddev is not excluded
    with pytest.warns(UserWarning, match=r"percentiles are the same:\['const', 'nulls', 'nan_only'\]"):
        product("IQR_standardization", t, list_of_cols="const|nulls|nan_only|f64")
    got = product("normalization", t, list_of_cols="const|nulls|nan_only|one", output_mode="append")
    assert set(got.column("const_scaled").to_pylist()) == {0.5} and got.column("nulls_scaled").null_count == t.num_rows
    assert got.column("nan_only_scaled").null_count == t.num_rows and got.column("one_scaled").to_pylist()[5] == 0.5


def test_errors():
    t = synthetic()
    for name in ("z_standardization", "IQR_standardization", "normalization"):
        with pytest.raises(TypeError, match="Invalid input for Column"):
            product(name, t, list_of_cols=["cat"])
        with pytest.raises(TypeError, match="output_mode"):
            product(name, t, list_of_cols="f64", output_mode="both")
        with pytest.warns(UserWarning, match="No .* Performed"):
            assert product(name, t, list_of_cols="f64", drop_cols="f64").column_names == t.column_names


def test_models_written_then_read(tmp_path):
    t = synthetic()
    mp = str(tmp_path)
    for name in ("z_standardization", "IQR_standardization", "normalization"):
        product(name, t, list_of_cols="all", model_path=mp)
        same_tables(product(name, t.slice(0, 500), list_of_cols="all", pre_existing_model=True, model_path=mp),
                    oracle(name, t.slice(0, 500), list_of_cols="all", pre_existing_model=True, model_path=mp))
    assert sorted(os.listdir(mp)) == ["IQR_standardization", "normalization", "z_standardization"]
    with pytest.raises(IndexError, match="list index out of range"):
        product("z_standardization", t.append_column("new", t.column("f64")), list_of_cols="new", pre_existing_model=True,
                model_path=mp)
    with pytest.raises(ValueError):
        product("normalization", t, list_of_cols="f64", pre_existing_model=True, model_path=mp)
    lo, hi, mins, maxs = SO.read_minmax_model(mp)
    names = SO._cols(t, "all", [], "replace", "")
    assert mins[names.index("nulls")] == SO.DOUBLE_MAX and maxs[names.index("nulls")] == -SO.DOUBLE_MAX   # recalled


def test_null_and_zero_parameters_give_all_null_columns(tmp_path):
    t = synthetic()
    mp = str(tmp_path)
    SO.write_param_model(mp, "z_standardization", ["f64", "i32", "f32", "i64"],
                         [[1.0, 0.0], [None, 2.0], [1.0, -0.0], [2.0, 3.0]])
    SO.write_param_model(mp, "IQR_standardization", ["f64"], [[1.0, None, 3.0]])
    got = product("z_standardization", t, list_of_cols="f64|i32|f32|i64", pre_existing_model=True, model_path=mp)
    same_tables(got, oracle("z_standardization", t, list_of_cols="f64|i32|f32|i64", pre_existing_model=True, model_path=mp))
    for c in ("f64", "i32", "f32"):
        assert got.column(c).null_count == t.num_rows and got.schema.field(c).type == pa.float64()
    assert got.column("i64").null_count == t.column("i64").null_count
    got = product("IQR_standardization", t, list_of_cols="f64", pre_existing_model=True, model_path=mp)
    assert got.column("f64").null_count == t.num_rows


def test_reads_minmax_model_in_sparks_layout(tmp_path):
    """A MinMaxScalerModel directory as Spark writes it: uuid'd part files, .crc files, _SUCCESS markers, a sparse
    vector, and min / max set in the paramMap."""
    import pyarrow.parquet as pq
    d = tmp_path / "normalization"
    (d / "metadata").mkdir(parents=True)
    (d / "data").mkdir()
    meta = {"class": "org.apache.spark.ml.feature.MinMaxScalerModel", "timestamp": 1, "sparkVersion": "3.2.1",
            "uid": "MinMaxScaler_0123456789ab", "paramMap": {"inputCol": "v", "outputCol": "s", "min": -1.0, "max": 1.0},
            "defaultParamMap": {"min": 0.0, "max": 1.0, "outputCol": "MinMaxScaler_0123456789ab__output"}}
    (d / "metadata" / "part-00000").write_text(json.dumps(meta) + "\n")
    (d / "metadata" / ".part-00000.crc").write_bytes(b"\0\1")
    (d / "metadata" / "_SUCCESS").write_text("")
    vec = pa.struct([pa.field("type", pa.int8(), False), pa.field("size", pa.int32()), pa.field("indices", pa.list_(pa.int32())),
                     pa.field("values", pa.list_(pa.float64()))])
    pq.write_table(pa.table({"originalMin": pa.array([{"type": 0, "size": 3, "indices": [1], "values": [-2.0]}], vec),
                             "originalMax": pa.array([{"type": 1, "size": None, "indices": None, "values": [90.0, 40.0, 5.0]}], vec)}),
                   str(d / "data" / "part-00000-5f1c2b9e-0000-4000-8000-000000000000-c000.snappy.parquet"))
    (d / "data" / "_SUCCESS").write_text("")
    t = synthetic()
    kw = dict(list_of_cols="f64|i32|const", pre_existing_model=True, model_path=str(tmp_path))
    got = product("normalization", t, **kw)
    same_tables(got, oracle("normalization", t, **kw))
    x = t.column("i32").to_pylist()
    g = got.column("i32").to_pylist()
    k = next(i for i, v in enumerate(x) if v is not None)
    assert g[k] == float(np.float32((x[k] + 2.0) * (2.0 / 42.0) - 1.0))


def test_partitioned_frame_equals_resident():
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.partitioned import PartitionedFrame
    t = synthetic(n=5000)
    for name in ("z_standardization", "normalization"):
        for mode in ("replace", "append"):
            res = product(name, t, list_of_cols="all", output_mode=mode)
            with stand_ins():
                pf = PartitionedFrame.from_frame(ColumnFrame.from_arrow(t), 1024)
                args = () if name == "normalization" else (None,)
                odf = _fn(name)(*args, pf, list_of_cols="all", output_mode=mode)
                got = _chunks_to_arrow(odf)
            if name == "z_standardization":           # merged moments: mean / stddev to a few ulps, not bit for bit
                assert got.column_names == res.column_names
                for c in res.column_names:
                    if pa.types.is_floating(res.schema.field(c).type):
                        a = got.column(c).to_numpy(zero_copy_only=False)
                        b = res.column(c).to_numpy(zero_copy_only=False)
                        assert np.allclose(a, b, rtol=1e-12, atol=1e-12, equal_nan=True), c
            else:
                same_tables(got, res)


def test_print_impact_tables(income_spark, capsys):
    """The "Before" / "After" describe() tables of notebook cell 35: counts and min / max as Spark prints them."""
    product("IQR_standardization", income_spark, list_of_cols=["fnlwgt", "hours-per-week", "age"], print_impact=True)
    out = capsys.readouterr().out.splitlines()
    assert out[0].strip() == "Before:" and any(line.strip() == "After:" for line in out)
    after = out[[i for i, line in enumerate(out) if line.strip() == "After:"][0] + 1:]
    rows = {line.split()[0]: line.split()[1:] for line in after[1:]}
    exp = _after(35)
    for j, c in enumerate(["fnlwgt", "hours-per-week", "age"]):
        assert rows["count"][j] == exp[c]["count"]
        assert rows["min"][j] == exp[c]["min"] and rows["max"][j] == exp[c]["max"]
    before = {line.split()[0]: line.split()[1:] for line in out[2:7]}
    assert before["min"] == ["12285", "1", "17"] and before["max"] == ["1484705", "94", "85"]
    product("normalization", income_spark, list_of_cols=["age"], print_impact=True)
    after = capsys.readouterr().out.splitlines()[-5:]
    assert after[-2].split()[1] == "0.0" and after[-1].split()[1] == "1.0"


def test_host_layer_reproduces_notebook(income_spark):
    check_notebook(product, income_spark)
