"""Row-level quality checks without a GPU: the oracle (oracle/row_checks.py) against the notebook tables and the reference unit
tests, and the product's host layer (argument checks, thresholds, result tables, treatments) with the two engine calls
replaced by the NumPy stand-ins below."""
import contextlib
import warnings

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

import cpu_engine
from golden_util import shown_close
from oracle import api as O
from oracle import row_checks as RC

DUP_CELLS = {7: {}, 8: dict(list_of_cols="all", drop_cols=["ifa"]),
             9: dict(list_of_cols=["age", "sex", "race", "workclass", "fnlwgt"]),
             10: dict(list_of_cols=["age", "sex", "race", "workclass", "fnlwgt"], treatment=True)}
NULL_CELLS = {12: {}, 13: dict(list_of_cols="all", drop_cols=["age"], treatment_threshold=0.4),
              14: dict(list_of_cols=["age", "sex", "race", "workclass", "fnlwgt"]),
              15: dict(list_of_cols="all", treatment=True, treatment_threshold=0.75)}


def _check_table(got, cell):
    assert list(got.columns) == cell["columns"]
    assert len(got) == len(cell["rows"])
    for r, exp in zip(got.values.tolist(), cell["rows"]):
        for g, e in zip(r, exp):
            assert shown_close(g, e), (r, exp)


def _unit_tables():
    null_t = O.table_from_rows([("27520a", 51, 9000, "HS-grad"), ("10a", 42, 7000, "Postgrad"), ("11a", 35, None, None),
                                ("1100b", 23, 6000, "HS-grad")], ["ifa", "age", "income", "education"])
    dup_t = O.table_from_rows([("27520a", 51, 9000, "HS-grad"), ("10a", 42, 7000, "Postgrad"), ("10a", 42, 7000, "Postgrad"),
                               ("11a", 35, None, None), ("1100b", 23, 6000, "HS-grad")], ["ifa", "age", "income", "education"])
    return null_t, dup_t


# ---- oracle ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cell", sorted(DUP_CELLS))
def test_oracle_duplicate_detection_notebook(income, nb_quality, cell):
    odf, stats = RC.duplicate_detection(income, print_impact=True, **DUP_CELLS[cell])
    _check_table(stats, nb_quality[cell])
    if cell == 10:
        assert odf.num_rows == 30601


@pytest.mark.parametrize("cell", sorted(NULL_CELLS))
def test_oracle_nullRows_detection_notebook(income, nb_quality, cell):
    odf, stats = RC.nullRows_detection(income, **NULL_CELLS[cell])
    _check_table(stats, nb_quality[cell])
    if cell == 15:
        assert odf.num_rows == income.num_rows     # threshold 0.75 of 20 columns: no row reaches 16 nulls


def test_oracle_reference_unit_tests():
    null_t, dup_t = _unit_tables()
    odf, st = RC.nullRows_detection(null_t, treatment=True, treatment_threshold=0.4)
    st = st.set_index("null_cols_count")
    assert odf.num_rows == 3
    assert (st.loc[0, "row_count"], st.loc[0, "row_pct"], st.loc[0, "treated"]) == (3, 0.75, 0)
    assert (st.loc[2, "row_count"], st.loc[2, "row_pct"], st.loc[2, "treated"]) == (1, 0.25, 1)
    odf, st = RC.duplicate_detection(dup_t, treatment=True, print_impact=True)
    v = dict(st.values.tolist())
    assert odf.num_rows == 4
    assert (v["rows_count"], v["unique_rows_count"], v["duplicate_rows"], v["duplicate_pct"]) == (5, 4, 1, 0.20)


def test_oracle_normalisation():
    nan2 = np.array([0x7ff8000000000000, 0xfff0000000000001], np.uint64).view(np.float64)
    t = pa.table({"x": pa.array(np.array([0.0, -0.0, nan2[0], nan2[1], 5.0, 6.0, 1.0]),
                                mask=np.array([0, 0, 0, 0, 1, 1, 0], bool)),
                  "s": pa.array(["a", "a", "b", "b", None, None, "a"])})
    assert RC.first_occurrence(t, ["x", "s"]).tolist() == [True, False, True, False, True, False, True]
    # a null differs from every value, even from the 0 under its lane
    t = pa.table({"i": pa.array(np.array([0, 0, 7]), mask=np.array([0, 1, 1], bool))})
    assert RC.first_occurrence(t, ["i"]).tolist() == [True, True, False]


# ---- the product's host layer with NumPy stand-ins for the two kernels ------------------------------------------------

def _valid_and_norm(fr, name):
    vals, valid = cpu_engine._values(fr, name)
    if vals.dtype.kind == "f":
        x = vals.astype(np.float64) + 0.0
        bits = np.where(np.isnan(x), np.int64(0x7ff8000000000000), x.view(np.int64))
    else:
        bits = vals.astype(np.int64)
    return np.where(valid, bits, 0), valid


def row_null_counts(fr, names, max_keep=None):
    import torch
    cnt = np.zeros(fr.n_rows, np.int64)
    for n in names:
        cnt += ~cpu_engine._values(fr, n)[1]
    hist = np.bincount(cnt, minlength=len(names) + 1).astype(np.uint64)
    keep = None
    if max_keep is not None:
        from anovos_b200.frame import _pack_validity
        keep = torch.from_numpy(_pack_validity(cnt <= max_keep).copy())
    return hist, keep


def row_distinct(fr, names, hash_bits=0):
    import torch
    from anovos_b200.frame import _pack_validity
    planes = []
    for n in names:
        b, v = _valid_and_norm(fr, n)
        planes += [b, v.astype(np.int64)]
    if fr.n_rows == 0:
        return 0, torch.zeros(1, dtype=torch.int32)
    first = ~pd.DataFrame(np.stack(planes, axis=1) if planes else np.zeros((fr.n_rows, 1))).duplicated().to_numpy()
    return int(first.sum()), torch.from_numpy(_pack_validity(first).copy())


@contextlib.contextmanager
def _stand_ins():
    from anovos_b200 import engine
    saved = engine.row_null_counts, engine.row_distinct
    with cpu_engine.installed():
        engine.row_null_counts, engine.row_distinct = row_null_counts, row_distinct
        try:
            yield
        finally:
            engine.row_null_counts, engine.row_distinct = saved


def _same_table(a, b):
    assert a.column_names == b.column_names and a.num_rows == b.num_rows
    for name in a.column_names:
        x, y = a.column(name).combine_chunks(), b.column(name).combine_chunks()
        assert x.type == y.type and x.is_valid().to_pylist() == y.is_valid().to_pylist(), name
        if pa.types.is_floating(x.type):
            bx, by = x.fill_null(0).to_numpy(), y.fill_null(0).to_numpy()
            assert np.array_equal(bx.view(np.int64 if bx.dtype == np.float64 else np.int32),
                                  by.view(np.int64 if by.dtype == np.float64 else np.int32)), name
        else:
            assert x.to_pylist() == y.to_pylist(), name


def _frames(income):
    null_t, dup_t = _unit_tables()
    rng = np.random.default_rng(5)
    n = 3001
    x = rng.choice(np.array([0.0, -0.0, np.nan, 1.5, -2.0]), n)
    synth = pa.table({"x": pa.array(x, mask=rng.random(n) < 0.2),
                      "i": pa.array(rng.integers(0, 3, n).astype(np.int32), mask=rng.random(n) < 0.1),
                      "s": pa.array(rng.choice(["a", "b", "c"], n)).dictionary_encode()})
    # a dictionary that repeats a string: codes 0 and 2 are the same value
    d = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, 3, n).astype(np.int32)), pa.array(["u", "v", "u"]))
    synth = synth.append_column("d", d)
    return {"income": income, "null_unit": null_t, "dup_unit": dup_t, "synthetic": synth}


@pytest.mark.parametrize("which", ["income", "null_unit", "dup_unit", "synthetic"])
def test_host_layer_equals_oracle(income, which):
    import anovos.data_analyzer.quality_checker as qc
    from anovos_b200.frame import ColumnFrame
    table = _frames(income)[which]
    plain = table.cast(pa.schema([pa.field(f.name, f.type.value_type if pa.types.is_dictionary(f.type) else f.type)
                                  for f in table.schema]))
    fr = ColumnFrame.from_arrow(table)
    with _stand_ins():
        for kw in ({}, dict(treatment=False), dict(drop_cols=[table.column_names[0]])):
            got = qc.duplicate_detection(None, fr, print_impact=True, **kw)
            exp = RC.duplicate_detection(plain, print_impact=True, **kw)
            assert got[1].toPandas().values.tolist() == exp[1].values.tolist(), kw
            if kw.get("treatment", True):
                _same_table(got[0].to_arrow(), exp[0])
        for thr in (0.0, 0.25, 0.4, 0.5, 0.75, 1.0):
            for treat in (False, True):
                got = qc.nullRows_detection(None, fr, treatment=treat, treatment_threshold=thr)
                exp = RC.nullRows_detection(plain, treatment=treat, treatment_threshold=thr)
                pd.testing.assert_frame_equal(got[1].toPandas(), exp[1], check_dtype=False)
                assert got[0].count() == exp[0].num_rows
                if treat:
                    _same_table(got[0].to_arrow(), exp[0])


def test_host_layer_argument_errors_and_warning(income):
    import anovos.data_analyzer.quality_checker as qc
    from anovos_b200.frame import ColumnFrame
    fr = ColumnFrame.from_arrow(income)
    with _stand_ins():
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            assert qc.duplicate_detection(None, fr, treatment=False, print_impact=False) is fr
        assert "Set print_impact=True" in str(w[0].message)
        for f in (qc.duplicate_detection, qc.nullRows_detection):
            with pytest.raises(TypeError, match="Invalid input for Column"):
                f(None, fr, list_of_cols=["no_such_column"])
            with pytest.raises(TypeError, match="Invalid input for Column"):
                f(None, fr, list_of_cols=["age"], drop_cols=["age"])
            with pytest.raises(TypeError, match="Non-Boolean input for treatment"):
                f(None, fr, list_of_cols="age|sex", treatment="maybe")
        for thr in (-0.1, 1.5):
            with pytest.raises(TypeError, match="Invalid input for Treatment Threshold Value"):
                qc.nullRows_detection(None, fr, treatment_threshold=thr)
        dt = ColumnFrame.from_arrow(pa.table({"a": pa.array([1, 2]), "when": pa.array([True, False])}))
        with pytest.raises(TypeError, match="dtypes the GPU path does not hold"):
            qc.duplicate_detection(None, dt, list_of_cols=["a", "when"], print_impact=True)
        # "all" leaves the boolean column out, like attributeType_segregation
        assert qc.duplicate_detection(None, dt, print_impact=True)[1].toPandas()["value"].tolist() == [2.0, 2.0, 0.0, 0.0]


def test_null_rows_max_keep():
    from anovos_b200.data_analyzer.quality_checker import _null_rows_max_keep
    for n in (1, 3, 4, 7, 20):
        for thr in (0.0, 0.1, 0.25, 0.4, 0.5, 0.75, 0.8, 0.99, 1.0):
            flagged = [(k > n * thr) if thr != 1 else (k == n) for k in range(n + 1)]
            assert flagged == [k > _null_rows_max_keep(n, thr) for k in range(n + 1)], (n, thr)
